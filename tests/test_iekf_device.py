"""The device-resident ESIKF loop (k_iekf_loop, the Woodbury form) on the seeded cases of tests/iekf_cases.py, through
srl_iekf_replay: the unchanged loop kernel, with a one-warp feeder per pass handing it the given sums.  Compared with the
50-digit truth (tests/iekf_reference.py) under the bounds of the Woodbury form (see test_iekf_algebra.py), and with the
host loop on the same sums for every discrete outcome whose margin exceeds both implementations' bounds."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import iekf_cases as IC
from sr_livo_b200 import capi, lio, synth
from test_iekf_algebra import MULTI, SINGLE, bounds, check_step, fragile, ref_step, state_err

pytestmark = pytest.mark.gpu
BIG = 2 ** 31 - 1


@pytest.fixture(scope="module")
def ctx():
    c = lio.Context(0)
    assert c.counter("device_loop_active") == 1
    yield c
    c.close()


def replay(ctx, case, delay=0, blocks=None):
    prm = IC.icp_params(**case.prm)
    st = capi.eskf_to_c(**case.state)
    fq, ft = np.array(case.state["q"], np.float64), np.array(case.state["p"], np.float64)
    summ = capi.IekfSummary()
    blk = np.ascontiguousarray(case.blocks if blocks is None else blocks, np.float64)
    rc = capi.lib().srl_iekf_replay(ctx.h, C.byref(st), capi.ptr(fq), capi.ptr(ft), C.byref(prm), capi.ptr(blk), blk.shape[0],
                                    int(delay), C.byref(summ))
    return dict(rc=rc, state=capi.eskf_from_c(st), frame_q=fq, frame_t=ft, passes=summ.passes_run, converged=summ.converged,
                trace=capi.summary_trace(summ), raw=np.frombuffer(st, np.float64).copy())


@pytest.mark.parametrize("case", SINGLE, ids=[c.name for c in SINGLE])
def test_device_step_against_the_truth(ctx, case):
    h = IC.host_loop(case)
    d = replay(ctx, case)
    prm = IC.icp_params(**case.prm)
    truth = ref_step(h["inputs"][0], prm)
    assert d["rc"] == h["status"] == capi.SRL_OK and d["passes"] == 1
    bd, _ = check_step(truth, d["trace"][0][:17], d["state"], d["state"]["cov"], "device", case.name)
    if not (fragile(truth, bd) or fragile(truth, bounds(truth, "host"))):
        assert d["converged"] == h["converged"] == int(truth.converged)
        assert np.array_equal(d["frame_t"], case.state["p"]) == truth.diverged


def _sequence_bound(h, prm, p):
    """First-order accumulation over the passes so far: the sum of both forms' per-step bounds."""
    tot = 0.0
    for inp in h["inputs"][:p + 1]:
        t = ref_step(inp, prm)
        tot += bounds(t, "device")["dx"] + bounds(t, "host")["dx"]
    return tot


@pytest.mark.parametrize("case", MULTI, ids=[c.name for c in MULTI])
def test_device_multi_pass_against_the_host_loop_and_the_truth(ctx, case):
    h = IC.host_loop(case)
    d = replay(ctx, case)
    prm = IC.icp_params(**case.prm)
    truths = [ref_step(inp, prm) for inp in h["inputs"]]
    robust = not any(fragile(t, bounds(t, "device")) or fragile(t, bounds(t, "host")) for t in truths)
    if robust:
        assert (d["rc"], d["passes"], d["converged"]) == (h["status"], h["passes"], h["converged"])
    for p in range(min(d["passes"], h["passes"])):
        b = _sequence_bound(h, prm, p)
        e = np.linalg.norm(d["trace"][p][:17] - h["trace"][p][:17])
        assert e <= b + 1e-15, f"{case.name} pass {p}: |d_x device - host| = {e:.3e} > {b:.3e}"
        # the truth of this step, evaluated on the host's input, is within the host's bound of the host's d_x (checked on the
        # CPU); the device's d_x is within the accumulated bound of both
        e_t = np.linalg.norm(d["trace"][p][:17] - truths[p].d_x)
        assert e_t <= b + 1e-15, f"{case.name} pass {p}: |d_x device - truth| = {e_t:.3e} > {b:.3e}"
    b = _sequence_bound(h, prm, h["passes"] - 1)
    assert state_err(d["state"], h["state"]) <= 2 * b + 1e-14
    tl = truths[-1]
    if tl.final:
        bc = bounds(tl, "device")["cov"] + bounds(tl, "host")["cov"]
        assert np.linalg.norm(d["state"]["cov"] - h["state"]["cov"], 2) <= bc * max(1, h["passes"]) + 1e-14


def test_warm_up_step_leaves_no_state_behind(ctx):
    """The loop's warm-up ("dry") step runs before pass 0 when pass 0's sums arrive late and is skipped when they are
    already there: the result is bitwise identical either way."""
    for case in (MULTI[-2], SINGLE[20], [c for c in SINGLE if c.name.startswith("pivot")][0]):
        runs = [replay(ctx, case, delay) for delay in (-1, 0, 20_000_000, -1, 20_000_000)]
        for r in runs[1:]:
            assert r["rc"] == runs[0]["rc"] and r["passes"] == runs[0]["passes"]
            assert np.array_equal(r["raw"], runs[0]["raw"]), case.name
            assert np.array_equal(r["trace"], runs[0]["trace"]), case.name


def test_statuses_at_a_chosen_pass(ctx):
    """[28] (residual count) and [31] (NaN-planarity count) of a chosen pass end both loops there with the same status."""
    case = [c for c in MULTI if c.prm.get("threshold_translation_norm") == 0.0][0]
    for p, col, val, want in ((2, 28, 5.0, capi.SRL_TOO_FEW_RESIDUALS), (1, 31, 1.0, capi.SRL_NAN_PLANARITY),
                              (0, 28, 19.0, capi.SRL_TOO_FEW_RESIDUALS), (3, 31, 3.0, capi.SRL_NAN_PLANARITY)):
        blocks = case.blocks.copy()
        blocks[p, col] = val
        c2 = IC.Case(case.name, case.state, blocks, case.prm)
        h = IC.host_loop(c2)
        d = replay(ctx, c2)
        assert d["rc"] == h["status"] == want
        assert d["passes"] == h["passes"] == p + 1
        if p:
            assert np.linalg.norm(d["trace"][p - 1][:17] - h["trace"][p - 1][:17]) <= _sequence_bound(h, IC.icp_params(**case.prm), p - 1) + 1e-15


def test_replay_rejects_fewer_blocks_than_passes(ctx):
    case = [c for c in MULTI if c.prm.get("num_iters_icp") == 3][0]
    d = replay(ctx, case, blocks=case.blocks[:3])
    assert d["rc"] == capi.SRL_BAD_ARG


def test_singular_covariance_on_the_device(ctx):
    """Exactly singular P (zero gravity block): the device never inverts P and returns the finite update, which is the
    limit of the reference's formula (the gravity block stays exactly zero); the host loop reports SRL_SINGULAR."""
    rng = np.random.default_rng(5)
    P = IC.singular_gravity()
    H = IC.normal_eq("rank6", rng, 1e2)
    case = IC.Case("singular", IC.base_state(rng, P), np.array([IC.pack32(H, H @ rng.normal(size=6) * 1e-3)]))
    assert IC.host_loop(case)["status"] == capi.SRL_SINGULAR
    d = replay(ctx, case)
    assert d["rc"] == capi.SRL_OK and d["passes"] == 1
    assert np.isfinite(d["raw"]).all()
    assert not d["state"]["cov"][15:17, :].any() and not d["state"]["cov"][:, 15:17].any()
    ne = IC.unpack32(case.blocks[0])
    T6 = IC.gain_T6(P, np.array(ne.HTH).reshape(6, 6))
    dx = -T6 @ np.array(ne.HTh)
    assert np.allclose(d["trace"][0][:17], dx, rtol=1e-9, atol=1e-15)


def test_replay_is_faithful_to_the_real_device_loop(small_world):
    """Drive the host loop on small_world with GPU passes, recording every pass's sums; replay them; the real device run
    (srl_update_iekf) and the replay agree: same passes, state to 1e-9."""
    sw = small_world["sweep"]
    prm = capi.r3live_params(max_num_residuals=BIG)
    L = lio.LioOptimization(max_voxels=1 << 18, sweep_capacity=8192)
    try:
        L.addPointsToMap(small_world["pts"])
        L.setKeypoints(sw.raw_xyz)
        P = synth.prior_covariance()
        st = capi.eskf_to_c(p=sw.t_init, q=sw.q_init, v=np.zeros(3), ba=np.zeros(3), bg=np.zeros(3), g=np.array([0.0, 0.0, 9.81]), cov=P)
        it = capi.IekfIter()
        assert capi.lib().srl_iekf_begin(C.byref(st), C.byref(prm), C.byref(it)) == 0
        fq, ft = sw.q_init.copy(), sw.t_init.copy()
        blocks = []
        while True:
            r = L.buildPlaneResiduals(prm, fq, ft, sw.t_last)
            blocks.append(IC.pack32(r.HTH, r.HTh, r.num_residuals))
            ne = IC.unpack32(blocks[-1])
            dx, done, div = np.zeros(17), C.c_int32(0), C.c_int32(0)
            assert capi.lib().srl_iekf_step(C.byref(it), C.byref(ne), C.byref(prm), C.byref(st), capi.ptr(fq), capi.ptr(ft),
                                            capi.ptr(dx), C.byref(done), C.byref(div)) == 0
            if done.value:
                break
        host_state, host_passes = capi.eskf_from_c(st), len(blocks)
        n_pass = int(it.max_num_iter) + 1
        blocks += [blocks[-1]] * (n_pass - len(blocks))
        start = dict(p=sw.t_init, q=sw.q_init, v=np.zeros(3), ba=np.zeros(3), bg=np.zeros(3), g=np.array([0.0, 0.0, 9.81]), cov=P)
        case = IC.Case("small_world", start, np.array(blocks), dict(num_iters_icp=prm.num_iters_icp, threshold_translation_norm=prm.threshold_translation_norm,
                                                                    threshold_orientation_norm=prm.threshold_orientation_norm, laser_point_cov=prm.laser_point_cov))
        rp = replay(L.ctx, case)
        L.eskf_pro = lio.EskfEstimator(p=sw.t_init.copy(), q=sw.q_init.copy(), cov=P.copy())
        summ, dq, dt = L.updateIEKF(prm, sw.t_last)
        assert rp["rc"] == capi.SRL_OK
        assert rp["passes"] == summ.passes_run == host_passes
        for f in ("p", "q", "v", "ba", "bg", "g"):
            assert np.allclose(rp["state"][f], getattr(L.eskf_pro, f), rtol=0, atol=1e-9), f
            assert np.allclose(rp["state"][f], host_state[f], rtol=0, atol=1e-9), f
        assert np.allclose(rp["state"]["cov"], L.eskf_pro.cov, rtol=1e-6, atol=1e-12)
    finally:
        L.close()
