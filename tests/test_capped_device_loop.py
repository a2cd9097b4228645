"""The residual cap (max_num_residuals < n, every shipped parameter file sets 600) on the device-resident updateIEKF loop.

The capped pass consumes keypoints in their own order and stops at k*, the keypoint at which the reference's loop breaks
(src/optimize.cpp:107).  Both loops process a pass as chunks of the same schedule (chunk 0 = [0, max(4096, 2 cap)), each
later one twice as long): the host-driven loop reads k2_cap_reduce's state back after every chunk, the device-resident
loop enqueues every chunk of every pass at once and the chunks after k* leave on the device.  Same boundaries, same
summation order: the device loop must reproduce the host-driven loop (and its pass sums bit for bit)."""
import ctypes as C

import numpy as np
import pytest

import capped_cases as CC
import degenerate_sets as D
import iekf_cases as IC
from oracle import oracle_py as O
from sr_livo_b200 import capi, lio, synth

pytestmark = pytest.mark.gpu
BIG = 2 ** 31 - 1
REL = 1e-5
FAR = CC.FAR   # keypoints moved this far have no neighbourhood: they never count toward the cap


@pytest.fixture(scope="module")
def L():
    obj = lio.LioOptimization(max_voxels=1 << 18, sweep_capacity=1 << 17)
    assert obj.ctx.counter("device_loop_active") == 1
    yield obj
    obj.close()


@pytest.fixture(scope="module")
def nan_world():
    return CC.nan_world()


def _eskf(sw):
    return dict(p=sw.t_init.copy(), q=sw.q_init.copy(), v=np.array([0.3, 0.0, 0.0]), ba=np.array([0.01, -0.02, 0.0]),
                bg=np.zeros(3), g=np.array([0.0, 0.0, 9.81]), cov=synth.prior_covariance())


def _update(L, raw, prm, e0, t_last, mode, variant=0):
    """One updateIEKF on `mode` (1 device-resident loop, 0 host-driven loop); what it returned or raised."""
    L.ctx.set_option("device_loop", mode)
    L.ctx.set_option("k1_variant", variant)
    try:
        L.setKeypoints(raw)
        L.eskf_pro = lio.EskfEstimator(**{k: np.array(v, copy=True) for k, v in e0.items()})
        try:
            summ, fq, ft = L.updateIEKF(prm, t_last)
            out = dict(err=None, summ=summ, fq=fq, ft=ft, e=L.eskf_pro)
        except RuntimeError as ex:   # RuntimeError("error") = NaN planarity (src/optimize.cpp:348); SrlError otherwise
            out = dict(err=ex if type(ex) is RuntimeError and str(ex) == "error" else repr(ex))
        out["chunks"] = L.ctx.counter("cap_chunks_run")
    finally:
        L.ctx.set_option("device_loop", 1)
        L.ctx.set_option("k1_variant", 0)
    return out


def _steps(summ):
    """Trace rows of the passes that ran an ESIKF step: a pass that ends the update with an error (too few residuals)
    has none (the host-driven loop leaves its row zero, the device-resident loop leaves it unwritten)."""
    return summ.passes_run if summ.success else summ.passes_run - 1


def _assert_loops_agree(d, h):
    """The tolerances of test_device_resident_loop_equals_host_driven_loop; discrete outcomes exactly."""
    assert (d["err"] is None) == (h["err"] is None), (d["err"], h["err"])
    assert d["chunks"] == h["chunks"]
    if d["err"] is not None:
        return
    sd, sh = d["summ"], h["summ"]
    assert (sd.success, sd.passes_run, sd.converged, sd.num_residuals_used) == (sh.success, sh.passes_run, sh.converged, sh.num_residuals_used)
    k = _steps(sd)
    assert np.allclose(sd.trace[:k], sh.trace[:k], rtol=1e-7, atol=1e-11)
    for f in ("p", "q", "v", "ba", "bg", "g"):
        assert np.allclose(getattr(d["e"], f), getattr(h["e"], f), rtol=1e-9, atol=1e-11), f
    assert np.allclose(d["e"].cov, h["e"].cov, rtol=1e-6, atol=1e-13)
    assert np.allclose(d["fq"], h["fq"], atol=1e-11) and np.allclose(d["ft"], h["ft"], atol=1e-11)


def _both_loops(L, raw, prm, e0, t_last, variant=0):
    d = _update(L, raw, prm, e0, t_last, 1, variant)
    h = _update(L, raw, prm, e0, t_last, 0, variant)
    _assert_loops_agree(d, h)
    return d, h


def _load(L, world):
    L.voxel_map.upload(*world["omap"].snapshot())
    return world["sweep"]


def _bounds(n, cap):
    b, chunk = [0], max(4096, 2 * max(cap, 1))
    while b[-1] < n:
        b.append(min(n, b[-1] + chunk))
        chunk *= 2
    return b


# ---- 1. device-resident capped loop against the host-driven one ----------------------------------------------------
@pytest.mark.parametrize("variant", [0, 1, 2], ids=["auto", "fast", "assoc"])
@pytest.mark.parametrize("frame", ["steady", "init"])
@pytest.mark.parametrize("cap", [600, 100, 1, -1, "n-1"])
def test_capped_device_loop_equals_host_loop(L, small_world, cap, frame, variant):
    sw = _load(L, small_world)
    raw = sw.raw_xyz
    cap = raw.shape[0] - 1 if cap == "n-1" else cap
    kw = dict(frame_id=5) if frame == "init" else dict()        # init frames: nb = 2, 15 iterations, k1_assoc alone
    prm = lio.r3live_params(max_num_residuals=cap, threshold_translation_norm=0.0, **kw)   # every pass runs
    d, h = _both_loops(L, raw, prm, _eskf(sw), sw.t_last, variant)
    assert d["err"] is None
    if cap <= 1:   # the pass stops at the first accepted / full keypoint: 1 residual < min_number_neighbors (src/optimize.cpp:155)
        assert not d["summ"].success and d["summ"].passes_run == 1 and d["summ"].num_residuals_used <= 1
    else:
        assert d["summ"].success and d["summ"].passes_run == (16 if frame == "init" else 6)
    assert d["chunks"] == d["summ"].passes_run        # 4000 keypoints: one chunk, k* found in it or not


# ---- 2. where k* falls in the chunk schedule (20k-point sweep) ---------------------------------------------------
def _first_accepted(L, raw, sw):
    """Index of the first keypoint with an accepted residual at the initial pose: put first, it is k* of cap -1."""
    L.setKeypoints(raw)
    g = L.buildPlaneResiduals(lio.r3live_params(max_num_residuals=BIG), sw.q_init, sw.t_init, sw.t_last, debug=True)
    return int(np.flatnonzero(g.status == 2)[0])


@pytest.mark.parametrize("cap,m,kstar_chunk", [
    (-1, 0, 0), (-1, 4095, 0), (-1, 4096, 1), (-1, 5000, 1), (-1, 12287, 1), (-1, 12288, 2), (-1, 13000, 2),
    (600, 13000, 2)])
def test_kstar_position_in_the_chunk_schedule(L, cfg1_world, cap, m, kstar_chunk):
    sw = _load(L, cfg1_world)
    real = sw.raw_xyz[_first_accepted(L, sw.raw_xyz, sw):]
    raw = np.concatenate([sw.raw_xyz[np.arange(m) % real.shape[0]] + FAR, real]) if m else real
    d, h = _both_loops(L, raw, lio.r3live_params(max_num_residuals=cap), _eskf(sw), sw.t_last)
    assert d["err"] is None and d["summ"].success == (cap > 1)   # cap -1: one residual, the update stops at pass 0
    assert d["chunks"] == h["chunks"] == d["summ"].passes_run * (kstar_chunk + 1)


def test_kstar_never_found(L, cfg1_world):
    """Fewer accepted keypoints than the cap: every chunk of every pass runs and the last one publishes."""
    sw = _load(L, cfg1_world)
    raw = np.concatenate([sw.raw_xyz[np.arange(30000) % 20000] + FAR, sw.raw_xyz[:3000]])
    cap = 4000
    n_chunks = len(_bounds(raw.shape[0], cap)) - 1
    assert n_chunks == 3
    d, h = _both_loops(L, raw, lio.r3live_params(max_num_residuals=cap), _eskf(sw), sw.t_last)
    assert d["err"] is None and d["summ"].success and d["summ"].num_residuals_used < cap
    assert d["chunks"] == h["chunks"] == d["summ"].passes_run * n_chunks


# ---- 3. pass 0 bit for bit ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("where", ["small_cap600", "chunk2"])
def test_first_pass_sums_equal_the_host_driven_pass_bit_for_bit(L, small_world, cfg1_world, where):
    """One pass (num_iters_icp = 0): the host-driven capped pass's sums, replayed into the unchanged loop kernel, give the
    device capped run's state bit for bit, so the device chunks summed exactly what the host-driven chunks summed."""
    if where == "small_cap600":
        sw = _load(L, small_world)
        raw = sw.raw_xyz
    else:
        sw = _load(L, cfg1_world)
        raw = np.concatenate([sw.raw_xyz[np.arange(13000) % 20000] + FAR, sw.raw_xyz])
    prm = lio.r3live_params(max_num_residuals=600, num_iters_icp=0)
    e0 = _eskf(sw)
    L.setKeypoints(raw)
    g = L.buildPlaneResiduals(prm, e0["q"], e0["p"], sw.t_last)
    assert g.success and g.num_residuals == 600
    n_chunks = 1 if where == "small_cap600" else 3
    assert L.ctx.counter("cap_chunks_run") == n_chunks   # this call's chunks, not added to an earlier update's
    L.buildPlaneResiduals(lio.r3live_params(max_num_residuals=BIG), e0["q"], e0["p"], sw.t_last)
    assert L.ctx.counter("cap_chunks_run") == 0
    blk = np.ascontiguousarray(IC.pack32(g.HTH, g.HTh, n_res=g.num_residuals)[None], np.float64)
    st = capi.eskf_to_c(**e0)
    fq, ft = e0["q"].copy(), e0["p"].copy()
    summ = capi.IekfSummary()
    rc = capi.lib().srl_iekf_replay(L.ctx.h, C.byref(st), capi.ptr(fq), capi.ptr(ft), C.byref(prm), capi.ptr(blk), 1, 0,
                                    C.byref(summ))
    assert rc == capi.SRL_OK and summ.passes_run == 1
    rep = capi.eskf_from_c(st)
    d = _update(L, raw, prm, e0, sw.t_last, 1)
    assert d["err"] is None and d["summ"].passes_run == 1 and d["chunks"] == n_chunks
    for f in ("p", "q", "v", "ba", "bg", "g", "cov"):
        assert np.array_equal(getattr(d["e"], f), rep[f]), f
    assert np.array_equal(d["fq"], fq) and np.array_equal(d["ft"], ft)


# ---- 4. against the oracle ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(max_num_residuals=600), dict(max_num_residuals=-1),
                                dict(max_num_residuals=600, frame_id=5, num_iters_icp=3),
                                dict(max_num_residuals=-1, frame_id=5, num_iters_icp=3)])
def test_capped_device_loop_matches_oracle(L, small_world, kw):
    om = small_world["omap"]
    sw = _load(L, small_world)
    n = 1500 if kw.get("frame_id") == 5 else sw.raw_xyz.shape[0]
    raw = sw.raw_xyz[:n]
    e0 = _eskf(sw)
    d = _update(L, raw, lio.r3live_params(**kw), e0, sw.t_last, 1)
    assert d["err"] is None and d["chunks"] == d["summ"].passes_run
    ref = om.update_iekf(raw, O.Eskf(**{k: v.copy() for k, v in e0.items()}), sw.t_last, O.r3live_params(**kw))
    summ, e = d["summ"], d["e"]
    assert summ.success == ref["success"] and summ.passes_run == ref["passes"]
    assert summ.num_residuals_used == ref["num_residuals_used"]
    k = _steps(summ)
    assert np.allclose(summ.trace[:k], ref["trace"][:k], rtol=REL, atol=1e-9)
    for f in ("p", "q", "v", "ba", "bg", "g"):
        assert np.allclose(getattr(e, f), getattr(ref["eskf"], f), rtol=REL, atol=1e-9), f
    assert np.allclose(e.cov, ref["eskf"].cov, rtol=1e-4, atol=1e-12)
    assert np.allclose(d["fq"], ref["frame_q"], atol=1e-9) and np.allclose(d["ft"], ref["frame_t"], atol=1e-9)


# ---- 5. NaN planarity and too few residuals ----------------------------------------------------------------------
@pytest.mark.parametrize("m,kstar_chunk", [(0, 0), (5000, 1), (13000, 2)])
def test_nan_planarity_before_at_and_after_kstar_on_both_loops(L, nan_world, m, kstar_chunk):
    """m keypoints without a neighbourhood in front: k* and the NaN keypoint in chunk 0, 1 or 2, so chunks before k*'s
    chunk are continued from and the ones after it are skipped."""
    L.voxel_map.upload(*nan_world["map"])
    e0 = dict(p=D.ZERO_T.copy(), q=D.IDENTITY_Q.copy(), v=np.zeros(3), ba=np.zeros(3), bg=np.zeros(3),
              g=np.array([0.0, 0.0, 9.81]), cov=synth.prior_covariance())
    for cap, where, kp in CC.capped_nan_cases(nan_world, m):
        for variant in (0, 2):
            # one pass: the NaN keypoint's place relative to k* is the one the cases were built for
            d, h = _both_loops(L, kp, lio.r3live_params(max_num_residuals=cap, num_iters_icp=0), e0, D.T_LAST, variant)
            assert (d["err"] is not None) == (where != "after"), (cap, where, variant, d["err"])
            assert d["err"] is None or isinstance(d["err"], RuntimeError), d["err"]
            assert d["chunks"] == kstar_chunk + 1, (cap, where, variant, d["chunks"])   # one pass, k* found in that chunk
            _both_loops(L, kp, lio.r3live_params(max_num_residuals=cap), e0, D.T_LAST, variant)   # every pass: the loops agree


def test_too_few_residuals_on_both_loops(L, small_world):
    """A gate that rejects every keypoint (no voxel holds more than 20 points): pass 0 ends the update with
    success = false, on both loops."""
    sw = _load(L, small_world)
    d, h = _both_loops(L, sw.raw_xyz, lio.r3live_params(max_num_residuals=600, threshold_voxel_occupancy=21), _eskf(sw), sw.t_last)
    assert d["err"] is None and not d["summ"].success and d["summ"].passes_run == 1 and d["summ"].num_residuals_used == 0
    assert d["chunks"] == 1                            # 4000 keypoints, never 600 accepted: the one chunk publishes


# ---- 6. back-to-back updates on one context ----------------------------------------------------------------------
def test_back_to_back_updates_equal_fresh_contexts(L, small_world, cfg1_world):
    """Stale status, stale k2 state and stale publications: a sequence of updates on one context (including one that
    ends early with chunks still enqueued and one that fails) gives what a fresh context gives for each of them."""
    sw1, sw2 = small_world["sweep"], cfg1_world["sweep"]
    far = np.concatenate([sw2.raw_xyz[np.arange(13000) % 20000] + FAR, sw2.raw_xyz])
    steps = [
        (small_world, sw1.raw_xyz, lio.r3live_params()),                                   # capped, converges early
        (small_world, sw1.raw_xyz, lio.r3live_params(max_num_residuals=BIG)),              # uncapped
        (cfg1_world, far, lio.r3live_params()),                                            # capped, k* in chunk 2
        (small_world, sw1.raw_xyz, lio.r3live_params(threshold_voxel_occupancy=21)),       # capped, too few residuals
        (small_world, sw1.raw_xyz[::-1].copy(), lio.r3live_params(max_num_residuals=100)),  # capped, must succeed
    ]
    expect_ok = [True, True, True, False, True]
    for i, (world, raw, prm) in enumerate(steps):
        sw = _load(L, world)
        a = _update(L, raw, prm, _eskf(sw), sw.t_last, 1)
        F = lio.LioOptimization(max_voxels=1 << 18, sweep_capacity=1 << 17)
        try:
            _load(F, world)
            b = _update(F, raw, prm, _eskf(sw), sw.t_last, 1)
        finally:
            F.close()
        assert a["err"] is None and b["err"] is None, i
        assert a["chunks"] == b["chunks"], i
        sa, sb = a["summ"], b["summ"]
        assert sa.success == sb.success == expect_ok[i], i
        assert (sa.passes_run, sa.converged, sa.num_residuals_used) == (sb.passes_run, sb.converged, sb.num_residuals_used), i
        assert np.array_equal(sa.trace[:_steps(sa)], sb.trace[:_steps(sb)]), i
        for f in ("p", "q", "v", "ba", "bg", "g", "cov"):
            assert np.array_equal(getattr(a["e"], f), getattr(b["e"], f)), (i, f)
        print(f"step {i}: {sa.passes_run} passes, converged {sa.converged}, {a['chunks']} chunks")


# ---- 7. the public interface -------------------------------------------------------------------------------------
def test_optimize_with_the_shipped_parameters_runs_on_the_device_loop(L, small_world):
    om = small_world["omap"]
    sw = _load(L, small_world)
    keep = L.gridSampling(sw.raw_xyz, 0.5)
    raw = sw.raw_xyz[keep]
    prm = lio.r3live_params()
    assert prm.max_num_residuals == 600 and prm.max_num_residuals < raw.shape[0]
    e0 = _eskf(sw)
    L.eskf_pro = lio.EskfEstimator(**{k: v.copy() for k, v in e0.items()})
    summ, fq, ft, world = L.optimize(raw, prm, sw.t_last)
    assert L.ctx.counter("device_loop_active") == 1 and L.ctx.counter("cap_chunks_run") == summ.passes_run > 0
    ref = om.update_iekf(raw, O.Eskf(**{k: v.copy() for k, v in e0.items()}), sw.t_last, O.r3live_params())
    assert summ.success == ref["success"] and summ.passes_run == ref["passes"]
    assert summ.num_residuals_used == ref["num_residuals_used"]
    for f in ("p", "q", "v", "ba", "bg", "g"):
        assert np.allclose(getattr(L.eskf_pro, f), getattr(ref["eskf"], f), rtol=REL, atol=1e-9), f
    assert np.allclose(fq, ref["frame_q"], atol=1e-9) and np.allclose(ft, ref["frame_t"], atol=1e-9)
    # src/optimize.cpp:441-445: the frame re-transformed with the final pose (un-normalised rotation, src/utility.cpp:317)
    assert np.allclose(world, raw @ O.quat_to_rot(fq).T + ft, rtol=0, atol=1e-9)
    assert np.allclose(world, raw @ O.quat_to_rot(ref["frame_q"]).T + ref["frame_t"], rtol=0, atol=1e-6)
