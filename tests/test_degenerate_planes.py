"""The per-keypoint plane fit of the scan-matching pass on degenerate neighbourhoods, on the GPU.

The parity suite fits planes to synthetic walls and floors only: well-conditioned scatter matrices.  Here every
neighbourhood is crafted (tests/degenerate_sets.py): exact and tilted planes, discs, poles, edges on both sides of the
closed-form eigensolver's gap cut, near-isotropic sets, rank 1 / rank 0, ulp-sized spreads, coordinates near the key
limit and in the double-width cell 0.  Each pass is compared row by row with the oracle, and both with the same
formulas evaluated at 50 digits from the stored FP32 points, under error bounds that follow the conditioning of the
problem: a failure then points at the kernel, not at an ill-posed row.

Also here: the signed acceptance gate at distance = dmax +- delta, and NaN planarity (the reference throws
std::runtime_error("error")) on every path: uncapped and capped passes, updateIEKF on the device-resident and the
host-driven loop, and the sharded update.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import degenerate_sets as D
from oracle import oracle_py as O

pytestmark = pytest.mark.gpu
BIG = 2 ** 31 - 1
REL = 1e-5
EPS = D.EPS
# (option, value) of every form of the pass: auto (k1_scan + k1_fit), k1_fast, k1_assoc, the split form, exact selection
VARIANTS = [("k1_variant", 0), ("k1_variant", 1), ("k1_variant", 2), ("k1_variant", 3), ("force_exact_selection", 1)]
VARIANT_IDS = ["auto", "fast", "assoc", "split", "exact"]


@pytest.fixture(scope="module")
def L():
    from sr_livo_b200 import lio
    obj = lio.LioOptimization(max_voxels=1 << 12, sweep_capacity=1 << 12)
    yield obj
    obj.close()


def _set_variant(L, opt):
    L.ctx.set_option("k1_variant", 0)
    L.ctx.set_option("force_exact_selection", 0)
    L.ctx.set_option("fast_force_ambiguous_mod", 0)
    if opt is not None:
        L.ctx.set_option(*opt)


@pytest.fixture(scope="module")
def crafted():
    """The crafted map split in two: clusters whose normal is defined, and the ones whose normal is not
    (poles, isotropic sets, rank 1), each with its keypoints and the 50-digit truth of every row."""
    cl = D.build_clusters(seed=0)
    out = {}
    for part, sel in (("defined", [c for c in cl if c.name not in D.UNDEFINED_NORMAL]),
                      ("undefined", [c for c in cl if c.name in D.UNDEFINED_NORMAL])):
        kp, owner = D.keypoints(sel)
        fits = [D.fit_truth(c.pts) for c in sel]
        truth = [D.row_truth(sel[o].pts, kp[i], fits[o]) for i, o in enumerate(owner)]
        out[part] = dict(clusters=sel, kp=kp, owner=owner, truth=truth, map=D.map_arrays(sel))
    return out


def _run(L, part, opt, prm_kw=None):
    from sr_livo_b200 import lio
    prm_kw = dict(max_num_residuals=BIG, **(prm_kw or {}))
    L.voxel_map.upload(*part["map"])
    om = O.OracleMap()
    om.load(*part["map"])
    L.setKeypoints(part["kp"])
    o = om.build_plane_residuals(part["kp"], D.IDENTITY_Q, D.ZERO_T, D.T_LAST, O.r3live_params(**prm_kw), debug=True)
    _set_variant(L, opt)
    try:
        g = L.buildPlaneResiduals(lio.r3live_params(**prm_kw), D.IDENTITY_Q, D.ZERO_T, D.T_LAST, debug=True)
    finally:
        _set_variant(L, None)
    return g, o


def _row_scales(kp, t):
    """Natural magnitude of each checked column of one row (normal, J, offset, distance, weight, a2D): the per-row
    relative comparison is taken against max(|value|, this), so a component that is ~0 is not held to 1e-5 of 0."""
    b = np.linalg.norm(kp)
    w = abs(t.weight) if t.weight == t.weight else 1.0
    return np.concatenate([np.ones(3), np.full(3, w), np.full(3, w * max(b, 1.0)), [np.linalg.norm(t.nearest),
                           np.linalg.norm(kp - t.nearest), 1.0, 1.0]])


def _truth_errors(row, kp, t, closed_form=False):
    """Errors of one plane row against the truth, and their conditioning-aware bounds: (names, errors, bounds).
    closed_form: the device's eigenvalues may come from the trigonometric solution of the cubic, whose acos loses up to
    half the digits where two eigenvalues nearly coincide (discs, edges): its planarity carries 3e-8 more
    (test_closed_form_eig.py holds the host model of it to that against the QR iteration)."""
    nb = D.normal_bound(t.fit)
    ab = D.a2d_bound(t.fit, t.a2D) + (3e-8 if closed_form else 0.0)
    p0 = t.nearest
    e_n = np.abs(row[3:6] - t.normal).max()
    e_d = abs(row[13] - t.distance)
    b_d = nb * np.linalg.norm(kp - p0) * 2 + 64 * EPS * (np.linalg.norm(kp) + np.linalg.norm(p0))
    e_o = abs(row[12] - t.offset)
    b_o = nb * np.linalg.norm(p0) * 2 + 64 * EPS * np.linalg.norm(p0)
    e_a = abs(row[15] - t.a2D)
    # weight = lambda_w a2D^2 + lambda_n exp(...): d weight / d a2D = 2 lambda_w a2D
    b_w = 2 * D.LAMBDA_W * (abs(t.a2D) + ab) * ab + 64 * EPS
    e_w = abs(row[14] - t.weight)
    return (("normal", e_n, nb), ("distance", e_d, b_d), ("offset", e_o, b_o), ("a2D", e_a, ab), ("weight", e_w, b_w))


@pytest.mark.parametrize("opt", VARIANTS, ids=VARIANT_IDS)
def test_plane_fit_on_well_posed_crafted_neighbourhoods(L, crafted, opt):
    """Exact and tilted planes, discs, edges at gap ratios 0.5e-3 .. 2e-3, ulp-sized spreads, the key limit, cell 0,
    random sets.  Status bit-exact; every row within 1e-5 of the oracle's (per row, not scaled by a column maximum);
    GPU and oracle both within the conditioning-aware bounds of the 50-digit truth."""
    part = crafted["defined"]
    g, o = _run(L, part, opt)
    kp, truth = part["kp"], part["truth"]
    assert o.num_fragile == 0                                   # vector_neighbors[0] is unambiguous everywhere
    assert all(D.normal_bound(t.fit) < 1e-7 and t.flip_margin > 1e-3 and abs(t.distance - D.DMAX) > 1e-6 for t in truth)
    want = np.array([t.status for t in truth])
    assert np.array_equal(o.status, want)                       # the oracle agrees with the truth on every gate
    assert np.array_equal(g.status, o.status)
    assert g.num_residuals == o.num_residuals and g.num_full_neighborhoods == o.num_full_neighborhoods == len(kp)
    assert g.success == o.success
    cols = np.r_[3:16]
    worst = {}
    for i, t in enumerate(truth):
        got, ref = g.plane[i, cols], o.plane[i, cols]
        scale = np.maximum(np.abs(ref), _row_scales(kp[i], t))
        bad = np.abs(got - ref) > REL * scale
        assert not bad.any(), (part["clusters"][part["owner"][i]].name, i, cols[bad], got[bad], ref[bad])
        for who, row in (("gpu", g.plane[i]), ("oracle", o.plane[i])):
            for name, err, bound in _truth_errors(row, kp[i], t, closed_form=who == "gpu"):
                assert err <= bound, (who, name, part["clusters"][part["owner"][i]].name, i, err, bound)
                worst[(who, name)] = max(worst.get((who, name), 0.0), err / bound)
        if t.status == 2:   # J against the truth: w n and w (b x n)
            for who, row in (("gpu", g.plane[i]), ("oracle", o.plane[i])):
                ab = D.a2d_bound(t.fit, t.a2D) + (3e-8 if who == "gpu" else 0.0)
                bJ = (D.normal_bound(t.fit) * abs(t.weight) * 2 + 2 * D.LAMBDA_W * ab) * (1 + np.linalg.norm(kp[i])) + 64 * EPS
                assert np.abs(row[6:12] - t.J).max() <= bJ, (who, "J", i)
    print("largest error / bound:", {f"{w}.{n}": f"{v:.2e}" for (w, n), v in sorted(worst.items())})


@pytest.mark.parametrize("opt", VARIANTS, ids=VARIANT_IDS)
def test_plane_fit_where_the_normal_is_undefined(L, crafted, opt):
    """Poles, (near-)isotropic sets and rank-1 sets (19 copies of a point plus one): the smallest eigenvalue is repeated,
    so the normal is any unit vector of its eigenspace and the GPU's choice need not be the oracle's.  What is defined
    is asserted: a2D and the weight against the truth, the normal lies in the eigenspace and is a unit vector, distance
    and offset are consistent with it, and the status wherever every admissible normal gives the same one.  How often
    the GPU's normal and status differ from the oracle's is printed."""
    part = crafted["undefined"]
    g, o = _run(L, part, opt)
    kp, truth = part["kp"], part["truth"]
    assert g.num_full_neighborhoods == o.num_full_neighborhoods == len(kp)
    n_diff = s_diff = 0
    determined = 0
    for i, t in enumerate(truth):
        name = part["clusters"][part["owner"][i]].name
        for who, row, st in (("gpu", g.plane[i], g.status[i]), ("oracle", o.plane[i], o.status[i])):
            ab = D.a2d_bound(t.fit, t.a2D) + (3e-8 if who == "gpu" else 0.0)
            assert abs(row[15] - t.a2D) <= ab, (who, name, i, row[15], t.a2D)
            assert abs(row[14] - t.weight) <= 2 * D.LAMBDA_W * (abs(t.a2D) + ab) * ab + 64 * EPS, (who, name, i)
            n = row[3:6]
            assert abs(np.linalg.norm(n) - 1.0) <= 8 * EPS, (who, name, i)
            lo, mid, hi = t.fit.evals
            # outside the eigenspace: the gap to the other eigenvalues is lambda_max - lambda_mid (poles, rank 1)
            if t.free_dim < 3:
                leak = np.abs(t.fixed_dirs @ n).max()
                assert leak <= D.C_EIG * EPS * hi / (hi - mid) + 64 * EPS, (who, name, i, leak)
            p0 = t.nearest
            assert abs(row[12] + n @ p0) <= 64 * EPS * np.linalg.norm(p0), (who, name, i)
            assert abs(row[13] - (n @ kp[i] + row[12])) <= 64 * EPS * (np.linalg.norm(kp[i]) + np.linalg.norm(p0)), (who, name, i)
            assert st == (2 if row[13] < D.DMAX else 1)
        if t.free_radius < D.DMAX - 1e-6:                       # every admissible normal accepts this keypoint
            determined += 1
            assert g.status[i] == o.status[i] == 2, (name, i)
        n_diff += int(np.abs(g.plane[i, 3:6] - o.plane[i, 3:6]).max() > 1e-6)
        s_diff += int(g.status[i] != o.status[i])
    assert determined >= len(kp) // 3
    print(f"{VARIANT_IDS[VARIANTS.index(opt)]}: undefined normal at {len(kp)} keypoints: GPU normal differs from the oracle's "
          f"at {n_diff}, status at {s_diff} (status determined by the geometry at {determined}, all equal)")


# ---- the signed acceptance gate ------------------------------------------------------------------------------------
DELTAS = [10.0 ** -e for e in range(2, 14)]


def _gate_world(seed=3):
    """Tilted planar clusters and keypoints at signed distance +(dmax +- delta) on the t_last side of the plane (the gate
    decides) and -(dmax +- delta) on the other side (always accepted: the gate is signed), delta = 1e-2 .. 1e-13."""
    rng = np.random.default_rng(seed)
    clusters, kps, gaps = [], [], []
    for c_i, key in enumerate([(8, 8, 4), (12, 8, 4), (8, 12, 4)]):
        lam = (0.0, 0.1, 0.25)
        cl = D.Cluster("tilted_plane", key, D._shaped(rng, lam, D.random_rotation(rng), D._centre(key)), lam=lam)
        fit = D.fit_truth(cl.pts)
        for delta in DELTAS:
            for side in (1, -1):
                for sgn in (1, -1):
                    target = side * (D.DMAX + sgn * delta)
                    u = rng.normal(size=3)
                    t = D.row_truth(cl.pts, fit.centre, fit)
                    u -= (u @ t.normal) * t.normal
                    kp = fit.centre + 0.1 * u / np.linalg.norm(u) + target * t.normal
                    for _ in range(4):                           # the nearest point moves with the keypoint: iterate
                        t = D.row_truth(cl.pts, kp, fit)
                        kp = kp + (target - t.distance) * t.normal
                    t = D.row_truth(cl.pts, kp, fit)
                    cl.kps.append(kp)
                    kps.append(kp)
                    gaps.append((delta, side, t.distance - D.DMAX, t))
        clusters.append(cl)
    return clusters, np.array(kps), gaps


@pytest.mark.parametrize("opt", VARIANTS, ids=VARIANT_IDS)
def test_acceptance_gate_at_dmax_plus_minus_delta(L, opt):
    from sr_livo_b200 import lio
    clusters, kp, gaps = _gate_world()
    keys, counts, xyz = D.map_arrays(clusters)
    L.voxel_map.upload(keys, counts, xyz)
    om = O.OracleMap()
    om.load(keys, counts, xyz)
    L.setKeypoints(kp)
    prm = dict(max_num_residuals=BIG)
    o = om.build_plane_residuals(kp, D.IDENTITY_Q, D.ZERO_T, D.T_LAST, O.r3live_params(**prm), debug=True)
    _set_variant(L, opt)
    try:
        g = L.buildPlaneResiduals(lio.r3live_params(**prm), D.IDENTITY_Q, D.ZERO_T, D.T_LAST, debug=True)
    finally:
        _set_variant(L, None)
    assert o.num_fragile == 0
    flips = 0
    for i, (delta, side, gap, t) in enumerate(gaps):
        assert abs(abs(gap) - delta) <= 1e-14 or side < 0     # the truth puts the keypoint where it was meant to be
        err = max(abs(g.plane[i, 13] - t.distance), abs(o.plane[i, 13] - t.distance))
        if side < 0:
            assert g.status[i] == o.status[i] == 2             # behind the plane: accepted however far (signed gate)
        elif abs(gap) > 2 * err:
            assert g.status[i] == o.status[i] == t.status, (i, delta, gap, err, g.status[i], o.status[i])
        else:
            flips += int(g.status[i] != o.status[i])
    max_err = max(abs(g.plane[i, 13] - t.distance) for i, (_, _, _, t) in enumerate(gaps))
    print(f"{VARIANT_IDS[VARIANTS.index(opt)]}: largest GPU distance error {max_err:.1e}; status differs from the oracle "
          f"at {flips} keypoints within that error of dmax")


def test_distance_exactly_dmax_is_rejected(L):
    """An exact FP32 plane z = 0.5, a keypoint at z = 0.75, max_dist_to_plane_icp = 0.25: the normal is (0, 0, 1) and the
    distance 0.25 exactly, so the keypoint is rejected (src/optimize.cpp:98 is `distance < max_dist_to_plane_icp`).  A
    second keypoint 2^-30 m lower is accepted."""
    from sr_livo_b200 import lio
    rng = np.random.default_rng(5)
    key = (8, 8, 0)
    x = 8.5 + rng.integers(-300, 300, D.K) * 2.0 ** -10
    y = 8.5 + rng.integers(-300, 300, D.K) * 2.0 ** -10
    pts = np.stack([x, y, np.full(D.K, 0.5)], 1).astype(np.float32)
    keys, counts, xyz = D.map_arrays([D.Cluster("zplane", key, pts)])
    kp = np.array([[8.4321, 8.5678, 0.75], [8.4321, 8.5678, 0.75 - 2.0 ** -30]])
    t_last = np.array([8.5, 8.5, 100.0])
    L.voxel_map.upload(keys, counts, xyz)
    om = O.OracleMap()
    om.load(keys, counts, xyz)
    L.setKeypoints(kp)
    prm = dict(max_num_residuals=BIG, max_dist_to_plane_icp=0.25)
    o = om.build_plane_residuals(kp, D.IDENTITY_Q, D.ZERO_T, t_last, O.r3live_params(**prm), debug=True)
    assert list(o.status) == [1, 2] and o.plane[0, 13] == 0.25 and list(o.plane[0, 3:6]) == [0.0, 0.0, 1.0]
    for opt in VARIANTS:
        _set_variant(L, opt)
        try:
            g = L.buildPlaneResiduals(lio.r3live_params(**prm), D.IDENTITY_Q, D.ZERO_T, t_last, debug=True)
        finally:
            _set_variant(L, None)
        assert list(g.status) == [1, 2], (opt, g.status, g.plane[:, 3:6], g.plane[:, 13] - 0.25)
        assert g.num_residuals == 1 and not g.success


# ---- NaN planarity -------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def nan_world():
    clusters, good, n_acc, n_rej = D.nan_world()
    keys, counts, xyz = D.map_arrays(clusters)
    om = O.OracleMap()
    om.load(keys, counts, xyz)
    o = om.build_plane_residuals(good, D.IDENTITY_Q, D.ZERO_T, D.T_LAST, O.r3live_params(max_num_residuals=BIG), debug=True)
    acc = good[o.status == 2]                                  # keypoints the oracle accepts: they decide k*
    assert acc.shape[0] >= 720
    return dict(map=(keys, counts, xyz), om=om, acc=acc, n_acc=n_acc, n_rej=n_rej)


def _raises_reference_error(fn):
    """The reference's `throw std::runtime_error("error")` (src/optimize.cpp:348-350): exactly RuntimeError("error"),
    not a subclass such as SrlError (which would mean the library returned some other status)."""
    try:
        fn()
    except RuntimeError as e:
        assert type(e) is RuntimeError and str(e) == "error", f"{type(e).__name__}: {e}"
        return True
    return False


@pytest.mark.parametrize("power", [2.0, 1.5, 0.0])
def test_nan_planarity_raises_on_every_uncapped_pass(L, nan_world, power):
    from sr_livo_b200 import lio
    L.voxel_map.upload(*nan_world["map"])
    kp = np.concatenate([nan_world["acc"][:150], nan_world["n_acc"][None], nan_world["acc"][150:300]])
    prm = dict(max_num_residuals=BIG, power_planarity=power)
    assert nan_world["om"].build_plane_residuals(kp, D.IDENTITY_Q, D.ZERO_T, D.T_LAST, O.r3live_params(**prm)).nan_planarity
    L.setKeypoints(kp)
    for opt in VARIANTS + [("fast_force_ambiguous_mod", 3)]:
        _set_variant(L, opt)
        try:
            raised = _raises_reference_error(
                lambda: L.buildPlaneResiduals(lio.r3live_params(**prm), D.IDENTITY_Q, D.ZERO_T, D.T_LAST))
        finally:
            _set_variant(L, None)
        assert raised, (opt, power)


def _capped_cases(w):
    """(cap, where, keypoints): the NaN keypoint before, at and after k*, the keypoint at which the reference's loop
    breaks (src/optimize.cpp:107): the cap-th accepted one (cap >= 1), the first with a full neighbourhood (cap <= 0)."""
    acc, n_acc, n_rej = w["acc"], w["n_acc"][None], w["n_rej"][None]
    cat = np.concatenate
    return [
        (600, "before", cat([acc[:10], n_acc, acc[10:700]])),
        (600, "at", cat([acc[:599], n_acc, acc[599:700]])),
        (600, "after", cat([acc[:650], n_acc, acc[650:700]])),
        (1, "before", cat([n_rej, acc[:50]])),
        (1, "at", cat([n_acc, acc[:50]])),
        (1, "after", cat([acc[:1], n_acc, acc[1:50]])),
        (-1, "at", cat([n_acc, acc[:50]])),
        (-1, "after", cat([acc[:1], n_rej, n_acc, acc[1:50]])),
    ]


@pytest.mark.parametrize("variant", [0, 2], ids=["auto", "assoc"])
@pytest.mark.parametrize("power", [2.0, 0.0])
def test_nan_planarity_on_the_capped_pass(L, nan_world, power, variant):
    """max_num_residuals below the sweep size: the keypoints are consumed in order and the pass stops at k*.  The
    reference throws if it reaches a NaN-planarity keypoint (before or at k*) and not otherwise; the oracle's
    nan_planarity is the expected answer.  power_planarity = 0 makes the weight finite (pow(NaN, 0) = 1), so NaN
    planarity must not be inferred from the Jacobian."""
    from sr_livo_b200 import lio
    L.voxel_map.upload(*nan_world["map"])
    for cap, where, kp in _capped_cases(nan_world):
        prm = dict(max_num_residuals=cap, power_planarity=power)
        o = nan_world["om"].build_plane_residuals(kp, D.IDENTITY_Q, D.ZERO_T, D.T_LAST, O.r3live_params(**prm))
        assert o.nan_planarity == (where != "after"), (cap, where)
        L.setKeypoints(kp)
        L.ctx.set_option("k1_variant", variant)
        try:
            res = []
            raised = _raises_reference_error(lambda: res.append(
                L.buildPlaneResiduals(lio.r3live_params(**prm), D.IDENTITY_Q, D.ZERO_T, D.T_LAST)))
        finally:
            L.ctx.set_option("k1_variant", 0)
        assert raised == o.nan_planarity, (cap, where, power)
        if not raised:
            g = res[0]
            assert g.num_residuals == o.num_residuals and g.success == o.success
            assert np.abs(g.HTH - o.HTH).max() <= REL * np.abs(o.HTH).max()
            assert np.abs(g.HTh - o.HTh).max() <= REL * np.abs(o.HTh).max()


def test_nan_planarity_raises_from_update_iekf_on_both_loops(L, nan_world):
    from sr_livo_b200 import lio, synth
    L.voxel_map.upload(*nan_world["map"])
    acc = nan_world["acc"]
    kp = np.concatenate([acc[:200], nan_world["n_acc"][None], acc[200:400]])
    prm = lio.r3live_params(max_num_residuals=BIG)
    try:
        for mode in (1, 0):
            L.ctx.set_option("device_loop", mode)
            L.setKeypoints(kp)
            L.eskf_pro = lio.EskfEstimator(p=D.ZERO_T.copy(), q=D.IDENTITY_Q.copy(), cov=synth.prior_covariance())
            assert _raises_reference_error(lambda: L.updateIEKF(prm, D.T_LAST)), mode
            # and the context is usable afterwards: the same sweep without that keypoint registers like the oracle
            L.setKeypoints(acc[:400])
            L.eskf_pro = lio.EskfEstimator(p=D.ZERO_T.copy(), q=D.IDENTITY_Q.copy(), cov=synth.prior_covariance())
            summ, fq, ft = L.updateIEKF(prm, D.T_LAST)
            ref = nan_world["om"].update_iekf(acc[:400], O.Eskf(p=D.ZERO_T.copy(), q=D.IDENTITY_Q.copy(), cov=synth.prior_covariance()),
                                              D.T_LAST, O.r3live_params(max_num_residuals=BIG))
            assert summ.success == ref["success"] and summ.passes_run == ref["passes"], mode
            assert np.allclose(ft, ref["frame_t"], atol=1e-9) and np.allclose(fq, ref["frame_q"], atol=1e-9)
    finally:
        L.ctx.set_option("device_loop", 1)


def test_doubles_that_round_to_one_fp32_point_through_insert(L):
    """20 distinct doubles that round to the same FP32 point, inserted with min_distance_points = 0: the insert test is
    strict (sq_dist > min_distance^2, src/lioOptimization.cpp:427) and compares against the stored FP32 value, so the
    GPU map must hold exactly what the oracle's holds.  If that is the 20 copies, the voxel is a rank-0 neighbourhood
    and a keypoint next to it makes the pass raise."""
    from sr_livo_b200 import lio
    base = np.array([10.3125, 20.6875, 4.4375])                           # exact in FP32
    pts = base + np.arange(-10, 10)[:, None] * np.array([2.0 ** -40, -(2.0 ** -41), 2.0 ** -42])
    assert len({tuple(p) for p in pts}) == 20 and np.all(pts.astype(np.float32) == base.astype(np.float32))
    L.voxel_map.clear()
    om = O.OracleMap()
    added = L.addPointsToMap(pts, min_distance_points=0.0)
    assert added == om.add_points(pts, min_distance_points=0.0)
    gk, gc, gx = L.voxel_map.download()
    ok, oc, ox = om.snapshot()
    assert np.array_equal(gk, ok) and np.array_equal(gc, oc) and np.array_equal(gx[0, :gc[0]], ox[0, :oc[0]])
    print(f"insert with min_distance_points = 0 stored {int(oc[0])} of 20 doubles that round to one FP32 point")
    if oc[0] == 20:
        kp = (base + [0.05, 0.03, -0.02])[None]
        o = om.build_plane_residuals(kp, D.IDENTITY_Q, D.ZERO_T, D.T_LAST, O.r3live_params(max_num_residuals=BIG))
        assert o.nan_planarity
        L.setKeypoints(kp)
        for opt in VARIANTS:
            _set_variant(L, opt)
            try:
                assert _raises_reference_error(lambda: L.buildPlaneResiduals(lio.r3live_params(max_num_residuals=BIG),
                                                                             D.IDENTITY_Q, D.ZERO_T, D.T_LAST)), opt
            finally:
                _set_variant(L, None)
    L.voxel_map.clear()


_NAN_DIST_WORKER = r"""
import os, sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], "tests"))
import numpy as np, torch.distributed as tdist
import degenerate_sets as D
from sr_livo_b200 import capi, dist, lio, synth
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
tdist.init_process_group("gloo", rank=rank, world_size=world)
clusters, good, n_acc, n_rej = D.nan_world()
L = lio.LioOptimization(max_voxels=1 << 12, sweep_capacity=4096)
L.voxel_map.upload(*D.map_arrays(clusters))
# the NaN keypoint (within dmax of its point: accepted whatever normal the zero scatter matrix yields, so its NaN
# Jacobian reaches the sums) lies in the last rank's shard only
kp = np.concatenate([good[:300], n_acc[None], good[300:400]])
b, e = dist.shard_range(kp.shape[0], rank, world)
assert (b <= 300 < e) == (rank == world - 1)
Dl = dist.DistributedLio(L, rank, world, native=True)
prm = lio.r3live_params(max_num_residuals=2 ** 31 - 1)
for mode in (1, 0):                                       # native device-resident loop, native host-driven loop
    L.ctx.set_option("device_loop", mode)
    Dl.set_keypoints(kp)
    L.eskf_pro = lio.EskfEstimator(p=D.ZERO_T.copy(), q=D.IDENTITY_Q.copy(), cov=synth.prior_covariance())
    try:
        Dl.updateIEKF(prm, D.T_LAST)
        raise SystemExit(f"rank {rank} device_loop {mode}: no exception")
    except RuntimeError as ex:
        if type(ex) is not RuntimeError or str(ex) != "error":
            raise SystemExit(f"rank {rank} device_loop {mode}: {type(ex).__name__}: {ex}")
    tdist.barrier()
Dl.close(); L.close(); tdist.destroy_process_group()
print("rank", rank, "ok")
"""


def test_nan_planarity_in_one_shard_raises_on_every_rank(tmp_path):
    """Sharded update, world 2 over the fused peer-memory exchange: the NaN-planarity keypoint sits in one rank's shard.
    The exchange hands every rank the NaN-planarity count, so both must raise the reference's error, on the native
    device-resident loop and on the native host-driven loop -- not report a timed-out exchange."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = tmp_path / "nan_dist_worker.py"
    script.write_text(_NAN_DIST_WORKER)
    port = 31700 + (os.getpid() % 1000)
    procs = []
    try:
        for r in range(2):
            env = dict(os.environ, RANK=str(r), WORLD_SIZE="2", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
            procs.append(subprocess.Popen([sys.executable, str(script), root], env=env, stdout=subprocess.PIPE,
                                          stderr=subprocess.STDOUT, text=True))
        outs = [p.communicate(timeout=600)[0] for p in procs]
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
                p.wait()
    for p, o in zip(procs, outs):
        assert p.returncode == 0 and " ok" in o, o[-3000:]
