"""Every form of the scan-matching pass on crafted near ties (tests/selection_sets.py), on the GPU, against the oracle.

The association is bit-exact: status, the transformed keypoint, the 20 neighbour ids in order and the bits of their
distances must equal the oracle's; the plane columns agree to 1e-5 (the device's closed-form eigensolver).  Each family
batch runs with debug output and without it: they are different k1_fit instances, and only the one without debug output
is the product, whose sums (HTH, HTh, loss_sum, num_residuals) are compared.  Every decided pair in the sets moves the
sums of its batch by far more than the tolerance of that comparison (`test_every_decided_pair_moves_the_sums`, CPU side).

The counters are held to the CPU model of the FP32 selection (tests/test_selection_model.py): per family and form, the
number of keypoints k1_scan / k1_fast flag lies within what the model predicts over the plausible FP32 evaluation orders.
"""
import collections

import numpy as np
import pytest

import selection_sets as S
from oracle import oracle_py as O

pytestmark = pytest.mark.gpu
BIG = 2 ** 31 - 1
REL = 1e-5
SUM_REL = 1e-6
DEFAULT_LANES = dict(split_lanes_per_keypoint=4, fast_lanes_per_keypoint=1)
PARAM_SETS = {"steady": {}, "init_frame": dict(frame_id=5), "K10": dict(max_number_neighbors=10, min_number_neighbors=10),
              "min5": dict(min_number_neighbors=5), "nb0": dict(voxel_neighborhood=0)}
TABLE = collections.defaultdict(lambda: collections.Counter())


@pytest.fixture(scope="module")
def lios():
    from sr_livo_b200 import lio
    out = {s: lio.LioOptimization(max_voxels=1 << 13, sweep_capacity=1 << 12, size_voxel_map=s) for s in S.SIZES}
    yield out
    for L in out.values():
        for k, v in DEFAULT_LANES.items():
            L.ctx.set_option(k, v)
        L.close()


@pytest.fixture(scope="module")
def batches():
    out = {}
    for fam in S.FAMILIES:
        for size in S.SIZES:
            b = S.build_batch(fam, size)
            out[(fam, size)] = (b, [S.measure(b, k) for k in range(len(b.hoods))])
    return out


def _options(L, form):
    L.ctx.set_option("k1_variant", 0)
    L.ctx.set_option("force_exact_selection", 0)
    L.ctx.set_option("fast_force_ambiguous_mod", 0)
    for k, v in DEFAULT_LANES.items():
        L.ctx.set_option(k, v)
    for k, v in (S.FORMS[form] if form else {}).items():
        L.ctx.set_option(k, v)


def _pass(L, b, form, prm_kw, debug):
    from sr_livo_b200 import lio
    L.voxel_map.upload(*b.map)
    L.setKeypoints(b.kp)
    _options(L, form)
    try:
        a0, e0 = L.ctx.counter("fast_ambiguous"), L.ctx.counter("exact_fallbacks")
        g = L.buildPlaneResiduals(lio.r3live_params(size_voxel_map=b.size, **prm_kw), S.IDENTITY_Q, S.ZERO_T, S.T_LAST, debug=debug)
        da, de = L.ctx.counter("fast_ambiguous") - a0, L.ctx.counter("exact_fallbacks") - e0
    finally:
        _options(L, None)
    return g, da, de


def _oracle(b, prm_kw, debug=True):
    om = O.OracleMap()
    om.load(*b.map)
    return om.build_plane_residuals(b.kp, S.IDENTITY_Q, S.ZERO_T, S.T_LAST, O.r3live_params(size_voxel_map=b.size, **prm_kw), debug=debug)


def _assert_rows_equal(g, o, b, tag):
    assert np.array_equal(g.status, o.status), (tag, np.flatnonzero(g.status != o.status)[:10])
    assert np.array_equal(g.world_xyz, o.world_xyz), tag
    full = o.status > 0
    bad = np.flatnonzero(np.any(g.nbr[full] != o.nbr[full], axis=(1, 2)))
    assert bad.size == 0, (tag, [b.hoods[i].variant for i in np.flatnonzero(full)[bad][:8]])
    assert np.array_equal(g.nbr_dist[full].view(np.uint64), o.nbr_dist[full].view(np.uint64)), tag
    cols = np.r_[3:16]
    got, ref = g.plane[full][:, cols], o.plane[full][:, cols]
    scale = np.maximum(np.abs(ref), 1.0)
    bad = np.flatnonzero(np.any(np.abs(got - ref) > REL * scale, axis=1))
    assert bad.size == 0, (tag, [b.hoods[i].variant for i in np.flatnonzero(full)[bad][:8]])
    assert g.num_residuals == o.num_residuals and g.num_full_neighborhoods == o.num_full_neighborhoods, tag


def _assert_sums_equal(g, o, tag):
    """o: the oracle's pass with debug rows; every component to SUM_REL of the sum of its absolute contributions."""
    assert g.num_residuals == o.num_residuals and g.success == o.success, tag
    sH, sh, sl = S.sum_scales(o)
    assert (np.abs(g.HTH - o.HTH) / sH).max() <= SUM_REL, (tag, (np.abs(g.HTH - o.HTH) / sH).max())
    assert (np.abs(g.HTh - o.HTh) / sh).max() <= SUM_REL, (tag, (np.abs(g.HTh - o.HTh) / sh).max())
    assert abs(g.loss_sum - o.loss_sum) <= SUM_REL * sl, tag


@pytest.mark.parametrize("form", list(S.FORMS))
@pytest.mark.parametrize("family", S.FAMILIES)
def test_every_form_decides_like_the_oracle(lios, batches, family, form):
    """Steady parameters (nb = 1, K = 20): rows bit-exact with debug output, sums without; the flag counter within the
    model's range."""
    flagged_gpu = flagged_lo = flagged_hi = 0
    for size in S.SIZES:
        b, meas = batches[(family, size)]
        o = _oracle(b, {"max_num_residuals": BIG})
        L = lios[size]
        g, da, _ = _pass(L, b, form, {"max_num_residuals": BIG}, True)
        _assert_rows_equal(g, o, b, (family, size, form, "debug"))
        g2, da2, _ = _pass(L, b, form, {"max_num_residuals": BIG}, False)
        _assert_sums_equal(g2, o, (family, size, form))
        if form in S.MODEL_FORM:
            lo = sum(S.predicted_flags(m, form)[0] for m in meas)
            hi = sum(S.predicted_flags(m, form)[1] for m in meas)
            assert lo <= da <= hi and lo <= da2 <= hi, (family, size, form, da, da2, lo, hi)
            flagged_gpu += da2
            flagged_lo += lo
            flagged_hi += hi
    if form in S.MODEL_FORM:
        t = TABLE[(family, form)]
        t.update(keypoints=sum(len(batches[(family, s)][0].hoods) for s in S.SIZES), gpu_flagged=flagged_gpu,
                 model_flagged_lo=flagged_lo, model_flagged_hi=flagged_hi)
        for size in S.SIZES:
            for m in batches[(family, size)][1]:
                t[S.branch(m, form)] += 1
        print(f"\n{family} {form}: {dict(t)}")


@pytest.mark.parametrize("pset", [p for p in PARAM_SETS if p != "steady"])
@pytest.mark.parametrize("family", S.FAMILIES)
def test_other_parameter_sets(lios, batches, family, pset):
    """nb = 2 (init frames), K = 10, min_number_neighbors = 5: k1_assoc alone, whose own FP32 bound sends the keypoints of
    families A and D to its exact fallback; voxel_neighborhood = 0: the fast forms over the keypoint's own voxel."""
    prm = dict(max_num_residuals=BIG, **PARAM_SETS[pset])
    fallbacks = 0
    for size in S.SIZES:
        b, _ = batches[(family, size)]
        o = _oracle(b, prm)
        for form in (None, "assoc", "exact"):
            g, _, de = _pass(lios[size], b, form, prm, True)
            _assert_rows_equal(g, o, b, (family, size, pset, form, "debug"))
            if form == "assoc":
                fallbacks += de
            g2, _, _ = _pass(lios[size], b, form, prm, False)
            _assert_sums_equal(g2, o, (family, size, pset, form))
    if family in "AD" and pset in ("init_frame", "K10", "min5"):
        assert fallbacks > 0, (family, pset)
    print(f"\n{family} {pset}: k1_assoc exact fallbacks {fallbacks}")


def test_occupancy_threshold_inside_the_window(lios, batches):
    """Family E with threshold_voxel_occupancy = 3: the two-point voxel next to the keypoint is not a candidate."""
    prm = dict(max_num_residuals=BIG, threshold_voxel_occupancy=3)
    for size in S.SIZES:
        b, _ = batches[("E", size)]
        o = _oracle(b, prm)
        o1 = _oracle(b, dict(max_num_residuals=BIG))
        assert np.any(o.nbr != o1.nbr)                          # the threshold changes the answer: the voxel is decisive
        for form in S.FORMS:
            g, _, _ = _pass(lios[size], b, form, prm, True)
            _assert_rows_equal(g, o, b, ("E", size, "occupancy3", form))
            g2, _, _ = _pass(lios[size], b, form, prm, False)
            _assert_sums_equal(g2, o, ("E", size, "occupancy3", form))


@pytest.mark.parametrize("form", ["split4", "split2", "assoc"])
def test_capped_pass_after_flagged_keypoints(lios, batches, form):
    """max_num_residuals with k* after several flagged keypoints (families A and B mixed, keypoint order)."""
    from sr_livo_b200 import lio
    size = 1.0
    b, meas = batches[("B", size)]
    o_full = _oracle(b, dict(max_num_residuals=BIG))
    acc = np.flatnonzero(o_full.status == 2)
    flagged_before = [k for k in range(len(meas)) if S.predicted_flags(meas[k], "split4")[0] and k < acc[len(acc) // 2]]
    assert len(flagged_before) >= 3
    cap = len(acc) // 2
    prm = dict(max_num_residuals=cap)
    o = _oracle(b, prm)
    g, _, _ = _pass(lios[size], b, form, prm, False)
    _assert_sums_equal(g, o, ("capped", form))
    assert o.num_residuals == cap


def test_square_root_ties_keep_the_neighbour_set(lios):
    """Pairs whose FP64 d^2 differ but whose square roots tie: the reference keeps whatever its heap leaves (documented
    deviation); the device ranks by d^2.  Status and the neighbour set are the same wherever the tie is not at the K-th
    boundary; how often the order or the boundary member differs is printed."""
    b = S.build_batch("D", 1.0, sqrt_ties=True)
    assert len(b.hoods) >= 4
    o = _oracle(b, dict(max_num_residuals=BIG))
    differ = 0
    for form in S.FORMS:
        g, _, _ = _pass(lios[1.0], b, form, dict(max_num_residuals=BIG), True)
        assert np.array_equal(g.status > 0, o.status > 0)
        for k in range(len(b.hoods)):
            sg = {tuple(r) for r in g.nbr[k].tolist()}
            so = {tuple(r) for r in o.nbr[k].tolist()}
            assert len(sg ^ so) <= 2, (form, k)                  # at most the tied pair trades places
            differ += int(not np.array_equal(g.nbr[k], o.nbr[k]))
    print(f"\nsquare-root ties: {len(b.hoods)} keypoints x {len(S.FORMS)} forms, neighbour list differs from the oracle's at {differ}")
