"""The pass sums on the device against exact sums of their per-keypoint terms (tests/pass_sum_reference.py).

Each case runs the pass once with debug outputs and twice without.  The debug run's per-keypoint rows give the exact
sums; its 32 sums must lie within gamma_h * sum |x| of them, with h the height of the form's summation tree (about
1e-14 of sum |x|, where test_gpu_parity.py allows 1e-5 of the largest entry).  The counts are exact, the NaN count 0.
The bound is not vacuous: it is below the median term of every component, so a keypoint lost or counted twice anywhere
in the tree breaks it.  Both product runs are bitwise equal, and equal to the debug run (same grid, same order).

Beyond one pass: the fallback launch's hand-over, the state carried from pass to pass, sharded ranges on one GPU and
the ordered residual cap (k2_cap_reduce).
"""
import numpy as np
import pytest

import pass_sum_cases as PC
import pass_sum_reference as R

pytestmark = pytest.mark.gpu
RATIOS = {}   # form -> largest |device - exact| / bound seen (printed at the end of the module)


@pytest.fixture(scope="module")
def L():
    from sr_livo_b200 import lio
    obj = lio.LioOptimization(max_voxels=1 << 18, sweep_capacity=1 << 20)
    obj.addPointsToMap(PC.map_points())
    yield obj
    obj.close()


@pytest.fixture(scope="module")
def pool(L):
    p = PC.twin_pool(L)
    assert p.shape[0] > 5000
    return p


@pytest.fixture(scope="module")
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _sums32(r):
    o = np.zeros(32)
    o[:21] = [r.HTH[i, j] for i, j in R.PAIRS]
    o[21:27] = r.HTh
    o[27] = r.loss_sum
    o[28], o[29], o[30] = r.num_residuals, r.num_full_neighborhoods, r.num_candidates_scanned
    return o


def _bits(r):
    return _sums32(r).tobytes()


def _prm(**kw):
    from sr_livo_b200 import lio
    return lio.r3live_params(max_num_residuals=PC.BIG, **kw)


def _run3(L, prm, q=PC.OFFSET_Q, t=PC.OFFSET_T):
    g = L.buildPlaneResiduals(prm, q, t, PC.T_LAST, debug=True)
    p1 = L.buildPlaneResiduals(prm, q, t, PC.T_LAST)
    p2 = L.buildPlaneResiduals(prm, q, t, PC.T_LAST)
    return g, p1, p2


def _within(form, got, ref, mag, h, comps=range(28)):
    comps = list(comps)
    bnd = R.bound(mag[comps], h)
    err = np.abs(got[comps] - ref[comps])
    ratio = float(np.max(np.where(bnd > 0, err / np.where(bnd > 0, bnd, 1.0), np.where(err > 0, np.inf, 0.0))))
    RATIOS[form] = max(RATIOS.get(form, 0.0), ratio)
    worst = comps[int(np.argmax(err - bnd))]
    assert np.all(err <= bnd), f"{form}: component {worst} off by {err[comps.index(worst)]:.3e}, bound {bnd[comps.index(worst)]:.3e}"


def _not_vacuous(g, h, mag):
    x = R.term_values(g.plane, g.status)
    bnd = R.bound(mag[:28], h)
    for c in range(28):
        nz = np.abs(x[c][x[c] != 0])
        if nz.size:
            assert bnd[c] < np.median(nz), (c, bnd[c], np.median(nz))


def _check_pass(form, g, p1, p2, n, h):
    assert h <= 100
    assert np.all(g.status == 2), "the scene's premise: every keypoint is accepted"
    ref, mag = R.exact_sums(g.plane, g.status)
    got = _sums32(g)
    _within(form, got, ref, mag, h)
    assert got[28] == ref[28] == n and got[29] == ref[29] == n
    assert _bits(p1) == _bits(p2), "two product runs differ"
    assert _bits(g) == _bits(p1), "the debug run differs from the product run"
    _not_vacuous(g, h, mag)
    return ref, mag


# ---- k1_fit (split form, the default) ----------------------------------------------------------------------------------
@pytest.mark.parametrize("lpk", [4, 2])
def test_fit_sums_at_block_chunk_and_grid_stride_edges(L, pool, sm_count, lpk):
    L.ctx.set_option("split_lanes_per_keypoint", lpk)
    try:
        for i, n in enumerate(PC.FIT_SIZES):
            L.setKeypoints(PC.resample(pool, n, seed=100 + i))
            g, p1, p2 = _run3(L, _prm())
            h = R.h_fallback(R.h_fit(n), n, sm_count)   # k1_scan may flag a few keypoints: the fallback then adds them
            _check_pass("k1_fit", g, p1, p2, n, h)
    finally:
        L.ctx.set_option("split_lanes_per_keypoint", 4)


def test_cancelling_and_offset_pose(L, pool, sm_count):
    """At the pose the twins were drawn from, J^T h cancels to below 1e-6 of sum |J h|; the bound still holds there.
    The same keypoints at an offset pose do not cancel."""
    n = 2 * 65537
    L.setKeypoints(PC.cancelling(pool, n // 2, seed=7))
    h = R.h_fallback(R.h_fit(n), n, sm_count)
    g, p1, p2 = _run3(L, _prm(), PC.POSE_Q, PC.POSE_T)
    ref, mag = _check_pass("k1_fit", g, p1, p2, n, h)
    assert np.all(np.abs(ref[21:27]) <= 1e-6 * mag[21:27]), "premise: J^T h cancels"
    g2, q1, q2 = _run3(L, _prm())
    _check_pass("k1_fit", g2, q1, q2, n, h)


# ---- k1_assoc -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["k1_variant_2", "init_frames_nb2"])
def test_assoc_sums_at_grid_stride_edges(L, pool, sm_count, mode):
    kw = dict(frame_id=5) if mode == "init_frames_nb2" else {}
    if mode == "k1_variant_2":
        L.ctx.set_option("k1_variant", 2)
    try:
        for i, n in enumerate(PC.assoc_sizes(sm_count)):
            L.setKeypoints(PC.resample(pool, n, seed=300 + i))
            g, p1, p2 = _run3(L, _prm(**kw))
            _check_pass("k1_assoc", g, p1, p2, n, R.h_assoc_any(n, sm_count))
    finally:
        L.ctx.set_option("k1_variant", 0)


def test_fast_sums(L, pool, sm_count):
    L.ctx.set_option("k1_variant", 1)
    lpk = L.ctx.counter("fast_lanes_per_keypoint")
    try:
        for i, n in enumerate(PC.FAST_SIZES):
            L.setKeypoints(PC.resample(pool, n, seed=500 + i))
            g, p1, p2 = _run3(L, _prm())
            _check_pass("k1_fast", g, p1, p2, n, R.h_fallback(R.h_fast(n, lpk), n, sm_count))
    finally:
        L.ctx.set_option("k1_variant", 0)


# ---- the fallback launch's hand-over ----------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [8193, 262145])
def test_fallback_hand_over(L, pool, sm_count, n):
    """fast_force_ambiguous_mod m flags keypoints k % m == 0: every one (m = 1, k1_fit's own part is zero), a seventh,
    keypoints 0 and n - 1, and only keypoint 0 (m > n).  Both launches' sums together are within the bound."""
    L.setKeypoints(PC.resample(pool, n, seed=600 + n))
    h = R.h_fallback(R.h_fit(n), n, sm_count)
    try:
        for m in (1, 7, n - 1, n + 5):
            L.ctx.set_option("fast_force_ambiguous_mod", m)
            before = L.ctx.counter("fast_ambiguous")
            g, p1, p2 = _run3(L, _prm())
            flagged = (L.ctx.counter("fast_ambiguous") - before) // 3
            assert flagged >= len(range(0, n, m)), (m, flagged)
            _check_pass("k1_fit + fallback", g, p1, p2, n, h)
    finally:
        L.ctx.set_option("fast_force_ambiguous_mod", 0)


# ---- pass-to-pass state --------------------------------------------------------------------------------------------
def test_pass_to_pass_state(L, pool, sm_count):
    """Tickets, chunk tickets, the scan count, `flagged` and `finalised` are reset by the pass that used them: a sequence
    of passes with and without flagged keypoints, growing and shrinking, each matches its own exact sums and differs
    from the pass before (no stale result forwarded)."""
    seq = [(262145, 0), (33, 7), (4097, 0), (4097, 7), (524289, 0)]
    prev = None
    try:
        for i, (n, mod) in enumerate(seq):
            L.ctx.set_option("fast_force_ambiguous_mod", mod)
            L.setKeypoints(PC.resample(pool, n, seed=700 + i))
            dq = PC.synth.quat_from_rotvec([1e-4 * i, 0.0, -1e-4 * i])
            q, t = PC.synth.quat_mul(PC.OFFSET_Q, dq), PC.OFFSET_T + 1e-3 * i
            g, p1, p2 = _run3(L, _prm(), q, t)
            _check_pass("k1_fit + fallback", g, p1, p2, n, R.h_fallback(R.h_fit(n), n, sm_count))
            if prev is not None:
                assert not np.array_equal(_sums32(g)[:28], prev[:28])
            prev = _sums32(g)
    finally:
        L.ctx.set_option("fast_force_ambiguous_mod", 0)


# ---- shards on one GPU --------------------------------------------------------------------------------------------
def test_shards_partition_the_sweep(L, pool, sm_count):
    n = 8193
    raw = PC.resample(pool, n, seed=800)
    L.setKeypoints(raw)
    whole = L.buildPlaneResiduals(_prm(), PC.OFFSET_Q, PC.OFFSET_T, PC.T_LAST, debug=True)
    w32 = _sums32(whole)
    try:
        for m in (1, 32, 4096, 4097, n - 1):
            parts = []
            for lo, hi in ((0, m), (m, n)):
                L.sweep.set_shard(lo, hi)
                g = L.buildPlaneResiduals(_prm(), PC.OFFSET_Q, PC.OFFSET_T, PC.T_LAST, debug=True)
                mem = np.any(g.world_xyz != 0.0, axis=1)   # the debug buffers are zeroed before each pass
                assert mem.sum() == hi - lo
                ref, mag = R.exact_sums(whole.plane, whole.status, members=mem)
                got = _sums32(g)
                _within("k1_fit shard", got, ref, mag, R.h_fallback(R.h_fit(hi - lo), n, sm_count))
                assert got[28] == ref[28] == hi - lo and got[29] == ref[29]
                assert np.array_equal(g.status[mem], whole.status[mem]) and not g.status[~mem].any()
                parts.append((mem, got))
            (ma, a), (mb, b) = parts
            assert np.all(ma ^ mb), "the two shards partition the sweep"
            assert a[28] + b[28] == w32[28] and a[29] + b[29] == w32[29] and a[30] + b[30] == w32[30]
            L.sweep.set_shard(m, m)
            e = L.buildPlaneResiduals(_prm(), PC.OFFSET_Q, PC.OFFSET_T, PC.T_LAST)
            assert not _sums32(e).any() and not e.success
    finally:
        L.sweep.set_shard(0, n)


# ---- the ordered residual cap (k2_cap_reduce) ---------------------------------------------------------------------
def test_capped_sums(L, pool):
    """k* (the cap-th accepted keypoint) on the first and the last keypoint of chunks 0 and 1 of cap_chunk_bounds, and a
    cap never reached.  The capped sums are within the k2_cap_reduce bound of the exact sum over accepted k <= k*."""
    from sr_livo_b200 import lio
    n = 20000
    rng = np.random.default_rng(900)
    cap = 100
    b = R.cap_chunk_bounds(n, cap)                       # [0, 4096, 12288, 20000]; the same for cap 1
    cases = [(1, 0, [0] + list(rng.choice(np.arange(1, n), 3000, replace=False)))]
    for kstar in (b[1] - 1, b[1], b[2] - 1):
        before = rng.choice(np.arange(0, kstar), cap - 1, replace=False)
        after = rng.choice(np.arange(kstar + 1, n), 2000, replace=False)
        cases.append((cap, kstar, [kstar] + list(before) + list(after)))
    cases.append((n - 1, None, list(rng.choice(np.arange(n), 9000, replace=False))))
    for i, (c, kstar, acc_at) in enumerate(cases):
        L.setKeypoints(PC.capped_layout(pool, n, acc_at, seed=910 + i))
        prm = lio.r3live_params(max_num_residuals=c)
        g = L.buildPlaneResiduals(prm, PC.OFFSET_Q, PC.OFFSET_T, PC.T_LAST, debug=True)
        visited = g.status != -1
        k_found = int(np.flatnonzero(visited).max())
        assert k_found == (n - 1 if kstar is None else kstar)
        assert np.all(visited[: k_found + 1]) and np.all(g.status[visited] >= 0)
        acc = np.zeros(n, bool)
        acc[acc_at] = True
        assert np.array_equal(g.status[visited] == 2, acc[visited]), "premise: accepted exactly where placed"
        b = R.cap_chunk_bounds(n, c)                     # one chunk of 20000 for cap n - 1
        run = next(j for j in range(len(b) - 1) if b[j + 1] > k_found) + 1
        assert L.ctx.counter("cap_chunks_run") == run
        ref, mag = R.exact_sums(g.plane, g.status, members=visited)
        got = _sums32(g)
        h = R.h_cap(b, run)
        _within("k2_cap_reduce", got, ref, mag, h)
        assert got[28] == ref[28] and got[29] == ref[29]
        _not_vacuous(g, h, mag)
        p = L.buildPlaneResiduals(prm, PC.OFFSET_Q, PC.OFFSET_T, PC.T_LAST)
        assert _bits(p) == _bits(g)


def test_report_ratios():
    """The largest |device - exact| / bound per form in this run (for DESIGN.md)."""
    for form, r in sorted(RATIOS.items()):
        print(f"pass-sum ratio {form}: {r:.3e}")
