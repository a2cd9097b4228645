"""CPU pins of the exact pass sums and of the rounding bound (tests/pass_sum_reference.py).

* The exact sum equals rational arithmetic (fractions.Fraction) on products whose factors span 2^-60 .. 2^60,
  including sets that cancel exactly.
* A plain restatement of each form's summation tree (k1_fit, k1_assoc with and without the fallback's hand-over,
  k1_fast, k2_cap_reduce) stays inside gamma_h * sum |x| on random terms, with every product rounded on its own and
  with every product fused into the first add that consumes it (emulated exactly with Fraction).
* On a real scene's terms the bound is tight enough to see a defect: dropping one keypoint's term, counting one twice
  or swapping two components puts the sum outside it.
"""
import os
from fractions import Fraction

import numpy as np
import pytest

import pass_sum_reference as R

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "scan_matching.npz")


# ---- restatements of the device summation trees (one component; leaves in the pass's keypoint order) -----------------
def _leaf(a, b):
    return float(a) * float(b)


def _fused(a, b, c):
    """fl(a * b + c) with the product exact: what DFMA computes."""
    return float(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def _warp_tree(a, b, lanes, shifts, fuse):
    """The 32-lane shuffle tree of one group: level 1 pairs lane l with l ^ shifts[0] (the lower lane keeps its own
    product, which DFMA may fuse into that add), later levels pair the partial sums."""
    v = {}
    s0 = shifts[0]
    for l in range(32):
        if l & s0:
            continue
        m = l ^ s0
        pa, pb = lanes.get(l), lanes.get(m)
        send = _leaf(a[pb], b[pb]) if pb is not None else 0.0
        if pa is None:
            v[l] = 0.0 + send
        elif fuse:
            v[l] = _fused(a[pa], b[pa], send)
        else:
            v[l] = _leaf(a[pa], b[pa]) + send
    for s in shifts[1:]:
        v = {l: v[l] + v[l ^ s] for l in v if not (l & s)}
    (x,) = v.values()
    return x


def _seq(vals):
    s = 0.0
    for x in vals:
        s += x
    return s


def model_fit(a, b, fuse):
    n = len(a)
    G = R.fit_grid(n)
    n_groups = -(-n // 32)
    acc = np.zeros((G, R.FAST_WARPS)).tolist()
    for g in range(n_groups):
        blk, w = g % G, (g // G) % R.FAST_WARPS
        lanes = {l: g * 32 + l for l in range(32) if g * 32 + l < n}
        acc[blk][w] += _warp_tree(a, b, lanes, (4, 2, 1, 8, 16), fuse)
    rows = [_seq(acc[blk]) for blk in range(G)]
    n_chunks = -(-G // R.CHUNK_BLOCKS)
    chunk_sums = []
    for c in range(n_chunks):
        in_chunk = min(R.CHUNK_BLOCKS, G - c * R.CHUNK_BLOCKS)
        per_warp = [_seq([rows[c * R.CHUNK_BLOCKS + r] if r < in_chunk else 0.0 for r in range(w, R.CHUNK_BLOCKS, R.FAST_WARPS)])
                    for w in range(R.FAST_WARPS)]
        chunk_sums.append(_seq(per_warp))
    return _seq([_seq(chunk_sums[w::R.FAST_WARPS]) for w in range(R.FAST_WARPS)])


def model_assoc(a, b, fuse, sm_count, per_sm, prev=None):
    n = len(a)
    G = R.assoc_grid(n, sm_count, per_sm)
    n_groups = -(-n // 32)
    acc = np.zeros((G, R.K1_WARPS)).tolist()
    for g in range(n_groups):
        blk, w = g % G, (g // G) % R.K1_WARPS
        lanes = {l: g * 32 + l for l in range(32) if g * 32 + l < n}
        acc[blk][w] += _warp_tree(a, b, lanes, (16, 8, 4, 2, 1), fuse)
    rows = [_seq(acc[blk]) for blk in range(G)]
    tot = _seq([_seq(rows[w::R.K1_WARPS]) for w in range(R.K1_WARPS)])
    return tot + prev if prev is not None else tot


def model_fast(a, b, fuse):
    n = len(a)
    G = R.fast_grid(n, 1)
    n_groups = -(-n // 32)
    acc = np.zeros((G, R.FAST_WARPS)).tolist()
    for g in range(n_groups):
        blk, w = g % G, (g // G) % R.FAST_WARPS
        lanes = {l: g * 32 + l for l in range(32) if g * 32 + l < n}
        acc[blk][w] += _warp_tree(a, b, lanes, (16, 8, 4, 2, 1), fuse)
    rows = [_seq(acc[blk]) for blk in range(G)]
    per_warp = []
    for w in range(R.FAST_WARPS):
        sacc = [0.0] * 8
        bb = w
        while bb + 7 * R.FAST_WARPS < G:
            for u in range(8):
                sacc[u] += rows[bb + u * R.FAST_WARPS]
            bb += 8 * R.FAST_WARPS
        while bb < G:
            sacc[0] += rows[bb]
            bb += R.FAST_WARPS
        per_warp.append(((sacc[0] + sacc[1]) + (sacc[2] + sacc[3])) + ((sacc[4] + sacc[5]) + (sacc[6] + sacc[7])))
    return _seq(per_warp)


def model_cap(a, b, fuse, bounds, chunks_run):
    out = 0.0
    for j in range(chunks_run):
        lo, hi = bounds[j], bounds[j + 1]
        acc = [0.0] * 1024
        for k in range(lo, hi):
            t = (k - lo) % 1024
            acc[t] = _fused(a[k], b[k], acc[t]) if fuse else acc[t] + _leaf(a[k], b[k])
        warps = []
        for w in range(32):
            v = {l: acc[32 * w + l] for l in range(32)}
            for s in (16, 8, 4, 2, 1):
                v = {l: v[l] + v[l ^ s] for l in v if not (l & s)}
            warps.append(v[0])
        out = out + _seq(warps)
    return out


# ---- random terms -----------------------------------------------------------------------------------------------------
def _wide_terms(rng, n, lo=-30, hi=30):
    """Factors with random 53-bit mantissas and exponents in [lo, hi]: products span 2^(2 lo) .. 2^(2 hi)."""
    def one():
        return rng.choice([-1.0, 1.0], n) * np.ldexp(rng.uniform(1.0, 2.0, n), rng.integers(lo, hi + 1, n))
    return one(), one()


def _frac_sum(a, b):
    return float(sum((Fraction(float(x)) * Fraction(float(y)) for x, y in zip(a, b)), Fraction(0)))


@pytest.mark.parametrize("seed", range(6))
def test_exact_sum_equals_rational_arithmetic(seed):
    rng = np.random.default_rng(seed)
    a, b = _wide_terms(rng, 400)
    assert R.exact_sum_of_products(a, b)[0] == _frac_sum(a, b)
    # exactly cancelling sets: every product appears with both signs, plus one tiny survivor
    a2 = np.concatenate([a, -a, [2.0 ** -60]])
    b2 = np.concatenate([b, b, [3.0]])
    perm = rng.permutation(a2.size)
    a2, b2 = a2[perm], b2[perm]
    assert R.exact_sum_of_products(a2, b2)[0] == _frac_sum(a2, b2) == 3.0 * 2.0 ** -60
    assert R.exact_sum_of_products(a[:0], b[:0])[0] == 0.0
    # near-cancellation: the rounded products alone sum to the wrong value, their errors carry the answer
    x = np.array([1.0 + 2.0 ** -30, -(1.0 + 2.0 ** -29)])
    y = np.array([1.0 + 2.0 ** -30, 1.0])
    assert R.exact_sum_of_products(x, y)[0] == _frac_sum(x, y) == 2.0 ** -60


def test_two_product_is_exact():
    rng = np.random.default_rng(9)
    a, b = _wide_terms(rng, 2000)
    p, e = R.two_product(a, b)
    for x, y, pp, ee in zip(a[:300], b[:300], p[:300], e[:300]):
        assert Fraction(float(pp)) + Fraction(float(ee)) == Fraction(float(x)) * Fraction(float(y))


def _scene_like(rng, n):
    """Terms with the spread of a real pass: factors over three decades, both signs, some near-cancelling."""
    a = rng.normal(0.0, 1.0, n) * 10.0 ** rng.uniform(-2.0, 1.0, n)
    b = rng.normal(0.0, 1.0, n) * 10.0 ** rng.uniform(-2.0, 1.0, n)
    return a, b


def _check(model_value, a, b, h):
    ref, mag = R.exact_sum_of_products(a, b)
    err = abs(model_value - ref)
    assert err <= R.gamma(h) * mag, (err, R.gamma(h) * mag)
    return err / max(R.gamma(h) * mag, 1e-300)


@pytest.mark.parametrize("n", [1, 31, 33, 129, 4097, 8193])
@pytest.mark.parametrize("fuse", [False, True])
def test_fit_tree_holds_its_bound(n, fuse):
    rng = np.random.default_rng(n)
    a, b = _scene_like(rng, n)
    _check(model_fit(a, b, fuse), a, b, R.h_fit(n))


def test_fit_tree_second_grid_stride_round():
    """n = 262 145: 2048 blocks, 64 chunks, the second grid-stride round holds one keypoint."""
    n = 262145
    rng = np.random.default_rng(1)
    a, b = _scene_like(rng, n)
    assert R.fit_grid(n) == R.MAX_GRID and R.h_fit(n) <= 100
    _check(model_fit(a, b, False), a, b, R.h_fit(n))


@pytest.mark.parametrize("n,per_sm", [(1, 1), (33, 2), (4223, 1), (8449, 2), (16897, 4)])
@pytest.mark.parametrize("fuse", [False, True])
def test_assoc_tree_holds_its_bound(n, per_sm, fuse):
    rng = np.random.default_rng(n + per_sm)
    a, b = _scene_like(rng, n)
    _check(model_assoc(a, b, fuse, 132, per_sm), a, b, R.h_assoc(n, 132, per_sm))


@pytest.mark.parametrize("fuse", [False, True])
def test_fallback_hand_over_holds_its_bound(fuse):
    """The first launch sums the unflagged keypoints, the fallback launch the flagged ones and then adds the first's."""
    rng = np.random.default_rng(5)
    n = 5000
    a, b = _scene_like(rng, n)
    flagged = np.zeros(n, bool)
    flagged[::7] = True
    af, bf = np.where(flagged, 0.0, a), np.where(flagged, 0.0, b)
    ag, bg = np.where(flagged, a, 0.0), np.where(flagged, b, 0.0)
    first = model_fit(af, bf, fuse)
    total = model_assoc(ag, bg, fuse, 132, 1, prev=first)
    _check(total, a, b, R.h_fallback(R.h_fit(n), n, 132))


@pytest.mark.parametrize("n", [1, 100, 5000])
@pytest.mark.parametrize("fuse", [False, True])
def test_fast_tree_holds_its_bound(n, fuse):
    rng = np.random.default_rng(n + 17)
    a, b = _scene_like(rng, n)
    _check(model_fast(a, b, fuse), a, b, R.h_fast(n, 1))


@pytest.mark.parametrize("fuse", [False, True])
def test_cap_tree_holds_its_bound(fuse):
    rng = np.random.default_rng(23)
    n = 15000
    a, b = _scene_like(rng, n)
    bounds = R.cap_chunk_bounds(n, 100)
    assert bounds == [0, 4096, 12288, 15000]
    for run in (1, 2, 3):
        hi = bounds[run]
        _check(model_cap(a, b, fuse, bounds, run), a[:hi], b[:hi], R.h_cap(bounds, run))


def test_bound_stays_near_1e_14_at_every_suite_size():
    for n in (1, 31, 32, 33, 127, 128, 129, 4095, 4096, 4097, 8193, 131072, 262143, 262144, 262145, 266241, 524289):
        assert R.h_fit(n) <= 100, n
        assert R.h_fallback(R.h_fit(n), n, 132) <= 100, n
    for p in (1, 2, 3, 4, 6, 8, 9, 12, 16):
        for d in (-1, 0, 1, 33):
            n = 32 * 132 * p + d
            assert R.h_assoc_any(n, 132, fallback=True) <= 100, n
    assert R.gamma(100) < 1.2e-14


# ---- a real scene's terms: the bound sees a defect ---------------------------------------------------------------------
@pytest.fixture(scope="module")
def scene():
    g = np.load(GOLDEN)
    plane, status = g["nb1_plane"], g["nb1_status"]
    assert np.count_nonzero(status == 2) > 300
    return plane, status


def _device_like(plane, status):
    """Components 0..27 as k1_fit sums them, keypoints in index order."""
    return np.array([model_fit(a, b, False) for a, b in R.term_factors(plane, status)])


def test_scene_terms_hold_the_bound(scene):
    plane, status = scene
    got = _device_like(plane, status)
    ref, mag = R.exact_sums(plane, status)
    n = len(status)
    bnd = R.bound(mag[:28], R.h_fit(n))
    assert np.all(np.abs(got - ref[:28]) <= bnd)
    # the bound is not vacuous: below the median magnitude of the component's terms
    x = R.term_values(plane, status)
    for c in range(28):
        nz = np.abs(x[c][x[c] != 0])
        assert bnd[c] < np.median(nz), c


def test_dropping_or_doubling_one_keypoint_breaks_the_bound(scene):
    plane, status = scene
    ref, mag = R.exact_sums(plane, status)
    bnd = R.bound(mag[:28], R.h_fit(len(status)))
    x = R.term_values(plane, status)
    # any one keypoint lost or counted twice moves some component by |x_k| > the bound
    assert np.all(np.any(np.abs(x) > bnd[:, None], axis=0))
    # and on the full restatement of k1_fit, for one keypoint each way
    acc = np.flatnonzero(status == 2)
    k = acc[len(acc) // 2]
    lost = status.copy()
    lost[k] = 1
    twice_p = np.concatenate([plane, plane[k:k + 1]])
    twice_s = np.concatenate([status, [2]])
    for p, st in ((plane, lost), (twice_p, twice_s)):
        got = _device_like(p, st)
        assert np.any(np.abs(got - ref[:28]) > bnd)


def test_swapping_two_components_breaks_the_bound(scene):
    plane, status = scene
    got = _device_like(plane, status)
    ref, mag = R.exact_sums(plane, status)
    bnd = R.bound(mag[:28], R.h_fit(len(status)))
    for i in range(28):
        for j in range(i + 1, 28):
            if ref[i] == ref[j]:
                continue
            sw = got.copy()
            sw[i], sw[j] = sw[j], sw[i]
            assert np.any(np.abs(sw - ref[:28]) > bnd), (i, j)
