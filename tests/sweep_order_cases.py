"""Seeded sweeps at the edges of the sweep order's kernels (tests/sweep_order_reference.py restates the order).

Three families, each case asserting its defining property as it is built:
  size_*   uniform keys at every size where the cluster kernel's geometry steps: keys per warp (per = 32 ceil(n / 512 / 32)
           steps at multiples of 16 384), empty CTAs, partial last rounds, a full cluster (131 072) and the sizes past it
           that CUB sorts while the cluster kernel stays in use;
  keys_*   keys built from target keys by inverting the Morton map: all equal, differing in one pass's digit only, every
           digit of a pass in one warp, a warp whose lanes share one digit in every round or all differ, ascending and
           descending runs, ties interleaved with other keys (stability), one digit holding a whole CTA's 8 192 keys;
  coord_*  coordinates at the floor and clamp: signed zeros and subnormals, one ulp either side of every integer in
           [-129, 128], -128 / 127 / below 128 / 128, infinities and NaNs, +-1e308 and 2^53 + 1.
"""
import functools

import numpy as np

import sweep_order_reference as R

SIZES = ([1, 2, 31, 32, 33, 255, 256, 257, 8191, 8192, 8193, 16383, 16384, 16385]
         + [16384 * k + d for k in range(2, 8) for d in (-1, 1)]
         + [65535, 65536, 65537, 131071, 131072, 131073, 1000003])
BIG = max(SIZES)   # sweep capacity the device tests need

_BUILDERS = {}


def _case(name):
    def deco(fn):
        _BUILDERS[name] = fn
        return fn
    return deco


def names():
    return list(_BUILDERS)


@functools.lru_cache(maxsize=None)
def build(name):
    """(n, 3) float64 points of the case (its property is asserted on the way)."""
    xyz = _BUILDERS[name]()
    assert xyz.dtype == np.float64 and xyz.ndim == 2 and xyz.shape[1] == 3
    return np.ascontiguousarray(xyz)


def _uniform_keys(n, rng):
    return rng.integers(0, 1 << 24, n, dtype=np.uint32)


# ---- sizes -------------------------------------------------------------------------------------------------------------
def _size_case(n):
    def fn():
        g = R.geometry(n)
        if n <= R.CAPACITY:
            assert g["cta_n"].sum() == n and g["per"] % 32 == 0 and 32 <= g["per"] <= 256
            assert g["per"] == 32 * -(-n // (512 * 32)), n   # steps at every multiple of 16 384
            if n == 16385:   # CTAs 0..7 full, one key in CTA 8, CTAs 9..15 empty
                assert g["per"] == 64 and list(g["cta_n"][:9]) == [2048] * 8 + [1] and not g["cta_n"][9:].any()
            if n == R.CAPACITY:   # every warp holds 8 full rounds
                assert g["per"] == 256 and np.all(g["end"] - g["begin"] == 256)
            if n % 32:   # the last non-empty warp ends in a partial round
                last = int(np.nonzero(g["end"] > g["begin"])[0][-1])
                assert (g["end"][last] - g["begin"][last]) % 32 == n % 32
        else:
            assert n > R.CAPACITY   # sorted by CUB while the cluster kernel stays in use
        return R.points_for_keys(_uniform_keys(n, np.random.default_rng(n)), np.random.default_rng(n + 1))
    return fn


for _n in SIZES:
    _case(f"size_{_n}")(_size_case(_n))


# ---- key patterns ------------------------------------------------------------------------------------------------------
def _pts(k, seed):
    return R.points_for_keys(np.asarray(k, np.uint32), np.random.default_rng(seed))


@_case("keys_all_equal_full")
def _():
    k = np.full(R.CAPACITY, 0xA5C3F1, np.uint32)
    return _pts(k, 1)


@_case("keys_all_equal_ragged")
def _():
    k = np.full(16385, 0x5A3C0E, np.uint32)
    assert R.geometry(16385)["cta_n"][8] == 1
    return _pts(k, 2)


def _one_digit_case(p):
    def fn():
        n = 50000
        rng = np.random.default_rng(10 + p)
        base = np.uint32(0x6B2D93) & ~(np.uint32(0xFF) << np.uint32(8 * p))
        k = base | (rng.integers(0, 256, n, dtype=np.uint32) << np.uint32(8 * p))
        for q in range(3):   # only digit p differs
            assert (len(np.unique(R.digit(k, q))) > 200) == (q == p)
        return _pts(k, 20 + p)
    return fn


for _p in range(3):
    _case(f"keys_only_digit{_p}")(_one_digit_case(_p))


@_case("keys_every_digit_in_one_warp")
def _():
    n = R.CAPACITY
    rng = np.random.default_rng(30)
    k = _uniform_keys(n, rng)
    g = R.geometry(n)
    w = 77                                   # warp 13 of CTA 2
    b, e = int(g["begin"][w]), int(g["end"][w])
    k[b:e] = (rng.permutation(256).astype(np.uint32) | (rng.permutation(256).astype(np.uint32) << np.uint32(8))
              | (rng.permutation(256).astype(np.uint32) << np.uint32(16)))
    assert e - b == 256 and all(len(np.unique(R.digit(k[b:e], p))) == 256 for p in range(3))
    return _pts(k, 31)


@_case("keys_warp_lanes_one_digit_and_all_distinct")
def _():
    n = R.CAPACITY
    rng = np.random.default_rng(40)
    k = _uniform_keys(n, rng)
    g = R.geometry(n)
    same, diff = 200, 201                     # two warps of CTA 6
    for r in range(R.ROUNDS):
        s = int(g["begin"][same]) + 32 * r
        k[s:s + 32] = rng.integers(0, 1 << 24, dtype=np.uint32)            # the round's 32 lanes share every digit
        d = int(g["begin"][diff]) + 32 * r
        k[d:d + 32] = sum(rng.choice(256, 32, replace=False).astype(np.uint32) << np.uint32(8 * p) for p in range(3))
    for r in range(R.ROUNDS):
        s, d = int(g["begin"][same]) + 32 * r, int(g["begin"][diff]) + 32 * r
        for p in range(3):
            assert len(np.unique(R.digit(k[s:s + 32], p))) == 1 and len(np.unique(R.digit(k[d:d + 32], p))) == 32
    return _pts(k, 41)


@_case("keys_ascending")
def _():
    k = np.sort(_uniform_keys(100000, np.random.default_rng(50)))
    assert np.all(np.diff(k.astype(np.int64)) >= 0)
    return _pts(k, 51)


@_case("keys_descending")
def _():
    k = np.sort(_uniform_keys(100000, np.random.default_rng(52)))[::-1].copy()
    assert np.all(np.diff(k.astype(np.int64)) <= 0)
    return _pts(k, 53)


@_case("keys_alternating_runs")
def _():
    rng = np.random.default_rng(54)
    runs = [np.sort(_uniform_keys(int(rng.integers(1, 3000)), rng)) for _ in range(60)]
    k = np.concatenate([r if i % 2 == 0 else r[::-1] for i, r in enumerate(runs)])
    assert len(runs) == 60 and 1 < k.size < R.CAPACITY
    return _pts(k, 55)


@_case("keys_ties_interleaved")
def _():
    n = R.CAPACITY
    rng = np.random.default_rng(60)
    k = _uniform_keys(n, rng)
    tied = rng.random(n) < 0.5
    k[tied] = 0x31D7A2                         # half the sweep shares one key, spread over every warp
    few = rng.random(n) < 0.2
    k[few] = rng.choice(np.array([0x000000, 0xFFFFFF, 0x31D7A1, 0x31D7A3], np.uint32), int(few.sum()))
    assert np.count_nonzero(k == 0x31D7A2) > n // 3
    return _pts(k, 61)


@_case("keys_few_distinct")
def _():
    n = 100003
    rng = np.random.default_rng(62)
    k = rng.choice(np.array([0x123456, 0x123457, 0x923456, 0x12A456], np.uint32), n)
    assert len(np.unique(k)) == 4
    return _pts(k, 63)


def _whole_cta_digit(seq_k, p, c):
    g = R.geometry(seq_k[0].size)
    lo = c * R.KEYS_PER_CTA
    assert g["cta_n"][c] == R.KEYS_PER_CTA
    return len(np.unique(R.digit(seq_k[p][lo:lo + R.KEYS_PER_CTA], p))) == 1


@_case("keys_cta0_minimum_digit_every_pass")
def _():
    n = R.CAPACITY
    rng = np.random.default_rng(70)
    k = sum(rng.integers(1, 256, n, dtype=np.uint32) << np.uint32(8 * p) for p in range(3)).astype(np.uint32)
    k[:R.KEYS_PER_CTA] = 0                     # digit 0 holds CTA 0's 8192 keys in every pass
    seq = R.pass_inputs(k)
    assert all(_whole_cta_digit(seq, p, 0) for p in range(3))
    return _pts(k, 71)


@_case("keys_cta15_maximum_digit_every_pass")
def _():
    n = R.CAPACITY
    rng = np.random.default_rng(72)
    k = sum(rng.integers(0, 255, n, dtype=np.uint32) << np.uint32(8 * p) for p in range(3)).astype(np.uint32)
    k[-R.KEYS_PER_CTA:] = 0xFFFFFF             # digit 255 holds CTA 15's 8192 keys in every pass
    seq = R.pass_inputs(k)
    assert all(_whole_cta_digit(seq, p, 15) for p in range(3))
    return _pts(k, 73)


@_case("keys_cta9_one_digit_pass0")
def _():
    n = R.CAPACITY
    rng = np.random.default_rng(74)
    k = _uniform_keys(n, rng)
    lo = 9 * R.KEYS_PER_CTA
    k[lo:lo + R.KEYS_PER_CTA] = (k[lo:lo + R.KEYS_PER_CTA] & np.uint32(0xFFFF00)) | np.uint32(0x80)
    seq = R.pass_inputs(k)
    assert _whole_cta_digit(seq, 0, 9) and not _whole_cta_digit(seq, 1, 9)
    return _pts(k, 75)


@_case("keys_one_digit_over_two_ctas_ragged")
def _():
    n = 16384 * 5 - 1                          # per = 160: warps of 5 rounds, CTAs of 5120 keys, the last one short of one
    rng = np.random.default_rng(76)
    k = _uniform_keys(n, rng)
    g = R.geometry(n)
    lo, hi = 3 * 32 * g["per"], 5 * 32 * g["per"]
    k[lo:hi] = (k[lo:hi] & np.uint32(0xFF00FF)) | np.uint32(0x4200)   # CTAs 3 and 4 share one digit of pass 1 ...
    k[lo:hi] &= np.uint32(0xFFFF00)                                     # ... and of pass 0 (digit 0: they stay together)
    assert g["per"] == 160 and g["cta_n"][3] == g["cta_n"][4] == 5120
    assert len(np.unique(R.digit(k[lo:hi], 0))) == 1 and len(np.unique(R.digit(k[lo:hi], 1))) == 1
    return _pts(k, 77)


# ---- coordinates ---------------------------------------------------------------------------------------------------------
TINY = np.nextafter(0.0, 1.0)   # the smallest subnormal
NAN_NEG = -np.float64("nan")
NAN_PAYLOAD = np.array([0x7FF00000DEADBEEF], np.uint64).view(np.float64)[0]
NAN_NEG_PAYLOAD = np.array([0xFFF4000000000001], np.uint64).view(np.float64)[0]

# value -> its cell, stated by hand (floor + 128, clamped to [0, 255]; NaN to 0)
SPECIAL = [
    (0.0, 128), (-0.0, 128), (TINY, 128), (-TINY, 127),
    (-128.0, 0), (np.nextafter(-128.0, -np.inf), 0), (np.nextafter(-128.0, np.inf), 0), (-127.0, 1),
    (127.0, 255), (np.nextafter(127.0, -np.inf), 254), (np.nextafter(128.0, -np.inf), 255), (128.0, 255),
    (np.inf, 255), (-np.inf, 0), (np.nan, 0), (NAN_NEG, 0), (NAN_PAYLOAD, 0), (NAN_NEG_PAYLOAD, 0),
    (1e308, 255), (-1e308, 0), (float(2 ** 53 + 1), 255), (-float(2 ** 53 + 1), 0),
]


def ulp_neighbours():
    """(values, cells): one ulp below, at and one ulp above every integer in [-129, 128]."""
    v, c = [], []
    for i in range(-129, 129):
        for x, cell in ((np.nextafter(float(i), -np.inf), i - 1 + 128), (float(i), i + 128), (np.nextafter(float(i), np.inf), i + 128)):
            v.append(x)
            c.append(min(max(cell, 0), 255))
    return np.array(v), np.array(c, np.uint32)


def _check_cells(xyz, want):
    assert np.array_equal(R.cells(xyz), want)


@_case("coord_zeros_and_subnormals")
def _():
    vals = np.array([0.0, -0.0, TINY, -TINY])
    g = np.stack(np.meshgrid(vals, vals, vals, indexing="ij"), -1).reshape(-1, 3)
    xyz = np.tile(g, (40, 1))                 # 64 combinations, 40 times each: ties among them
    want = np.where(np.signbit(xyz) & (xyz != 0), 127, 128).astype(np.uint32)
    _check_cells(xyz, want)
    assert np.array_equal(np.signbit(xyz[:64]).sum(0), [32, 32, 32])
    return xyz


@_case("coord_ulp_around_integers")
def _():
    v, c = ulp_neighbours()
    rng = np.random.default_rng(80)
    m = v.size
    idx = np.concatenate([np.stack([np.arange(m), rng.permutation(m), rng.permutation(m)], 1),
                          rng.integers(0, m, (20 * m, 3))])
    xyz = v[idx]
    _check_cells(xyz, c[idx])
    assert m == 3 * 258
    return xyz


@_case("coord_special_values")
def _():
    v = np.array([x for x, _ in SPECIAL])
    c = np.array([y for _, y in SPECIAL], np.uint32)
    m = v.size
    g = np.stack(np.meshgrid(np.arange(m), np.arange(m), np.arange(m), indexing="ij"), -1).reshape(-1, 3)   # every triple
    xyz = v[g]
    _check_cells(xyz, c[g])
    assert np.isnan(xyz).any() and np.isinf(xyz).any() and xyz.shape[0] == m ** 3
    return xyz


@_case("coord_special_values_full_cluster")
def _():
    v = np.concatenate([np.array([x for x, _ in SPECIAL]), ulp_neighbours()[0]])
    c = np.concatenate([np.array([y for _, y in SPECIAL], np.uint32), ulp_neighbours()[1]])
    rng = np.random.default_rng(81)
    idx = rng.integers(0, v.size, (R.CAPACITY, 3))
    xyz = v[idx]
    _check_cells(xyz, c[idx])
    return xyz


@_case("coord_special_values_cub")
def _():
    v = np.array([x for x, _ in SPECIAL])
    c = np.array([y for _, y in SPECIAL], np.uint32)
    rng = np.random.default_rng(82)
    idx = rng.integers(0, v.size, (300007, 3))
    xyz = v[idx]
    _check_cells(xyz, c[idx])
    assert xyz.shape[0] > R.CAPACITY
    return xyz
