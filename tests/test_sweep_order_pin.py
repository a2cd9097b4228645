"""CPU pins of the sweep-order restatement (tests/sweep_order_reference.py) and of the edge cases built on it.

The numpy restatement is held to a plain per-point one: an explicit floor with C's fmin / fmax rules for NaN operands and
a bit-by-bit interleave, sorted by (key, index).  The cluster geometry is held to a direct count of the keys each warp and
CTA owns.  Building every case asserts the property it claims.
"""
import math

import numpy as np
import pytest

import sweep_order_cases as C
import sweep_order_reference as R


# ---- the per-point restatement -------------------------------------------------------------------------------------------
def c_floor(x):
    if math.isnan(x) or math.isinf(x):
        return x
    return float(math.floor(x))


def c_fmax(a, b):   # C fmax: a NaN operand is dropped
    if math.isnan(a):
        return b
    if math.isnan(b):
        return a
    return a if a > b else b


def c_fmin(a, b):
    if math.isnan(a):
        return b
    if math.isnan(b):
        return a
    return a if a < b else b


def cell_py(x):
    return int(c_fmin(c_fmax(c_floor(float(x)) + 128.0, 0.0), 255.0))


def key_py(p):
    c = [cell_py(v) for v in p]
    k = 0
    for i in range(8):
        for a in range(3):
            k |= ((c[a] >> i) & 1) << (3 * i + a)
    return k


def _sample(name, limit=20000):
    xyz = C.build(name)
    if xyz.shape[0] <= limit:
        return np.arange(xyz.shape[0]), xyz
    idx = np.sort(np.random.default_rng(len(name)).choice(xyz.shape[0], limit, replace=False))
    return idx, xyz[idx]


@pytest.mark.parametrize("name", C.names())
def test_case_builds_with_its_property(name):
    xyz = C.build(name)
    assert xyz.shape[0] >= 1


@pytest.mark.parametrize("name", C.names())
def test_numpy_keys_are_the_per_point_keys(name):
    idx, xyz = _sample(name)
    got = R.keys(xyz)
    assert got.dtype == np.uint32
    want = np.array([key_py(p) for p in xyz.tolist()], np.uint32)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, (idx[bad[:5]], xyz[bad[:5]], got[bad[:5]], want[bad[:5]])


@pytest.mark.parametrize("name", [n for n in C.names() if C.build(n).shape[0] <= 140000])
def test_numpy_order_is_the_order_of_key_and_index(name):
    xyz = C.build(name)
    k = R.keys(xyz).tolist()
    want = sorted(range(len(k)), key=lambda i: (k[i], i))
    assert np.array_equal(R.order(xyz), np.array(want, np.uint32))


def test_cells_at_the_named_values():
    for x, cell in C.SPECIAL:
        assert cell_py(x) == cell, x
        assert R.cells(np.array([[x, x, x]]))[0].tolist() == [cell] * 3, x
    v, c = C.ulp_neighbours()
    assert [cell_py(x) for x in v] == c.tolist()


def test_nan_payloads_and_signs_are_what_the_cases_say():
    bits = np.array([C.NAN_PAYLOAD, C.NAN_NEG_PAYLOAD, C.NAN_NEG]).view(np.uint64)
    assert all(math.isnan(x) for x in (C.NAN_PAYLOAD, C.NAN_NEG_PAYLOAD, C.NAN_NEG))
    assert bits[0] == 0x7FF00000DEADBEEF and bits[1] >> 63 == 1 and bits[2] >> 63 == 1
    assert np.array([np.nan]).view(np.uint64)[0] not in bits[:2]   # not the default NaN
    assert C.TINY > 0 and C.TINY / 2 == 0.0
    assert float(2 ** 53 + 1) == 2.0 ** 53


def test_morton_inverse_and_points_for_keys():
    rng = np.random.default_rng(3)
    k = np.concatenate([rng.integers(0, 1 << 24, 100000, dtype=np.uint32), np.array([0, 0xFFFFFF, 0x924924, 0x492492, 0x249249], np.uint32)])
    assert np.array_equal(R.morton(R.unmorton(k)), k)
    assert np.array_equal(R.keys(R.points_for_keys(k, rng)), k)
    for frac in (0.0, np.nextafter(1.0, 0.0), 0.5):   # fractions at both ends of the cell
        assert np.array_equal(R.keys(R.points_for_keys(k, rng, frac=np.full((k.size, 3), frac))), k)
    c = R.unmorton(k)
    for j in range(0, k.size, 997):
        assert key_py(c[j].astype(np.float64) - 128.0) == k[j]


def test_pass_inputs_are_a_plain_lsd_sort():
    rng = np.random.default_rng(4)
    k = rng.integers(0, 1 << 24, 3000, dtype=np.uint32)
    k[::7] = k[3]
    seq = R.pass_inputs(k)
    cur = k.tolist()
    for p in range(3):
        assert seq[p].tolist() == cur
        buckets = [[] for _ in range(256)]
        for x in cur:
            buckets[(x >> (8 * p)) & 255].append(x)
        cur = [x for b in buckets for x in b]
    assert cur == sorted(k.tolist())


@pytest.mark.parametrize("n", sorted(set([s for s in C.SIZES if s <= R.CAPACITY] + list(range(1, 2000, 37)) + [R.CAPACITY - 31, 114688, 114689])))
def test_geometry_is_a_direct_count(n):
    g = R.geometry(n)
    per = g["per"]
    # the least multiple of 32 that lets 16 x 32 warps hold n keys, at most 8 rounds
    assert per % 32 == 0 and 512 * per >= n and (per == 32 or 512 * (per - 32) < n) and per <= 256
    warp = np.arange(n) // per
    per_warp = np.bincount(warp, minlength=512)
    per_cta = np.bincount(warp // 32, minlength=16)
    assert per_warp.size == 512 and per_cta.size == 16
    assert np.array_equal(g["end"] - g["begin"], per_warp)
    assert np.array_equal(g["cta_n"], per_cta)
    # every warp's range is consecutive and starts where the previous one ended
    assert g["begin"][0] == 0 and np.array_equal(g["begin"][1:], g["end"][:-1]) and g["end"][-1] == n
