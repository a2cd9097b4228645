"""buildFrame's models on the CPU (tests/build_frame_model.py):

- the numpy std::shuffle equals the standard library's compiled std::shuffle (oracle/srl_shuffle_probe.cpp) for both draw
  rules: permutations and the engine's next output, two shuffles in a row on one engine, n = 0 .. 2^17 + 1;
- forced rejections: replayed word streams whose chosen words the draw rejects;
- the parallel resolution equals a sequential Fisher-Yates on the same swap targets;
- the oracle's buildFrame equals the reference's own buildFrame (oracle/_ref/libsrl_build_frame_ref.so) bit for bit.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import pytest

import build_frame_model as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBES = {0: os.path.join(ROOT, "oracle", "_ref", "libsrl_shuffle_probe.so"),
          1: os.path.join(ROOT, "oracle", "_ref", "libsrl_shuffle_probe_div.so")}
SIZES = [0, 1, 2, 3, 4, 5, 6, 7, 8, 31, 100, 101, 1000, 4097, 65536, (1 << 17), (1 << 17) + 1]
_probes = {}


def probe(rule):
    if rule not in _probes:
        if not os.path.exists(PROBES[rule]):
            pytest.skip(f"{PROBES[rule]} not built (make -C oracle)")
        L = C.CDLL(PROBES[rule])
        L.probe_int128.restype = C.c_int32
        L.probe_shuffle_mt.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
        L.probe_shuffle_mt.restype = C.c_uint64
        L.probe_shuffle_replay.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p]
        L.probe_shuffle_replay.restype = C.c_int64
        assert L.probe_int128() == (1 if rule == 0 else 0)
        _probes[rule] = L
    return _probes[rule]


def probe_mt(rule, sizes):
    sizes = np.ascontiguousarray(sizes, np.int64)
    out = np.zeros(int(sizes.sum()), np.int32)
    nxt = probe(rule).probe_shuffle_mt(sizes.ctypes.data, len(sizes), out.ctypes.data)
    return np.split(out, np.cumsum(sizes)[:-1]), int(nxt)


def probe_replay(rule, words, n):
    w = np.ascontiguousarray(words, np.uint64)
    out = np.zeros(n, np.int32)
    used = probe(rule).probe_shuffle_replay(w.ctypes.data, w.shape[0], n, out.ctypes.data)
    return out, int(used)


@pytest.mark.parametrize("rule", [0, 1])
@pytest.mark.parametrize("n", SIZES)
def test_model_shuffle_equals_compiled_shuffle(rule, n):
    # two shuffles on one engine, as buildFrame's: n, then a smaller second one
    m = n // 3
    perms, nxt = probe_mt(rule, [n, m])
    words = M.mt19937_64(M.num_draws(n) + M.num_draws(m) + 64)
    p1, pos = M.shuffle(n, words, 0, rule)
    p2, pos = M.shuffle(m, words, pos, rule)
    assert np.array_equal(p1, perms[0]) and np.array_equal(p2, perms[1])
    assert int(words[pos]) == nxt


def test_the_two_rules_differ():
    n = 100001
    assert not np.array_equal(probe_mt(0, [n])[0][0], probe_mt(1, [n])[0][0])


def _rejected_word(rule, r):
    # Lemire: low 64 bits of w * r below (2^64 - r) % r (w = 0 whenever r is no power of two); division: w >= r * floor(max / r)
    return 0 if rule == 0 else M.MASK


@pytest.mark.parametrize("rule", [0, 1])
@pytest.mark.parametrize("n", [5, 6, 101, 1000])
def test_forced_rejections(rule, n):
    rng = np.random.default_rng(n + 10 * rule)
    D = M.num_draws(n)
    pool = np.arange(1 if n % 2 == 0 else 0, D)   # (the draw in [0, 2) has a power-of-two range: Lemire never rejects it)
    chosen = sorted(rng.choice(pool, size=min(3, pool.size), replace=False).tolist())
    words, rejected = [], 0
    for d in range(D):
        if d in chosen:
            i = (2 * d if n % 2 == 0 else 2 * d + 1)
            r = (i + 1) * (i + 2)
            for _ in range(1 + (d == chosen[0])):     # the first chosen draw is rejected twice in a row
                words.append(_rejected_word(rule, r)); rejected += 1
        words.append(int(rng.integers(0, 1 << 63)) * 2 + 1)
    words += [12345] * 4
    words = np.array(words, np.uint64)
    want, used = probe_replay(rule, words, n)
    got, pos = M.shuffle(n, words, 0, rule)
    assert used == pos == D + rejected
    assert np.array_equal(got, want)


@pytest.mark.parametrize("n", [0, 1, 2, 3, 10, 257, 4096, 4097, 20001])
def test_parallel_resolution_equals_sequential_fisher_yates(n):
    rng = np.random.default_rng(n)
    for trial in range(4):
        if trial == 0:
            j = M.shuffle_targets(n, M.mt19937_64(M.num_draws(n) + 8))[0]
        elif trial == 1:
            j = np.zeros(n, np.int64)                               # every step swaps with position 0
        elif trial == 2:
            j = np.arange(n)                                        # every step a self-swap
        else:
            j = np.array([rng.integers(0, k + 1) if k else 0 for k in range(n)], np.int64)
        assert np.array_equal(M.resolve(j), M.fisher_yates(j)), trial


needs_ref = pytest.mark.skipif(not M.reference_available(), reason="oracle/_ref/libsrl_build_frame_ref.so not built (needs the reference tree)")
FIELDS = ("raw_point", "point", "imu_point", "relative_time", "alpha_time", "timestamp")


def reference_frame(R, c):
    return R.build_frame(c)


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))


@needs_ref
@pytest.mark.parametrize("case", M.cases(), ids=lambda c: c["name"])
def test_oracle_build_frame_equals_the_reference(case):
    R = M.ReferenceBuildFrame()
    ref = reference_frame(R, case)
    o = M.build_frame(case)
    assert np.array_equal(o["source_index"], ref["source_index"])
    for k in FIELDS:
        assert same_bits(np.ascontiguousarray(o[k], np.float64), ref[k]), k
    end = case["begin"] + case["offset"]
    sc = ref["scalars"]
    assert sc["time_sweep_begin"] == case["begin"] and sc["time_sweep_end"] == end and sc["offset_end"] == case["offset"]
    dt = 0.0
    if case["index_frame"] > 1:
        dt -= case["begin"] - case["prev_time_sweep_end"]
    assert sc["dt_offset"] == dt


@needs_ref
def test_cases_reach_the_branches():
    """The cases exercise what they are named for (against the reference, so the claim does not rest on the model)."""
    R = M.ReferenceBuildFrame()
    by = {c["name"]: c for c in M.cases()}
    c = by["no_time_const_f5"]
    ref = reference_frame(R, dict(c, voxel_size=0.0))
    end = c["begin"] + c["offset"]
    inside = (c["ts"] >= c["begin"]) & (c["ts"] <= end)
    assert sorted(ref["source_index"].tolist()) == np.flatnonzero(inside).tolist()     # erase, both boundaries kept
    assert (c["ts"] == c["begin"]).any() and (c["ts"] == end).any() and (~inside).any()
    c = by["alpha_clamp"]
    ref = reference_frame(R, dict(c, voxel_size=0.0))
    assert (ref["alpha_time"] == 1.0 - 1e-5).any()
    c = by["imu_walk_stops_early"]
    ref = reference_frame(R, dict(c, voxel_size=0.0))
    zero = (ref["imu_point"] == 0.0).all(axis=1)
    assert zero.any() and (~zero).any()
    c = by["frame25_steady_size"]
    assert len(reference_frame(R, c)["source_index"]) < len(reference_frame(R, dict(c, index_frame=3))["source_index"])
