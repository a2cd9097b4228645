"""buildFrame's edge cases on the CPU: the numpy model (tests/build_frame_model.build_frame) equals the reference's own
buildFrame (ref_build_frame in oracle/_ref/libsrl_build_frame_ref.so) on every case of tests/build_frame_edge_cases.py:

- the source-index sequence (the erase, both shuffles, the cells);
- relative_time, alpha_time, timestamp, the points and the cloudFrame scalars bit for bit, NaN compared by position;
- on one engine-rejection frame per rule, shuffle 1 really rejects at the listed draw (checked with the plain scalar draw), and the
  words consumed are the draws of both shuffles plus the rejected ones.  The reference is built with __int128 (rule 0): at
  the rule-1 sizes it is compared under rule 0, and the rule-1 shuffles are held to the model, which
  tests/test_build_frame_model.py pins to the compiled std::shuffle without __int128.  The other rejection frames take about
  half a minute each on one CPU thread; the device file compares all of them with the reference.
"""
from __future__ import annotations

import numpy as np
import pytest

import build_frame_edge_cases as E
import build_frame_model as M

pytestmark = pytest.mark.skipif(not M.reference_available(), reason="oracle/_ref/libsrl_build_frame_ref.so not built (needs the reference tree)")
FIELDS = ("raw_point", "point", "imu_point", "relative_time", "alpha_time", "timestamp")


def same_bits(a, b) -> bool:
    """Equal shapes, NaN at the same entries, every other entry bit for bit."""
    a, b = np.ascontiguousarray(a, np.float64), np.ascontiguousarray(b, np.float64)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint64), b[~nb].view(np.uint64))


def check_equal(o, ref, c):
    assert np.array_equal(o["source_index"], ref["source_index"])
    for k in FIELDS:
        assert same_bits(o[k], ref[k]), k
    sc, end = ref["scalars"], c["begin"] + c["offset"]
    assert (sc["time_sweep_begin"], sc["time_sweep_end"], sc["time_frame_begin"], sc["time_frame_end"]) == (c["begin"], end, c["begin"], end)
    assert (sc["offset_begin"], sc["offset_end"]) == (0.0, c["offset"])
    assert sc["dt_offset"] == (-(c["begin"] - c["prev_time_sweep_end"]) if c["index_frame"] > 1 else 0.0)


def check_rejection(o, c, rule):
    """Shuffle 1 rejects first at c["first_rejection"] under c["rule"]; the words are D1 + D2 + rejections."""
    rej1, rej2 = o["rejected"]
    n1, m = o["n_timestamped"], len(o["source_index"])
    D1, D2 = M.num_draws(n1), (M.num_draws(m) if c["voxel_size"] > 0 else 0)
    assert o["engine_words"] == D1 + D2 + len(rej1) + len(rej2)
    print(f"{c['name']} rule {rule}: n {n1}, shuffle 1 draws {D1}, rejected {rej1}, shuffle 2 draws {D2}, rejected {rej2}, "
          f"engine words {o['engine_words']}")
    if rule != c["rule"]:
        return
    assert rej1 and rej1[0] == c["first_rejection"]
    words = M.mt19937_64(D1 + 16)
    d = rej1[0]
    i = 2 * d + (n1 % 2)
    rng = 2 if (n1 % 2 == 0 and d == 0) else (i + 1) * (i + 2)
    # the plain draw takes word d + 1 for draw d: word d fails its test
    assert M.draw(words, d, rng, rule)[1] == d + 2


@pytest.mark.parametrize("rule", [0, 1])
@pytest.mark.parametrize("n", [0, 1, 2, 3, 6, 7, 101, 4097, 20001])
def test_array_shuffle_equals_the_sequential_model(n, rule):
    """shuffle_fast (which build_frame uses) against the sequential shuffle, on the engine and with rejected words forced at
    the first draw, twice in a row in the middle and at the last draw."""
    D = M.num_draws(n)
    words = M.mt19937_64(D + 64)
    streams = [(words, [])]
    if D >= 3:
        at = sorted({1 if n % 2 == 0 else 0, D // 2, D - 1})
        forced = words.copy()
        for d in reversed(at):
            forced = np.insert(forced, d, [np.uint64(0 if rule == 0 else M.MASK)] * (2 if d == D // 2 else 1))
        streams.append((forced, sorted(at + [D // 2])))
    for w, rejected in streams:
        start = 0 if rejected else 5   # the engine stream from a later word too
        perm, pos = M.shuffle(n, w, start, rule)
        fast = M.shuffle_fast(n, w, start, rule)
        assert np.array_equal(fast[0], perm) and fast[1] == pos and fast[2] == rejected


@pytest.mark.parametrize("name", ["reject_rule0_odd", "reject_rule1_even"])
def test_array_shuffle_equals_compiled_shuffle_at_rejection_sizes(name):
    """Two shuffles in a row on one default-seeded engine, as buildFrame's, against the compiled std::shuffle of both rules."""
    from test_build_frame_model import probe_mt
    c = E.rejection_case(name)
    n = len(c["ts"])
    m = n // 3
    words = M.mt19937_64(M.num_draws(n) + M.num_draws(m) + 64)
    for rule in (0, 1):
        perms, nxt = probe_mt(rule, [n, m])
        p1, pos, rej = M.shuffle_fast(n, words, 0, rule)
        p2, pos, _ = M.shuffle_fast(m, words, pos, rule)
        assert np.array_equal(p1, perms[0]) and np.array_equal(p2, perms[1]) and int(words[pos]) == nxt
        if rule == c["rule"]:
            assert rej[0] == c["first_rejection"]


@pytest.mark.parametrize("name", ["reject_rule0_odd", "reject_rule1_even"])
def test_rejection_frame_model_equals_the_reference(name):
    c = E.rejection_case(name)
    o = M.build_frame(c, rule=0)
    check_equal(o, M.ReferenceBuildFrame().build_frame(c), c)
    check_rejection(o, c, 0)
    if c["rule"] == 1 and c["voxel_size"] > 0:
        check_rejection(M.build_frame(c, rule=1), c, 1)


@pytest.mark.parametrize("case", E.edge_cases(), ids=lambda c: c["name"])
def test_edge_case_model_equals_the_reference(case):
    check_equal(M.build_frame(case), M.ReferenceBuildFrame().build_frame(case), case)


def test_reuse_sequence_on_one_reference_object():
    R = M.ReferenceBuildFrame()
    for c in E.reuse_sequence():
        check_equal(M.build_frame(c), R.build_frame(c), c)


def test_edge_cases_reach_their_branches():
    """What each case is named for holds in the reference's output, so the claim does not rest on the model."""
    R = M.ReferenceBuildFrame()
    by = {c["name"]: c for c in E.edge_cases()}
    # the initial and steady cells keep different sets at 19 and 20
    assert len(R.build_frame(by["index19"])["source_index"]) != len(R.build_frame(dict(by["index19"], index_frame=20))["source_index"])
    assert len(R.build_frame(by["index20"])["source_index"]) != len(R.build_frame(dict(by["index20"], index_frame=19))["source_index"])
    assert len(R.build_frame(by["erase_all"])["source_index"]) == 0
    for name in ("nan_stamp_pte1_mc1", "nan_stamp_pte0_mc1"):   # both branches keep the NaN stamps
        ref = R.build_frame(dict(by[name], voxel_size=0.0))
        assert sorted(ref["source_index"][np.isnan(ref["timestamp"])].tolist()) == [0, 1000, 1999]
    ref = R.build_frame(dict(by["inf_stamp_pte1"], voxel_size=0.0))
    assert np.isinf(ref["timestamp"]).sum() == 5 and (ref["alpha_time"][ref["timestamp"] == np.inf] == 1.0 - 1e-5).all()
    ref = R.build_frame(dict(by["inf_stamp_pte0"], voxel_size=0.0))
    assert not np.isinf(ref["timestamp"]).any()
    ref = R.build_frame(dict(by["zero_offset_pte1_mc1"], voxel_size=0.0, index_frame=5))
    a = ref["alpha_time"]
    assert np.isnan(a).any() and (a == -np.inf).any() and (a == 1.0 - 1e-5).any()
    c = by["zero_offset_pte0_mc1"]
    ref = R.build_frame(dict(c, voxel_size=0.0))
    assert (ref["timestamp"] == c["begin"]).all() and len(ref["timestamp"]) == 4
    for mc in (1, 0):
        c = by[f"epoch_ends_erase_mc{mc}"]
        ts = R.build_frame(dict(c, voxel_size=0.0))["timestamp"]
        assert (ts == c["begin"]).sum() == 300 and (ts == c["begin"] + c["offset"]).sum() == 300 and len(ts) == 2980
    assert len(by["states4097_mc1"]["states"]) == 4097 and len(by["states4096_mc0"]["states"]) == 4096
