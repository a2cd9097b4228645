"""The restatement of cloudProcessing and of libstdc++'s std::sort (tests/cloud_processing_ref.py) pinned against this compiler's
std::sort (oracle/_ref/libsrl_sort_probe.so) and against the reference's own handlers compiled unmodified
(oracle/_ref/libsrl_cloud_processing_ref.so), bit for bit.  CPU only."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cloud_processing_ref as R  # noqa: E402

need_probe = pytest.mark.skipif(not R.have_probe(), reason="oracle/_ref/libsrl_sort_probe.so not built")
need_ref = pytest.mark.skipif(not R.have_reference(), reason="oracle/_ref/libsrl_cloud_processing_ref.so not built")

SIZES = list(range(0, 41)) + [n + d for p in (6, 7, 8, 9, 10, 11, 12) for n in (1 << p,) for d in (-1, 0, 1)]


def key_sets(n, rng):
    yield "random", rng.random(n)
    yield "few", rng.integers(0, 4, n).astype(float)
    yield "equal", np.zeros(n)
    yield "ties16", np.repeat(rng.permutation(n // 16 + 1), 16)[:n].astype(float)
    yield "ties128", np.repeat(rng.permutation(n // 128 + 1), 128)[:n].astype(float)
    yield "sorted", np.arange(n, dtype=float)
    yield "reversed", np.arange(n, dtype=float)[::-1].copy()
    yield "organ", np.concatenate([np.arange(n // 2), np.arange(n - n // 2)[::-1]]).astype(float)


@need_probe
@pytest.mark.parametrize("n", SIZES)
def test_introsort_equals_std_sort(n):
    P = R.SortProbe()
    rng = np.random.default_rng(n)
    for kind, keys in key_sets(n, rng):
        want = P.perm(keys, np.float64)
        assert np.array_equal(R.introsort(list(keys)), want), kind
        assert np.array_equal(R.introsort(list(keys), partition="scan"), want), kind


@need_probe
@pytest.mark.parametrize("dtype", [np.float32, np.uint32])
def test_introsort_equals_std_sort_on_the_narrow_key_types(dtype):
    P = R.SortProbe()
    rng = np.random.default_rng(7)
    for n in (17, 100, 1000, 5000):
        keys = np.repeat(rng.integers(0, 1 << 20, n // 16 + 1), 16)[:n].astype(dtype)
        assert np.array_equal(R.introsort([float(k) for k in keys]), P.perm(keys, dtype))


@need_probe
@pytest.mark.parametrize("n", [200, 1000, 3000])
def test_median_of_3_killer_takes_the_heapsort_fallback(n):
    keys = R.median_of_3_killer(n)
    perm, heapsorts = R.introsort(list(keys), return_heapsorts=True)
    assert heapsorts >= 1
    assert np.array_equal(perm, R.SortProbe().perm(keys, np.float64))
    assert np.array_equal(R.introsort(list(keys), partition="scan"), perm)


def test_scan_partition_equals_the_sequential_loop():
    rng = np.random.default_rng(3)
    for trial in range(300):
        n = int(rng.integers(17, 200))
        keys = rng.integers(0, int(rng.integers(1, 20)), n).astype(float)
        s1 = R._Sorter([(k, i) for i, k in enumerate(keys)])
        s2 = R._Sorter([(k, i) for i, k in enumerate(keys)], partition="scan")
        for s in (s1, s2):
            s.move_median_to_first(0, 1, n // 2, n - 1)
        c1 = s1._partition_seq(1, n, 0)
        c2 = s2._partition_scan(1, n, 0)
        assert c1 == c2 and s1.a == s2.a, trial


def _same(ref, me):
    xyz, rel, ts = ref.drain()
    gx, gr, gt = R.as_arrays(me.queue)
    me.queue = []
    assert len(gt) == len(ts)
    for a, b in ((gx, xyz), (gr, rel), (gt, ts)):
        assert np.array_equal(a.view(np.int64), b.view(np.int64))
    le, given, sweep_id, interval = ref.state()
    assert le == me.last_end_time and sweep_id == me.sweep_id and interval == me.getSweepInterval()
    return given


@need_ref
@pytest.mark.parametrize("name", list(R.SCENES))
def test_handlers_equal_the_reference(name):
    lt, ns, rate, tu, blind, f, _ = R.SCENES[name]
    ref, me = R.ReferenceCP(lt, ns, rate, tu, blind, f), R.CloudProcessingRef(lt, ns, rate, tu, blind, f)
    for kind, msg, stamp in R.scene_messages(name):
        if kind == "livox":
            ref.livox(msg, stamp), me.livoxHandler(msg, stamp)
        else:
            ref.process(msg, stamp), me.process(msg, stamp)
        given = _same(ref, me)
        if kind == "cloud":
            assert given == me.given_offset_time
    ref.close()


@need_ref
@pytest.mark.parametrize("f,blind", [(1, 0.1), (4, 0.1), (1, 4.0), (4, 4.0)])
def test_livox_gates(f, blind):
    """duplicates next to filtered records, x at 0.7 and 2.0, |coord| around 1e8 and past 2^31 (IS_VALID's abs is the float one)"""
    ref, me = R.ReferenceCP(R.LIVOX, 6, 10, R.NS, blind, f), R.CloudProcessingRef(R.LIVOX, 6, 10, R.NS, blind, f)
    for m in range(6):
        rec = R.livox_records(100 + m, 1500, dup_every=3, big=True)
        ref.livox(rec, 1.7e9 + 0.1 * m), me.livoxHandler(rec, 1.7e9 + 0.1 * m)
        _same(ref, me)
    ref.close()


@need_ref
@pytest.mark.parametrize("lt", [R.VELO, R.OUST, R.ROBO])
@pytest.mark.parametrize("given", [True, False])
@pytest.mark.parametrize("f,blind", [(1, 0.1), (4, 4.0)])
def test_cloud_handlers_over_five_messages(lt, given, f, blind):
    tu = R.SEC if lt == R.ROBO else R.NS
    ref, me = R.ReferenceCP(lt, 32, 10, tu, blind, f), R.CloudProcessingRef(lt, 32, 10, tu, blind, f)
    for m in range(5):
        c = R.cloud2(lt, 200 + m, 32, 64, given=given, scan_rate=10)
        ref.process(c, 1.7e9 + 0.1 * m), me.process(c, 1.7e9 + 0.1 * m)
        _same(ref, me)
    ref.close()


def test_cut_stops_at_the_first_later_timestamp():
    me = R.CloudProcessingRef(R.OUST, 16, 20, R.NS, 0.1, 1)
    me.process(R.cloud2(R.OUST, 1, 16, 32), 1.7e9)
    ts = np.array([q[4] for q in me.queue])
    t = ts[40]   # inside a 16-way tie
    popped = me.cut(t)
    assert len(popped) == int(np.argmax(ts >= t)) and all(p[4] < t for p in popped)
    assert me.cut(np.inf) and me.cut(np.inf) == []
