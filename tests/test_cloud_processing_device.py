"""cloudProcessing on the device (row N10) against the reference's own handlers recorded in tests/golden/cloud_processing.npz,
and the device std::sort against the restated libstdc++ introsort."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cloud_processing_ref as R  # noqa: E402
import build_frame_model as M  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cloud_processing.npz")
GIVEN = [s for s in R.SCENES if "yaw" not in s]
YAW = [s for s in R.SCENES if "yaw" in s]


@pytest.fixture(scope="module")
def ctx():
    from sr_livo_b200 import lio
    c = lio.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def make_cp(ctx, name, capacity=1 << 16):
    from sr_livo_b200 import lio
    lt, ns, rate, tu, blind, f, _ = R.SCENES[name]
    return lio.CloudProcessing(ctx, lt, ns, rate, tu, blind, f, capacity=capacity)


def feed(cp, kind, msg, stamp, on_device):
    import torch
    raw = np.frombuffer(np.ascontiguousarray(msg).tobytes(), np.uint8)
    buf = torch.from_numpy(raw.copy()).cuda() if on_device else raw
    if kind == "livox":
        return cp.livoxHandler(buf, stamp, stride=msg.dtype.itemsize)
    return cp.process(buf, R.cloud_layout(cp.params.lidar_type), stamp)


def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.int64)


@pytest.mark.parametrize("on_device", [False, True])
@pytest.mark.parametrize("name", GIVEN)
def test_given_time_paths_equal_the_reference(ctx, golden, name, on_device):
    cp = make_cp(ctx, name, capacity=256)   # far below one message: the queue grows
    for m, (kind, msg, stamp) in enumerate(R.scene_messages(name)):
        feed(cp, kind, msg, stamp, on_device)
        k = f"{name}/{m}"
        n, xyz, ts = cp.cut(np.inf)
        gx, gr, gt, st = golden[k + "/xyz"], golden[k + "/rel"], golden[k + "/ts"], golden[k + "/state"]
        assert n == len(gt), (m, n, len(gt))
        assert np.array_equal(bits(xyz), bits(gx)) and np.array_equal(bits(ts), bits(gt)), m
        info = cp.info()
        assert info.last_end_time == st[0] and info.sweep_id == (int(st[2]) if kind == "cloud" else 0)
        if kind == "cloud":
            assert bool(info.given_offset_time) == bool(st[1])
    cp.close()


def test_relative_time_and_growth(ctx, golden):
    name = "ouster_given_f1"
    cp = make_cp(ctx, name, capacity=16)
    tot_x, tot_r, tot_t = [], [], []
    for m, (kind, msg, stamp) in enumerate(R.scene_messages(name)):
        feed(cp, kind, msg, stamp, False)
        k = f"{name}/{m}"
        tot_x.append(golden[k + "/xyz"]), tot_r.append(golden[k + "/rel"]), tot_t.append(golden[k + "/ts"])
    xyz, rel, ts = cp.queue()
    assert cp.info().capacity >= len(ts) > 16
    assert np.array_equal(bits(xyz), bits(np.concatenate(tot_x))) and np.array_equal(bits(rel), bits(np.concatenate(tot_r)))
    assert np.array_equal(bits(ts), bits(np.concatenate(tot_t)))
    cp.close()


def test_unaligned_livox_records_with_a_wider_stride(ctx):
    from sr_livo_b200 import lio
    rec = R.livox_records(5, 2000, stride=23)
    ref = R.CloudProcessingRef(R.LIVOX, 6, 10, R.NS, 0.1, 4)
    ref.livoxHandler(rec, 1.7e9)
    cp = lio.CloudProcessing(ctx, **lio.r3live_lidar_params())
    feed(cp, "livox", rec, 1.7e9, True)
    xyz, rel, ts = cp.queue()
    gx, gr, gt = R.as_arrays(ref.queue)
    assert np.array_equal(bits(xyz), bits(gx)) and np.array_equal(bits(rel), bits(gr)) and np.array_equal(bits(ts), bits(gt))
    assert cp.info().last_end_time == ref.last_end_time
    cp.close()


def test_cut_between_equal_timestamps(ctx):
    name = "ouster_given_f1"
    cp = make_cp(ctx, name)
    kind, msg, stamp = R.scene_messages(name)[0]
    feed(cp, kind, msg, stamp, False)
    _, _, ts = cp.queue()
    # a timestamp shared by a column's rings: the cut pops everything strictly before it
    vals, counts = np.unique(ts, return_counts=True)
    t = vals[np.flatnonzero(counts > 1)[len(vals) // 4 if len(vals) > 4 else 0]]
    expect = int(np.argmax(~(ts < t))) if np.any(~(ts < t)) else len(ts)
    n, xyz, got = cp.cut(t)
    assert n == expect and np.array_equal(bits(got), bits(ts[:expect]))
    info = cp.info()
    assert info.size == len(ts) - expect and info.front_timestamp == ts[expect]
    n2, _, _ = cp.cut(np.inf)
    assert n2 == len(ts) - expect and cp.info().size == 0 and np.isnan(cp.info().front_timestamp)
    assert cp.cut(np.inf)[0] == 0   # a cut on an empty queue stops at once
    cp.close()


def test_undefined_cases(ctx):
    from sr_livo_b200 import lio
    from sr_livo_b200.capi import SrlError
    # a Livox message with nothing left: nothing appended, last_end_time kept
    cp = lio.CloudProcessing(ctx, **lio.r3live_lidar_params())
    rec = R.livox_records(1, 50)
    rec["x"] = np.float32(0.5)
    assert cp.livoxHandler(rec, 1.7e9) == 0 and cp.info().last_end_time == -1.0 and cp.info().size == 0
    cp.close()
    # ring >= N_SCANS on the yaw path, NaN time field, NaN xyz on the yaw path: SRL_BAD_ARG, nothing appended, no state change
    for lt, mutate in ((R.OUST, "ring"), (R.VELO, "nan_time"), (R.VELO, "nan_xyz")):
        cp = lio.CloudProcessing(ctx, lt, 16, 10, R.NS, 4.0, 1)
        good = R.cloud2(lt, 3, 16, 64, given=mutate == "nan_time")
        cp.process(np.frombuffer(good.tobytes(), np.uint8), R.cloud_layout(lt), 1.7e9)
        before = cp.info()
        c = R.cloud2(lt, 4, 16, 64, given=mutate == "nan_time")
        if mutate == "ring":
            c["ring"][17] = 16
        elif mutate == "nan_time":
            c["time"][100] = np.nan
        else:
            c["x"][40] = np.nan
        with pytest.raises(SrlError, match="SRL_BAD_ARG"):
            cp.process(np.frombuffer(c.tobytes(), np.uint8), R.cloud_layout(lt), 1.8e9)
        after = cp.info()
        assert (after.size, after.last_end_time, after.sweep_id, after.given_offset_time) == \
            (before.size, before.last_end_time, before.sweep_id, before.given_offset_time)
        cp.close()


# The yaw path runs CUDA's atan2 (within 2 ulp), not glibc's.  An angle error of a few ulp of 180 degrees moves relative_time =
# (yaw_first - yaw) / (0.361 * SCAN_RATE) by about 1e-14 ms; the bound below is 100 times that.  The scenes' distinct keys lie
# more than YAW_MIN_GAP apart (asserted on the restated keys), so the order must be glibc's exactly; the ties (every ring's first
# point at 0) are exact.  Timestamps (relative_time / 1000 + stamp, one ulp ~ 2.4e-7 s at 1.7e9 s) may differ by one rounding.
YAW_REL_ABS = 1e-12   # ms
YAW_MIN_GAP = 1e-10   # ms: 100 times YAW_REL_ABS; two keys each within YAW_REL_ABS cannot swap


@pytest.mark.parametrize("name", YAW)
def test_yaw_path_within_bound(ctx, golden, name):
    cp = make_cp(ctx, name)
    worst_rel, worst_rel_ulp, worst_ts = 0.0, 0, 0
    for m, (kind, msg, stamp) in enumerate(R.scene_messages(name)):
        assert R.yaw_gap_ok(msg, R.SCENES[name][2], YAW_MIN_GAP)
        feed(cp, kind, msg, stamp, False)
        k = f"{name}/{m}"
        xyz, rel, ts = cp.queue()
        assert cp.cut(np.inf)[0] == len(ts)
        gx, gr, gt = golden[k + "/xyz"], golden[k + "/rel"], golden[k + "/ts"]
        assert len(ts) == len(gt)
        assert np.array_equal(bits(xyz), bits(gx)), "order differs"
        if len(ts):
            worst_rel = max(worst_rel, float(np.abs(rel - gr).max()))
            worst_rel_ulp = max(worst_rel_ulp, int(np.abs(bits(rel) - bits(gr)).max()))
            worst_ts = max(worst_ts, int(np.abs(bits(ts) - bits(gt)).max()))
        # the ring-first points: relative_time 0 and timestamp 0 exactly
        assert np.array_equal(gr == 0.0, rel == 0.0) and np.array_equal(gt == 0.0, ts == 0.0)
        assert abs(cp.info().last_end_time - golden[k + "/state"][0]) <= np.spacing(golden[k + "/state"][0])
    print(f"{name}: max |relative_time - glibc's| = {worst_rel:.3g} ms ({worst_rel_ulp} ulp), max timestamp difference {worst_ts} ulp")
    assert worst_rel <= YAW_REL_ABS and worst_ts <= 1
    cp.close()


def test_padded_rows_equal_packed_rows(ctx):
    """PointCloud2 rows row_step bytes apart with padding after width * point_step: the same points as the packed message"""
    from sr_livo_b200 import lio
    lt, rows, cols = R.OUST, 16, 64
    c = R.cloud2(lt, 9, rows, cols)
    step = c.dtype.itemsize
    width, pad = 128, 40
    packed = np.frombuffer(c.tobytes(), np.uint8)
    padded = np.full((len(c) // width, width * step + pad), 0xAB, np.uint8)
    padded[:, :width * step] = packed.reshape(-1, width * step)
    out = []
    for data, extra in ((packed, {}), (padded.reshape(-1), dict(width=width, row_step=width * step + pad))):
        cp = lio.CloudProcessing(ctx, lt, 16, 20, R.NS, 0.1, 1)
        cp.process(data, dict(R.cloud_layout(lt), **extra), 1.7e9)
        out.append(cp.queue())
        cp.close()
    for a, b in zip(*out):
        assert np.array_equal(bits(a), bits(b))
    assert len(out[0][2]) > 0
    cp = lio.CloudProcessing(ctx, lt, 16, 20, R.NS, 0.1, 1)
    from sr_livo_b200.capi import SrlError
    with pytest.raises(SrlError, match="SRL_BAD_ARG"):   # row_step below width * point_step
        cp.process(padded.reshape(-1), dict(R.cloud_layout(lt), width=width, row_step=width * step - 1), 1.7e9)
    cp.close()


@pytest.mark.parametrize("n", [0, 1, 2, 16, 17, 40, 1000, 4097, 70000])
@pytest.mark.parametrize("kind", ["random", "ties128", "equal", "organ"])
def test_device_sort_equals_introsort(ctx, n, kind):
    from sr_livo_b200 import lio
    rng = np.random.default_rng(n)
    keys = {"random": rng.random(n), "ties128": np.repeat(rng.permutation(n // 128 + 1), 128)[:n].astype(float),
            "equal": np.zeros(n), "organ": np.concatenate([np.arange(n // 2), np.arange(n - n // 2)[::-1]]).astype(float)}[kind]
    assert np.array_equal(lio.device_sort_permutation(ctx, keys), R.introsort(list(keys)))


def test_device_sort_heapsort_fallback(ctx):
    from sr_livo_b200 import lio
    keys = R.median_of_3_killer(3000)
    ref, h_ref = R.introsort(list(keys), return_heapsorts=True)
    got, h = lio.device_sort_permutation(ctx, keys, return_heapsorts=True)
    assert h_ref >= 1 and h == h_ref
    assert np.array_equal(got, ref)


def test_cut_chains_into_build_frame(ctx, golden):
    from sr_livo_b200 import lio
    name = "ouster_given_ntu"
    L = lio.LioOptimization(max_voxels=1 << 12, sweep_capacity=1 << 12)
    cp = make_cp(L.ctx, name)
    kind, msg, stamp = R.scene_messages(name)[1]
    feed(cp, kind, msg, stamp, True)
    t_end = stamp + 0.04
    states = [dict(timestamp=stamp, quat=[0, 0, 0, 1], trans=[0, 0, 0], vel=[1, 0, 0], un_acc=[0, 0, 0], un_gyr=[0, 0, 0.1]),
              dict(timestamp=t_end, quat=[0, 0, 0.02, 0.9998], trans=[0.05, 0, 0], vel=[1, 0, 0], un_acc=[0, 0, 0], un_gyr=[0, 0, 0.1])]
    st = M.capi_imu_states(states)
    n, xyz_d, ts_d = cp.cut(t_end, device=True)
    assert n > 0
    xyz_h, ts_h = xyz_d.cpu().numpy(), ts_d.cpu().numpy()
    a = L.buildFrame(xyz_d, ts_d, st, stamp, t_end, 3, point_time_enable=cp.isPointTimeEnable()).download()
    b = L.buildFrame(xyz_h, ts_h, st, stamp, t_end, 3, point_time_enable=cp.isPointTimeEnable()).download()
    for k in a:
        assert np.array_equal(np.asarray(a[k]).view(np.uint8), np.asarray(b[k]).view(np.uint8)), k
    cp.close()
    L.close()
