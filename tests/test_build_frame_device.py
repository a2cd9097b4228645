"""srl_build_frame (srl_frame.cu) against the reference's own buildFrame (oracle/_ref/libsrl_build_frame_ref.so) and the shuffle
models (tests/build_frame_model.py):

- every discrete decision equals the reference's: the source-index sequence covers the erase, both shuffles, the cells and
  the tr1 order; relative_time, alpha_time and timestamp are bit for bit, the points bit for bit or within 1e-11 m where
  the undistortion calls libm (slerp, so3ToQuat);
- the device permutation equals the models for both draw rules, on the engine and on replayed streams with rejections;
- three frames built on the GPU and inserted through srl_map_insert_device give the reference's voxel_map, and frame 3's
  keypoints are the reference's.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import build_frame_model as M
from oracle import reference_py as Rf

needs_ref = pytest.mark.skipif(not M.reference_available(), reason="oracle/_ref/libsrl_build_frame_ref.so not built (needs the reference tree)")
XYZ = ("raw_point", "point", "imu_point")
SCALAR = ("relative_time", "alpha_time", "timestamp")


@pytest.fixture(scope="module")
def L():
    from sr_livo_b200 import lio
    L = lio.LioOptimization(max_voxels=1 << 16, sweep_capacity=8192)
    yield L
    L.close()


def gpu_frame(L, c, frame=None):
    L.R_imu_lidar, L.t_imu_lidar = np.asarray(c["R_il"], float), np.asarray(c["t_il"], float)
    return L.buildFrame(c["raw"], c["ts"], M.capi_imu_states(c["states"]), c["begin"], c["offset"], c["index_frame"], c["q_pred"], c["t_pred"],
                        c["point_time_enable"], c["motion_compensation"], c["init_num_frames"], c["init_voxel_size"], c["voxel_size"],
                        c["prev_time_sweep_end"], frame=frame)


def ref_frame(R, c):
    return R.build_frame(c)


@needs_ref
@pytest.mark.gpu
@pytest.mark.parametrize("case", M.cases(), ids=lambda c: c["name"])
def test_device_build_frame_equals_the_reference(L, case):
    R = M.ReferenceBuildFrame()
    ref = ref_frame(R, case)
    f = gpu_frame(L, case)
    g = f.download()
    assert np.array_equal(g["source_index"], ref["source_index"])
    for k in SCALAR:
        assert np.array_equal(g[k].view(np.uint64), ref[k].view(np.uint64)), k
    for k in XYZ:
        eq = (g[k] == ref[k]).all(axis=1)
        err = np.abs(g[k] - ref[k]).max() if g[k].size else 0.0
        print(f"{case['name']} {k}: {int(eq.sum())}/{eq.size} rows bit for bit, max |diff| {err:.3g} m")
        assert err <= 1e-11, (k, err)
    # transformAllImuPoint and transformPoint call no libm function: given the same imu_point they are bit for bit
    same = (g["imu_point"] == ref["imu_point"]).all(axis=1)
    assert np.array_equal(g["raw_point"][same], ref["raw_point"][same])
    assert np.array_equal(g["point"][same], ref["point"][same])
    info = f.info
    sc = ref["scalars"]
    assert (info.time_sweep_begin, info.time_sweep_end, info.dt_offset, info.offset_end) == \
        (sc["time_sweep_begin"], sc["time_sweep_end"], sc["dt_offset"], sc["offset_end"])
    assert info.n_points == len(ref["source_index"])


def replay(L, words, n, rule):
    from sr_livo_b200 import capi
    perm = np.zeros(max(n, 1), np.uint32)
    used, nxt = C.c_size_t(0), C.c_uint64(0)
    w = None if words is None else np.ascontiguousarray(words, np.uint64)
    rc = capi.lib().srl_shuffle_replay(L.ctx.h, None if w is None else w.ctypes.data, 0 if w is None else w.shape[0], n, rule,
                                       perm.ctypes.data, C.byref(used), C.byref(nxt))
    assert rc == capi.SRL_OK, capi.lib().srl_last_error(L.ctx.h)
    return perm[:n].astype(np.int64), used.value, nxt.value


@pytest.mark.gpu
@pytest.mark.parametrize("on_host", [0, 1])
@pytest.mark.parametrize("rule", [0, 1])
@pytest.mark.parametrize("n", [0, 1, 2, 3, 4, 7, 100, 101, 4097, 100000, (1 << 17) + 1])
def test_device_shuffle_on_the_engine_equals_the_model(L, n, rule, on_host):
    L.ctx.set_option("shuffle_on_host", on_host)
    try:
        perm, used, nxt = replay(L, None, n, rule)
    finally:
        L.ctx.set_option("shuffle_on_host", 0)
    words = M.mt19937_64(M.num_draws(n) + 64)
    want, pos = M.shuffle(n, words, 0, rule)
    assert np.array_equal(perm, want)
    assert used == pos and nxt == int(words[pos])


@pytest.mark.gpu
@pytest.mark.parametrize("on_host", [0, 1])
@pytest.mark.parametrize("rule", [0, 1])
@pytest.mark.parametrize("n", [5, 6, 1001, 100000])
def test_device_shuffle_with_rejections_equals_the_model(L, n, rule, on_host):
    rng = np.random.default_rng(n + rule)
    D = M.num_draws(n)
    words = M.mt19937_64(D + 64).copy()
    # reject draws at the start, in the middle (twice in a row) and at the end: 0 (Lemire) / all ones (division)
    bad = np.uint64(0 if rule == 0 else M.MASK)
    first = 1 if n % 2 == 0 else 0
    at = sorted({first, D // 2, D - 1})
    for d in reversed(at):
        words = np.insert(words, d, [bad] * (2 if d == D // 2 else 1))
    L.ctx.set_option("shuffle_on_host", on_host)
    try:
        perm, used, nxt = replay(L, words, n, rule)
    finally:
        L.ctx.set_option("shuffle_on_host", 0)
    want, pos = M.shuffle(n, words, 0, rule)
    assert pos > D
    assert np.array_equal(perm, want) and used == pos and nxt == int(words[pos])


@needs_ref
@pytest.mark.gpu
def test_shuffle_rule_option(L):
    c = M.make_case("rule1", n=20000, seed=21)
    L.ctx.set_option("shuffle_rule", 1)
    try:
        g = gpu_frame(L, c).download()
    finally:
        L.ctx.set_option("shuffle_rule", 0)
    assert np.array_equal(g["source_index"], M.build_frame(c, rule=1)["source_index"])
    assert not np.array_equal(g["source_index"], M.build_frame(c, rule=0)["source_index"])
    from sr_livo_b200.capi import SRL_BAD_ARG, SrlError
    with pytest.raises(SrlError) as ei:
        L.ctx.set_option("shuffle_rule", 2)
    assert ei.value.code == SRL_BAD_ARG


@pytest.mark.gpu
def test_bad_motion_compensation_is_rejected(L):
    from sr_livo_b200.capi import SRL_BAD_ARG, SrlError
    c = M.make_case("bad", n=10, seed=22, motion_compensation=2)
    with pytest.raises(SrlError) as ei:
        gpu_frame(L, c)
    assert ei.value.code == SRL_BAD_ARG


def _map_dict(keys, counts, xyz):
    return {tuple(k): x[:cnt].copy() for k, cnt, x in zip(keys.tolist(), counts.tolist(), xyz)}


@needs_ref
@pytest.mark.skipif(not Rf.available(), reason="oracle/_ref/libsrl_reference.so not built (needs the reference tree)")
@pytest.mark.gpu
def test_three_frame_stream_map_and_keypoints(L):
    """Frames 1-3 of a stream built on the GPU and chained through the existing entry points by device pointer."""
    from sr_livo_b200 import capi
    R, B = Rf.Reference(), M.ReferenceBuildFrame()   # the reference's map and its buildFrame
    L.voxel_map.clear()
    frame = None
    prev_end = 0.0
    for index_frame in (1, 2, 3):
        c = M.make_case(f"stream{index_frame}", n=30000, seed=40 + index_frame, begin=1.7e9 + 0.1 * index_frame, index_frame=index_frame,
                        scale=30.0)
        c["prev_time_sweep_end"] = prev_end
        frame = gpu_frame(L, c, frame)
        ref = ref_frame(B, c)
        n = len(frame)
        ptrs = frame.device_ptrs()
        assert np.array_equal(frame.download()["source_index"], ref["source_index"])
        if index_frame < 3:
            # stateEstimation's addPointsToMap of frames 1-2 (no optimisation, identity pose)
            added = C.c_int64(0)
            rc = capi.lib().srl_map_insert_device(L.voxel_map.h, C.c_void_p(ptrs["point"]), n, 0.1, 0, C.byref(added))
            assert rc == capi.SRL_OK
            R.add_points_to_map(ref["point"], voxel_size=1.0, max_num_points_in_voxel=20, min_distance_points=0.1, min_num_points=0)
            g = _map_dict(*L.voxel_map.download())
            o = _map_dict(*[R.snapshot()[k] for k in ("keys", "counts", "xyz")])
            assert g.keys() == o.keys()
            bad = [k for k in o if not np.array_equal(g[k].view(np.uint32), o[k].view(np.uint32))]
            assert not bad, bad[:5]
        else:
            # optimize()'s gridSampling of point_frame (src/optimize.cpp:431) at sample_voxel_size 1.5
            out = np.zeros(n, np.uint32)
            m = C.c_size_t(0)
            rc = capi.lib().srl_grid_sampling(L.ctx.h, C.c_void_p(ptrs["point"]), n, 1.5, out.ctypes.data, C.byref(m))
            assert rc == capi.SRL_OK
            want = np.zeros(n, np.int32)
            k = Rf.lib().ref_grid_sampling(ref["point"].ctypes.data, n, 1.5, want.ctypes.data)
            assert np.array_equal(out[:m.value].astype(np.int64), want[:k].astype(np.int64))
        prev_end = frame.info.time_sweep_end
