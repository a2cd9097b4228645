"""Row N4 with blocks of more than 20 points: the colour map on the GPU against the oracle, bit for bit, for capacities 20 to
128 (the shipped map_options use 50 and 100), with wrapped and aliased keys; and the argument checks that keep such maps
out of the LIO path.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle_py as O

from color_map_cases import FINE, SIZE, camera, sweep, voxel_exact_count

pytestmark = pytest.mark.gpu

CAPS = [20, 21, 31, 32, 33, 50, 64, 65, 100, 128]


@pytest.fixture(scope="module")
def ctx():
    from sr_livo_b200 import lio
    c = lio.Context()
    yield c
    c.close()


def _cam(cam15):
    from sr_livo_b200 import capi
    c = capi.Camera()
    c.q_camera_world[:] = cam15[0:4].tolist(); c.t_camera_world[:] = cam15[4:7].tolist(); c.t_world_camera[:] = cam15[7:10].tolist()
    c.fx, c.fy, c.cx, c.cy, c.fov_margin = cam15[10:15].tolist()
    c.cols, c.rows = 640, 480
    return c


def _by_key(d):
    return {tuple(k): i for i, k in enumerate(d["keys"].tolist())}


def _assert_same(cmg, cmo, cap):
    g, o = cmg.download(), cmo.snapshot()
    nv = o["keys"].shape[0]
    assert g["xyz"].shape == (nv, cap, 3) and g["rgb"].shape == (nv, cap, 3) and g["n_rgb"].shape == (nv, cap)
    st, oc = cmg.stats(), cmo.counts()
    assert (st["voxels"], st["rgb_points"], st["recent"], st["new_recent"]) == (oc["voxels"], oc["rgb_points"], oc["recent"], oc["new_recent"])
    assert st["points"] == int(o["counts"].sum())
    o_rgb, o_recent = cmo.lists()
    assert np.array_equal(g["rgb_points"], o_rgb)                    # rgb_points_vec in order, index in block up to cap - 1
    assert np.array_equal(g["recent"].astype(np.int32), o_recent)    # voxels_recent_visited in order
    gi, oi = _by_key(g), _by_key(o)
    assert gi.keys() == oi.keys()
    for k, j in oi.items():
        i = gi[k]
        assert g["counts"][i] == o["counts"][j], k
        for f in ("xyz", "rgb", "n_rgb", "cov", "obs_dist", "last_obs"):
            assert np.array_equal(g[f][i], o[f][j]), (k, f)
        assert g["last_visited"][i] == o["last_visited"][j], k
    return g, o


@pytest.mark.parametrize("cap", CAPS)
def test_color_map_capacity_matches_the_oracle(ctx, cap):
    from sr_livo_b200 import lio
    rng = np.random.default_rng(cap)
    cmg = lio.ColorVoxelMap(ctx, voxel_size=SIZE, max_num_points_in_voxel=cap, max_voxels=1 << 15, min_distance_points=FINE)
    cmo = O.OracleColorMap(voxel_size=SIZE, max_num_points_in_voxel=cap, min_distance_points=FINE)
    try:
        exact = voxel_exact_count(rng, cap)
        s1, s2 = sweep(seed=500 + cap), sweep(seed=600 + cap) + rng.normal(0, 0.003, (1, 3))
        feeds = [(exact, dict(add_point_step=1, time_sweep_end=1.0, time_last_process=0.0, to_rendering=False)),   # recent list kept
                 (s1, dict(add_point_step=1, time_sweep_end=1.1, time_last_process=1.0, to_rendering=True)),       # ... then published
                 (s2, dict(add_point_step=4, time_sweep_end=1.2, time_last_process=1.1, to_rendering=False)),
                 (s1[:5000] + 0.004, dict(add_point_step=1, time_sweep_end=1.3, time_last_process=1.2, to_rendering=True))]
        for n, (pts, kw) in enumerate(feeds):
            assert cmg.addPoints(pts, **kw) == cmo.add_points(pts, **kw)
            if n == 0:                                                     # exactly cap and cap + 1 offered: all full at cap
                g, o = _assert_same(cmg, cmo, cap)
                assert np.all(o["counts"] == cap) and o["counts"].size == 24
                continue
            if kw["to_rendering"]:
                for k, pos in enumerate([(0.0, 0.0, 0.0), (400.0, 0.0, 0.0)]):
                    img = rng.integers(0, 256, (480, 640, 3), dtype=np.uint8)
                    cam15, obs = camera(pos), kw["time_sweep_end"] + 0.01 * (k + 1)
                    assert cmg.renderPointsInRecentVoxel(_cam(cam15), img, obs) == cmo.render(cam15, img, obs)
            g, o = _assert_same(cmg, cmo, cap)
        # the scene reaches what it is meant to: full blocks, colours past point 32, wrapped keys
        assert o["counts"].max() == cap
        full = o["counts"] == cap
        assert (o["n_rgb"][full][:, cap - 1] >= 1).any()                   # the last slot of a full block was rendered
        assert (g["rgb_points"][:, 3] == cap - 1).any()
        assert (np.abs(o["keys"][:, 0].astype(np.int64)) > 3000).any()
        vox = C.c_void_p(lio.lib().srl_color_map_voxels(cmg.h))
        nv, npts = C.c_int64(0), C.c_int64(0)
        assert lio.lib().srl_map_stats(vox, C.byref(nv), C.byref(npts)) == 0
        assert (nv.value, npts.value) == (o["keys"].shape[0], int(o["counts"].sum()))
    finally:
        cmg.close()


def test_keys_past_int32_nan_and_inf_are_dropped(ctx):
    """|x / size| >= 2^31, NaN and +-inf drop the point (the int32 conversion the reference relies on is undefined there);
    everything else is stored as the oracle stores it."""
    from sr_livo_b200 import lio
    rng = np.random.default_rng(3)
    good = sweep(seed=9, n_dense=4000)
    bad = np.array([[3e7, 0.0, 4.0], [0.0, -2.2e7, 4.0], [np.nan, 0.0, 1.0], [np.inf, 0.0, 1.0], [0.0, 0.0, -np.inf]])
    pts = np.concatenate([good[:3000], bad, good[3000:]])
    cmg = lio.ColorVoxelMap(ctx, voxel_size=SIZE, max_num_points_in_voxel=50, max_voxels=1 << 14, min_distance_points=FINE)
    cmo = O.OracleColorMap(voxel_size=SIZE, max_num_points_in_voxel=50, min_distance_points=FINE)
    try:
        kw = dict(add_point_step=1, time_sweep_end=1.0, time_last_process=0.0, to_rendering=True)
        assert cmg.addPoints(pts, **kw) == cmo.add_points(good, **kw)
        _assert_same(cmg, cmo, 50)
        img = rng.integers(0, 256, (480, 640, 3), dtype=np.uint8)
        assert cmg.renderPointsInRecentVoxel(_cam(camera((0.0, 0.0, 0.0))), img, 1.05) == cmo.render(camera((0.0, 0.0, 0.0)), img, 1.05)
        _assert_same(cmg, cmo, 50)
    finally:
        cmg.close()


def _err(ctx):
    from sr_livo_b200 import capi
    return capi.lib().srl_last_error(ctx.h).decode()


def test_color_map_create_rejects_bad_capacities(ctx):
    from sr_livo_b200 import capi
    L = capi.lib()
    h = C.c_void_p()
    for cap, max_voxels in [(0, 1024), (129, 1024), (-5, 1024), (50, 0),
                            (128, 1 << 25),                       # 2^25 * 128 = 2^32 ids: not below 2^32
                            (100, -(-(1 << 32) // 100)),          # the smallest pool whose ids reach 2^32
                            (21, -(-(1 << 32) // 21))]:
        assert L.srl_color_map_create(ctx.h, SIZE, cap, max_voxels, FINE, C.byref(h)) == capi.SRL_BAD_ARG, (cap, max_voxels)
        assert not h.value
        assert "srl_color_map_create" in _err(ctx)
    assert "2^32" in _err(ctx)
    assert L.srl_map_create(ctx.h, 1.0, 21, 1024, C.byref(h)) == capi.SRL_BAD_ARG   # the LIO map keeps its 20-point limit


def _snapshot(cm):
    d = cm.download()
    return {k: v.copy() for k, v in d.items()}, cm.stats()


@pytest.mark.parametrize("cap", [50, 21])
def test_lio_entry_points_reject_wide_blocks_and_leave_the_map_alone(ctx, cap):
    import torch
    from sr_livo_b200 import capi, lio
    L = capi.lib()
    cm = lio.ColorVoxelMap(ctx, voxel_size=SIZE, max_num_points_in_voxel=cap, max_voxels=1 << 12, min_distance_points=FINE)
    sw = lio.Sweep(ctx, 4096)
    comm = C.c_void_p()
    assert L.srl_comm_create(ctx.h, 0, 1, C.byref(comm)) == capi.SRL_OK
    try:
        pts = sweep(seed=11, n_dense=3000)
        cm.addPoints(pts, to_rendering=True)
        before, st_before = _snapshot(cm)
        vox = C.c_void_p(L.srl_color_map_voxels(cm.h))
        xyz = np.ascontiguousarray(pts[:2000])
        sw.upload(xyz)
        dev = torch.from_numpy(xyz).cuda()
        prm = lio.r3live_params(size_voxel_map=SIZE)
        fr = lio.make_frame([0, 0, 0, 1], [0, 0, 0], [0, 0, 0])
        ne = capi.NormalEq()
        st = lio.EskfEstimator().to_c()
        fq, ft, tl = np.array([0.0, 0, 0, 1]), np.zeros(3), np.zeros(3)
        R, ti = np.eye(3).reshape(9).copy(), np.zeros(3)
        summ = capi.IekfSummary()
        d_out = torch.zeros(32, dtype=torch.float64, device="cuda")
        n = C.c_int64(0)
        keys, counts = np.zeros((1, 3), np.int16), np.ones(1, np.int32)
        up_xyz = np.zeros((1, cap, 3), np.float32)
        p = capi.ptr
        calls = {
            "srl_map_insert": lambda: L.srl_map_insert(vox, p(xyz), xyz.shape[0], FINE, 0, C.byref(n)),
            "srl_map_insert_device": lambda: L.srl_map_insert_device(vox, C.c_void_p(dev.data_ptr()), xyz.shape[0], FINE, 0, C.byref(n)),
            "srl_map_insert_sweep": lambda: L.srl_map_insert_sweep(vox, sw.h, p(fq), p(ft), p(R), p(ti), FINE, 0, C.byref(n)),
            "srl_map_upload": lambda: L.srl_map_upload(vox, p(keys), p(counts), p(up_xyz), 1),
            "srl_map_remove_far": lambda: L.srl_map_remove_far(vox, p(np.zeros(3)), 0.5, C.byref(n)),
            "srl_build_plane_residuals": lambda: L.srl_build_plane_residuals(ctx.h, vox, sw.h, C.byref(fr), C.byref(prm), C.byref(ne), None),
            "srl_build_plane_residuals_async": lambda: L.srl_build_plane_residuals_async(ctx.h, vox, sw.h, C.byref(fr), C.byref(prm),
                                                                                          C.c_void_p(d_out.data_ptr())),
            "srl_update_iekf": lambda: L.srl_update_iekf(ctx.h, vox, sw.h, C.byref(st), p(fq), p(ft), p(tl), p(R), p(ti), C.byref(prm), C.byref(summ)),
            "srl_update_iekf_dist": lambda: L.srl_update_iekf_dist(ctx.h, comm, vox, sw.h, C.byref(st), p(fq), p(ft), p(tl), p(R), p(ti),
                                                                   C.byref(prm), C.byref(summ)),
            "srl_optimize_host": lambda: L.srl_optimize_host(ctx.h, vox, sw.h, p(xyz), xyz.shape[0], C.byref(st), p(fq), p(ft), p(tl), p(R), p(ti),
                                                             C.byref(prm), C.byref(summ), None),
            "srl_optimize_host_dist": lambda: L.srl_optimize_host_dist(ctx.h, comm, vox, sw.h, p(xyz), xyz.shape[0], C.byref(st), p(fq), p(ft),
                                                                       p(tl), p(R), p(ti), C.byref(prm), C.byref(summ), None, None, None),
        }
        for name, call in calls.items():
            rc = call()
            assert rc == capi.SRL_BAD_ARG, (name, rc)
            assert _err(ctx) == f"map has {cap} points per block; the LIO path needs 20", name
            after, st_after = _snapshot(cm)
            assert st_after == st_before, name
            for k in before:
                assert np.array_equal(before[k], after[k]), (name, k)
    finally:
        L.srl_comm_destroy(comm)
        sw.close()
        cm.close()


def test_narrow_color_map_still_takes_the_lio_insert(ctx):
    """A colour map of cap <= 20 keeps the LIO block layout and still works with the LIO entry points."""
    from sr_livo_b200 import capi, lio
    L = capi.lib()
    cm = lio.ColorVoxelMap(ctx, voxel_size=SIZE, max_num_points_in_voxel=20, max_voxels=1 << 12, min_distance_points=FINE)
    try:
        vox = C.c_void_p(L.srl_color_map_voxels(cm.h))
        pts = sweep(seed=12, n_dense=2000)                 # 1000 of its points lie past |x / size| = 32768, where keys wrap in
                                                           # both maps as in the reference (DESIGN.md section 5)
        n = C.c_int64(0)
        assert L.srl_map_insert(vox, capi.ptr(np.ascontiguousarray(pts)), pts.shape[0], FINE, 0, C.byref(n)) == capi.SRL_OK
        om = O.OracleMap()
        assert n.value == om.add_points(pts, SIZE, 20, FINE, 0) > 0
    finally:
        cm.close()
