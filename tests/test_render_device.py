"""The colour renderer on the GPU (srl_color_map_render_recent, k_color_render) on the crafted scenes of render_cases: the
device equals the restatement (render_reference) and the oracle after every rendering, with a host image and with an
exact-size device image passed through the C ABI.  The boundary and depth scenes also go through
selectPointsForProjection, which projects with the same project_in_image.  A negative or NaN fov_margin is refused and
leaves the colour state untouched.

A voxel listed twice in the recent list would be fused twice in a row (the `mult > 1` branch of k_color_render), but
addPointsToMap publishes each voxel once (src/lioOptimization.cpp:485-490, 523-549; DESIGN.md section 5), so that branch
cannot be reached through the API and no scene here builds such a list.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle_py as O
from oracle import tracker_oracle as TO

import render_cases as RC
from render_cases import assert_state, bits, padded

pytestmark = pytest.mark.gpu


def _cam(r):
    from sr_livo_b200 import capi
    c = capi.Camera()
    cam15 = r.cam.cam15
    c.q_camera_world[:] = cam15[0:4].tolist(); c.t_camera_world[:] = cam15[4:7].tolist(); c.t_world_camera[:] = cam15[7:10].tolist()
    c.fx, c.fy, c.cx, c.cy, c.fov_margin = cam15[10:15].tolist()
    c.cols, c.rows = r.cam.cols, r.cam.rows
    return c


def _map(ctx, sc):
    from sr_livo_b200 import lio
    cm = lio.ColorVoxelMap(ctx, RC.VOXEL, RC.CAP, 1 << 12, RC.FINE, initial_voxels=64)
    assert cm.addPoints(sc.points, 1, 1.0, 0.0, True) == sc.points.shape[0]
    st = cm.stats()
    assert st["recent"] == st["voxels"]
    return cm


def _render_device_image(cm, r):
    """srl_color_map_render_recent with the image as an exact-size CUDA tensor"""
    import torch
    from sr_livo_b200 import capi
    img = torch.from_numpy(np.ascontiguousarray(r.img)).cuda()
    assert img.numel() == r.cam.rows * r.cam.cols * 3
    n = C.c_int64(0)
    rc = capi.lib().srl_color_map_render_recent(cm.h, C.byref(_cam(r)), C.c_void_p(img.data_ptr()), float(r.obs_time), C.byref(n))
    assert rc == capi.SRL_OK, capi.STATUS_NAMES[rc]
    torch.cuda.synchronize()
    return n.value


@pytest.mark.parametrize("name", list(RC.SCENES))
def test_device_equals_the_restatement_and_the_oracle(name):
    from sr_livo_b200 import lio
    sc = RC.scene(name)
    ctx = lio.Context()
    host, dev = _map(ctx, sc), _map(ctx, sc)
    oc = O.OracleColorMap(voxel_size=RC.VOXEL, max_num_points_in_voxel=RC.CAP, min_distance_points=RC.FINE)
    try:
        assert oc.add_points(sc.points, 1, 1.0, 0.0, True) == sc.points.shape[0]
        for k, r in enumerate(sc.renders):
            assert host.renderPointsInRecentVoxel(_cam(r), r.img, r.obs_time) == sc.counts[k], (name, k)
            assert _render_device_image(dev, r) == sc.counts[k], (name, k)
            assert oc.render(r.cam.cam15, padded(r.img), r.obs_time, rows=r.cam.rows) == sc.counts[k], (name, k)
            g_host, g_dev = host.download(), dev.download()
            assert_state(g_host, sc, k, "device, host image")
            assert_state(g_dev, sc, k, "device, device image")
            assert_state(oc.snapshot(), sc, k, "oracle")
            assert all(bits(g_host[f]) == bits(g_dev[f]) for f in g_host)
    finally:
        host.close(); dev.close(); ctx.close()


@pytest.mark.parametrize("name", RC.PROJECTION_SCENES)
def test_selection_on_the_boundary_and_depth_scenes(name):
    """selectPointsForProjection with every rendering's camera, both candidate modes, against the oracle: key/index and uv bits.
    minimum_depth is 0 so the depth scene's points (distance ~0.001) reach the pcz cut."""
    from sr_livo_b200 import lio
    sc = RC.scene(name)
    ctx = lio.Context()
    cm = _map(ctx, sc)
    oc = TO.OracleColorMap(voxel_size=RC.VOXEL, max_num_points_in_voxel=RC.CAP, min_distance_points=RC.FINE)
    try:
        assert oc.add_points(sc.points, 1, 1.0, 0.0, True) == sc.points.shape[0]
        total = 0
        for r in sc.renders:
            for use_all in (False, True):
                for md in (1.0, 5.0):
                    kw = dict(minimum_dis=md, use_all_points=use_all, minimum_depth=0.0)
                    ids, _, uv = cm.selectPointsForProjection(_cam(r), **kw)
                    ki_o, uv_o = oc.select(r.cam.cam15, r.cam.rows, r.cam.cols, **kw)
                    assert np.array_equal(cm.gatherPoints(ids)["key_index"], ki_o), (name, kw)
                    assert bits(uv) == bits(uv_o), (name, kw)
                    total += ids.shape[0]
        assert total > 0
    finally:
        cm.close(); ctx.close()


@pytest.mark.parametrize("fov", [-0.4, -1e-300, float("nan")])
def test_negative_or_nan_margin_is_refused_and_the_state_is_untouched(fov):
    from sr_livo_b200 import capi, lio
    sc = RC.scene("gate")
    ctx = lio.Context()
    cm = _map(ctx, sc)
    try:
        r0 = sc.renders[0]
        assert cm.renderPointsInRecentVoxel(_cam(r0), r0.img, r0.obs_time) == sc.counts[0]
        before = {f: bits(v) for f, v in cm.download().items()}
        c = _cam(r0)
        c.fov_margin = fov
        with pytest.raises(capi.SrlError) as e:
            cm.renderPointsInRecentVoxel(c, r0.img, r0.obs_time + 1.0)
        assert e.value.code == capi.SRL_BAD_ARG
        n = C.c_int64(-5)
        img = np.ascontiguousarray(r0.img)
        assert capi.lib().srl_color_map_render_recent(cm.h, C.byref(c), img.ctypes.data, r0.obs_time + 1.0, C.byref(n)) == capi.SRL_BAD_ARG
        assert {f: bits(v) for f, v in cm.download().items()} == before
        # the selection still takes the margin when it is a number (it reads no image)
        if fov == fov:
            cm.selectPointsForProjection(c)
        r1 = sc.renders[1]
        assert cm.renderPointsInRecentVoxel(_cam(r1), r1.img, r1.obs_time) == sc.counts[1]
    finally:
        cm.close(); ctx.close()
