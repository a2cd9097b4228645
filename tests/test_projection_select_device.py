"""selectPointsForProjection on the GPU (srl_color_map_select_for_projection) and the tracker's per-point reads
(srl_color_map_gather_points), against the oracle bit for bit, and against the reference's own compiled code
(oracle/_ref/libsrl_tracker_ref.so) where that library was built.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import tracker_oracle as O

import tracker_ref as TR
from projection_cases import (COLS, FINE, HALVES_CAM, ROWS, SIZE, camera, halves_points, map_sweeps, select_params, ulp_pairs, with_fov)
from publish_cases import render_images

pytestmark = pytest.mark.gpu


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _cam(cam15, rows=ROWS, cols=COLS):
    from sr_livo_b200 import capi
    c = capi.Camera()
    c.q_camera_world[:] = cam15[0:4].tolist(); c.t_camera_world[:] = cam15[4:7].tolist(); c.t_world_camera[:] = cam15[7:10].tolist()
    c.fx, c.fy, c.cx, c.cy, c.fov_margin = cam15[10:15].tolist()
    c.cols, c.rows = cols, rows
    return c


def _fill(cap, sweeps, renders=1, to_rendering=None, with_ref=False, initial_voxels=64, max_voxels=1 << 16):
    from sr_livo_b200 import lio
    ctx = lio.Context()
    cm = lio.ColorVoxelMap(ctx, SIZE, cap, max_voxels, FINE, initial_voxels=initial_voxels)
    oc = O.OracleColorMap(voxel_size=SIZE, max_num_points_in_voxel=cap, min_distance_points=FINE)
    ref = TR.TrackerReference(SIZE, cap, FINE) if with_ref else None
    for s, pts in enumerate(sweeps):
        t_end, t_proc = 1.0 + 0.1 * s, 1.0 * s
        tr = True if to_rendering is None else to_rendering[s]
        cm.addPoints(pts, 1, t_end, t_proc, tr)
        oc.add_points(pts, 1, t_end, t_proc, tr)
        if ref:
            ref.add_points(pts, 1, t_end, t_proc, tr)
        for k, img in enumerate(render_images(100 * cap + s, renders)):
            cam15, obs = camera((0.02 * k, 0.0, 0.0)), t_end + 0.01 * (k + 1)
            n = cm.renderPointsInRecentVoxel(_cam(cam15), img, obs)
            assert n == oc.render(cam15, img, obs)
            if ref:
                assert ref.render(cam15, img, obs) == n
    return ctx, cm, oc, ref


def _check(cm, oc, cam15, ref=None, **kw):
    """device == oracle (and == the compiled reference when given): key/index, uv bits, and xyz = the oracle's stored floats"""
    ids, xyz, uv = cm.selectPointsForProjection(_cam(cam15), **kw)
    ki_o, uv_o = oc.select(cam15, ROWS, COLS, **kw)
    g = cm.gatherPoints(ids)
    assert np.array_equal(g["key_index"], ki_o), kw
    assert np.array_equal(bits(uv), bits(uv_o)), kw
    want = oc.gather(ki_o)
    assert want is not None and np.array_equal(bits(xyz), bits(want["xyz"])), kw
    if ref is not None:
        ki_r, uv_r = ref.select(cam15, ROWS, COLS, **kw)
        assert np.array_equal(ki_r, ki_o) and np.array_equal(bits(uv_r), bits(uv)), kw
    assert cm.countPointsForProjection(_cam(cam15), **kw) == ids.shape[0]
    return ids


@pytest.mark.parametrize("cap", [20, 50, 100])
def test_map_scenes_match_oracle(cap):
    ctx, cm, oc, _ = _fill(cap, map_sweeps(seed=cap), renders=2)
    try:
        assert cm.capacity()["committed_voxels"] > 64
        for _, fov, kw in select_params():
            for pos in ((0.0, 0.0, 0.0), (0.13, -0.07, 0.5)):
                _check(cm, oc, with_fov(camera(pos), fov), **kw)
    finally:
        cm.close(); ctx.close()


def test_empty_recent_list_falls_back_and_halves_and_ulp_pairs():
    sweeps = map_sweeps(seed=3)
    ctx, cm, oc, _ = _fill(50, sweeps, renders=0)
    try:
        cm.addPoints(sweeps[0][:100], 1, 7.0, 7.0, True); oc.add_points(sweeps[0][:100], 1, 7.0, 7.0, True)
        assert cm.stats()["recent"] == oc.num_recent() == 0
        for md in (5.0, 10.0):
            ids = _check(cm, oc, camera((0, 0, 0)), minimum_dis=md)
            assert np.array_equal(ids, cm.selectPointsForProjection(_cam(camera((0, 0, 0))), minimum_dis=md, use_all_points=True)[0])
    finally:
        cm.close(); ctx.close()
    for md in (5.0, 10.0):
        ctx, cm, oc, _ = _fill(50, [halves_points(md)], renders=0)
        try:
            for use_all in (False, True):
                ids, xyz, uv = cm.selectPointsForProjection(_cam(HALVES_CAM), minimum_dis=md, use_all_points=use_all)
                ki_o, uv_o = oc.select(HALVES_CAM, ROWS, COLS, minimum_dis=md, use_all_points=use_all)
                assert np.array_equal(cm.gatherPoints(ids)["key_index"], ki_o) and np.array_equal(bits(uv), bits(uv_o))
                assert (uv[:, 0] < 0).any()
        finally:
            cm.close(); ctx.close()
    for reverse in (False, True):
        ctx, cm, oc, _ = _fill(50, [ulp_pairs(seed=21 + reverse, n=12, reverse=reverse)], renders=0)
        try:
            for md in (10.0, 40.0 / 1.5):
                for use_all in (False, True):
                    _check(cm, oc, camera((0, 0, 0)), minimum_dis=md, use_all_points=use_all)
        finally:
            cm.close(); ctx.close()


def test_recent_list_after_sweeps_without_rendering():
    sweeps = map_sweeps(seed=8)
    ctx, cm, oc, _ = _fill(50, [sweeps[0], sweeps[1], sweeps[0][::2] + 0.002], renders=1, to_rendering=[False, False, True])
    try:
        for md in (5.0, 10.0, 40.0 / 1.5):
            _check(cm, oc, with_fov(camera((0, 0, 0)), -0.4), minimum_dis=md)
    finally:
        cm.close(); ctx.close()


def _snapshot(cm):
    d = cm.download()
    return {k: bits(v).tobytes() for k, v in d.items()}, cm.stats()


def test_outputs_host_device_count_and_the_map_is_untouched():
    import torch
    ctx, cm, oc, _ = _fill(50, map_sweeps(seed=5), renders=2)
    try:
        cam = _cam(with_fov(camera((0, 0, 0)), -0.4))
        before = _snapshot(cm)
        ids, xyz, uv = cm.selectPointsForProjection(cam, minimum_dis=10.0)
        n = ids.shape[0]
        assert n > 0 and cm.countPointsForProjection(cam, minimum_dis=10.0) == n
        d = (torch.empty(n + 5, dtype=torch.int32, device="cuda"), torch.empty((n + 5, 3), dtype=torch.float32, device="cuda"),
             torch.empty((n + 5, 2), dtype=torch.float32, device="cuda"))
        gi, gx, gu = cm.selectPointsForProjection(cam, minimum_dis=10.0, out=d)
        assert gi.is_cuda and np.array_equal(gi.cpu().numpy().view(np.uint32), ids)
        assert np.array_equal(bits(gx.cpu().numpy()), bits(xyz)) and np.array_equal(bits(gu.cpu().numpy()), bits(uv))
        pinned = (torch.empty(n, dtype=torch.int32).pin_memory(), None, torch.empty((n, 2), dtype=torch.float32).pin_memory())
        pi, px, pu = cm.selectPointsForProjection(cam, minimum_dis=10.0, out=pinned)
        assert px is None and np.array_equal(pi.numpy().view(np.uint32), ids) and np.array_equal(bits(pu.numpy()), bits(uv))
        mixed = (None, torch.empty((n, 3), dtype=torch.float32, device="cuda"), np.empty((n, 2), np.float32))
        _, mx, mu = cm.selectPointsForProjection(cam, minimum_dis=10.0, out=mixed)
        assert np.array_equal(bits(mx.cpu().numpy()), bits(xyz)) and np.array_equal(bits(mu), bits(uv))
        # gather by device ids
        g_dev = cm.gatherPoints(gi)
        g_host = cm.gatherPoints(ids)
        assert all(np.array_equal(bits(g_dev[k]), bits(g_host[k])) for k in g_host)
        # max_points too small: SRL_BAD_ARG and nothing written
        from sr_livo_b200 import capi
        small = (np.full(n - 1, 0xABCDABCD, np.uint32), np.full((n - 1, 3), -7.0, np.float32), np.full((n - 1, 2), -7.0, np.float32))
        with pytest.raises(capi.SrlError) as e:
            cm.selectPointsForProjection(cam, minimum_dis=10.0, out=small)
        assert e.value.code == capi.SRL_BAD_ARG
        assert (small[0] == 0xABCDABCD).all() and (small[1] == -7.0).all() and (small[2] == -7.0).all()
        for kw in (dict(use_all_points=True), dict(skip_step=3), dict(minimum_dis=40.0 / 1.5)):
            cm.selectPointsForProjection(cam, **kw)
        assert _snapshot(cm) == before                              # the map and both lists, byte for byte
    finally:
        cm.close(); ctx.close()


def test_bad_arguments_are_refused():
    from sr_livo_b200 import capi, lio
    ctx, cm, oc, _ = _fill(20, map_sweeps(seed=6), renders=1)
    try:
        cam15 = camera((0, 0, 0))
        for kw in (dict(minimum_dis=0.0), dict(minimum_dis=-1.0), dict(minimum_dis=float("nan")), dict(minimum_dis=float("inf")),
                   dict(skip_step=0)):
            with pytest.raises(capi.SrlError) as e:
                cm.selectPointsForProjection(_cam(cam15), **kw)
            assert e.value.code == capi.SRL_BAD_ARG, kw
        for c in (_cam(cam15, rows=1), _cam(cam15, cols=0), _cam(with_fov(cam15, 1e12)), _cam(with_fov(cam15, float("nan")))):
            with pytest.raises(capi.SrlError) as e:
                cm.selectPointsForProjection(c)
            assert e.value.code == capi.SRL_BAD_ARG
        ids, _, _ = cm.selectPointsForProjection(_cam(cam15), use_all_points=True)
        st = cm.stats()
        d = cm.download()
        v = int(np.nonzero(d["counts"] < 20)[0][0])                 # a voxel with a free slot: its next index is not a point
        bad = [np.uint32(1 << 31), np.uint32(v * 20 + d["counts"][v]), np.uint32(st["voxels"] * 20)]
        for b in bad:
            with pytest.raises(capi.SrlError) as e:
                cm.gatherPoints(np.r_[ids[:3], b].astype(np.uint32))
            assert e.value.code == capi.SRL_BAD_ARG
        # eviction would move the colour map's blocks under its point ids: refused
        n = C.c_int64(0)
        vox = C.c_void_p(capi.lib().srl_color_map_voxels(cm.h))
        loc = np.zeros(3)
        assert capi.lib().srl_map_remove_far(vox, capi.ptr(loc), 0.5, C.byref(n)) == capi.SRL_BAD_ARG
        assert cm.stats() == st
    finally:
        cm.close(); ctx.close()


def test_one_cell_with_thousands_of_candidates():
    rng = np.random.default_rng(17)
    pts = np.stack([rng.uniform(-0.15, 0.15, 40000), rng.uniform(-0.15, 0.15, 40000), rng.uniform(150.0, 160.0, 40000)], axis=1)
    ctx, cm, oc, _ = _fill(50, [pts], renders=0, initial_voxels=256)
    try:
        assert cm.stats()["rgb_points"] > 5000
        cam15 = camera((0, 0, 0))
        for md in (10.0, 40.0 / 1.5):
            ids = _check(cm, oc, cam15, minimum_dis=md, use_all_points=True)
            assert ids.shape[0] <= 4
    finally:
        cm.close(); ctx.close()


def test_use_all_points_over_a_million_rgb_points():
    g = np.arange(1100) * 0.015 + 0.003
    gx, gy = np.meshgrid(g - 8.0, g - 8.0, indexing="ij")
    pts = np.stack([gx.ravel(), gy.ravel(), np.full(gx.size, 9.0) + 0.001 * np.sin(gx.ravel() * 7.0)], axis=1)
    ctx, cm, oc, _ = _fill(50, [pts], renders=1, initial_voxels=4096, max_voxels=1 << 17)
    try:
        assert cm.stats()["rgb_points"] >= 1_000_000
        for md, skip, fov in ((5.0, 1, 0.0001), (10.0, 3, -0.4)):
            ids = _check(cm, oc, with_fov(camera((0.3, -0.2, 0.0)), fov), minimum_dis=md, skip_step=skip, use_all_points=True)
            assert ids.shape[0] > 1000
    finally:
        cm.close(); ctx.close()


def test_gather_equals_the_oracle_state_after_two_renderings():
    ctx, cm, oc, _ = _fill(50, map_sweeps(seed=12), renders=2)
    try:
        rgb, _ = oc.lists()
        ids_all, _, _ = cm.selectPointsForProjection(_cam(camera((0, 0, 0))), minimum_dis=1e-3, use_all_points=True, maximum_depth=1e30,
                                                     minimum_depth=-1.0)
        ids = np.r_[ids_all, cm.selectPointsForProjection(_cam(camera((0, 0, 0))), minimum_dis=10.0)[0]].astype(np.uint32)
        got = cm.gatherPoints(ids)
        want = oc.gather(got["key_index"])
        assert want is not None
        for k in ("xyz", "rgb", "n_rgb", "cov"):
            assert np.array_equal(bits(got[k]), bits(want[k])), k
        assert got["n_rgb"].max() >= 2
    finally:
        cm.close(); ctx.close()


@pytest.mark.skipif(not TR.available(), reason="oracle/_ref/libsrl_tracker_ref.so not built")
def test_against_the_compiled_reference():
    ctx, cm, oc, ref = _fill(50, map_sweeps(seed=50), renders=2, with_ref=True)
    try:
        for _, fov, kw in select_params()[::3]:
            _check(cm, oc, with_fov(camera((0.0, 0.0, 0.0)), fov), ref=ref, **kw)
        # refreshPointsForProjection: the camera the reference derives, fov_margin -0.4, 10 px cells, the recent voxels
        q_wc = np.array([0.01, -0.02, 0.015, 1.0]); q_wc /= np.linalg.norm(q_wc)
        ki, q_cw, t_cw = ref.refresh(q_wc, [0.05, 0.0, -0.1], 300.0, 300.0, 320.25, 239.75, ROWS, COLS, 1)
        cam15 = np.concatenate([q_cw, t_cw, [0.05, 0.0, -0.1], [300.0, 300.0, 320.25, 239.75, -0.4]])
        ids, _, _ = cm.selectPointsForProjection(_cam(cam15), minimum_dis=10.0)
        assert ki.shape[0] > 0 and np.array_equal(cm.gatherPoints(ids)["key_index"], ki)
    finally:
        cm.close(); ctx.close()
