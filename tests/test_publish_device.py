"""The published maps on the GPU: srl_map_insert_published / srl_map_insert_sweep_published (the registered cloud of
addPointsToMap) and srl_color_map_export (pubColorPoints / saveColorPoints), against the oracle bit for bit, and against the
reference's own compiled code (oracle/_ref/libsrl_publish_ref.so) where that library was built.
"""
import numpy as np
import pytest

from oracle import publish_oracle as O

import publish_ref as PR
from color_map_cases import FINE, SIZE, camera, sweep
from publish_cases import CAP, MIN_DIST, lio_stream, render_images, small_color_points

pytestmark = pytest.mark.gpu


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _cam(cam15):
    from sr_livo_b200 import capi
    c = capi.Camera()
    c.q_camera_world[:] = cam15[0:4].tolist(); c.t_camera_world[:] = cam15[4:7].tolist(); c.t_world_camera[:] = cam15[7:10].tolist()
    c.fx, c.fy, c.cx, c.cy, c.fov_margin = cam15[10:15].tolist()
    c.cols, c.rows = 640, 480
    return c


def _download_bytes(vm):
    keys, counts, xyz = vm.download()
    return bits(keys).tobytes() + bits(counts).tobytes() + bits(xyz).tobytes()


@pytest.mark.parametrize("mode", ["host", "device", "sweep"])
@pytest.mark.parametrize("voxel_size,min_num_points", [(1.0, 0), (0.5, 0), (1.0, 3), (0.5, 3)])
def test_registered_cloud_matches_oracle(mode, voxel_size, min_num_points):
    import torch
    from sr_livo_b200 import lio
    L = lio.LioOptimization(max_voxels=1 << 16, sweep_capacity=1 << 13, size_voxel_map=voxel_size, initial_voxels=256)
    P = lio.LioOptimization(max_voxels=1 << 16, sweep_capacity=1 << 13, size_voxel_map=voxel_size, initial_voxels=256)
    om = O.OracleMap()
    try:
        for k, (pts, tz) in enumerate(lio_stream(seed=int(40 * voxel_size) + min_num_points, voxel_size=voxel_size)):
            mnp = 0 if k == 0 else min_num_points
            if mode == "sweep":   # identity rotation and extrinsics: the registered points are raw + t, one rounding
                t = np.array([0.25, -0.5, tz])
                raw = pts - t
                world = raw + t
                L.setKeypoints(raw); P.setKeypoints(raw)
                added, a = L.addSweepToMapPublished([0, 0, 0, 1], t, MIN_DIST, mnp)
                plain = P.addSweepToMap([0, 0, 0, 1], t, MIN_DIST, mnp)
            else:
                world = pts
                src = torch.from_numpy(np.ascontiguousarray(pts)).cuda() if mode == "device" else pts
                added, a = L.addPointsToMapPublished(src, tz, MIN_DIST, mnp)
                if mode == "device":
                    assert a.is_cuda
                    a = a.cpu().numpy()
                plain = P.addPointsToMap(pts, MIN_DIST, mnp)
            b_added, b = om.add_points_published(world, tz, voxel_size, CAP, MIN_DIST, mnp)
            assert added == plain == b_added, k
            assert a.shape == b.shape and np.array_equal(bits(a), bits(b)), k
        assert _download_bytes(L.voxel_map) == _download_bytes(P.voxel_map)   # the map is the plain insert's, byte for byte
        assert L.voxel_map.capacity()["committed_voxels"] > 256
    finally:
        L.close(); P.close()


def test_registered_cloud_counts_an_uploaded_empty_voxel_as_found():
    """A voxel uploaded with count 0 is in the slot table, so its first point is appended to a found voxel and published."""
    from sr_livo_b200 import lio
    L = lio.LioOptimization(max_voxels=1 << 10, sweep_capacity=64)
    om = O.OracleMap()
    keys = np.array([[2, 3, 4], [5, 5, 5]], np.int16)
    counts = np.array([0, 1], np.int32)
    xyz = np.zeros((2, CAP, 3), np.float32)
    xyz[1, 0] = [5.5, 5.5, 5.5]
    try:
        L.voxel_map.upload(keys, counts, xyz)
        om.load(keys, counts, xyz)
        pts = np.array([[2.5, 3.5, 4.5], [2.9, 3.1, 4.2], [5.1, 5.2, 5.3], [7.5, 7.5, 7.5], [7.2, 7.2, 7.2]])
        added, a = L.addPointsToMapPublished(pts, 1.0, MIN_DIST, 0)
        b_added, b = om.add_points_published(pts, 1.0, 1.0, CAP, MIN_DIST, 0)
        assert added == b_added == 5 and np.array_equal(bits(a), bits(b))
        assert a.shape[0] == 4 and a[0, 0] == np.float32(2.5)    # only the creator of voxel (7, 7, 7) is left out
    finally:
        L.close()


def test_max_out_below_n_leaves_the_map_unchanged():
    from sr_livo_b200 import capi, lio
    L = lio.LioOptimization(max_voxels=1 << 14, sweep_capacity=1 << 13)
    try:
        stream = lio_stream(seed=5, voxel_size=1.0)
        L.addPointsToMap(stream[0][0], MIN_DIST)
        before = _download_bytes(L.voxel_map), L.mapSize()
        pts, tz = stream[1]
        with pytest.raises(capi.SrlError) as e:
            L.addPointsToMapPublished(pts, tz, MIN_DIST, 0, out=np.empty((pts.shape[0] - 1, 4), np.float32))
        assert e.value.code == capi.SRL_BAD_ARG
        L.setKeypoints(pts)
        with pytest.raises(capi.SrlError) as e:
            L.addSweepToMapPublished([0, 0, 0, 1], [0, 0, 0], MIN_DIST, 0, out=np.empty((pts.shape[0] - 1, 4), np.float32))
        assert e.value.code == capi.SRL_BAD_ARG
        assert (_download_bytes(L.voxel_map), L.mapSize()) == before
    finally:
        L.close()


def _color_pair(cap, sweeps, renders, initial_voxels=64, with_ref=False):
    from sr_livo_b200 import lio
    ctx = lio.Context()
    cm = lio.ColorVoxelMap(ctx, SIZE, cap, 1 << 16, FINE, initial_voxels=initial_voxels)
    oc = O.OracleColorMap(voxel_size=SIZE, max_num_points_in_voxel=cap, min_distance_points=FINE)
    ref = PR.PublishReference() if with_ref else None
    for s, pts in enumerate(sweeps):
        t_end, t_proc = 1.0 + 0.1 * s, 1.0 * s
        cm.addPoints(pts, 1, t_end, t_proc, True)
        oc.add_points(pts, add_point_step=1, time_sweep_end=t_end, time_last_process=t_proc, to_rendering=True)
        if ref:
            ref.add_points_to_map(pts, 0.0, color_voxel_size=SIZE, color_max_points=cap, color_min_distance=FINE, add_point_step=1,
                                  time_sweep_end=t_end, time_last_process=t_proc, to_rendering=True)
        for k, img in enumerate(render_images(100 * cap + s, renders)):
            cam15, obs = camera((0.02 * k, 0.0, 0.0)), t_end + 0.01 * (k + 1)
            n = cm.renderPointsInRecentVoxel(_cam(cam15), img, obs)
            assert n == oc.render(cam15, img, obs)
            if ref:
                assert ref.color_render(cam15, img, obs) == n
    return ctx, cm, oc, ref


@pytest.mark.parametrize("cap", [50, 100])
def test_color_export_matches_oracle(cap):
    import torch
    rng = np.random.default_rng(cap)
    first = sweep(seed=11 * cap)
    ctx, cm, oc, _ = _color_pair(cap, [first, first + rng.normal(0, 0.003, first.shape)], renders=2)
    try:
        assert cm.capacity()["committed_voxels"] > 64        # the map grew while it was fed
        top = oc.max_n_rgb()
        for order in (0, 1):
            for mv in (-1, 0, 1, 3, top + 1):
                want = oc.export(mv, order)
                got = cm.exportColorPoints(mv, order)
                assert np.array_equal(bits(got[0]), bits(want[0])) and np.array_equal(got[1], want[1]), (order, mv)
                assert cm.countColorPoints(mv, order) == want[0].shape[0]
                dx = torch.empty((want[0].shape[0] + 7, 3), dtype=torch.float32, device="cuda")
                dr = torch.empty((want[0].shape[0] + 7, 3), dtype=torch.uint8, device="cuda")
                gx, gr = cm.exportColorPoints(mv, order, dx, dr)
                assert np.array_equal(bits(gx.cpu().numpy()), bits(want[0])) and np.array_equal(gr.cpu().numpy(), want[1]), (order, mv)
                px = torch.empty((want[0].shape[0], 3), dtype=torch.float32).pin_memory()   # page-locked host output
                pr = torch.empty((want[0].shape[0], 3), dtype=torch.uint8).pin_memory()
                gx, gr = cm.exportColorPoints(mv, order, px, pr)
                assert np.array_equal(bits(gx.numpy()), bits(want[0])) and np.array_equal(gr.numpy(), want[1]), (order, mv)
        assert cm.pubColorPoints(1)[0].shape[0] == oc.export(1, 0)[0].shape[0]
        from sr_livo_b200 import capi
        n = cm.countColorPoints(-1, 0)
        with pytest.raises(capi.SrlError):
            cm.exportColorPoints(-1, 0, np.empty((n - 1, 3), np.float32), np.empty((n - 1, 3), np.uint8))
    finally:
        cm.close(); ctx.close()


@pytest.mark.parametrize("k", [0, 1, 2])
def test_color_export_of_tiny_maps(k):
    ctx, cm, oc, _ = _color_pair(50, [small_color_points(k)], renders=1)
    try:
        for order in (0, 1):
            for mv in (-1, 0, 1):
                want, got = oc.export(mv, order), cm.exportColorPoints(mv, order)
                assert np.array_equal(bits(got[0]), bits(want[0])) and np.array_equal(got[1], want[1]), (order, mv)
        assert cm.countColorPoints(-1, 1) == max(k - 1, 0)
    finally:
        cm.close(); ctx.close()


def read_pcd_xyzrgb(path):
    """A small reader of binary PCD v0.7 files with fields x y z rgb (float32 each)."""
    with open(path, "rb") as f:
        data = f.read()
    header, rest = {}, data
    while True:
        line, rest = rest.split(b"\n", 1)
        if line.startswith(b"#"):
            continue
        key, _, val = line.decode("ascii").partition(" ")
        header[key] = val
        if key == "DATA":
            break
    assert header["VERSION"] == "0.7" and header["FIELDS"] == "x y z rgb" and header["SIZE"] == "4 4 4 4"
    assert header["TYPE"] == "F F F F" and header["COUNT"] == "1 1 1 1" and header["HEIGHT"] == "1"
    assert header["VIEWPOINT"] == "0 0 0 1 0 0 0" and header["DATA"] == "binary"
    n = int(header["POINTS"])
    assert int(header["WIDTH"]) == n and len(rest) == 16 * n
    rec = np.frombuffer(rest, np.float32).reshape(n, 4)
    packed = rec.view(np.uint32)[:, 3]
    rgb = np.stack([(packed >> 16) & 255, (packed >> 8) & 255, packed & 255], axis=1).astype(np.uint8)
    return rec[:, :3].copy(), rgb, (packed >> 24).astype(np.uint8)


def test_saved_pcd_round_trips(tmp_path):
    first = sweep(seed=3)
    ctx, cm, oc, _ = _color_pair(50, [first], renders=2)
    try:
        path = str(tmp_path / "rgb_map.pcd")
        xyz, rgb = cm.saveColorPoints(path, min_views=1)
        rx, rr, alpha = read_pcd_xyzrgb(path)
        want = oc.export(1, 1)
        assert xyz.shape[0] > 0 and np.array_equal(bits(rx), bits(want[0])) and np.array_equal(rr, want[1]) and (alpha == 255).all()
        assert np.array_equal(bits(xyz), bits(rx)) and np.array_equal(rgb, rr)
    finally:
        cm.close(); ctx.close()


@pytest.mark.skipif(not PR.available(), reason="oracle/_ref/libsrl_publish_ref.so not built")
def test_against_the_compiled_reference():
    from sr_livo_b200 import lio
    L = lio.LioOptimization(max_voxels=1 << 16, sweep_capacity=1 << 13, size_voxel_map=0.5, initial_voxels=256)
    ref = PR.PublishReference()
    try:
        for k, (pts, tz) in enumerate(lio_stream(seed=77, voxel_size=0.5)):
            a_added, a = ref.add_points_to_map(pts, tz, 0.5, CAP, MIN_DIST, 0)
            added, g = L.addPointsToMapPublished(pts, tz, MIN_DIST, 0)
            assert added == a_added and np.array_equal(bits(g), bits(a)), k
    finally:
        L.close()
    first = sweep(seed=9)
    ctx, cm, oc, ref = _color_pair(50, [first, first + np.random.default_rng(9).normal(0, 0.003, first.shape)], renders=2, with_ref=True)
    try:
        for order in (0, 1):
            for mv in (-1, 0, 1, 3):
                want, got = ref.export(mv, order), cm.exportColorPoints(mv, order)
                assert np.array_equal(bits(got[0]), bits(want[0])) and np.array_equal(got[1], want[1]), (order, mv)
    finally:
        cm.close(); ctx.close()
