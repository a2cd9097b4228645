"""The colour map at the counts and sizes of a long run on the GPU (scenes: tests/color_map_long_run_cases.py).

Wrap scenes: about 65,550 renderings of a few hundred points, so N_rgb runs through its short range, wraps to -32768, comes
back to 0 and re-initialises.  Every rendering's count equals the oracle's and the restated count; after every checkpoint
the device's colour state (srl_color_map_download_state), its per-id reads (srl_color_map_gather_points) and both exports at
every min_views equal the oracle bit for bit.  At the checkpoint where points stand on both sides of the wrap,
vioPhotometric over all the scene's points uses exactly those at N_rgb >= 3 and equals the 50-digit restatement.

Lattice maps of 2^22 - 1, 2^22, 2^22 + 1 and 2^23 + 5 rgb points: the export runs in one, two and three chunks of 2^22
positions, with flags on both sides of every chunk boundary and chunks without a flag.  exportColorPoints and
countColorPoints equal the oracle's export in both orders at every min_views, into pageable, pinned and CUDA outputs; a
max_points one short is refused and writes nothing; the saved PCD round-trips; and on the largest map the projection
selection over all its candidates and the per-id reads of ids past 2^22 equal the oracle.
"""
import numpy as np
import pytest

from oracle import publish_oracle as PO
from oracle import tracker_oracle as TO

import color_map_long_run_cases as L
import vio_cases as VC
import vio_reference as VR
from test_color_map_long_run_pin import bits, oracle_snapshot, point_state
from test_publish_device import read_pcd_xyzrgb

pytestmark = pytest.mark.gpu
WRAP = {c.name: c for c in L.wrap_cases()}
TOL, TOL_COV = 1e-11, 1e-10          # tests/test_vio_device.py: the device within rounding of the 50-digit truth


@pytest.fixture(scope="module")
def ctx():
    from sr_livo_b200 import lio
    c = lio.Context()
    yield c
    c.close()


def _cam(cam15, cols, rows):
    from sr_livo_b200 import capi
    c = capi.Camera()
    c.q_camera_world[:] = cam15[0:4].tolist(); c.t_camera_world[:] = cam15[4:7].tolist(); c.t_world_camera[:] = cam15[7:10].tolist()
    c.fx, c.fy, c.cx, c.cy, c.fov_margin = cam15[10:15].tolist()
    c.cols, c.rows = cols, rows
    return c


def _ids_and_keys(cm, d):
    """every stored point's id (block * block_pts + index, blocks in download order) and its (voxel key, index in block)"""
    block_pts = max(cm.cap, 20)
    ids, ki = [], []
    for v, (k, c) in enumerate(zip(d["keys"].tolist(), d["counts"].tolist())):
        for i in range(c):
            ids.append(v * block_pts + i)
            ki.append(tuple(k) + (i,))
    return np.array(ids, np.uint32), np.array(ki, np.int16).reshape(-1, 4)


def _same_export(got, want):
    return np.array_equal(bits(got[0]), bits(want[0])) and np.array_equal(np.asarray(got[1]), want[1])


def _vio_photometric(ctx, cm, ids, g):
    """vioPhotometric over the given points with the colour state gathered from the device, against the restatement"""
    from sr_livo_b200 import lio
    ip = lio.ImageProcessing(ctx, **lio.ntu_camera_params())
    try:
        cols, rows = ip.output_size()
        K = ip.camera_intrinsic()
        st = lio.CameraState([0.0, 0.0, 0.0, 1.0], L.HOME, np.eye(3), np.zeros(3), K[0, 0], K[1, 1], K[0, 2], K[1, 2], 0.002)
        state = VC.state_array(st)
        cov = VC.initial_covariance()
        ip.setCovariance(cov)
        rng = np.random.default_rng(17)
        vel = rng.normal(scale=20.0, size=(len(ids), 2))
        img = VC.textured_image(rows, cols, 23)
        r = ip.vioPhotometric(cm, st, ids, vel, 40, img)
        it, used, _ = ip.vio_last_summary(1)
        t = VR.vio_update(False, state, cov, g["xyz"], np.zeros((len(ids), 2), np.float32), vel, g["rgb"], g["cov"], g["n_rgb"], 40, img)
        assert not VC.fragile(t, False, len(ids))
        assert int(r) == t["result"] == 1 and (it, used) == (t["iterations"], t["used"])
        assert used == int((g["n_rgb"] >= 3).sum()) >= 10 and (g["n_rgb"] < 0).any()
        assert np.abs(t["state"] - state).max() > 1e-6, "the update moved nothing"
        s, c = VC.state_array(st), ip.covariance()
        assert np.all(np.abs(s - t["state"]) <= TOL * (1 + np.abs(t["state"]))), np.abs(s - t["state"]).max()
        assert np.abs(c - t["cov"]).max() <= TOL_COV * np.abs(t["cov"]).max()
    finally:
        ip.close()


@pytest.mark.parametrize("name", list(WRAP))
def test_wrap_scene_device_equals_oracle(ctx, name):
    from sr_livo_b200 import lio
    case = WRAP[name]
    cm = lio.ColorVoxelMap(ctx, L.SIZE, case.cap, 1 << 10, L.FINE)
    po = PO.OracleColorMap(voxel_size=L.SIZE, max_num_points_in_voxel=case.cap, min_distance_points=L.FINE)
    to = TO.OracleColorMap(voxel_size=L.SIZE, max_num_points_in_voxel=case.cap, min_distance_points=L.FINE)
    kw = dict(add_point_step=1, time_sweep_end=1.0, time_last_process=0.0, to_rendering=True)
    try:
        n_pts = case.points.shape[0]
        assert cm.addPoints(case.points, **kw) == po.add_points(case.points, **kw) == to.add_points(case.points, **kw) == n_pts
        counts, rendered = L.model_counts(case)
        marks = set(L.checkpoints(case))
        imgs = L.images(case.cap)
        cams = {}
        ids = keys = None
        seen_marks, vio_done = set(), False
        for k in range(1, case.renders + 1):
            cam15, img, t = case.camera_of(k), imgs[k % len(imgs)], case.obs_time(k)
            key = cam15.tobytes()
            if key not in cams:
                cams[key] = _cam(cam15, L.COLS, L.ROWS)
            n = cm.renderPointsInRecentVoxel(cams[key], img, t)
            assert n == po.render(cam15, img, t) == to.render(cam15, img, t) == rendered[k - 1], (k, n, rendered[k - 1])
            if k not in marks:
                continue
            d = cm.download()
            if ids is None:
                ids, keys = _ids_and_keys(cm, d)
            a, b = point_state(d), point_state(oracle_snapshot(po))
            assert a.keys() == b.keys() and all(a[p] == b[p] for p in b), k
            seen_marks.update(int(v) for v in np.unique(d["n_rgb"][d["n_rgb"] != 0]) if int(v) in L.COUNT_MARKS)
            g, o = cm.gatherPoints(ids), to.gather(keys)
            assert np.array_equal(g["key_index"], keys), k
            for f in ("xyz", "rgb", "n_rgb", "cov"):
                assert np.array_equal(bits(g[f]), bits(o[f])), (k, f)
            for order in (0, 1):
                for mv in L.WRAP_MIN_VIEWS:
                    assert _same_export(cm.exportColorPoints(mv, order), po.export(mv, order)), (k, order, mv)
            c = counts[k - 1]
            if not vio_done and min(c.values()) < 0 < max(c.values()):
                _vio_photometric(ctx, cm, ids, g)
                vio_done = True
        assert vio_done and seen_marks == set(L.COUNT_MARKS) - {0}
    finally:
        cm.close()


# ---- the lattice maps --------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=L.LATTICE_SIZES, ids=lambda n: f"n{n}")
def lattice(request, ctx):
    """the device map and the oracle of the published maps fed the lattice plan; the tracker's oracle too for the largest"""
    from sr_livo_b200 import lio
    n = request.param
    cm = lio.ColorVoxelMap(ctx, L.SIZE, 100, 1 << 18, L.FINE, initial_voxels=4096)
    po = PO.OracleColorMap(voxel_size=L.SIZE, max_num_points_in_voxel=100, min_distance_points=L.FINE)
    to = TO.OracleColorMap(voxel_size=L.SIZE, max_num_points_in_voxel=100, min_distance_points=L.FINE) if n == max(L.LATTICE_SIZES) else None
    cam15 = L.camera15(L.LATTICE_CAMERA, rows=L.LATTICE_ROWS, cols=L.LATTICE_COLS)
    cam = _cam(cam15, L.LATTICE_COLS, L.LATTICE_ROWS)
    img = np.ascontiguousarray(np.random.default_rng(5).integers(0, 256, (L.LATTICE_ROWS, L.LATTICE_COLS, 3), dtype=np.uint8))
    for s, (lo, hi, reps) in enumerate(L.lattice_plan(n)):
        pts = L.lattice_points(lo, hi)
        kw = dict(add_point_step=1, time_sweep_end=1.0 + s, time_last_process=0.5 + s, to_rendering=True)
        stored = cm.addPoints(pts, **kw)
        assert stored == po.add_points(pts, **kw) == hi - lo
        if to is not None:
            to.add_points(pts, **kw)
        for r in range(reps):
            got = cm.renderPointsInRecentVoxel(cam, img, 10.0 + s + r)
            assert got == po.render(cam15, img, 10.0 + s + r)
            if to is not None:
                to.render(cam15, img, 10.0 + s + r)
    assert cm.stats()["rgb_points"] == po.num_rgb_points() == n
    yield dict(n=n, cm=cm, po=po, to=to, cam=cam, cam15=cam15, counts=L.lattice_counts(n))
    cm.close()


def test_lattice_export_matches_oracle(lattice):
    import torch
    n, cm, po, counts = lattice["n"], lattice["cm"], lattice["po"], lattice["counts"]
    lat = L.lattice_points(0, n).astype(np.float32)
    for order in (0, 1):
        for mv in L.LATTICE_MIN_VIEWS:
            want = po.export(mv, order)
            total = want[0].shape[0]
            # the oracle's export is the restated one: insertion order, flags from the restated counts
            pos = L.export_positions(counts, mv, order)
            assert total == pos.shape[0] and np.array_equal(bits(want[0]), bits(lat[pos])), (order, mv)
            assert cm.countColorPoints(mv, order) == total
            assert _same_export(cm.exportColorPoints(mv, order), want), (order, mv)
            if total == 0:
                continue
            px = torch.empty((total, 3), dtype=torch.float32).pin_memory()
            pr = torch.empty((total, 3), dtype=torch.uint8).pin_memory()
            gx, gr = cm.exportColorPoints(mv, order, px, pr)
            assert _same_export((gx.numpy(), gr.numpy()), want), (order, mv)
            for rows in (total, total + 7):
                dx = torch.full((rows, 3), float("nan"), dtype=torch.float32, device="cuda")
                dr = torch.full((rows, 3), 7, dtype=torch.uint8, device="cuda")
                gx, gr = cm.exportColorPoints(mv, order, dx, dr)
                assert gx.shape[0] == total and _same_export((gx.cpu().numpy(), gr.cpu().numpy()), want), (order, mv, rows)
                assert torch.isnan(dx[total:]).all() and (dr[total:] == 7).all()            # nothing past the last point
            del px, pr, dx, dr


def test_lattice_export_one_row_short_is_refused(lattice):
    from sr_livo_b200 import capi
    cm = lattice["cm"]
    for order in (0, 1):
        total = cm.countColorPoints(-1, order)
        x = np.full((total - 1, 3), np.float32(-3.5))
        r = np.full((total - 1, 3), 9, np.uint8)
        with pytest.raises(capi.SrlError) as e:
            cm.exportColorPoints(-1, order, x, r)
        assert e.value.code == capi.SRL_BAD_ARG
        assert (x == np.float32(-3.5)).all() and (r == 9).all()


def test_lattice_saved_pcd_round_trips(lattice, tmp_path):
    if lattice["n"] != L.CHUNK + 1:
        pytest.skip("saved at 2^22 + 1 points: one chunk of exactly 2^22 positions in save order")
    cm, po = lattice["cm"], lattice["po"]
    path = str(tmp_path / "rgb_map.pcd")
    xyz, rgb = cm.saveColorPoints(path, min_views=0)
    rx, rr, alpha = read_pcd_xyzrgb(path)
    want = po.export(0, 1)
    assert xyz.shape[0] == L.CHUNK and np.array_equal(bits(rx), bits(want[0])) and np.array_equal(rr, want[1]) and (alpha == 255).all()


def test_lattice_selection_and_reads_past_2p22(lattice):
    if lattice["to"] is None:
        pytest.skip("run on the largest lattice")
    cm, to, cam, cam15 = lattice["cm"], lattice["to"], lattice["cam"], lattice["cam15"]
    ids, xyz, uv = cm.selectPointsForProjection(cam, minimum_dis=1.0, use_all_points=True)
    ki, ouv = to.select(cam15, rows=L.LATTICE_ROWS, cols=L.LATTICE_COLS, minimum_dis=1.0, use_all_points=True)
    assert len(ids) == len(ki) > 1000
    g = cm.gatherPoints(ids)
    o = to.gather(ki)
    assert np.array_equal(g["key_index"], ki) and np.array_equal(bits(xyz), bits(o["xyz"])) and np.array_equal(bits(uv), bits(ouv))
    high = ids > (1 << 22)
    assert high.sum() > 100
    gh, oh = cm.gatherPoints(ids[high]), to.gather(ki[high])
    for f in ("xyz", "rgb", "n_rgb", "cov"):
        assert np.array_equal(bits(gh[f]), bits(oh[f])), f
    assert (oh["n_rgb"] > 0).any()
