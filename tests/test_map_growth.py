"""Maps that grow on demand (srl_map_create_growable / srl_color_map_create_growable): every case feeds a growable map and
a twin created fixed at the limit the same inputs, and the two must agree bit for bit after every step, while the growable
map's capacity shows the doubling and a slot-table load of at most 0.5.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import oracle_py as O

from color_map_cases import FINE, SIZE, camera, sweep

pytestmark = pytest.mark.gpu

VS = 0.5              # LIO stream voxel size: the street stream below then grows from 1024 voxels through five doublings


def _stream_sweeps(n_sweeps=34):
    """Config-4 stream on the synthetic street: a small first sweep seeds the map, then 6000-point Livox sweeps 4 m apart."""
    from sr_livo_b200 import synth
    return [synth.make_sweep(3000 if i == 0 else 6000, seed=5000 + i, position=(4.0 * i, 3.0, 1.8)) for i in range(n_sweeps)]


def _params():
    from sr_livo_b200 import lio
    return lio.r3live_params(max_num_residuals=2 ** 31 - 1, size_voxel_map=VS)


def _map_state(m):
    keys, counts, xyz = m.download()
    return keys.tobytes() + counts.tobytes() + xyz.tobytes(), m.stats()


def _by_key(keys, counts, xyz):
    return {tuple(k): (c, x[:c].tobytes()) for k, c, x in zip(keys.tolist(), counts.tolist(), xyz)}


def _check_capacity(cap, n_voxels, history):
    assert n_voxels <= cap["committed_voxels"] and 2 * cap["committed_voxels"] <= cap["slot_capacity"]   # load <= 0.5
    if not history or history[-1] != cap["committed_voxels"]:
        if history:
            assert cap["committed_voxels"] >= 2 * history[-1]                                           # grows by doubling (or more)
        history.append(cap["committed_voxels"])


def test_lio_stream_growable_equals_fixed_and_oracle():
    from sr_livo_b200 import lio, synth
    sweeps = _stream_sweeps()
    limit = 1 << 17
    G = lio.LioOptimization(max_voxels=limit, initial_voxels=1024, sweep_capacity=8192, size_voxel_map=VS)
    F = lio.LioOptimization(max_voxels=limit, sweep_capacity=8192, size_voxel_map=VS)
    om = O.OracleMap()
    prm, P = _params(), synth.prior_covariance()
    history = [1024]
    try:
        assert G.voxel_map.capacity()["committed_voxels"] == 1024
        assert F.voxel_map.capacity()["committed_voxels"] == limit
        first = synth.registered_points(sweeps[0])
        assert G.addPointsToMap(first) == F.addPointsToMap(first) == om.add_points(first, VS)
        assert _map_state(G.voxel_map) == _map_state(F.voxel_map)
        _check_capacity(G.voxel_map.capacity(), G.voxel_map.stats()[0], history)
        for sw in sweeps[1:]:
            outs = []
            for L in (G, F):
                L.setKeypoints(sw.raw_xyz)
                L.eskf_pro = lio.EskfEstimator(p=sw.t_init.copy(), q=sw.q_init.copy(), cov=P.copy())
                summ, fq, ft = L.updateIEKF(prm, sw.t_last)
                e = L.eskf_pro
                outs.append((summ, fq, ft, np.concatenate([e.p, e.q, e.v, e.ba, e.bg, e.g, e.cov.reshape(-1)]).tobytes()))
            (sg, qg, tg, eg), (sf, qf, tf, ef) = outs
            assert eg == ef and qg.tobytes() == qf.tobytes() and tg.tobytes() == tf.tobytes()
            assert (sg.success, sg.passes_run, sg.num_residuals_used, sg.converged) == (sf.success, sf.passes_run, sf.num_residuals_used, sf.converged)
            assert sg.trace.tobytes() == sf.trace.tobytes()
            world = synth.registered_points(sw, qg, tg)
            assert G.addPointsToMap(world) == F.addPointsToMap(world) == om.add_points(world, VS)
            sgm, sfm = _map_state(G.voxel_map), _map_state(F.voxel_map)
            assert sgm == sfm
            _check_capacity(G.voxel_map.capacity(), sgm[1][0], history)
        assert len(history) >= 6, history                                  # 1024 and at least five growth steps
        assert F.voxel_map.capacity()["committed_voxels"] == limit        # the fixed map never grows
        assert _by_key(*G.voxel_map.download()) == _by_key(*om.snapshot(cap=20))
    finally:
        G.close(); F.close()


@pytest.fixture(scope="module")
def ctx():
    from sr_livo_b200 import lio
    c = lio.Context()
    yield c
    c.close()


def _twins(ctx, initial, limit, **kw):
    from sr_livo_b200 import lio
    return (lio.VoxelHashMap(ctx, VS, 20, limit, initial_voxels=initial, **kw), lio.VoxelHashMap(ctx, VS, 20, limit, **kw))


def _street_points(n_sweeps):
    from sr_livo_b200 import synth
    return [synth.registered_points(sw) for sw in _stream_sweeps(n_sweeps)]


def test_upload_past_initial_voxels(ctx):
    om = O.OracleMap()
    for p in _street_points(4):
        om.add_points(p, VS)
    keys, counts, xyz = om.snapshot(cap=20)
    assert keys.shape[0] > 3 * 1024
    g, f = _twins(ctx, 1024, 1 << 15)
    try:
        g.upload(keys, counts, xyz); f.upload(keys, counts, xyz)
        assert _map_state(g) == _map_state(f)
        assert g.capacity()["committed_voxels"] >= keys.shape[0]
        extra = _street_points(6)[5]
        assert g.insert(extra) == f.insert(extra) == om.add_points(extra, VS)
        assert _map_state(g) == _map_state(f)
        assert _by_key(*g.download()) == _by_key(*om.snapshot(cap=20))
    finally:
        g.close(); f.close()


def test_remove_far_then_growth(ctx):
    pts = _street_points(26)
    om = O.OracleMap()
    g, f = _twins(ctx, 1024, 1 << 16)
    try:
        for p in pts[:6]:
            assert g.insert(p) == f.insert(p) == om.add_points(p, VS)
        before = g.capacity()
        here = (20.0, 3.0, 1.8)
        assert g.remove_far(here, 40.0) == f.remove_far(here, 40.0) == om.remove_far(here, 40.0) > 0
        assert g.capacity() == before                                    # nothing shrinks
        for p in pts[6:]:
            assert g.insert(p) == f.insert(p) == om.add_points(p, VS)
            assert _map_state(g) == _map_state(f)
        assert g.capacity()["committed_voxels"] > before["committed_voxels"]
        assert _by_key(*g.download()) == _by_key(*om.snapshot(cap=20))
    finally:
        g.close(); f.close()


def test_insert_past_the_limit_is_refused_and_the_map_stays_usable(ctx):
    from sr_livo_b200 import capi
    pts = _street_points(8)
    limit = 4096
    g, f = _twins(ctx, 1024, limit)
    try:
        g.insert(pts[0]); f.insert(pts[0])
        state = _map_state(g)
        assert state == _map_state(f) and state[1][0] < limit
        big = np.concatenate(pts[1:])
        for m in (g, f):
            with pytest.raises(capi.SrlError) as ei:
                m.insert(big)
            assert ei.value.code == capi.SRL_MAP_FULL
            assert _map_state(m) == state                                 # the download is unchanged
        assert g.capacity()["committed_voxels"] <= limit
        small = pts[1][:500]
        assert g.insert(small) == f.insert(small) > 0
        assert _map_state(g) == _map_state(f)
    finally:
        g.close(); f.close()


def _cam(cam15):
    from sr_livo_b200 import capi
    c = capi.Camera()
    c.q_camera_world[:] = cam15[0:4].tolist(); c.t_camera_world[:] = cam15[4:7].tolist(); c.t_world_camera[:] = cam15[7:10].tolist()
    c.fx, c.fy, c.cx, c.cy, c.fov_margin = cam15[10:15].tolist()
    c.cols, c.rows = 640, 480
    return c


def _color_state(cm):
    d = cm.download()
    return {k: v.tobytes() for k, v in d.items()}, cm.stats()


def _assert_color_equals_oracle(cm, cmo):
    d, st = cm.download(), cm.stats()
    o, oc = cmo.snapshot(), cmo.counts()
    assert (st["voxels"], st["rgb_points"], st["recent"], st["new_recent"]) == (oc["voxels"], oc["rgb_points"], oc["recent"], oc["new_recent"])
    o_rgb, o_recent = cmo.lists()
    assert np.array_equal(d["rgb_points"], o_rgb) and np.array_equal(d["recent"].astype(np.int32), o_recent)
    gi = {tuple(k): i for i, k in enumerate(d["keys"].tolist())}
    assert gi.keys() == {tuple(k) for k in o["keys"].tolist()}
    for j, k in enumerate(o["keys"].tolist()):
        i = gi[tuple(k)]
        for fld in ("counts", "xyz", "rgb", "n_rgb", "cov", "obs_dist", "last_obs", "last_visited"):
            assert np.array_equal(d[fld][i], o[fld][j]), (k, fld)


@pytest.mark.parametrize("initial", [1024, 1])
@pytest.mark.parametrize("cap", [50, 100])
def test_color_map_growable_equals_fixed(ctx, cap, initial):
    """The colour-map scenes (dense surfaces, wrapped and aliased keys), shifted 1 m per frame so that the map keeps growing,
    with a rendering after every frame; the recent list is published every fourth frame, so it also grows."""
    from sr_livo_b200 import lio
    limit = 1 << 14
    g = lio.ColorVoxelMap(ctx, SIZE, cap, limit, FINE, initial_voxels=initial)
    f = lio.ColorVoxelMap(ctx, SIZE, cap, limit, FINE)
    cmo = O.OracleColorMap(voxel_size=SIZE, max_num_points_in_voxel=cap, min_distance_points=FINE)
    rng = np.random.default_rng(cap + initial)
    n_frames, seen = 12, []
    try:
        c0 = g.capacity()
        assert c0["committed_voxels"] == initial and c0["committed_rgb_points"] == initial * cap
        for fr in range(n_frames):
            pts = sweep(seed=300 + fr, n_dense=20000) + [0.0, 1.0 * fr, 0.0]
            kw = dict(add_point_step=1, time_sweep_end=1.0 + 0.1 * fr, time_last_process=0.9 + 0.1 * fr, to_rendering=(fr % 4 == 3 or fr == 0))
            assert g.addPoints(pts, **kw) == f.addPoints(pts, **kw) == cmo.add_points(pts, **kw)
            img = rng.integers(0, 256, (480, 640, 3), dtype=np.uint8)
            cam15, obs = camera((0.0, 1.0 * fr, 0.0)), kw["time_sweep_end"] + 0.05
            assert g.renderPointsInRecentVoxel(_cam(cam15), img, obs) == f.renderPointsInRecentVoxel(_cam(cam15), img, obs) == cmo.render(cam15, img, obs)
            assert _color_state(g) == _color_state(f)
            c = g.capacity()
            st = g.stats()
            assert st["voxels"] <= c["committed_voxels"] and st["rgb_points"] <= c["committed_rgb_points"] <= 2 ** 32
            assert 2 * c["committed_rgb_points"] <= c["fine_capacity"]
            seen.append(c)
            if fr in (0, n_frames - 1):
                _assert_color_equals_oracle(g, cmo)
        assert seen[-1]["committed_voxels"] > initial and seen[-1]["committed_rgb_points"] > initial * cap
        assert seen[-1]["committed_bytes"] < f.capacity()["committed_bytes"]
    finally:
        g.close(); f.close()


def test_narrow_color_map_grown_through_the_lio_insert(ctx):
    """A cap-20 colour map takes srl_map_insert on its voxel map: the colour arrays grow with the blocks, so the colour
    kernels that follow address only committed memory."""
    from sr_livo_b200 import capi, lio, synth
    L = capi.lib()
    g = lio.ColorVoxelMap(ctx, SIZE, 20, 1 << 15, FINE, initial_voxels=1024)
    f = lio.ColorVoxelMap(ctx, SIZE, 20, 1 << 15, FINE)
    sw = synth.make_sweep(20000, seed=7001, position=(1.0, 3.0, 1.8))
    pts = np.ascontiguousarray(synth.registered_points(sw))
    try:
        for cm in (g, f):
            vox = C.c_void_p(L.srl_color_map_voxels(cm.h))
            n = C.c_int64(0)
            assert L.srl_map_insert(vox, capi.ptr(pts), pts.shape[0], 0.15, 0, C.byref(n)) == capi.SRL_OK
        assert g.capacity()["committed_voxels"] > 1024
        assert _color_state(g) == _color_state(f)
        more = np.ascontiguousarray(synth.registered_points(synth.make_sweep(20000, seed=7002, position=(3.0, 3.0, 1.8))))
        kw = dict(add_point_step=1, time_sweep_end=1.0, time_last_process=0.0, to_rendering=True)
        assert g.addPoints(more, **kw) == f.addPoints(more, **kw)
        R = np.array([[0.0, -1.0, 0.0], [0.0, 0.0, -1.0], [1.0, 0.0, 0.0]])
        pos = np.array([3.0, 3.0, 1.8])
        cam15 = np.concatenate([[0.5, -0.5, 0.5, 0.5], -R @ pos, pos, [300.0, 300.0, 320.0, 240.0, 0.01]])
        img = np.random.default_rng(5).integers(0, 256, (480, 640, 3), dtype=np.uint8)
        for obs in (1.05, 1.1):                                          # a point's first fusion is not counted
            assert g.renderPointsInRecentVoxel(_cam(cam15), img, obs) == f.renderPointsInRecentVoxel(_cam(cam15), img, obs)
            assert _color_state(g) == _color_state(f)
        assert (g.download()["n_rgb"] > 0).any()
    finally:
        g.close(); f.close()


def test_create_growable_rejects_bad_initial_voxels(ctx):
    from sr_livo_b200 import capi
    L = capi.lib()
    h = C.c_void_p()
    for init, lim in ((0, 1024), (2048, 1024)):
        assert L.srl_map_create_growable(ctx.h, 1.0, 20, init, lim, C.byref(h)) == capi.SRL_BAD_ARG
        assert L.srl_color_map_create_growable(ctx.h, 0.1, 50, init, lim, 0.01, C.byref(h)) == capi.SRL_BAD_ARG


_DIST_WORKER = r"""
import os, sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], "tests"))
import numpy as np, torch, torch.distributed as tdist
from sr_livo_b200 import dist, lio, synth
from test_map_growth import VS, _params, _stream_sweeps
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
tdist.init_process_group("gloo", rank=rank, world_size=world)
L = lio.LioOptimization(device=rank, max_voxels=1 << 17, initial_voxels=1024, sweep_capacity=8192, size_voxel_map=VS)
D = dist.DistributedLio(L, rank, world, native=True)
sweeps = _stream_sweeps(12)
L.addPointsToMap(synth.registered_points(sweeps[0]))
prm = _params()
for sw in sweeps[1:]:
    D.set_keypoints(sw.raw_xyz)
    L.eskf_pro = lio.EskfEstimator(p=sw.t_init.copy(), q=sw.q_init.copy(), cov=synth.prior_covariance())
    out = D.updateIEKF(prm, sw.t_last)
    L.addPointsToMap(synth.registered_points(sw, out["frame_q"], out["frame_t"]))
    keys, counts, xyz = L.voxel_map.download()
    t = torch.from_numpy(np.concatenate([L.eskf_pro.p, L.eskf_pro.q, L.eskf_pro.cov.reshape(-1), xyz.reshape(-1).astype(np.float64),
                                         [float(L.voxel_map.capacity()["committed_voxels"])]]))
    lst = [torch.zeros_like(t) for _ in range(world)]
    tdist.all_gather(lst, t)
    assert all(torch.equal(lst[0], x) for x in lst)
assert L.voxel_map.capacity()["committed_voxels"] > 1024
D.close(); L.close(); tdist.destroy_process_group()
print("rank", rank, "ok")
"""


def test_two_ranks_grow_alike(tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = tmp_path / "growth_worker.py"
    script.write_text(_DIST_WORKER)
    port = 29900 + (os.getpid() % 1000)
    procs = []
    for r in range(2):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE="2", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        procs.append(subprocess.Popen([sys.executable, str(script), root], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = [p.communicate(timeout=600)[0] for p in procs]
    for p, o in zip(procs, outs):
        assert p.returncode == 0, o[-3000:]
