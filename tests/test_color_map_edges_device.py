"""The colour map's insertion at its edges on the GPU: for every case of tests/color_map_edge_cases.py, fed from a host array
and from a CUDA tensor, on a map committed for max_voxels and on one grown from initial_voxels, the device equals the plain
restatement (tests/color_map_reference.py) after every call: points stored, stats(), rgb_points_vec and the published
recent list in order, per voxel the keys, counts, float positions and last_visited bit for bit.  The colour state of the
points a call stores is at its reset values and that of older points is unchanged.  After every rendering call one seeded
image is rendered on the device and on the oracle, with the same count and colour state.  During the run of calls without
rendering, the map commits no more memory: those calls list nothing.
"""
import numpy as np
import pytest

from oracle import oracle_py as O

import color_map_edge_cases as E
from color_map_cases import camera
from color_map_reference import ColorMapRef
from test_color_map_edges_pin import assert_same_lists, assert_same_voxels, voxels_of

pytestmark = pytest.mark.gpu
CASES = {c.name: c for c in E.all_cases()}
STATE = ("rgb", "n_rgb", "cov", "obs_dist", "last_obs")


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


def _state(d) -> dict:
    """(voxel key, index in block) -> the colour state of that point, as bytes"""
    out = {}
    for v, (k, c) in enumerate(zip(d["keys"].tolist(), d["counts"].tolist())):
        for i in range(c):
            out[tuple(k) + (i,)] = tuple(np.ascontiguousarray(d[f][v, i]).tobytes() for f in STATE)
    return out


def _reset():
    return tuple(np.zeros(1, dt).tobytes() * n for dt, n in ((np.int16, 3), (np.int16, 1), (np.float32, 3), (np.float64, 1),
                                                             (np.float64, 1)))


def _camera_for(xyz):
    """A camera 1.5 m behind the median of the call's finite, nearby points, looking along +z."""
    f = xyz[np.all(np.isfinite(xyz) & (np.abs(xyz) < 1e4), axis=1)]
    c = np.median(f, axis=0) if f.size else np.zeros(3)
    return camera(c - [0.0, 0.0, 1.5])


@pytest.mark.parametrize("kind", ["fixed", "growable"])
@pytest.mark.parametrize("source", ["host", "cuda"])
@pytest.mark.parametrize("name", list(CASES))
def test_device_equals_restatement(ctx, name, source, kind):
    import torch
    from sr_livo_b200 import lio
    case = CASES[name]
    cm = lio.ColorVoxelMap(ctx, case.size, case.cap, case.max_voxels, case.fine,
                           initial_voxels=None if kind == "fixed" else case.initial_voxels)
    m = ColorMapRef(case.size, case.cap, case.fine)
    om = O.OracleColorMap(voxel_size=case.size, max_num_points_in_voxel=case.cap, min_distance_points=case.fine)
    rng = np.random.default_rng(len(name))
    prev, committed, coloured = {}, [], 0
    try:
        for i, (xyz, kw) in enumerate(case.calls):
            src = xyz if source == "host" else torch.from_numpy(np.ascontiguousarray(xyz)).cuda()
            try:
                got = cm.addPoints(src, **kw)
            except lio.SrlError as e:
                raise AssertionError(f"call {i}: {e}") from e
            want = m.add_points(xyz, **kw)
            f, fkw = E.feed_for_reference(xyz, kw, case)
            assert om.add_points(f, **fkw) == want, i
            assert got == want, (i, got, want)
            assert cm.stats() == m.stats(), i
            committed.append(cm.capacity()["committed_bytes"])
            d = cm.download()
            assert_same_lists(d["rgb_points"], d["recent"], m, i)
            assert_same_voxels(voxels_of(d), m.voxels(), i)
            state = _state(d)
            assert all(state[k] == v for k, v in prev.items()), i                      # older points untouched
            assert all(v == _reset() for k, v in state.items() if k not in prev), i    # new points at rgbPoint::reset()
            if kw["to_rendering"]:
                cam15 = _camera_for(xyz)
                img = rng.integers(0, 256, (480, 640, 3), dtype=np.uint8)
                obs = kw["time_sweep_end"] + 0.01 if np.isfinite(kw["time_sweep_end"]) else 0.5
                n = cm.renderPointsInRecentVoxel(_cam(cam15), img, obs)
                assert n == om.render(cam15, img, obs), i
                d = cm.download()
                o = om.snapshot()
                coloured = int((o["n_rgb"] > 0).sum())
                o_state = _state(o)
                state = _state(d)
                assert state.keys() == o_state.keys() and all(state[k] == o_state[k] for k in o_state), i
            prev = state
        if name == "no_image_run":
            # calls 1 .. 11 store nothing (cap 1) and list nothing: not a byte more is committed
            assert len(set(committed[:E.NO_IMAGE_CALLS])) == 1, committed
            assert cm.stats()["recent"] == E.NO_IMAGE_VOXELS
        if name.startswith(("cap_", "sequence_", "no_image")):
            assert coloured > 0                 # the renderings reached stored points
    finally:
        cm.close()
