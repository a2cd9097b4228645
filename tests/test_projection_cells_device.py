"""The map tracker's projection cells on the GPU at the shipped camera sizes and at the FoV window's edges
(tests/projection_cell_cases.py): selectPointsForProjection (srl_color_map_select_for_projection) against the oracle and the
reference's compiled selection, and updateAndAppendTrackPoints (srl_flow_tracker_update_and_append) against the sequential
restatement and the reference's compiled tracker, bit for bit; refusals that change nothing; empty windows."""
import numpy as np
import pytest

from oracle import tracker_oracle as O

import flow_tracker_ref as RF
import flow_tracker_reference as FR
import projection_cell_cases as P
import tracker_ref as TR
from render_reference import Camera

pytestmark = pytest.mark.gpu


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _cam(cam15, cols, rows):
    from sr_livo_b200 import capi
    c = [float(a) for a in cam15]
    import ctypes as C
    return capi.Camera((C.c_double * 4)(*c[0:4]), (C.c_double * 3)(*c[4:7]), (C.c_double * 3)(*c[7:10]), c[10], c[11], c[12], c[13], c[14],
                       int(cols), int(rows))


@pytest.fixture(scope="module")
def ctx():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from sr_livo_b200 import lio
    c = lio.Context(0)
    yield c
    c.close()


def test_resized_cameras_match_the_image_preparation(ctx):
    from sr_livo_b200 import lio
    for name, cols, rows, md, _, resized in P.cameras():
        if resized is None:
            continue
        p, in_cols = resized
        in_rows = int(round(p["image_height"] * in_cols / p["image_width"]))
        ip = lio.ImageProcessing(ctx, **p, cols=in_cols, rows=in_rows)
        try:
            assert ip.output_size() == (cols, rows) and 40.0 / ip.scale_factor() == md, name
        finally:
            ip.close()


def _select_all(cm, oc, ref, cam15, cols, rows, kw, what):
    ids, xyz, uv = cm.selectPointsForProjection(_cam(cam15, cols, rows), **kw)
    ki_o, uv_o = oc.select(cam15, rows, cols, **kw)
    g = cm.gatherPoints(ids)
    assert np.array_equal(g["key_index"], ki_o), what
    assert np.array_equal(bits(uv), bits(uv_o)), what
    want = oc.gather(ki_o)
    assert want is not None and np.array_equal(bits(xyz), bits(want["xyz"])), what
    if ref is not None:
        ki_r, uv_r = ref.select(cam15, rows, cols, **kw)
        assert np.array_equal(ki_r, ki_o) and np.array_equal(bits(uv_r), bits(uv)), what
    return ids, xyz, uv


def _snapshot(cm):
    d = cm.download()
    return {k: bits(v).tobytes() for k, v in d.items()}, cm.stats()


def test_selection_equals_the_oracle_on_every_case(ctx):
    """every (camera, margin, d): the unshifted call from both sources, then one call per edge target (lo, the double below
    it, H, the double above it, per axis); the empty windows select nothing"""
    from sr_livo_b200 import lio
    use_ref = TR.available()
    empty = 0
    for n_case, (name, fov, cols, rows, d, _) in enumerate(P.selection_cases()):
        pts, targets = P.selection_points(fov, cols, rows, d)
        cm = lio.ColorVoxelMap(ctx, P.VOXEL, P.CAP, 1 << 14, P.FINE)
        oc = O.OracleColorMap(P.VOXEL, P.CAP, P.FINE)
        ref = TR.TrackerReference(P.VOXEL, P.CAP, P.FINE) if use_ref else None
        try:
            cm.addPoints(pts, 1, 1.0, 0.0, True)
            assert oc.add_points(pts) == len(pts) == cm.stats()["rgb_points"], name
            if ref:
                ref.add_points(pts)
            calls = [((0.0, 0.0), None)] + [(P.target_shift(pts, t), t) for t in targets]
            before = _snapshot(cm) if n_case % 40 == 0 else None
            for (tu, tv), t in calls:
                cam15 = P.window_cam15(fov, tu, tv)
                for use_all in ((False, True) if t is None else (True,)):
                    kw = dict(minimum_dis=d, use_all_points=use_all, minimum_depth=0.0, maximum_depth=200.0)
                    ids, xyz, uv = _select_all(cm, oc, ref, cam15, cols, rows, kw, (name, tu, tv, use_all))
                    if P.edges(fov, cols) is None or P.edges(fov, rows) is None:
                        assert len(ids) == 0, name
                        empty += 1
                    if before is not None:
                        assert cm.countPointsForProjection(_cam(cam15, cols, rows), **kw) == len(ids)
                        _host_device_agree(cm, _cam(cam15, cols, rows), kw, ids, xyz, uv)
            if before is not None:
                assert _snapshot(cm) == before, name                 # the map and both lists, byte for byte
        finally:
            cm.close()
    assert empty > 50


def _host_device_agree(cm, cam, kw, ids, xyz, uv):
    import torch
    n = len(ids)
    d = (torch.empty(n + 3, dtype=torch.int32, device="cuda"), torch.empty((n + 3, 3), dtype=torch.float32, device="cuda"),
         torch.empty((n + 3, 2), dtype=torch.float32, device="cuda"))
    gi, gx, gu = cm.selectPointsForProjection(cam, out=d, **kw)
    assert np.array_equal(gi.cpu().numpy().view(np.uint32), ids) and np.array_equal(bits(gx.cpu().numpy()), bits(xyz))
    assert np.array_equal(bits(gu.cpu().numpy()), bits(uv))


def test_selection_through_the_shipped_intrinsics(ctx):
    from sr_livo_b200 import lio
    for name, cols, rows, md, k, _ in P.cameras():
        if k is None:
            continue
        pts = P.scene_points(cols, rows, k, seed=cols)
        cm = lio.ColorVoxelMap(ctx, 0.25, 20, 1 << 14, 0.01)
        oc = O.OracleColorMap(0.25, 20, 0.01)
        ref = TR.TrackerReference(0.25, 20, 0.01) if TR.available() else None
        try:
            cm.addPoints(pts, 1, 1.0, 0.0, True)
            oc.add_points(pts)
            if ref:
                ref.add_points(pts)
            for fov in P.FOVS:
                for d in P.cell_sizes(fov, cols, rows, md):
                    _select_all(cm, oc, ref, P.shipped_cam15(fov, k), cols, rows, dict(minimum_dis=d, use_all_points=True), (name, fov, d))
        finally:
            cm.close()


# ---- updateAndAppendTrackPoints ------------------------------------------------------------------------------------------------
class _Env:
    """a colour map holding one case's points, one voxel each, in row order; row -> point id"""

    def __init__(self, ctx, case):
        from sr_livo_b200 import lio
        self.cm = lio.ColorVoxelMap(ctx, P.TRACK_VOXEL, P.CAP, 1 << 14, P.FINE)
        pts = case["points"].astype(np.float64)
        for p in pts:
            self.cm.addPoints(p.reshape(1, 3), 1, 1.0, 0.0, True)
        xyz = self.cm.download()["xyz"].reshape(-1, 3)
        rows_of = {tuple(r.view(np.uint32).tolist()): i for i, r in enumerate(np.ascontiguousarray(xyz, np.float32))}
        self.ids = np.array([rows_of[tuple(p.view(np.uint32).tolist())] for p in np.ascontiguousarray(case["points"], np.float32)], np.uint32)
        assert np.all(np.diff(self.ids.astype(np.int64)) > 0), "ids must follow the rows"
        self.pos = {int(i): tuple(float(a) for a in p) for i, p in zip(self.ids, case["points"])}
        self.xyz = xyz

    def close(self):
        self.cm.close()


def _tracker(ctx, env, case):
    from sr_livo_b200 import lio
    lk = lio.LKOpticalFlowKernel(ctx, **lio.tracker_lk_params())
    t = lio.OpticalFlowTracker(ctx, env.cm, lk, case["max_points"])
    return t, lk


def _state(t, ids):
    last = t.last()
    return (bits(last[0]).tobytes(), bits(last[1]).tobytes(), bits(t.outlierCounts(ids)).tobytes(), t.counts())


def _check(t, m, env, what):
    ml = m.last_arrays()
    dl = t.last()
    assert np.array_equal(dl[0], ml[0]) and np.array_equal(bits(dl[1]), bits(ml[1])), what
    want = np.array([m.count.get(int(i), 0) for i in env.ids], np.int16)
    assert np.array_equal(t.outlierCounts(env.ids), want), what
    assert t.counts()["last"] == len(ml[0])


def test_update_and_append_equals_the_restatement_on_every_case(ctx):
    """init, then the case's updates; after every call last (order, uv bits) and every point's outlier count equal the
    restatement's and, where it was built, the compiled reference's"""
    erased = appended = 0
    for case in P.tracker_cases():
        env = _Env(ctx, case)
        t, lk = _tracker(ctx, env, case)
        ref = RF.FlowTrackerReference(env.xyz, case["max_points"]) if RF.available() else None
        try:
            m = FR.FlowTrackerModel(env.pos, case["max_points"])
            gray = np.zeros((case["rows"], case["cols"]), np.uint8)
            ids0 = env.ids[case["init_rows"]]
            t.init(gray, 1.0, ids0, case["init_uv"])
            m.init(1.0, ids0, case["init_uv"], lambda p: None)
            if ref:
                ref.init(1.0, ids0, case["init_uv"], lambda p: None)
            _check(t, m, env, (case["name"], "init"))
            start = set(m.last)
            for k, (cam15, cand, md) in enumerate(case["steps"]):
                c = env.ids[np.array(cand, np.int64)]
                t.updateAndAppendTrackPoints(_cam(cam15, case["cols"], case["rows"]), c, md)
                m.update_and_append(Camera(cam15, case["rows"], case["cols"]), c, md)
                _check(t, m, env, (case["name"], k))
                if ref:
                    ref.update_and_append(cam15, case["cols"], case["rows"], c, md)
                    assert np.array_equal(ref.last_arrays()[0], m.last_arrays()[0])
                    assert np.array_equal(bits(ref.last_arrays()[1]), bits(m.last_arrays()[1]))
                    assert np.array_equal(ref.counts(env.ids), t.outlierCounts(env.ids)), (case["name"], k)
            assert m.leading_unprojected == 0
            if case["fov"] >= 0.5:                                   # an empty window appends nothing
                assert set(m.last) <= start
            erased += len(start - set(m.last))
            appended += len(set(m.last) - start)
        finally:
            t.close(); lk.close(); env.close()
            if ref:
                ref.close()
    assert erased > 0 and appended > 0


def test_refusals_change_nothing(ctx):
    """a non-finite margin, a window with a >= 1e9, a / d >= 1e300 and an image narrower or lower than 2 pixels: both entry
    points refuse, and the sets, counts, outlier counts and map bytes stay as they were"""
    from sr_livo_b200 import capi, lio
    case = next(c for c in P.tracker_cases() if c["name"].startswith("thr+-752"))
    env = _Env(ctx, case)
    t, lk = _tracker(ctx, env, case)
    try:
        cols, rows = case["cols"], case["rows"]
        t.init(np.zeros((rows, cols), np.uint8), 1.0, env.ids[case["init_rows"]], case["init_uv"])
        cam15, cand, md = case["steps"][0]
        t.updateAndAppendTrackPoints(_cam(cam15, cols, rows), env.ids[np.array(cand)], md)     # counts of 1 to keep
        huge = 1.0 - 1e9 / 1024.0
        bad = [(P.window_cam15(float("nan")), cols, rows, md), (P.window_cam15(float("inf")), cols, rows, md),
               (P.window_cam15(-float("inf")), cols, rows, md), (P.window_cam15(huge), 1024, 1024, md),
               (P.window_cam15(0.005), cols, rows, 1e-298), (P.window_cam15(0.005), 1, rows, md), (P.window_cam15(0.005), cols, 1, md),
               (P.window_cam15(0.005), 0, 0, md)]
        state, snap = _state(t, env.ids), _snapshot(env.cm)
        for cam15b, c, r, d in bad:
            for call in (lambda: t.updateAndAppendTrackPoints(_cam(cam15b, c, r), env.ids[np.array(cand)], d),
                         lambda: env.cm.selectPointsForProjection(_cam(cam15b, c, r), minimum_dis=d),
                         lambda: env.cm.countPointsForProjection(_cam(cam15b, c, r), minimum_dis=d)):
                with pytest.raises(lio.SrlError) as e:
                    call()
                assert e.value.code == capi.SRL_BAD_ARG, (cam15b[14], c, r, d)
                assert _state(t, env.ids) == state and _snapshot(env.cm) == snap
        # just inside each limit: accepted
        ok = [(P.window_cam15(float(np.nextafter(huge, 0.0))), 1024, 1024, md), (P.window_cam15(0.005), cols, rows, 1e-297),
              (P.window_cam15(0.005), 2, 2, md)]
        for cam15b, c, r, d in ok:
            env.cm.selectPointsForProjection(_cam(cam15b, c, r), minimum_dis=d)
    finally:
        t.close(); lk.close(); env.close()
