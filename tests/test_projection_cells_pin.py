"""The cell layout of the map tracker's projection selection and optical-flow tracker, without a GPU.

  * srl::cell_axis restated (projection_cell_cases.cell_axis) and its bound checked at every shipped camera size, FoV margin and
    cell size of the cases: the outermost accepted coordinates of each axis and their neighbouring doubles give fields in
    [0, 2^bits - 2], so no cell packs to the all-ones `none`, and the two fields fit 64 bits (DESIGN.md section 4).
  * The reference's own compiled selectPointsForProjection (oracle/_ref/libsrl_tracker_ref.so) equals the oracle
    (oracle/tracker_oracle.py) on every selection case: ids in order and uv bits.
  * The reference's own compiled opticalFlowTracker (oracle/_ref/libsrl_flow_tracker_ref.so) equals the sequential restatement
    (tests/flow_tracker_reference.py) after every call of every tracker case: order, uv bits and outlier counts.
The last two skip when those libraries were not built (they need the reference tree to build)."""
import math

import numpy as np
import pytest

import flow_tracker_ref as RF
import flow_tracker_reference as FR
import projection_cell_cases as P
import tracker_ref as TR
from render_reference import Camera

HUGE_FOVS = (1.0 - 1e9 / 1024.0, float(np.nextafter(1.0 - 1e9 / 1024.0, 0.0)), 2e6, -1e7, 1e300)


def _extremes(fov, size):
    """the outermost accepted coordinates of one axis and the accepted doubles next to them"""
    e = P.edges(fov, size)
    if e is None:
        return []
    lo, _, H, _ = e
    return sorted({lo, P.nxt(lo) if P.nxt(lo) <= H else lo, H, P.prv(H) if P.prv(H) >= lo else H})


def _layouts():
    for name, cols, rows, md, _, _ in P.cameras():
        for fov in P.FOVS + HUGE_FOVS:
            for d in P.cell_sizes(fov, cols, rows, md) if abs(fov) < 1e6 else (md, 1e-3, 1.0):
                yield name, cols, rows, fov, d


def test_cell_axis_bound_at_the_shipped_shapes():
    checked = refused = ends = 0
    for name, cols, rows, fov, d in _layouts():
        lay_u, lay_v = P.cell_axis(fov, cols, d), P.cell_axis(fov, rows, d)
        if lay_u is None or lay_v is None:
            refused += 1
            lo_u, hi_u = P.bounds(fov, cols)
            assert max(abs(lo_u), abs(hi_u), abs(fov * rows + 1.0), abs((1.0 - fov) * rows)) >= 1e9 or not math.isfinite(fov)
            continue
        assert lay_u[1] + lay_v[1] <= 64, (name, fov, d)
        end = lay_u[1] + lay_v[1]
        none = (1 << end) - 1
        us, vs = _extremes(fov, cols), _extremes(fov, rows)
        for u in us:
            for v in vs:
                assert P.accepted(u, fov, cols) and P.accepted(v, fov, rows)
                fu, fv, key = P.key_fields(u, v, d, lay_u, lay_v)
                assert 0 <= fu <= (1 << lay_u[1]) - 2 and 0 <= fv <= (1 << lay_v[1]) - 2, (name, fov, d, u, v, fu, fv)
                assert key != none and key < (1 << end)
                ends += fu >= (1 << (lay_u[1] - 1)) + (1 << (lay_u[1] - 2)) or fv >= (1 << (lay_v[1] - 1)) + (1 << (lay_v[1] - 2))
                checked += 1
    assert checked > 5000 and refused >= 3 and ends > 0
    # the refusals of cell_axis, one at a time: a non-finite margin, a window with a >= 1e9, a / d >= 1e300
    assert P.cell_axis(float("nan"), 752, 40.0) is None and P.cell_axis(float("inf"), 752, 40.0) is None
    assert P.cell_axis(HUGE_FOVS[0], 1024, 40.0) is None and P.cell_axis(HUGE_FOVS[1], 1024, 40.0) == (-(2 * 10 ** 9 + 2), 32)
    assert P.cell_axis(0.005, 752, 1e-298) is None and P.cell_axis(0.005, 752, 1e-297) is not None


def test_bound_cells_reach_twice_the_coordinate():
    """the d of bound_ds puts the outermost accepted coordinate x at cell +-d, about 2x: the case the 2a + 1 bound is for"""
    seen = set()
    for name, cols, rows, md, _, _ in P.cameras():
        for fov in P.FOVS:
            for d in P.bound_ds(fov, cols, rows):
                xs = [x for size in (cols, rows) for x in _extremes(fov, size) if 0.5 < abs(x) / d < 0.5 + 1e-9]
                assert xs, (name, fov, d)
                for x in xs:
                    c = P.cell(x, d)
                    assert abs(c) == int(d) and abs(c) > 2 * abs(x) - 2
                    seen.add(c > 0)
    assert seen == {True, False}


def test_shifts_put_the_anchors_on_the_edges():
    n = 0
    for name, fov, cols, rows, d, _ in P.selection_cases()[::5]:
        pts, targets = P.selection_points(fov, cols, rows, d)
        for axis, t, k in targets:
            tu, tv = P.target_shift(pts, (axis, t, k))
            u, v, ok = P.project_window(pts[k], fov, cols, rows, tu, tv)
            assert (u, v)[axis] == t
            n += 1
    assert n > 500


def _ki(pts, k):
    """the (voxel key, index in block) the map gives point k when every point is stored in order"""
    from map_reference import voxel_of
    key = voxel_of(tuple(float(a) for a in pts[k]), P.VOXEL)
    return key + (sum(voxel_of(tuple(float(a) for a in q), P.VOXEL) == key for q in pts[:k]),)


@pytest.mark.skipif(not TR.available(), reason="oracle/_ref/libsrl_tracker_ref.so not built (needs the reference tree)")
def test_compiled_selection_equals_the_oracle_on_every_case():
    from oracle import tracker_oracle as O
    hit = miss = 0
    for name, fov, cols, rows, d, _ in P.selection_cases():
        pts, targets = P.selection_points(fov, cols, rows, d)
        oc = O.OracleColorMap(P.VOXEL, P.CAP, P.FINE)
        ref = TR.TrackerReference(P.VOXEL, P.CAP, P.FINE)
        assert oc.add_points(pts) == ref.add_points(pts) == len(pts), name
        calls = [((0.0, 0.0), None)] + [(P.target_shift(pts, t), t) for t in targets]
        for (tu, tv), t in calls:
            cam = P.window_cam15(fov, tu, tv)
            for use_all in ((False, True) if t is None else (True,)):
                kw = dict(minimum_dis=d, use_all_points=use_all, minimum_depth=0.0, maximum_depth=200.0)
                ki_o, uv_o = oc.select(cam, rows, cols, **kw)
                ki_r, uv_r = ref.select(cam, rows, cols, **kw)
                assert np.array_equal(ki_o, ki_r) and np.array_equal(uv_o.view(np.uint32), uv_r.view(np.uint32)), (name, tu, tv, use_all)
            if t is not None:
                axis, val, k = t
                sel = {tuple(int(a) for a in r) for r in ki_o}
                inside = P.project_window(pts[k], fov, cols, rows, tu, tv)[2]
                if not inside:
                    assert _ki(pts, k) not in sel, (name, t)
                else:
                    hit += _ki(pts, k) in sel
                    miss += _ki(pts, k) not in sel
    assert hit > 1000 and hit > 4 * miss


@pytest.mark.skipif(not TR.available(), reason="oracle/_ref/libsrl_tracker_ref.so not built (needs the reference tree)")
def test_compiled_selection_equals_the_oracle_through_the_shipped_intrinsics():
    from oracle import tracker_oracle as O
    n = 0
    for name, cols, rows, md, k, _ in P.cameras():
        if k is None:
            continue
        pts = P.scene_points(cols, rows, k, seed=cols)
        oc, ref = O.OracleColorMap(0.25, 20, 0.01), TR.TrackerReference(0.25, 20, 0.01)
        assert oc.add_points(pts) == ref.add_points(pts)
        for fov in P.FOVS:
            for d in P.cell_sizes(fov, cols, rows, md):
                kw = dict(minimum_dis=d, use_all_points=True)
                ki_o, uv_o = oc.select(P.shipped_cam15(fov, k), rows, cols, **kw)
                ki_r, uv_r = ref.select(P.shipped_cam15(fov, k), rows, cols, **kw)
                assert np.array_equal(ki_o, ki_r) and np.array_equal(uv_o.view(np.uint32), uv_r.view(np.uint32)), (name, fov, d)
                n += len(ki_o)
    assert n > 10000


def loop1_errors(case, cam):
    """the error loop 1 measures for each init entry (row order), the stale projection carried over entries behind the camera"""
    pos = case["points"].astype(np.float64)
    uv = dict(zip(case["init_rows"], [tuple(float(a) for a in r) for r in case["init_uv"]]))
    out, ud = {}, None
    for r in sorted(uv):
        z_ok, _, u, v = FR.project_full(cam, pos[r])
        if z_ok:
            ud = (u, v)
        if ud is not None:
            a, b = ud[0] - uv[r][0], ud[1] - uv[r][1]
            out[r] = math.sqrt(a * a + b * b)
    return out


def run_tracker(tracker, case, model_like, snap):
    """init then the case's updates on a FlowTrackerModel (model_like) or a FlowTrackerReference; snap() after every call"""
    ids, uv = np.array(case["init_rows"], np.uint32), case["init_uv"]
    tracker.init(1.0, ids, uv, lambda p: None)
    snap("init")
    for k, (cam15, cand, md) in enumerate(case["steps"]):
        c = np.array(cand, np.uint32)
        if model_like:
            tracker.update_and_append(Camera(cam15, case["rows"], case["cols"]), c, md)
        else:
            tracker.update_and_append(cam15, case["cols"], case["rows"], c, md)
        snap(f"append{k}")


def test_tracker_cases_reach_their_thresholds_and_edges():
    """the crafted errors are exactly thr, 2 thr and one double above, at widths where thr is not a float (752: 4.7), and the
    survivors of the edge cases sit exactly on their edge"""
    widths = set()
    from map_reference import voxel_of
    for case in P.tracker_cases():
        keys = [voxel_of(tuple(float(a) for a in p), P.TRACK_VOXEL) for p in case["points"]]
        assert len(set(keys)) == len(keys), "one voxel per point"
        cam = Camera(case["steps"][0][0], case["rows"], case["cols"])
        err = loop1_errors(case, cam)
        for r, e in case["errors"].items():
            assert err[r] == e, (case["name"], r, err[r], e)
            widths.add(case["cols"])
        assert all(P.project_window(case["points"][r], case["fov"], case["cols"], case["rows"], *case["steps"][0][0][4:6])[0] is None
                   for r in case["init_rows"] if case["points"][r][2] < 0)
        assert case["points"][min(case["init_rows"])][2] > 0, "an entry behind the camera must not come first"
    assert {752, 1280} <= widths and float(np.float32(P.thr_of(752))) != P.thr_of(752)


@pytest.mark.skipif(not RF.available(), reason="oracle/_ref/libsrl_flow_tracker_ref.so not built (needs the reference tree)")
def test_compiled_tracker_equals_the_restatement_on_every_case():
    erased = appended = 0
    for case in P.tracker_cases():
        pos = {i: tuple(float(a) for a in p) for i, p in enumerate(case["points"])}
        rows_all = np.arange(len(case["points"]), dtype=np.uint32)
        m = FR.FlowTrackerModel(pos, case["max_points"])
        r = RF.FlowTrackerReference(case["points"], case["max_points"])
        try:
            tm, tr = [], []
            run_tracker(m, case, True, lambda tag: tm.append((tag, *m.last_arrays(),
                                                              np.array([m.count.get(int(i), 0) for i in rows_all], np.int16))))
            run_tracker(r, case, False, lambda tag: tr.append((tag, *r.last_arrays(), r.counts(rows_all))))
            assert m.leading_unprojected == 0
            for a, b in zip(tm, tr):
                assert a[0] == b[0]
                for x, y in zip(a[1:], b[1:]):
                    assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), (case["name"], a[0])
            erased += len(set(tm[0][1].tolist()) - set(tm[-1][1].tolist()))
            appended += len(set(tm[-1][1].tolist()) - set(tm[0][1].tolist()))
        finally:
            r.close()
    assert erased > 0 and appended > 0
