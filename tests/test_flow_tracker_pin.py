"""The plain restatement of the optical-flow tracker's bookkeeping (tests/flow_tracker_reference.py) against the reference's own
opticalFlowTracker.cpp, compiled unmodified (oracle/flow_tracker.mk, tests/flow_tracker_ref.py) where it was built, and against
its outputs frozen in tests/golden/flow_tracker.npz (tests/golden/make_flow_tracker_golden.py) everywhere: bit for bit after
every call of the pin sequences (tests/flow_tracker_cases.py: run_pin), last and cur with their order, uv and velocity bits,
every point's is_out_lier_count and the number of Lucas-Kanade calls.

The sequences cover the 30-point rule, dt of 0, just below 1e-5, 1e-5 and negative, all-zero, all-one and alternating masks,
unsorted and repeated inliers, zero inliers, a throwing and a skipped PnP step, candidate lists in and out of order and with
repeats, interior points behind the camera, two cell sizes, and (maximum_tracked_points 120) a full set that takes one more."""
import os

import numpy as np
import pytest

import flow_tracker_cases as FC
import flow_tracker_ref as RF
import flow_tracker_reference as FR

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "flow_tracker.npz")
FIELDS = ("last_ids", "last_uv", "cur_ids", "cur_uv", "cur_vel", "counts", "lk_calls")


def _model(max_points):
    xyz = FC.pin_points()
    m = FR.FlowTrackerModel({i: tuple(float(a) for a in p) for i, p in enumerate(xyz)}, max_points)
    return m, FC.run_pin(m, True, max_points)


def _same(a, b):
    a, b = np.atleast_1d(np.asarray(a)), np.atleast_1d(np.asarray(b))
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def _compare(trace, other, what):
    assert [s[0] for s in trace] == [s[0] for s in other]
    for x, y in zip(trace, other):
        for f, a, b in zip(FIELDS, x[1:], y[1:]):
            assert _same(a, b), (what, x[0], f)


@pytest.mark.parametrize("max_points", FC.PIN_MAX_POINTS)
def test_restatement_equals_the_golden_reference_outputs(max_points):
    m, trace = _model(max_points)
    assert m.leading_unprojected == 0, "the pin sequences keep points behind the camera off the front of last"
    g = np.load(GOLDEN)
    golden = []
    for k, s in enumerate(trace):
        golden.append((s[0],) + tuple(g[f"max{max_points}.{k:02d}.{s[0]}.{f}"] for f in FIELDS))
    _compare(trace, golden, "golden")
    sizes = [len(s[1]) for s in trace if s[0].startswith("append")]
    if max_points == 120:
        assert max(sizes) == max_points + 1 and max_points in sizes
    assert any(len(s[3]) == 0 for s in trace) and any((s[6] != 0).any() for s in trace)


@pytest.mark.skipif(not RF.available(), reason="oracle/_ref/libsrl_flow_tracker_ref.so not built (needs the reference tree)")
@pytest.mark.parametrize("max_points", FC.PIN_MAX_POINTS)
def test_compiled_reference_equals_the_restatement(max_points):
    _, trace = _model(max_points)
    r = RF.FlowTrackerReference(FC.pin_points(), max_points)
    try:
        _compare(trace, FC.run_pin(r, False, max_points), "compiled reference")
    finally:
        r.close()


@pytest.mark.skipif(not RF.available(), reason="oracle/_ref/libsrl_flow_tracker_ref.so not built (needs the reference tree)")
def test_compiled_reference_interior_entry_behind_the_camera_takes_the_previous_projection():
    """an interior entry whose camera z < 0.001 measures its error against the previous entry's projection, in the reference and
    in the restatement alike (a leading one reads uninitialised doubles in the reference: DESIGN.md section 5)"""
    xyz = FC.pin_points()
    behind = int(np.flatnonzero(xyz[:, 2] < 0)[0])
    front = [i for i in range(behind) if xyz[i, 2] > 0][:40]
    cam = FC.model_camera(FC.cam15())
    uv = np.array([FR.project_full(cam, xyz[i])[2:] for i in front], np.float32)
    ids = np.array(front + [behind], np.uint32)
    uv = np.r_[uv, [[50.0, 50.0]]].astype(np.float32)
    m = FR.FlowTrackerModel({i: tuple(float(a) for a in p) for i, p in enumerate(xyz)}, 300)
    r = RF.FlowTrackerReference(xyz, 300)
    try:
        for t in (m, r):
            t.init(1.0, ids, uv, lambda p: None)
        m.update_and_append(cam, [], 40.0)
        r.update_and_append(FC.cam15(), FC.COLS, FC.ROWS, [], 40.0)
        assert m.leading_unprojected == 0                         # the behind point is interior here
        assert _same(m.last_arrays()[0], r.last_arrays()[0]) and _same(m.last_arrays()[1], r.last_arrays()[1])
    finally:
        r.close()
