"""The plain restatement of the optical-flow tracker's bookkeeping (tests/flow_tracker_reference.py) on hand-worked inputs: the
decisions opticalFlowTracker.cpp makes at its edges, each computed here by hand from the source.  The device is checked
against this restatement in test_flow_tracker_device.py."""
import math

import numpy as np

import flow_tracker_cases as FC
import flow_tracker_reference as FR

F32 = np.float32


def _grid(n):
    """n points of the exact grid (x, y, 2) and their exact projections under the unmoved camera"""
    _, _, exact = FC.scene_points()
    cam = FC.model_camera(FC.cam15())
    pos, proj = {}, {}
    for i, p in enumerate(exact[:n]):
        pos[i] = tuple(p)
        _, res, u, v = FR.project_full(cam, p)
        assert res and u == math.floor(u) + 0.125 and v == math.floor(v)
        proj[i] = (u, v)
    return pos, proj, cam


def _no_lk(p):
    raise AssertionError("Lucas-Kanade called")


def test_init_keeps_the_last_of_repeated_ids():
    m = FR.FlowTrackerModel({}, 300)
    m.init(0.0, [5, 3, 5], [(1, 1), (2, 2), (3, 3)], lambda p: None)
    assert m.last == {3: (F32(2), F32(2)), 5: (F32(3), F32(3))} and m.lk_calls == 1


def test_fewer_than_thirty_points_skip_lucas_kanade_and_keep_last():
    pos, proj, _ = _grid(29)
    m = FR.FlowTrackerModel(pos, 300)
    m.init(1.0, list(proj), [proj[i] for i in proj], lambda p: None)
    assert m.track_image(2.0, _no_lk, FC.COLS, FC.ROWS) is False
    assert m.last_time == 2.0 and m.cur == {} and len(m.last) == 29


def test_velocities_and_the_time_step_rule():
    """(1e-3f, 1e-3f) when now - last_image_time < 1e-5 (zero, just below, negative), else 0.5 / dt rounded to float"""
    pos, proj, _ = _grid(30)
    for now in (1.0, 1.0 + 9.99e-6, 0.0, 1.0 + 1e-5, 1.1):
        m = FR.FlowTrackerModel(pos, 300)
        m.init(1.0, list(proj), [proj[i] for i in proj], lambda p: None)
        assert m.track_image(now, lambda p: (p + F32(0.5), np.ones(len(p), np.uint8)), FC.COLS, FC.ROWS)
        d = now - 1.0
        want = float(F32(0.5 / d)) if d >= 1e-5 else float(F32(1e-3))
        assert len(m.cur) >= 20 and np.all(m.cur_arrays()[2] == want), (now, want)


def test_margin_bounds():
    """if2dPointsAvailable(x, y, 1.0, 0.05) on 640 x 480: x >= 33, ceil(x) < 608, y >= 25, ceil(y) < 456"""
    assert FR.in_margin(33.0, 25.0, 640, 480) and not FR.in_margin(float(np.nextafter(F32(33), F32(0))), 25.0, 640, 480)
    assert FR.in_margin(607.0, 455.0, 640, 480) and not FR.in_margin(float(np.nextafter(F32(607), F32(700))), 100.0, 640, 480)
    assert not FR.in_margin(100.0, float(np.nextafter(F32(455), F32(500))), 640, 480)


def test_remove_outliers_rules():
    pos, proj, _ = _grid(40)
    m = FR.FlowTrackerModel(pos, 300)
    m.cur = {i: ((F32(i), F32(i)), (0.0, 0.0)) for i in range(9)}
    m.last = {100: (F32(0), F32(0))}
    assert m.remove_outliers([0]) is False and list(m.last) == [100]          # fewer than 10: nothing changes
    m.cur = {i * 2: ((F32(i), F32(-i)), (1.0, 2.0)) for i in range(10)}
    assert m.remove_outliers([7, 2, 2, 9]) is True
    assert sorted(m.last) == [4, 14, 18] and m.last[14] == (F32(7), F32(-7)) and sorted(m.cur) == [4, 14, 18]
    m.cur = {i: ((F32(i), F32(i)), (0.0, 0.0)) for i in range(10)}
    assert m.remove_outliers([]) is True and m.last == {} and m.cur == {}


def test_append_thresholds_and_counts():
    """thr = 4 on 640 columns: error 4 resets the count, just above 4 counts once and erases the second time, above 8 erases at
    once; a NaN error (leading entry behind the camera) keeps the entry and resets its count"""
    pos, proj, cam = _grid(5)
    pos[99] = (0.0, 0.0, -1.0)                                  # behind the camera, the smallest id below
    m = FR.FlowTrackerModel({**pos, -1: pos[99]}, 300)
    eps4 = float(np.nextafter(F32(proj[1][0] + 4.0), F32(1e9))) - proj[1][0]
    m.last = {-1: (F32(0), F32(0)), 0: (F32(proj[0][0] + 4.0), F32(proj[0][1])), 1: (F32(proj[1][0] + eps4), F32(proj[1][1])),
              2: (F32(proj[2][0] + 8.0), F32(proj[2][1])), 3: (F32(proj[3][0] + 8.5), F32(proj[3][1])),
              4: (F32(proj[4][0]), F32(proj[4][1]))}
    m.count = {-1: 1, 0: 1}
    m.update_and_append(cam, [], 40.0)
    assert sorted(m.last) == [-1, 0, 1, 2, 4] and m.count[-1] == 0 and m.count[0] == 0 and m.count[1] == 1 and m.count[2] == 1
    assert m.count[3] == 0
    m.update_and_append(cam, [], 40.0)
    assert sorted(m.last) == [-1, 0, 4] and m.count[1] == 0 and m.count[2] == 0


def test_append_size_rule_and_reentry():
    """size0 < max: candidates enter until the set holds max; size0 >= max: only the first non-member candidate may enter, so
    the set can reach max + 1; an erased point is no member and comes straight back as a candidate"""
    pos, proj, cam = _grid(40)
    uv = {i: (F32(proj[i][0]), F32(proj[i][1])) for i in proj}
    for max_points, size0, want in ((12, 10, 12), (10, 10, 11), (9, 10, 11)):
        m = FR.FlowTrackerModel(pos, max_points)
        m.last = {i: uv[i] for i in range(size0)}
        m.update_and_append(cam, list(range(39, 9, -1)), 1.0)
        assert len(m.last) == want, (max_points, size0, len(m.last))
    m = FR.FlowTrackerModel(pos, 300)
    m.last = {0: (F32(proj[0][0] + 20.0), F32(proj[0][1]))}
    m.update_and_append(cam, [0], 1.0)
    assert m.last == {0: uv[0]} and m.count[0] == 0
