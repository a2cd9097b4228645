"""selectPointsForProjection, the reference's own code against the oracle, bit for bit and in order.

Left: oracle/_ref/libsrl_tracker_ref.so, the reference's rgbMapTracker::selectPointsForProjection / refreshPointsForProjection
compiled from its sources over a colour map its addPointsToMap fills and its renderer colours (oracle/tracker.mk).  Right: the
oracle's restatement (orc_color_select), which the GPU tests use as their yardstick.  Also: a numpy model of the prefix-min
characterisation the device's parallel form rests on, against the sequential rule (no library needed).

CPU only; the reference comparisons are skipped when the reference library was not built.
"""
import numpy as np
import pytest

from oracle import tracker_oracle as O

import tracker_ref as TR
from projection_cases import (COLS, FINE, HALVES_CAM, ROWS, SIZE, camera, halves_points, map_sweeps, prefix_min_winners, select_params,
                              sequential_winners, ulp_pairs, with_fov)
from publish_cases import render_images

needs_ref = pytest.mark.skipif(not TR.available(), reason="oracle/_ref/libsrl_tracker_ref.so not built (needs the reference tree)")


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _fill(cap, sweeps, renders=1, to_rendering=None, with_ref=True):
    oc = O.OracleColorMap(voxel_size=SIZE, max_num_points_in_voxel=cap, min_distance_points=FINE)
    ref = TR.TrackerReference(SIZE, cap, FINE) if with_ref else None
    for s, pts in enumerate(sweeps):
        t_end, t_proc = 1.0 + 0.1 * s, 1.0 * s
        tr = True if to_rendering is None else to_rendering[s]
        oc.add_points(pts, 1, t_end, t_proc, tr)
        if ref:
            ref.add_points(pts, 1, t_end, t_proc, tr)
        for k, img in enumerate(render_images(100 * cap + s, renders)):
            cam, obs = camera((0.02 * k, 0.0, 0.0)), t_end + 0.01 * (k + 1)
            n = oc.render(cam, img, obs)
            if ref:
                assert ref.render(cam, img, obs) == n
    if ref:
        assert ref.num_rgb_points() == oc.num_rgb_points() and ref.num_recent() == oc.num_recent()
    return oc, ref


def _agree(ref, oc, cam15, rows=ROWS, cols=COLS, **kw):
    a, b = ref.select(cam15, rows, cols, **kw), oc.select(cam15, rows, cols, **kw)
    assert np.array_equal(a[0], b[0]), kw
    assert np.array_equal(bits(a[1]), bits(b[1])), kw
    return b


@needs_ref
@pytest.mark.parametrize("cap", [20, 50, 100])
def test_map_scenes_reference_equals_oracle(cap):
    oc, ref = _fill(cap, map_sweeps(seed=cap), renders=2)
    sizes = {}
    for name, fov, kw in select_params():
        for pos in ((0.0, 0.0, 0.0), (0.13, -0.07, 0.5)):
            ki, _ = _agree(ref, oc, with_fov(camera(pos), fov), **kw)
            sizes[name, pos] = ki.shape[0]
    p0 = (0.0, 0.0, 0.0)
    assert min(v for (_, pos), v in sizes.items() if pos == p0) > 0
    # the scene exercises what it should: skip_step, the source and the margin change the selection
    assert sizes["md5-skip1-recent-fov0.0001", p0] != sizes["md5-skip1-all-fov0.0001", p0]
    assert sizes["md10-skip1-recent-fov-0.4", p0] >= sizes["md10-skip1-recent-fov0.0001", p0]


@needs_ref
def test_empty_recent_list_falls_back_to_rgb_points():
    sweeps = map_sweeps(seed=3)
    # a last sweep whose end time equals time_last_process: nothing is appended, the published recent list is empty
    oc = O.OracleColorMap(voxel_size=SIZE, max_num_points_in_voxel=50, min_distance_points=FINE)
    ref = TR.TrackerReference(SIZE, 50, FINE)
    for s, pts in enumerate(sweeps):
        oc.add_points(pts, 1, 1.0 + 0.1 * s, 1.0 * s, True); ref.add_points(pts, 1, 1.0 + 0.1 * s, 1.0 * s, True)
    oc.add_points(sweeps[0][:100], 1, 7.0, 7.0, True); ref.add_points(sweeps[0][:100], 1, 7.0, 7.0, True)
    assert oc.num_recent() == ref.num_recent() == 0
    for md in (5.0, 10.0):
        a = _agree(ref, oc, camera((0, 0, 0)), minimum_dis=md, use_all_points=False)
        b = oc.select(camera((0, 0, 0)), minimum_dis=md, use_all_points=True)
        assert np.array_equal(a[0], b[0]) and a[0].shape[0] > 0


@needs_ref
def test_recent_list_after_sweeps_without_rendering():
    """to_rendering off for two sweeps, then on: the rendering sweep clears voxels_recent_visited_temp before it publishes the
    list (src/lioOptimization.cpp:523-527), so the list the tracker reads holds each voxel once; both sides agree on it."""
    sweeps = map_sweeps(seed=8)
    third = sweeps[0][::2] + 0.002
    oc, ref = _fill(50, [sweeps[0], sweeps[1], third], renders=1, to_rendering=[False, False, True])
    _, rec = oc.lists()
    assert rec.shape[0] > 0 and np.unique(rec, axis=0).shape[0] == rec.shape[0]
    for md in (5.0, 10.0, 40.0 / 1.5):
        _agree(ref, oc, with_fov(camera((0, 0, 0)), -0.4), minimum_dis=md)


@needs_ref
@pytest.mark.parametrize("md", [5.0, 10.0])
def test_exact_halves_reference_equals_oracle(md):
    pts = halves_points(md)
    oc, ref = _fill(50, [pts], renders=0)
    for use_all in (False, True):
        ki, uv = _agree(ref, oc, HALVES_CAM, minimum_dis=md, use_all_points=use_all)
        assert (uv[:, 0] < 0).any() and (uv[:, 1] < 0).any()            # negative halves were selected
        if use_all:   # every point is alone in its cell: each one selected, half away from zero
            assert ki.shape[0] == np.count_nonzero(pts[:, 1] * 64.0 >= -191.0)


@needs_ref
@pytest.mark.parametrize("reverse", [False, True])
def test_ulp_pairs_reference_equals_oracle(reverse):
    pts = ulp_pairs(seed=21 + reverse, n=12, reverse=reverse)
    oc, ref = _fill(50, [pts], renders=0)
    picks = []
    for md in (10.0, 40.0 / 1.5):
        for use_all in (False, True):
            ki, _ = _agree(ref, oc, camera((0, 0, 0)), minimum_dis=md, use_all_points=use_all)
            picks.append(ki.shape[0])
    # within a pair the float comparison decides; the 40/1.5 px cells hold each pair together, so that selection has at most
    # one point per pair
    assert picks[2] <= 12 and picks[3] <= 12


@needs_ref
@pytest.mark.parametrize("cap", [20, 50])
def test_refresh_equals_oracle_select_from_the_derived_camera(cap):
    oc, ref = _fill(cap, map_sweeps(seed=40 + cap), renders=1)
    rng = np.random.default_rng(cap)
    for frame_id, pos in enumerate([(0.0, 0.0, 0.0), (0.11, -0.05, 0.3), (-0.2, 0.1, -0.4)]):
        axis = rng.normal(size=3)
        axis /= np.linalg.norm(axis)
        ang = 0.05 * (frame_id + 1)
        q_wc = np.r_[np.sin(ang / 2) * axis, np.cos(ang / 2)]
        ki, q_cw, t_cw = ref.refresh(q_wc, pos, 300.0, 300.0, 320.25, 239.75, ROWS, COLS, frame_id)
        cam15 = np.concatenate([q_cw, t_cw, pos, [300.0, 300.0, 320.25, 239.75, -0.4]])
        want, _ = oc.select(cam15, ROWS, COLS, minimum_dis=10.0, skip_step=1, use_all_points=False)
        assert ki.shape[0] > 0 and np.array_equal(ki, want), frame_id
        again, _, _ = ref.refresh(q_wc, pos, 300.0, 300.0, 320.25, 239.75, ROWS, COLS, frame_id)   # same frame_id: early return
        assert np.array_equal(again, ki)


def _adversarial_sequences(rng):
    out = []
    base = np.float32(4.0)
    ulp = float(np.spacing(base))
    for _ in range(200):
        k = int(rng.integers(1, 40))
        kind = rng.integers(0, 5)
        if kind == 0:    # depths within a float ulp of one float value: rounding up and down decides
            d = float(base) + rng.integers(-2, 3, k) * ulp / 4 + rng.uniform(-1e-12, 1e-12, k)
        elif kind == 1:  # exact repeats (a voxel listed twice): the later copy takes the cell when its float rounds up
            v = float(base) + rng.choice([ulp / 4, -ulp / 4, ulp / 3])
            d = np.full(k, v)
        elif kind == 2:  # decreasing, then increasing within the rounding gap
            d = float(base) + np.r_[np.linspace(ulp, -ulp, k // 2 + 1), np.linspace(-ulp, ulp, k - k // 2 - 1)] / 2
        elif kind == 3:  # far points with random gaps
            d = rng.uniform(100.0, 100.0 + 4 * float(np.spacing(np.float32(100.0))), k)
        else:
            d = rng.uniform(0.1, 200.0, k)
        cells = rng.integers(0, 1 + int(rng.integers(1, 4)), k)
        out.append((d, cells))
    return out


def test_prefix_min_characterisation_equals_the_sequential_rule():
    rng = np.random.default_rng(2024)
    seen_later_farther = seen_repeat = False
    for d, c in _adversarial_sequences(rng):
        want = sequential_winners(d.tolist(), c.tolist())
        assert prefix_min_winners(d, c) == want
        for cell in np.unique(c):
            idx = np.nonzero(c == cell)[0]
            w = [j for j in want if c[j] == cell][0]
            first = idx[0]
            if w != first and d[w] > d[first]:
                seen_later_farther = True                  # a farther later point beat a nearer one whose depth rounded up
            if w != first and d[w] == d[first]:
                seen_repeat = True                         # a repeat replaced its own earlier copy
    assert seen_later_farther and seen_repeat


def test_counter_intuitive_cases_by_hand():
    d0 = 4.0 + float(np.spacing(np.float32(4.0))) * 0.6     # float(d0) rounds up above d0
    assert float(np.float32(d0)) > d0
    # farther later beats nearer earlier: d1 > d0 but d1 < float(d0)
    d1 = d0 + float(np.spacing(np.float32(4.0))) * 0.05
    assert sequential_winners([d0, d1], [0, 0]) == prefix_min_winners([d0, d1], [0, 0]) == [1]
    # the same depth twice: the later copy takes the cell
    assert sequential_winners([d0, d0], [7, 7]) == prefix_min_winners([d0, d0], [7, 7]) == [1]
    # a depth that rounds down: the later equal copy does not
    d2 = 4.0 + float(np.spacing(np.float32(4.0))) * 0.1
    assert float(np.float32(d2)) < d2
    assert sequential_winners([d2, d2], [1, 1]) == prefix_min_winners([d2, d2], [1, 1]) == [0]
