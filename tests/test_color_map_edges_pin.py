"""The colour map's insertion at its edges on the CPU: the plain restatement (tests/color_map_reference.py) against the oracle
on every case of tests/color_map_edge_cases.py after every call (points stored, counts, rgb_points_vec and the published
recent list in order, per voxel the keys, counts, float positions in order and last_visited bit for bit), and against the
reference's own compiled addPointsToMap where oracle/_ref was built.  Also checks that each family reaches its edge.

The reference's static_cast<short> is undefined for NaN, +-inf and |q| >= 2^31; the restatement drops such points, so the
oracle and the reference are fed the other selected points only (color_map_edge_cases.feed_for_reference).
"""
import numpy as np
import pytest

from oracle import oracle_py as O
from oracle import reference_py as R

import color_map_edge_cases as E
from color_map_reference import ColorMapRef
from map_reference import f32, voxel_of

CASES = {c.name: c for c in E.all_cases()}


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def voxels_of(snap) -> dict:
    """key -> ((count, 3) float32 positions, last_visited) of an oracle / reference / device snapshot"""
    return {tuple(k): (np.ascontiguousarray(x[:c]), lv)
            for k, c, x, lv in zip(snap["keys"].tolist(), snap["counts"].tolist(), snap["xyz"], snap["last_visited"].tolist())}


def assert_same_voxels(got: dict, want: dict, where):
    assert got.keys() == want.keys(), where
    for k, (xyz, lv) in want.items():
        g_xyz, g_lv = got[k]
        assert g_xyz.shape == xyz.shape and np.array_equal(bits(g_xyz), bits(xyz)), (where, k)
        assert np.array([g_lv]).view(np.int64)[0] == np.array([lv]).view(np.int64)[0], (where, k, g_lv, lv)


def assert_same_lists(rgb, recent, m: ColorMapRef, where):
    w_rgb, w_recent = m.lists()
    assert np.array_equal(np.asarray(rgb, np.int16).reshape(-1, 4), w_rgb), where
    assert np.array_equal(np.asarray(recent, np.int32).reshape(-1, 3), w_recent), where


@pytest.mark.parametrize("name", list(CASES))
def test_restatement_equals_oracle(name):
    case = CASES[name]
    m = ColorMapRef(case.size, case.cap, case.fine)
    om = O.OracleColorMap(voxel_size=case.size, max_num_points_in_voxel=case.cap, min_distance_points=case.fine)
    for i, (xyz, kw) in enumerate(case.calls):
        want = m.add_points(xyz, **kw)
        f, fkw = E.feed_for_reference(xyz, kw, case)
        assert om.add_points(f, **fkw) == want, i
        c = om.counts()
        st = m.stats()
        assert (c["voxels"], c["rgb_points"], c["recent"], c["new_recent"]) == (st["voxels"], st["rgb_points"], st["recent"], st["new_recent"]), i
        snap = om.snapshot()
        assert int(snap["counts"].sum()) == st["points"], i
        assert_same_lists(*om.lists(), m, i)
        assert_same_voxels(voxels_of(snap), m.voxels(), i)


@pytest.mark.skipif(not R.available(), reason="oracle/_ref/libsrl_reference.so not built (needs the reference tree)")
@pytest.mark.parametrize("name", list(CASES))
def test_restatement_equals_compiled_reference(name):
    case = CASES[name]
    m = ColorMapRef(case.size, case.cap, case.fine)
    ref = R.Reference()
    for i, (xyz, kw) in enumerate(case.calls):
        want = m.add_points(xyz, **kw)
        f, fkw = E.feed_for_reference(xyz, kw, case)
        before = ref.num_points(1)
        ref.add_points_to_map(f, color_voxel_size=case.size, color_max_points=case.cap, color_min_distance=case.fine,
                              add_point_step=fkw["add_point_step"], time_sweep_end=fkw["time_sweep_end"],
                              time_last_process=fkw["time_last_process"], to_rendering=fkw["to_rendering"])
        assert ref.num_points(1) - before == want, i
        c, st = ref.color_counts(), m.stats()
        assert (c["voxels"], c["rgb_points"], c["recent"], c["new_recent"]) == (st["voxels"], st["rgb_points"], st["recent"], st["new_recent"]), i
        assert ref.num_points(1) == st["points"], i
        assert_same_lists(*ref.color_lists(), m, i)
        assert_same_voxels(voxels_of(ref.snapshot(1, case.cap, color=True)), m.voxels(), i)


def test_cases_reach_their_edges():
    total = {}
    for case in CASES.values():
        ev = E.replay(case).events
        missing = [e for e in case.expect if not ev[e]]
        assert not missing, (case.name, missing)
        for k, v in ev.items():
            total[k] = total.get(k, 0) + v
    # a listed voxel with no point stored by that call, a straddling cell won across voxels after a full voxel refused a
    # point in it, gates decided within one double of 1e-5, dropped points, blocks filled to cap - 1
    for e in ("listed_without_a_stored_point", "cell_won_across_voxels", "cell_claimed_after_refusal", "gate_within_one_double",
              "dropped", "index_cap_minus_1", "stored_in_claimed_cell", "refused"):
        assert total.get(e, 0) > 0, e
    assert {c.cap for c in CASES.values()} >= {1, 2, 20, 21, 50, 100, 128}
    assert {c.fine for c in CASES.values() if c.size == E.SIZE} >= {0.01, 0.1, 0.03, 0.15}
    steps = {kw["add_point_step"] for c in CASES.values() for _, kw in c.calls}
    assert steps >= {1, 2, 3, 7, 49, 50, 51, E.BIG_STEP}
    # fine cells whose probe chains wrap the 1024-slot table and still collide at 2048 slots, in both calls of the growth
    # case (the first commits 1024 fine slots, the second 2048)
    growth = CASES["fine_chain_across_growth"]
    for xyz, _ in growth.calls:
        cells = {voxel_of(tuple(f32(v) for v in p), growth.fine) for p in xyz}
        assert sum(E.chained(k) for k in cells) >= 100

