"""The colour map past the short range of N_rgb on the CPU: the reference's own compiled code against the oracle on the wrap
scenes of tests/color_map_long_run_cases.py, and the reference's short counter and vioPhotometric's N_rgb < 3 skip read
directly, with no restatement in between.

Left: oracle/_ref/libsrl_reference.so (the colour state, ref_map_snapshot) and oracle/_ref/libsrl_publish_ref.so (the clouds
pubColorPoints and saveColorPoints hand over), both fed the same calls.  Right: the oracle of the published maps (its
snapshot and orc_color_export).  Skipped where the reference libraries were not built.  The lattice plan's reach (flags on
both sides of every chunk boundary, a chunk without a flag) is checked on its plain restatement, which needs nothing built.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import publish_oracle as PO
from oracle import reference_py as R

import color_map_long_run_cases as L
import publish_ref as PR
import vio_cases as VC
import vio_ref as RF
import vio_reference as VR

CASES = {c.name: c for c in L.wrap_cases()}
STATE = ("rgb", "n_rgb", "cov", "obs_dist", "last_obs")
needs_ref = pytest.mark.skipif(not (R.available() and PR.available()),
                               reason="oracle/_ref/libsrl_reference.so / libsrl_publish_ref.so not built (needs the reference tree)")


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def oracle_snapshot(oc) -> dict:
    """the colour state of an oracle of the published maps (publish_oracle.OracleColorMap), as ref_map_snapshot returns it"""
    lib, cap = PO.lib(), oc.cap
    nv = int(lib.orc_color_num_voxels(oc._h))
    a = dict(keys=np.zeros((nv, 3), np.int16), counts=np.zeros(nv, np.int32), xyz=np.zeros((nv, cap, 3), np.float32),
             rgb=np.zeros((nv, cap, 3), np.int16), n_rgb=np.zeros((nv, cap), np.int16), cov=np.zeros((nv, cap, 3), np.float32),
             obs_dist=np.zeros((nv, cap)), last_obs=np.zeros((nv, cap)), last_visited=np.zeros(nv))
    lib.orc_color_snapshot(oc._h, cap, *[a[k].ctypes.data_as(C.c_void_p) for k in ("keys", "counts", "xyz", "rgb", "n_rgb", "cov",
                                                                                   "obs_dist", "last_obs", "last_visited")])
    return a


def point_state(snap) -> dict:
    """(voxel key, index in block) -> the colour state of that point, as bytes"""
    out = {}
    for v, (k, c) in enumerate(zip(snap["keys"].tolist(), snap["counts"].tolist())):
        for i in range(c):
            out[tuple(k) + (i,)] = tuple(np.ascontiguousarray(snap[f][v, i]).tobytes() for f in STATE)
    return out


def point_counts(snap) -> dict:
    """(voxel key, index in block) -> N_rgb"""
    return {tuple(k) + (i,): int(snap["n_rgb"][v, i]) for v, (k, c) in enumerate(zip(snap["keys"].tolist(), snap["counts"].tolist()))
            for i in range(c)}


def group_of_points(case, snap) -> dict:
    """(voxel key, index in block) -> the group of the scene that point belongs to (found by its float position)"""
    where = {np.asarray(case.points[i], np.float32).tobytes(): g for g, idx in case.groups.items() for i in idx.tolist()}
    return {tuple(k) + (i,): where[snap["xyz"][v, i].tobytes()] for v, (k, c) in enumerate(zip(snap["keys"].tolist(), snap["counts"].tolist()))
            for i in range(c)}


def counts_match_groups(counts_after: dict, snap, where: dict) -> bool:
    """every point's N_rgb is its group's restated count"""
    got = point_counts(snap)
    return got.keys() == where.keys() and all(got[p] == counts_after[g] for p, g in where.items())


@needs_ref
@pytest.mark.parametrize("name", list(CASES))
def test_wrap_scene_reference_equals_oracle(name):
    case = CASES[name]
    ref, pub = R.Reference(), PR.PublishReference()
    oc = PO.OracleColorMap(voxel_size=L.SIZE, max_num_points_in_voxel=case.cap, min_distance_points=L.FINE)
    kw = dict(add_point_step=1, time_sweep_end=1.0, time_last_process=0.0, to_rendering=True)
    stored = oc.add_points(case.points, **kw)
    assert stored == case.points.shape[0]
    ref.add_points_to_map(case.points, color_voxel_size=L.SIZE, color_max_points=case.cap, color_min_distance=L.FINE, **kw)
    pub.add_points_to_map(case.points, 0.0, color_voxel_size=L.SIZE, color_max_points=case.cap, color_min_distance=L.FINE, **kw)
    counts, rendered = L.model_counts(case)
    marks = set(L.checkpoints(case))
    imgs = L.images(case.cap)
    where, straddled = None, False
    for k in range(1, case.renders + 1):
        cam, img, t = case.camera_of(k), imgs[k % len(imgs)], case.obs_time(k)
        n = oc.render(cam, img, t)
        assert ref.color_render(cam, img, t) == n and pub.color_render(cam, img, t) == n, k
        assert n == rendered[k - 1], (k, n, rendered[k - 1])
        if k not in marks:
            continue
        rs, os_ = ref.snapshot(1, case.cap, color=True), oracle_snapshot(oc)
        if where is None:
            where = group_of_points(case, rs)
        # the reference's own short: each point at its group's restated count, no harness convention in between
        assert counts_match_groups(counts[k - 1], rs, where), (k, counts[k - 1])
        a, b = point_state(rs), point_state(os_)
        assert a.keys() == b.keys() and all(a[p] == b[p] for p in b), k
        for order in (0, 1):
            for mv in L.WRAP_MIN_VIEWS:
                x, y = pub.export(mv, order), oc.export(mv, order)
                assert np.array_equal(bits(x[0]), bits(y[0])) and np.array_equal(x[1], y[1]), (k, order, mv)
        c = counts[k - 1]
        straddled |= min(c.values()) < 0 < max(c.values())
    assert straddled


@pytest.mark.skipif(not R.available(), reason="oracle/_ref/libsrl_reference.so not built (needs the reference tree)")
def test_reference_counter_is_a_wrapping_short():
    """one point viewed 65,537 times by the reference's own renderer: N_rgb -32768 after 32,768 views, 0 after 65,536, and the
    next view takes updateRgb's first-view branch again: it is not counted and leaves the state the first view left"""
    ref = R.Reference()
    p = np.array([[0.2051, 0.2543, 2.0562]])
    ref.add_points_to_map(p, color_voxel_size=L.SIZE, color_max_points=50, color_min_distance=L.FINE, add_point_step=1,
                          time_sweep_end=1.0, time_last_process=0.0, to_rendering=True)
    imgs = L.images(3)
    cam = L.camera15(L.HOME)

    def view(k):
        return ref.color_render(cam, imgs[0] if k in (1, 65537) else imgs[k % len(imgs)], 1.0 + L.DT * k)

    def state():
        s = ref.snapshot(1, 50, color=True)
        return {f: s[f][0, 0].copy() for f in STATE}

    assert view(1) == 0
    first = state()
    assert first["n_rgb"] == 1 and np.all(first["cov"] == 15.0)
    at = {}
    for k in range(2, 65537):
        assert view(k) == 1, k
        if k in (32767, 32768, 32769, 65535, 65536):
            at[k] = state()
    assert [int(at[k]["n_rgb"]) for k in sorted(at)] == [32767, -32768, -32767, -1, 0]
    assert np.all(at[32768]["cov"] > 0) and np.all(np.isfinite(at[32768]["cov"]))      # reported while negative
    assert np.all(at[65536]["cov"] == 0)                                               # N_rgb == 0: not reported
    assert view(65537) == 0
    again = state()
    assert int(again["n_rgb"]) == 1 and np.array_equal(again["rgb"], first["rgb"]) and np.array_equal(again["cov"], first["cov"])
    assert again["obs_dist"] == first["obs_dist"] and again["last_obs"] == 1.0 + L.DT * 65537
    assert view(65538) == 1 and int(state()["n_rgb"]) == 2


VIO_COUNTS = np.array([-32768, -1, 0, 2, 3, 32767], np.int16)


@pytest.mark.skipif(not RF.available(), reason="oracle/_ref/libsrl_vio_ref.so not built (needs the reference tree)")
def test_vio_photometric_skips_exactly_the_counts_below_three():
    """vioPhotometric's `N_rgb < 3` skip (src/imageProcessing.cpp:465) on wrapped counts: the compiled reference gives the
    same bits when every skipped count is replaced by 0 and every kept one by 40, and other bits when the 2s become 3s; the
    restatement uses exactly the points at 3 and 32767 and agrees with the reference within rounding"""
    c = VC.make_case(61, "ntu", n=60)
    cov = VC.initial_covariance()
    n_rgb = np.resize(VIO_COUNTS, 60).astype(np.int16)
    kept = n_rgb >= 3

    def run(counts):
        return RF.update(1, c["state"], cov, c["xyz"], c["uv"], c["vel"], c["rgb"], c["cov_rgb"], counts, c["n_new_visited"], c["img"])

    s, cv, r, _ = run(n_rgb)
    assert r[1] == 1
    s0, cv0, r0, _ = run(np.where(kept, 40, 0).astype(np.int16))
    assert r0 == r and np.array_equal(bits(s0), bits(s)) and np.array_equal(bits(cv0), bits(cv))
    s3, cv3, _, _ = run(np.where(n_rgb == 2, 3, n_rgb).astype(np.int16))
    assert not np.array_equal(bits(s3), bits(s))
    t = VR.vio_update(False, c["state"], cov, c["xyz"], c["uv"], c["vel"], c["rgb"], c["cov_rgb"], n_rgb, c["n_new_visited"], c["img"])
    assert t["result"] == r[1] and t["used"] == int(kept.sum())
    assert np.all(np.abs(s - t["state"]) <= 1e-13 * (1 + np.abs(t["state"])))
    assert np.abs(cv - t["cov"]).max() <= 1e-12 * np.abs(t["cov"]).max()


@pytest.mark.parametrize("n", L.LATTICE_SIZES)
def test_lattice_plan_reaches_the_chunk_edges(n):
    """the lattice maps' restated N_rgb put flags on both sides of every chunk boundary at min_views 1, leave a whole chunk
    unflagged at 2 where there are three chunks, flag everything at -1 and 0 and nothing at 3; the sizes take one, two and
    three chunks in publish and save order"""
    counts = L.lattice_counts(n)
    assert counts.max() == 2 and counts.min() == 0
    for order in (0, 1):
        m = n if order == 0 else n - 1
        assert L.chunk_flags(counts, -1, order) == L.chunk_flags(counts, 0, order) and sum(L.chunk_flags(counts, 0, order)) == m
        assert sum(L.chunk_flags(counts, 3, order)) == 0
        idx = np.arange(n) if order == 0 else np.arange(n - 1, 0, -1)
        flagged = counts[idx] >= 1
        for b in range(L.CHUNK, m, L.CHUNK):
            assert flagged[b - 1] and flagged[b], (order, b)
        per = L.chunk_flags(counts, 2, order)
        if len(per) == 3:
            assert 0 in per and any(per), (order, per)
    chunks = {order: len(L.chunk_flags(counts, 0, order)) for order in (0, 1)}
    assert chunks == {L.CHUNK - 1: {0: 1, 1: 1}, L.CHUNK: {0: 1, 1: 1}, L.CHUNK + 1: {0: 2, 1: 1}, 2 * L.CHUNK + 5: {0: 3, 1: 3}}[n]
