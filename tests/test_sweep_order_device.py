"""The sweep's Morton order on the device against the stable sort of restated keys (tests/sweep_order_reference.py).

Every case of tests/sweep_order_cases.py, in each order mode ("cluster_order": 1 the cluster kernel with CTA-local digit
order, 2 its direct scatter, 3 its first version, 0 CUB) and in both states of the library's own check:
  checking   the option set right before the upload: the library runs CUB too and compares (counter -1 while checking;
             0 would mean the cluster order differed and CUB's was kept);
  trusted    after four warm-up uploads (counter 1): nothing compares the cluster kernel's product any more.
Sweeps come from host memory and from a CUDA tensor; one sweep handle serves every case, long and short ones in turn.
The order read back (Sweep.order) is a permutation of range(n) and equals the restated order word for word.

Over the small_world map, three edge sweeps give bit-identical pass sums in all four modes.
"""
import ctypes
import functools

import numpy as np
import pytest

import sweep_order_cases as C
import sweep_order_reference as R

pytestmark = pytest.mark.gpu
MODES = (1, 2, 3, 0)
STATES = ("checking", "trusted")
WARM = np.random.default_rng(5).uniform(-60.0, 60.0, (3000, 3))   # the warm-up sweep of the trusted state
BIG = 2 ** 31 - 1


@functools.lru_cache(maxsize=None)
def _want(name):
    return R.order(C.build(name))


@pytest.fixture(scope="module")
def S():
    from sr_livo_b200 import lio
    ctx = lio.Context(0)
    sw = lio.Sweep(ctx, C.BIG)
    yield ctx, sw
    sw.close()
    ctx.close()


def _enter(ctx, sw, mode, state):
    """Select `mode`; in the trusted state also run the four checked uploads that make the library trust the kernel."""
    ctx.set_option("cluster_order", mode)
    if state == "trusted":
        for _ in range(4):
            sw.upload(WARM)
        assert ctx.counter("cluster_order_active") == (1 if mode else 0)


def _assert_state(ctx, mode, state):
    active = ctx.counter("cluster_order_active")
    if mode == 0:
        assert active == 0
    elif state == "trusted":
        assert active == 1, "a sweep past the cluster's capacity retired the kernel"
    else:
        assert active == -1, f"cluster_order_active {active}: the cluster order differed from CUB's (0) or the checks ran out"


def _assert_order(got, want):
    n = want.size
    assert got.dtype == np.uint32 and got.shape == (n,)
    seen = np.bincount(got.astype(np.int64), minlength=n) if n else np.zeros(0, np.int64)
    assert seen.size == n and np.all(seen == 1), \
        f"not a permutation: {int(np.count_nonzero(seen == 0))} keypoints missing, {int(np.count_nonzero(seen > 1))} repeated, max {int(got.max())}"
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, f"{bad.size} positions differ, first at {bad[0]}: {got[bad[:4]]} vs {want[bad[:4]]}"


@pytest.mark.parametrize("state", STATES)
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", C.names())
def test_order_is_the_stable_order_of_the_restated_keys(S, name, mode, state):
    import torch
    ctx, sw = S
    xyz, want = C.build(name), _want(name)
    _enter(ctx, sw, mode, state)
    sw.upload(xyz)
    got_host = sw.order()
    _assert_state(ctx, mode, state)
    _enter(ctx, sw, mode, state)
    d = torch.from_numpy(xyz).cuda()
    torch.cuda.synchronize()
    sw.set_device(d.data_ptr(), xyz.shape[0])
    got_dev = sw.order()
    del d
    _assert_state(ctx, mode, state)
    _assert_order(got_host, want)
    _assert_order(got_dev, want)


@pytest.mark.parametrize("mode", MODES)
def test_one_handle_long_short_long(S, mode):
    """No key of an earlier upload leaks into a shorter one, and a longer one after it is whole."""
    ctx, sw = S
    _enter(ctx, sw, mode, "trusted")
    for name in ("keys_ties_interleaved", "size_33", "size_131072", "size_1", "coord_special_values_cub", "size_16385",
                 "size_131072"):
        sw.upload(C.build(name))
        _assert_order(sw.order(), _want(name))
        _assert_state(ctx, mode, "trusted")


def test_order_read_back_changes_nothing(S):
    """Reading the order neither recomputes it nor uses up one of the library's four checks."""
    ctx, sw = S
    xyz = C.build("size_16385")
    ctx.set_option("cluster_order", 1)
    sw.upload(xyz)
    launches, active = ctx.kernel_launches, ctx.counter("cluster_order_active")
    a, b = sw.order(), sw.order()
    assert np.array_equal(a, b) and ctx.kernel_launches == launches and ctx.counter("cluster_order_active") == active == -1
    for _ in range(2):
        sw.upload(xyz)
        assert ctx.counter("cluster_order_active") == -1
    sw.upload(xyz)                       # the fourth checked upload
    assert ctx.counter("cluster_order_active") == 1
    _assert_order(sw.order(), _want("size_16385"))


def test_order_read_back_arguments(S):
    from sr_livo_b200 import capi
    ctx, sw = S
    L = capi.lib()
    ctx.set_option("cluster_order", 1)
    xyz = C.build("size_257")
    sw.upload(xyz)
    n = ctypes.c_int64(-1)
    assert L.srl_sweep_download_order(sw.h, None, 0, ctypes.byref(n)) == capi.SRL_OK and n.value == 257
    short = np.full(256, 7, np.uint32)
    assert L.srl_sweep_download_order(sw.h, capi.ptr(short), 256, ctypes.byref(n)) == capi.SRL_BAD_ARG
    assert np.all(short == 7)
    full = np.empty(257, np.uint32)
    assert L.srl_sweep_download_order(sw.h, capi.ptr(full), 257, None) == capi.SRL_OK
    _assert_order(full, _want("size_257"))
    assert L.srl_sweep_download_order(None, None, 0, None) == capi.SRL_BAD_ARG
    sw.upload(np.zeros((0, 3)))
    assert sw.order().shape == (0,)


# ---- the product pass over edge sweeps --------------------------------------------------------------------------------
def _edge_sweeps(sweep):
    rng = np.random.default_rng(90)
    raw = sweep.raw_xyz
    ragged = raw[rng.integers(0, raw.shape[0], 16385)] + rng.normal(0.0, 0.02, (16385, 3))
    g = R.geometry(16385)
    assert g["cta_n"][8] == 1 and not g["cta_n"][9:].any()
    # one cell: a sweep point well inside its cell, 20 000 points around it kept inside the cell
    fr = raw - np.floor(raw)
    p = raw[np.nonzero(np.all((fr > 0.3) & (fr < 0.7), axis=1))[0][0]]
    lo = np.floor(p)
    one = np.clip(p + rng.normal(0.0, 0.05, (20000, 3)), lo, np.nextafter(lo + 1.0, -np.inf))
    assert len(np.unique(R.keys(one))) == 1
    # cell faces and points past +-128 m
    faces = raw.copy()
    faces[::2] = np.round(faces[::2])
    far = raw * (rng.uniform(130.0, 300.0, (raw.shape[0], 1)) / np.linalg.norm(raw, axis=1, keepdims=True))
    edges = np.concatenate([faces, far, raw])
    assert np.all(np.isfinite(edges)) and np.any(np.abs(far) > 128.0) and np.count_nonzero(edges == np.round(edges)) > raw.shape[0]
    return dict(ragged=ragged, one_cell=one, faces_and_far=edges)


@pytest.fixture(scope="module")
def W(small_world):
    from sr_livo_b200 import lio
    L = lio.LioOptimization(max_voxels=1 << 18, sweep_capacity=1 << 17)
    keys, counts, xyz = small_world["omap"].snapshot()
    L.voxel_map.upload(keys, counts, xyz)
    yield L, small_world["sweep"], _edge_sweeps(small_world["sweep"])
    L.close()


@pytest.mark.parametrize("which", ["ragged", "one_cell", "faces_and_far"])
def test_pass_sums_are_the_same_in_every_mode(W, which):
    from sr_livo_b200 import lio
    L, sw, sweeps = W
    xyz = sweeps[which]
    prm = lio.r3live_params(max_num_residuals=BIG)
    out = {}
    for mode in MODES:
        _enter(L.ctx, L.sweep, mode, "trusted")
        L.setKeypoints(xyz)
        _assert_order(L.sweep.order(), R.order(xyz))
        out[mode] = L.buildPlaneResiduals(prm, sw.q_init, sw.t_init, sw.t_last)
        _assert_state(L.ctx, mode, "trusted")
    assert out[0].num_residuals > 0
    for mode in (1, 2, 3):
        assert out[mode].num_residuals == out[0].num_residuals, mode
        assert out[mode].HTH.tobytes() == out[0].HTH.tobytes(), mode
        assert out[mode].HTh.tobytes() == out[0].HTh.tobytes(), mode
