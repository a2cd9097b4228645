"""srl_build_frame (srl_frame.cu) at its edges (tests/build_frame_edge_cases.py) against the reference's own buildFrame
(oracle/_ref/libsrl_build_frame_ref.so) and the model (tests/build_frame_model.py):

- every case equals the reference as test_build_frame_device.py compares it (source indices, stamps and times bit for bit,
  points bit for bit or within 1e-11 m where the undistortion calls libm), NaN by position, and info's engine_words,
  shuffle_rejections and n_timestamped equal the model's;
- the engine-rejection frames run shuffle 1's host redo inside srl_build_frame with shuffle 2 continuing the engine after
  it; rule 1 and shuffle_on_host = 1 equal the model there too;
- one frame object reused across growth, shrinking and growth again; host and device inputs give the same bytes;
- a refused call returns its code and leaves the frame it was given downloading what it held before, grown or not.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import build_frame_edge_cases as E
import build_frame_model as M

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not M.reference_available(), reason="oracle/_ref/libsrl_build_frame_ref.so not built (needs the reference tree)")]
XYZ = ("raw_point", "point", "imu_point")
SCALAR = ("relative_time", "alpha_time", "timestamp")


@pytest.fixture(scope="module")
def L():
    from sr_livo_b200 import lio
    L = lio.LioOptimization(max_voxels=1 << 16, sweep_capacity=8192)
    yield L
    L.close()


@pytest.fixture
def new_frame(L):
    """CloudFrame(L.ctx, capacity) closed at the test's end, also when it fails, so that its device memory goes with the test."""
    from sr_livo_b200 import lio
    made = []

    def make(capacity):
        made.append(lio.CloudFrame(L.ctx, capacity))
        return made[-1]
    yield make
    for f in made:
        f.close()


def call(L, c, frame, raw=None, ts=None, n_states=None):
    """srl_build_frame on case c into frame: (return code, info).  raw / ts: device addresses instead of c's host arrays."""
    from sr_livo_b200 import capi
    h_raw, h_ts = np.ascontiguousarray(c["raw"], np.float64).reshape(-1, 3), np.ascontiguousarray(c["ts"], np.float64)
    states = M.capi_imu_states(c["states"])
    st = (capi.ImuState * len(states))(*states)
    p = capi.BuildFrameParams()
    p.timestamp_begin, p.timestamp_offset = c["begin"], c["offset"]
    p.point_time_enable, p.motion_compensation = int(bool(c["point_time_enable"])), c["motion_compensation"]
    p.index_frame, p.init_num_frames = c["index_frame"], c["init_num_frames"]
    p.init_voxel_size, p.voxel_size, p.prev_time_sweep_end = c["init_voxel_size"], c["voxel_size"], c["prev_time_sweep_end"]
    for name in ("R_il", "t_il", "q_pred", "t_pred"):
        getattr(p, name)[:] = [float(v) for v in np.asarray(c[name], float).reshape(-1)]
    info = capi.BuildFrameInfo()
    rc = capi.lib().srl_build_frame(L.ctx.h, C.c_void_p(raw) if raw else capi.ptr(h_raw), C.c_void_p(ts) if ts else capi.ptr(h_ts),
                                    h_raw.shape[0], st, len(states) if n_states is None else n_states, C.byref(p), frame.h, C.byref(info))
    frame.info = info
    return rc, info


def build(L, c, frame):
    from sr_livo_b200 import capi
    rc, _ = call(L, c, frame)
    assert rc == capi.SRL_OK, capi.lib().srl_last_error(L.ctx.h)
    return frame


def same_bits(a, b) -> bool:
    a, b = np.ascontiguousarray(a, np.float64), np.ascontiguousarray(b, np.float64)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint64), b[~nb].view(np.uint64))


def check_reference(f, ref, name):
    g = f.download()
    assert np.array_equal(g["source_index"], ref["source_index"])
    for k in SCALAR:
        assert same_bits(g[k], ref[k]), k
    for k in XYZ:
        nan = np.isnan(g[k])
        assert np.array_equal(nan, np.isnan(ref[k])), k
        err = np.abs(g[k][~nan] - ref[k][~nan]).max() if (~nan).any() else 0.0
        print(f"{name} {k}: {int((g[k] == ref[k]).all(axis=1).sum())}/{len(g[k])} rows bit for bit, {int(nan.any(axis=1).sum())} NaN rows, "
              f"max |diff| {err:.3g} m")
        assert err <= 1e-11, (k, err)
    same = (g["imu_point"] == ref["imu_point"]).all(axis=1)   # no libm after imu_point
    assert np.array_equal(g["raw_point"][same], ref["raw_point"][same]) and np.array_equal(g["point"][same], ref["point"][same])
    info, sc = f.info, ref["scalars"]
    assert (info.time_sweep_begin, info.time_sweep_end, info.time_frame_begin, info.time_frame_end, info.offset_begin, info.offset_end) == \
        (sc["time_sweep_begin"], sc["time_sweep_end"], sc["time_frame_begin"], sc["time_frame_end"], sc["offset_begin"], sc["offset_end"])
    assert same_bits(info.dt_offset, sc["dt_offset"])
    assert info.n_points == len(ref["source_index"]) == len(f)


def check_model(f, o):
    info = f.info
    assert (info.engine_words, info.shuffle_rejections, info.n_timestamped) == (o["engine_words"], sum(map(len, o["rejected"])), o["n_timestamped"])


def fields(info) -> list:
    """info's fields but the host clock (stage_ms)."""
    return [getattr(info, k) for k, _ in info._fields_ if k != "stage_ms"]


def with_options(L, rule, on_host, fn):
    L.ctx.set_option("shuffle_rule", rule)
    L.ctx.set_option("shuffle_on_host", on_host)
    try:
        return fn()
    finally:
        L.ctx.set_option("shuffle_rule", 0)
        L.ctx.set_option("shuffle_on_host", 0)


@pytest.mark.parametrize("name", E.REJECTION_NAMES)
def test_rejection_frame_equals_the_reference_and_the_model(L, new_frame, name):
    c = E.rejection_case(name)
    o = M.build_frame(c, rule=0)
    f = build(L, c, new_frame(len(c["ts"])))
    check_reference(f, M.ReferenceBuildFrame().build_frame(c), name)
    check_model(f, o)
    info = f.info
    print(f"{name} rule 0: first rejected draw {o['rejected'][0][:1]}, rejections {info.shuffle_rejections}, engine words {info.engine_words}")
    if c["rule"] == 0:
        assert o["rejected"][0][0] == c["first_rejection"] and info.shuffle_rejections >= 1
    # the host Fisher-Yates on the host engine, same rule
    g = with_options(L, 0, 1, lambda: build(L, c, f))
    assert np.array_equal(g.download()["source_index"], o["source_index"])
    check_model(g, o)
    if c["voxel_size"] > 0:   # rule 1: rejects at every one of these sizes
        o1 = M.build_frame(c, rule=1)
        assert o1["rejected"][0][0] == 2_579_772
        for on_host in (0, 1):
            g = with_options(L, 1, on_host, lambda: build(L, c, f))
            assert np.array_equal(g.download()["source_index"], o1["source_index"])
            check_model(g, o1)
        print(f"{name} rule 1: first rejected draw {o1['rejected'][0][:1]}, rejections {g.info.shuffle_rejections}, "
              f"engine words {g.info.engine_words}")


@pytest.mark.parametrize("case", E.edge_cases(), ids=lambda c: c["name"])
def test_edge_case_equals_the_reference_and_the_model(L, new_frame, case):
    f = build(L, case, new_frame(max(len(case["ts"]), 1)))
    check_reference(f, M.ReferenceBuildFrame().build_frame(case), case["name"])
    check_model(f, M.build_frame(case))


def test_one_frame_reused_across_growth(L, new_frame):
    """Created for 4096 points; frame_reserve grows to max(n, 2 * capacity), so the block moves exactly at 5000, 9000 and
    40000."""
    R = M.ReferenceBuildFrame()
    f = new_frame(4096)
    prev = f.device_ptrs()["point"]
    for c, grows in zip(E.reuse_sequence(), (True, False, True, False, True, False, False)):
        build(L, c, f)
        check_reference(f, R.build_frame(c), c["name"])
        check_model(f, M.build_frame(c))
        now = f.device_ptrs()["point"]
        assert (now != prev) == grows, c["name"]
        prev = now


@pytest.mark.parametrize("name", ["nan_stamp_pte0_mc1", "epoch_ends_erase_mc0", "index20", "inf_stamp_pte1", "states4096_mc0"])
def test_host_and_device_inputs_give_the_same_bytes(L, new_frame, name):
    import torch
    from sr_livo_b200 import capi
    c = next(c for c in E.edge_cases() if c["name"] == name)
    want = build(L, c, new_frame(len(c["ts"])))
    d_raw = torch.from_numpy(np.ascontiguousarray(c["raw"], np.float64)).cuda()
    d_ts = torch.from_numpy(np.ascontiguousarray(c["ts"], np.float64)).cuda()
    torch.cuda.synchronize()
    for raw, ts in ((d_raw.data_ptr(), d_ts.data_ptr()), (d_raw.data_ptr(), None), (None, d_ts.data_ptr())):
        f = new_frame(1024)
        rc, info = call(L, c, f, raw=raw, ts=ts)
        assert rc == capi.SRL_OK
        g, w = f.download(), want.download()
        assert all(g[k].tobytes() == w[k].tobytes() for k in g)
        assert fields(info) == fields(want.info)


REFUSALS = [
    ("no_states", dict(), dict(n_states=0)),
    ("init_size_zero", dict(index_frame=19, init_voxel_size=0.0), {}),
    ("init_size_negative", dict(index_frame=0, init_voxel_size=-0.2), {}),
    ("init_size_nan", dict(index_frame=3, init_voxel_size=float("nan")), {}),
    ("imu_walk_4097_states", dict(motion_compensation=0, n_states=4097, edges=False, early=0.0), {}),
]


@pytest.mark.parametrize("grow", [False, True], ids=["fits", "grows"])
@pytest.mark.parametrize("name,case_kw,call_kw", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_refused_call_leaves_the_frame_as_it_was(L, new_frame, name, case_kw, call_kw, grow):
    """The frame holds a build from 3000 points in a 4096-point block; the refused call has 2000 points, or 10000 (past the block:
    the refusal after stage 1 comes after the frame has grown)."""
    from sr_livo_b200 import capi
    f = new_frame(4096)
    build(L, M.make_case("held", n=3000, seed=400, index_frame=4), f)
    before = f.download()
    c = M.make_case(name, n=10000 if grow else 2000, seed=401, **case_kw)
    rc, _ = call(L, c, f, **call_kw)
    assert rc == capi.SRL_BAD_ARG
    print(name, capi.lib().srl_last_error(L.ctx.h))
    after = f.download()
    assert len(f) == len(before["source_index"]) > 0 and all(after[k].tobytes() == before[k].tobytes() for k in before)
