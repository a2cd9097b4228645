"""The Python binding's marshalling, checked on the CPU: lio.lib is replaced by a recorder that logs each C call instead of
running it.  Every public method that takes a buffer is fed numpy arrays of the right dtype and ones that need converting,
CPU torch tensors of the exact and of a wrong dtype, strided views, padded rows and reversed rows; the test checks the
address, count and pitch the C call receives, or the TypeError / ValueError raised before any C call.  Handles are made with
object.__new__, so no library handle and no GPU is involved."""
import ctypes as C
import types

import numpy as np
import pytest

from sr_livo_b200 import capi, lio

torch = pytest.importorskip("torch")


class Recorder:
    """Stands in for the loaded library: each srl_* call is logged as (name, args) and returns SRL_OK, out-parameters left
    at their zeros."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if not name.startswith("srl_"):
            raise AttributeError(name)

        def call(*args):
            self.calls.append((name, args))
            return capi.SRL_OK
        return call

    def only(self, name):
        """the arguments of the one call of `name`, pointers as ints"""
        got = [a for n, a in self.calls if n == name]
        assert len(got) == 1, (name, [n for n, _ in self.calls])
        return [a.value if isinstance(a, C.c_void_p) else a for a in got[0]]


HANDLES = dict(Context="srl_ctx_destroy", VoxelHashMap="srl_map_destroy", ColorVoxelMap="srl_color_map_destroy",
               Sweep="srl_sweep_destroy", CloudFrame="srl_cloud_frame_destroy", LKOpticalFlowKernel="srl_lk_destroy",
               ImageProcessing="srl_image_destroy", OpticalFlowTracker="srl_flow_tracker_destroy",
               CloudProcessing="srl_lidar_destroy")


@pytest.fixture
def rec(monkeypatch):
    r = Recorder()
    monkeypatch.setattr(lio, "lib", lambda: r)
    r.made = []
    yield r
    for o in r.made:     # no fake handle may reach the real library's destroy calls after the recorder is gone
        o.h = None


def make(rec, cls, h=0x1000, **attrs):
    o = object.__new__(cls)
    o.h = C.c_void_p(h)
    o.__dict__.update(attrs)
    rec.made.append(o)
    return o


def objects(rec):
    ctx = make(rec, lio.Context, 0x10, device=0)
    d = dict(ctx=ctx, cmap=make(rec, lio.ColorVoxelMap, 0x20, ctx=ctx, cap=20),
             vmap=make(rec, lio.VoxelHashMap, 0x30, ctx=ctx, cap=20, voxel_size=1.0),
             lk=make(rec, lio.LKOpticalFlowKernel, 0x40, ctx=ctx, params=capi.LkParams(21, 21, 3, 3, 10, 0.05, 8, 1e-4)),
             ip=make(rec, lio.ImageProcessing, 0x50, ctx=ctx), ft=make(rec, lio.OpticalFlowTracker, 0x60, ctx=ctx),
             cp=make(rec, lio.CloudProcessing, 0x70, ctx=ctx), frame=make(rec, lio.CloudFrame, 0x80, ctx=ctx, info=None))
    opt = object.__new__(lio.LioOptimization)
    opt.__dict__.update(ctx=ctx, voxel_map=d["vmap"], sweep=make(rec, lio.Sweep, 0x90, ctx=ctx, capacity=64, n=6),
                        R_imu_lidar=np.eye(3), t_imu_lidar=np.zeros(3), eskf_pro=lio.EskfEstimator())
    d["opt"] = opt
    d["state"] = types.SimpleNamespace(c=capi.VioState())
    d["camera"] = capi.Camera(cols=4, rows=3)
    return d


F32, F64, U8, U32, I32 = np.float32, np.float64, np.uint8, np.uint32, np.int32
ROWS = 5


def _ids(a):
    return np.arange(ROWS, dtype=np.uint32) if a is None else a


# name: (C function, index of the address, index of the count, dtype, values per row, numpy input converted, the call)
# The other arguments are fixed to buffers of ROWS rows that the rule accepts.
def _f32(w):
    return np.zeros((ROWS, w), F32)


ROW_CASES = {
    "VoxelHashMap.insert_published": ("srl_map_insert_published", 1, 2, F64, 3, True,
                                      lambda o, a: o["vmap"].insert_published(a, 0.5, out=_f32(4))),
    "VoxelHashMap.insert_published.out": ("srl_map_insert_published", 6, 7, F32, 4, False,
                                          lambda o, a: o["vmap"].insert_published(np.zeros((ROWS, 3)), 0.5, out=a)),
    "LioOptimization.addPointsToMapPublished": ("srl_map_insert_published", 1, 2, F64, 3, True,
                                                lambda o, a: o["opt"].addPointsToMapPublished(a, 0.5, out=_f32(4))),
    "LioOptimization.addSweepToMapPublished.out": ("srl_map_insert_sweep_published", 8, 9, F32, 4, False,
                                                   lambda o, a: o["opt"].addSweepToMapPublished([0, 0, 0, 1], [0, 0, 0], out=a)),
    "LioOptimization.buildFrame.raw_xyz": ("srl_build_frame", 1, 3, F64, 3, True,
                                           lambda o, a: o["opt"].buildFrame(a, np.zeros(ROWS), [], 0.0, 0.0, 0, frame=o["frame"])),
    "ColorVoxelMap.addPoints": ("srl_color_map_add_points", 1, 2, F64, 3, True, lambda o, a: o["cmap"].addPoints(a)),
    "ColorVoxelMap.exportColorPoints.xyz": ("srl_color_map_export", 3, 5, F32, 3, False,
                                            lambda o, a: o["cmap"].exportColorPoints(xyz=a, rgb=np.zeros((ROWS, 3), U8))),
    "ColorVoxelMap.exportColorPoints.rgb": ("srl_color_map_export", 4, 5, U8, 3, False,
                                            lambda o, a: o["cmap"].exportColorPoints(xyz=_f32(3), rgb=a)),
    "ColorVoxelMap.pubColorPoints.xyz": ("srl_color_map_export", 3, 5, F32, 3, False,
                                         lambda o, a: o["cmap"].pubColorPoints(1, a, np.zeros((ROWS, 3), U8))),
    "ColorVoxelMap.selectPointsForProjection.ids": ("srl_color_map_select_for_projection", 3, 6, U32, 1, False,
                                                    lambda o, a: o["cmap"].selectPointsForProjection(o["camera"], out=(a, None, None))),
    "ColorVoxelMap.selectPointsForProjection.xyz": ("srl_color_map_select_for_projection", 4, 6, F32, 3, False,
                                                    lambda o, a: o["cmap"].selectPointsForProjection(o["camera"], out=(None, a, None))),
    "ColorVoxelMap.selectPointsForProjection.uv": ("srl_color_map_select_for_projection", 5, 6, F32, 2, False,
                                                   lambda o, a: o["cmap"].selectPointsForProjection(o["camera"], out=(None, None, a))),
    "ColorVoxelMap.gatherPoints": ("srl_color_map_gather_points", 1, 2, U32, 1, True, lambda o, a: o["cmap"].gatherPoints(a)),
    "LKOpticalFlowKernel.trackImage.last_pts": ("srl_lk_track_image", 5, 6, F32, 2, False,
                                                lambda o, a: o["lk"].trackImage(np.zeros((3, 4), U8), a)),
    "LKOpticalFlowKernel.trackImage.curr": ("srl_lk_track_image", 7, 6, F32, 2, False,
                                            lambda o, a: o["lk"].trackImage(np.zeros((3, 4), U8), _f32(2), out=(a, np.ones(ROWS, U8)))),
    "ImageProcessing.vioEsikf.ids": ("srl_image_vio_esikf", 3, 6, U32, 1, False,
                                     lambda o, a: o["ip"].vioEsikf(o["cmap"], o["state"], a, _f32(2), np.zeros((ROWS, 2)), 4)),
    "ImageProcessing.vioEsikf.uv": ("srl_image_vio_esikf", 4, 6, F32, 2, False,
                                    lambda o, a: o["ip"].vioEsikf(o["cmap"], o["state"], _ids(None), a, np.zeros((ROWS, 2)), 4)),
    "ImageProcessing.vioEsikf.velocity": ("srl_image_vio_esikf", 5, 6, F64, 2, False,
                                          lambda o, a: o["ip"].vioEsikf(o["cmap"], o["state"], _ids(None), _f32(2), a, 4)),
    "ImageProcessing.vioPhotometric.ids": ("srl_image_vio_photometric", 3, 5, U32, 1, False,
                                           lambda o, a: o["ip"].vioPhotometric(o["cmap"], o["state"], a, np.zeros((ROWS, 2)), 4,
                                                                               np.zeros((3, 4, 3), U8))),
    "ImageProcessing.vioPhotometric.velocity": ("srl_image_vio_photometric", 4, 5, F64, 2, False,
                                                lambda o, a: o["ip"].vioPhotometric(o["cmap"], o["state"], _ids(None), a, 4,
                                                                                    np.zeros((3, 4, 3), U8))),
    "OpticalFlowTracker.init.ids": ("srl_flow_tracker_init", 6, 8, U32, 1, False,
                                    lambda o, a: o["ft"].init(np.zeros((3, 4), U8), 1.0, a, _f32(2))),
    "OpticalFlowTracker.init.uv": ("srl_flow_tracker_init", 7, 8, F32, 2, False,
                                   lambda o, a: o["ft"].init(np.zeros((3, 4), U8), 1.0, _ids(None), a)),
    "OpticalFlowTracker.rejectMatches": ("srl_flow_tracker_reject_matches", 1, 2, U8, 1, True, lambda o, a: o["ft"].rejectMatches(a)),
    "OpticalFlowTracker.removeOutlierUsingRansacPnp": ("srl_flow_tracker_remove_outliers", 1, 2, I32, 1, True,
                                                       lambda o, a: o["ft"].removeOutlierUsingRansacPnp(a)),
    "OpticalFlowTracker.updateAndAppendTrackPoints": ("srl_flow_tracker_update_and_append", 3, 4, U32, 1, False,
                                                      lambda o, a: o["ft"].updateAndAppendTrackPoints(o["camera"], a, 40.0)),
    "device_sort_permutation": ("srl_lidar_sort_replay", 1, 2, F64, 1, True, lambda o, a: lio.device_sort_permutation(o["ctx"], a)),
}

# a dtype of the same kind the rule does not take for each dtype (an int64 for 32-bit ids: the 4-byte float is refusal 2)
OTHER = {F32: np.float64, F64: np.float32, U8: np.int16, U32: np.int64, I32: np.int64}

KINDS = ["numpy", "numpy_converted", "numpy_strided", "list", "torch", "torch_other_dtype", "torch_strided", "torch_int32_ids"]


def _input(kind, dtype, w):
    shape = (ROWS, w) if w > 1 else (ROWS,)
    base = np.arange(ROWS * w, dtype=np.float64).reshape(shape) % 7
    if kind == "numpy":
        return base.astype(dtype)
    if kind == "numpy_converted":
        return base.astype(OTHER[dtype])
    if kind == "numpy_strided":
        return np.repeat(base.astype(dtype), 2, axis=0)[::2]
    if kind == "list":
        return base.astype(dtype).tolist()
    if kind == "torch":
        return torch.from_numpy(base.astype(dtype))
    if kind == "torch_other_dtype":
        return torch.from_numpy(base.astype(OTHER[dtype]))
    if kind == "torch_strided":
        return torch.from_numpy(np.repeat(base.astype(dtype), 2, axis=0))[::2]
    return torch.from_numpy(base.astype(np.int32))


def _address(a):
    return a.ctypes.data if isinstance(a, np.ndarray) else a.data_ptr()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case", list(ROW_CASES))
def test_row_buffers(rec, case, kind):
    fn, i_p, i_n, dtype, w, convert, call = ROW_CASES[case]
    if kind == "torch_int32_ids" and dtype != U32:
        pytest.skip("int32 tensors stand for uint32 ids only")
    if (kind == "torch_strided" and case in ("device_sort_permutation", "ColorVoxelMap.selectPointsForProjection.ids")
            or kind == "torch_other_dtype" and case == "device_sort_permutation"):
        pytest.skip("one of the test_refused_* cases")
    o = objects(rec)
    a = _input(kind, dtype, w)
    taken = kind in ("numpy", "torch", "torch_int32_ids") or (convert and kind.startswith(("numpy", "list")))
    if not taken:
        with pytest.raises(TypeError):
            call(o, a)
        assert not [n for n, _ in rec.calls if n == fn]
        return
    call(o, a)
    args = rec.only(fn)
    assert args[i_n] == ROWS
    if kind in ("numpy", "torch", "torch_int32_ids"):
        assert args[i_p] == _address(a)          # used in place
    else:
        assert args[i_p] not in (None, 0)        # a converted copy


def test_outputs_count_their_rows_and_are_returned_as_given(rec):
    o = objects(rec)
    xyz, rgb = torch.zeros((9, 3), dtype=torch.float32), np.zeros((7, 3), U8)
    gx, gr = o["cmap"].exportColorPoints(xyz=xyz, rgb=rgb)
    args = rec.only("srl_color_map_export")
    assert args[3:6] == [xyz.data_ptr(), rgb.ctypes.data, 7]
    assert gx.untyped_storage().data_ptr() == xyz.data_ptr() and gr.base is rgb       # the first n (here 0) rows of each
    ids, uv = torch.zeros(8, dtype=torch.int32), np.zeros((6, 2), F32)
    o["cmap"].selectPointsForProjection(o["camera"], out=(ids, None, uv))
    args = rec.only("srl_color_map_select_for_projection")
    assert args[3:7] == [ids.data_ptr(), None, uv.ctypes.data, 6]
    with pytest.raises(ValueError):
        o["cmap"].exportColorPoints(xyz=xyz)
    with pytest.raises(ValueError):
        o["lk"].trackImage(np.zeros((3, 4), U8), _f32(2), out=(_f32(2)[:4], np.ones(ROWS, U8)))


def test_defaults_follow_the_input(rec):
    o = objects(rec)
    xyz = torch.zeros((ROWS, 3), dtype=torch.float64)
    stored, cloud = o["vmap"].insert_published(xyz, 0.5)
    args = rec.only("srl_map_insert_published")
    assert isinstance(cloud, torch.Tensor) and cloud.dtype == torch.float32 and args[7] == ROWS
    curr, status, _ = o["lk"].trackImage(np.zeros((3, 4), U8), torch.zeros((ROWS, 2), dtype=torch.float32))
    assert isinstance(curr, torch.Tensor) and tuple(curr.shape) == (ROWS, 2) and tuple(status.shape) == (ROWS,)
    assert bool((status == 1).all())
    curr, status, _ = o["lk"].trackImage(np.zeros((3, 4), U8), _f32(2))
    assert isinstance(curr, np.ndarray) and curr.shape == (ROWS, 2) and status.dtype == U8 and (status == 1).all()
    args = [a for n, a in rec.calls if n == "srl_lk_track_image"][-1]
    assert args[7].value == curr.ctypes.data and args[8].value == status.ctypes.data


def test_length_mismatches_are_refused(rec):
    o = objects(rec)
    with pytest.raises(ValueError):
        o["ip"].vioEsikf(o["cmap"], o["state"], _ids(None), _f32(2)[:4], np.zeros((ROWS, 2)), 4)
    with pytest.raises(ValueError):
        o["ip"].vioPhotometric(o["cmap"], o["state"], _ids(None), np.zeros((4, 2)), 4, np.zeros((3, 4, 3), U8))
    with pytest.raises(ValueError):
        o["ft"].init(np.zeros((3, 4), U8), 1.0, _ids(None), _f32(2)[:4])
    with pytest.raises(ValueError):
        o["cmap"].addPoints(np.zeros(7))                     # not whole rows of 3
    assert rec.calls == []


def test_none_and_empty_lists(rec):
    o = objects(rec)
    o["ft"].rejectMatches(None)
    assert rec.only("srl_flow_tracker_reject_matches")[1:] == [None, 0]
    o["ft"].removeOutlierUsingRansacPnp(None)
    assert rec.only("srl_flow_tracker_remove_outliers")[1:3] == [None, 0]
    rec.calls.clear()
    o["ft"].removeOutlierUsingRansacPnp(np.zeros(0, I32))     # zero inliers, which a NULL pointer would not say
    p, n = rec.only("srl_flow_tracker_remove_outliers")[1:3]
    assert p not in (None, 0) and n == 0


def test_message_bytes(rec):
    o = objects(rec)
    rec_ = np.zeros(4, dtype=[("x", "<f4"), ("pad", "V15")])          # a structured array is taken as its bytes
    o["cp"].livoxHandler(rec_, 1.0)
    assert rec.only("srl_lidar_livox")[1:4] == [rec_.ctypes.data, 4, 19]
    data = torch.zeros(7 * 16, dtype=torch.uint8)
    o["cp"].process(data, dict(point_step=16, x=0, y=4, z=8, time=12), 1.0)
    assert rec.only("srl_lidar_process")[1:3] == [data.data_ptr(), 7]
    rec.calls.clear()
    words = torch.zeros(2 * 12, dtype=torch.int32)                   # 96 bytes of rows padded from 40 to 48 bytes
    o["cp"].process(words, dict(point_step=10, x=0, y=4, z=8, time=-1, width=4, row_step=48), 1.0)
    assert rec.only("srl_lidar_process")[1:3] == [words.data_ptr(), 8]
    with pytest.raises(TypeError):
        o["cp"].livoxHandler(torch.zeros(38, dtype=torch.uint8)[::2], 1.0)
    o["cp"].livoxHandler(np.zeros(76, U8)[::2], 1.0)                # numpy is made contiguous
    assert rec.calls[-1][1][2] == 2


def test_render_image(rec):
    o = objects(rec)
    img = np.zeros((3, 4, 3), U8)
    o["cmap"].renderPointsInRecentVoxel(o["camera"], img, 1.0)
    assert rec.only("srl_color_map_render_recent")[2] == img.ctypes.data
    rec.calls.clear()
    o["cmap"].renderPointsInRecentVoxel(o["camera"], img.astype(np.int64), 1.0)      # numpy is converted
    assert rec.only("srl_color_map_render_recent")[2] not in (None, 0, img.ctypes.data)
    t = torch.zeros((3, 4, 3), dtype=torch.uint8)
    rec.calls.clear()
    o["cmap"].renderPointsInRecentVoxel(o["camera"], t, 1.0)
    assert rec.only("srl_color_map_render_recent")[2] == t.data_ptr()
    rec.calls.clear()
    for bad in (t.float(), torch.zeros((3, 8, 3), dtype=torch.uint8)[:, ::2]):
        with pytest.raises(TypeError):
            o["cmap"].renderPointsInRecentVoxel(o["camera"], bad, 1.0)
    assert rec.calls == []


# (C function, index of the address; cols, rows and pitch follow it; pixel bytes, the call)
IMAGE_CASES = {
    "ImageProcessing.process": ("srl_image_process", 1, 3, lambda o, a: o["ip"].process(a)),
    "ImageProcessing.vioPhotometric": ("srl_image_vio_photometric", 7, 3,
                                       lambda o, a: o["ip"].vioPhotometric(o["cmap"], o["state"], _ids(None), np.zeros((ROWS, 2)), 4, a)),
    "LKOpticalFlowKernel.trackImage": ("srl_lk_track_image", 1, 1, lambda o, a: o["lk"].trackImage(a, _f32(2))),
    "OpticalFlowTracker.init": ("srl_flow_tracker_init", 1, 1, lambda o, a: o["ft"].init(a, 1.0, _ids(None), _f32(2))),
    "OpticalFlowTracker.trackImage": ("srl_flow_tracker_track_image", 1, 1, lambda o, a: o["ft"].trackImage(a, 1.0)),
}
IMAGE_KINDS = ["numpy", "numpy_padded", "torch", "torch_padded", "numpy_other_dtype", "torch_other_dtype", "pixel_stride",
               "channels_strided", "wrong_ndim", "list"]


def _image(kind, px):
    shape = (6, 4, 3) if px == 3 else (6, 4)
    a = (np.arange(int(np.prod(shape))) % 251).astype(U8).reshape(shape)
    wide = np.zeros((6, 9) + shape[2:], U8)
    if kind == "numpy":
        return a
    if kind == "numpy_padded":
        return wide[:, 2:6]
    if kind == "torch":
        return torch.from_numpy(a)
    if kind == "torch_padded":
        return torch.from_numpy(wide)[:, 2:6]
    if kind == "numpy_other_dtype":
        return a.astype(np.int16)
    if kind == "torch_other_dtype":
        return torch.from_numpy(a.astype(np.float32))
    if kind == "pixel_stride":
        return np.zeros((6, 8) + shape[2:], U8)[:, ::2]
    if kind == "channels_strided":
        return np.zeros((6, 4, 6), U8)[:, :, ::2] if px == 3 else np.zeros((6, 4, 2), U8)[:, :, 0]
    if kind == "wrong_ndim":
        return np.zeros((6, 4, 1), U8) if px == 1 else np.zeros((6, 12), U8)
    return a.tolist()


@pytest.mark.parametrize("kind", IMAGE_KINDS)
@pytest.mark.parametrize("case", list(IMAGE_CASES))
def test_images(rec, case, kind):
    fn, i_p, px, call = IMAGE_CASES[case]
    o = objects(rec)
    a = _image(kind, px)
    if kind not in ("numpy", "numpy_padded", "torch", "torch_padded"):
        with pytest.raises(TypeError):
            call(o, a)
        assert not [n for n, _ in rec.calls if n == fn]
        return
    call(o, a)
    args = rec.only(fn)
    pitch = (9 if kind.endswith("padded") else 4) * px
    assert args[i_p:i_p + 4] == [_address(a), 4, 6, pitch]


# ---- the buffers the C ABI would misread, refused before any call ---------------------------------------------------------
def test_refused_sort_keys_of_another_dtype(rec):
    o = objects(rec)
    for keys in (torch.arange(10, dtype=torch.float32), torch.arange(20, dtype=torch.float64)[::2]):
        with pytest.raises(TypeError):
            lio.device_sort_permutation(o["ctx"], keys)
    assert rec.calls == []


def test_refused_float_point_ids(rec):
    o = objects(rec)
    with pytest.raises(TypeError):
        o["cmap"].gatherPoints(torch.zeros(4, dtype=torch.float32))
    assert rec.calls == []


def test_refused_strided_selection_ids(rec):
    o = objects(rec)
    with pytest.raises(TypeError):
        o["cmap"].selectPointsForProjection(o["camera"], out=(torch.zeros(16, dtype=torch.int32)[::2], None, None))
    assert rec.calls == []


@pytest.mark.parametrize("case", list(IMAGE_CASES))
def test_refused_reversed_rows(rec, case):
    fn, _, px, call = IMAGE_CASES[case]
    o = objects(rec)
    with pytest.raises(TypeError):
        call(o, _image("numpy", px)[::-1])
    assert not [n for n, _ in rec.calls if n == fn]


def test_refused_shapes_without_assert(rec):
    """python -O strips assert statements: the image shape of the renderer and the timestamp count of buildFrame are checked
    with ValueError instead"""
    o = objects(rec)
    for img in (np.zeros((3, 5, 3), U8), torch.zeros((4, 4, 3), dtype=torch.uint8)):
        with pytest.raises(ValueError):
            o["cmap"].renderPointsInRecentVoxel(o["camera"], img, 1.0)
    for ts in (np.zeros(ROWS - 1), torch.zeros(ROWS + 1, dtype=torch.float64)):
        with pytest.raises(ValueError):
            o["opt"].buildFrame(torch.zeros((ROWS, 3), dtype=torch.float64), ts, [], 0.0, 0.0, 0, frame=o["frame"])
    with pytest.raises(ValueError):
        o["opt"].buildFrame(np.zeros((ROWS, 3)), np.zeros(ROWS - 1), [], 0.0, 0.0, 0, frame=o["frame"])
    assert rec.calls == []


# ---- handles -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(HANDLES))
def test_close_destroys_once(rec, name):
    cls = getattr(lio, name)
    half = object.__new__(cls)          # a constructor that failed before the handle existed
    half.close()
    half.__del__()
    assert rec.calls == []
    o = make(rec, cls, 0x1234)
    o.close()
    o.close()
    o.__del__()
    assert [(n, a[0].value) for n, a in rec.calls] == [(HANDLES[name], 0x1234)]


def test_destroy_errors_are_swallowed_by_del(rec, monkeypatch):
    def boom():
        raise RuntimeError("library gone")
    o = make(rec, lio.Sweep, 0x99)
    monkeypatch.setattr(lio, "lib", boom)
    o.__del__()
    with pytest.raises(RuntimeError):
        o.close()


def test_lio_optimization_closes_sweep_then_map_then_ctx(rec):
    o = objects(rec)["opt"]
    o.close()
    assert [n for n, _ in rec.calls] == ["srl_sweep_destroy", "srl_map_destroy", "srl_ctx_destroy"]
