"""Host-side mirror of the reference's interface for the scan-matching path, over the C ABI.

Names and argument meaning follow the reference so the parity tests read like its call sites:

  voxelHashMap                          include/cloudMap.h:171          -> VoxelHashMap
  lioOptimization::addPointsToMap       src/lioOptimization.cpp:520-554 -> LioOptimization.addPointsToMap
  lioOptimization::mapSize              src/lioOptimization.cpp:574-581 -> LioOptimization.mapSize
  lioOptimization::buildPlaneResiduals  src/optimize.cpp:18-131         -> LioOptimization.buildPlaneResiduals
  lioOptimization::updateIEKF           src/optimize.cpp:133-314        -> LioOptimization.updateIEKF
  lioOptimization::optimize             src/optimize.cpp:428-448        -> LioOptimization.optimize (keypoints given)
  eskfEstimator (state + observe)       src/eskfEstimator.cpp           -> EskfEstimator
  addPointToPcl / publishCLoudWorld     src/lioOptimization.cpp:432,552 -> LioOptimization.addPointsToMapPublished
  pubColorPoints / saveColorPoints      src/lioOptimization.cpp:1210,1386 -> ColorVoxelMap.pubColorPoints / saveColorPoints
  rgbMapTracker::selectPointsForProjection src/rgbMapTracker.cpp:45     -> ColorVoxelMap.selectPointsForProjection / gatherPoints
  LKOpticalFlowKernel::trackImage       src/lkpyramid.cpp:755           -> LKOpticalFlowKernel.trackImage
  imageProcessing::process (:91-125)    src/imageProcessing.cpp:91      -> ImageProcessing.process
  opticalFlowTracker                    src/opticalFlowTracker.cpp      -> OpticalFlowTracker
  cloudProcessing + getMeasurements' pops src/cloudProcessing.cpp        -> CloudProcessing

Error behaviour: optimizeSummary.success=false <-> OptimizeSummary.success False (SRL_TOO_FEW_RESIDUALS);
the reference's `throw std::runtime_error("error")` on NaN planarity <-> RuntimeError; everything else raises
SrlError.  No CPU fallback exists: without the CUDA library/GPU every call fails loudly.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass, field
from types import SimpleNamespace

import numpy as np

from . import capi
from .capi import (DebugOut, EskfState, Frame, IcpParams, IekfSummary, NormalEq, SrlError, f64, lib, ptr,
                   r3live_params)

NS = capi.NS


def _check(ctx, rc, ok=(capi.SRL_OK,), what=""):
    """Raise SrlError unless rc is in `ok`, with ctx's last error message (or `what` for a call that takes no ctx)."""
    if rc not in ok:
        raise SrlError(rc, lib().srl_last_error(ctx).decode() if ctx else what)
    return rc


def _buffer(a, dtype, width=1, *, convert=False, image=False):
    """The one rule by which a caller's buffer reaches the C ABI, which tells host from device memory per pointer.

    `a` is a numpy array or a torch tensor on the host or a CUDA device.  A tensor must have exactly `dtype` (an int32 tensor
    also stands for uint32 point ids: torch has no uint32 arithmetic) and is never copied.  A numpy array must have exactly
    `dtype`, unless convert=True: then any array-like is copied as C-contiguous `dtype` when it is not so already, and must
    hold whole rows.  dtype None takes any dtype and counts bytes.

    A row buffer is C-contiguous with `width` values per row: returns (a, address, rows).  An image (image=True) is
    (rows, cols), or (rows, cols, width) for width > 1, with contiguous pixels and a row pitch of at least one row of
    pixels, padding allowed: returns (a, address, rows, cols, pitch in bytes).  `a` is the converted copy when one was made,
    which the caller keeps alive across the C call."""
    name = "any" if dtype is None else np.dtype(dtype).name
    if type(a).__module__.split(".")[0] == "torch":
        got = str(a.dtype).replace("torch.", "")
        if dtype is not None and got != name and (name, got) != ("uint32", "int32"):
            raise TypeError(f"expected a torch.{name} tensor, got torch.{got}")
        p, shape, strides, item, contiguous = a.data_ptr(), tuple(a.shape), a.stride(), a.element_size(), a.is_contiguous()
    else:
        if convert:
            a = np.ascontiguousarray(a, dtype)
            if a.size % width:
                raise ValueError(f"expected whole rows of {width} values, got {a.size}")
        if not isinstance(a, np.ndarray) or (dtype is not None and a.dtype != dtype):
            raise TypeError(f"expected a numpy {name} array or a torch tensor, got {type(a).__name__} {getattr(a, 'dtype', '')}")
        p, shape, item, contiguous = a.ctypes.data, a.shape, a.itemsize, a.flags.c_contiguous
        strides = tuple(s // item for s in a.strides)
    if image:
        pixel = (width,) if width > 1 else ()
        if (len(shape) != 2 + len(pixel) or tuple(shape[2:]) != pixel or tuple(strides[1:]) != pixel[::-1] + (1,)
                or strides[0] < shape[1] * width):
            raise TypeError(f"expected a (rows, cols{', %d' % width if pixel else ''}) image with contiguous pixels and rows at "
                            f"least cols pixels apart in address order, got shape {tuple(shape)} and strides {tuple(strides)}")
        return a, p, shape[0], shape[1], strides[0] * item
    if not contiguous:
        raise TypeError("expected a C-contiguous buffer")
    return a, p, math.prod(shape) * item // (width * (1 if dtype is None else item))


def _empty_like_input(a, rows, width, dtype):
    if isinstance(a, np.ndarray):
        return np.empty((rows, width), dtype)
    import torch
    return torch.empty((rows, width), dtype=getattr(torch, np.dtype(dtype).name), device=a.device)


def _device_view(ctx, p, rows, width, dtype):
    """A torch view of `rows` x `width` values of `dtype` at address p of ctx's device (memory the library owns): no copy."""
    import torch
    shape = (rows,) if width == 1 else (rows, width)
    dev = torch.device("cuda", ctx.device)
    if rows == 0:
        return torch.empty(shape, dtype=getattr(torch, np.dtype(dtype).name), device=dev)
    view = dict(shape=shape, typestr=np.dtype(dtype).str, data=(p, False), version=3, strides=None)
    return torch.as_tensor(SimpleNamespace(__cuda_array_interface__=view), device=dev)


class _Handle:
    """Owns the C handle `h`.  close() releases it once with the `_destroy` call, and does nothing on an object whose
    constructor failed before it had one; __del__ closes and swallows errors."""
    _destroy = ""
    h = None

    def close(self):
        if self.h:
            getattr(lib(), self._destroy)(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def write_pcd_xyzrgb(path: str, xyz, rgb) -> None:
    """A binary PCD v0.7 file of pcl::PointXYZRGB points as pcl::io::savePCDFileBinary writes one: fields x y z rgb, 16 bytes per
    point, rgb the float whose bits are a << 24 | r << 16 | g << 8 | b with a = 255 (what PointXYZRGB's constructors set).
    Header layout and alpha are taken from PCL's published sources (DESIGN.md section 2)."""
    xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
    rgb = np.ascontiguousarray(rgb, np.uint8).reshape(-1, 3)
    n = xyz.shape[0]
    assert rgb.shape[0] == n
    rec = np.empty((n, 4), np.float32)
    rec[:, :3] = xyz
    c = rgb.astype(np.uint32)
    rec.view(np.uint32)[:, 3] = (np.uint32(255) << 24) | (c[:, 0] << 16) | (c[:, 1] << 8) | c[:, 2]
    header = ("# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS x y z rgb\nSIZE 4 4 4 4\nTYPE F F F F\nCOUNT 1 1 1 1\n"
              f"WIDTH {n}\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS {n}\nDATA binary\n")
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        f.write(rec.tobytes())


class Context(_Handle):
    """srl_ctx: one per host thread / GPU. `stream` may be a raw cudaStream_t (e.g. torch's current stream)."""

    _destroy = "srl_ctx_destroy"

    def __init__(self, device: int = 0, stream: int | None = None):
        h = C.c_void_p()
        rc = lib().srl_ctx_create(device, C.c_void_p(stream) if stream else None, C.byref(h))
        if rc != capi.SRL_OK:
            raise SrlError(rc, "srl_ctx_create failed: no usable CUDA device (this path has no CPU fallback)")
        self.h = h
        self.device = device

    def synchronize(self):
        _check(self.h, lib().srl_ctx_synchronize(self.h))

    @property
    def kernel_launches(self) -> int:
        return int(lib().srl_ctx_kernel_launches(self.h))

    def set_option(self, name: str, value: int):
        _check(self.h, lib().srl_ctx_set_option(self.h, name.encode(), int(value)))

    def counter(self, name: str) -> int:
        v = C.c_int64(0)
        _check(self.h, lib().srl_ctx_get_counter(self.h, name.encode(), C.byref(v)))
        return v.value

    def set_timing(self, enable: bool = True):
        _check(self.h, lib().srl_ctx_set_timing(self.h, 1 if enable else 0))

    def pass_time(self, reset: bool = False):
        """(summed k1_assoc device time in ms, launches) measured with CUDA events on the ctx stream."""
        ms, n = C.c_double(0), C.c_int64(0)
        _check(self.h, lib().srl_ctx_pass_time(self.h, C.byref(ms), C.byref(n), 1 if reset else 0))
        return ms.value, n.value


class VoxelHashMap(_Handle):
    """HBM-resident voxelHashMap (include/cloudMap.h:171).

    max_voxels is the limit (SRL_MAP_FULL past it); initial_voxels (None = max_voxels) is what is committed at creation,
    and the map grows from there on demand, doubling, up to max_voxels."""

    _destroy = "srl_map_destroy"

    def __init__(self, ctx: Context, voxel_size: float = 1.0, max_num_points_in_voxel: int = 20,
                 max_voxels: int = 1 << 20, initial_voxels: int | None = None):
        self.ctx = ctx
        self.cap = max_num_points_in_voxel
        self.voxel_size = voxel_size
        h = C.c_void_p()
        init = max_voxels if initial_voxels is None else initial_voxels
        _check(ctx.h, lib().srl_map_create_growable(ctx.h, voxel_size, max_num_points_in_voxel, init, max_voxels, C.byref(h)))
        self.h = h

    def capacity(self) -> dict:
        """What is committed now: voxels, slot-table slots and device bytes."""
        v = [C.c_size_t(0) for _ in range(3)]
        _check(self.ctx.h, lib().srl_map_capacity(self.h, *[C.byref(x) for x in v]))
        return dict(zip(("committed_voxels", "slot_capacity", "committed_bytes"), [x.value for x in v]))

    def clear(self):
        _check(self.ctx.h, lib().srl_map_clear(self.h))

    def remove_far(self, location, distance: float) -> int:
        """removePointsFarFromLocation (src/lioOptimization.cpp:556-572): number of voxels erased."""
        loc = f64(location).reshape(3)
        n = C.c_int64(0)
        _check(self.ctx.h, lib().srl_map_remove_far(self.h, ptr(loc), float(distance), C.byref(n)))
        return int(n.value)

    def stats(self):
        nv, npts = C.c_int64(0), C.c_int64(0)
        _check(self.ctx.h, lib().srl_map_stats(self.h, C.byref(nv), C.byref(npts)))
        return nv.value, npts.value

    def upload(self, keys, counts, xyz):
        keys = np.ascontiguousarray(keys, np.int16).reshape(-1, 3)
        counts = np.ascontiguousarray(counts, np.int32)
        xyz = np.ascontiguousarray(xyz, np.float32).reshape(keys.shape[0], self.cap, 3)
        _check(self.ctx.h, lib().srl_map_upload(self.h, ptr(keys), ptr(counts), ptr(xyz), keys.shape[0]))

    def download(self):
        nv, _ = self.stats()
        keys = np.zeros((nv, 3), np.int16)
        counts = np.zeros(nv, np.int32)
        xyz = np.zeros((nv, self.cap, 3), np.float32)
        got = C.c_int64(0)
        _check(self.ctx.h, lib().srl_map_download(self.h, ptr(keys), ptr(counts), ptr(xyz), nv, C.byref(got)))
        return keys, counts, xyz

    def insert(self, xyz_world, min_distance_points: float = 0.15, min_num_points: int = 0) -> int:
        xyz = f64(xyz_world).reshape(-1, 3)
        added = C.c_int64(0)
        _check(self.ctx.h, lib().srl_map_insert(self.h, ptr(xyz), xyz.shape[0], min_distance_points, min_num_points,
                                                C.byref(added)))
        return added.value

    def insert_device(self, d_ptr: int, n: int, min_distance_points: float = 0.15, min_num_points: int = 0) -> int:
        added = C.c_int64(0)
        _check(self.ctx.h, lib().srl_map_insert_device(self.h, C.c_void_p(d_ptr), n, min_distance_points,
                                                       min_num_points, C.byref(added)))
        return added.value

    def insert_published(self, xyz_world, translation_z: float, min_distance_points: float = 0.15, min_num_points: int = 0, out=None):
        """insert + the cloud addPointsToMap publishes (srl_map_insert_published): (points stored, xyzi) with xyzi the first
        n_published rows of `out` (n x 4 float32: x, y, z, intensity, sweep order).  xyz_world is an (n, 3) float64 numpy array
        or torch tensor (host or CUDA); out, when not given, is allocated like the input."""
        xyz_world, p_in, n = _buffer(xyz_world, np.float64, 3, convert=True)
        out = _empty_like_input(xyz_world, n, 4, np.float32) if out is None else out
        _, p_out, max_out = _buffer(out, np.float32, 4)
        added, n_pub = C.c_int64(0), C.c_int64(0)
        _check(self.ctx.h, lib().srl_map_insert_published(self.h, C.c_void_p(p_in), n, min_distance_points, min_num_points, float(translation_z),
                                                          C.c_void_p(p_out), max_out, C.byref(added), C.byref(n_pub)))
        return added.value, out[:n_pub.value]


def r3live_map_options() -> dict:
    """`map_options` of config/r3live.yaml:71-76 (config/ntu.yaml:70-75 has the same values): the colour map's parameters."""
    return dict(size_voxel_map=0.1, max_num_points_in_voxel=50, min_distance_points=0.01, add_point_step=1, pub_point_minimum_views=1)


def r3live_compressed_map_options() -> dict:
    """`map_options` of config/r3live_compressed.yaml:71-76."""
    return dict(size_voxel_map=0.1, max_num_points_in_voxel=100, min_distance_points=0.01, add_point_step=1, pub_point_minimum_views=3)


class ColorVoxelMap(_Handle):
    """color_voxel_map + hashmap_3d_points + rgb_points_vec + voxels_recent_visited (include/lioOptimization.h:275-291,
    include/rgbMapTracker.h:38), fed by the colour branch of addPointsToMap and coloured by renderPointsInRecentVoxel.

    1 <= max_num_points_in_voxel <= 128.  Each point slot costs about 92-124 B of HBM (position, colour state, rgb id, fine
    cell slots), so the shipped map_options (0.1 m, 50 or 100 points) committed for 2^20 voxels take about 5-11 GB.
    max_voxels is the limit; initial_voxels (None = max_voxels) is what is committed at creation, and the map grows from
    there on demand, so a long run needs no guess of its size: initial_voxels=4096, max_voxels=1 << 20.
    The yaml values: ColorVoxelMap(ctx, o["size_voxel_map"], o["max_num_points_in_voxel"], max_voxels, o["min_distance_points"])
    with o = r3live_map_options(), and addPoints(..., add_point_step=o["add_point_step"])."""

    _destroy = "srl_color_map_destroy"

    def __init__(self, ctx: Context, voxel_size: float = 1.0, max_num_points_in_voxel: int = 20, max_voxels: int = 1 << 16,
                 min_distance_points: float = 0.15, initial_voxels: int | None = None):
        self.ctx, self.cap = ctx, max_num_points_in_voxel
        h = C.c_void_p()
        init = max_voxels if initial_voxels is None else initial_voxels
        _check(ctx.h, lib().srl_color_map_create_growable(ctx.h, voxel_size, max_num_points_in_voxel, init, max_voxels, min_distance_points,
                                                          C.byref(h)))
        self.h = h

    def capacity(self) -> dict:
        """What is committed now: voxels, fine-set slots, rgb points and device bytes of the whole colour map."""
        v = [C.c_size_t(0) for _ in range(4)]
        _check(self.ctx.h, lib().srl_color_map_capacity(self.h, *[C.byref(x) for x in v]))
        return dict(zip(("committed_voxels", "fine_capacity", "committed_rgb_points", "committed_bytes"), [x.value for x in v]))

    def stats(self) -> dict:
        v = [C.c_int64(0) for _ in range(5)]
        _check(self.ctx.h, lib().srl_color_map_stats(self.h, *[C.byref(x) for x in v]))
        return dict(zip(("voxels", "points", "rgb_points", "recent", "new_recent"), [x.value for x in v]))

    def addPoints(self, xyz_world, add_point_step: int = 1, time_sweep_end: float = 1.0, time_last_process: float = 0.0,
                  to_rendering: bool = True) -> int:
        """the loop of src/lioOptimization.cpp:533-551 over the registered frame: an (n, 3) float64 numpy array or torch tensor
        (host or CUDA).  Returns the number of points stored."""
        xyz_world, p, n = _buffer(xyz_world, np.float64, 3, convert=True)
        stored = C.c_int64(0)
        _check(self.ctx.h, lib().srl_color_map_add_points(self.h, C.c_void_p(p), n, add_point_step, time_sweep_end, time_last_process,
                                                          1 if to_rendering else 0, C.byref(stored)))
        return stored.value

    def renderPointsInRecentVoxel(self, camera: "capi.Camera", image_bgr, obs_time: float) -> int:
        """rgbMapTracker::renderPointsInRecentVoxel (srl_color_map_render_recent) with a (rows, cols, 3) BGR8 image: a numpy array,
        or a contiguous torch.uint8 tensor on the host or a CUDA device (ImageProcessing.process's rgb output as it is); returns
        render_point_count.  camera.fov_margin must be >= 0 (SRL_BAD_ARG otherwise, NaN included, and the map is untouched):
        a negative margin would sample outside the image, which the reference leaves undefined.  The selection
        (selectPointsForProjection) still takes negative margins."""
        if tuple(np.shape(image_bgr)) != (camera.rows, camera.cols, 3):
            raise ValueError(f"expected a ({camera.rows}, {camera.cols}, 3) image, got {tuple(np.shape(image_bgr))}")
        image_bgr, p_img, _ = _buffer(image_bgr, np.uint8, 3, convert=True)
        n = C.c_int64(0)
        _check(self.ctx.h, lib().srl_color_map_render_recent(self.h, C.byref(camera), C.c_void_p(p_img), float(obs_time), C.byref(n)))
        return n.value

    def exportColorPoints(self, min_views: int = 1, order: int = 0, xyz=None, rgb=None):
        """srl_color_map_export: the rgb_points_vec entries with N_rgb >= min_views as ((n, 3) float32 positions, (n, 3) uint8 r, g, b).
        order 0 is pubColorPoints' order, order 1 saveColorPoints'.  xyz / rgb (numpy arrays or torch tensors, host or CUDA) receive
        the points when given (the first n rows are returned), else numpy arrays are allocated."""
        if (xyz is None) != (rgb is None):
            raise ValueError("give both xyz and rgb, or neither")
        n = C.c_int64(0)
        if xyz is None:
            _check(self.ctx.h, lib().srl_color_map_export(self.h, int(min_views), int(order), None, None, 0, C.byref(n)))
            xyz, rgb = np.empty((n.value, 3), np.float32), np.empty((n.value, 3), np.uint8)
        _, p_xyz, cap = _buffer(xyz, np.float32, 3)
        _, p_rgb, cap_rgb = _buffer(rgb, np.uint8, 3)
        _check(self.ctx.h, lib().srl_color_map_export(self.h, int(min_views), int(order), C.c_void_p(p_xyz), C.c_void_p(p_rgb),
                                                      min(cap, cap_rgb), C.byref(n)))
        return xyz[:n.value], rgb[:n.value]

    def countColorPoints(self, min_views: int = 1, order: int = 0) -> int:
        """How many points exportColorPoints(min_views, order) hands out."""
        n = C.c_int64(0)
        _check(self.ctx.h, lib().srl_color_map_export(self.h, int(min_views), int(order), None, None, 0, C.byref(n)))
        return n.value

    def pubColorPoints(self, min_views: int = 1, xyz=None, rgb=None):
        """pubColorPoints (src/lioOptimization.cpp:1210-1241): rgb_points_vec from index 0 up (one round of threadPubColorPoints'
        topics, concatenated).  min_views is map_options.pub_point_minimum_views: 1 in r3live_map_options(), 3 in
        r3live_compressed_map_options()."""
        return self.exportColorPoints(min_views, 0, xyz, rgb)

    def saveColorPoints(self, path: str | None = None, min_views: int = 1):
        """saveColorPoints (src/lioOptimization.cpp:1386-1426): rgb_points_vec from the last index down to 1 (index 0 is never
        saved); with a path, also writes the binary PCD (write_pcd_xyzrgb) the reference writes to rgb_map.pcd."""
        xyz, rgb = self.exportColorPoints(min_views, 1)
        if path is not None:
            write_pcd_xyzrgb(path, xyz, rgb)
        return xyz, rgb

    def selectPointsForProjection(self, camera: "capi.Camera", minimum_dis: float = 5.0, skip_step: int = 1, use_all_points: bool = False,
                                  minimum_depth: float = 0.1, maximum_depth: float = 200.0, out=None):
        """rgbMapTracker::selectPointsForProjection (src/rgbMapTracker.cpp:45-152, srl_color_map_select_for_projection):
        (ids, xyz, uv) of the selected points in point_index order — uint32 point ids, (n, 3) float32 positions, (n, 2) float32
        cv::Point2f(u_f, v_f).  refreshPointsForProjection is minimum_dis=10 from a camera with fov_margin -0.4; the first image
        uses minimum_dis = track_windows_size / image_scale_factor.  out = (ids, xyz, uv) buffers (numpy arrays or torch tensors,
        host or CUDA; any may be None) receive the points and their first n rows are returned; without it numpy arrays are made."""
        prm = capi.ProjectionParams(float(minimum_dis), int(skip_step), 1 if use_all_points else 0, float(minimum_depth), float(maximum_depth))
        n = C.c_int64(0)
        if out is None:
            st = self.stats()
            total = st["rgb_points"] if use_all_points or st["recent"] == 0 else st["recent"]
            bound = (total + max(int(skip_step), 1) - 1) // max(int(skip_step), 1)
            out = (np.empty(bound, np.uint32), np.empty((bound, 3), np.float32), np.empty((bound, 2), np.float32))
        ids, xyz, uv = out
        addrs, caps = [], []
        for a, dt, w in ((ids, np.uint32, 1), (xyz, np.float32, 3), (uv, np.float32, 2)):
            if a is None:
                addrs.append(None)
                continue
            _, p, rows = _buffer(a, dt, w)
            addrs.append(C.c_void_p(p))
            caps.append(rows)
        _check(self.ctx.h, lib().srl_color_map_select_for_projection(self.h, C.byref(camera), C.byref(prm), addrs[0], addrs[1], addrs[2],
                                                                      min(caps) if caps else 0, C.byref(n)))
        k = n.value
        return tuple(None if a is None else a[:k] for a in (ids, xyz, uv))

    def countPointsForProjection(self, camera: "capi.Camera", minimum_dis: float = 5.0, skip_step: int = 1, use_all_points: bool = False,
                                 minimum_depth: float = 0.1, maximum_depth: float = 200.0) -> int:
        """How many points selectPointsForProjection with the same arguments returns."""
        prm = capi.ProjectionParams(float(minimum_dis), int(skip_step), 1 if use_all_points else 0, float(minimum_depth), float(maximum_depth))
        n = C.c_int64(0)
        _check(self.ctx.h, lib().srl_color_map_select_for_projection(self.h, C.byref(camera), C.byref(prm), None, None, None, 0, C.byref(n)))
        return n.value

    def gatherPoints(self, ids) -> dict:
        """srl_color_map_gather_points: the state of each point id as numpy arrays — xyz (n, 3) float32, rgb (n, 3) int16 (the BGR
        state), n_rgb (n,) int16, cov (n, 3) float32, key_index (n, 4) int16 (voxel key, index in block).  ids: a uint32 numpy array
        or a torch tensor (host or CUDA; int32 holds the ids' bits).  An id that names no stored point raises SrlError."""
        ids, p, n = _buffer(ids, np.uint32, convert=True)
        out = dict(xyz=np.empty((n, 3), np.float32), rgb=np.empty((n, 3), np.int16), n_rgb=np.empty(n, np.int16),
                   cov=np.empty((n, 3), np.float32), key_index=np.empty((n, 4), np.int16))
        _check(self.ctx.h, lib().srl_color_map_gather_points(self.h, C.c_void_p(p), n, *[ptr(out[k]) for k in ("xyz", "rgb", "n_rgb", "cov",
                                                                                                                "key_index")]))
        return out

    def download(self) -> dict:
        """voxel contents + colour state (block order) + the two lists."""
        st = self.stats()
        nv, cap = st["voxels"], self.cap
        out = dict(keys=np.zeros((nv, 3), np.int16), counts=np.zeros(nv, np.int32), xyz=np.zeros((nv, cap, 3), np.float32),
                   rgb=np.zeros((nv, cap, 3), np.int16), n_rgb=np.zeros((nv, cap), np.int16), cov=np.zeros((nv, cap, 3), np.float32),
                   obs_dist=np.zeros((nv, cap)), last_obs=np.zeros((nv, cap)), last_visited=np.zeros(nv),
                   rgb_points=np.zeros((st["rgb_points"], 4), np.int16), recent=np.zeros((st["recent"], 3), np.int16))
        vox = C.c_void_p(lib().srl_color_map_voxels(self.h))
        got = C.c_int64(0)
        _check(self.ctx.h, lib().srl_map_download(vox, ptr(out["keys"]), ptr(out["counts"]), ptr(out["xyz"]), nv, C.byref(got)))
        _check(self.ctx.h, lib().srl_color_map_download_state(self.h, nv, ptr(out["rgb"]), ptr(out["n_rgb"]), ptr(out["cov"]), ptr(out["obs_dist"]),
                                                              ptr(out["last_obs"]), ptr(out["last_visited"])))
        _check(self.ctx.h, lib().srl_color_map_download_lists(self.h, ptr(out["rgb_points"]), ptr(out["recent"])))
        return out


class Sweep(_Handle):
    """The keypoints of one reconstructed sweep, resident in HBM (raw LiDAR-frame points, FP64)."""

    _destroy = "srl_sweep_destroy"

    def __init__(self, ctx: Context, capacity: int):
        self.ctx = ctx
        self.capacity = capacity
        self.n = 0
        h = C.c_void_p()
        _check(ctx.h, lib().srl_sweep_create(ctx.h, capacity, C.byref(h)))
        self.h = h

    def upload(self, raw_xyz):
        raw = f64(raw_xyz).reshape(-1, 3)
        _check(self.ctx.h, lib().srl_sweep_upload(self.h, ptr(raw), raw.shape[0]))
        self.n = raw.shape[0]

    def set_device(self, d_ptr: int, n: int):
        _check(self.ctx.h, lib().srl_sweep_set_device(self.h, C.c_void_p(d_ptr), n))
        self.n = n

    def set_shard(self, begin: int, end: int):
        _check(self.ctx.h, lib().srl_sweep_set_shard(self.h, begin, end))

    def order(self) -> np.ndarray:
        """The Morton order the passes visit the keypoints in: (n,) uint32, entry s = the keypoint at sorted position s."""
        n = C.c_int64(0)
        _check(self.ctx.h, lib().srl_sweep_download_order(self.h, None, 0, C.byref(n)))
        out = np.empty(n.value, np.uint32)
        _check(self.ctx.h, lib().srl_sweep_download_order(self.h, ptr(out), out.size, C.byref(n)))
        return out


class CloudFrame(_Handle):
    """The frame buildFrame hands to stateEstimation, resident in HBM (srl_cloud_frame), final frame order."""

    _destroy = "srl_cloud_frame_destroy"
    FIELDS = (("raw_point", 3, np.float64), ("point", 3, np.float64), ("imu_point", 3, np.float64), ("relative_time", 1, np.float64),
              ("alpha_time", 1, np.float64), ("timestamp", 1, np.float64), ("source_index", 1, np.int32))

    def __init__(self, ctx: Context, capacity: int = 1 << 17):
        self.ctx = ctx
        self.info = None
        h = C.c_void_p()
        _check(ctx.h, lib().srl_cloud_frame_create(ctx.h, capacity, C.byref(h)))
        self.h = h

    def __len__(self) -> int:
        return int(lib().srl_cloud_frame_size(self.h))

    def device_ptrs(self) -> dict:
        """Device addresses of the fields (valid until the next build into this frame)."""
        p = capi.CloudFramePtrs()
        _check(self.ctx.h, lib().srl_cloud_frame_device(self.h, C.byref(p)))
        return {name: getattr(p, name) for name, _, _ in self.FIELDS}

    def download(self) -> dict:
        n = len(self)
        out = {name: np.zeros((n, k) if k > 1 else n, dt) for name, k, dt in self.FIELDS}
        _check(self.ctx.h, lib().srl_cloud_frame_download(self.h, *[ptr(out[name]) for name, _, _ in self.FIELDS]))
        return out


@dataclass
class EskfEstimator:
    """eskfEstimator state (src/eskfEstimator.cpp:3-21); q = (x, y, z, w)."""
    p: np.ndarray = field(default_factory=lambda: np.zeros(3))
    q: np.ndarray = field(default_factory=lambda: np.array([0.0, 0.0, 0.0, 1.0]))
    v: np.ndarray = field(default_factory=lambda: np.zeros(3))
    ba: np.ndarray = field(default_factory=lambda: np.zeros(3))
    bg: np.ndarray = field(default_factory=lambda: np.zeros(3))
    g: np.ndarray = field(default_factory=lambda: np.array([0.0, 0.0, 9.81]))
    cov: np.ndarray = field(default_factory=lambda: np.eye(NS))

    def to_c(self) -> EskfState:
        return capi.eskf_to_c(self.p, self.q, self.v, self.ba, self.bg, self.g, self.cov)

    @staticmethod
    def from_c(s: EskfState) -> "EskfEstimator":
        return EskfEstimator(**capi.eskf_from_c(s))

    def observe(self, d_x) -> "EskfEstimator":
        """eskfEstimator::observe (src/eskfEstimator.cpp:219-230)."""
        s = self.to_c()
        d = f64(d_x)
        _check(None, lib().srl_eskf_observe(C.byref(s), ptr(d)), what="srl_eskf_observe")
        return EskfEstimator.from_c(s)


@dataclass
class OptimizeSummary:
    """optimizeSummary (include/lioOptimization.h) + what the GPU pass reports."""
    success: bool
    num_residuals_used: int
    passes_run: int = 1
    converged: bool = False
    trace: np.ndarray | None = None


@dataclass
class PlaneResiduals:
    HTH: np.ndarray
    HTh: np.ndarray
    loss_sum: float
    num_residuals: int
    num_full_neighborhoods: int
    num_candidates_scanned: int
    success: bool
    world_xyz: np.ndarray | None = None
    status: np.ndarray | None = None
    nbr: np.ndarray | None = None
    nbr_dist: np.ndarray | None = None
    plane: np.ndarray | None = None


def make_frame(q_cur, t_cur, t_last, R_il=None, t_il=None) -> Frame:
    fr = Frame()
    for name, val, n in (("q_cur", q_cur, 4), ("t_cur", t_cur, 3), ("t_last", t_last, 3),
                         ("R_il", np.eye(3) if R_il is None else R_il, 9),
                         ("t_il", np.zeros(3) if t_il is None else t_il, 3)):
        a = f64(val).reshape(-1)
        assert a.size == n, name
        for i in range(n):
            getattr(fr, name)[i] = a[i]
    return fr


class LioOptimization:
    """The scan-matching members of `class lioOptimization` (include/lioOptimization.h:334-353) on one GPU."""

    def __init__(self, device: int = 0, stream: int | None = None, max_voxels: int = 1 << 20,
                 sweep_capacity: int = 1 << 17, size_voxel_map: float = 1.0, max_num_points_in_voxel: int = 20,
                 R_imu_lidar=None, t_imu_lidar=None, initial_voxels: int | None = None):
        self.ctx = Context(device, stream)
        self.voxel_map = VoxelHashMap(self.ctx, size_voxel_map, max_num_points_in_voxel, max_voxels, initial_voxels)
        self.sweep = Sweep(self.ctx, sweep_capacity)
        self.R_imu_lidar = np.eye(3) if R_imu_lidar is None else f64(R_imu_lidar).reshape(3, 3)
        self.t_imu_lidar = np.zeros(3) if t_imu_lidar is None else f64(t_imu_lidar)
        self.eskf_pro = EskfEstimator()

    def close(self):
        self.sweep.close()
        self.voxel_map.close()
        self.ctx.close()

    # ---- src/lioOptimization.cpp:520-554 (voxel_size is the map's own)
    def addPointsToMap(self, points_world, min_distance_points: float = 0.15, min_num_points: int = 0) -> int:
        return self.voxel_map.insert(points_world, min_distance_points, min_num_points)

    def addSweepToMap(self, frame_q, frame_t, min_distance_points: float = 0.15, min_num_points: int = 0) -> int:
        """stateEstimation's tail (src/lioOptimization.cpp:1027): the resident sweep, re-transformed with the final pose
        (src/optimize.cpp:441-445), goes into the map without leaving the device."""
        q, t = f64(frame_q), f64(frame_t)
        R, ti = f64(self.R_imu_lidar).reshape(9), f64(self.t_imu_lidar)
        added = C.c_int64(0)
        _check(self.ctx.h, lib().srl_map_insert_sweep(self.voxel_map.h, self.sweep.h, ptr(q), ptr(t), ptr(R), ptr(ti),
                                                      min_distance_points, min_num_points, C.byref(added)))
        return added.value

    def addPointsToMapPublished(self, points_world, translation_z: float, min_distance_points: float = 0.15, min_num_points: int = 0,
                                out=None):
        """addPointsToMap and the cloud it publishes (publishCLoudWorld, src/lioOptimization.cpp:552): (points stored, xyzi), xyzi
        (n_published, 4) float32 x, y, z, intensity = 50 * (z - translation_z), in sweep order (VoxelHashMap.insert_published)."""
        return self.voxel_map.insert_published(points_world, translation_z, min_distance_points, min_num_points, out)

    def addSweepToMapPublished(self, frame_q, frame_t, min_distance_points: float = 0.15, min_num_points: int = 0, out=None):
        """addSweepToMap and the cloud it publishes, intensity relative to frame_t[2] (srl_map_insert_sweep_published).  out: n x 4
        float32 (numpy or torch, host or CUDA); a numpy array is allocated when not given."""
        q, t = f64(frame_q), f64(frame_t)
        R, ti = f64(self.R_imu_lidar).reshape(9), f64(self.t_imu_lidar)
        out = np.empty((self.sweep.n, 4), np.float32) if out is None else out
        _, p_out, max_out = _buffer(out, np.float32, 4)
        added, n_pub = C.c_int64(0), C.c_int64(0)
        _check(self.ctx.h, lib().srl_map_insert_sweep_published(self.voxel_map.h, self.sweep.h, ptr(q), ptr(t), ptr(R), ptr(ti),
                                                                min_distance_points, min_num_points, C.c_void_p(p_out), max_out,
                                                                C.byref(added), C.byref(n_pub)))
        return added.value, out[:n_pub.value]

    # ---- src/lioOptimization.cpp:786-893
    def buildFrame(self, raw_xyz, timestamp, imu_states, timestamp_begin: float, timestamp_offset: float, index_frame: int,
                   q_pred=None, t_pred=None, point_time_enable: bool = True, motion_compensation: int = 1, init_num_frames: int = 20,
                   init_voxel_size: float = 0.2, voxel_size: float = 0.5, prev_time_sweep_end: float = 0.0,
                   frame: "CloudFrame | None" = None) -> CloudFrame:
        """buildFrame over a cut sweep: raw_xyz n*3 and timestamp n as host arrays, or torch tensors (host or CUDA, read in place;
        CloudProcessing.cut(t, device=True) gives such views).  imu_states: a list of capi.ImuState.  motion_compensation: 0 IMU, 1 CONSTANT_VELOCITY.  Returns the
        device-resident frame (into `frame` when given), with the cloudFrame scalars in frame.info (capi.BuildFrameInfo)."""
        raw_xyz, p_raw, n = _buffer(raw_xyz, np.float64, 3, convert=True)
        timestamp, p_ts, n_ts = _buffer(timestamp, np.float64, convert=True)
        if n_ts != n:
            raise ValueError(f"raw_xyz holds {n} points and timestamp {n_ts}")
        states = (capi.ImuState * len(imu_states))(*imu_states)
        p = capi.BuildFrameParams()
        p.timestamp_begin, p.timestamp_offset = float(timestamp_begin), float(timestamp_offset)
        p.point_time_enable, p.motion_compensation = int(bool(point_time_enable)), int(motion_compensation)
        p.index_frame, p.init_num_frames = int(index_frame), int(init_num_frames)
        p.init_voxel_size, p.voxel_size = float(init_voxel_size), float(voxel_size)
        p.prev_time_sweep_end = float(prev_time_sweep_end)
        for name, val in (("R_il", f64(self.R_imu_lidar).reshape(9)), ("t_il", f64(self.t_imu_lidar)),
                          ("q_pred", f64([0, 0, 0, 1] if q_pred is None else q_pred)), ("t_pred", f64(np.zeros(3) if t_pred is None else t_pred))):
            getattr(p, name)[:] = list(val)
        frame = frame if frame is not None else CloudFrame(self.ctx, max(n, 1))
        info = capi.BuildFrameInfo()
        _check(self.ctx.h, lib().srl_build_frame(self.ctx.h, C.c_void_p(p_raw), C.c_void_p(p_ts), n, states, len(imu_states), C.byref(p),
                                                 frame.h, C.byref(info)))
        frame.info = info
        return frame

    # ---- src/lioOptimization.cpp:574-581
    def mapSize(self) -> int:
        return self.voxel_map.stats()[1]

    # ---- src/lioOptimization.cpp:556-572
    def removePointsFarFromLocation(self, location, distance: float) -> int:
        return self.voxel_map.remove_far(location, distance)

    # ---- src/utility.cpp:188-201, called at src/optimize.cpp:431
    def gridSampling(self, points_world, size_voxel_subsampling: float) -> np.ndarray:
        """Frame indices of the keypoints (first point of every cell), in the reference's order."""
        xyz = f64(points_world).reshape(-1, 3)
        out = np.zeros(xyz.shape[0], np.uint32)
        m = C.c_size_t(0)
        _check(self.ctx.h, lib().srl_grid_sampling(self.ctx.h, ptr(xyz), xyz.shape[0], size_voxel_subsampling, ptr(out), C.byref(m)))
        return out[:m.value].copy()

    # ---- src/utility.cpp:203-332 (row N3): undistortion and the sweep-end re-expression
    @staticmethod
    def _imu_states(states):
        """states: sequence of dicts / objects with timestamp, quat (x,y,z,w), trans, vel, un_acc, un_gyr."""
        from .capi import ImuState
        arr = (ImuState * len(states))()
        for a, s_ in zip(arr, states):
            g = (lambda k: s_[k]) if isinstance(s_, dict) else (lambda k: getattr(s_, k))
            a.timestamp = float(g("timestamp"))
            for name, m in (("quat", 4), ("trans", 3), ("vel", 3), ("un_acc", 3), ("un_gyr", 3)):
                v = np.asarray(g(name), np.float64).reshape(m)
                getattr(a, name)[:] = v.tolist()
        return arr

    def distortFrameByConstant(self, raw_xyz, relative_time_ms, imu_states, time_frame_begin: float) -> np.ndarray:
        raw = f64(raw_xyz).reshape(-1, 3)
        rel = f64(relative_time_ms).reshape(-1)
        st = self._imu_states(imu_states)
        out = np.zeros_like(raw)
        R, t = f64(self.R_imu_lidar).reshape(9), f64(self.t_imu_lidar)
        _check(self.ctx.h, lib().srl_distort_frame_by_constant(self.ctx.h, ptr(raw), ptr(rel), raw.shape[0], C.cast(st, C.c_void_p),
                                                               len(imu_states), float(time_frame_begin), ptr(R), ptr(t), ptr(out)))
        return out

    def distortFrameByImu(self, raw_xyz, relative_time_ms, imu_states, time_frame_begin: float, imu_xyz_in=None):
        """Returns (imu_xyz, n_written); imu_xyz_in supplies the values kept by points the reference's walk never reaches."""
        raw = f64(raw_xyz).reshape(-1, 3)
        rel = f64(relative_time_ms).reshape(-1)
        st = self._imu_states(imu_states)
        out = np.zeros_like(raw) if imu_xyz_in is None else f64(imu_xyz_in).reshape(-1, 3).copy()
        nw = C.c_int64(0)
        R, t = f64(self.R_imu_lidar).reshape(9), f64(self.t_imu_lidar)
        _check(self.ctx.h, lib().srl_distort_frame_by_imu(self.ctx.h, ptr(raw), ptr(rel), raw.shape[0], C.cast(st, C.c_void_p),
                                                          len(imu_states), float(time_frame_begin), ptr(R), ptr(t), ptr(out), C.byref(nw)))
        return out, int(nw.value)

    def transformAllImuPoint(self, imu_xyz, last_imu_state) -> np.ndarray:
        imu = f64(imu_xyz).reshape(-1, 3)
        st = self._imu_states([last_imu_state])
        out = np.zeros_like(imu)
        R, t = f64(self.R_imu_lidar).reshape(9), f64(self.t_imu_lidar)
        _check(self.ctx.h, lib().srl_transform_all_imu_point(self.ctx.h, ptr(imu), imu.shape[0], C.cast(st, C.c_void_p), ptr(R), ptr(t), ptr(out)))
        return out

    def setKeypoints(self, raw_xyz):
        """std::vector<point3D> keypoints (raw_point members), uploaded once per sweep."""
        self.sweep.upload(raw_xyz)

    # ---- src/optimize.cpp:18-131 (+ :160-170,:235,:239)
    def buildPlaneResiduals(self, cur_icp_options: IcpParams, q_cur, t_cur, t_last, debug: bool = False) -> PlaneResiduals:
        fr = make_frame(q_cur, t_cur, t_last, self.R_imu_lidar, self.t_imu_lidar)
        ne = NormalEq()
        n = self.sweep.n
        K = cur_icp_options.max_number_neighbors
        arrs = {}
        dbg = None
        if debug:
            arrs = dict(world_xyz=np.zeros((n, 3)), status=np.zeros(n, np.int32), nbr=np.zeros((n, K, 4), np.int16),
                        nbr_dist=np.zeros((n, K)), plane=np.zeros((n, 16)))
            dbg = DebugOut(*[ptr(arrs[k]) for k in ("world_xyz", "status", "nbr", "nbr_dist", "plane")])
        rc = lib().srl_build_plane_residuals(self.ctx.h, self.voxel_map.h, self.sweep.h, C.byref(fr),
                                             C.byref(cur_icp_options), C.byref(ne),
                                             C.byref(dbg) if dbg is not None else None)
        if rc == capi.SRL_NAN_PLANARITY:
            raise RuntimeError("error")   # src/optimize.cpp:348-350
        _check(self.ctx.h, rc, ok=(capi.SRL_OK, capi.SRL_TOO_FEW_RESIDUALS))
        return PlaneResiduals(HTH=np.array(ne.HTH).reshape(6, 6), HTh=np.array(ne.HTh), loss_sum=ne.loss_sum,
                              num_residuals=ne.num_residuals, num_full_neighborhoods=ne.num_full_neighborhoods,
                              num_candidates_scanned=ne.num_candidates_scanned, success=(rc == capi.SRL_OK), **arrs)

    def _call_buffers(self):
        """Argument marshalling of the per-sweep calls, built once: a persistent srl_eskf_state with a float64 view over it,
        one float64 block for frame_q | frame_t | t_last | R_il | t_il with precomputed pointers, one srl_iekf_summary.
        (Fresh numpy arrays + ctypes pointer objects per call were ~20 us of Python inside every timed sweep.)"""
        b = getattr(self, "_bufs", None)
        if b is None:
            st = capi.EskfState()
            blk = np.zeros(4 + 3 + 3 + 9 + 3, np.float64)
            base = blk.ctypes.data
            b = self._bufs = dict(st=st, st_view=np.frombuffer(st, dtype=np.float64), st_ref=C.byref(st), blk=blk,
                                  p_fq=C.c_void_p(base), p_ft=C.c_void_p(base + 32), p_tl=C.c_void_p(base + 56),
                                  p_R=C.c_void_p(base + 80), p_ti=C.c_void_p(base + 152), summ=IekfSummary())
            b["summ_ref"] = C.byref(b["summ"])
        return b

    def _marshal(self, b, t_last, frame_q, frame_t):
        e, v, blk = self.eskf_pro, b["st_view"], b["blk"]
        v[0:3] = e.p; v[3:7] = e.q; v[7:10] = e.v; v[10:13] = e.ba; v[13:16] = e.bg; v[16:19] = e.g
        v[19:] = np.asarray(e.cov, np.float64).reshape(-1)
        blk[0:4] = e.q if frame_q is None else frame_q
        blk[4:7] = e.p if frame_t is None else frame_t
        blk[7:10] = t_last
        blk[10:19] = np.asarray(self.R_imu_lidar, np.float64).reshape(-1)
        blk[19:22] = self.t_imu_lidar

    def _unmarshal(self, b, rc):
        if rc == capi.SRL_NAN_PLANARITY:
            raise RuntimeError("error")
        _check(self.ctx.h, rc, ok=(capi.SRL_OK, capi.SRL_TOO_FEW_RESIDUALS))
        a = b["st_view"].copy()
        self.eskf_pro = EskfEstimator(p=a[0:3], q=a[3:7], v=a[7:10], ba=a[10:13], bg=a[13:16], g=a[16:19], cov=a[19:].reshape(NS, NS))
        summ = b["summ"]
        blk = b["blk"]
        return OptimizeSummary(success=bool(summ.success) and rc == capi.SRL_OK, num_residuals_used=summ.num_residuals_used,
                               passes_run=summ.passes_run, converged=bool(summ.converged), trace=capi.summary_trace(summ)), \
            blk[0:4].copy(), blk[4:7].copy()

    # ---- src/optimize.cpp:133-314
    def updateIEKF(self, cur_icp_options: IcpParams, t_last, frame_q=None, frame_t=None):
        b = self._call_buffers()
        self._marshal(b, t_last, frame_q, frame_t)
        rc = lib().srl_update_iekf(self.ctx.h, self.voxel_map.h, self.sweep.h, b["st_ref"], b["p_fq"], b["p_ft"], b["p_tl"],
                                   b["p_R"], b["p_ti"], C.byref(cur_icp_options), b["summ_ref"])
        return self._unmarshal(b, rc)

    # ---- src/optimize.cpp:428-448 with the keypoints already selected (gridSampling is a "next" row)
    def optimize(self, raw_xyz, cur_icp_options: IcpParams, t_last, frame_q=None, frame_t=None, want_world: bool = True,
                 world_out=None):
        """world_out: optional (n,3) float64 C-contiguous array to receive the re-transformed frame (pass a pinned
        buffer to avoid staging); raw_xyz may likewise live in pinned memory."""
        raw = f64(raw_xyz).reshape(-1, 3)
        n = raw.shape[0]
        b = self._call_buffers()
        self._marshal(b, t_last, frame_q, frame_t)
        world = (world_out if world_out is not None else np.empty((n, 3))) if want_world else None
        rc = lib().srl_optimize_host(self.ctx.h, self.voxel_map.h, self.sweep.h, ptr(raw), n, b["st_ref"], b["p_fq"], b["p_ft"],
                                     b["p_tl"], b["p_R"], b["p_ti"], C.byref(cur_icp_options), b["summ_ref"],
                                     ptr(world) if want_world else None)
        self.sweep.n = n
        summ, fq, ft = self._unmarshal(b, rc)
        return summ, fq, ft, world


COUNT, EPS = 1, 2   # cv::TermCriteria::COUNT, ::EPS


def tracker_lk_params() -> dict:
    """The LKOpticalFlowKernel opticalFlowTracker's constructor makes (src/opticalFlowTracker.cpp:5-8): a 21 x 21 window, 3 levels,
    COUNT | EPS with 10 iterations and epsilon 0.05, flags cv_OPTFLOW_LK_GET_MIN_EIGENVALS (8), the default min_eig_threshold."""
    return dict(win_size=(21, 21), max_level=3, criteria=(COUNT | EPS, 10, 0.05), flags=8, min_eig_threshold=1e-4)


class LKOpticalFlowKernel(_Handle):
    """LKOpticalFlowKernel (include/lkpyramid.h:65-131, srl_lk_*): the optical-flow tracker's pyramidal Lucas-Kanade on the GPU, bit
    for bit the reference.  criteria = (type, max_count, epsilon) as cv::TermCriteria; the defaults are the reference's own
    constructor defaults.  Each image's pyramid stays on the device as the previous image of the next call."""

    _destroy = "srl_lk_destroy"

    def __init__(self, ctx: Context, win_size=(21, 21), max_level: int = 3, criteria=(COUNT | EPS, 30, 0.01), flags: int = 0,
                 min_eig_threshold: float = 1e-4):
        self.ctx = ctx
        t, c, e = criteria
        self.params = capi.LkParams(int(win_size[0]), int(win_size[1]), int(max_level), int(t), int(c), float(e), int(flags),
                                    float(min_eig_threshold))
        h = C.c_void_p()
        _check(ctx.h, lib().srl_lk_create(ctx.h, C.byref(self.params), C.byref(h)))
        self.h = h

    def trackImage(self, gray, last_pts, out=None):
        """trackImage (src/lkpyramid.cpp:755-795): (curr_pts (n, 2) float32, status (n,) uint8, n_tracked).  gray: (rows, cols) uint8
        with unit column stride (a numpy array or a torch tensor, host or CUDA; rows may be padded); last_pts: (n, 2) float32 (the
        selection's uv as it comes).  out = (curr_pts, status) buffers receive the result; without it they are made on last_pts'
        side (numpy, or a torch tensor on its device), status filled with ones.  The first image only builds its pyramid:
        curr_pts = last_pts, status as it was, n_tracked 0."""
        _, p_img, rows, cols, pitch = _buffer(gray, np.uint8, image=True)
        _, p_last, n = _buffer(last_pts, np.float32, 2)
        if out is None:
            curr = _empty_like_input(last_pts, n, 2, np.float32)
            status = _empty_like_input(last_pts, n, 1, np.uint8).reshape(-1)
            status[:] = 1
        else:
            curr, status = out
        _, p_curr, n_curr = _buffer(curr, np.float32, 2)
        _, p_st, n_st = _buffer(status, np.uint8)
        if n_curr < n or n_st < n:
            raise ValueError("out buffers hold fewer points than last_pts")
        k = C.c_int64(0)
        _check(self.ctx.h, lib().srl_lk_track_image(self.h, C.c_void_p(p_img), int(cols), int(rows), int(pitch), C.c_void_p(p_last), n,
                                                    C.c_void_p(p_curr), C.c_void_p(p_st), C.byref(k)))
        return curr[:n], status[:n], k.value

    def getMaxLevel(self) -> int:
        v = C.c_int32(0)
        _check(self.ctx.h, lib().srl_lk_info(self.h, C.byref(v), None, None))
        return v.value

    def level(self, which: int, level: int):
        """Test hook: (padded image, padded (Ix, Iy) int16 buffer) of a pyramid level; which 0 is the last image's, 1 the one before."""
        ml, cols, rows = C.c_int32(0), C.c_int32(0), C.c_int32(0)
        _check(self.ctx.h, lib().srl_lk_info(self.h, C.byref(ml), C.byref(cols), C.byref(rows)))
        w, h = cols.value, rows.value
        for _ in range(level):
            w, h = (w + 1) // 2, (h + 1) // 2
        shape = (h + 2 * self.params.win_h, w + 2 * self.params.win_w)
        img, der = np.zeros(shape, np.uint8), np.zeros(shape + (2,), np.int16)
        _check(self.ctx.h, lib().srl_lk_download_level(self.h, int(which), int(level), ptr(img), ptr(der)))
        return img, der

    def lastTimes(self) -> tuple[float, float]:
        """(ms of image upload + pyramid + derivatives, ms of the point tracking) of the last trackImage, CUDA events."""
        a, b = C.c_double(0), C.c_double(0)
        _check(self.ctx.h, lib().srl_lk_last_times(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value


def r3live_camera_params() -> dict:
    """camera_parameter of config/r3live.yaml (and r3live_compressed.yaml): a 1280 x 1024 camera."""
    return dict(image_width=1280, image_height=1024, camera_intrinsic=[863.4241, 0.0, 640.6808, 0.0, 863.4171, 518.3392, 0.0, 0.0, 1.0],
                camera_dist_coeffs=[-0.1080, 0.1050, -1.2872e-04, 5.7923e-05, -0.0222])


def ntu_camera_params() -> dict:
    """camera_parameter of config/ntu.yaml: a 752 x 480 camera."""
    return dict(image_width=752, image_height=480, camera_intrinsic=[425.0259, 0.0, 386.0152, 0.0, 426.7976, 241.9130, 0.0, 0.0, 1.0],
                camera_dist_coeffs=[-0.2881, 0.0746, 7.7845e-04, -2.2779e-04, 0.0])


class ImageProcessing(_Handle):
    """The image preparation of imageProcessing::process (src/imageProcessing.cpp:91-125,166-200, srl_image_*) on the GPU, bit for
    bit OpenCV's: undistortion (initUndistortRectifyMap CV_16SC2 + remap INTER_LINEAR), COLOR_RGB2GRAY and CLAHE clip 3 for
    gray_image, BGR2YCrCb, CLAHE clip 1 on Y and YCrCb2BGR for rgb_image.  Construction is the first-image step for inputs of
    cols x rows (the yaml's size unless given): the scale factor, the scaled intrinsics (camera_intrinsic()) and the map.
    ImageProcessing(ctx, **r3live_camera_params())."""

    _destroy = "srl_image_destroy"

    def __init__(self, ctx: Context, image_width: int, image_height: int, camera_intrinsic, camera_dist_coeffs, cols: int | None = None,
                 rows: int | None = None):
        self.ctx = ctx
        k = np.asarray(camera_intrinsic, np.float64).reshape(-1)
        d = np.asarray(camera_dist_coeffs, np.float64).reshape(-1)
        if k.size != 9 or d.size != 5:
            raise ValueError("camera_intrinsic has 9 values and camera_dist_coeffs 5")
        self.params = capi.ImageParams(int(image_width), int(image_height), (C.c_double * 9)(*k), (C.c_double * 5)(*d))
        self.input_size = (int(image_width if cols is None else cols), int(image_height if rows is None else rows))
        h = C.c_void_p()
        _check(ctx.h, lib().srl_image_create(ctx.h, C.byref(self.params), self.input_size[0], self.input_size[1], C.byref(h)))
        self.h = h

    def _info(self):
        c, r, t, s, k = C.c_int32(0), C.c_int32(0), C.c_int32(0), C.c_double(0), np.zeros(9, np.float64)
        _check(self.ctx.h, lib().srl_image_info(self.h, C.byref(c), C.byref(r), C.byref(t), C.byref(s), ptr(k)))
        return c.value, r.value, t.value, s.value, k

    def output_size(self) -> tuple[int, int]:
        """(out_cols, out_rows) of rgb_image and gray_image."""
        return self._info()[:2]

    def tiles(self) -> int:
        """CLAHE's grid: tiles x tiles."""
        return self._info()[2]

    def scale_factor(self) -> float:
        """image_scale_factor = image_width / input cols."""
        return self._info()[3]

    def camera_intrinsic(self) -> np.ndarray:
        """(3, 3) K with fx, cx, fy, cy divided by the scale factor: what srl_camera and the vision updates use."""
        return self._info()[4].reshape(3, 3)

    def process(self, image_bgr, out=None):
        """process:120-125 for one (rows, cols, 3) BGR8 image (numpy or torch, host or CUDA; rows may be padded, as a ROS step is):
        (rgb_image (out_rows, out_cols, 3) BGR8, gray_image (out_rows, out_cols)).  out = (rgb, gray) buffers (contiguous, numpy or
        torch, host or CUDA) receive them; without it numpy arrays are returned."""
        _, p_img, rows, cols, pitch = _buffer(image_bgr, np.uint8, 3, image=True)
        oc, orows = self.output_size()
        if out is None:
            rgb, gray = np.empty((orows, oc, 3), np.uint8), np.empty((orows, oc), np.uint8)
        else:
            rgb, gray = out
        _, p_rgb, n_rgb = _buffer(rgb, np.uint8, 3)
        _, p_gray, n_gray = _buffer(gray, np.uint8)
        if n_rgb < oc * orows or n_gray < oc * orows:
            raise ValueError(f"out buffers must hold {orows} x {oc} pixels")
        _check(self.ctx.h, lib().srl_image_process(self.h, C.c_void_p(p_img), int(cols), int(rows), int(pitch), C.c_void_p(p_rgb),
                                                   C.c_void_p(p_gray)))
        return rgb, gray

    def maps(self):
        """Test hook: (map1 (out_rows, out_cols, 2) int16, map2 (out_rows, out_cols) uint16), OpenCV's CV_16SC2 + CV_16UC1 pair."""
        oc, orows = self.output_size()
        m1, m2 = np.zeros((orows, oc, 2), np.int16), np.zeros((orows, oc), np.uint16)
        _check(self.ctx.h, lib().srl_image_download_maps(self.h, ptr(m1), ptr(m2)))
        return m1, m2

    def last_times(self) -> tuple[float, float, float]:
        """(upload ms, remap + colour planes ms, both CLAHEs ms) of the last process, CUDA events."""
        a, b, c = C.c_double(0), C.c_double(0), C.c_double(0)
        _check(self.ctx.h, lib().srl_image_last_times(self.h, C.byref(a), C.byref(b), C.byref(c)))
        return a.value, b.value, c.value

    def covariance(self) -> np.ndarray:
        """imageProcessing::covariance (11, 11): setInitialCov at construction, then what the camera updates leave."""
        c = np.zeros((11, 11), np.float64)
        _check(self.ctx.h, lib().srl_image_covariance(self.h, None, ptr(c)))
        return c

    def setCovariance(self, cov) -> None:
        c = np.ascontiguousarray(np.asarray(cov, np.float64).reshape(11, 11))
        _check(self.ctx.h, lib().srl_image_covariance(self.h, ptr(c), None))

    def vioEsikf(self, cmap: "ColorVoxelMap", state: "CameraState", ids, uv, velocity, n_new_visited: int) -> bool:
        """imageProcessing::vioEsikf (src/imageProcessing.cpp:220-380, srl_image_vio_esikf) over the tracked set in the caller's
        order: ids (n,) uint32 colour-map point ids, uv (n, 2) float32 matched points (LKOpticalFlowKernel.trackImage's output
        as it is), velocity (n, 2) float64 image velocities; numpy arrays or torch tensors, host or CUDA.  n_new_visited is the
        colour map's stats()["recent"] after the rendering insert.  Updates `state` and the covariance in place; returns the reference's
        result."""
        _, p_ids, n = _buffer(ids, np.uint32)
        _, p_uv, n_uv = _buffer(uv, np.float32, 2)
        _, p_vel, n_vel = _buffer(velocity, np.float64, 2)
        if n_uv != n or n_vel != n:
            raise ValueError("ids, uv and velocity must hold the same number of points")
        r = C.c_int32(0)
        _check(self.ctx.h, lib().srl_image_vio_esikf(self.h, cmap.h, C.byref(state.c), C.c_void_p(p_ids), C.c_void_p(p_uv),
                                                     C.c_void_p(p_vel), n, int(n_new_visited), C.byref(r)))
        return bool(r.value)

    def vioPhotometric(self, cmap: "ColorVoxelMap", state: "CameraState", ids, velocity, n_new_visited: int, rgb_image) -> bool:
        """imageProcessing::vioPhotometric (:402-552, srl_image_vio_photometric) on the prepared rgb_image ((out_rows, out_cols,
        3) BGR8, process()'s rgb output; numpy or torch, host or CUDA, rows may be padded); ids and velocity as for vioEsikf."""
        _, p_ids, n = _buffer(ids, np.uint32)
        _, p_vel, n_vel = _buffer(velocity, np.float64, 2)
        if n_vel != n:
            raise ValueError("ids and velocity must hold the same number of points")
        _, p_img, rows, cols, pitch = _buffer(rgb_image, np.uint8, 3, image=True)
        r = C.c_int32(0)
        _check(self.ctx.h, lib().srl_image_vio_photometric(self.h, cmap.h, C.byref(state.c), C.c_void_p(p_ids), C.c_void_p(p_vel), n,
                                                           int(n_new_visited), C.c_void_p(p_img), int(cols), int(rows), int(pitch),
                                                           C.byref(r)))
        return bool(r.value)

    def vio_last_summary(self, which: int) -> tuple[int, int, float]:
        """(iterations run, points used, acc_residual) of the last vioEsikf (0) or vioPhotometric (1)."""
        it, used, acc = C.c_int32(0), C.c_int32(0), C.c_double(0)
        _check(self.ctx.h, lib().srl_image_vio_last_summary(self.h, int(which), C.byref(it), C.byref(used), C.byref(acc)))
        return it.value, used.value, acc.value

    def vio_last_times(self) -> tuple[float, float]:
        """(vioEsikf ms, vioPhotometric ms): device time of each update's last launch, CUDA events."""
        a, b = C.c_double(0), C.c_double(0)
        _check(self.ctx.h, lib().srl_image_vio_last_times(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value


_NO_INLIERS = np.zeros(1, np.int32)


class OpticalFlowTracker(_Handle):
    """opticalFlowTracker (src/opticalFlowTracker.cpp, srl_flow_tracker_*): the tracked point sets of the camera frame kept on the
    device from one image to the next, in colour-map point id order.  lk is the LKOpticalFlowKernel it tracks with
    (LKOpticalFlowKernel(ctx, **tracker_lk_params()) as the reference's constructor makes it); cmap holds the points.

    Per image, as imageProcessing::process calls it: trackImage(gray, t) -> (caller's findFundamentalMat on matches(),
    rejectMatches(mask)) -> (caller's solvePnPRansac on current(), removeOutlierUsingRansacPnp(inliers)) -> the camera updates on
    current(device=True) -> render -> refresh selection -> updateAndAppendTrackPoints(camera, selected ids, 40 / scale).
    Point lists are numpy arrays or torch tensors, host or CUDA; the set accessors return numpy copies, or with device=True
    torch views of the tracker's own memory, valid until its next call."""

    _destroy = "srl_flow_tracker_destroy"

    def __init__(self, ctx: Context, cmap: "ColorVoxelMap", lk: "LKOpticalFlowKernel", maximum_tracked_points: int = 300):
        self.ctx, self.cmap, self.lk = ctx, cmap, lk
        h = C.c_void_p()
        _check(ctx.h, lib().srl_flow_tracker_create(ctx.h, cmap.h, lk.h, int(maximum_tracked_points), C.byref(h)))
        self.h = h

    def init(self, gray, image_time: float, ids, uv) -> None:
        """init / setTrackPoints (:188-211): last = {ids[i]: uv[i]}, both image times = image_time, and the Lucas-Kanade call
        on gray (its first image: the pyramid only).  ids: uint32 point ids (int32 tensors hold their bits); uv: (n, 2) float32."""
        _, p_img, rows, cols, pitch = _buffer(gray, np.uint8, image=True)
        _, p_ids, n = _buffer(ids, np.uint32)
        _, p_uv, n_uv = _buffer(uv, np.float32, 2)
        if n_uv != n:
            raise ValueError("ids and uv must hold the same number of points")
        _check(self.ctx.h, lib().srl_flow_tracker_init(self.h, C.c_void_p(p_img), int(cols), int(rows), int(pitch), float(image_time),
                                                       C.c_void_p(p_ids), C.c_void_p(p_uv), n))

    def trackImage(self, gray, image_time: float) -> bool:
        """trackImage(p_frame, -20) (:111-186) on gray_image at time_sweep_end; returns whether Lucas-Kanade ran (not below 30
        tracked points)."""
        _, p_img, rows, cols, pitch = _buffer(gray, np.uint8, image=True)
        called = C.c_int32(0)
        _check(self.ctx.h, lib().srl_flow_tracker_track_image(self.h, C.c_void_p(p_img), int(cols), int(rows), int(pitch), float(image_time),
                                                              C.byref(called)))
        return bool(called.value)

    def rejectMatches(self, mask=None) -> None:
        """findFundamentalMat's status over matches() (one uint8 per match, non-zero = inlier); None = all inliers."""
        if mask is None:
            _check(self.ctx.h, lib().srl_flow_tracker_reject_matches(self.h, None, 0))
            return
        mask, p, n = _buffer(mask, np.uint8, convert=True)
        _check(self.ctx.h, lib().srl_flow_tracker_reject_matches(self.h, C.c_void_p(p), n))

    def removeOutlierUsingRansacPnp(self, inliers=None) -> bool:
        """removeOutlierUsingRansacPnp(p_frame, 1) (:267-323) with solvePnPRansac's inlier indices into current() (int32, any
        order, repeats allowed); None = all.  False (nothing changed) below 10 current points."""
        r = C.c_int32(0)
        if inliers is None:
            _check(self.ctx.h, lib().srl_flow_tracker_remove_outliers(self.h, None, 0, C.byref(r)))
            return bool(r.value)
        inliers, p, n = _buffer(inliers, np.int32, convert=True)
        p = C.c_void_p(p) if n else ptr(_NO_INLIERS)   # an empty list is zero inliers, which a NULL pointer would not say
        _check(self.ctx.h, lib().srl_flow_tracker_remove_outliers(self.h, p, n, C.byref(r)))
        return bool(r.value)

    def updateAndAppendTrackPoints(self, camera: "capi.Camera", candidates, mini_distance: float) -> None:
        """updateAndAppendTrackPoints(p_frame, map_tracker, mini_distance) (:13-102): camera is the frame's after the updates
        (fov_margin 0.005), candidates the refresh selection's point ids in its order (points_rgb_vec_for_projection)."""
        _, p, n = _buffer(candidates, np.uint32)
        _check(self.ctx.h, lib().srl_flow_tracker_update_and_append(self.h, C.byref(camera), float(mini_distance), C.c_void_p(p), n))

    def _sets(self) -> "capi.FlowTrackerSets":
        s = capi.FlowTrackerSets()
        _check(self.ctx.h, lib().srl_flow_tracker_sets(self.h, C.byref(s)))
        return s

    def counts(self) -> dict:
        s = self._sets()
        return dict(match=s.n_match, cur=s.n_cur, last=s.n_last)

    def _arrays(self, device, spec):
        out = []
        for p, n, w, dt in spec:
            t = _device_view(self.ctx, p, n, w, dt)
            out.append(t if device else (t.cpu().numpy().view(np.uint32) if dt == np.int32 else t.cpu().numpy()))
        return tuple(out)

    def matches(self, device: bool = False):
        """(ids, last uv (n, 2) float32, new uv (n, 2) float32): what trackImage's Lucas-Kanade tracked, in last order — the two
        point lists findFundamentalMat is given.  ids are uint32 (numpy) or int32 holding their bits (device)."""
        s = self._sets()
        return self._arrays(device, [(s.match_ids, s.n_match, 1, np.int32), (s.match_last_uv, s.n_match, 2, np.float32),
                                     (s.match_uv, s.n_match, 2, np.float32)])

    def current(self, device: bool = False):
        """(ids, uv (n, 2) float32, velocity (n, 2) float64): map_rgb_points_in_cur_image_pose and the points' image_velocity, what
        vioEsikf / vioPhotometric take."""
        s = self._sets()
        return self._arrays(device, [(s.cur_ids, s.n_cur, 1, np.int32), (s.cur_uv, s.n_cur, 2, np.float32), (s.cur_velocity, s.n_cur, 2, np.float64)])

    def last(self, device: bool = False):
        """(ids, uv (n, 2) float32): map_rgb_points_in_last_image_pose."""
        s = self._sets()
        return self._arrays(device, [(s.last_ids, s.n_last, 1, np.int32), (s.last_uv, s.n_last, 2, np.float32)])

    def lastImageTime(self) -> float:
        return self._sets().last_image_time

    def outlierCounts(self, ids) -> np.ndarray:
        """Test hook: rgbPoint::is_out_lier_count of each point id, int16."""
        ids = np.ascontiguousarray(ids, np.uint32).reshape(-1)
        out = np.zeros(ids.size, np.int16)
        _check(self.ctx.h, lib().srl_flow_tracker_outlier_counts(self.h, ptr(ids), ids.size, ptr(out)))
        return out


def _quat_to_rot(q):
    """Eigen's Quaterniond::toRotationMatrix, q = (x, y, z, w)."""
    x, y, z, w = (float(v) for v in q)
    tx, ty, tz = 2.0 * x, 2.0 * y, 2.0 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return np.array([[1.0 - (tyy + tzz), txy - twz, txz + twy], [txy + twz, 1.0 - (txx + tzz), tyz - twx],
                     [txz - twy, tyz + twx, 1.0 - (txx + tyy)]])


def _rot_to_quat(m):
    """Eigen's Quaterniond(Matrix3d), as (x, y, z, w)."""
    q = [0.0] * 4
    t = m[0, 0] + m[1, 1] + m[2, 2]
    if t > 0:
        t = np.sqrt(t + 1.0); q[3] = 0.5 * t; t = 0.5 / t
        q[0] = (m[2, 1] - m[1, 2]) * t; q[1] = (m[0, 2] - m[2, 0]) * t; q[2] = (m[1, 0] - m[0, 1]) * t
    else:
        i = 0
        if m[1, 1] > m[0, 0]:
            i = 1
        if m[2, 2] > m[i, i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        t = np.sqrt(m[i, i] - m[j, j] - m[k, k] + 1.0); q[i] = 0.5 * t; t = 0.5 / t
        q[3] = (m[k, j] - m[j, k]) * t; q[j] = (m[j, i] + m[i, j]) * t; q[k] = (m[k, i] + m[i, k]) * t
    return np.array(q)


def _mm3(a, b):
    """3 x 3 product with Eigen's fixed-size reduction order c0 + (c1 + c2)."""
    return np.array([[a[i, 0] * b[0, j] + (a[i, 1] * b[1, j] + a[i, 2] * b[2, j]) for j in range(3)] for i in range(3)])


def _mv3(a, v):
    return np.array([a[i, 0] * v[0] + (a[i, 1] * v[1] + a[i, 2] * v[2]) for i in range(3)])


class CameraState:
    """The p_state fields the camera updates read and write (srl_vio_state).  The constructor derives the camera poses as
    lioOptimization::stateEstimation does before process (src/lioOptimization.cpp:1073-1075): q_world_camera =
    Quaterniond(rotation.toRotationMatrix() * R_imu_camera), t_world_camera = rotation.toRotationMatrix() * t_imu_camera +
    translation, then refreshPoseForProjection.  Quaternions are (x, y, z, w); R_imu_camera is (3, 3)."""

    def __init__(self, rotation, translation, R_imu_camera, t_imu_camera, fx: float, fy: float, cx: float, cy: float,
                 time_td: float = 0.0):
        rq = np.asarray(rotation, np.float64).reshape(4)
        tr = np.asarray(translation, np.float64).reshape(3)
        ric = np.asarray(R_imu_camera, np.float64).reshape(3, 3)
        tic = np.asarray(t_imu_camera, np.float64).reshape(3)
        rw = _quat_to_rot(rq)
        q_wc = _rot_to_quat(_mm3(rw, ric))
        t_wc = _mv3(rw, tic) + tr
        n2 = (q_wc[0] * q_wc[0] + q_wc[2] * q_wc[2]) + (q_wc[1] * q_wc[1] + q_wc[3] * q_wc[3])
        q_cw = np.array([-q_wc[0] / n2, -q_wc[1] / n2, -q_wc[2] / n2, q_wc[3] / n2])   # Quaterniond::inverse
        t_cw = _mv3(-_quat_to_rot(q_cw), t_wc)
        c = capi.VioState()
        c.rotation[:] = rq.tolist(); c.translation[:] = tr.tolist(); c.R_imu_camera[:] = ric.reshape(-1).tolist()
        c.t_imu_camera[:] = tic.tolist()
        c.fx, c.fy, c.cx, c.cy, c.time_td = float(fx), float(fy), float(cx), float(cy), float(time_td)
        c.q_world_camera[:] = q_wc.tolist(); c.t_world_camera[:] = t_wc.tolist()
        c.q_camera_world[:] = q_cw.tolist(); c.t_camera_world[:] = t_cw.tolist()
        self.c = c

    def __getattr__(self, name):
        c = self.__dict__.get("c")
        if c is None or name not in dict(capi.VioState._fields_):
            raise AttributeError(name)
        v = getattr(c, name)
        if isinstance(v, float):
            return v
        a = np.array(v[:], np.float64)
        return a.reshape(3, 3) if name == "R_imu_camera" else a

    def camera(self, cols: int, rows: int, fov_margin: float) -> "capi.Camera":
        """The srl_camera of this state for the renderer (renderPointsInRecentVoxel) and the selection (selectPointsForProjection)."""
        c = self.c
        return capi.Camera((C.c_double * 4)(*c.q_camera_world), (C.c_double * 3)(*c.t_camera_world), (C.c_double * 3)(*c.t_world_camera),
                           c.fx, c.fy, c.cx, c.cy, float(fov_margin), int(cols), int(rows))


def r3live_lidar_params(**kw) -> dict:
    """config/r3live.yaml: Livox, 6 lines, 10 Hz, ns, blind 0.1 m, point_filter_num 4"""
    return dict(dict(lidar_type=1, n_scans=6, scan_rate=10, time_unit=3, blind=0.1, point_filter_num=4), **kw)


def ntu_lidar_params(**kw) -> dict:
    """config/ntu.yaml: Ouster, 16 rings, 20 Hz, ns, blind 4 m, point_filter_num 4"""
    return dict(dict(lidar_type=3, n_scans=16, scan_rate=20, time_unit=3, blind=4.0, point_filter_num=4), **kw)


class CloudProcessing(_Handle):
    """cloudProcessing (src/cloudProcessing.cpp, srl_lidar_*) with its point_buffer kept on the device.  Messages are byte buffers
    as they come off the wire: numpy arrays (a structured array is taken as its bytes) or torch uint8 tensors, host or CUDA.

    livoxHandler(records, stamp): CustomMsg points, `stride` bytes apart (19 for the packed ROS layout).
    process(data, layout, stamp): PointCloud2 data; layout = dict(point_step, x, y, z, time, ring) byte offsets (msg->fields),
    and for rows padded past width * point_step also width and row_step (msg->width, msg->row_step).
    cut(t): getMeasurements' pops (front().timestamp < t) as (count, raw_xyz, timestamp) torch views of the queue's memory
    (device=True, valid until the next handler call) or numpy copies; the views go to srl_build_frame as they are:
        n, xyz, ts = cp.cut(t, device=True)
        frame = lio_opt.buildFrame(xyz, ts, states, ..., point_time_enable=cp.isPointTimeEnable())"""

    _destroy = "srl_lidar_destroy"

    def __init__(self, ctx: Context, lidar_type: int, n_scans: int, scan_rate: int, time_unit: int, blind: float,
                 point_filter_num: int, capacity: int = 1 << 18):
        self.ctx = ctx
        self.params = capi.LidarParams(int(lidar_type), int(n_scans), int(scan_rate), int(time_unit), float(blind),
                                       int(point_filter_num), 0)
        h = C.c_void_p()
        _check(ctx.h, lib().srl_lidar_create(ctx.h, C.byref(self.params), int(capacity), C.byref(h)))
        self.h = h

    def livoxHandler(self, records, stamp: float, stride: int = 19) -> int:
        records, p, nbytes = _buffer(records, None, convert=True)
        n = C.c_int64(0)
        _check(self.ctx.h, lib().srl_lidar_livox(self.h, C.c_void_p(p), nbytes // stride, stride, float(stamp), C.byref(n)))
        return n.value

    def process(self, data, layout: dict, stamp: float) -> int:
        data, p, nbytes = _buffer(data, None, convert=True)
        y = capi.Cloud2Layout(int(layout["point_step"]), int(layout["x"]), int(layout["y"]), int(layout["z"]), int(layout["time"]),
                              int(layout.get("ring", -1)), int(layout.get("width", 0)), int(layout.get("row_step", 0)))
        n_pts = (nbytes // y.row_step) * y.width if y.row_step else nbytes // y.point_step
        n = C.c_int64(0)
        _check(self.ctx.h, lib().srl_lidar_process(self.h, C.c_void_p(p), n_pts, C.byref(y), float(stamp), C.byref(n)))
        return n.value

    def cut(self, t: float, device: bool = False):
        n, xyz, ts = C.c_int64(0), C.c_void_p(), C.c_void_p()
        _check(self.ctx.h, lib().srl_lidar_cut(self.h, float(t), C.byref(n), C.byref(xyz), C.byref(ts)))
        k = n.value
        xyz_t, ts_t = _device_view(self.ctx, xyz.value, k, 3, np.float64), _device_view(self.ctx, ts.value, k, 1, np.float64)
        if device:
            return k, xyz_t, ts_t
        return k, xyz_t.cpu().numpy(), ts_t.cpu().numpy()

    def info(self) -> "capi.LidarInfo":
        i = capi.LidarInfo()
        _check(self.ctx.h, lib().srl_lidar_info_get(self.h, C.byref(i)))
        return i

    def isPointTimeEnable(self) -> bool:
        return bool(self.info().given_offset_time)

    def getSweepInterval(self) -> float:
        return self.info().sweep_interval

    def queue(self):
        """the whole point_buffer, front first: (raw_xyz n x 3, relative_time, timestamp) numpy copies"""
        n = self.info().size
        xyz, rel, ts = np.empty((n, 3)), np.empty(n), np.empty(n)
        _check(self.ctx.h, lib().srl_lidar_download(self.h, ptr(xyz), ptr(rel), ptr(ts)))
        return xyz, rel, ts


def device_sort_permutation(ctx: Context, keys, return_heapsorts: bool = False):
    """The device std::sort's permutation of float64 keys (host or CUDA): perm[p] = the index of the key that ends at p."""
    keys, p, n = _buffer(keys, np.float64, convert=True)
    perm = np.empty(n, np.int32)
    h = C.c_int32(0)
    _check(ctx.h, lib().srl_lidar_sort_replay(ctx.h, C.c_void_p(p), n, ptr(perm), C.byref(h)))
    return (perm, h.value) if return_heapsorts else perm


__all__ = ["Context", "VoxelHashMap", "ColorVoxelMap", "Sweep", "EskfEstimator", "LioOptimization", "OptimizeSummary", "PlaneResiduals",
           "IcpParams", "r3live_params", "r3live_map_options", "r3live_compressed_map_options", "make_frame", "SrlError", "write_pcd_xyzrgb",
           "LKOpticalFlowKernel", "tracker_lk_params", "OpticalFlowTracker", "ImageProcessing", "CameraState", "r3live_camera_params", "ntu_camera_params",
           "CloudProcessing", "r3live_lidar_params", "ntu_lidar_params", "device_sort_permutation"]
