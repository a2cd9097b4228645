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

Error behaviour: optimizeSummary.success=false <-> OptimizeSummary.success False (SRL_TOO_FEW_RESIDUALS);
the reference's `throw std::runtime_error("error")` on NaN planarity <-> RuntimeError; everything else raises
SrlError.  No CPU fallback exists: without the CUDA library/GPU every call fails loudly.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from . import capi
from .capi import (DebugOut, EskfState, Frame, IcpParams, IekfSummary, NormalEq, SrlError, f64, lib, ptr,
                   r3live_params)

NS = capi.NS


def _check(ctx, rc, ok=(capi.SRL_OK,)):
    if rc not in ok:
        raise SrlError(rc, lib().srl_last_error(ctx).decode() if ctx else "")
    return rc


def _is_tensor(a) -> bool:
    return type(a).__module__.split(".")[0] == "torch"


def _addr(a, dtype, width):
    """(address, rows) of a C-contiguous buffer of `width` elements of `dtype` per row: a numpy array (host) or a torch tensor
    (host or CUDA; the C ABI tells host from device per pointer)."""
    if _is_tensor(a):
        if str(a.dtype) != "torch." + np.dtype(dtype).name or not a.is_contiguous():
            raise TypeError(f"expected a contiguous torch.{np.dtype(dtype).name} tensor")
        return a.data_ptr(), a.numel() // width
    if not (isinstance(a, np.ndarray) and a.dtype == dtype and a.flags.c_contiguous):
        raise TypeError(f"expected a C-contiguous {np.dtype(dtype).name} array")
    return a.ctypes.data, a.size // width


def _empty_like_input(a, rows, width, dtype):
    if _is_tensor(a):
        import torch
        return torch.empty((rows, width), dtype=getattr(torch, np.dtype(dtype).name), device=a.device)
    return np.empty((rows, width), dtype)


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


class Context:
    """srl_ctx: one per host thread / GPU. `stream` may be a raw cudaStream_t (e.g. torch's current stream)."""

    def __init__(self, device: int = 0, stream: int | None = None):
        h = C.c_void_p()
        rc = lib().srl_ctx_create(device, C.c_void_p(stream) if stream else None, C.byref(h))
        if rc != capi.SRL_OK:
            raise SrlError(rc, "srl_ctx_create failed: no usable CUDA device (this path has no CPU fallback)")
        self.h = h
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            lib().srl_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

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


class VoxelHashMap:
    """HBM-resident voxelHashMap (include/cloudMap.h:171).

    max_voxels is the limit (SRL_MAP_FULL past it); initial_voxels (None = max_voxels) is what is committed at creation,
    and the map grows from there on demand, doubling, up to max_voxels."""

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

    def close(self):
        if getattr(self, "h", None):
            lib().srl_map_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

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
        if not _is_tensor(xyz_world):
            xyz_world = f64(xyz_world).reshape(-1, 3)
        p_in, n = _addr(xyz_world, np.float64, 3)
        out = _empty_like_input(xyz_world, n, 4, np.float32) if out is None else out
        p_out, max_out = _addr(out, np.float32, 4)
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


class ColorVoxelMap:
    """color_voxel_map + hashmap_3d_points + rgb_points_vec + voxels_recent_visited (include/lioOptimization.h:275-291,
    include/rgbMapTracker.h:38), fed by the colour branch of addPointsToMap and coloured by renderPointsInRecentVoxel.

    1 <= max_num_points_in_voxel <= 128.  Each point slot costs about 92-124 B of HBM (position, colour state, rgb id, fine
    cell slots), so the shipped map_options (0.1 m, 50 or 100 points) committed for 2^20 voxels take about 5-11 GB.
    max_voxels is the limit; initial_voxels (None = max_voxels) is what is committed at creation, and the map grows from
    there on demand, so a long run needs no guess of its size: initial_voxels=4096, max_voxels=1 << 20.
    The yaml values: ColorVoxelMap(ctx, o["size_voxel_map"], o["max_num_points_in_voxel"], max_voxels, o["min_distance_points"])
    with o = r3live_map_options(), and addPoints(..., add_point_step=o["add_point_step"])."""

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

    def close(self):
        if getattr(self, "h", None):
            lib().srl_color_map_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def stats(self) -> dict:
        v = [C.c_int64(0) for _ in range(5)]
        _check(self.ctx.h, lib().srl_color_map_stats(self.h, *[C.byref(x) for x in v]))
        return dict(zip(("voxels", "points", "rgb_points", "recent", "new_recent"), [x.value for x in v]))

    def addPoints(self, xyz_world, add_point_step: int = 1, time_sweep_end: float = 1.0, time_last_process: float = 0.0,
                  to_rendering: bool = True) -> int:
        """the loop of src/lioOptimization.cpp:533-551 over the registered frame (host array or a device pointer + n)."""
        xyz = f64(xyz_world).reshape(-1, 3)
        stored = C.c_int64(0)
        _check(self.ctx.h, lib().srl_color_map_add_points(self.h, ptr(xyz), xyz.shape[0], add_point_step, time_sweep_end, time_last_process,
                                                          1 if to_rendering else 0, C.byref(stored)))
        return stored.value

    def renderPointsInRecentVoxel(self, camera: "capi.Camera", image_bgr, obs_time: float) -> int:
        """rgbMapTracker::renderPointsInRecentVoxel (srl_color_map_render_recent) with a (rows, cols, 3) BGR8 host image; returns
        render_point_count.  camera.fov_margin must be >= 0 (SRL_BAD_ARG otherwise, NaN included, and the map is untouched):
        a negative margin would sample outside the image, which the reference leaves undefined.  The selection
        (selectPointsForProjection) still takes negative margins."""
        img = np.ascontiguousarray(image_bgr, np.uint8)
        assert img.shape == (camera.rows, camera.cols, 3)
        n = C.c_int64(0)
        _check(self.ctx.h, lib().srl_color_map_render_recent(self.h, C.byref(camera), ptr(img), float(obs_time), C.byref(n)))
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
        p_xyz, cap = _addr(xyz, np.float32, 3)
        p_rgb, cap_rgb = _addr(rgb, np.uint8, 3)
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
            if _is_tensor(a) and str(a.dtype) == "torch.int32" and dt == np.uint32:
                p, rows = a.data_ptr(), a.numel()          # torch has no uint32 of its own: int32 holds the ids' bits
            else:
                p, rows = _addr(a, dt, w)
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
        if _is_tensor(ids):
            p, n = ids.data_ptr(), ids.numel()
            if ids.element_size() != 4 or not ids.is_contiguous():
                raise TypeError("expected a contiguous 32-bit tensor of point ids")
        else:
            ids = np.ascontiguousarray(ids, np.uint32).reshape(-1)
            p, n = ids.ctypes.data, ids.size
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


class Sweep:
    """The keypoints of one reconstructed sweep, resident in HBM (raw LiDAR-frame points, FP64)."""

    def __init__(self, ctx: Context, capacity: int):
        self.ctx = ctx
        self.capacity = capacity
        self.n = 0
        h = C.c_void_p()
        _check(ctx.h, lib().srl_sweep_create(ctx.h, capacity, C.byref(h)))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            lib().srl_sweep_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def upload(self, raw_xyz):
        raw = f64(raw_xyz).reshape(-1, 3)
        _check(self.ctx.h, lib().srl_sweep_upload(self.h, ptr(raw), raw.shape[0]))
        self.n = raw.shape[0]

    def set_device(self, d_ptr: int, n: int):
        _check(self.ctx.h, lib().srl_sweep_set_device(self.h, C.c_void_p(d_ptr), n))
        self.n = n

    def set_shard(self, begin: int, end: int):
        _check(self.ctx.h, lib().srl_sweep_set_shard(self.h, begin, end))


class CloudFrame:
    """The frame buildFrame hands to stateEstimation, resident in HBM (srl_cloud_frame), final frame order."""

    FIELDS = (("raw_point", 3, np.float64), ("point", 3, np.float64), ("imu_point", 3, np.float64), ("relative_time", 1, np.float64),
              ("alpha_time", 1, np.float64), ("timestamp", 1, np.float64), ("source_index", 1, np.int32))

    def __init__(self, ctx: Context, capacity: int = 1 << 17):
        self.ctx = ctx
        self.info = None
        h = C.c_void_p()
        _check(ctx.h, lib().srl_cloud_frame_create(ctx.h, capacity, C.byref(h)))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            lib().srl_cloud_frame_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

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
        rc = lib().srl_eskf_observe(C.byref(s), ptr(d))
        if rc != capi.SRL_OK:
            raise SrlError(rc, "srl_eskf_observe")
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
        p_out, max_out = _addr(out, np.float32, 4)
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
        """buildFrame over a cut sweep given as host arrays (raw_xyz n*3, timestamp n; capi.lib().srl_build_frame takes device
        pointers too).  imu_states: a list of capi.ImuState.  motion_compensation: 0 IMU, 1 CONSTANT_VELOCITY.  Returns the
        device-resident frame (into `frame` when given), with the cloudFrame scalars in frame.info (capi.BuildFrameInfo)."""
        raw = f64(raw_xyz).reshape(-1, 3)
        ts = f64(timestamp).reshape(-1)
        assert ts.shape[0] == raw.shape[0]
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
        frame = frame if frame is not None else CloudFrame(self.ctx, max(raw.shape[0], 1))
        info = capi.BuildFrameInfo()
        _check(self.ctx.h, lib().srl_build_frame(self.ctx.h, ptr(raw), ptr(ts), raw.shape[0], states, len(imu_states), C.byref(p),
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


class LKOpticalFlowKernel:
    """LKOpticalFlowKernel (include/lkpyramid.h:65-131, srl_lk_*): the optical-flow tracker's pyramidal Lucas-Kanade on the GPU, bit
    for bit the reference.  criteria = (type, max_count, epsilon) as cv::TermCriteria; the defaults are the reference's own
    constructor defaults.  Each image's pyramid stays on the device as the previous image of the next call."""

    def __init__(self, ctx: Context, win_size=(21, 21), max_level: int = 3, criteria=(COUNT | EPS, 30, 0.01), flags: int = 0,
                 min_eig_threshold: float = 1e-4):
        self.ctx = ctx
        t, c, e = criteria
        self.params = capi.LkParams(int(win_size[0]), int(win_size[1]), int(max_level), int(t), int(c), float(e), int(flags),
                                    float(min_eig_threshold))
        h = C.c_void_p()
        _check(ctx.h, lib().srl_lk_create(ctx.h, C.byref(self.params), C.byref(h)))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            lib().srl_lk_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def trackImage(self, gray, last_pts, out=None):
        """trackImage (src/lkpyramid.cpp:755-795): (curr_pts (n, 2) float32, status (n,) uint8, n_tracked).  gray: (rows, cols) uint8
        with unit column stride (a numpy array or a torch tensor, host or CUDA; rows may be padded); last_pts: (n, 2) float32 (the
        selection's uv as it comes).  out = (curr_pts, status) buffers receive the result; without it they are made on last_pts'
        side (numpy, or a torch tensor on its device), status filled with ones.  The first image only builds its pyramid:
        curr_pts = last_pts, status as it was, n_tracked 0."""
        if _is_tensor(gray):
            if str(gray.dtype) != "torch.uint8" or gray.dim() != 2 or gray.stride(1) != 1:
                raise TypeError("expected a 2-D torch.uint8 image with unit column stride")
            p_img, rows, cols, pitch = gray.data_ptr(), gray.shape[0], gray.shape[1], gray.stride(0)
        else:
            if not (isinstance(gray, np.ndarray) and gray.dtype == np.uint8 and gray.ndim == 2 and gray.strides[1] == 1):
                raise TypeError("expected a 2-D uint8 array with unit column stride")
            p_img, rows, cols, pitch = gray.ctypes.data, gray.shape[0], gray.shape[1], gray.strides[0]
        p_last, n = _addr(last_pts, np.float32, 2)
        if out is None:
            curr = _empty_like_input(last_pts, n, 2, np.float32)
            status = _empty_like_input(last_pts, n, 1, np.uint8).reshape(-1)
            status[:] = 1
        else:
            curr, status = out
        p_curr, n_curr = _addr(curr, np.float32, 2)
        p_st, n_st = _addr(status, np.uint8, 1)
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


__all__ = ["Context", "VoxelHashMap", "ColorVoxelMap", "Sweep", "EskfEstimator", "LioOptimization", "OptimizeSummary", "PlaneResiduals",
           "IcpParams", "r3live_params", "r3live_map_options", "r3live_compressed_map_options", "make_frame", "SrlError", "write_pcd_xyzrgb",
           "LKOpticalFlowKernel", "tracker_lk_params"]
