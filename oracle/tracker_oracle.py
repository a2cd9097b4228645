"""ctypes binding of the oracle of the map tracker's projection selection (oracle/_build/libsrl_tracker_oracle.so:
oracle/srl_tracker_oracle.cpp, which is srl_oracle.cpp as it is plus orc_color_select and orc_color_gather; built by
oracle/tracker.mk).

TEST INFRASTRUCTURE ONLY.  The library carries its own copy of the whole oracle, so the colour maps used with the two new entry
points are created, fed and rendered through that same library (the handles of oracle_py's library are not interchangeable).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(_HERE, "_build", "libsrl_tracker_oracle.so")
_lib = None


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(PATH):
        r = subprocess.run(["make", "-C", _HERE, "-f", "tracker.mk", "_build/libsrl_tracker_oracle.so"], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("oracle/_build/libsrl_tracker_oracle.so could not be built:\n" + r.stdout + r.stderr)
    L = C.CDLL(PATH)
    P, I64, I32, D = C.c_void_p, C.c_int64, C.c_int32, C.c_double
    L.orc_color_create.restype = P
    L.orc_color_destroy.argtypes = [P]
    L.orc_color_add_points.argtypes = [P, P, I64, D, I32, D, I32, D, D, I32]
    L.orc_color_add_points.restype = I64
    L.orc_color_render.argtypes = [P, P, P, I32, I32, D]
    L.orc_color_render.restype = I64
    for f in ("orc_color_num_voxels", "orc_color_num_rgb_points", "orc_color_num_recent"):
        getattr(L, f).argtypes = [P]
        getattr(L, f).restype = I64
    L.orc_color_lists.argtypes = [P, P, P]
    L.orc_color_select.argtypes = [P, P, I32, I32, D, I32, I32, D, D, P, P, I64]
    L.orc_color_select.restype = I64
    L.orc_color_gather.argtypes = [P, P, I64, P, P, P, P]
    L.orc_color_gather.restype = I32
    _lib = L
    return L


class OracleColorMap:
    """The colour map of oracle_py.OracleColorMap (same restatement) + selectPointsForProjection and the per-point reads."""

    def __init__(self, voxel_size=1.0, max_num_points_in_voxel=20, min_distance_points=0.15):
        self._h = C.c_void_p(lib().orc_color_create())
        self.voxel_size, self.cap, self.min_dist = voxel_size, max_num_points_in_voxel, min_distance_points

    def __del__(self):
        try:
            if self._h:
                lib().orc_color_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def add_points(self, xyz, add_point_step=1, time_sweep_end=1.0, time_last_process=0.0, to_rendering=True) -> int:
        xyz = np.ascontiguousarray(xyz, np.float64).reshape(-1, 3)
        return int(lib().orc_color_add_points(self._h, _ptr(xyz), xyz.shape[0], self.voxel_size, self.cap, self.min_dist, add_point_step,
                                              time_sweep_end, time_last_process, 1 if to_rendering else 0))

    def render(self, cam15, image_bgr, obs_time) -> int:
        cam = np.ascontiguousarray(cam15, np.float64).reshape(15)
        img = np.ascontiguousarray(image_bgr, np.uint8)
        return int(lib().orc_color_render(self._h, _ptr(cam), _ptr(img), img.shape[0], img.shape[1], float(obs_time)))

    def num_rgb_points(self) -> int:
        return int(lib().orc_color_num_rgb_points(self._h))

    def num_recent(self) -> int:
        return int(lib().orc_color_num_recent(self._h))

    def lists(self):
        """(rgb_points_vec as (n, 4) int16 voxel key + index in block, voxels_recent_visited as (m, 3) int32 keys)"""
        rgb = np.zeros((self.num_rgb_points(), 4), np.int16)
        rec = np.zeros((self.num_recent(), 3), np.int32)
        lib().orc_color_lists(self._h, _ptr(rgb), _ptr(rec))
        return rgb, rec

    def select(self, cam15, rows=480, cols=640, minimum_dis=5.0, skip_step=1, use_all_points=False, minimum_depth=0.1, maximum_depth=200.0):
        """selectPointsForProjection: ((n, 4) int16 voxel key + index in block, (n, 2) float32 u_f, v_f) in point_index order."""
        cam = np.ascontiguousarray(cam15, np.float64).reshape(15)
        args = (self._h, _ptr(cam), int(rows), int(cols), float(minimum_dis), int(skip_step), 1 if use_all_points else 0, float(minimum_depth),
                float(maximum_depth))
        n = int(lib().orc_color_select(*args, None, None, 0))
        ki, uv = np.zeros((n, 4), np.int16), np.zeros((n, 2), np.float32)
        if n:
            assert lib().orc_color_select(*args, _ptr(ki), _ptr(uv), n) == n
        return ki, uv

    def gather(self, key_index):
        """the state of the points named by (n, 4) key_index as a dict like ColorVoxelMap.gatherPoints (None for an unknown entry)."""
        ki = np.ascontiguousarray(key_index, np.int16).reshape(-1, 4)
        n = ki.shape[0]
        out = dict(xyz=np.zeros((n, 3), np.float32), rgb=np.zeros((n, 3), np.int16), n_rgb=np.zeros(n, np.int16), cov=np.zeros((n, 3), np.float32))
        if lib().orc_color_gather(self._h, _ptr(ki), n, _ptr(out["xyz"]), _ptr(out["rgb"]), _ptr(out["n_rgb"]), _ptr(out["cov"])) != 0:
            return None
        out["key_index"] = ki.copy()
        return out
