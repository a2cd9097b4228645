"""ctypes binding of the oracle of the published maps (oracle/_build/libsrl_publish_oracle.so: oracle/srl_publish_oracle.cpp,
which is srl_oracle.cpp as it is plus orc_map_add_points_published and orc_color_export; built by oracle/publish.mk).

TEST INFRASTRUCTURE ONLY.  The library carries its own copy of the whole oracle, so the maps used with the two new entry points
are created, fed and rendered through that same library (the handles of oracle_py's library are not interchangeable).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(_HERE, "_build", "libsrl_publish_oracle.so")
_lib = None


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(PATH):
        r = subprocess.run(["make", "-C", _HERE, "-f", "publish.mk", "_build/libsrl_publish_oracle.so"], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("oracle/_build/libsrl_publish_oracle.so could not be built:\n" + r.stdout + r.stderr)
    L = C.CDLL(PATH)
    P, I64, I32, D = C.c_void_p, C.c_int64, C.c_int32, C.c_double
    L.orc_map_create.restype = P
    L.orc_map_destroy.argtypes = [P]
    L.orc_map_num_voxels.argtypes = [P]
    L.orc_map_num_voxels.restype = I64
    L.orc_map_snapshot.argtypes = [P, I32, P, P, P]
    L.orc_map_snapshot.restype = I64
    L.orc_map_load.argtypes = [P, P, P, P, I64, I32]
    L.orc_map_remove_far.argtypes = [P, P, D]
    L.orc_map_remove_far.restype = I64
    L.orc_map_add_points_published.argtypes = [P, P, I64, D, I32, D, I32, D, P, C.POINTER(I64)]
    L.orc_map_add_points_published.restype = I64
    L.orc_color_create.restype = P
    L.orc_color_destroy.argtypes = [P]
    L.orc_color_add_points.argtypes = [P, P, I64, D, I32, D, I32, D, D, I32]
    L.orc_color_add_points.restype = I64
    L.orc_color_render.argtypes = [P, P, P, I32, I32, D]
    L.orc_color_render.restype = I64
    for f in ("orc_color_num_voxels", "orc_color_num_rgb_points"):
        getattr(L, f).argtypes = [P]
        getattr(L, f).restype = I64
    L.orc_color_snapshot.argtypes = [P, I32] + [P] * 9
    L.orc_color_snapshot.restype = I64
    L.orc_color_export.argtypes = [P, I32, I32, P, P]
    L.orc_color_export.restype = I64
    _lib = L
    return L


class OracleMap:
    """voxelHashMap + addPointsToMap with the cloud publishCLoudWorld sends."""

    def __init__(self):
        self._h = C.c_void_p(lib().orc_map_create())

    def __del__(self):
        try:
            if self._h:
                lib().orc_map_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def add_points_published(self, xyz, translation_z, voxel_size=1.0, max_num_points_in_voxel=20, min_distance_points=0.15,
                             min_num_points=0):
        """(points stored, (n_published, 4) float32 x, y, z, intensity in sweep order) — addPointToPcl, src/lioOptimization.cpp:432,
        1346-1355."""
        xyz = _f64(xyz).reshape(-1, 3)
        out = np.zeros((xyz.shape[0], 4), np.float32)
        n_pub = C.c_int64(0)
        added = lib().orc_map_add_points_published(self._h, _ptr(xyz), xyz.shape[0], voxel_size, max_num_points_in_voxel,
                                                   min_distance_points, min_num_points, float(translation_z), _ptr(out), C.byref(n_pub))
        return int(added), out[:n_pub.value].copy()

    def remove_far(self, location, distance: float) -> int:
        """removePointsFarFromLocation (src/lioOptimization.cpp:556-572): voxels erased."""
        loc = _f64(location).reshape(3)
        return int(lib().orc_map_remove_far(self._h, _ptr(loc), float(distance)))

    def snapshot(self, cap=20):
        n = int(lib().orc_map_num_voxels(self._h))
        keys, counts, xyz = np.zeros((n, 3), np.int16), np.zeros(n, np.int32), np.zeros((n, cap, 3), np.float32)
        assert lib().orc_map_snapshot(self._h, cap, _ptr(keys), _ptr(counts), _ptr(xyz)) == n
        return keys, counts, xyz

    def load(self, keys, counts, xyz):
        keys = np.ascontiguousarray(keys, np.int16); counts = np.ascontiguousarray(counts, np.int32)
        xyz = np.ascontiguousarray(xyz, np.float32)
        lib().orc_map_load(self._h, _ptr(keys), _ptr(counts), _ptr(xyz), keys.shape[0], xyz.shape[1])


class OracleColorMap:
    """The colour map of oracle_py.OracleColorMap (same restatement) + pubColorPoints / saveColorPoints."""

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
        xyz = _f64(xyz).reshape(-1, 3)
        return int(lib().orc_color_add_points(self._h, _ptr(xyz), xyz.shape[0], self.voxel_size, self.cap, self.min_dist, add_point_step,
                                              time_sweep_end, time_last_process, 1 if to_rendering else 0))

    def render(self, cam15, image_bgr, obs_time) -> int:
        cam = _f64(cam15).reshape(15)
        img = np.ascontiguousarray(image_bgr, np.uint8)
        return int(lib().orc_color_render(self._h, _ptr(cam), _ptr(img), img.shape[0], img.shape[1], float(obs_time)))

    def num_rgb_points(self) -> int:
        return int(lib().orc_color_num_rgb_points(self._h))

    def max_n_rgb(self) -> int:
        """the largest N_rgb of any stored point"""
        nv, cap = int(lib().orc_color_num_voxels(self._h)), self.cap
        a = {k: np.zeros(s, t) for k, s, t in (("keys", (nv, 3), np.int16), ("counts", nv, np.int32), ("xyz", (nv, cap, 3), np.float32),
                                               ("rgb", (nv, cap, 3), np.int16), ("n_rgb", (nv, cap), np.int16),
                                               ("cov", (nv, cap, 3), np.float32), ("obs_dist", (nv, cap), np.float64),
                                               ("last_obs", (nv, cap), np.float64), ("last_visited", nv, np.float64))}
        lib().orc_color_snapshot(self._h, cap, *[_ptr(a[k]) for k in ("keys", "counts", "xyz", "rgb", "n_rgb", "cov", "obs_dist",
                                                                      "last_obs", "last_visited")])
        return int(a["n_rgb"].max()) if nv else 0

    def export(self, min_views, order):
        """pubColorPoints (order 0) / saveColorPoints (order 1): ((n, 3) float32 positions, (n, 3) uint8 r, g, b)."""
        n = int(lib().orc_color_export(self._h, int(min_views), int(order), None, None))
        xyz, rgb = np.zeros((n, 3), np.float32), np.zeros((n, 3), np.uint8)
        if n:
            lib().orc_color_export(self._h, int(min_views), int(order), _ptr(xyz), _ptr(rgb))
        return xyz, rgb
