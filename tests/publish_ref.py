"""ctypes binding of oracle/_ref/libsrl_publish_ref.so (oracle/publish.mk, oracle/srl_publish_harness.cpp): the reference's own
addPointsToMap, pubColorPoints and saveColorPoints, compiled from its sources, with the clouds they publish and save captured.

Test infrastructure: the tests skip what needs it when the library was not built (it needs the reference tree to build).
"""
import ctypes as C
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libsrl_publish_ref.so")
_lib = None


def available() -> bool:
    return os.path.exists(PATH)


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(PATH)
        P, I64, I32, D = C.c_void_p, C.c_int64, C.c_int32, C.c_double
        L.pub_create.restype = P
        L.pub_destroy.argtypes = [P]
        L.pub_add_points_to_map.argtypes = [P, P, I64, D, I32, D, I32, D, D, I32, D, I32, D, D, I32, P, C.POINTER(I64)]
        L.pub_add_points_to_map.restype = I64
        L.pub_color_render.argtypes = [P, P, P, I32, I32, D]
        L.pub_color_render.restype = I64
        L.pub_color_num_rgb_points.argtypes = [P]
        L.pub_color_num_rgb_points.restype = I64
        L.pub_color_export.argtypes = [P, I32, I32, P, P]
        L.pub_color_export.restype = I64
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


class PublishReference:
    """One lioOptimization object of the reference whose published clouds are observable."""

    def __init__(self):
        self._h = C.c_void_p(lib().pub_create())

    def __del__(self):
        try:
            if self._h:
                lib().pub_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def add_points_to_map(self, world_xyz, translation_z, voxel_size=1.0, max_num_points_in_voxel=20, min_distance_points=0.15,
                          min_num_points=0, color_voxel_size=0.1, color_max_points=20, color_min_distance=0.01, add_point_step=4,
                          time_sweep_end=1.0, time_last_process=-1e5, to_rendering=False):
        """addPointsToMap (both maps): (points stored in the LIO map, (n_published, 4) float32 cloud of publishCLoudWorld)."""
        xyz = np.ascontiguousarray(world_xyz, np.float64).reshape(-1, 3)
        out = np.zeros((xyz.shape[0], 4), np.float32)
        n_pub = C.c_int64(0)
        added = lib().pub_add_points_to_map(self._h, _ptr(xyz), xyz.shape[0], voxel_size, max_num_points_in_voxel, min_distance_points,
                                            min_num_points, float(translation_z), color_voxel_size, color_max_points, color_min_distance,
                                            add_point_step, time_sweep_end, time_last_process, 1 if to_rendering else 0, _ptr(out),
                                            C.byref(n_pub))
        assert added >= 0, "addPointsToMap did not publish exactly one cloud"
        return int(added), out[:n_pub.value].copy()

    def color_render(self, cam15, image_bgr, obs_time) -> int:
        cam = np.ascontiguousarray(cam15, np.float64).reshape(15)
        img = np.ascontiguousarray(image_bgr, np.uint8)
        return int(lib().pub_color_render(self._h, _ptr(cam), _ptr(img), img.shape[0], img.shape[1], float(obs_time)))

    def num_rgb_points(self) -> int:
        return int(lib().pub_color_num_rgb_points(self._h))

    def export(self, min_views, order):
        """order 0: pubColorPoints, 1: saveColorPoints -> ((n, 3) float32, (n, 3) uint8 r, g, b)."""
        n = int(lib().pub_color_export(self._h, int(min_views), int(order), None, None))
        assert n >= 0, "no cloud was handed over"
        xyz, rgb = np.zeros((n, 3), np.float32), np.zeros((n, 3), np.uint8)
        if n:
            assert lib().pub_color_export(self._h, int(min_views), int(order), _ptr(xyz), _ptr(rgb)) == n
        return xyz, rgb
