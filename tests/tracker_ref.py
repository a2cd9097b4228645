"""ctypes binding of oracle/_ref/libsrl_tracker_ref.so (oracle/tracker.mk, oracle/srl_tracker_harness.cpp): the reference's own
selectPointsForProjection and refreshPointsForProjection, compiled from its sources, over a colour map its addPointsToMap fills.

Test infrastructure: the tests skip what needs it when the library was not built (it needs the reference tree to build).
"""
import ctypes as C
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libsrl_tracker_ref.so")
_lib = None


def available() -> bool:
    return os.path.exists(PATH)


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(PATH)
        P, I64, I32, D = C.c_void_p, C.c_int64, C.c_int32, C.c_double
        L.trk_create.restype = P
        L.trk_destroy.argtypes = [P]
        L.trk_add_points_to_map.argtypes = [P, P, I64, D, I32, D, I32, D, D, I32]
        L.trk_add_points_to_map.restype = I64
        L.trk_color_render.argtypes = [P, P, P, I32, I32, D]
        L.trk_color_render.restype = I64
        for f in ("trk_color_num_recent", "trk_color_num_rgb_points"):
            getattr(L, f).argtypes = [P]
            getattr(L, f).restype = I64
        L.ref_color_select.argtypes = [P, P, I32, I32, D, I32, I32, D, D, P, P, I64]
        L.ref_color_select.restype = I64
        L.ref_color_refresh.argtypes = [P, P, P, D, D, D, D, I32, I32, I32, P, I64, P, P]
        L.ref_color_refresh.restype = I64
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


class TrackerReference:
    """One lioOptimization object of the reference: its colour map and its rgbMapTracker."""

    def __init__(self, voxel_size=0.1, max_num_points_in_voxel=50, min_distance_points=0.01):
        self._h = C.c_void_p(lib().trk_create())
        self.voxel_size, self.cap, self.min_dist = voxel_size, max_num_points_in_voxel, min_distance_points

    def __del__(self):
        try:
            if self._h:
                lib().trk_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def add_points(self, xyz, add_point_step=1, time_sweep_end=1.0, time_last_process=0.0, to_rendering=True) -> int:
        xyz = np.ascontiguousarray(xyz, np.float64).reshape(-1, 3)
        return int(lib().trk_add_points_to_map(self._h, _ptr(xyz), xyz.shape[0], self.voxel_size, self.cap, self.min_dist, add_point_step,
                                               time_sweep_end, time_last_process, 1 if to_rendering else 0))

    def render(self, cam15, image_bgr, obs_time) -> int:
        cam = np.ascontiguousarray(cam15, np.float64).reshape(15)
        img = np.ascontiguousarray(image_bgr, np.uint8)
        return int(lib().trk_color_render(self._h, _ptr(cam), _ptr(img), img.shape[0], img.shape[1], float(obs_time)))

    def num_recent(self) -> int:
        return int(lib().trk_color_num_recent(self._h))

    def num_rgb_points(self) -> int:
        return int(lib().trk_color_num_rgb_points(self._h))

    def select(self, cam15, rows=480, cols=640, minimum_dis=5.0, skip_step=1, use_all_points=False, minimum_depth=0.1, maximum_depth=200.0):
        cam = np.ascontiguousarray(cam15, np.float64).reshape(15)
        args = (self._h, _ptr(cam), int(rows), int(cols), float(minimum_dis), int(skip_step), 1 if use_all_points else 0, float(minimum_depth),
                float(maximum_depth))
        n = int(lib().ref_color_select(*args, None, None, 0))
        ki, uv = np.zeros((n, 4), np.int16), np.zeros((n, 2), np.float32)
        if n:
            assert lib().ref_color_select(*args, _ptr(ki), _ptr(uv), n) == n
        return ki, uv

    def refresh(self, q_world_camera, t_world_camera, fx, fy, cx, cy, rows, cols, frame_id):
        """updatePoseForProjection(frame, -0.4) + refreshPointsForProjection: ((n, 4) key_index of points_rgb_vec_for_projection,
        q_camera_world (x, y, z, w), t_camera_world) as the tracker derived them."""
        q = np.ascontiguousarray(q_world_camera, np.float64).reshape(4)
        t = np.ascontiguousarray(t_world_camera, np.float64).reshape(3)
        q_cw, t_cw = np.zeros(4), np.zeros(3)
        args = (self._h, _ptr(q), _ptr(t), float(fx), float(fy), float(cx), float(cy), int(rows), int(cols), int(frame_id))
        n = int(lib().ref_color_refresh(*args, None, 0, _ptr(q_cw), _ptr(t_cw)))
        assert n >= 0
        ki = np.zeros((n, 4), np.int16)
        if n:   # the same frame_id again returns early and leaves the selection as it is
            assert lib().ref_color_refresh(*args, _ptr(ki), n, _ptr(q_cw), _ptr(t_cw)) == n
        return ki, q_cw, t_cw
