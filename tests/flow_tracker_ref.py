"""ctypes binding of oracle/_ref/libsrl_flow_tracker_ref.so (oracle/flow_tracker.mk, oracle/srl_flow_tracker_harness.cpp): the
reference's own opticalFlowTracker::init, trackImage, removeOutlierUsingRansacPnp and updateAndAppendTrackPoints, compiled
unmodified over the stand-in headers.  Lucas-Kanade, findFundamentalMat and solvePnPRansac are the test's: a Python function
for Lucas-Kanade and for the mask, a list of inliers (or a throw) for the PnP step.

Test infrastructure: the tests skip what needs it when the library was not built (it needs the reference tree to build).
"""
import ctypes as C
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libsrl_flow_tracker_ref.so")
LK_FN = C.CFUNCTYPE(None, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_uint8))
MASK_FN = C.CFUNCTYPE(None, C.c_int, C.POINTER(C.c_uint8))
_lib = None
_NO_INLIERS = np.zeros(1, np.int32)


def available() -> bool:
    return os.path.exists(PATH)


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(PATH)
        P, I32, I64, D = C.c_void_p, C.c_int32, C.c_int64, C.c_double
        L.ft_ref_set_callbacks.argtypes = [LK_FN, MASK_FN]
        L.ft_ref_set_callbacks.restype = None
        L.ft_ref_lk_calls.restype = C.c_long
        L.ft_ref_create.argtypes = [I32, I32, P]
        L.ft_ref_create.restype = P
        L.ft_ref_destroy.argtypes = [P]
        L.ft_ref_destroy.restype = None
        L.ft_ref_set_counts.argtypes = [P, P, I32, P]
        L.ft_ref_set_counts.restype = None
        L.ft_ref_get_counts.argtypes = [P, P, I32, P]
        L.ft_ref_get_counts.restype = None
        L.ft_ref_init.argtypes = [P, D, P, P, I32]
        L.ft_ref_init.restype = I64
        L.ft_ref_track.argtypes = [P, D, I32, I32]
        L.ft_ref_track.restype = I64
        L.ft_ref_remove_outliers.argtypes = [P, P, I32, I32, C.POINTER(I32)]
        L.ft_ref_remove_outliers.restype = I64
        L.ft_ref_update.argtypes = [P, P, I32, I32, D, P, I32]
        L.ft_ref_update.restype = I64
        L.ft_ref_get.argtypes = [P, I32, P, P, P]
        L.ft_ref_get.restype = I32
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class FlowTrackerReference:
    """xyz: (n_points, 3) stored positions, point id = row.  Every call returns the reference's wall time in ns in self.ns."""

    def __init__(self, xyz, maximum_tracked_points: int = 300):
        self.xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
        self.h = lib().ft_ref_create(int(maximum_tracked_points), len(self.xyz), _p(self.xyz))
        self.ns = 0
        self._lk = None
        self._mask = None

    def close(self):
        if self.h:
            lib().ft_ref_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _callbacks(self, lk, mask_fn):
        def lk_c(n, last, cur, status):
            pts = np.ctypeslib.as_array(last, (n, 2)).copy()
            out = lk(pts)
            if out is None:                 # init's call: the first image, points copied, status untouched
                return
            new_uv, st = out
            np.ctypeslib.as_array(cur, (n, 2))[:] = np.asarray(new_uv, np.float32).reshape(n, 2)
            np.ctypeslib.as_array(status, (n,))[:] = np.asarray(st, np.uint8).reshape(n)

        def mask_c(n, m):
            if mask_fn is not None:
                np.ctypeslib.as_array(m, (n,))[:] = np.asarray(mask_fn(n), np.uint8).reshape(n)

        self._lk, self._mask = LK_FN(lk_c), MASK_FN(mask_c)   # kept alive while the library may call them
        lib().ft_ref_set_callbacks(self._lk, self._mask)

    @staticmethod
    def lk_calls() -> int:
        return int(lib().ft_ref_lk_calls())

    def set_counts(self, ids, counts):
        ids = np.ascontiguousarray(ids, np.uint32)
        c = np.ascontiguousarray(counts, np.int16)
        lib().ft_ref_set_counts(self.h, _p(ids), len(ids), _p(c))

    def counts(self, ids):
        ids = np.ascontiguousarray(ids, np.uint32)
        out = np.zeros(len(ids), np.int16)
        lib().ft_ref_get_counts(self.h, _p(ids), len(ids), _p(out))
        return out

    def init(self, image_time, ids, uv, lk):
        """lk(points) is called for the first image too; its result there is ignored (return None)"""
        self._callbacks(lambda p: (lk(p), None)[1], None)
        ids = np.ascontiguousarray(ids, np.uint32)
        uv = np.ascontiguousarray(uv, np.float32).reshape(-1, 2)
        self.ns = lib().ft_ref_init(self.h, float(image_time), _p(ids), _p(uv), len(ids))

    def track_image(self, image_time, lk, cols, rows, mask_fn=None):
        """mask_fn(n) -> findFundamentalMat's status over the n matches (None: all inliers)"""
        self._callbacks(lk, mask_fn)
        self.ns = lib().ft_ref_track(self.h, float(image_time), int(cols), int(rows))

    def remove_outliers(self, inliers, throws=False) -> bool:
        r = C.c_int32(0)
        a = None if inliers is None else np.ascontiguousarray(inliers, np.int32).reshape(-1)
        p = None if a is None else _p(a if a.size else _NO_INLIERS)   # an empty list is zero inliers, not "all of cur"
        self.ns = lib().ft_ref_remove_outliers(self.h, p, 0 if a is None else a.size, 1 if throws else 0, C.byref(r))
        return bool(r.value)

    def update_and_append(self, cam15, cols, rows, candidates, mini_distance):
        c = np.ascontiguousarray(cam15, np.float64).reshape(15)
        cand = np.ascontiguousarray(candidates, np.uint32)
        self.ns = lib().ft_ref_update(self.h, _p(c), int(cols), int(rows), float(mini_distance), _p(cand), len(cand))

    def last_arrays(self):
        n = lib().ft_ref_get(self.h, 0, None, None, None)
        ids, uv = np.zeros(n, np.uint32), np.zeros((n, 2), np.float32)
        lib().ft_ref_get(self.h, 0, _p(ids), _p(uv), None)
        return ids, uv

    def cur_arrays(self):
        n = lib().ft_ref_get(self.h, 1, None, None, None)
        ids, uv, vel = np.zeros(n, np.uint32), np.zeros((n, 2), np.float32), np.zeros((n, 2), np.float64)
        lib().ft_ref_get(self.h, 1, _p(ids), _p(uv), _p(vel))
        return ids, uv, vel
