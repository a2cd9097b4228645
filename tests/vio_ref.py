"""ctypes binding of oracle/_ref/libsrl_vio_ref.so (oracle/vio.mk, oracle/srl_vio_harness.cpp): the reference's own
imageProcessing::vioEsikf / vioPhotometric and cloudFrame::getRgb, compiled unmodified over the stand-in headers.

Test infrastructure: the tests skip what needs it when the library was not built (it needs the reference tree to build).
"""
import ctypes as C
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libsrl_vio_ref.so")
_lib = None


def available() -> bool:
    return os.path.exists(PATH)


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(PATH)
        P, I32, I64, D = C.c_void_p, C.c_int32, C.c_int64, C.c_double
        L.vio_ref_update.argtypes = [I32, P, P, I32, P, P, P, P, P, P, I32, P, I32, I32, P]
        L.vio_ref_update.restype = I64
        L.vio_ref_get_rgb.argtypes = [P, I32, I32, D, D, P]
        L.vio_ref_get_rgb.restype = None
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def update(which, state, cov, xyz, uv, vel, rgb, cov_rgb, n_rgb, n_new_visited, img=None):
    """which 0 vioEsikf, 1 vioPhotometric, 2 both in process's order.  state: 38 doubles (srl_vio_state's layout).
    Returns (state', cov', (result esikf, result photometric) with -1 where not run, nanoseconds)."""
    st = np.array(state, np.float64).reshape(38).copy()
    cv = np.array(cov, np.float64).reshape(11, 11).copy()
    n = len(xyz)
    xyz = np.ascontiguousarray(xyz, np.float32)
    uv = None if uv is None else np.ascontiguousarray(uv, np.float32)
    vel = np.ascontiguousarray(vel, np.float64)
    rgb = np.ascontiguousarray(rgb, np.int16)
    cov_rgb = np.ascontiguousarray(cov_rgb, np.float32)
    n_rgb = np.ascontiguousarray(n_rgb, np.int16)
    res = np.zeros(2, np.int32)
    rows = cols = 0
    if img is not None:
        img = np.ascontiguousarray(img, np.uint8)
        rows, cols = img.shape[:2]
    ns = lib().vio_ref_update(int(which), _p(st), _p(cv), n, _p(xyz), _p(uv), _p(vel), _p(rgb), _p(cov_rgb), _p(n_rgb),
                              int(n_new_visited), _p(img), cols, rows, _p(res))
    return st, cv, (int(res[0]), int(res[1])), int(ns)


def get_rgb(img, u, v):
    """cloudFrame::getRgb(u, v, 0, &dx, &dy): (value, dx, dy) as three float64 3-vectors."""
    img = np.ascontiguousarray(img, np.uint8)
    out = np.zeros(9, np.float64)
    lib().vio_ref_get_rgb(_p(img), img.shape[1], img.shape[0], float(u), float(v), _p(out))
    return out[:3], out[3:6], out[6:]
