"""ctypes binding of oracle/_ref/libsrl_lk_ref.so (oracle/lk.mk, oracle/srl_lk_harness.cpp): the reference's own
LKOpticalFlowKernel (src/lkpyramid.cpp), compiled unmodified over the OpenCV stand-in of oracle/shim_lk/.

Test infrastructure: the tests skip what needs it when the library was not built (it needs the reference tree to build).
"""
import ctypes as C
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libsrl_lk_ref.so")
_lib = None


def available() -> bool:
    return os.path.exists(PATH)


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(PATH)
        P, I64, I32, D, SZ = C.c_void_p, C.c_int64, C.c_int32, C.c_double, C.c_size_t
        L.lk_create.argtypes = [I32, I32, I32, I32, I32, D, I32, D]
        L.lk_create.restype = P
        L.lk_destroy.argtypes = [P]
        L.lk_destroy.restype = None
        L.lk_track.argtypes = [P, P, I32, I32, SZ, P, I64, P, P]
        L.lk_track.restype = I32
        L.lk_info.argtypes = [P, C.POINTER(I32), C.POINTER(I32), C.POINTER(I32), C.POINTER(I32), C.POINTER(D)]
        L.lk_info.restype = None
        L.lk_level.argtypes = [P, I32, I32, C.POINTER(I32), C.POINTER(I32), P, P]
        L.lk_level.restype = I32
        L.lk_pyr_down.argtypes = [P, I32, I32, P]
        L.lk_pyr_down.restype = None
        L.lk_copy_make_border.argtypes = [P, I32, I32, I32, I32, I32, I32, I32, I32, I32, I32, I32, I32, I32, P, C.POINTER(I32), C.POINTER(I32)]
        L.lk_copy_make_border.restype = I32
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


class LKReference:
    """One LKOpticalFlowKernel of the reference (include/lkpyramid.h:100-106 constructor)."""

    def __init__(self, win_size=(21, 21), max_level=3, criteria=(3, 30, 0.01), flags=0, min_eig_threshold=1e-4):
        t, c, e = criteria
        self._h = C.c_void_p(lib().lk_create(int(win_size[0]), int(win_size[1]), int(max_level), int(t), int(c), float(e), int(flags),
                                             float(min_eig_threshold)))

    def close(self):
        if self._h:
            lib().lk_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def track(self, gray, last_pts, status_in=None):
        """trackImage: (curr_pts (n, 2) float32, status (n,) uint8, return value).  status_in (default ones) is what the status
        vector holds before the call; the first call leaves it as it is."""
        img = np.ascontiguousarray(gray, np.uint8)
        pts = np.ascontiguousarray(last_pts, np.float32).reshape(-1, 2)
        n = pts.shape[0]
        curr = np.zeros((n, 2), np.float32)
        st = np.ones(n, np.uint8) if status_in is None else np.array(status_in, np.uint8).reshape(n)
        ret = lib().lk_track(self._h, _ptr(img), img.shape[1], img.shape[0], img.strides[0], _ptr(pts), n, _ptr(curr), _ptr(st))
        assert ret >= 0, "trackImage returned vectors of the wrong size"
        return curr, st, int(ret)

    def info(self) -> dict:
        ml, ww, wh, mc = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32()
        eps = C.c_double()
        lib().lk_info(self._h, C.byref(ml), C.byref(ww), C.byref(wh), C.byref(mc), C.byref(eps))
        return dict(max_level=ml.value, win=(ww.value, wh.value), max_count=mc.value, epsilon=eps.value)

    def level(self, which, level):
        """(padded image (rows + 2 win_h, cols + 2 win_w) uint8, derivative buffer (..., ..., 2) int16) of a pyramid level:
        which 0 is the last image's pyramid, 1 the one before it."""
        cols, rows = C.c_int32(), C.c_int32()
        if lib().lk_level(self._h, which, level, C.byref(cols), C.byref(rows), None, None) != 0:
            raise IndexError(level)
        ww, wh = self.info()["win"]
        img = np.zeros((rows.value + 2 * wh, cols.value + 2 * ww), np.uint8)
        der = np.zeros((rows.value + 2 * wh, cols.value + 2 * ww, 2), np.int16)
        assert lib().lk_level(self._h, which, level, C.byref(cols), C.byref(rows), _ptr(img), _ptr(der)) == 0
        return img, der


def pyr_down(src):
    src = np.ascontiguousarray(src, np.uint8)
    h, w = src.shape
    dst = np.zeros(((h + 1) // 2, (w + 1) // 2), np.uint8)
    lib().lk_pyr_down(_ptr(src), w, h, _ptr(dst))
    return dst


def copy_make_border(whole, roi, top, bottom, left, right, border, inplace=False):
    """The stand-in's copyMakeBorder of the ROI (x, y, w, h) of `whole` ((rows, cols) uint8 or (rows, cols, 2) int16)."""
    whole = np.ascontiguousarray(whole)
    elem = 1 if whole.dtype == np.uint8 else 4
    rows, cols = whole.shape[:2]
    x, y, w, h = roi
    dc, dr = C.c_int32(), C.c_int32()
    args = [_ptr(whole), cols, rows, elem, x, y, w, h, top, bottom, left, right, border, 1 if inplace else 0]
    assert lib().lk_copy_make_border(*args, None, C.byref(dc), C.byref(dr)) == 0
    out = np.zeros((dr.value, dc.value) + whole.shape[2:], whole.dtype)
    assert lib().lk_copy_make_border(*args, _ptr(out), C.byref(dc), C.byref(dr)) == 0
    return out
