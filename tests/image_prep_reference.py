"""Plain numpy restatement of the camera image preparation of imageProcessing::process (src/imageProcessing.cpp:91-125,166-200),
one short function per OpenCV stage, each in OpenCV's own integer or float order:

  initUndistortRectifyMap(K, dist, I, K, size, CV_16SC2)   undistort_maps
  remap(bgr, map1, map2, INTER_LINEAR, BORDER_CONSTANT 0)  remap_bilinear
  cvtColor(COLOR_RGB2GRAY) / (BGR2YCrCb, YCrCb2BGR)        rgb2gray / bgr2ycrcb / ycrcb2bgr
  createCLAHE(clip, (t, t))->apply                         clahe
  the whole recipe                                         process

No cv2 here: tests compare this file with the golden vectors (made by cv2) and, when cv2 is importable, with cv2 itself.
"""
from __future__ import annotations

import numpy as np

F32 = np.float32


def _cv_round(v: np.ndarray) -> np.ndarray:
    """saturate_cast<int>(double) as x86-64 cvRound has it: nearest even; INT_MIN outside the int range and for NaN."""
    r = np.rint(v)
    ok = (r >= -2147483648.0) & (r <= 2147483647.0)
    out = np.full(r.shape, -2147483648, np.int64)
    out[ok] = r[ok].astype(np.int64)
    return out


def inv3(K: np.ndarray) -> np.ndarray:
    """Mat::inv(DECOMP_LU) of a 3x3 double matrix: cofactors times 1 / det3, each product rounded."""
    a = np.asarray(K, np.float64).reshape(3, 3)
    d = (a[0, 0] * (a[1, 1] * a[2, 2] - a[1, 2] * a[2, 1]) - a[0, 1] * (a[1, 0] * a[2, 2] - a[1, 2] * a[2, 0])
         + a[0, 2] * (a[1, 0] * a[2, 1] - a[1, 1] * a[2, 0]))
    d = 1.0 / d
    return np.array([
        (a[1, 1] * a[2, 2] - a[1, 2] * a[2, 1]) * d, (a[0, 2] * a[2, 1] - a[0, 1] * a[2, 2]) * d, (a[0, 1] * a[1, 2] - a[0, 2] * a[1, 1]) * d,
        (a[1, 2] * a[2, 0] - a[1, 0] * a[2, 2]) * d, (a[0, 0] * a[2, 2] - a[0, 2] * a[2, 0]) * d, (a[0, 2] * a[1, 0] - a[0, 0] * a[1, 2]) * d,
        (a[1, 0] * a[2, 1] - a[1, 1] * a[2, 0]) * d, (a[0, 1] * a[2, 0] - a[0, 0] * a[2, 1]) * d, (a[0, 0] * a[1, 1] - a[0, 1] * a[1, 0]) * d,
    ], np.float64)


def first_image(image_width: int, image_height: int, camera_intrinsic, cols: int) -> tuple[float, np.ndarray, int, int, int]:
    """process's first-image step (:93-104): (image_scale_factor, scaled K, out_cols, out_rows, CLAHE tiles).  cv::Size of a
    double truncates; the tile grid is imageEqualize's (:169), square and taken from the output's cols."""
    s = image_width * 1.0 / cols
    K = np.array(camera_intrinsic, np.float64).reshape(3, 3).copy()
    K[0, 0] /= s
    K[0, 2] /= s
    K[1, 1] /= s
    K[1, 2] /= s
    out_cols, out_rows = int(image_width / s), int(image_height / s)
    return s, K, out_cols, out_rows, clahe_tiles(out_cols)


def clahe_tiles(cols: int) -> int:
    return int(max(cols * 32.0 / 640, 4.0))


def undistort_coords(K: np.ndarray, dist, out_cols: int, out_rows: int) -> tuple[np.ndarray, np.ndarray]:
    """(32 u, 32 v) (rows, cols) float64 of initUndistortRectifyMap with R = I and newK = K, before cvRound: per row, _x/_y/_w
    start at i*ir[1] + ir[2], ... and step by += ir[0], ...; the rational model with k4..k6 = s1..s4 = 0 and no tilt."""
    ir = inv3(K)
    fx, fy, u0, v0 = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    k1, k2, p1, p2, k3 = (float(v) for v in dist)
    i = np.arange(out_rows, dtype=np.float64)
    _x, _y, _w = i * ir[1] + ir[2], i * ir[4] + ir[5], i * ir[7] + ir[8]
    u32 = np.empty((out_rows, out_cols), np.float64)
    v32 = np.empty((out_rows, out_cols), np.float64)
    for j in range(out_cols):
        w = 1.0 / _w
        x, y = _x * w, _y * w
        x2, y2 = x * x, y * y
        r2, _2xy = x2 + y2, 2 * x * y
        kr = (1 + ((k3 * r2 + k2) * r2 + k1) * r2) / (1 + ((0.0 * r2 + 0.0) * r2 + 0.0) * r2)
        xd = x * kr + p1 * _2xy + p2 * (r2 + 2 * x2) + 0.0 * r2 + 0.0 * r2 * r2
        yd = y * kr + p1 * (r2 + 2 * y2) + p2 * _2xy + 0.0 * r2 + 0.0 * r2 * r2
        u32[:, j] = (fx * 1.0 * xd + u0) * 32
        v32[:, j] = (fy * 1.0 * yd + v0) * 32
        _x, _y, _w = _x + ir[0], _y + ir[3], _w + ir[6]
    return u32, v32


def undistort_maps(K: np.ndarray, dist, out_cols: int, out_rows: int) -> tuple[np.ndarray, np.ndarray]:
    """(map1 (rows, cols, 2) int16, map2 (rows, cols) uint16) of initUndistortRectifyMap(..., CV_16SC2) with R = I and newK = K:
    iu = cvRound(32 u), map1 = (iu >> 5, iv >> 5) saturated to int16, map2 = (iv & 31) * 32 + (iu & 31)."""
    u32, v32 = undistort_coords(K, dist, out_cols, out_rows)
    iu, iv = _cv_round(u32), _cv_round(v32)
    # saturate_cast<short>, as OpenCV's vectorised rows pack map1: an iu of INT_MIN (NaN or out of the int range) gives -32768,
    # and a coordinate past +-32767 px stays outside the image instead of wrapping back into it
    map1 = np.stack([np.clip(iu >> 5, -32768, 32767).astype(np.int16), np.clip(iv >> 5, -32768, 32767).astype(np.int16)], axis=-1)
    map2 = ((iv & 31) * 32 + (iu & 31)).astype(np.uint16)
    return map1, map2


def saturated(map1: np.ndarray) -> np.ndarray:
    """(rows, cols) bool: the map entries whose source coordinate saturated map1 in either component.  Every tap of such an
    entry lies outside the image; a vectorised OpenCV may give their map2 a different last bit."""
    return ((map1 == -32768) | (map1 == 32767)).any(axis=-1)


def remap_bilinear(src: np.ndarray, map1: np.ndarray, map2: np.ndarray) -> np.ndarray:
    """remap INTER_LINEAR of a (rows, cols, cn) uint8 image with fixed-point maps: 15-bit weights (32 - fx)(32 - fy) * 32, ...,
    taps outside the image read 0."""
    h, w = src.shape[:2]
    sx, sy = map1[..., 0].astype(np.int64), map1[..., 1].astype(np.int64)
    fx, fy = (map2 & 31).astype(np.int64), ((map2 >> 5) & 31).astype(np.int64)
    acc = np.zeros(map2.shape + src.shape[2:], np.int64)
    for dy, dx, wt in ((0, 0, (32 - fx) * (32 - fy)), (0, 1, fx * (32 - fy)), (1, 0, (32 - fx) * fy), (1, 1, fx * fy)):
        X, Y = sx + dx, sy + dy
        inside = (X >= 0) & (X < w) & (Y >= 0) & (Y < h)
        v = src[np.where(inside, Y, 0), np.where(inside, X, 0)].astype(np.int64)
        v[~inside] = 0
        acc += v * (wt * 32).reshape(wt.shape + (1,) * (src.ndim - 2))
    return ((acc + (1 << 14)) >> 15).astype(np.uint8)


def rgb2gray(img: np.ndarray) -> np.ndarray:
    """COLOR_RGB2GRAY on 8 bits: channel 0 weighted as R, 15-bit weights."""
    c = img.astype(np.int64)
    return ((c[..., 0] * 9798 + c[..., 1] * 19235 + c[..., 2] * 3735 + (1 << 14)) >> 15).astype(np.uint8)


def bgr2ycrcb(img: np.ndarray) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """COLOR_BGR2YCrCb on 8 bits, 14-bit weights: (Y, Cr, Cb)."""
    b, g, r = (img[..., k].astype(np.int64) for k in range(3))
    y = (b * 1868 + g * 9617 + r * 4899 + (1 << 13)) >> 14
    cr = ((r - y) * 11682 + (128 << 14) + (1 << 13)) >> 14
    cb = ((b - y) * 9241 + (128 << 14) + (1 << 13)) >> 14
    return tuple(np.clip(v, 0, 255).astype(np.uint8) for v in (y, cr, cb))


def ycrcb2bgr(y: np.ndarray, cr: np.ndarray, cb: np.ndarray) -> np.ndarray:
    """COLOR_YCrCb2BGR on 8 bits, 14-bit weights."""
    Y, Cr, Cb = (v.astype(np.int64) for v in (y, cr, cb))
    b = Y + (((Cb - 128) * 29049 + (1 << 13)) >> 14)
    g = Y + (((Cb - 128) * -5636 + (Cr - 128) * -11698 + (1 << 13)) >> 14)
    r = Y + (((Cr - 128) * 22987 + (1 << 13)) >> 14)
    return np.clip(np.stack([b, g, r], axis=-1), 0, 255).astype(np.uint8)


def _reflect101(p: np.ndarray, n: int) -> np.ndarray:
    p = p.copy()
    while True:
        bad = (p < 0) | (p >= n)
        if not bad.any():
            return p
        p = np.where(p < 0, -p, np.where(p >= n, 2 * n - p - 2, p))


def clahe_sums(img: np.ndarray, clip: float, t: int) -> tuple[np.ndarray, int, int]:
    """(prefix sums (t * t, 256) int64 of the clipped and redistributed histograms, tile width, tile height) of CLAHE's
    histogram pass.  A size that is not a multiple of the grid in either dimension pads both, by t - size % t (a full t where
    it divides), with REFLECT_101, bottom and right."""
    h, w = img.shape
    if w % t == 0 and h % t == 0:
        ext = img
    else:
        ys, xs = _reflect101(np.arange(h + t - h % t), h), _reflect101(np.arange(w + t - w % t), w)
        ext = img[ys[:, None], xs[None, :]]
    th, tw = ext.shape[0] // t, ext.shape[1] // t
    area = th * tw
    tiles = ext[:th * t, :tw * t].reshape(t, th, t, tw).transpose(0, 2, 1, 3).reshape(t * t, area)
    hist = np.zeros((t * t, 256), np.int64)
    np.add.at(hist, (np.repeat(np.arange(t * t), area), tiles.reshape(-1).astype(np.int64)), 1)
    limit = max(int(clip * area / 256), 1)
    clipped = np.maximum(hist - limit, 0).sum(axis=1)
    hist = np.minimum(hist, limit) + (clipped // 256)[:, None]
    residual = clipped % 256
    step = np.maximum(256 // np.maximum(residual, 1), 1)
    i = np.arange(256)[None, :]
    hist += ((residual[:, None] > 0) & (i % step[:, None] == 0) & (i // step[:, None] < residual[:, None])).astype(np.int64)
    return np.cumsum(hist, axis=1), tw, th


def clahe_luts(img: np.ndarray, clip: float, t: int) -> tuple[np.ndarray, int, int]:
    """(lut (t, t, 256) uint8, tile width, tile height): cvRound((float)sum * (255.f / area)) of clahe_sums, clamped."""
    sums, tw, th = clahe_sums(img, clip, t)
    lut = np.rint(sums.astype(F32) * (F32(255) / F32(tw * th)))
    return np.clip(lut, 0, 255).astype(np.uint8).reshape(t, t, 256), tw, th


def clahe(img: np.ndarray, clip: float, t: int) -> np.ndarray:
    """createCLAHE(clip, (t, t))->apply on a uint8 plane: the LUTs, then the bilinear blend of the four nearest tiles' LUTs in
    CLAHE_Interpolation_Body's float32 expression."""
    lut, tw, th = clahe_luts(img, clip, t)
    h, w = img.shape

    def axis(n, size):
        tf = np.arange(n).astype(F32) * (F32(1) / F32(size)) - F32(0.5)
        t1 = np.floor(tf).astype(np.int64)
        a = tf - t1.astype(F32)
        return np.maximum(t1, 0), np.minimum(t1 + 1, t - 1), a, F32(1) - a

    x1, x2, xa, xa1 = axis(w, tw)
    y1, y2, ya, ya1 = axis(h, th)
    v = img.astype(np.int64)
    Y1, Y2, X1, X2 = y1[:, None], y2[:, None], x1[None, :], x2[None, :]
    l1a, l1b = lut[Y1, X1, v].astype(F32), lut[Y1, X2, v].astype(F32)
    l2a, l2b = lut[Y2, X1, v].astype(F32), lut[Y2, X2, v].astype(F32)
    xa, xa1, ya, ya1 = xa[None, :], xa1[None, :], ya[:, None], ya1[:, None]
    res = (l1a * xa1 + l1b * xa) * ya1 + (l2a * xa1 + l2b * xa) * ya
    return np.clip(np.rint(res), 0, 255).astype(np.uint8)


def process(bgr: np.ndarray, map1: np.ndarray, map2: np.ndarray, t: int) -> tuple[np.ndarray, np.ndarray]:
    """(rgb_image (rows, cols, 3) BGR8, gray_image (rows, cols)) of process:120-125 for one image."""
    und = remap_bilinear(bgr, map1, map2)
    gray = clahe(rgb2gray(und), 3.0, t)
    y, cr, cb = bgr2ycrcb(und)
    return ycrcb2bgr(clahe(y, 1.0, t), cr, cb), gray


def prepare(bgr: np.ndarray, image_width: int, image_height: int, camera_intrinsic, camera_dist_coeffs):
    """The first-image step and process for one image: (rgb, gray, map1, map2, scale factor, scaled K, tiles)."""
    s, K, oc, orows, t = first_image(image_width, image_height, camera_intrinsic, bgr.shape[1])
    map1, map2 = undistort_maps(K, camera_dist_coeffs, oc, orows)
    rgb, gray = process(bgr, map1, map2, t)
    return rgb, gray, map1, map2, s, K, t
