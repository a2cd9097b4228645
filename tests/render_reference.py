"""A plain restatement of the colour renderer, independent of the C++ oracle: renderPointsInRecentVoxel
(src/rgbMapTracker.cpp:181-237) -> project3dPointInThisImage (src/lioOptimization.cpp:142-198) -> getSubPixel<cv::Vec3b>
(:71-98) -> rgbPoint::updateRgb (src/cloudMap.cpp:59-101), one point at a time.

Every operation is one IEEE operation in the reference's order: Python floats and numpy float64 scalars are binary64 with
round-to-nearest-even per operation, numpy float32 scalars are binary32.  Nothing is vectorised, nothing is fused.

Two exact layers sit beside it:
  * `Fraction` certifies the crafted ties (a tap product that is exactly k + 1/2) and gives the exact bilinear value;
  * `exact_cov_chain` runs updateRgb's covariance recursion in mpmath at 80 digits, without the float / double roundings.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from fractions import Fraction

import mpmath
import numpy as np

F32 = np.float32
SIGMA = 15.0                 # image_obs_cov (src/rgbMapTracker.cpp:176)
PROCESS_NOISE = 0.1          # process_noise_sigma (src/cloudMap.cpp:56)


def quat_to_rot(q):
    """Eigen::Quaterniond::toRotationMatrix, q = (x, y, z, w), as a row-major list of 9 doubles."""
    x, y, z, w = (float(a) for a in q)
    tx, ty, tz = 2.0 * x, 2.0 * y, 2.0 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return [1.0 - (tyy + tzz), txy - twz, txz + twy,
            txy + twz, 1.0 - (txx + tzz), tyz - twx,
            txz - twy, tyz + twx, 1.0 - (txx + tyy)]


@dataclass
class Camera:
    """the 15 doubles the oracle and the reference take (q_camera_world x,y,z,w, t_camera_world, t_world_camera, fx, fy, cx,
    cy, fov_margin) and the image size"""
    cam15: np.ndarray
    rows: int
    cols: int

    def __post_init__(self):
        self.cam15 = np.asarray(self.cam15, np.float64).reshape(15)
        self.R = quat_to_rot(self.cam15[0:4])
        self.t_cw = [float(a) for a in self.cam15[4:7]]
        self.t_wc = [float(a) for a in self.cam15[7:10]]
        self.fx, self.fy, self.cx, self.cy, self.fov = (float(a) for a in self.cam15[10:15])


def stored(p):
    """a world point as the colour map stores it: float32, widened back to double"""
    return tuple(float(F32(a)) for a in p)


def camera_point(cam: Camera, p):
    """q_camera_world.toRotationMatrix() * point_world + t_camera_world, each row reduced as c0 + (c1 + c2)"""
    x, y, z = stored(p)
    R = cam.R
    return tuple((R[3 * i] * x + (R[3 * i + 1] * y + R[3 * i + 2] * z)) + cam.t_cw[i] for i in range(3))


def window(cam: Camera):
    """if2dPointsAvailable's bounds: (u_lo, u_hi, v_lo, v_hi) with u >= u_lo and ceil(u) < u_hi"""
    f = cam.fov
    return f * cam.cols + 1, (1 - f) * cam.cols, f * cam.rows + 1, (1 - f) * cam.rows


def project(cam: Camera, p):
    """project3dTo2d (scale 1) then if2dPointsAvailable: (u, v) or None.  Also returns why a point fell out."""
    pcx, pcy, pcz = camera_point(cam, p)
    if pcz < 0.001:
        return None, "depth"
    u = pcx * cam.fx / pcz + cam.cx
    v = pcy * cam.fy / pcz + cam.cy
    u_lo, u_hi, v_lo, v_hi = window(cam)
    if not (u >= u_lo and math.ceil(u) < u_hi and v >= v_lo and math.ceil(v) < v_hi):
        return None, "window"
    return (u, v), "in"


def distance(cam: Camera, p):
    """(point_world - t_world_camera).norm(), the 3-term sum as c0 + (c1 + c2)"""
    x, y, z = stored(p)
    dx, dy, dz = x - cam.t_wc[0], y - cam.t_wc[1], z - cam.t_wc[2]
    return math.sqrt(dx * dx + (dy * dy + dz * dz))


def round_half_even_u8(x: float) -> int:
    """cv::saturate_cast<uchar>(double): cvRound (half to even) then clamp to [0, 255].  Python's round() of a float is exact
    and rounds halves to even."""
    return min(255, max(0, round(x)))


@dataclass
class Sample:
    color: tuple            # the three channels as getSubPixel<Vec3b> returns them (double of the uchar)
    taps: list              # per channel the four rounded products (a, b, c, d)
    raw_sums: tuple         # per channel a + b + c + d without saturation
    weights: tuple          # (w00, w10, w01, w11) as doubles
    rc: tuple               # (floor_row, floor_col)


def tap_rc(img_rows, img_cols, r, c):
    """the pixel a tap names; the +1 taps past the last row / column only ever carry weight 0 (checked by the caller)"""
    return min(r, img_rows - 1), min(c, img_cols - 1)


def sub_pixel(img, u: float, v: float) -> Sample:
    """getSubPixel<cv::Vec3b>(img, v, u, 0): four products rounded half to even and clamped, then three saturated sums"""
    rows, cols = img.shape[0], img.shape[1]
    fr, fc = math.floor(v), math.floor(u)
    frac_r, frac_c = v - fr, u - fc
    w00 = (1.0 - frac_r) * (1.0 - frac_c)
    w10 = frac_r * (1.0 - frac_c)
    w01 = (1.0 - frac_r) * frac_c
    w11 = frac_r * frac_c
    spots = [((fr, fc), w00), ((fr + 1, fc), w10), ((fr, fc + 1), w01), ((fr + 1, fc + 1), w11)]
    for (r, c), w in spots:
        assert r >= 0 and c >= 0
        if r >= rows or c >= cols:
            assert w == 0.0, (u, v, r, c, w)     # a tap outside the image carries weight 0 exactly
    color, taps, raw = [], [], []
    for ch in range(3):
        t = [round_half_even_u8(float(img[tap_rc(rows, cols, r, c) + (ch,)]) * w) for (r, c), w in spots]
        s = min(255, t[0] + t[1])
        s = min(255, s + t[2])
        s = min(255, s + t[3])
        color.append(float(s))
        taps.append(t)
        raw.append(sum(t))
    return Sample(tuple(color), taps, tuple(raw), (w00, w10, w01, w11), (fr, fc))


def exact_bilinear(img, u: float, v: float):
    """the bilinear value at the exact (u, v) in rational arithmetic, per channel"""
    U, V = Fraction(u), Fraction(v)
    fr, fc = math.floor(V), math.floor(U)
    ar, ac = V - fr, U - fc
    rows, cols = img.shape[0], img.shape[1]
    out = []
    for ch in range(3):
        acc = Fraction(0)
        for (r, c), w in (((fr, fc), (1 - ar) * (1 - ac)), ((fr + 1, fc), ar * (1 - ac)), ((fr, fc + 1), (1 - ar) * ac),
                          ((fr + 1, fc + 1), ar * ac)):
            if w:
                acc += int(img[r, c, ch]) * w
        out.append(acc)
    return out


def exact_tap_products(img, u: float, v: float):
    """per channel the four products pixel * weight with the weights as the doubles getSubPixel computes, in Fraction"""
    s = sub_pixel(img, u, v)
    fr, fc = s.rc
    rows, cols = img.shape[0], img.shape[1]
    spots = [(fr, fc), (fr + 1, fc), (fr, fc + 1), (fr + 1, fc + 1)]
    return [[int(img[tap_rc(rows, cols, r, c) + (ch,)]) * Fraction(w) for (r, c), w in zip(spots, s.weights)] for ch in range(3)]


def is_tie(x: Fraction) -> bool:
    """x == k + 1/2 for an integer k"""
    return (x - Fraction(1, 2)).denominator == 1


def short_of_int(x) -> int:
    """(short)(int)x as g++ compiles it on x86-64: cvttsd2si gives INT_MIN for NaN and out-of-range values (low 16 bits 0),
    then the low 16 bits.  The device's cvt.rzi.s32.f64 gives 0 for NaN but saturates a finite out-of-range value, so such a
    value would not be a pinned case: refuse it."""
    x = float(x)
    if math.isnan(x):
        return 0
    t = math.trunc(x)
    assert -2 ** 31 <= t < 2 ** 31, x
    return int(np.int32(t).astype(np.int16))


@dataclass
class PointState:
    """rgbPoint's colour state: rgb (BGR shorts), N_rgb, cov_rgb (floats), observe_distance, last_observe_time"""
    rgb: list = field(default_factory=lambda: [0, 0, 0])
    n_rgb: int = 0
    cov: list = field(default_factory=lambda: [F32(0.0)] * 3)
    obs_dist: float = 0.0
    last_obs: float = 0.0


def update_rgb(st: PointState, color, dist: float, obs_time: float) -> int:
    """rgbPoint::updateRgb with observe_sigma_ = (15, 15, 15).  float <-> double as written there: cov_rgb is a float, the
    products cov_rgb * cov_rgb are float products, everything else double.  Returns 1 when the fusion counts."""
    if st.obs_dist != 0 and dist > st.obs_dist * 1.2:
        return 0
    if st.n_rgb == 0:
        st.last_obs, st.obs_dist = obs_time, dist
        st.rgb = [int(np.int16(round(c))) for c in color]       # (short)round(x) of an integral double
        st.cov = [F32(SIGMA)] * 3
        st.n_rgb = 1
        return 0
    with np.errstate(all="ignore"):                             # 1 / 0, 0 * inf: IEEE results, as the reference computes them
        for i in range(3):
            cov = F32(np.float64(st.cov[i]) + np.float64(PROCESS_NOISE) * (np.float64(obs_time) - np.float64(st.last_obs)))
            old_sigma = np.float64(cov)
            c2 = np.float64(cov * cov)                          # float * float, widened
            cov = F32(np.sqrt(np.float64(1.0) / (np.float64(1.0) / c2 + np.float64(1.0) / (np.float64(SIGMA) * np.float64(SIGMA)))))
            n2 = np.float64(cov * cov)
            mix = np.float64(st.rgb[i]) / (old_sigma * old_sigma) + np.float64(color[i]) / (np.float64(SIGMA) * np.float64(SIGMA))
            st.rgb[i] = short_of_int(n2 * mix)
            st.cov[i] = cov
    if dist < st.obs_dist:
        st.obs_dist = dist
    st.last_obs = obs_time
    st.n_rgb += 1
    return 1


@dataclass
class Observation:
    """what one rendering did to one point"""
    why: str                 # "depth", "window" or "in"
    uv: tuple | None = None
    dist: float | None = None
    sample: Sample | None = None
    first: bool = False      # the point's first observation (N_rgb was 0)
    fused: int = 0           # counted by render_point_count


def render(states: list, points, cam: Camera, img, obs_time: float):
    """renderPointsInRecentVoxel over every point (each voxel of the recent list once): returns (render_point_count, the
    per-point observations).  `img` is exactly rows x cols x 3."""
    assert img.shape == (cam.rows, cam.cols, 3)
    count, obs = 0, []
    for st, p in zip(states, points):
        uv, why = project(cam, p)
        if uv is None:
            obs.append(Observation(why))
            continue
        d = distance(cam, p)
        s = sub_pixel(img, uv[0], uv[1])
        first = st.n_rgb == 0
        f = update_rgb(st, s.color, d, obs_time)
        count += f
        obs.append(Observation(why, uv, d, s, first and st.n_rgb == 1, f))
    return count, obs


def exact_cov_chain(obs_times, fused_flags, digits=80):
    """updateRgb's covariance recursion at `digits` digits with no intermediate float / double rounding: 15 at the first
    observation, then per fusion c <- sqrt(1 / (1 / (c + 0.1 * dt)^2 + 1 / 15^2)) with 0.1 the double constant and dt the
    exact difference of the double times.  Returns the value after each entry (None before the first observation)."""
    with mpmath.workdps(digits):
        c, last, out = None, None, []
        q = mpmath.mpf(PROCESS_NOISE)
        for t, f in zip(obs_times, fused_flags):
            if f == "first":
                c, last = mpmath.mpf(SIGMA), mpmath.mpf(t)
            elif f:
                s = c + q * (mpmath.mpf(t) - last)
                c = mpmath.sqrt(1 / (1 / (s * s) + 1 / mpmath.mpf(SIGMA) ** 2))
                last = mpmath.mpf(t)
            out.append(None if c is None else float(c))
        return out
