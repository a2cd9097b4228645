"""A plain sequential restatement of the optical-flow tracker's bookkeeping (src/opticalFlowTracker.cpp): init / setTrackPoints
(:188-211), trackImage (:111-186, distance -20), removeOutlierUsingRansacPnp (:267-323) with given inliers and
updateAndAppendTrackPoints (:13-102), over Python dicts walked in sorted point-id order (the device's stand-in for the
reference's rgbPoint* order).

Every operation is one IEEE operation in the reference's order: Python floats are binary64, numpy float32 scalars binary32.
The Lucas-Kanade call is a function the caller passes (the device's own tracker, pinned bit for bit by row N6), so the
restatement decides when it runs and a device that runs it at another time tracks other images.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np

from render_reference import Camera, camera_point

F32 = np.float32


def std_round(x: float) -> float:
    """std::round: half away from zero"""
    if x < 0:
        return -std_round(-x)
    r = math.floor(x)
    return float(r + 1 if x - r >= 0.5 else r)


def cell(x: float, d: float) -> int:
    """(int)(std::round(x / d) * d)"""
    return int(std_round(x / d) * d)


def project_full(cam: Camera, p):
    """project3dTo2d then if2dPointsAvailable with the camera's own margin: (z_ok, res, u, v); u, v are None when z < 0.001"""
    pcx, pcy, pcz = camera_point(cam, p)
    if pcz < 0.001:
        return False, False, None, None
    u = pcx * cam.fx / pcz + cam.cx
    v = pcy * cam.fy / pcz + cam.cy
    f = cam.fov
    res = u >= f * cam.cols + 1 and math.ceil(u) < (1 - f) * cam.cols and v >= f * cam.rows + 1 and math.ceil(v) < (1 - f) * cam.rows
    return True, res, u, v


def in_margin(x: float, y: float, cols: int, rows: int) -> bool:
    """if2dPointsAvailable(x, y, 1.0, 0.05)"""
    m = 0.05
    return x >= m * cols + 1 and math.ceil(x) < (1 - m) * cols and y >= m * rows + 1 and math.ceil(y) < (1 - m) * rows


def velocity(cur: F32, last: F32, dt: float) -> float:
    """one component of (cur - last) / dt in cv::Point_<float> arithmetic, widened to double; 1e-3f when dt < 1e-5"""
    if dt < 1e-5:
        return float(F32(1e-3))
    with np.errstate(over="ignore"):
        return float(F32(float(F32(cur) - F32(last)) / dt))


@dataclass
class Match:
    id: int
    last_uv: tuple
    uv: tuple
    vel: tuple
    in_margin: bool


class FlowTrackerModel:
    """positions: point id -> stored (x, y, z) floats"""

    def __init__(self, positions: dict, maximum_tracked_points: int = 300):
        self.pos = positions
        self.max = maximum_tracked_points
        self.last: dict[int, tuple] = {}            # id -> (F32 u, F32 v)
        self.cur: dict[int, tuple] = {}             # id -> ((F32 u, F32 v), (vx, vy))
        self.matches: list[Match] = []
        self.count: dict[int, int] = {}             # rgbPoint::is_out_lier_count
        self.last_time = None
        self.lk_calls = 0
        self.leading_unprojected = 0                # entries that met the reference's uninitialised u_d, v_d

    def _last_uv(self):
        ids = sorted(self.last)
        return ids, np.array([self.last[i] for i in ids], np.float32).reshape(-1, 2)

    def init(self, image_time: float, ids, uv, lk):
        self.last = {}
        for i, p in zip(np.asarray(ids, np.uint32).tolist(), np.asarray(uv, np.float32).reshape(-1, 2)):
            self.last[int(i)] = (F32(p[0]), F32(p[1]))   # a later duplicate overwrites
        self.last_time = image_time
        lk(self._last_uv()[1])                           # the pyramid only on the first image
        self.lk_calls += 1

    def track_image(self, image_time: float, lk, cols: int, rows: int) -> bool:
        self.cur = {}
        self.matches = []
        dt = image_time - self.last_time
        if len(self.last) < 30:
            self.last_time = image_time
            return False
        ids, last_uv = self._last_uv()
        new_uv, status = lk(last_uv)
        self.lk_calls += 1
        for k, i in enumerate(ids):
            if not status[k]:
                continue
            a, b = (F32(new_uv[k, 0]), F32(new_uv[k, 1])), (F32(last_uv[k, 0]), F32(last_uv[k, 1]))
            vel = (velocity(a[0], b[0], dt), velocity(a[1], b[1], dt))
            self.matches.append(Match(i, b, a, vel, in_margin(float(a[0]), float(a[1]), cols, rows)))
        self.reject_matches(None)
        self.last_time = image_time
        return True

    def reject_matches(self, mask):
        if mask is not None:
            assert len(mask) == len(self.matches)
        self.cur = {m.id: (m.uv, m.vel) for k, m in enumerate(self.matches) if m.in_margin and (mask is None or mask[k])}

    def remove_outliers(self, inliers) -> bool:
        if len(self.cur) < 10:
            return False
        order = sorted(self.cur)
        idx = range(len(order)) if inliers is None else [int(k) for k in inliers]
        for k in idx:
            if not 0 <= k < len(order):
                raise IndexError(k)
        new = {order[k]: self.cur[order[k]] for k in idx}
        self.cur = dict(new)
        self.last = {i: uv for i, (uv, _) in new.items()}
        return True

    def update_and_append(self, cam: Camera, candidates, mini_distance: float):
        thr = 2.0 * cam.cols / 320.0
        occupied = set()
        ud = vd = None
        kept = {}
        for i in sorted(self.last):
            uv = self.last[i]
            z_ok, res, u, v = project_full(cam, self.pos[i])
            if z_ok:
                ud, vd = u, v
            if ud is None:
                err = math.nan                            # the reference reads uninitialised doubles here
                self.leading_unprojected += 1
            else:
                a, b = ud - float(uv[0]), vd - float(uv[1])
                err = math.sqrt(a * a + b * b)
            c = self.count.get(i, 0)
            if err > thr:
                c += 1
                if c > 1 or err > thr * 2:
                    self.count[i] = 0
                    continue
                self.count[i] = c
            else:
                self.count[i] = 0
            if res:
                occupied.add((cell(ud, mini_distance), cell(vd, mini_distance)))
            kept[i] = uv
        for i in np.asarray(candidates, np.uint32).tolist():
            if i in kept:
                continue
            _, res, u, v = project_full(cam, self.pos[i])
            if res:
                key = (cell(u, mini_distance), cell(v, mini_distance))
                if key not in occupied:
                    occupied.add(key)
                    kept[i] = (F32(u), F32(v))
            if len(kept) >= self.max:
                break
        self.last = kept

    # the sets as arrays in id order, for comparisons
    def last_arrays(self):
        ids = sorted(self.last)
        return np.array(ids, np.uint32), np.array([self.last[i] for i in ids], np.float32).reshape(-1, 2)

    def cur_arrays(self):
        ids = sorted(self.cur)
        return (np.array(ids, np.uint32), np.array([self.cur[i][0] for i in ids], np.float32).reshape(-1, 2),
                np.array([self.cur[i][1] for i in ids], np.float64).reshape(-1, 2))

    def match_arrays(self):
        return (np.array([m.id for m in self.matches], np.uint32), np.array([m.last_uv for m in self.matches], np.float32).reshape(-1, 2),
                np.array([m.uv for m in self.matches], np.float32).reshape(-1, 2))
