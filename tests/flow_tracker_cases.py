"""Scenes and sequences for the optical-flow tracker's bookkeeping (row N9).

  * CAM15 / camera(): an identity-rotation 640 x 480 camera (fx = fy = 400, cx = 320, cy = 240), so a point (x, y, 2) with x
    and y multiples of 1/64 projects to exact pixel coordinates: crafted errors and cells land exactly on their thresholds.
  * scene_points(): points in front of the camera (depth 3 to 12 m), points behind it (camera z < 0.001), and a grid of
    exact points at depth 2; each in its own voxel and fine cell, so the colour map stores every one.
  * SEQUENCE: per image, the time step, the fundamental-matrix mask, the PnP inliers and the camera's drift.
"""
from __future__ import annotations

import numpy as np

from render_reference import Camera

COLS, ROWS = 640, 480
FX = FY = 400.0
CX, CY = 320.0, 240.0


def cam15(t_cw=(0.0, 0.0, 0.0), fov=0.005, q_cw=(0.0, 0.0, 0.0, 1.0)):
    """q_camera_world (x, y, z, w), t_camera_world, t_world_camera, fx, fy, cx, cy, fov_margin"""
    t = np.asarray(t_cw, np.float64)
    return np.r_[np.asarray(q_cw, np.float64), t, -t, FX, FY, CX, CY, fov]


def model_camera(c15):
    return Camera(c15, ROWS, COLS)


def device_camera(capi, c15):
    c = [float(a) for a in c15]
    import ctypes as C
    return capi.Camera((C.c_double * 4)(*c[0:4]), (C.c_double * 3)(*c[4:7]), (C.c_double * 3)(*c[7:10]), c[10], c[11], c[12], c[13], c[14],
                       COLS, ROWS)


def scene_points(seed: int = 900, n_front: int = 2500, n_behind: int = 40):
    """(front, behind, exact): float64 (n, 3) arrays of points whose float32 values are what the map stores"""
    rng = np.random.default_rng(seed)
    z = rng.uniform(3.0, 12.0, n_front)
    u = rng.uniform(-0.5 * COLS, 1.5 * COLS, n_front)
    v = rng.uniform(-0.5 * ROWS, 1.5 * ROWS, n_front)
    front = np.stack([(u - CX) * z / FX, (v - CY) * z / FY, z], 1)
    behind = np.stack([rng.uniform(-3, 3, n_behind), rng.uniform(-3, 3, n_behind), rng.uniform(-6.0, -0.5, n_behind)], 1)
    gx, gy = np.meshgrid(np.arange(-6, 7) * 4.0, np.arange(-4, 5) * 4.0)
    # (x, y, 2) with x, y on a 1/16 grid: u = x * 400 / 2 + 320 exactly
    exact = np.stack([gx.ravel() / 16.0 + 1.0 / 64.0, gy.ravel() / 16.0, np.full(gx.size, 2.0)], 1)
    return (front.astype(np.float32).astype(np.float64), behind.astype(np.float32).astype(np.float64),
            exact.astype(np.float32).astype(np.float64))


# per image: (dt, mask kind, inlier kind, camera drift in metres along x)
SEQUENCE = [
    (0.1, None, None, 0.0),
    (0.1, "ones", "all_list", 0.002),
    (0.1, "alternate", "unsorted_dups", 0.004),
    (0.0, None, "skip", 0.004),
    (9.99e-6, "zeros", None, 0.006),
    (1e-5, None, "half", 0.01),
    (-0.05, "alternate", None, 0.03),
    (0.1, None, "zero", 0.03),
    (0.1, "ones", None, 0.05),
    (0.1, None, "unsorted_dups", 0.05),
    (0.1, None, None, 0.12),
    (0.1, "alternate", "half", 0.12),
]


def mask_for(kind, n: int, rng):
    if kind is None:
        return None
    if kind == "ones":
        return np.ones(n, np.uint8)
    if kind == "zeros":
        return np.zeros(n, np.uint8)
    return (np.arange(n) % 2).astype(np.uint8)


def inliers_for(kind, n: int, rng):
    """None = all of cur; 'skip' = the caller's RANSAC failed: no call"""
    if kind in (None, "skip"):
        return kind
    if kind == "all_list":
        return np.arange(n, dtype=np.int32)
    if kind == "zero":
        return np.zeros(0, np.int32)
    if kind == "half":
        return np.sort(rng.choice(n, max(n // 2, 1), replace=False)).astype(np.int32)
    k = rng.choice(n, max(n // 2, 1), replace=True)                     # unsorted, with repeats
    return rng.permutation(np.r_[k, k[: len(k) // 3]]).astype(np.int32)


# ---- CPU sequences for the pin of the restatement against the reference's own compiled tracker (test_flow_tracker_pin.py) and
# tests/golden/flow_tracker.npz.  Point ids are rows of pin_points(): the exact grid first, then random points in front with
# points behind the camera among them.  A behind point is never the first entry of `last` here: the reference reads
# uninitialised doubles for such a leading entry (DESIGN.md section 5), which test_flow_tracker_device.py pins against the
# restatement only.
def pin_points(seed: int = 1900):
    front, behind, exact = scene_points(seed, n_front=900, n_behind=30)
    return np.r_[exact, front[:450], behind, front[450:]].astype(np.float32)


def pin_lk(step: int):
    """a Lucas-Kanade stand-in, a pure function of its input: points move by a per-image float shift, every 7th (by position)
    loses its status, every 11th jumps 300 px (out of the 0.05 margin)"""
    dx, dy = np.float32(0.375 * ((step % 5) - 2)), np.float32(0.25 * ((step % 3) - 1))

    def lk(pts):
        pts = np.asarray(pts, np.float32).reshape(-1, 2)
        new = (pts + np.array([dx, dy], np.float32)).astype(np.float32)
        new[10::11, 0] += np.float32(300.0)
        status = np.ones(len(pts), np.uint8)
        status[(step % 7)::7] = 0
        return new, status
    return lk


PIN_MAX_POINTS = (300, 120)     # 120: the set reaches maximum_tracked_points, and max + 1 through the first non-member

# per image: (dt, mask kind, inlier kind, camera drift along x, candidate order); inlier kind "throw": the caller's RANSAC threw
PIN_SEQUENCE = [
    (0.1, None, None, 0.0, "order"),
    (0.1, "alternate", "unsorted_dups", 0.003, "reverse"),
    (0.0, "ones", "throw", 0.006, "order"),
    (9.99e-6, None, "half", 0.01, "dups"),
    (1e-5, "zeros", None, 0.02, "order"),
    (-0.05, None, "skip", 0.02, "reverse"),
    (0.1, "alternate", "zero", 0.04, "order"),
    (0.1, None, None, 0.08, "dups"),
    (0.1, None, "half", 0.15, "order"),
]


def pin_candidates(kind, n_points, rng):
    ids = np.arange(n_points, dtype=np.uint32)
    if kind == "reverse":
        return ids[::-1].copy()
    if kind == "dups":
        return np.r_[ids, rng.choice(ids, n_points // 4)].astype(np.uint32)
    return rng.permutation(ids).astype(np.uint32)


def run_pin(tracker, model_like: bool, max_points: int = 300, seed: int = 3):
    """the PIN_SEQUENCE on `tracker` (a FlowTrackerModel or a FlowTrackerReference); returns the trace: after every call, last,
    cur and every point's is_out_lier_count, and the number of Lucas-Kanade calls"""
    xyz = pin_points()
    ids_all = np.arange(len(xyz), dtype=np.uint32)
    rng = np.random.default_rng(seed)
    trace = []
    calls0 = [tracker.lk_calls if model_like else type(tracker).lk_calls()]

    def snap(tag):
        last = tracker.last_arrays()
        cur = tracker.cur_arrays()
        counts = (np.array([tracker.count.get(int(i), 0) for i in ids_all], np.int16) if model_like else tracker.counts(ids_all))
        calls = (tracker.lk_calls if model_like else type(tracker).lk_calls()) - calls0[0]
        trace.append((tag, last[0], last[1], cur[0], cur[1], cur[2], counts, np.int64(calls)))

    cam0 = model_camera(cam15())
    init_ids = np.flatnonzero(xyz[:, 2] > 0)[:max_points].astype(np.uint32)
    init_uv = []
    from flow_tracker_reference import project_full
    for i in init_ids:
        _, _, u, v = project_full(cam0, xyz[i])
        init_uv.append((u + 0.5 * (i % 5), v))
    behind = np.flatnonzero(xyz[:, 2] < 0)[:6].astype(np.uint32)
    init_ids = np.r_[behind, init_ids, init_ids[:7]]                                           # interior points behind, repeats
    init_uv = np.r_[np.full((len(behind), 2), 50.0), np.array(init_uv), np.array(init_uv[:7]) + 1.0].astype(np.float32)
    time = 5.0
    tracker.init(time, init_ids, init_uv, lambda p: None)
    snap("init")
    for k, (dt, mk, ik, drift, ck) in enumerate(PIN_SEQUENCE):
        time += dt
        lk = pin_lk(k)
        mask_fn = None if mk is None else (lambda n, mk=mk: mask_for(mk, n, None))
        if model_like:
            tracker.track_image(time, lk, COLS, ROWS)
            if mask_fn is not None:
                tracker.reject_matches(mask_fn(len(tracker.matches)))
        else:
            tracker.track_image(time, lk, COLS, ROWS, mask_fn)
        snap(f"track{k}")
        n_cur = len(tracker.cur_arrays()[0])
        inl = inliers_for(ik if ik != "throw" else "skip", n_cur, rng)
        if ik == "throw" and not model_like:
            tracker.remove_outliers(np.arange(n_cur), throws=True)
        elif not (isinstance(inl, str) and inl == "skip"):
            tracker.remove_outliers(inl)
        snap(f"pnp{k}")
        c15 = cam15((drift, 0.0, 0.0))
        cand = pin_candidates(ck, len(xyz), rng)
        if model_like:
            tracker.update_and_append(model_camera(c15), cand, 40.0 / (1 + k % 2))
        else:
            tracker.update_and_append(c15, COLS, ROWS, cand, 40.0 / (1 + k % 2))
        snap(f"append{k}")
    return trace
