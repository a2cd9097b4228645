"""Seeded scenes for the colour map at the counts and sizes of a long run: the view counter N_rgb past its short range, and
the export past its 2^22-position chunk.

Wrap scene (`wrap_cases`).  A few hundred points in four 0.1 m voxels and one nearer point, inserted once and rendered about
65,550 times by a fixed 64 x 48 camera, so every point is seen on nearly every render and its N_rgb runs through
1 .. 32767, -32768 .. -1, 0 and, on the next view, the re-initialising branch of updateRgb (count back to 1).  Two groups are
held back on purpose, so points sit at different counts at every checkpoint:
  * group "side" (one voxel) leaves the window on a few early renders: the camera is moved 0.2 m along y;
  * group "near" (one point at 0.56 m) is gated by distance (> 1.2 * observe_distance) on a few other early renders: the
    camera is moved 0.2 m back along z, which moves the far points by under 10 %.
`model_counts` restates the counter per group (the short wrap and the re-initialisation) and `checkpoints` lists the renders
after which some group has just reached one of COUNT_MARKS; one of them holds points on both sides of the wrap.

Lattice maps (`lattice_points`, `lattice_plan`).  Points on a lattice of pitch 0.025 m at 0.0125 + 0.025 i, off every voxel
and fine-cell face: 64 points per voxel (cap 100), each alone in its 0.01 m cell, so rgb_points_vec is the insertion order.
The lattice is 2048 points along x, 4 along z (one voxel thick) and as many rows along y as the size needs (< 327 m on every
axis, so no fine key wraps).  The points are inserted in sweeps; after the sweeps that hold the windows around the chunk
boundaries (publish order 2^22, 2^23; save order n - 1 - 2^22, n - 1 - 2^23) the map is rendered by a camera 100 m away that
sees every listed voxel, once for the inner windows and twice for the last one.  `lattice_counts` restates N_rgb per point.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

SIZE, FINE = 0.1, 0.01
CHUNK = 1 << 22
ROWS, COLS = 48, 64
FX = FY = 200.0
COUNT_MARKS = (1, 2, 3, 32766, 32767, -32768, -32767, -1, 0)
# export filters of the wrap scene: both ends of the short range, around 0 and the renderer's usual thresholds
WRAP_MIN_VIEWS = (-32768, -32767, -1, 0, 1, 2, 3, 32766, 32767, 32768)


def wrap16(k: int) -> int:
    return ((k + 0x8000) & 0xFFFF) - 0x8000


def camera15(position, rows=ROWS, cols=COLS):
    """identity rotation, camera at `position` looking along +z: the 15 doubles the oracle and the reference take"""
    pos = np.asarray(position, np.float64)
    return np.concatenate([[0.0, 0.0, 0.0, 1.0], -pos, pos, [FX, FY, cols / 2.0 + 0.25, rows / 2.0 - 0.25, 0.0001]])


# ---- the wrap scene ----------------------------------------------------------------------------------------------------
HOME = (0.2, 0.25, 0.0)          # the usual camera
SIDE_CAM = (0.2, 0.05, 0.0)      # "side" leaves the window, the rest stays in it
BACK_CAM = (0.2, 0.25, -0.2)     # "near" is gated by distance, the rest is not
SIDE_RENDERS = (5, 9, 10)        # 1-based render numbers at which the camera is at SIDE_CAM
BACK_RENDERS = (14, 15, 16, 17, 30)
VIEWS_TO_REACH = 65536 + 3       # views after which a point is back at 3


@dataclass
class WrapCase:
    name: str
    cap: int
    t0: float                    # obs_time of render k is t0 + DT * k
    points: np.ndarray           # (n, 3) float64 world points, one insertion call
    groups: dict                 # group name -> indices into points that the map stores (all of them here)
    renders: int = 0

    def camera_of(self, k: int):
        return camera15(SIDE_CAM if k in SIDE_RENDERS else BACK_CAM if k in BACK_RENDERS else HOME)

    def obs_time(self, k: int) -> float:
        return self.t0 + DT * k


DT = 0.1


def _cells(vkey, n, rng):
    """n points of voxel vkey (all keys > 0) in n distinct 0.01 m cells, 2 mm clear of every cell face"""
    per = 10
    cells = rng.permutation(per ** 3)[:n]
    out = []
    for c in cells.tolist():
        ijk = np.array([c // (per * per), (c // per) % per, c % per], np.float64)
        out.append(np.asarray(vkey) * SIZE + (ijk + 0.2 + 0.6 * rng.random(3)) * FINE)
    return np.array(out)


def _wrap_points(cap, seed):
    rng = np.random.default_rng(seed)
    main = [(1, 1, 20), (2, 1, 20), (3, 1, 20)]
    n_main = (min(cap, 60), 30, 24)
    pts = [_cells(k, n, rng) for k, n in zip(main, n_main)]
    side = _cells((1, 3, 20), 20, rng)
    near = np.array([[0.2051, 0.2543, 0.5562]])
    allp = np.concatenate(pts + [side, near])
    n_all = allp.shape[0]
    groups = dict(main=np.arange(0, n_all - 21), side=np.arange(n_all - 21, n_all - 1), near=np.array([n_all - 1]))
    return allp, groups


def wrap_cases() -> list[WrapCase]:
    out = []
    for cap, t0, name in ((50, 1.0, "cap50"), (100, 1.0, "cap100"), (100, 1.7e9, "cap100_epoch")):
        pts, groups = _wrap_points(cap, 7 + cap)
        c = WrapCase(name, cap, t0, pts, groups)
        c.renders = VIEWS_TO_REACH + len(SIDE_RENDERS) + len(BACK_RENDERS)
        out.append(c)
    return out


def seen(group: str, k: int) -> bool:
    """whether render k views the points of a group (the window and the distance gate)"""
    if group == "side":
        return k not in SIDE_RENDERS
    if group == "near":                  # out of the window at SIDE_CAM, gated at BACK_CAM
        return k not in BACK_RENDERS and k not in SIDE_RENDERS
    return True


def model_counts(case: WrapCase):
    """per render k (1-based): the count of each group after it, and how many of the scene's points render k counted
    (updateRgb returns 0 on the first view and on the re-initialising view at N_rgb == 0)"""
    n = {g: 0 for g in case.groups}
    counts, rendered = [], []
    for k in range(1, case.renders + 1):
        r = 0
        for g, idx in case.groups.items():
            if not seen(g, k):
                continue
            if n[g] == 0:
                n[g] = 1
            else:
                n[g] = wrap16(n[g] + 1)
                r += len(idx)
        counts.append(dict(n))
        rendered.append(r)
    return counts, rendered


def checkpoints(case: WrapCase) -> list[int]:
    """the renders after which some group has just been viewed and stands at one of COUNT_MARKS"""
    counts, _ = model_counts(case)
    out = []
    for k in range(1, case.renders + 1):
        now = counts[k - 1]
        if any(seen(g, k) and now[g] in COUNT_MARKS for g in case.groups):
            out.append(k)
    return out


def images(seed: int, n: int = 5) -> list[np.ndarray]:
    rng = np.random.default_rng(seed)
    return [np.ascontiguousarray(rng.integers(0, 256, (ROWS, COLS, 3), dtype=np.uint8)) for _ in range(n)]


# ---- the lattice maps --------------------------------------------------------------------------------------------------
LATTICE_NX, LATTICE_NZ = 2048, 4
PITCH = 0.025
LATTICE_SIZES = (CHUNK - 1, CHUNK, CHUNK + 1, 2 * CHUNK + 5)
WINDOW = 2000
# N_rgb filters of the lattice exports: everything (-1, 0), the rendered windows (1), the last window (2), nothing (3)
LATTICE_MIN_VIEWS = (-1, 0, 1, 2, 3)
LATTICE_CAMERA = (25.6, 12.8, -100.0)
LATTICE_COLS, LATTICE_ROWS = 640, 480


def lattice_index(j):
    j = np.asarray(j, np.int64)
    return j % LATTICE_NZ, (j // LATTICE_NZ) % LATTICE_NX, j // (LATTICE_NZ * LATTICE_NX)   # iz, ix, iy


def lattice_points(begin: int, end: int) -> np.ndarray:
    """points begin .. end - 1 of the lattice in insertion order, (n, 3) float64 (exact in float32)"""
    iz, ix, iy = lattice_index(np.arange(begin, end))
    return np.stack([0.0125 + PITCH * ix, 0.0125 + PITCH * iy, 0.0125 + PITCH * iz], axis=1).astype(np.float32).astype(np.float64)


def lattice_voxel(j):
    """a dense id of the voxel of point j: its (ix // 4, iy // 4); the lattice is one voxel thick"""
    _, ix, iy = lattice_index(j)
    return (iy // 4) * (LATTICE_NX // 4) + ix // 4


def lattice_plan(n: int):
    """[(begin, end, renders after it)] covering 0 .. n - 1: windows of +-WINDOW around the boundaries of the chunks in both
    orders, rendered once; the last window rendered twice; the stretches between them not rendered"""
    marks = {0}
    for b in (CHUNK, 2 * CHUNK):
        for j in (b, n - 1 - b):
            if 0 < j < n:
                marks.add(j)
    wins = []
    for j in sorted(marks):
        lo, hi = max(0, j - WINDOW), min(n, j + WINDOW)
        if wins and lo <= wins[-1][1]:
            wins[-1] = (wins[-1][0], max(wins[-1][1], hi))
        else:
            wins.append((lo, hi))
    if wins[-1][1] >= n - WINDOW:
        wins[-1] = (wins[-1][0], n)
    else:
        wins.append((n - WINDOW, n))
    plan, at = [], 0
    for i, (lo, hi) in enumerate(wins):
        if lo > at:
            plan.append((at, lo, 0))
        plan.append((lo, hi, 2 if i == len(wins) - 1 else 1))
        at = hi
    assert at == n and plan[0][0] == 0
    return plan


def lattice_counts(n: int) -> np.ndarray:
    """N_rgb of every point after the plan: the number of renders whose recent list holds the point's voxel and that come after
    the point's insertion (the camera sees every listed voxel and never moves, so no gate fires)"""
    vox = lattice_voxel(np.arange(n))
    counts = np.zeros(n, np.int16)
    for lo, hi, reps in lattice_plan(n):
        if reps:
            listed = np.zeros(int(vox.max()) + 1, bool)
            listed[np.unique(vox[lo:hi])] = True
            counts[:hi] += (listed[vox[:hi]] * reps).astype(np.int16)
    return counts


def export_positions(counts: np.ndarray, min_views: int, order: int) -> np.ndarray:
    """the rgb_points_vec indices an export hands out, in its order (save order: n - 1 down to 1)"""
    n = counts.shape[0]
    idx = np.arange(n) if order == 0 else np.arange(n - 1, 0, -1)
    return idx[counts[idx].astype(np.int32) >= min_views]


def chunk_flags(counts: np.ndarray, min_views: int, order: int) -> list[int]:
    """flagged positions per 2^22-position chunk of an export"""
    n = counts.shape[0]
    m = n if order == 0 else max(n - 1, 0)
    idx = np.arange(n) if order == 0 else np.arange(n - 1, 0, -1)
    f = counts[idx].astype(np.int32) >= min_views
    return [int(f[b:b + CHUNK].sum()) for b in range(0, m, CHUNK)]
