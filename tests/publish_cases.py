"""Scenes for the published maps: the registered cloud of addPointsToMap (addPointToPcl) and the coloured map of
pubColorPoints / saveColorPoints.

lio_stream: a stream like the reference's own start (the first frame fills the map, then insert -> insert) whose later sweeps
mix, shuffled together,
  * near-copies of stored points (minimum-distance rejections),
  * a grid of points inside a few stored voxels, more than the cap leaves room for (the voxel fills up mid-sweep),
  * groups of points in voxels the map does not have yet (the first point creates the voxel and is not published; the
    next ones find it and are),
all around a vehicle at a large |z|, so that intensity = 50 * (z - translation.z) exercises the float rounding.
"""
import numpy as np

from color_map_cases import camera, patch

MIN_DIST = 0.1
CAP = 20


def lio_stream(seed, voxel_size, z0=1234.5678):
    """[(points (n, 3) float64, translation_z)] for the first frame and two inserts."""
    rng = np.random.default_rng(seed)
    s = voxel_size
    first = rng.uniform([-6 * s, -6 * s, z0 - 1.5 * s], [6 * s, 6 * s, z0 + 1.5 * s], (2500, 3))
    out = [(first, z0 - 1.7)]
    for k in range(2):
        near = first[rng.choice(first.shape[0], 500, replace=False)] + rng.normal(0.0, 0.04 * s, (500, 3))
        # a 5 x 5 x 5 grid (spacing 0.18 s) in each of four stored voxels: 125 candidates for at most 20 slots.  Keys truncate
        # toward zero, so the grid keeps the sign of the stored point it is built around.
        g = (np.stack(np.meshgrid(*[np.arange(5)] * 3, indexing="ij"), -1).reshape(-1, 3) * 0.18 + 0.07) * s
        picks = first[rng.choice(first.shape[0], 4, replace=False)]
        key, sign = np.trunc(picks / s), np.where(picks < 0, -1.0, 1.0)
        full = np.concatenate([sg * (np.abs(kk) * s + g) for kk, sg in zip(key, sign)])
        # 40 new voxels beyond the first frame's box, 6 points each, 0.15 s apart along a diagonal
        centers = rng.uniform([8 * s, -8 * s, z0 - 2 * s], [14 * s, 8 * s, z0 + 2 * s], (40, 3)) + 20 * s * k
        fresh = np.concatenate([c + np.outer(np.arange(6) * 0.15 * s, [1.0, 0.5, 0.25]) * 0.5 for c in centers])
        pts = np.concatenate([near, full, fresh, rng.uniform(-6 * s, 6 * s, (300, 3)) + [0, 0, z0]])
        out.append((pts[rng.permutation(pts.shape[0])], z0 + 0.37 * (k + 1) + rng.uniform(-0.5, 0.5)))
    return out


def small_color_points(k):
    """k points in distinct 0.01 m cells and 0.1 m voxels in front of a camera at the origin."""
    return np.array([[0.05 + 0.2 * i, 0.03 - 0.1 * i, 4.03] for i in range(k)], np.float64).reshape(-1, 3)


def render_images(seed, n):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (480, 640, 3), dtype=np.uint8) for _ in range(n)]


__all__ = ["lio_stream", "small_color_points", "render_images", "camera", "patch", "MIN_DIST", "CAP"]
