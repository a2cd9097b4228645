"""Scenes for rgbMapTracker::selectPointsForProjection (src/rgbMapTracker.cpp:45-152).

  * map_sweeps: the colour-map sweeps of color_map_cases (dense patches in front of the camera, clusters at +-400 m far past
    the 200 m depth bound, points far behind the camera), a second noisy pass over the first, and points placed at the depth
    bounds and just in front of the camera plane.
  * halves_points / HALVES_CAM: points whose u_f / minimum_dis and v_f / minimum_dis are exact halves, negative ones included,
    seen by a camera with fov_margin -0.4 (the window reaches 255 px left of and above the image).
  * ulp_pairs: pairs of points in one pixel cell whose depths sit within one float ulp: the second point's depth lies strictly
    between the first's double depth and its float rounding, so the sequential rule's float-against-double comparison decides.
  * select_params: the parameter sets every scene runs (minimum_dis 5, 10 and 40 / 1.5; skip_step 1 and 3; both candidate
    sources; fov_margin 0.0001 and -0.4; the shipped depth bounds and a few others).
"""
import numpy as np

from color_map_cases import FINE, SIZE, camera, patch, sweep

MIN_DIS = (5.0, 10.0, 40.0 / 1.5)
ROWS, COLS = 480, 640


def with_fov(cam15, fov):
    c = np.array(cam15, np.float64)
    c[14] = fov
    return c


def depth(p, t_wc=(0.0, 0.0, 0.0)):
    """(point_world - t_world_camera).norm() of stored floats: sqrt(dx^2 + (dy^2 + dz^2)) in FP64."""
    p = np.asarray(p, np.float32).astype(np.float64)
    d = p - np.asarray(t_wc, np.float64)
    return np.sqrt(d[..., 0] * d[..., 0] + (d[..., 1] * d[..., 1] + d[..., 2] * d[..., 2]))


def project(p, cam15):
    """u_f, v_f of an identity-rotation camera (the cameras of these scenes): (pc * f) / pcz + c, products rounded one by one."""
    p = np.asarray(p, np.float32).astype(np.float64)
    pc = p + np.asarray(cam15[4:7])
    return (pc[..., 0] * cam15[10]) / pc[..., 2] + cam15[12], (pc[..., 1] * cam15[11]) / pc[..., 2] + cam15[13]


def cell(x, minimum_dis):
    """int(std::round(x / minimum_dis) * minimum_dis): half away from zero, the product truncated."""
    q = np.asarray(x, np.float64) / minimum_dis
    r = np.where(q >= 0, np.floor(q + 0.5), -np.floor(-q + 0.5))
    # floor(q + 0.5) can round q + 0.5 up for q just below a half; std::round does not: correct those
    r = np.where((q >= 0) & (r - q > 0.5), r - 1, r)
    r = np.where((q < 0) & (q - r > 0.5), r + 1, r)
    return np.trunc(r * minimum_dis).astype(np.int64)


def bound_points():
    """points on the camera axis at the depth bounds 0.1 and 200 (exact floats: 0.125 and 200 with minimum_depth 0.125), just
    past them, and just in front of the camera plane (pcz < 0.001)."""
    return np.array([[0.0, 0.0, 200.0], [0.01, 0.01, 200.0], [0.0, 0.02, 200.0001], [0.0, 0.0, 0.125], [0.01, 0.0, 0.12],
                     [0.02, 0.0, 0.0005], [0.03, 0.01, 0.0009], [0.0, 0.03, -0.5], [0.3, 0.2, 199.99]], np.float64)


def map_sweeps(seed, n_dense=6000):
    """two sweeps of the colour-map scenes (the second a noisy copy of the first plus the bound points)."""
    rng = np.random.default_rng(seed)
    first = sweep(seed, n_dense=n_dense)
    second = np.concatenate([first[: first.shape[0] // 2] + rng.normal(0, 0.003, (first.shape[0] // 2, 3)), bound_points(),
                             patch(rng, 800, (1.5, -0.8, 9.0), half=0.6)])
    return [first, second[rng.permutation(second.shape[0])]]


# fx = fy = 256, cx = cy = 0, camera at the origin: u_f = 64 * x / (z / 4) is exact for x = u / 64 at z = 4
HALVES_CAM = np.concatenate([[0.0, 0.0, 0.0, 1.0], [0.0, 0.0, 0.0], [0.0, 0.0, 0.0], [256.0, 256.0, 0.0, 0.0, -0.4]])


def halves_points(minimum_dis):
    """a grid of points at z = 4 whose u_f and v_f are odd multiples of minimum_dis / 2 (u_f / minimum_dis = k + 1/2), from
    -247.5 px (left of the image) to 247.5 px."""
    h = minimum_dis / 2.0
    us = h * (2 * np.arange(-int(247.5 / minimum_dis) - 1, int(247.5 / minimum_dis) + 1) + 1)
    vs = us[:: max(1, us.size // 12)]
    g = np.array([[u / 64.0, v / 64.0, 4.0] for u in us for v in vs], np.float64)
    u_f, v_f = project(g, HALVES_CAM)
    assert np.array_equal(u_f, g[:, 0] * 64.0) and np.all(np.abs(np.mod(u_f / minimum_dis, 1.0) - 0.5) == 0.0)
    return g


def ulp_pairs(seed, n, minimum_dis=40.0 / 1.5, reverse=False):
    """n pairs (a, b) in the same `minimum_dis` cell of camera((0, 0, 0)), 0.12 m apart in x (different voxels and fine cells),
    with depth(b) strictly between depth(a) and float(depth(a)).  Found by walking b's float x and z by a few ulps around the
    point of a's depth.  The pairs sit on a grid 0.3 m apart, so no two pairs share a voxel.  a comes first in the returned
    order (b first with reverse)."""
    rng = np.random.default_rng(seed)
    cam = camera((0.0, 0.0, 0.0))
    out = []
    i = 0
    while len(out) < n and i < 40 * n:
        gx, gy = 0.25 + 0.3 * (len(out) % 3), -0.6 + 0.3 * (len(out) // 3)
        i += 1
        a = np.array([gx + rng.uniform(0, 0.05), gy + rng.uniform(0, 0.05), rng.uniform(3.5, 6.0)], np.float32)
        da = float(depth(a))
        fa = float(np.float32(da))
        if fa == da:
            continue
        lo, hi = min(da, fa), max(da, fa)
        bx, by = np.float32(a[0] + np.float32(0.12)), a[1]
        bz0 = np.float32(np.sqrt(da * da - float(bx) ** 2 - float(by) ** 2))
        found = None
        for dz in range(-3, 4):
            bz = np.float32(bz0)
            for _ in range(abs(dz)):
                bz = np.nextafter(bz, np.float32(np.inf if dz > 0 else -np.inf))
            xs = [bx]
            for s in (np.inf, -np.inf):
                x = bx
                for _ in range(300):
                    x = np.nextafter(x, np.float32(s))
                    xs.append(x)
            for x in xs:
                b = np.array([x, by, bz], np.float32)
                db = float(depth(b))
                if lo < db < hi:
                    found = b
                    break
            if found is not None:
                break
        if found is None:
            continue
        ua, va = project(a, cam)
        ub, vb = project(found, cam)
        if cell(ua, minimum_dis) != cell(ub, minimum_dis) or cell(va, minimum_dis) != cell(vb, minimum_dis):
            continue
        out.append((found, a) if reverse else (a, found))
    assert len(out) == n, len(out)
    return np.array(out, np.float64).reshape(-1, 3)


def select_params():
    """(name, camera fov_margin, kwargs of select) for every scene."""
    out = []
    for md in MIN_DIS:
        for skip in (1, 3):
            for use_all in (False, True):
                for fov in (0.0001, -0.4):
                    out.append((f"md{md:.3g}-skip{skip}-{'all' if use_all else 'recent'}-fov{fov}", fov,
                                dict(minimum_dis=md, skip_step=skip, use_all_points=use_all)))
    out.append(("bounds-0.125-200", 0.0001, dict(minimum_dis=5.0, minimum_depth=0.125, maximum_depth=200.0, use_all_points=True)))
    out.append(("bounds-0-199.995", -0.4, dict(minimum_dis=10.0, minimum_depth=0.0, maximum_depth=199.995, use_all_points=True)))
    out.append(("bounds-4.03-4.05", 0.0001, dict(minimum_dis=10.0, minimum_depth=4.03, maximum_depth=4.05)))
    return out


def sequential_winners(depths, cells):
    """selectPointsForProjection's per-cell rule walked in index order: a candidate takes its cell when the cell is empty or the
    float the cell stores is > its depth (float widened against the double); the cell then stores (float)depth.  Returns the
    winners' indices in ascending order."""
    holder, stored = {}, {}
    for j, (d, c) in enumerate(zip(depths, cells)):
        if c not in stored or float(stored[c]) > d:
            holder[c], stored[c] = j, np.float32(d)
    return sorted(holder.values())


def prefix_min_winners(depths, cells):
    """the characterisation: per cell, the last candidate whose depth is below the minimum of the float depths before it in
    the cell, or the first candidate.  Stable sort by cell, segmented exclusive min-scan, segmented last-flagged reduction."""
    depths = np.asarray(depths, np.float64)
    cells = np.asarray(cells, np.int64)
    if depths.size == 0:
        return []
    order = np.argsort(cells, kind="stable")
    c, d = cells[order], depths[order]
    f = d.astype(np.float32)
    start = np.r_[True, c[1:] != c[:-1]]
    seg = np.cumsum(start) - 1
    pre = np.empty(d.size, np.float32)
    for s in np.unique(seg):
        idx = np.nonzero(seg == s)[0]
        run = np.minimum.accumulate(f[idx])
        pre[idx] = np.r_[np.float32(np.inf), run[:-1]]
    flag = d < pre.astype(np.float64)
    win = []
    for s in np.unique(seg):
        idx = np.nonzero((seg == s) & flag)[0]
        win.append(order[idx[-1]])
    return sorted(int(w) for w in win)


__all__ = ["MIN_DIS", "ROWS", "COLS", "FINE", "SIZE", "camera", "with_fov", "depth", "project", "cell", "bound_points", "map_sweeps",
           "HALVES_CAM", "halves_points", "ulp_pairs", "select_params", "sequential_winners", "prefix_min_winners"]
