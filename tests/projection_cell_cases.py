"""Cases for the pixel cells of the map tracker's two cell users: selectPointsForProjection (srl_color_map_select_for_projection)
and updateAndAppendTrackPoints (srl_flow_tracker_update_and_append), at the shipped camera sizes and at the FoV window's edges.

Both reduce a projected coordinate x to the cell int(std::round(x / d) * d) and pack the two cells of a point into one sort key
laid out by srl::cell_axis: per axis an offset -b (b = ceil(2a) + 2, a the larger magnitude of the window's bounds) and `bits`
bits, the all-ones key meaning "no cell".  cell_axis() below restates that layout.

Cameras.  The image sizes are the shipped ones: ntu 752 x 480 and r3live 1280 x 1024 at scale factor 1, the same cameras after
an image resize (resized_size() restates ImageProcessing's output size and scale factor, which the GPU tests hold against the
library), and 2 x 2 and 2 x 1024 images.  The crafted points are seen through a *window camera*: identity rotation, fx = fy =
1, cx = cy = 0, translation (tu, tv, 0).  A point (x, y, z) with z a power of two then projects to u = (x + tu) / z exactly, so
one float point and a per-call translation put u on any chosen double: with the shipped principal points the sum + cx puts
coordinates near the low edge on a grid far coarser than their ulp, and the window test reads only cols, rows and the margin.
scene_points() adds points seen through the shipped intrinsics themselves.

Selection cases (selection_cases): per camera, FoV margin and cell size d, one map of
  * a grid over the window and a little past it (z = 2^-8);
  * anchors (z = 2^-9, so they are nearer than the grid and win their cells) at the four window edges of each axis;
  * exact halves of d, (k + 1/2) d, at both ends of the window, around 0 and at random in between, for every d whose halves
    are floats;
and the calls (tu, tv) that put an anchor exactly on lo = fov * size + 1, the double below it, the largest double H with
ceil(H) < (1 - fov) * size, and the double above H.  The cell sizes include, per axis and side, the d that puts the outermost
accepted coordinate just past d / 2, so its cell is +-d, about twice the coordinate: the one case where a key field gets near
the end of its range.

Tracker cases (tracker_cases): a `last` set, candidates and two updates (count 0, then count 1) per case, at 752, 1280 and the
resized widths:
  * thr-*: reprojection errors exactly thr = 2 cols / 320 and 2 thr and one double above each, as the reference computes
    them (the norm of (u_d - u, v_d - v) with v_d - v = 0);
  * edge-*: survivors on a window edge, candidates on the same cell, on the double past the edge and on neighbouring cells;
  * entries behind the camera right after edge and threshold entries, so the stale projection they are measured against is
    an edge one (never the first entry: the reference reads uninitialised doubles there);
  * fov 0.5, an empty window: nothing is appended and loop 1 still erases.
Points are rows of the case's `points`; a row is a point id for the compiled reference, and the GPU tests map rows to the
colour map's ids (voxels of TRACK_VOXEL, one per point, added in row order, so the order is the same).
"""
from __future__ import annotations

import math
from fractions import Fraction

import numpy as np

from map_reference import voxel_of

F32 = np.float32
GRID_Z = 2.0 ** -8             # above project3dTo2d's 0.001 and a power of two, so u = (x + tu) / z is exact
ANCHOR_Z = 2.0 ** -9
VOXEL = 2.0 ** -8              # the colour map the cases fill: a voxel per pixel of the grid, fine cells of a quarter pixel
FINE = 2.0 ** -10
TRACK_VOXEL = FINE             # the tracker cases' map: a voxel per point, so point ids follow the order points are added
CAP = 20
FOVS = (0.005, 0.0001, 0.0, -0.4, -10.0, 0.5, 0.5000000000000001, 0.75, 2.0)
BASE_D = (0.75, 1.5, 5.0, 10.0, 40.0 / 1.5, 40.0, 80.0, 1e-3)
HALVES_D = (0.75, 1.5, 5.0, 10.0, 40.0, 80.0)          # (k + 1/2) d is a float for these


def nxt(x: float) -> float:
    return float(np.nextafter(x, np.inf))


def prv(x: float) -> float:
    return float(np.nextafter(x, -np.inf))


# ---- cameras -------------------------------------------------------------------------------------------------------------
def resized_size(params: dict, in_cols: int):
    """imageProcessing's first-image step for inputs in_cols wide: scale factor s = image_width / in_cols, output size
    (int(image_width / s), int(image_height / s)), and the tracker's mini_distance 40 / s"""
    s = params["image_width"] * 1.0 / in_cols
    return int(params["image_width"] / s), int(params["image_height"] / s), s, 40.0 / s


def cameras():
    """(name, cols, rows, mini_distance, intrinsics (fx, fy, cx, cy) or None, (params, in_cols) for the resized ones)"""
    from sr_livo_b200 import lio
    out = []
    for name, p, in_cols in (("ntu", lio.ntu_camera_params(), 500), ("r3live", lio.r3live_camera_params(), 960)):
        k = p["camera_intrinsic"]
        out.append((name, p["image_width"], p["image_height"], 40.0, (k[0], k[4], k[2], k[5]), None))
        c, r, s, md = resized_size(p, in_cols)
        assert s != 1.0
        out.append((f"{name}-resized", c, r, md, (k[0] / s, k[4] / s, k[2] / s, k[5] / s), (p, in_cols)))
    out.append(("tiny-2x2", 2, 2, 40.0, None, None))
    out.append(("thin-2x1024", 2, 1024, 40.0, None, None))
    return out


def window_cam15(fov: float, tu: float = 0.0, tv: float = 0.0):
    """q_camera_world, t_camera_world, t_world_camera, fx, fy, cx, cy, fov_margin of the window camera"""
    return np.array([0.0, 0.0, 0.0, 1.0, tu, tv, 0.0, -tu, -tv, 0.0, 1.0, 1.0, 0.0, 0.0, fov], np.float64)


def shipped_cam15(fov: float, k):
    return np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, k[0], k[1], k[2], k[3], fov], np.float64)


# ---- the layout and the window -----------------------------------------------------------------------------------------
def cell_axis(fov: float, size: int, d: float):
    """srl::cell_axis: (offset, bits) of one axis, or None where it refuses"""
    if not math.isfinite(fov):
        return None
    lo, hi = fov * size + 1.0, (1.0 - fov) * size
    a = max(abs(lo), abs(hi))
    if not (a < 1e9) or not (a / d < 1e300):
        return None
    b = math.ceil(2.0 * a) + 2.0
    if not b <= 2147483647.0:
        return None
    span = 2 * int(b) + 2
    bits = 0
    while (1 << bits) < span:
        bits += 1
    return -int(b), bits


def std_round(x: float) -> float:
    """std::round: half away from zero"""
    if x < 0:
        return -std_round(-x)
    r = math.floor(x)
    return float(r + 1 if x - r >= 0.5 else r)


def cell(x: float, d: float) -> int:
    """int(std::round(x / d) * d)"""
    return int(std_round(x / d) * d)


def bounds(fov: float, size: int):
    """if2dPointsAvailable's two doubles for one axis: x >= lo and ceil(x) < hi"""
    return fov * size + 1.0, (1.0 - fov) * size


def accepted(x: float, fov: float, size: int) -> bool:
    lo, hi = bounds(fov, size)
    return x >= lo and math.ceil(x) < hi


def edges(fov: float, size: int):
    """(lo, the double below lo, H, the double above H): H is the largest double with ceil(H) < hi.  Certified with exact
    rationals; None when the window is empty"""
    lo, hi = bounds(fov, size)
    H = float(math.ceil(hi) - 1)
    if H < lo:
        return None
    flo, fhi = Fraction(lo), Fraction(hi)
    for x, want in ((lo, True), (prv(lo), False), (H, True), (nxt(H), False)):
        fx = Fraction(x)
        assert (fx >= flo and math.ceil(fx) < fhi) == want, (fov, size, x)
    return lo, prv(lo), H, nxt(H)


def bound_ds(fov: float, cols: int, rows: int):
    """per axis and side, the d with x / d just past 1/2 for the outermost accepted coordinate x: its cell is +-d"""
    out = []
    for size in (cols, rows):
        e = edges(fov, size)
        if e is None:
            continue
        for x in (e[0], e[2]):
            if x == 0.0:
                continue
            d = 2.0 * abs(x) * (1.0 - 2.0 ** -40)
            assert abs(x) / d > 0.5 and abs(cell(x, d)) == abs(int(d)) and abs(int(d)) >= 2 * abs(x) - 1
            out.append(d)
    return out


def cell_sizes(fov: float, cols: int, rows: int, mini_distance: float):
    """the d of every (camera, margin): the base list, the camera's own, one larger than the window, the bound ones"""
    lo_u, hi_u = bounds(fov, cols)
    lo_v, hi_v = bounds(fov, rows)
    big = 4.0 * max(abs(lo_u), abs(hi_u), abs(lo_v), abs(hi_v)) + 8.0
    out = list(BASE_D) + [mini_distance, big] + bound_ds(fov, cols, rows)
    return sorted(set(out))


def key_fields(u: float, v: float, d: float, lay_u, lay_v):
    """the two fields of a point's key and the key"""
    fu, fv = cell(u, d) - lay_u[0], cell(v, d) - lay_v[0]
    return fu, fv, (fu << lay_v[1]) | fv


# ---- the map of a selection case -------------------------------------------------------------------------------------------
def _dedupe(pts):
    """drop points whose fine cell (int16 keys of 2^-10) another point already claimed, or whose voxel holds CAP points"""
    seen, count, out = set(), {}, []
    for p in pts:
        p = tuple(float(F32(a)) for a in p)
        f, k = voxel_of(p, FINE), voxel_of(p, VOXEL)
        if f is None or k is None or f in seen or count.get(k, 0) >= CAP:
            continue
        seen.add(f)
        count[k] = count.get(k, 0) + 1
        out.append(p)
    return np.array(out, np.float64).reshape(-1, 3)


def _mid(fov, size):
    lo, hi = bounds(fov, size)
    return float(np.clip(math.floor((lo + hi) / 2.0), -16000, 16000))


def _axis_span(fov, size):
    lo, hi = bounds(fov, size)
    a, b = (lo, hi) if lo <= hi else (hi, lo)
    return max(a - 3.0, -16000.0), min(b + 3.0, 16000.0)


def anchors(fov, cols, rows):
    """the anchor points and, per target, (axis, target value, anchor index): u = (x + tu) / ANCHOR_Z"""
    mu, mv = _mid(fov, cols), _mid(fov, rows)
    pts, targets = [], []
    for axis, size, other in ((0, cols, mv), (1, rows, mu)):
        e = edges(fov, size)
        if e is None:
            continue
        for t_in, t_out in ((e[0], e[1]), (e[2], e[3])):
            xy = [0.0, 0.0]
            xy[axis] = float(F32(t_in * ANCHOR_Z))
            xy[1 - axis] = float(F32(other * ANCHOR_Z))
            p = (xy[0], xy[1], ANCHOR_Z)
            if p not in pts:                                       # lo and H coincide in a one-pixel window
                pts.append(p)
            for t in (t_in, t_out):
                targets.append((axis, t, pts.index(p)))
    return pts, targets


def halves(fov, size, d, rng, n_random=40):
    """coordinates (k + 1/2) d inside the window's span: the outermost ones, those around 0 and random ones"""
    lo, hi = _axis_span(fov, size)
    k0, k1 = math.ceil(lo / d - 0.5), math.floor(hi / d - 0.5)
    if k1 < k0:
        return []
    ks = set(range(k0, min(k0 + 4, k1 + 1))) | set(range(max(k1 - 3, k0), k1 + 1)) | {k for k in range(-4, 4) if k0 <= k <= k1}
    if k1 - k0 > 8:
        ks |= set(int(k) for k in rng.integers(k0, k1 + 1, n_random))
    out = []
    for k in sorted(ks):
        x = (k + 0.5) * d
        if float(F32(x * GRID_Z)) == x * GRID_Z and (x * GRID_Z) / GRID_Z / d == k + 0.5:
            out.append(x)
    return out


def selection_points(fov, cols, rows, d, seed=0):
    """(points, anchor targets): the map of one selection case (see the module docstring)"""
    rng = np.random.default_rng(seed)
    pts, targets = anchors(fov, cols, rows)
    (ul, uh), (vl, vh) = _axis_span(fov, cols), _axis_span(fov, rows)
    us, vs = np.linspace(ul, uh, 20), np.linspace(vl, vh, 20)
    grid = [(u * GRID_Z, v * GRID_Z, GRID_Z) for u in us for v in vs]
    if d in HALVES_D:
        mu, mv = _mid(fov, cols) + 0.5 * d, _mid(fov, rows) + 0.5 * d
        grid += [(x * GRID_Z, mv * GRID_Z, GRID_Z) for x in halves(fov, cols, d, rng)]
        grid += [(mu * GRID_Z, y * GRID_Z, GRID_Z) for y in halves(fov, rows, d, rng)]
        hu, hv = halves(fov, cols, d, rng, 6), halves(fov, rows, d, rng, 6)
        grid += [(x * GRID_Z, y * GRID_Z, GRID_Z) for x in hu[:4] + hu[-4:] for y in hv[:4] + hv[-4:]]
    out = _dedupe(pts + grid)
    # the anchors come first and survive the dedupe, so the target indices still name them
    assert np.array_equal(out[: len(pts)], np.array(pts, np.float32).astype(np.float64).reshape(-1, 3))
    return out, targets


def target_shift(points, target):
    """(tu, tv) that put the anchor of `target` exactly on its value"""
    axis, t, k = target
    s = t * ANCHOR_Z
    sh = s - points[k][axis]
    assert float(np.float64(points[k][axis]) + sh) == s and (points[k][axis] + sh) / ANCHOR_Z == t
    return (sh, 0.0) if axis == 0 else (0.0, sh)


def project_window(p, fov, cols, rows, tu, tv):
    """u, v and acceptance of a stored point under the window camera, as project_in_image computes them"""
    x, y, z = (float(F32(a)) for a in p)
    if z < 0.001:
        return None, None, False
    u, v = (x + tu) * 1.0 / z + 0.0, (y + tv) * 1.0 / z + 0.0
    return u, v, accepted(u, fov, cols) and accepted(v, fov, rows)


def selection_cases():
    """(name, fov, cols, rows, d, intrinsics or None): every (camera, margin, d)"""
    out = []
    for name, cols, rows, md, k, _ in cameras():
        for fov in FOVS:
            for d in cell_sizes(fov, cols, rows, md):
                out.append((f"{name}-fov{fov!r}-d{d!r}", fov, cols, rows, d, None))
    return out


def scene_points(cols, rows, k, seed=0, n=1500):
    """points in front of a camera with the shipped intrinsics k, projecting over the window and a little past it: (n, 3)"""
    rng = np.random.default_rng(seed)
    z = rng.uniform(2.0, 6.0, n)
    u = rng.uniform(-0.2 * cols, 1.2 * cols, n)
    v = rng.uniform(-0.2 * rows, 1.2 * rows, n)
    return np.stack([(u - k[2]) * z / k[0], (v - k[3]) * z / k[1], z], 1).astype(np.float32).astype(np.float64)


# ---- tracker cases -----------------------------------------------------------------------------------------------------------
def thr_of(cols: int) -> float:
    return 2.0 * cols / 320.0


def _exact_sum(a: float, b: float) -> bool:
    return Fraction(a) + Fraction(b) == Fraction(a + b)


def _cand_offsets(d):
    return (0.0, 0.5, -0.5, 0.25 * d, 0.5 * d, -0.5 * d, d, -d, 2.0 * d)


def tracker_cases():
    """dicts: name, cols, rows, fov, max_points, points (n, 3) float32 rows, init_rows, init_uv (float32), steps: list of
    (cam15, candidate rows, mini_distance), and for certification `errors`: row -> the error loop 1 must compute"""
    cams = [(c, r, md) for name, c, r, md, _, _ in cameras() if name in ("ntu", "r3live", "ntu-resized", "r3live-resized")]
    out = []
    for cols, rows, md in cams:
        thr = thr_of(cols)
        for fov in (0.005, -0.4):
            for tag, e in (("thr", thr), ("thr+", nxt(thr)), ("2thr", 2.0 * thr), ("2thr+", nxt(2.0 * thr))):
                out.append(_thr_case(f"{tag}-{cols}x{rows}-fov{fov}", cols, rows, fov, md, e))
            for axis in (0, 1):
                for side in (0, 1):
                    out.append(_edge_case(f"edge-{'uv'[axis]}{'lo' if side == 0 else 'hi'}-{cols}x{rows}-fov{fov}", cols, rows, fov, md,
                                          axis, side))
        out.append(_thr_case(f"empty-{cols}x{rows}-fov0.5", cols, rows, 0.5, md, nxt(thr)))
    return out


def _behind(k):
    return (float(F32(0.25 + 0.001 * k)), -0.25, -1.0)


def _thr_case(name, cols, rows, fov, md, e):
    """loop-1 errors exactly e: u_d = e + u with v_d = v, u_d put on its double by tu = e * 2^-8 (u_d = (x + tu) * 2^8 with
    x = u * 2^-8)"""
    tu = e * GRID_Z
    pts, init_rows, init_uv, errors = [], [], [], {}
    lo_v, hi_v = bounds(fov, rows)
    v0 = max(math.ceil(lo_v) + 3, 3)
    k = 0
    for j, u in enumerate((-3.5, -1.0, 0.0, 0.5, 1.0, 2.25, 3.0)):
        if not _exact_sum(u, e):
            continue
        v = float(v0 + 37 * j)
        pts.append((u * GRID_Z, v * GRID_Z, GRID_Z))
        init_rows.append(len(pts) - 1); init_uv.append((u, v)); errors[len(pts) - 1] = e
        if j % 2 == 0:                                            # a point behind the camera right after it: the same error
            pts.append(_behind(k)); k += 1
            init_rows.append(len(pts) - 1); init_uv.append((u, v)); errors[len(pts) - 1] = e
    # one far behind entry (erased at once) and candidates on the tracked points' cells and beside them
    pts.append(_behind(k)); init_rows.append(len(pts) - 1); init_uv.append((u - 100.0, v))
    cand = []
    for r in list(errors):
        x, y, z = pts[r]
        if z < 0:
            continue
        for off in _cand_offsets(md):
            pts.append((float(F32(x + off * GRID_Z)), y + 0.25 * GRID_Z, GRID_Z))
            cand.append(len(pts) - 1)
    cam = window_cam15(fov, tu, 0.0)
    steps = [(cam, cand, md), (cam, cand[::-1], md)]
    return dict(name=name, cols=cols, rows=rows, fov=fov, max_points=300, points=_as_points(pts), init_rows=init_rows,
                init_uv=np.array(init_uv, F32), steps=steps, errors=errors)


def _edge_case(name, cols, rows, fov, md, axis, side):
    """a survivor exactly on one window edge (lo or H of one axis), candidates on the same cell, on the double past the edge
    and around it; the second update uses the d that puts this edge's cell at +-d"""
    size = (cols, rows)[axis]
    e = edges(fov, size)
    t = e[0] if side == 0 else e[2]
    past = e[1] if side == 0 else e[3]
    other = _mid(fov, (rows, cols)[axis])
    shift = [0.0, 0.0]
    shift[axis] = t * GRID_Z
    pts, init_rows, init_uv = [], [], []

    def point(c, o, exact=False):
        """the point at coordinate c (near t; exactly c when `exact`) on `axis` and o on the other"""
        xy = [0.0, 0.0]
        xy[axis] = float(F32((c - t) * GRID_Z))
        xy[1 - axis] = float(F32(o * GRID_Z))
        assert not exact or (xy[axis] + shift[axis]) / GRID_Z == c, (name, c)
        return (xy[0], xy[1], GRID_Z)

    def uv(c, o):
        return (c, o) if axis == 0 else (o, c)

    # survivors: on the edge, then a point behind the camera (measured against the edge projection), and one a cell inside
    inward = 1.0 if side == 0 else -1.0
    for c, o, exact in ((t, other, True), (t + inward * (md + 1.0), other + 3.0, False)):
        pts.append(point(c, o, exact)); init_rows.append(len(pts) - 1); init_uv.append(uv(float(F32(c)), o))
        pts.append(_behind(len(pts))); init_rows.append(len(pts) - 1); init_uv.append(uv(float(F32(c)), o))
    cand = []
    # a quarter pixel apart on the other axis: two points closer than that in both coordinates would share a fine cell
    for j, (c, exact) in enumerate(((past, True), (t, True), (nxt(t) if side == 0 else prv(t), True), (t + inward * 0.5, False),
                                    (t + inward * 0.5 * md, False), (t + inward * md, False), (t + inward * 2.0 * md, False))):
        for o in (other + 0.25 * (j + 1), other + 2.0 + 0.25 * j, other + md + 0.25 * j):
            pts.append(point(c, o, exact)); cand.append(len(pts) - 1)
    cam = window_cam15(fov, *shift)
    bd = 2.0 * abs(t) * (1.0 - 2.0 ** -40) if t != 0.0 else md
    steps = [(cam, cand, md), (cam, cand[::-1], bd), (cam, cand, md)]
    return dict(name=name, cols=cols, rows=rows, fov=fov, max_points=300, points=_as_points(pts), init_rows=init_rows,
                init_uv=np.array(init_uv, F32), steps=steps, errors={})


def _as_points(pts):
    p = np.array(pts, np.float64).reshape(-1, 3)
    assert np.array_equal(p.astype(np.float32).astype(np.float64), p), "case points must be floats"
    return p.astype(np.float32)


__all__ = ["F32", "GRID_Z", "ANCHOR_Z", "VOXEL", "FINE", "TRACK_VOXEL", "CAP", "FOVS", "BASE_D", "HALVES_D", "resized_size", "cameras", "window_cam15",
           "shipped_cam15", "cell_axis", "cell", "std_round", "bounds", "accepted", "edges", "bound_ds", "cell_sizes", "key_fields",
           "selection_points", "target_shift", "project_window", "selection_cases", "scene_points", "thr_of", "tracker_cases"]
