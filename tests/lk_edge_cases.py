"""Crafted cases of the pyramidal Lucas-Kanade tracker at the places where it makes a discrete or rounding-sensitive decision.

Each case is two images and one point set: the first image only builds its pyramid, the second tracks the points from it.
The families, each with a coverage check that reads the restatement's trace (tests/lk_track_reference.py) and asserts that
the family reaches its edge:
  saturation   0/255 stripes, blocks, step edges and binary noise against their inversion, a whole-pixel shift and a partial
               inversion: |Scharr| 4080, |diff| 8160 and madd pairs past 2^24, where the int -> float conversions round;
  thresholds   min_eig_threshold exactly at a point's minEig, one float above it and a double under half an ulp above it;
               faint specks whose D lands on both sides of FLT_EPSILON and whose minEig goes negative; epsilon exactly at
               an iteration's double ddot and one double below it; the max_count / epsilon clamps and criteria types; the
               oscillation rule mined for |dx + pdx| as close to 0.01 as the scenes get, on both sides;
  borders      at every level of 161x97 and 1281x1023 (levels of odd sizes, cols_l != cols >> l), the last float inside and
               the first float outside each of the four limits of the first check; points carried out during the iteration;
               patches wholly and partly in the zero-derivative border;
  non_finite   NaN payloads (quiet and signalling, either sign) in x, y or both, +-inf, +-2^31, +-2147483520, +-3e9, 1e30,
               -0.0 and subnormals;
  shapes       the level-count truncation exactly on its boundary (21x21, 3x31, 31x3), the smallest accepted images, win 3
               at 1280x1024 (level 8), windows 4..25 that move the SSE chunk boundaries, n = 1, 2, 3, 5 and 4097.

Images come from integer arithmetic only (as tests/lk_cases.py), so every machine builds the same bytes.
"""
from __future__ import annotations

import functools
from dataclasses import dataclass, field

import numpy as np

import lk_cases as K
import lk_track_reference as T

F = np.float32
SHIPPED = dict(win_size=(21, 21), max_level=3, criteria=(3, 10, 0.05), flags=8, min_eig_threshold=1e-4)


@dataclass
class Case:
    name: str
    frames: list            # [I, J]: I builds the first pyramid, J is tracked against it
    pts: np.ndarray         # (n, 2) float32
    kw: dict                # LKOpticalFlowKernel parameters
    expect: dict = field(default_factory=dict)   # what the family's coverage check needs


def kw_with(**over) -> dict:
    d = dict(SHIPPED)
    d.update(over)
    return d


def restate(case: Case, exact: bool = False):
    """(curr, status, ret, trace, restated kernel) of a case on the restatement."""
    r = T.LKRestated(**case.kw, exact=exact)
    r.track(case.frames[0], case.pts)
    curr, st, ret = r.track(case.frames[1], case.pts)
    return curr, st, ret, r.trace, r


def _texture(cols: int, rows: int, seed: int, passes: int = 2, gain: int = 3) -> np.ndarray:
    """A smooth noise world of (rows + 2 MARGIN, cols + 2 MARGIN) for K.sample."""
    rng = np.random.default_rng(seed)
    w = K._binomial(rng.integers(0, 256, (rows + 2 * K.MARGIN, cols + 2 * K.MARGIN)), passes)
    return np.clip((w - 128) * gain + 128, 0, 255)


def textured_pair(cols: int, rows: int, seed: int, dx256: int = 0, dy256: int = 0):
    w = _texture(cols, rows, seed)
    return K.sample(w, cols, rows), K.sample(w, cols, rows, dx256, dy256)


def _grid(cols, rows, step, off=0.0):
    y, x = np.mgrid[0:rows:step, 0:cols:step]
    return np.stack([x.ravel() + off, y.ravel() + off], 1).astype(np.float32)


# ---- saturation -------------------------------------------------------------------------------------------------------------

def _shift(img, dx, dy):
    """img moved by whole pixels (content at (x, y) goes to (x + dx, y + dy)), edges replicated."""
    p = np.pad(img, ((abs(dy), abs(dy)), (abs(dx), abs(dx))), mode="edge")
    r, c = img.shape
    return p[abs(dy) - dy:abs(dy) - dy + r, abs(dx) - dx:abs(dx) - dx + c]


@functools.lru_cache(maxsize=None)
def saturation() -> list[Case]:
    cols, rows = 160, 120
    y, x = np.mgrid[0:rows, 0:cols]
    rng = np.random.default_rng(101)
    stripes = np.where((x // 4) % 2 == 1, 255, 0).astype(np.uint8)                 # 4 px stripes, period 8
    hstripes = np.where((y // 2) % 2 == 1, 255, 0).astype(np.uint8)                # 2 px stripes
    checker = np.where(((x // 8) + (y // 8)) % 2 == 1, 255, 0).astype(np.uint8)
    step = np.where(x + 0 * y >= cols // 2, 255, 0).astype(np.uint8)
    bs = rng.integers(2, 7)
    binary = (np.kron(rng.integers(0, 2, (rows // 2 + 1, cols // 2 + 1)), np.ones((2, 2), np.int64))[:rows, :cols] * 255).astype(np.uint8)
    blocks = (np.kron(rng.integers(0, 2, (rows // bs + 1, cols // bs + 1)), np.ones((bs, bs), np.int64))[:rows, :cols] * 255).astype(np.uint8)
    partial = lambda im: np.where(x < cols // 2, 255 - im, im).astype(np.uint8)
    pts = np.concatenate([_grid(cols, rows, 5), _grid(cols, rows, 11, 0.5)])
    cases = []
    for name, I in (("stripes", stripes), ("hstripes", hstripes), ("checker", checker), ("step", step), ("binary", binary), ("blocks", blocks)):
        for jname, J in (("inverted", 255 - I), ("shift2", _shift(I, 2, -1)), ("partial", partial(I))):
            cases.append(Case(f"saturation_{name}_{jname}", [I, np.ascontiguousarray(J, np.uint8)], pts, kw_with()))
    return cases


# ---- thresholds -------------------------------------------------------------------------------------------------------------

THR_KW = kw_with(max_level=0, criteria=(3, 10, 0.05))


@functools.lru_cache(maxsize=None)
def _thr_scene():
    I, J = textured_pair(160, 120, 202, 77, -51)
    rng = np.random.default_rng(203)
    pts = (rng.integers(30 * 256, 130 * 256, (40, 2)) / 256.0).astype(np.float32)
    pts[:, 1] = np.minimum(pts[:, 1], F(95))
    return I, J, pts


def _mine_min_eig():
    """(points, [(target index, minEig)]): two interior points that converge, by their level-0 minEig."""
    I, J, pts = _thr_scene()
    _, st, _, tr, _ = restate(Case("", [I, J], pts, dict(THR_KW, min_eig_threshold=1e-4)))
    ok = np.flatnonzero((st == 1) & (tr[0]["exit"] != T.OUTSIDE_ITER) & (tr[0]["min_eig"] > 0))
    return pts, [(int(i), F(tr[0]["min_eig"][i])) for i in ok[:2]]


def min_eig_cases() -> list[Case]:
    I, J, pts = _thr_scene()
    _, targets = _mine_min_eig()
    cases = []
    for t, m in targets:
        up = np.nextafter(m, F(np.inf))
        half_ulp = float(m) + 0.4 * (float(up) - float(m))     # a double under half an ulp above m: rounds to m
        assert F(half_ulp) == m and half_ulp > float(m)
        for tag, thr, rejected in (("exact", float(m), False), ("next_float", float(up), True), ("under_half_ulp", half_ulp, False)):
            cases.append(Case(f"min_eig_{t}_{tag}", [I, J], pts, dict(THR_KW, min_eig_threshold=thr), dict(target=t, rejected=rejected)))
    return cases


@functools.lru_cache(maxsize=None)
def _faint_scene():
    """On the left, flat 128 with sparse specks raised 1-3 levels (D around FLT_EPSILON); on the right, a diagonal 2 | 250 step
    edge with sparse +1 specks: Ix = Iy on the edge, so A is rank one but for the specks, and minEig rounds to either sign."""
    cols, rows = 240, 120
    rng = np.random.default_rng(301)
    y, x = np.mgrid[0:rows, 0:cols]
    I = np.where(x < 120, 128, np.where((x - 120) + y >= 120, 250, 2)).astype(np.int64)
    sp = rng.random((rows, cols)) < np.where(x < 120, 0.01, 0.002)
    I[sp] += np.where(x[sp] < 120, rng.integers(1, 4, sp.sum()), 1)
    I = I.astype(np.uint8)
    J = _shift(I, 1, 0).astype(np.uint8)
    left = np.stack([rng.integers(25 * 256, 100 * 256, 3000), rng.integers(25 * 256, 95 * 256, 3000)], 1) / 256.0
    t = rng.integers(30 * 256, 90 * 256, 3000) / 256.0
    diag = np.stack([240 - t + rng.integers(-1024, 1024, 3000) / 256.0, t], 1)
    return I, J, np.concatenate([left, diag]).astype(np.float32)


@functools.lru_cache(maxsize=None)
def _mine_faint():
    """The faint scene's points whose D lies nearest FLT_EPSILON below and above it (refined by sub-pixel steps around the
    nearest of a first pass), and points with a negative minEig."""
    I, J, pts = _faint_scene()
    eps = float(T.FLT_EPSILON)

    def run(p):
        _, _, _, tr, _ = restate(Case("", [I, J], p, dict(THR_KW, min_eig_threshold=-1.0)))
        return tr[0]["D"].astype(np.float64), tr[0]["min_eig"]

    def nearest(D, k):
        below, above = np.flatnonzero(D < eps), np.flatnonzero(D >= eps)
        return below[np.argsort(eps - D[below])][:k], above[np.argsort(D[above] - eps)][:k]

    D, me = run(pts)
    seeds = pts[np.concatenate(nearest(D, 6))]
    steps = np.stack(np.meshgrid(np.arange(-16, 16) / 256.0, np.arange(-4, 4) / 256.0), -1).reshape(-1, 2)
    fine = (seeds[:, None, :] + steps[None]).reshape(-1, 2).astype(np.float32)
    Df, _ = run(fine)
    below, above = nearest(Df, 12)
    return np.concatenate([fine[below], fine[above], pts[np.flatnonzero(me < 0)[:12]]])


def faint_cases() -> list[Case]:
    I, J, _ = _faint_scene()
    sel = _mine_faint()
    return [Case(f"faint_thr{t}", [I, J], sel, dict(THR_KW, min_eig_threshold=t)) for t in (0.0, -1.0)]


EPS_KW = kw_with(max_level=0, criteria=(3, 30, 0.0))


@functools.lru_cache(maxsize=None)
def _mine_eps():
    """[(point index, iteration j, ddot_j)]: iterations whose ddot is below every earlier one of the point, which no other
    rule ended, so that epsilon = ddot_j stops the point exactly at j."""
    I, J, pts = _thr_scene()
    _, _, _, tr, _ = restate(Case("", [I, J], pts, EPS_KW))
    out = []
    for i in range(len(pts)):
        n = int(tr[0]["iters"][i])
        dd = tr[0]["ddot"][i, :n]
        for j in range(1, n - 1):
            if 0 < dd[j] < dd[:j].min():
                out.append((i, j, float(dd[j])))
                break
        if len(out) == 8:
            break
    return out


def eps_cases() -> list[Case]:
    I, J, pts = _thr_scene()
    cases = []
    for i, j, dd in _mine_eps():
        for tag, e, stops in (("exact", dd, True), ("next_down", float(np.nextafter(dd, 0.0)), False)):
            cases.append(Case(f"eps_{i}_{j}_{tag}", [I, J], pts, dict(EPS_KW, criteria=(3, 30, e)), dict(target=i, j=j, stops=stops)))
    return cases


# (type, max_count, epsilon) -> the (max_count, epsilon) setTerminationCriteria makes
CRITERIA = [((3, 0, 0.05), (0, 0.05)), ((3, 1, 0.05), (1, 0.05)), ((3, 100, 0.0), (100, 0.0)), ((3, -5, 0.05), (0, 0.05)),
            ((3, 101, 0.0), (100, 0.0)), ((3, 30, -1.0), (30, 0.0)), ((3, 30, 11.0), (30, 10.0)), ((0, 5, 0.5), (30, 0.01)),
            ((1, 5, 0.5), (5, 0.01)), ((2, 5, 0.5), (30, 0.5))]


def criteria_cases() -> list[Case]:
    I, J = textured_pair(160, 120, 401, 300, -200)
    pts = _grid(160, 120, 9, 0.25)
    return [Case(f"criteria_{c[0]}_{c[1]}_{c[2]}", [I, J], pts, kw_with(criteria=c), dict(term=t)) for c, t in CRITERIA]


OSC_KW = kw_with(max_level=1, criteria=(3, 100, 0.0))


@functools.lru_cache(maxsize=None)
def _osc_scene():
    I, J = textured_pair(320, 240, 501, 128, 128)          # half a pixel each way: the rule fires now and then
    rng = np.random.default_rng(502)
    pts = (rng.integers(24 * 256, 296 * 256, (3000, 2)) / 256.0).astype(np.float32)
    pts[:, 1] = np.clip(pts[:, 1], 24, 216)
    return I, J, pts


def osc_margins(tr_level: dict) -> np.ndarray:
    """Per point and iteration j >= 1: max(|dx_j + dx_{j-1}|, |dy_j + dy_{j-1}|) - 0.01 in double (the rule fires below 0),
    NaN where the iteration did not run or the epsilon rule ended it first."""
    dx, dy, dd = tr_level["dx"], tr_level["dy"], tr_level["ddot"]
    sx = np.abs(dx[:, 1:] + dx[:, :-1]).astype(np.float64)
    sy = np.abs(dy[:, 1:] + dy[:, :-1]).astype(np.float64)
    return np.maximum(sx, sy) - 0.01


@functools.lru_cache(maxsize=None)
def _mine_osc():
    I, J, pts = _osc_scene()
    _, _, _, tr, _ = restate(Case("", [I, J], pts, OSC_KW))
    m = osc_margins(tr[0])
    pos = np.where(np.isnan(m) | (m < 0), np.inf, m).min(1)       # closest miss of each point
    neg = np.where(np.isnan(m) | (m >= 0), np.inf, -m).min(1)     # closest hit
    a, b = np.argsort(pos)[:10], np.argsort(neg)[:10]
    return np.unique(np.concatenate([a[np.isfinite(pos[a])], b[np.isfinite(neg[b])]]))


def osc_cases() -> list[Case]:
    I, J, pts = _osc_scene()
    return [Case("oscillation", [I, J], pts[_mine_osc()], OSC_KW)]


def thresholds() -> list[Case]:
    return min_eig_cases() + faint_cases() + eps_cases() + criteria_cases() + osc_cases()


# ---- borders ----------------------------------------------------------------------------------------------------------------

def _first_check(p: np.float32, level: int, half: np.float32) -> int:
    """The restatement's first-check integer of one coordinate at a level: cvFloor(p * 2^-level - half)."""
    return int(T.cv_floor(T.fmul_x86(np.array([p], np.float32), F(1.0 / (1 << level))) - half)[0])


def limit_pair(lim: int, level: int, half: np.float32, low_side: bool) -> tuple[np.float32, np.float32]:
    """(the last float coordinate whose first-check integer is the limit lim, the adjacent float, whose integer is past it).
    low_side: the limit is -W (outside below it), else cols_l - 1 (outside above it)."""
    s = 1 << level
    edge = lim if low_side else lim + 1        # the first-check value exactly at the integer step
    p = F((edge + float(half)) * s)
    assert _first_check(p, level, half) == edge
    toward = F(-np.inf)                        # walk down one float at a time until the integer changes
    while True:
        q = np.nextafter(p, toward)
        if _first_check(q, level, half) != edge:
            return (p, q) if low_side else (q, p)
        p = q


@functools.lru_cache(maxsize=None)
def borders() -> list[Case]:
    cases = []
    for (cols, rows), seed in (((161, 97), 601), ((1281, 1023), 602)):
        kw = kw_with(criteria=(3, 10, 0.05))
        ml = T.level_count(cols, rows, kw["win_size"], kw["max_level"])
        W, H = kw["win_size"]
        hx, hy = F((W - 1) * 0.5), F((H - 1) * 0.5)
        pts, tags = [], []
        for level in range(ml + 1):
            lc, lr = cols, rows
            for _ in range(level):
                lc, lr = (lc + 1) // 2, (lr + 1) // 2
            cx, cy = F(cols * 0.5 + 0.25), F(rows * 0.5 + 0.25)
            for side, (lim, up, half, axis) in {"left": (-W, True, hx, 0), "right": (lc - 1, False, hx, 0),
                                                "top": (-H, True, hy, 1), "bottom": (lr - 1, False, hy, 1)}.items():
                pin, pout = limit_pair(lim, level, half, up)
                for p, inside in ((pin, True), (pout, False)):
                    pt = [cx, cy]
                    pt[axis] = p
                    pts.append(pt)
                    tags.append((level, side, axis, lim if inside else lim + (-1 if up else 1), inside))
                if up:   # ipx = -W with most of the weight on the image's first column: a patch that is not all border
                    for frac in (0.5, 0.875, 0.9921875):
                        pt = [cx, cy]
                        pt[axis] = F((lim + frac + float(half)) * (1 << level))
                        pts.append(pt)
                        tags.append((level, side, axis, lim, True))
        # carried out during the iteration: 1-2 px inside the level-0 limits, J moved 6 px toward each edge
        for d in (1.0, 1.5, 2.0):
            pts += [[F(-W + hx + d), F(rows * 0.5)], [F(cols - 1 + hx + 1 - d), F(rows * 0.5)],
                    [F(cols * 0.5), F(-H + hy + d)], [F(cols * 0.5), F(rows - 1 + hy + 1 - d)]]
        # patches wholly in the zero-derivative border (ipx = -W, a = 0 at level 0) and partly in it
        pts += [[F(-W + hx), F(rows * 0.5)], [F(cols * 0.5), F(-H + hy)], [F(-W + hx), F(-H + hy)], [F(-5), F(rows * 0.5)],
                [F(cols + 4), F(rows * 0.5)], [F(cols * 0.5), F(rows + 3.5)]]
        pts = np.array(pts, np.float32)
        w = _texture(cols, rows, seed)
        I = K.sample(w, cols, rows)
        for name, (dx, dy) in (("still", (40, -30)), ("left", (6 * 256, 0)), ("right", (-6 * 256, 0)), ("up", (0, 6 * 256)), ("down", (0, -6 * 256))):
            J = K.sample(w, cols, rows, dx, dy)
            cases.append(Case(f"borders_{cols}x{rows}_{name}", [I, J], pts, kw, dict(tags=tags)))
    return cases


# ---- non-finite and huge coordinates ----------------------------------------------------------------------------------------

NAN_BITS = [0x7FC00000, 0xFFC00000, 0x7FC00001, 0x7FD23456, 0xFFEABCDE, 0x7F800001, 0x7FA00000, 0xFF800123]   # quiet, then signalling
SPECIALS = [np.inf, -np.inf, 2.0 ** 31, -2.0 ** 31, 2147483520.0, -2147483520.0, 3e9, -3e9, 1e30, -0.0, 1e-45, 1e-40, -1e-40,
            1.1754942e-38]


@functools.lru_cache(maxsize=None)
def non_finite() -> list[Case]:
    vals = [np.array([b], np.uint32).view(np.float32)[0] for b in NAN_BITS] + [F(v) for v in SPECIALS]
    pts = []
    for v in vals:
        pts += [[v, F(60.5)], [F(80.25), v], [v, v]]
    pts += [[F(-0.0), F(-0.0)], [F(1e-40), F(60.0)], [F(80.0), F(-1e-40)]]
    pts = np.array(pts, np.float32)
    I, J = textured_pair(160, 120, 701, 90, 60)
    return [Case("non_finite", [I, J], pts, kw_with()), Case("non_finite_count0", [I, J], pts, kw_with(criteria=(3, 0, 0.05)))]


# ---- shapes -----------------------------------------------------------------------------------------------------------------

def _shape_case(name, cols, rows, win, max_level, n, seed, expect_levels=None):
    I, J = textured_pair(cols, rows, seed, 70, -45)
    rng = np.random.default_rng(seed + 1)
    pts = np.stack([rng.integers(-256, (cols + 1) * 256, n), rng.integers(-256, (rows + 1) * 256, n)], 1) / 256.0
    return Case(name, [I, J], pts.astype(np.float32), kw_with(win_size=win, max_level=max_level), dict(levels=expect_levels))


@functools.lru_cache(maxsize=None)
def shapes() -> list[Case]:
    c = []
    # the truncation (w + 1) / 2 <= win exactly on its boundary
    for cols, rows, lv in ((42, 120, 0), (43, 120, 1), (120, 42, 0), (120, 43, 1), (84, 200, 1), (85, 200, 2)):
        c.append(_shape_case(f"trunc21_{cols}x{rows}", cols, rows, (21, 21), 3, 64, 800 + cols + rows, lv))
    for cols, rows, lv in ((6, 200, 0), (7, 200, 1), (200, 62, 0), (200, 63, 1)):
        c.append(_shape_case(f"trunc3x31_{cols}x{rows}", cols, rows, (3, 31), 3, 64, 810 + cols + rows, lv))
        c.append(_shape_case(f"trunc31x3_{rows}x{cols}", rows, cols, (31, 3), 3, 64, 820 + cols + rows, lv))
    # the smallest accepted images
    for win in ((21, 21), (3, 31), (31, 3), (3, 3)):
        c.append(_shape_case(f"smallest_{win[0]}x{win[1]}", win[0] + 1, win[1] + 1, win, 3, 16, 830 + win[0], 0))
    c.append(_shape_case("win3_level8", 1280, 1024, (3, 3), 8, 300, 840, 8))
    for w in (4, 7, 9, 15, 17, 23, 24, 25):
        c.append(_shape_case(f"win{w}", 200, 150, (w, w), 3, 200, 850 + w))
    c.append(_shape_case("win3x31", 200, 150, (3, 31), 3, 200, 880))
    c.append(_shape_case("win31x3", 200, 150, (31, 3), 3, 200, 881))
    for n in (1, 2, 3, 5, 4097):
        c.append(_shape_case(f"n{n}", 160, 120, (21, 21), 3, n, 890 + n))
    return c


FAMILIES = {"saturation": saturation, "thresholds": thresholds, "borders": borders, "non_finite": non_finite, "shapes": shapes}


def all_cases() -> list[Case]:
    return [c for f in FAMILIES.values() for c in f()]
