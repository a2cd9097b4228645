"""A plain numpy restatement of the reference's pyramidal Lucas-Kanade (LKOpticalFlowKernel::trackImage, src/lkpyramid.cpp):
opencvBuildOpticalFlowPyramid (:510-625), calcSharrDeriv (:57-154) and calculateLKOpticalFlow (:174-496, err == nullptr),
with a per-point, per-level trace of every decision it makes.

How it stays the reference's arithmetic:
  - the integer work (pyrDown, Scharr, the 14-bit bilinear weights, the window patch, the temporal differences, the madd
    pairs) is exact int64; the SSE2 path and the scalar tail compute the same integers;
  - every float32 operation is a numpy float32 operation, elementwise over the points (the same IEEE single rounding as one
    float32 scalar at a time), in the reference's order, and no Python double enters a float32 expression: the constants are
    np.float32, and the two double compares (ddot <= epsilon, |dx + pdx| < 0.01) run on float64 arrays;
  - each SSE lane of a sum is a strictly sequential float32 chain, np.cumsum(..., dtype=np.float32) along the chain (an
    accumulate, never pairwise: np.sum must not be used), then the lanes fold as the reference folds them;
  - cvRound is round-half-to-even (np.rint); cvFloor is (int)v - (i > v), with (int)v = INT_MIN outside the int range and for
    NaN (cvttss2si), in 32-bit wrap-around;
  - a NaN coordinate is carried as x86 carries it: the product of a NaN and a finite float is that NaN with its quiet bit set.

The trace (LKRestated.trace, one dict per level) holds, per point: ipx/ipy, A11/A12/A22, D, minEig, every iteration's delta and
ddot, the exit (EXITS), and the largest |Scharr| (interpolated derivative), |diff| and |madd pair| the point touched.  With
exact=True it also holds the unrounded int64 sums of the A and b chains and the sums of their |terms|.
"""
from __future__ import annotations

import numpy as np

F = np.float32
INT_MIN = -(1 << 31)
FLT_EPSILON = F(np.finfo(np.float32).eps)
FLT_SCALE = F(1.0 / (1 << 20))
W_BITS = 14
EXITS = ("outside", "min_eig", "D", "eps", "oscillation", "count", "outside_iter")
OUTSIDE, MIN_EIG, DET, EPS, OSC, COUNT, OUTSIDE_ITER = range(7)
CHUNK = 2048                      # points per vectorised block


def pyr_down(src: np.ndarray) -> np.ndarray:
    """[1 4 6 4 1]^2 / 256 at (2x, 2y), REFLECT_101, (s + 128) >> 8."""
    h, w = src.shape
    p = np.pad(src.astype(np.int64), 2, mode="reflect")
    k = np.array([1, 4, 6, 4, 1], np.int64)
    rows = sum(k[i] * p[i:i + h, :] for i in range(5))
    full = sum(k[j] * rows[:, j:j + w] for j in range(5))
    return ((full[::2, ::2] + 128) >> 8).astype(np.uint8)


def scharr(img: np.ndarray) -> np.ndarray:
    """calcSharrDeriv with REFLECT_101 rows and columns: (Ix, Iy) int16."""
    p = np.pad(img.astype(np.int64), 1, mode="reflect")
    c = lambda dy, dx: p[1 + dy:p.shape[0] - 1 + dy, 1 + dx:p.shape[1] - 1 + dx]
    ix = 3 * (c(-1, 1) + c(1, 1)) + 10 * c(0, 1) - 3 * (c(-1, -1) + c(1, -1)) - 10 * c(0, -1)
    iy = 3 * (c(1, -1) + c(1, 1)) + 10 * c(1, 0) - 3 * (c(-1, -1) + c(-1, 1)) - 10 * c(-1, 0)
    return np.stack([ix, iy], -1).astype(np.int16)


def level_count(cols: int, rows: int, win: tuple[int, int], max_level: int) -> int:
    """The max_level opencvBuildOpticalFlowPyramid returns (:609-619)."""
    w, h = cols, rows
    for level in range(max_level + 1):
        w, h = (w + 1) // 2, (h + 1) // 2
        if w <= win[0] or h <= win[1]:
            return level
    return max_level


def pyramid(img: np.ndarray, win: tuple[int, int], max_level: int) -> list[tuple[np.ndarray, np.ndarray]]:
    """(padded level uint8 with a REFLECT_101 border of the window, padded (Ix, Iy) int16 with a zero border) per level."""
    ww, wh = win
    out, lvl = [], np.ascontiguousarray(img, np.uint8)
    for level in range(max_level + 1):
        if level:
            lvl = pyr_down(lvl)
        out.append((np.pad(lvl, ((wh, wh), (ww, ww)), mode="reflect"), np.pad(scharr(lvl), ((wh, wh), (ww, ww), (0, 0)))))
    return out


def cv_floor(v: np.ndarray) -> np.ndarray:
    """cvFloor on float32: (int)v - (i > v), (int)v = INT_MIN outside [-2^31, 2^31) and for NaN, 32-bit wrap-around."""
    v = np.asarray(v, np.float32)
    inside = (v >= F(-2147483648.0)) & (v < F(2147483648.0))
    i = np.where(inside, np.where(inside, v, F(0)).astype(np.int64), INT_MIN)
    r = i - (i.astype(np.float32) > v)
    return ((r - INT_MIN) & 0xFFFFFFFF) + INT_MIN


def cv_round(v: np.ndarray) -> np.ndarray:
    return np.rint(np.asarray(v, np.float32)).astype(np.int64)


def quiet(v: np.ndarray) -> np.ndarray:
    """A float32 NaN with its quiet bit set (x86's result of an operation on that NaN)."""
    return (np.asarray(v, np.float32).view(np.uint32) | np.uint32(0x00400000)).view(np.float32)


def fmul_x86(a: np.ndarray, s) -> np.ndarray:
    """a * s in float32 with a NaN `a` carried as x86 carries it (the NaN, quietened); s is a finite float32."""
    a = np.asarray(a, np.float32)
    return np.where(np.isnan(a), quiet(a), a * F(s))


def termination(criteria) -> tuple[int, float]:
    """setTerminationCriteria (:670-682): (max_count, epsilon)."""
    t, c, e = criteria
    max_count = 30 if (t & 1) == 0 else min(max(int(c), 0), 100)
    epsilon = 0.01 if (t & 2) == 0 else min(max(float(e), 0.0), 10.0)
    return max_count, epsilon


def weights(a: np.ndarray, b: np.ndarray):
    """The 14-bit bilinear weights: cvRound(((1 - a)(1 - b)) * 16384) and so on, iw11 the remainder."""
    one, s = F(1), F(1 << W_BITS)
    w00 = cv_round((one - a) * (one - b) * s)
    w01 = cv_round(a * (one - b) * s)
    w10 = cv_round((one - a) * b * s)
    return w00, w01, w10, (1 << W_BITS) - w00 - w01 - w10


def _gather(buf: np.ndarray, ix: np.ndarray, iy: np.ndarray, W: int, H: int) -> np.ndarray:
    """The (H + 1) x (W + 1) block of a padded buffer at padded (iy + H, ix + W), per point."""
    r = (iy + H)[:, None] + np.arange(H + 1)
    c = (ix + W)[:, None] + np.arange(W + 1)
    return buf[r[:, :, None], c[:, None, :]].astype(np.int64)


def _interp(P: np.ndarray, w, shift: int) -> np.ndarray:
    w00, w01, w10, w11 = (x.reshape((-1,) + (1,) * (P.ndim - 1)) for x in w)
    s = P[:, :-1, :-1] * w00 + P[:, :-1, 1:] * w01 + P[:, 1:, :-1] * w10 + P[:, 1:, 1:] * w11
    assert np.abs(s).max(initial=0) < 1 << 31   # the SSE2 path's 32-bit sums
    return (s + (1 << (shift - 1))) >> shift


def _chain(terms: np.ndarray) -> np.ndarray:
    """The last element of a sequential float32 sum along axis 1 (0 for an empty chain): (n, L, lanes) -> (n, lanes)."""
    if terms.shape[1] == 0:
        return np.zeros((terms.shape[0],) + terms.shape[2:], np.float32)
    return np.cumsum(terms, axis=1, dtype=np.float32)[:, -1]


def a_sums(dIw: np.ndarray) -> np.ndarray:
    """iA11, iA12, iA22 (:257-330) of interpolated derivatives dIw (n, H, W, 2) int64: (n, 3) float32, before FLT_SCALE."""
    n, H, W, _ = dIw.shape
    nc4 = W // 4
    out = np.empty((n, 3), np.float32)
    head = dIw[:, :, :4 * nc4].reshape(n, H * nc4, 4, 2).astype(np.float32)   # (point, chunk in row-major order, lane, comp)
    tail = dIw[:, :, 4 * nc4:].reshape(n, -1, 2)
    for m, (p, q) in enumerate(((0, 0), (0, 1), (1, 1))):
        lanes = _chain(head[..., p] * head[..., q])                                # exact products (|I| <= 4080)
        t = _chain((tail[..., p] * tail[..., q]).astype(np.float32)[..., None])[:, 0]
        out[:, m] = t + (((lanes[:, 0] + lanes[:, 1]) + lanes[:, 2]) + lanes[:, 3])
    return out


def b_sums(diff: np.ndarray, dIw: np.ndarray):
    """ib1, ib2 (:382-435) of differences diff (n, H, W) and derivatives dIw (n, H, W, 2): ((n, 2) float32, largest |madd pair|)."""
    n, H, W = diff.shape
    nc8 = W // 8
    d = diff[:, :, :8 * nc8].reshape(n, H, nc8, 2, 4)          # (.., chunk, half, j): pixel 8c + 4 half + j
    g = dIw[:, :, :8 * nc8].reshape(n, H, nc8, 2, 4, 2)
    pairs = (d[..., None] * g).sum(3).reshape(n, H * nc8, 4, 2)  # one _mm_madd_epi16 pair: pixel j and j + 4, Ix or Iy
    madd = np.abs(pairs).reshape(n, -1).max(1, initial=0)
    # qb0 lane k = (pixel pair k >> 1, comp k & 1), qb1 lane k = (pixel pair 2 + (k >> 1), comp k & 1)
    qb0 = _chain(pairs[:, :, 0:2, :].reshape(n, -1, 4).astype(np.float32))
    qb1 = _chain(pairs[:, :, 2:4, :].reshape(n, -1, 4).astype(np.float32))
    bbuf = qb0 + qb1
    tail = (diff[:, :, 8 * nc8:, None] * dIw[:, :, 8 * nc8:]).reshape(n, -1, 2)
    t = _chain(tail.astype(np.float32))
    ib = np.stack([t[:, 0] + (bbuf[:, 0] + bbuf[:, 2]), t[:, 1] + (bbuf[:, 1] + bbuf[:, 3])], 1)
    return ib, madd


def _exact(dIw: np.ndarray, diff: np.ndarray | None):
    """Unrounded int64 sums and sums of |terms| of the A chains (diff None) or the b chains."""
    if diff is None:
        ix, iy = dIw[..., 0], dIw[..., 1]
        terms = np.stack([ix * ix, ix * iy, iy * iy], -1).reshape(len(dIw), -1, 3)
    else:
        terms = (diff[..., None] * dIw).reshape(len(dIw), -1, 2)
    return terms.sum(1), np.abs(terms).sum(1), terms.shape[1]


def track_level(lv, level: int, max_level: int, win: tuple[int, int], max_count: int, epsilon: float, min_eig: np.float32,
                prev_pts: np.ndarray, next_pts: np.ndarray, status: np.ndarray, exact: bool = False) -> dict:
    """calculateLKOpticalFlow for one level over all points; next_pts and status are updated in place.  lv = (I padded, dI
    padded, J padded, cols, rows).  Returns the level's trace."""
    Ipad, dIpad, Jpad, cols, rows = lv
    W, H = win
    n = len(prev_pts)
    hwx, hwy = F((W - 1) * 0.5), F((H - 1) * 0.5)
    sc = F(1.0 / (1 << level))
    mc = max(max_count, 1)
    tr = dict(ipx=np.zeros(n, np.int64), ipy=np.zeros(n, np.int64), A11=np.full(n, np.nan, np.float32), A12=np.full(n, np.nan, np.float32),
              A22=np.full(n, np.nan, np.float32), D=np.full(n, np.nan, np.float32), min_eig=np.full(n, np.nan, np.float32),
              exit=np.full(n, -1, np.int8), iters=np.zeros(n, np.int64), dx=np.full((n, mc), np.nan, np.float32),
              dy=np.full((n, mc), np.nan, np.float32), ddot=np.full((n, mc), np.nan, np.float64), inx=np.zeros((n, mc), np.int64),
              iny=np.zeros((n, mc), np.int64), scharr=np.zeros(n, np.int64), diff=np.zeros(n, np.int64), madd=np.zeros(n, np.int64))
    if exact:
        tr.update(A_sum=np.full((n, 3), np.nan, np.float32), A_exact=np.zeros((n, 3), np.int64), A_abs=np.zeros((n, 3), np.int64),
                  b_sum=np.full((n, mc, 2), np.nan, np.float32), b_exact=np.zeros((n, mc, 2), np.int64), b_abs=np.zeros((n, mc, 2), np.int64),
                  A_terms=0, b_terms=0)
    px = fmul_x86(prev_pts[:, 0], sc)
    py = fmul_x86(prev_pts[:, 1], sc)
    if level == max_level:
        nx, ny = px.copy(), py.copy()
    else:
        nx, ny = fmul_x86(next_pts[:, 0], F(2)), fmul_x86(next_pts[:, 1], F(2))
    next_pts[:, 0], next_pts[:, 1] = nx, ny
    px, py = px - hwx, py - hwy
    ipx, ipy = cv_floor(px), cv_floor(py)
    tr["ipx"], tr["ipy"] = ipx, ipy
    out = (ipx < -W) | (ipx >= cols) | (ipy < -H) | (ipy >= rows)
    tr["exit"][out] = OUTSIDE
    if level == 0:
        status[out] = 0
    for s in range(0, n, CHUNK):
        idx = np.flatnonzero(~out[s:s + CHUNK]) + s
        if len(idx):
            _track_block(idx, Ipad, dIpad, Jpad, cols, rows, W, H, hwx, hwy, max_count, epsilon, min_eig, level,
                         px, py, ipx, ipy, nx, ny, next_pts, status, tr, exact)
    return tr


def _track_block(idx, Ipad, dIpad, Jpad, cols, rows, W, H, hwx, hwy, max_count, epsilon, min_eig, level,
                 px, py, ipx, ipy, nx0, ny0, next_pts, status, tr, exact):
    w = weights(px[idx] - ipx[idx].astype(np.float32), py[idx] - ipy[idx].astype(np.float32))
    Iw = _interp(_gather(Ipad, ipx[idx], ipy[idx], W, H), w, W_BITS - 5)
    dIw = _interp(_gather(dIpad, ipx[idx], ipy[idx], W, H), w, W_BITS)
    tr["scharr"][idx] = np.abs(dIw).reshape(len(idx), -1).max(1)
    iA = a_sums(dIw)
    if exact:
        tr["A_sum"][idx] = iA
        tr["A_exact"][idx], tr["A_abs"][idx], tr["A_terms"] = _exact(dIw, None)
    A11, A12, A22 = iA[:, 0] * FLT_SCALE, iA[:, 1] * FLT_SCALE, iA[:, 2] * FLT_SCALE
    D = A11 * A22 - A12 * A12
    dd = A11 - A22
    min_eig_v = ((A22 + A11) - np.sqrt(dd * dd + F(4) * A12 * A12)) / F(2 * W * H)
    tr["A11"][idx], tr["A12"][idx], tr["A22"][idx], tr["D"][idx], tr["min_eig"][idx] = A11, A12, A22, D, min_eig_v
    rej_eig = min_eig_v < min_eig
    rej = rej_eig | (D < FLT_EPSILON)
    tr["exit"][idx[rej_eig]] = MIN_EIG
    tr["exit"][idx[rej & ~rej_eig]] = DET
    if level == 0:
        status[idx[rej]] = 0
    keep = ~rej
    idx, Iw, dIw, A11, A12, A22 = idx[keep], Iw[keep], dIw[keep], A11[keep], A12[keep], A22[keep]
    Dinv = F(1) / D[keep]
    nx, ny = nx0[idx] - hwx, ny0[idx] - hwy
    pdx, pdy = np.zeros(len(idx), np.float32), np.zeros(len(idx), np.float32)
    live = np.arange(len(idx))
    tr["exit"][idx] = COUNT
    for j in range(max_count):
        if not len(live):
            break
        g = idx[live]
        inx, iny = cv_floor(nx[live]), cv_floor(ny[live])
        tr["inx"][g, j], tr["iny"][g, j] = inx, iny
        o = (inx < -W) | (inx >= cols) | (iny < -H) | (iny >= rows)
        tr["exit"][g[o]] = OUTSIDE_ITER
        if level == 0:
            status[g[o]] = 0
        live, g, inx, iny = live[~o], g[~o], inx[~o], iny[~o]
        if not len(live):
            break
        tr["iters"][g] = j + 1
        wj = weights(nx[live] - inx.astype(np.float32), ny[live] - iny.astype(np.float32))
        diff = _interp(_gather(Jpad, inx, iny, W, H), wj, W_BITS - 5) - Iw[live]
        tr["diff"][g] = np.maximum(tr["diff"][g], np.abs(diff).reshape(len(g), -1).max(1))
        ib, madd = b_sums(diff, dIw[live])
        tr["madd"][g] = np.maximum(tr["madd"][g], madd)
        if exact:
            tr["b_sum"][g, j] = ib
            tr["b_exact"][g, j], tr["b_abs"][g, j], tr["b_terms"] = _exact(dIw[live], diff)
        b1, b2 = ib[:, 0] * FLT_SCALE, ib[:, 1] * FLT_SCALE
        a11, a12, a22, dinv = A11[live], A12[live], A22[live], Dinv[live]
        dx = (a12 * b2 - a22 * b1) * dinv
        dy = (a12 * b1 - a11 * b2) * dinv
        nx[live] = nx[live] + dx
        ny[live] = ny[live] + dy
        cx, cy = nx[live] + hwx, ny[live] + hwy
        ddot = dx.astype(np.float64) * dx.astype(np.float64) + dy.astype(np.float64) * dy.astype(np.float64)
        tr["dx"][g, j], tr["dy"][g, j], tr["ddot"][g, j] = dx, dy, ddot
        stop = ddot <= np.float64(epsilon)
        osc = ~stop & (j > 0) & (np.abs(dx + pdx[live]).astype(np.float64) < np.float64(0.01)) & \
            (np.abs(dy + pdy[live]).astype(np.float64) < np.float64(0.01))
        cx = np.where(osc, cx - dx * F(0.5), cx)
        cy = np.where(osc, cy - dy * F(0.5), cy)
        next_pts[g, 0], next_pts[g, 1] = cx, cy
        tr["exit"][g[stop]] = EPS
        tr["exit"][g[osc]] = OSC
        pdx[live], pdy[live] = dx, dy
        live = live[~(stop | osc)]


class LKRestated:
    """The restated LKOpticalFlowKernel: the same constructor and trackImage (:755-795) as tests/lk_ref.py's LKReference."""

    def __init__(self, win_size=(21, 21), max_level=3, criteria=(3, 30, 0.01), flags=0, min_eig_threshold=1e-4, exact=False):
        self.win = (int(win_size[0]), int(win_size[1]))
        self.max_level = int(max_level)
        self.max_count, self.epsilon = termination(criteria)
        self.min_eig = F(min_eig_threshold)      # calculateLKOpticalFlow's float parameter
        self.exact = exact
        self.prev = None                          # the previous image's pyramid
        self.curr = None
        self.trace = []

    def track(self, gray, last_pts, status_in=None):
        """(curr_pts (n, 2) float32, status (n,) uint8, return value); the trace of the call is self.trace[level]."""
        img = np.ascontiguousarray(gray, np.uint8)
        pts = np.ascontiguousarray(last_pts, np.float32).reshape(-1, 2)
        n = len(pts)
        if self.prev is None:
            self.max_level = level_count(img.shape[1], img.shape[0], self.win, self.max_level)
        self.curr = pyramid(img, self.win, self.max_level)
        self.trace = []
        if self.prev is None:               # the first image
            self.prev = self.curr
            st = np.ones(n, np.uint8) if status_in is None else np.array(status_in, np.uint8).reshape(n)
            return pts.copy(), st, 0
        curr, st = pts.copy(), np.ones(n, np.uint8)
        traces = {}
        for level in range(self.max_level, -1, -1):
            (I, dI), (J, _) = self.prev[level], self.curr[level]
            rows, cols = I.shape[0] - 2 * self.win[1], I.shape[1] - 2 * self.win[0]
            traces[level] = track_level((I, dI, J, cols, rows), level, self.max_level, self.win, self.max_count, self.epsilon,
                                        self.min_eig, pts, curr, st, self.exact)
        self.trace = [traces[l] for l in range(self.max_level + 1)]
        self.prev, self.curr = self.curr, self.prev
        return curr, st, int(st.sum())

    def info(self) -> dict:
        return dict(max_level=self.max_level, win=self.win, max_count=self.max_count, epsilon=self.epsilon)

    def level(self, which, level):
        """(padded image, padded derivative buffer) of a level: which 0 the last image's, 1 the one before (as LKReference)."""
        return (self.prev if which == 0 else self.curr)[level]
