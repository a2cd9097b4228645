"""Seeded cases of the pyramidal Lucas-Kanade tracker (LKOpticalFlowKernel::trackImage, src/lkpyramid.cpp:755-795).

Images are generated, not stored, with integer arithmetic only (numpy's integer draws, shifts and sums), so every machine
builds the same bytes: a smooth noise texture with rectangles (edges and corners), a half-plane edge and one flat patch,
seen through a camera that moves by sub-pixel shifts, a larger shift, a small rotation, a brightness step and a blur.

Point sets reach every branch of calculateLKOpticalFlow: corners (converge), the flat patch (minEig rejects), points near and
beyond the borders at coarse and fine levels (the out-of-image `continue` at level > 0, status cleared at level 0), and random
points everywhere, where max_count = 1 exhausts the iterations and the oscillation rule fires now and then.
"""
from __future__ import annotations

import numpy as np

MARGIN = 48                   # world pixels around the frame, so every transform samples inside the world
R3LIVE = (1280, 1024)         # (cols, rows) of r3live's camera
NTU = (752, 480)


def _binomial(a: np.ndarray, passes: int) -> np.ndarray:
    """[1 2 1] / 4 along both axes, `passes` times, on int64, edges replicated, rounded down."""
    a = a.astype(np.int64)
    for _ in range(passes):
        p = np.pad(a, 1, mode="edge")
        a = (p[:-2, 1:-1] + 2 * p[1:-1, 1:-1] + p[2:, 1:-1] + 2) >> 2
        p = np.pad(a, 1, mode="edge")
        a = (p[1:-1, :-2] + 2 * p[1:-1, 1:-1] + p[1:-1, 2:] + 2) >> 2
    return a


def world(cols: int, rows: int, seed: int) -> tuple[np.ndarray, dict]:
    """(int64 world image of (rows + 2 MARGIN, cols + 2 MARGIN), features in frame coordinates: corners, flat patch box)."""
    rng = np.random.default_rng(seed)
    H, W = rows + 2 * MARGIN, cols + 2 * MARGIN
    img = _binomial(rng.integers(0, 256, (H, W)), 3)
    img = (img - 128) * 2 + 128
    corners = []
    yy, xx = np.mgrid[0:H, 0:W]
    n_rect = max(4, (cols * rows) // 40000)
    for _ in range(n_rect):
        w, h = int(rng.integers(12, max(13, cols // 6))), int(rng.integers(12, max(13, rows // 6)))
        x0, y0 = int(rng.integers(MARGIN, W - MARGIN - w)), int(rng.integers(MARGIN, H - MARGIN - h))
        img[y0:y0 + h, x0:x0 + w] += int(rng.integers(40, 90)) * (1 if rng.integers(0, 2) else -1)
        corners += [(x0 - MARGIN, y0 - MARGIN), (x0 + w - MARGIN, y0 - MARGIN), (x0 - MARGIN, y0 + h - MARGIN), (x0 + w - MARGIN, y0 + h - MARGIN)]
    # a half-plane edge a*x + b*y > c with integer coefficients
    a, b = int(rng.integers(-5, 6)), int(rng.integers(1, 6))
    img = img + np.where(a * (xx - W // 2) + b * (yy - H // 2) > 0, 30, 0)
    img = np.clip(img, 0, 255)
    # one flat patch, no texture at all
    fw, fh = max(cols // 8, 40), max(rows // 8, 40)
    fx0, fy0 = MARGIN + cols // 2 - fw // 2, MARGIN + rows // 5
    img[fy0:fy0 + fh, fx0:fx0 + fw] = 128
    return img, dict(corners=np.array(corners, np.int64), flat=(fx0 - MARGIN, fy0 - MARGIN, fw, fh))


def sample(img: np.ndarray, cols: int, rows: int, dx256: int = 0, dy256: int = 0, cos16: int = 65536, sin16: int = 0) -> np.ndarray:
    """The frame of (rows, cols) seeing the world shifted by (dx, dy) / 256 px and rotated by (cos16, sin16) / 65536 about the
    frame centre: source = R (x - c) + c + d in 1/256 px, integer bilinear with 8-bit weights, rounded."""
    y, x = np.mgrid[0:rows, 0:cols].astype(np.int64)
    cx, cy = cols // 2, rows // 2
    xs = ((cos16 * (x - cx) - sin16 * (y - cy)) >> 8) + (cx + MARGIN) * 256 + dx256
    ys = ((sin16 * (x - cx) + cos16 * (y - cy)) >> 8) + (cy + MARGIN) * 256 + dy256
    ix, fx = xs >> 8, xs & 255
    iy, fy = ys >> 8, ys & 255
    v = ((256 - fx) * (256 - fy) * img[iy, ix] + fx * (256 - fy) * img[iy, ix + 1] + (256 - fx) * fy * img[iy + 1, ix] +
         fx * fy * img[iy + 1, ix + 1] + 32768) >> 16
    return v.astype(np.uint8)


# (dx256, dy256, cos16, sin16, brightness, blur passes) of each frame of a sequence
SEQUENCE = [
    (0, 0, 65536, 0, 0, 0),
    (95, -156, 65536, 0, 0, 0),          # (0.37, -0.61) px
    (307, 205, 65536, 0, 0, 0),          # (1.2, 0.8) px
    (1536, -1024, 65536, 0, 0, 0),       # (6, -4) px: the coarse levels carry it
    (1600, -900, 65532, 686, 0, 0),      # a rotation of 0.6 degrees about the centre
    (1700, -820, 65532, 686, 14, 0),     # a brightness step
    (1760, -760, 65532, 686, 14, 1),     # a blur
]


def frames(cols: int, rows: int, seed: int, count: int | None = None) -> list[np.ndarray]:
    """`count` frames (default: the whole SEQUENCE; longer sequences keep drifting by the last step)."""
    img, _ = world(cols, rows, seed)
    count = len(SEQUENCE) if count is None else count
    out = []
    for k in range(count):
        if k < len(SEQUENCE):
            dx, dy, c, s, bright, blur = SEQUENCE[k]
        else:
            dx, dy, c, s, bright, blur = SEQUENCE[-1]
            dx, dy = dx + 60 * (k - len(SEQUENCE) + 1), dy + 45 * (k - len(SEQUENCE) + 1)
            dx, dy = max(min(dx, (MARGIN - 8) * 256), -(MARGIN - 8) * 256), max(min(dy, (MARGIN - 8) * 256), -(MARGIN - 8) * 256)
        f = sample(img, cols, rows, dx, dy, c, s).astype(np.int64)
        if blur:
            f = _binomial(f, blur)
        out.append(np.clip(f + bright, 0, 255).astype(np.uint8))
    return out


def points(cols: int, rows: int, seed: int, n: int) -> np.ndarray:
    """(n, 2) float32 points on a 1/256 px grid (exact in float32): corners of the world's rectangles, the flat patch, bands
    near and beyond every border, and uniform points over the whole frame."""
    _, feat = world(cols, rows, seed)
    rng = np.random.default_rng(seed + 7)
    parts = []
    c = feat["corners"]
    c = c[(c[:, 0] >= 0) & (c[:, 0] < cols) & (c[:, 1] >= 0) & (c[:, 1] < rows)]
    if len(c):
        k = min(len(c), max(n // 6, 1))
        parts.append(c[rng.choice(len(c), k, replace=False)] * 256 + rng.integers(-128, 129, (k, 2)))
    fx0, fy0, fw, fh = feat["flat"]
    k = max(n // 12, 1)
    parts.append(np.stack([rng.integers(fx0 * 256 + 4096, (fx0 + fw) * 256 - 4096, k), rng.integers(fy0 * 256 + 2048, (fy0 + fh) * 256 - 2048, k)], 1))
    k = max(n // 6, 1)   # near and beyond the borders: within 40 px of an edge, on either side
    side = rng.integers(0, 4, k)            # left, right, top, bottom
    ax, ay = rng.integers(0, cols * 256, k), rng.integers(0, rows * 256, k)
    across = rng.integers(-40 * 256, 40 * 256, k)
    bx = np.select([side == 0, side == 1], [across, (cols - 1) * 256 - across], ax)
    by = np.select([side == 2, side == 3], [across, (rows - 1) * 256 - across], ay)
    parts.append(np.stack([bx, by], 1))
    used = sum(len(p) for p in parts)
    k = max(n - used, 0)
    parts.append(np.stack([rng.integers(0, cols * 256, k), rng.integers(0, rows * 256, k)], 1))
    p = np.concatenate(parts)[:n]
    return (p.astype(np.float64) / 256.0).astype(np.float32)


# parameter cases: (name, win (w, h), max_level, (criteria type, max_count, epsilon), flags, min_eig_threshold)
SHIPPED = ("shipped", (21, 21), 3, (3, 10, 0.05), 8, 1e-4)   # opticalFlowTracker's constructor (src/opticalFlowTracker.cpp:5-8)
PARAM_CASES = [
    SHIPPED,
    ("win3", (3, 3), 3, (3, 10, 0.05), 8, 1e-4),
    ("win8", (8, 8), 3, (3, 10, 0.05), 0, 1e-4),
    ("win16x12", (16, 12), 3, (3, 10, 0.05), 0, 1e-4),
    ("win31", (31, 31), 3, (3, 10, 0.05), 0, 1e-4),
    ("level0", (21, 21), 0, (3, 10, 0.05), 8, 1e-4),
    ("level5", (21, 21), 5, (3, 10, 0.05), 8, 1e-4),
    ("count1", (21, 21), 3, (3, 1, 0.05), 8, 1e-4),
    ("count30", (21, 21), 3, (3, 30, 0.05), 8, 1e-4),
    ("eps0", (21, 21), 3, (3, 30, 0.0), 8, 1e-4),
    ("default_criteria", (21, 21), 3, (1, 30, 0.01), 4, 1e-3),
]


# the runs of tests/golden/lk_track.npz: (name, (cols, rows), seed, points, parameter case, frames).  Each frame after the first
# tracks the previous frame's output points (all of them, whatever their status).
GOLDEN_RUNS = [
    ("r3live_300", R3LIVE, 11, 300, SHIPPED, 4),
    ("ntu_300", NTU, 12, 300, SHIPPED, len(SEQUENCE)),
    ("r3live_20000", R3LIVE, 13, 20000, SHIPPED, 3),
    ("odd_161x97", (161, 97), 14, 300, SHIPPED, 4),        # max_level 3 -> 2
    ("trunc_330x50", (330, 50), 15, 200, SHIPPED, 3),      # max_level 3 -> 1
    ("level5_r3live", R3LIVE, 16, 300, PARAM_CASES[6], 3),
] + [(f"param_{c[0]}", (320, 240), 20 + i, 200, c, 4) for i, c in enumerate(PARAM_CASES[1:]) if c[0] != "level5"]


def run_inputs(run):
    """(frames, initial points, kernel kwargs) of a GOLDEN_RUNS entry."""
    name, (cols, rows), seed, n, case, count = run
    _, win, max_level, criteria, flags, min_eig = case
    kw = dict(win_size=win, max_level=max_level, criteria=criteria, flags=flags, min_eig_threshold=min_eig)
    return frames(cols, rows, seed, count), points(cols, rows, seed, n), kw


def level_digest(levels) -> str:
    """sha256 over the (padded image, derivative buffer) pairs of a pyramid, level 0 first."""
    import hashlib
    h = hashlib.sha256()
    for img, der in levels:
        h.update(np.ascontiguousarray(img, np.uint8).tobytes())
        h.update(np.ascontiguousarray(der, np.int16).tobytes())
    return h.hexdigest()


def image_digest(img) -> str:
    import hashlib
    return hashlib.sha256(np.ascontiguousarray(img, np.uint8).tobytes()).hexdigest()
