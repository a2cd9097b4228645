"""Edge cases of the camera image preparation (imageProcessing::process, src/imageProcessing.cpp:91-125,166-200): the map's
int16 saturation, CLAHE grids that pad one or both sides many times over, inputs whose size disagrees with the yaml's, crafted
CLAHE histograms, LUT rounding ties, colour-conversion clamps and a map full of 1/32 rounding ties.

Like tests/image_prep_cases.py, images are generated with integer arithmetic only, so every machine builds the same bytes.
Each case states in a comment what it is for; test_image_prep_edges_pin.py asserts the premises (saturated entries, the
grid, the identity map, the residuals reached, the clamps) on the cases as built.
"""
from __future__ import annotations

import hashlib
from dataclasses import dataclass

import numpy as np

import image_prep_cases as IC

def camera(cols, rows, fx, fy, cx, cy, dist=(0.0, 0.0, 0.0, 0.0, 0.0)):
    return dict(image_width=cols, image_height=rows, camera_intrinsic=[fx, 0.0, cx, 0.0, fy, cy, 0.0, 0.0, 1.0],
                camera_dist_coeffs=list(dist))


MILD = (-0.1713, 0.0621, 4.1e-04, -2.7e-04, -0.0117)   # a generic barrel lens, no entry near an int16 limit

# fx = fy = 60 over 320 x 240 puts the corners at |x| ~ 2.7, where a large positive k3 drives u far past +-32767 px.  Both widths
# are multiples of 32, so no saturating entry falls in the scalar tail of a vectorised OpenCV row (which wraps); cx, cy are
# off the integer grid, because with astronomic coefficients and an integer principal point an FMA-dispatched OpenCV row
# start gives y = -2e-16 where the scalar order gives 0.
OVERFLOW = camera(320, 240, 60.0, 60.0, 160.1, 120.2, (50.0, 900.0, 0.3, -0.2, 4000.0))
OVERFLOW_HUGE = camera(320, 240, 60.0, 60.0, 160.1, 120.2, (1e6, 1e9, 0.0, 0.0, 1e12))

# round intrinsics with distortion: many 32 u, 32 v land exactly on a 1/32 rounding tie, which a vectorised OpenCV may round
# the other way depending on its build; the device follows the scalar order, so this one is held to the restatement only
TIES = camera(320, 240, 150.0, 150.0, 160.0, 120.0, (-0.25, 0.0625, 0.0, 0.0, 0.0))


@dataclass(frozen=True)
class Case:
    name: str
    camera: dict
    cols: int                  # input size
    rows: int
    image: str                 # "texture", "uniform", "clahe_400", "clahe_240" or "palette"
    seed: int
    grid: tuple | None = None  # (t, tw, th) the case is built to reach
    opencv: bool = True        # False: outside what every OpenCV build agrees on (the tie-heavy map)

    def bgr(self) -> np.ndarray:
        return make_image(self.image, self.cols, self.rows, self.seed, self.grid)


CASES = [
    # map overflow: 70 888 entries saturate map1; unfixed, the wrapped ones land inside the textured image
    Case("overflow", OVERFLOW, 320, 240, "texture", 101),
    # every entry but a few at the centre saturates, many from cvRound's INT_MIN; OpenCV writes 0 there, a wrapped map
    # samples pixel (0, y) of the uniform 200 image
    Case("overflow_huge", OVERFLOW_HUGE, 320, 240, "uniform", 102),
    # t = 64 from cols, 1-row tiles: 48 padding rows reflected (REFLECT_101) several times over a 16-row plane
    Case("wide_1280x16", camera(1280, 16, 900.7, 899.3, 640.3, 8.1, MILD), 1280, 16, "texture", 103, (64, 21, 1)),
    # t = 50 divides the cols but not the 20 rows: both sides pad, 30 reflected rows over 20
    Case("wide_1000x20", camera(1000, 20, 700.3, 701.1, 500.2, 10.4, MILD), 1000, 20, "texture", 104, (50, 21, 1)),
    # the 4-tile floor on a tall plane: t = 4 divides both sides, tiles of 10 x 225
    Case("tall_40x900", camera(40, 900, 500.1, 499.7, 20.3, 450.2, MILD), 40, 900, "texture", 105, (4, 10, 225)),
    # t = 10 divides the rows only, t = 32 the cols only: each pads both sides, a full tile on the side it divides
    Case("rows_divide_219x160", camera(219, 160, 180.3, 179.6, 109.7, 80.4, MILD), 219, 160, "texture", 106, (10, 22, 17)),
    Case("cols_divide_640x50", camera(640, 50, 450.2, 449.1, 320.6, 25.3, MILD), 640, 50, "texture", 107, (32, 21, 2)),
    # an input wider than the yaml: s = 0.5 doubles the intrinsics, 1504 x 960 output, t = 75 pads both sides
    Case("ntu_1504", IC.NTU, 1504, 960, "texture", 108, (75, 21, 13)),
    # an input with fewer rows than the output: the output's 240 rows come from image_height / s, the bottom ones read
    # outside the 200-row input and one row straddles its last row
    Case("ntu_short_rows", IC.NTU, 376, 200, "texture", 109, (18, 21, 14)),
    # crafted CLAHE histograms on an identity map: grey (v, v, v) makes gray = Y = v and Cr = Cb = 128, so one plane drives
    # clip 3 (limit 4) and clip 1 (limit 1) over 1024 tiles of 20 x 20 and every clipped residual 0..255 of both
    Case("clahe_640", camera(640, 640, 431.7, 431.7, 320.3, 319.6), 640, 640, "clahe_400", 110, (32, 20, 20)),
    # tiles of 20 x 12: area 240, so clip 1 gives (int)(240 / 256) = 0, floored to a limit of 1 (clip 3: limit 2)
    Case("clahe_floor", camera(320, 192, 150.0, 150.0, 160.0, 96.0), 320, 192, "clahe_240", 111, (16, 20, 12)),
    # 255.f / 510 = 0.5 exactly: every odd prefix sum is a rounding tie of the LUT (the grid pads 405 rows to 408)
    Case("lut_tie_16x405", camera(16, 405, 300.3, 300.1, 7.9, 202.4, MILD), 16, 405, "texture", 112, (4, 5, 102)),
    # 255.f / 1020 = 0.25 exactly: prefix sums of 2 mod 4 are ties
    Case("lut_tie_16x1020", camera(16, 1020, 300.3, 300.1, 7.9, 509.6, MILD), 16, 1020, "texture", 113, (4, 4, 255)),
    # the BGR cube's corners and pure primaries on an identity map: pure red's Cr is 256 before BGR2YCrCb's clamp, cyan's Cr
    # is 0 and yellow's Cb 1, the lowest any 8-bit BGR reaches; YCrCb2BGR of the equalised Y' clamps below 0 and above 255
    # (a pixel with Y' = 0 cannot clamp: Y = 0 forces Cr, Cb >= 128)
    Case("colour_extremes", camera(160, 960, 211.3, 211.3, 80.3, 479.6), 160, 960, "palette", 114, (8, 20, 120)),
    Case("map_ties", TIES, 320, 240, "texture", 115, opencv=False),
]
BY_NAME = {c.name: c for c in CASES}
OPENCV_CASES = [c.name for c in CASES if c.opencv]

# the colours of the palette image: the eight cube corners, then primaries and secondaries at lower intensities
PALETTE = np.array([(0, 0, 0), (255, 255, 255), (255, 0, 0), (0, 255, 0), (0, 0, 255), (255, 255, 0), (255, 0, 255), (0, 255, 255),
                    (128, 0, 0), (0, 128, 0), (0, 0, 128), (0, 64, 0), (0, 128, 128), (128, 128, 0)], np.uint8)


def _clahe_tile(k: int, area: int, rng: np.random.Generator) -> np.ndarray:
    """The `area` values of crafted tile k, shuffled.
    k < 256: d = k + 1 distinct values spread over 0..255 in near-equal counts; at limit 1 the clipped mass is area - d, so
      the 256 tiles give 256 consecutive residuals (all of 0..255 at area 400).
    k < 512 (area 400): one value with 4 + r pixels (r = k - 256), the rest in bins of at most 4: at limit 4 clipped = r.
    k < 653 (area 400): one value with 4 + c pixels, c = 256..396, the rest in bins of at most 4: clipped / 256 = 1.
    otherwise: n5 = (k - 653) % 81 bins at 5 (one above limit 4), the rest at exactly 4."""
    if k < 256:
        d = min(k + 1, area)
        vals = (np.arange(d) * 256) // d
        counts = np.full(d, area // d)
        counts[:area % d] += 1
    else:
        if k < 653:
            head = [4 + (k - 256)]          # r = 0..255, then c = 256..396
            fours, tail = divmod(area - head[0], 4)
        else:
            n5 = (k - 653) % 81
            head = [5] * n5
            fours, tail = divmod(area - 5 * n5, 4)
        counts = np.array(head + [4] * fours + ([tail] if tail else []))
        start = int(rng.integers(0, 256))
        vals = (start + (np.arange(counts.size) * 256) // counts.size) % 256
    out = np.repeat(vals, counts).astype(np.uint8)
    assert out.size == area, (k, out.size)
    return rng.permutation(out)


def _clahe_plane(cols: int, rows: int, t: int, seed: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    th, tw = rows // t, cols // t
    assert th * t == rows and tw * t == cols
    plane = np.empty((rows, cols), np.uint8)
    for k in range(t * t):
        ty, tx = divmod(k, t)
        plane[ty * th:(ty + 1) * th, tx * tw:(tx + 1) * tw] = _clahe_tile(k, tw * th, rng).reshape(th, tw)
    return plane


def make_image(kind: str, cols: int, rows: int, seed: int, grid=None) -> np.ndarray:
    """(rows, cols, 3) uint8 BGR image."""
    if kind == "texture":
        return IC.make_image("texture", cols, rows, seed)
    if kind == "uniform":
        return np.full((rows, cols, 3), 200, np.uint8)
    if kind in ("clahe_400", "clahe_240"):
        return _clahe_plane(cols, rows, grid[0], seed)[..., None].repeat(3, axis=2)
    if kind == "palette":
        # per-pixel grey noise with half of its 4 x 4 blocks painted in palette colours: the noise spreads each tile's Y
        # histogram, so CLAHE moves Y' away from Y and the saturated colours' reconstruction leaves [0, 255] on both sides
        rng = np.random.default_rng(seed)
        out = rng.integers(0, 256, (rows, cols)).astype(np.uint8)[..., None].repeat(3, axis=2)
        colour = PALETTE[rng.integers(0, PALETTE.shape[0], (rows // 4, cols // 4))].repeat(4, axis=0).repeat(4, axis=1)
        painted = (rng.integers(0, 16, (rows // 4, cols // 4)) < 8).repeat(4, axis=0).repeat(4, axis=1)
        out[painted] = colour[painted]
        return out
    raise ValueError(kind)


def digest(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()
