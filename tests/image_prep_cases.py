"""Seeded cases of the camera image preparation (imageProcessing::process, src/imageProcessing.cpp:91-125,166-200).

Images are generated, not stored, with integer arithmetic only (numpy's integer draws, shifts and sums), so every machine
builds the same bytes.  The textured image holds a smooth noise texture, rectangles (edges), a flat field, saturated 0 and
255 regions and a horizontal gradient; the constant image puts a whole tile's mass in one bin, so CLAHE's residual loop runs
with a step above 1; the two-level image splits it over two bins.

Cameras: r3live and ntu at their shipped sizes (ntu's 37-tile grid pads both dimensions), inputs narrower than the yaml width
(640: scale 2; 212: 211 output columns; 465: 371 rows), a strongly distorted camera whose taps fall partly and wholly outside
the image, a small odd size (10 tiles), a size under 80 columns (the 4-tile floor, where the Y plane's clip limit falls to 1)
and the 16 x 16 minimum.
"""
from __future__ import annotations

import hashlib
from dataclasses import dataclass

import numpy as np

R3LIVE = dict(image_width=1280, image_height=1024, camera_intrinsic=[863.4241, 0.0, 640.6808, 0.0, 863.4171, 518.3392, 0.0, 0.0, 1.0],
              camera_dist_coeffs=[-0.1080, 0.1050, -1.2872e-04, 5.7923e-05, -0.0222])
NTU = dict(image_width=752, image_height=480, camera_intrinsic=[425.0259, 0.0, 386.0152, 0.0, 426.7976, 241.9130, 0.0, 0.0, 1.0],
           camera_dist_coeffs=[-0.2881, 0.0746, 7.7845e-04, -2.2779e-04, 0.0])
# strong barrel-to-pincushion terms: the corners' taps land far outside the image, the edges' straddle it.  The values are not
# round on purpose: a map entry on an exact 1/32 tie is rounded by whichever lane order an OpenCV build vectorises with.
STRONG = dict(image_width=320, image_height=240, camera_intrinsic=[231.4517, 0.0, 158.3371, 0.0, 229.8813, 121.6629, 0.0, 0.0, 1.0],
              camera_dist_coeffs=[0.8123, 0.4417, 0.0123, -0.0091, 0.2571])
SQUARE = dict(image_width=64, image_height=64, camera_intrinsic=[52.3117, 0.0, 31.7243, 0.0, 51.9871, 32.2119, 0.0, 0.0, 1.0],
              camera_dist_coeffs=[-0.2113, 0.0517, 1.3e-03, -7.1e-04, 0.0])

FULL_LIMIT = 40000   # output pixels up to which the golden file stores whole maps and images; larger cases keep SHA-256 digests


@dataclass(frozen=True)
class Case:
    name: str
    camera: dict
    cols: int          # input size
    rows: int
    image: str         # "texture", "constant" or "two_level"
    seed: int

    def bgr(self) -> np.ndarray:
        return make_image(self.image, self.cols, self.rows, self.seed)


CASES = [
    Case("r3live", R3LIVE, 1280, 1024, "texture", 1),
    Case("ntu", NTU, 752, 480, "texture", 2),
    Case("r3live_half", R3LIVE, 640, 512, "texture", 3),
    Case("r3live_212", R3LIVE, 212, 170, "texture", 4),
    Case("r3live_465", R3LIVE, 465, 372, "texture", 5),
    Case("strong", STRONG, 320, 240, "texture", 6),
    Case("strong_small", STRONG, 160, 120, "texture", 7),
    Case("odd_203", NTU, 203, 157, "texture", 8),
    Case("narrow_60", NTU, 60, 50, "texture", 9),
    Case("min_16", SQUARE, 16, 16, "texture", 10),
    Case("constant", NTU, 188, 120, "constant", 11),
    Case("two_level", NTU, 188, 120, "two_level", 12),
    Case("constant_r3live", R3LIVE, 1280, 1024, "constant", 13),
]
BY_NAME = {c.name: c for c in CASES}


def _smooth(a: np.ndarray, passes: int) -> np.ndarray:
    """[1 2 1] / 4 along both axes, `passes` times, on int64, edges replicated, rounded down."""
    for _ in range(passes):
        p = np.pad(a, 1, mode="edge")
        a = (p[:-2, 1:-1] + 2 * p[1:-1, 1:-1] + p[2:, 1:-1] + 2) >> 2
        p = np.pad(a, 1, mode="edge")
        a = (p[1:-1, :-2] + 2 * p[1:-1, 1:-1] + p[1:-1, 2:] + 2) >> 2
    return a


def make_image(kind: str, cols: int, rows: int, seed: int) -> np.ndarray:
    """(rows, cols, 3) uint8 BGR image."""
    rng = np.random.default_rng(seed)
    if kind == "constant":
        return np.full((rows, cols, 3), (37, 141, 203), np.uint8)
    if kind == "two_level":
        yy, xx = np.mgrid[0:rows, 0:cols]
        return np.where((((xx // 7) + (yy // 5)) % 2 == 0)[..., None], np.uint8(60), np.uint8(190)).repeat(3, axis=2).astype(np.uint8)
    img = np.empty((rows, cols, 3), np.int64)
    for c in range(3):
        img[..., c] = _smooth(rng.integers(0, 256, (rows, cols)).astype(np.int64), 2)
        img[..., c] = (img[..., c] - 128) * 3 + 128
    for _ in range(max(3, cols * rows // 30000)):
        w, h = int(rng.integers(2, max(3, cols // 5))), int(rng.integers(2, max(3, rows // 5)))
        x0, y0 = int(rng.integers(0, cols - w + 1)), int(rng.integers(0, rows - h + 1))
        img[y0:y0 + h, x0:x0 + w] += rng.integers(-90, 91, 3)
    xx = np.arange(cols)[None, :]
    g0 = rows // 3
    img[g0:g0 + max(1, rows // 8)] = (xx * 255 // max(cols - 1, 1))[..., None]                       # gradient band
    img[:max(1, rows // 10), :max(1, cols // 6)] = 0                                                   # saturated dark
    img[rows - max(1, rows // 10):, cols - max(1, cols // 6):] = 255                                   # saturated bright
    fx0, fy0 = cols // 2, rows // 2
    img[fy0:fy0 + max(1, rows // 6), fx0:fx0 + max(1, cols // 6)] = (96, 128, 160)                    # flat field
    return np.clip(img, 0, 255).astype(np.uint8)


def digest(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def padded(img: np.ndarray, extra: int = 13) -> np.ndarray:
    """The same image as a view whose rows are cols * 3 + extra bytes apart (a padded ROS step)."""
    rows, cols, _ = img.shape
    buf = np.zeros((rows, cols * 3 + extra), np.uint8)
    buf[:, :cols * 3] = img.reshape(rows, cols * 3)
    return np.lib.stride_tricks.as_strided(buf, shape=(rows, cols, 3), strides=(cols * 3 + extra, 3, 1))
