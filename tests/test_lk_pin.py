"""CPU pins of the pyramidal Lucas-Kanade's test infrastructure (no GPU):
  - the OpenCV stand-in's pyrDown and copyMakeBorder (oracle/shim_lk/srl_lk_cv.h, parity unpinned against OpenCV itself) against an
    independent numpy restatement: np.pad(mode="reflect") is BORDER_REFLECT_101, mode="constant" BORDER_CONSTANT;
  - the case generator's frames against the digests in tests/golden/lk_track.npz (its bytes are part of the pin);
  - the compiled reference (oracle/_ref/libsrl_lk_ref.so) against the golden file, and its pyramid against the numpy restatement.
"""
import os

import numpy as np
import pytest

import lk_cases as K
import lk_ref as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lk_track.npz")
needs_ref = pytest.mark.skipif(not R.available(), reason="oracle/_ref/libsrl_lk_ref.so not built (needs the reference tree)")
REFLECT_101, CONSTANT, ISOLATED = 4, 0, 16


def np_pyr_down(src):
    """[1 4 6 4 1]^2 / 256 at (2x, 2y), REFLECT_101, (s + 128) >> 8."""
    h, w = src.shape
    p = np.pad(src.astype(np.int64), 2, mode="reflect")
    k = np.array([1, 4, 6, 4, 1], np.int64)
    rows = sum(k[i] * p[i:i + h, :] for i in range(5))
    full = sum(k[j] * rows[:, j:j + w] for j in range(5))
    return ((full[::2, ::2] + 128) >> 8).astype(np.uint8)


def np_scharr(img):
    """calcSharrDeriv with REFLECT_101 rows and columns: (Ix, Iy) int16."""
    p = np.pad(img.astype(np.int64), 1, mode="reflect")
    c = lambda dy, dx: p[1 + dy:p.shape[0] - 1 + dy, 1 + dx:p.shape[1] - 1 + dx]
    ix = 3 * (c(-1, 1) + c(1, 1)) + 10 * c(0, 1) - 3 * (c(-1, -1) + c(1, -1)) - 10 * c(0, -1)
    iy = 3 * (c(1, -1) + c(1, 1)) + 10 * c(1, 0) - 3 * (c(-1, -1) + c(-1, 1)) - 10 * c(-1, 0)
    return np.stack([ix, iy], -1).astype(np.int16)


@needs_ref
@pytest.mark.parametrize("shape", [(97, 161), (50, 330), (480, 752), (7, 9), (2, 3), (31, 64)])
def test_stand_in_pyr_down(shape):
    img = np.random.default_rng(shape[0] * 1000 + shape[1]).integers(0, 256, shape).astype(np.uint8)
    assert np.array_equal(R.pyr_down(img), np_pyr_down(img))


@needs_ref
@pytest.mark.parametrize("pad", [(3, 3, 3, 3), (21, 21, 21, 21), (12, 16, 8, 31), (0, 2, 5, 0)])
def test_stand_in_copy_make_border(pad):
    t, b, l, r = pad
    rng = np.random.default_rng(sum(pad))
    img = rng.integers(0, 256, (40, 57)).astype(np.uint8)
    der = rng.integers(-4080, 4081, (40, 57, 2)).astype(np.int16)
    whole = (0, 0, 57, 40)
    assert np.array_equal(R.copy_make_border(img, whole, t, b, l, r, REFLECT_101), np.pad(img, ((t, b), (l, r)), mode="reflect"))
    assert np.array_equal(R.copy_make_border(der, whole, t, b, l, r, CONSTANT), np.pad(der, ((t, b), (l, r), (0, 0))))
    # the in-place case: the source is a ROI of the destination (BORDER_ISOLATED: the border is not taken from the parent)
    big = rng.integers(0, 256, (40 + t + b, 57 + l + r)).astype(np.uint8)
    inner = big[t:t + 40, l:l + 57]
    got = R.copy_make_border(big, (l, t, 57, 40), t, b, l, r, REFLECT_101 | ISOLATED, inplace=True)
    assert np.array_equal(got, np.pad(inner, ((t, b), (l, r)), mode="reflect"))
    bigd = rng.integers(-4080, 4081, (40 + t + b, 57 + l + r, 2)).astype(np.int16)
    got = R.copy_make_border(bigd, (l, t, 57, 40), t, b, l, r, CONSTANT | ISOLATED, inplace=True)
    assert np.array_equal(got, np.pad(bigd[t:t + 40, l:l + 57], ((t, b), (l, r), (0, 0))))
    # without BORDER_ISOLATED a ROI's border comes from its parent where the parent has pixels
    roi = (10, 6, 30, 20)
    got = R.copy_make_border(img, roi, 3, 3, 3, 3, REFLECT_101)
    assert np.array_equal(got, img[3:29, 7:43])


@needs_ref
@pytest.mark.parametrize("size", [(161, 97), (330, 50), (96, 64)])
def test_reference_pyramid_matches_numpy(size):
    """The reference's padded levels and derivative buffers = the numpy restatement: level 0 the image, level l pyrDown of l-1,
    REFLECT_101 padding of the window's size, Scharr inside, zero border."""
    cols, rows = size
    f = K.frames(cols, rows, 3, 1)[0]
    ref = R.LKReference((21, 21), 3, (3, 10, 0.05), 8, 1e-4)
    ref.track(f, np.zeros((0, 2), np.float32))
    lvl = f
    for l in range(ref.info()["max_level"] + 1):
        if l:
            lvl = np_pyr_down(lvl)
        img, der = ref.level(0, l)
        assert np.array_equal(img, np.pad(lvl, 21, mode="reflect")), l
        assert np.array_equal(der, np.pad(np_scharr(lvl), ((21, 21), (21, 21), (0, 0)))), l


def test_generator_matches_golden():
    g = np.load(GOLDEN)
    for run in K.GOLDEN_RUNS:
        frames, _, _ = K.run_inputs(run)
        for k, f in enumerate(frames):
            assert K.image_digest(f) == str(g[f"{run[0]}/image{k}"]), (run[0], k)


@needs_ref
@pytest.mark.parametrize("run", K.GOLDEN_RUNS, ids=[r[0] for r in K.GOLDEN_RUNS])
def test_reference_matches_golden(run):
    g = np.load(GOLDEN)
    frames, pts, kw = K.run_inputs(run)
    ref = R.LKReference(**kw)
    last = pts
    for k, f in enumerate(frames):
        curr, st, ret = ref.track(f, last)
        key = f"{run[0]}/"
        assert np.array_equal(curr.view(np.uint32), g[key + f"pts{k}"].view(np.uint32)), k
        assert np.array_equal(st, g[key + f"status{k}"]) and ret == int(g[key + f"ret{k}"]), k
        ml = ref.info()["max_level"]
        assert K.level_digest([ref.level(0, l) for l in range(ml + 1)]) == str(g[key + f"levels{k}"]), k
        last = curr
    assert ref.info()["max_level"] == int(g[f"{run[0]}/max_level"])


@needs_ref
def test_golden_reaches_every_branch():
    """The golden runs converge, reject flat patches, lose points over the border and keep most points tracked."""
    g = np.load(GOLDEN)
    frames, pts, kw = K.run_inputs(K.GOLDEN_RUNS[1])
    tracked = [int(g[f"ntu_300/ret{k}"]) for k in range(1, len(frames))]
    assert all(150 < t < 300 for t in tracked), tracked
    st = g["ntu_300/status1"]
    fx0, fy0, fw, fh = K.world(752, 480, 12)[1]["flat"]
    flat = (pts[:, 0] > fx0 + 11) & (pts[:, 0] < fx0 + fw - 12) & (pts[:, 1] > fy0 + 11) & (pts[:, 1] < fy0 + fh - 12)
    assert flat.sum() > 5 and not st[flat].any()
    outside = (pts[:, 0] < -21) | (pts[:, 1] < -21) | (pts[:, 0] > 752 + 20) | (pts[:, 1] > 480 + 20)
    assert outside.sum() > 3 and not st[outside].any()
