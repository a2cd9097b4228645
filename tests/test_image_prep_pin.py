"""Pins the camera image preparation's restatement (image_prep_reference) to OpenCV: against the golden vectors that
tests/golden/make_image_golden.py made with cv2, against cv2 itself when it is importable, and the recipe's own rules
(the tile formula, the truncated output size, the channel order of the grey conversion)."""
import os

import numpy as np
import pytest

import image_prep_cases as IC
import image_prep_reference as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "image_prep.npz")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def check_against_golden(g, case, rgb, gray, map1, map2):
    n = case.name
    assert tuple(g[f"{n}/shape"]) == gray.shape
    outs = (("map1", map1), ("map2", map2), ("gray", gray), ("rgb", rgb))
    if f"{n}/gray" in g:
        for k, a in outs:
            assert np.array_equal(a, g[f"{n}/{k}"]), (n, k, int((a != g[f"{n}/{k}"]).sum()))
    else:
        for k, a in outs:
            assert IC.digest(a) == str(g[f"{n}/{k}_sha"]), (n, k)


@pytest.mark.parametrize("name", [c.name for c in IC.CASES])
def test_restatement_equals_golden(golden, name):
    case = IC.BY_NAME[name]
    bgr = case.bgr()
    assert IC.digest(bgr) == str(golden[f"{name}/input_sha"]), "the case generator changed"
    rgb, gray, map1, map2, *_ = R.prepare(bgr, **case.camera)
    check_against_golden(golden, case, rgb, gray, map1, map2)


@pytest.mark.parametrize("name", ["r3live_212", "strong_small", "odd_203", "narrow_60", "min_16", "two_level"])
def test_restatement_equals_live_cv2(name):
    cv2 = pytest.importorskip("cv2")
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(GOLDEN)))
    from make_image_golden import opencv_recipe
    case = IC.BY_NAME[name]
    bgr = case.bgr()
    want = opencv_recipe(bgr, **case.camera)
    got = R.prepare(bgr, **case.camera)[:4]
    for w, g in zip(want, got):
        assert np.array_equal(w, g)
    # each stage on its own, on the distorted camera's undistorted image
    und = R.remap_bilinear(bgr, got[2], got[3])
    assert np.array_equal(und, cv2.remap(bgr, got[2], got[3], cv2.INTER_LINEAR))
    assert np.array_equal(R.rgb2gray(und), cv2.cvtColor(und, cv2.COLOR_RGB2GRAY))
    ycc = cv2.cvtColor(und, cv2.COLOR_BGR2YCrCb)
    assert all(np.array_equal(a, ycc[..., k]) for k, a in enumerate(R.bgr2ycrcb(und)))
    assert np.array_equal(R.ycrcb2bgr(ycc[..., 0], ycc[..., 1], ycc[..., 2]), cv2.cvtColor(ycc, cv2.COLOR_YCrCb2BGR))


def test_first_image_step_truncates_and_scales():
    s, K, oc, orows, t = R.first_image(1280, 1024, IC.R3LIVE["camera_intrinsic"], 212)
    assert (oc, orows) == (211, 169) and s == 1280 / 212
    assert K[0, 0] == 863.4241 / s and K[0, 2] == 640.6808 / s and K[1, 1] == 863.4171 / s and K[1, 2] == 518.3392 / s
    assert K[2, 2] == 1.0 and K[0, 1] == 0.0
    assert R.first_image(1280, 1024, IC.R3LIVE["camera_intrinsic"], 465)[2:4] == (464, 371)
    assert R.first_image(1280, 1024, IC.R3LIVE["camera_intrinsic"], 640)[:1] == (2.0,)
    assert R.first_image(752, 480, IC.NTU["camera_intrinsic"], 752)[2:] == (752, 480, 37)


def test_tile_grid_is_square_from_cols_with_a_floor_of_four():
    assert [R.clahe_tiles(c) for c in (1280, 752, 640, 203, 80, 79, 60, 16)] == [64, 37, 32, 10, 4, 4, 4, 4]
    # non-square image: both dimensions of the grid come from cols, and a grid that divides neither side pads both
    lut, tw, th = R.clahe_luts(np.zeros((480, 752), np.uint8), 3.0, 37)
    assert lut.shape == (37, 37, 256) and (tw, th) == (21, 13)
    # a side the grid divides still gets a full extra tile's width when the other side needs padding
    assert R.clahe_luts(np.zeros((50, 64), np.uint8), 1.0, 4)[1:] == (17, 13)


def test_gray_weights_channel_zero_as_red():
    px = np.zeros((1, 3, 3), np.uint8)
    px[0, 0, 0] = px[0, 1, 1] = px[0, 2, 2] = 255
    # 15-bit weights 9798 / 19235 / 3735 with channel 0 (B of the BGR image) weighted as R
    assert R.rgb2gray(px).tolist() == [[76, 150, 29]]
    assert R.bgr2ycrcb(px)[0].tolist() == [[29, 150, 76]]
