"""Pins the camera image preparation's restatement (image_prep_reference) to OpenCV on the edge cases of
image_prep_edge_cases: against the SHA-256 digests of tests/golden/image_prep_edges.npz (made with cv2 by
make_image_edges_golden.py) and against cv2 itself when it is importable, which counts the entries that differ.  map2 is
compared at the unsaturated entries only: a vectorised OpenCV may give a saturated entry's map2 another last bit, which no
image can show because every tap of such an entry is outside.  Then the
premises each case is built on: the saturated entries and what a wrapping map would do instead, the grid, the identity map
of the crafted planes, every clipped residual, the exact LUT scales, the colour clamps, the rows read outside the input and
the map's rounding ties."""
import os
import sys

import numpy as np
import pytest

import image_prep_edge_cases as EC
import image_prep_reference as R

F32 = np.float32
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "image_prep_edges.npz")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def check_against_golden(g, case, rgb, gray, map1, map2):
    """The outputs' SHA-256 digests equal the golden file's; map2's over the entries where map1 did not saturate."""
    n = case.name
    assert tuple(g[f"{n}/shape"]) == gray.shape
    sat = R.saturated(map1)
    for k, a in (("map1", map1), ("map2_unsat", map2[~sat]), ("gray", gray), ("rgb", rgb)):
        assert EC.digest(a) == str(g[f"{n}/{k}_sha"]), (n, k)


def _opencv_recipe():
    sys.path.insert(0, os.path.dirname(GOLDEN))
    from make_image_golden import opencv_recipe
    return opencv_recipe


def _maps_raw(case):
    """(32 u, 32 v, scaled K, out_cols, out_rows, t) of the case's camera before cvRound."""
    cam = case.camera
    s, K, oc, orows, t = R.first_image(cam["image_width"], cam["image_height"], cam["camera_intrinsic"], case.cols)
    u, v = R.undistort_coords(K, cam["camera_dist_coeffs"], oc, orows)
    return u, v, K, oc, orows, t


@pytest.mark.parametrize("name", EC.OPENCV_CASES)
def test_restatement_equals_golden(golden, name):
    case = EC.BY_NAME[name]
    bgr = case.bgr()
    assert EC.digest(bgr) == str(golden[f"{name}/input_sha"]), "the case generator changed"
    rgb, gray, map1, map2, *_ = R.prepare(bgr, **case.camera)
    check_against_golden(golden, case, rgb, gray, map1, map2)


@pytest.mark.parametrize("name", EC.OPENCV_CASES)
def test_restatement_equals_live_cv2(name):
    cv2 = pytest.importorskip("cv2")
    cv2.setNumThreads(1)
    case = EC.BY_NAME[name]
    bgr = case.bgr()
    rgb_w, gray_w, m1_w, m2_w = _opencv_recipe()(bgr, **case.camera)
    rgb, gray, map1, map2, *_ = R.prepare(bgr, **case.camera)
    sat = R.saturated(map1)
    assert np.array_equal(map1, m1_w), int((map1 != m1_w).any(-1).sum())
    assert np.array_equal(map2[~sat], m2_w[~sat]), int((map2 != m2_w)[~sat].sum())
    assert np.array_equal(gray, gray_w), int((gray != gray_w).sum())
    assert np.array_equal(rgb, rgb_w), int((rgb != rgb_w).any(-1).sum())


@pytest.mark.parametrize("name, n_saturated", [("overflow", 70888), ("overflow_huge", 76778)])
def test_overflow_cameras_saturate_and_a_wrapped_map_would_differ(name, n_saturated):
    case = EC.BY_NAME[name]
    bgr = case.bgr()
    u, v, _, oc, orows, _ = _maps_raw(case)
    rgb, gray, map1, map2, *_ = R.prepare(bgr, **case.camera)
    sat = R.saturated(map1)
    assert oc % 32 == 0 and int(sat.sum()) == n_saturated
    iu, iv = R._cv_round(u), R._cv_round(v)
    # every tap of a saturated entry is outside the image, so it samples the border value 0
    sx, sy = map1[..., 0].astype(np.int64), map1[..., 1].astype(np.int64)
    assert (((sx[sat] < -1) | (sx[sat] >= case.cols)) | ((sy[sat] < -1) | (sy[sat] >= case.rows))).all()
    # the plain (short) cast of the unfixed kernel: wrapped entries whose taps land inside the image, and different pixels
    wrapped = np.stack([(iu >> 5).astype(np.int16), (iv >> 5).astype(np.int16)], axis=-1)
    wx, wy = wrapped[..., 0].astype(np.int64), wrapped[..., 1].astype(np.int64)
    inside = sat & (wx >= 0) & (wx < case.cols) & (wy >= 0) & (wy < case.rows)
    assert inside.sum() > 0
    und_w = R.remap_bilinear(bgr, wrapped, map2)
    assert (und_w != R.remap_bilinear(bgr, map1, map2)).any(-1).sum() > 0
    if name == "overflow_huge":
        # cvRound's INT_MIN (outside the int range) on most entries: OpenCV keeps -32768, a wrap gives 0, a real column
        assert (iu == -2**31).sum() > 60000
        assert (R.process(bgr, wrapped, map2, R.clahe_tiles(oc))[0] != rgb).any(-1).sum() > 70000


@pytest.mark.parametrize("name", [c.name for c in EC.CASES if c.grid])
def test_grid_premise(name):
    case = EC.BY_NAME[name]
    gray = R.prepare(case.bgr(), **case.camera)[1]
    t, tw, th = case.grid
    assert R.clahe_tiles(gray.shape[1]) == t
    assert R.clahe_luts(gray, 3.0, t)[1:] == (tw, th)
    if name == "wide_1280x16":
        assert gray.shape == (16, 1280) and th * t - 16 == 48   # 48 padding rows reflected over 16
    if name == "tall_40x900":
        assert gray.shape[1] % t == 0 and gray.shape[0] % t == 0
    if name in ("rows_divide_219x160", "cols_divide_640x50"):
        assert (gray.shape[0] % t == 0) != (gray.shape[1] % t == 0)


def test_input_size_premises():
    wide = EC.BY_NAME["ntu_1504"]
    s, K, oc, orows, t = R.first_image(752, 480, EC.IC.NTU["camera_intrinsic"], wide.cols)
    assert s == 0.5 and (oc, orows, t) == (1504, 960, 75) and K[0, 0] == 2 * EC.IC.NTU["camera_intrinsic"][0]
    short = EC.BY_NAME["ntu_short_rows"]
    _, _, map1, map2, *_ = R.prepare(short.bgr(), **short.camera)
    assert map1.shape[0] == 240 > short.rows
    sy, fy = map1[..., 1].astype(np.int64), map2 >> 5
    assert (sy >= short.rows).sum() > 1000                               # wholly below the input
    assert ((sy == short.rows - 1) & (fy > 0)).sum() > 100               # one tap on the last row, the other below it


@pytest.mark.parametrize("name", ["clahe_640", "clahe_floor", "colour_extremes"])
def test_crafted_cases_have_an_identity_map(name):
    case = EC.BY_NAME[name]
    _, _, map1, map2, *_ = R.prepare(case.bgr(), **case.camera)
    yy, xx = np.mgrid[0:case.rows, 0:case.cols]
    assert (map2 == 0).all() and np.array_equal(map1[..., 0], xx) and np.array_equal(map1[..., 1], yy)


def _tile_hists(plane, t):
    h, w = plane.shape
    th, tw = h // t, w // t
    tiles = plane.reshape(t, th, t, tw).transpose(0, 2, 1, 3).reshape(t * t, th * tw).astype(np.int64)
    hist = np.zeros((t * t, 256), np.int64)
    np.add.at(hist, (np.repeat(np.arange(t * t), th * tw), tiles.reshape(-1)), 1)
    return hist, th * tw


def test_crafted_planes_reach_every_residual():
    case = EC.BY_NAME["clahe_640"]
    bgr = case.bgr()
    t = case.grid[0]
    gray_in = R.rgb2gray(bgr)
    y, cr, cb = R.bgr2ycrcb(bgr)
    # grey BGR: one plane is both CLAHEs' input, and rgb_image is Y' itself
    assert np.array_equal(gray_in, bgr[..., 0]) and np.array_equal(y, bgr[..., 0]) and (cr == 128).all() and (cb == 128).all()
    rgb, gray, *_ = R.prepare(bgr, **case.camera)
    assert np.array_equal(rgb, R.clahe(y, 1.0, t)[..., None].repeat(3, axis=2))
    hist, area = _tile_hists(bgr[..., 0], t)
    assert area == 400
    for clip, limit in ((3.0, 4), (1.0, 1)):
        assert max(int(clip * area / 256), 1) == limit
        clipped = np.maximum(hist - limit, 0).sum(axis=1)
        assert set((clipped % 256).tolist()) == set(range(256)), clip
        assert (clipped >= 256).any() and (clipped < 256).any()
        assert limit == 1 or (clipped == 0).any()
    # bins exactly at limit 4 and one above it, in tiles that clip nothing more than those
    assert ((hist == 4).any(axis=1) & (hist == 5).any(axis=1) & (hist <= 5).all(axis=1)).sum() > 50
    floor = EC.BY_NAME["clahe_floor"]
    hist, area = _tile_hists(floor.bgr()[..., 0], floor.grid[0])
    assert area == 240 and int(1.0 * area / 256) == 0 and int(3.0 * area / 256) == 2
    assert len(set((np.maximum(hist - 1, 0).sum(axis=1) % 256).tolist())) == 240


@pytest.mark.parametrize("name, scale", [("lut_tie_16x405", 0.5), ("lut_tie_16x1020", 0.25)])
def test_lut_scale_is_exact_and_ties_are_read(name, scale):
    case = EC.BY_NAME[name]
    rgb, gray, map1, map2, s, K, t = R.prepare(case.bgr(), **case.camera)
    gray_in = R.rgb2gray(R.remap_bilinear(case.bgr(), map1, map2))
    sums, tw, th = R.clahe_sums(gray_in, 3.0, t)
    assert F32(255) / F32(tw * th) == scale
    prod = sums.astype(np.float64) * scale
    tie = prod - np.floor(prod) == 0.5
    assert tie.sum() > 100
    # the tied LUT entries at values the tile's own pixels hold: the blend reads them
    h = gray_in.shape[0]
    present = np.zeros_like(tie)
    for ty in range(t):
        for tx in range(t):
            vals = gray_in[ty * th:min((ty + 1) * th, h), tx * tw:(tx + 1) * tw]
            present[ty * t + tx, np.unique(vals)] = True
    assert (tie & present).sum() > 50


def test_colour_extremes_clamp():
    case = EC.BY_NAME["colour_extremes"]
    bgr = case.bgr()
    assert all((bgr.reshape(-1, 3) == c).all(axis=1).any() for c in EC.PALETTE)
    b, g, r = (bgr[..., k].astype(np.int64) for k in range(3))
    y = (b * 1868 + g * 9617 + r * 4899 + (1 << 13)) >> 14
    cr = ((r - y) * 11682 + (128 << 14) + (1 << 13)) >> 14
    cb = ((b - y) * 9241 + (128 << 14) + (1 << 13)) >> 14
    assert cr.max() == 256 and cr.min() == 0 and cb.min() == 1 and cb.max() == 255
    Y, Cr, Cb = R.bgr2ycrcb(bgr)
    yp = R.clahe(Y, 1.0, case.grid[0]).astype(np.int64)
    assert yp.max() == 255 and (yp != Y).mean() > 0.5
    cr, cb = Cr.astype(np.int64) - 128, Cb.astype(np.int64) - 128
    pre = np.stack([yp + ((cb * 29049 + (1 << 13)) >> 14), yp + ((cb * -5636 + cr * -11698 + (1 << 13)) >> 14),
                    yp + ((cr * 22987 + (1 << 13)) >> 14)], axis=-1)
    assert (pre < 0).any(-1).sum() > 500 and (pre > 255).any(-1).sum() > 5000
    rgb = R.prepare(bgr, **case.camera)[0]
    assert np.array_equal(rgb, np.clip(pre, 0, 255).astype(np.uint8))


def test_tie_heavy_map_differs_from_cv2_only_near_ties():
    case = EC.BY_NAME["map_ties"]
    u, v, *_ = _maps_raw(case)
    du, dv = np.abs(u - np.floor(u) - 0.5), np.abs(v - np.floor(v) - 0.5)
    assert ((du == 0) | (dv == 0)).sum() >= 10
    cv2 = pytest.importorskip("cv2")
    cv2.setNumThreads(1)
    _, _, m1_w, m2_w = _opencv_recipe()(case.bgr(), **case.camera)
    _, _, map1, map2, *_ = R.prepare(case.bgr(), **case.camera)
    diff = (map1 != m1_w).any(-1) | (map2 != m2_w)
    # a different lane order moves u, v by a few ulps: only an entry within that of a tie can round the other way
    near = np.minimum(du / np.maximum(np.abs(u), 1), dv / np.maximum(np.abs(v), 1)) < 1e-13
    assert not (diff & ~near).any()
