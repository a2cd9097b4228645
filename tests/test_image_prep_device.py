"""The camera image preparation on the GPU (srl_image_*: k_img_map, k_img_remap, k_img_clahe_lut, k_img_clahe_apply) against
the golden vectors (OpenCV's own outputs) and the restatement (image_prep_reference), bit for bit: the undistortion maps,
and gray_image / rgb_image of every case from host and device inputs, with padded row pitches, into host and device
outputs.  Then the chain: the device outputs fed to the Lucas-Kanade tracker and the colour renderer give the bits the
golden images give.  Finally every SRL_BAD_ARG of the C ABI, after which the object still works."""
import ctypes as C

import numpy as np
import pytest

import image_prep_cases as IC
import image_prep_reference as R
import render_cases as RC
from test_image_prep_pin import GOLDEN, check_against_golden

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def ctx():
    from sr_livo_b200 import lio
    c = lio.Context(0)
    yield c
    c.close()


def _want(case):
    """(rgb, gray, map1, map2, scale, K, tiles) of the restatement; the golden test of the restatement pins it to OpenCV."""
    return R.prepare(case.bgr(), **case.camera)


@pytest.mark.parametrize("name", [c.name for c in IC.CASES])
def test_maps_and_images_equal_golden_and_restatement(ctx, golden, name):
    import torch
    from sr_livo_b200 import lio
    case = IC.BY_NAME[name]
    bgr = case.bgr()
    rgb_w, gray_w, m1_w, m2_w, s_w, K_w, t_w = _want(case)
    ip = lio.ImageProcessing(ctx, **case.camera, cols=case.cols, rows=case.rows)
    try:
        assert ip.output_size() == (gray_w.shape[1], gray_w.shape[0])
        assert ip.tiles() == t_w and ip.scale_factor() == s_w
        assert np.array_equal(ip.camera_intrinsic(), K_w)
        m1, m2 = ip.maps()
        assert np.array_equal(m1, m1_w), int((m1 != m1_w).sum())
        assert np.array_equal(m2, m2_w), int((m2 != m2_w).sum())
        # host in, host out (numpy, contiguous and with a padded pitch)
        for src in (bgr, IC.padded(bgr)):
            rgb, gray = ip.process(src)
            check_against_golden(golden, case, rgb, gray, m1, m2)
            assert np.array_equal(rgb, rgb_w) and np.array_equal(gray, gray_w)
        # device in (contiguous and padded), device out; host in, device out; device in, host out
        d_img = torch.from_numpy(bgr).cuda()
        d_pad = torch.zeros((case.rows, case.cols * 3 + 29), dtype=torch.uint8, device="cuda")
        d_pad[:, :case.cols * 3] = d_img.reshape(case.rows, -1)
        d_pad = d_pad[:, :case.cols * 3].view(case.rows, case.cols, 3)
        assert d_pad.stride(0) == case.cols * 3 + 29
        oc, orows = ip.output_size()
        for src in (d_img, d_pad, bgr):
            out = (torch.full((orows, oc, 3), 7, dtype=torch.uint8, device="cuda"), torch.full((orows, oc), 7, dtype=torch.uint8, device="cuda"))
            rgb, gray = ip.process(src, out=out)
            assert rgb is out[0] and gray is out[1]
            assert np.array_equal(rgb.cpu().numpy(), rgb_w) and np.array_equal(gray.cpu().numpy(), gray_w)
        rgb, gray = ip.process(d_pad, out=(np.empty((orows, oc, 3), np.uint8), torch.empty((orows, oc), dtype=torch.uint8)))
        assert np.array_equal(rgb, rgb_w) and np.array_equal(gray.numpy(), gray_w)
        up, rm, cl = ip.last_times()
        assert up >= 0 and rm >= 0 and cl >= 0
    finally:
        ip.close()


def test_device_gray_tracks_as_the_golden_gray(ctx):
    import torch
    from sr_livo_b200 import lio
    case = IC.BY_NAME["ntu"]
    frames = [case.bgr(), np.roll(case.bgr(), (2, 3), axis=(0, 1))]
    want = [R.prepare(f, **case.camera)[1] for f in frames]
    ip = lio.ImageProcessing(ctx, **case.camera)
    oc, orows = ip.output_size()
    rng = np.random.default_rng(3)
    pts = np.stack([rng.uniform(40, oc - 40, 300), rng.uniform(40, orows - 40, 300)], axis=1).astype(np.float32)
    lk_dev = lio.LKOpticalFlowKernel(ctx, **lio.tracker_lk_params())
    lk_host = lio.LKOpticalFlowKernel(ctx, **lio.tracker_lk_params())
    try:
        for f, g in zip(frames, want):
            gray = torch.empty((orows, oc), dtype=torch.uint8, device="cuda")
            rgb = torch.empty((orows, oc, 3), dtype=torch.uint8, device="cuda")
            ip.process(torch.from_numpy(f).cuda(), out=(rgb, gray))
            a = lk_dev.trackImage(gray, pts)
            b = lk_host.trackImage(g, pts)
        assert a[2] == b[2] and a[2] > 100
        assert np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)) and np.array_equal(a[1], b[1])
    finally:
        lk_dev.close(), lk_host.close(), ip.close()


def test_device_rgb_renders_as_the_golden_rgb(ctx):
    import torch
    from sr_livo_b200 import capi, lio
    case = IC.BY_NAME["r3live_212"]
    rgb_w = R.prepare(case.bgr(), **case.camera)[0]
    ip = lio.ImageProcessing(ctx, **case.camera, cols=case.cols, rows=case.rows)
    oc, orows = ip.output_size()
    K = ip.camera_intrinsic()
    rgb = torch.empty((orows, oc, 3), dtype=torch.uint8, device="cuda")
    ip.process(torch.from_numpy(case.bgr()).cuda(), out=(rgb, torch.empty((orows, oc), dtype=torch.uint8, device="cuda")))
    cam = capi.Camera()
    cam.q_camera_world[:] = [0.0, 0.0, 0.0, 1.0]   # (x, y, z, w): the identity
    cam.fx, cam.fy, cam.cx, cam.cy, cam.fov_margin = K[0, 0], K[1, 1], K[0, 2], K[1, 2], 0.01
    cam.cols, cam.rows = oc, orows
    rng = np.random.default_rng(5)
    z = rng.uniform(3.5, 4.5, 600)
    u, v = rng.uniform(0, oc, 600), rng.uniform(0, orows, 600)
    pts = np.stack([(u - K[0, 2]) / K[0, 0] * z, (v - K[1, 2]) / K[1, 1] * z, z], axis=1).astype(np.float32).astype(np.float64)
    out = []
    for img in (rgb, rgb_w):
        cm = lio.ColorVoxelMap(ctx, RC.VOXEL, RC.CAP, 1 << 12, RC.FINE, initial_voxels=64)
        assert cm.addPoints(pts, 1, 1.0, 0.0, True) > 0 and cm.stats()["recent"] > 0
        # a point's first observation only seeds its colour; the second one is fused and counted
        n = cm.renderPointsInRecentVoxel(cam, img, 1.0) + cm.renderPointsInRecentVoxel(cam, img, 2.0)
        out.append((n, *cm.exportColorPoints(1)))
        cm.close()
    ip.close()
    assert out[0][0] == out[1][0] > 100
    assert np.array_equal(out[0][1], out[1][1]) and np.array_equal(out[0][2], out[1][2])


def test_bad_arguments_leave_the_object_usable(ctx):
    from sr_livo_b200 import capi
    L = capi.lib()
    case = IC.BY_NAME["odd_203"]

    def params(**kw):
        cam = dict(case.camera, **kw)
        return capi.ImageParams(cam["image_width"], cam["image_height"], (C.c_double * 9)(*cam["camera_intrinsic"]),
                                (C.c_double * 5)(*cam["camera_dist_coeffs"]))

    h = C.c_void_p()
    bad_create = [(params(), 0, 157), (params(), 203, -1), (params(image_width=0), 203, 157), (params(), 40000, 157),
                  (params(camera_intrinsic=[np.nan] + case.camera["camera_intrinsic"][1:]), 203, 157),
                  (params(camera_dist_coeffs=[np.inf, 0, 0, 0, 0]), 203, 157),
                  (params(camera_intrinsic=[0.0] * 8 + [1.0]), 203, 157),     # no inverse
                  (params(image_width=15, image_height=15), 15, 15)]          # a 15 x 15 output
    for prm, cols, rows in bad_create:
        assert L.srl_image_create(ctx.h, C.byref(prm), cols, rows, C.byref(h)) == capi.SRL_BAD_ARG
        assert not h.value

    assert L.srl_image_create(ctx.h, C.byref(params()), case.cols, case.rows, C.byref(h)) == capi.SRL_OK
    try:
        oc, orows = C.c_int32(0), C.c_int32(0)
        assert L.srl_image_info(h, C.byref(oc), C.byref(orows), None, None, None) == capi.SRL_OK
        bgr = case.bgr()
        rgb, gray = np.empty((orows.value, oc.value, 3), np.uint8), np.empty((orows.value, oc.value), np.uint8)
        p = lambda a: C.c_void_p(a.ctypes.data)
        pitch = case.cols * 3
        assert L.srl_image_last_times(h, None, None, None) == capi.SRL_BAD_ARG
        for args in [(None, case.cols, case.rows, pitch, p(rgb), p(gray)), (p(bgr), case.cols, case.rows, pitch, None, p(gray)),
                     (p(bgr), case.cols, case.rows, pitch, p(rgb), None), (p(bgr), case.cols + 1, case.rows, pitch + 3, p(rgb), p(gray)),
                     (p(bgr), case.cols, case.rows - 1, pitch, p(rgb), p(gray)), (p(bgr), case.cols, case.rows, pitch - 1, p(rgb), p(gray))]:
            assert L.srl_image_process(h, *args) == capi.SRL_BAD_ARG
        assert L.srl_image_process(h, p(bgr), case.cols, case.rows, pitch, p(rgb), p(gray)) == capi.SRL_OK
        rgb_w, gray_w = _want(case)[:2]
        assert np.array_equal(rgb, rgb_w) and np.array_equal(gray, gray_w)
    finally:
        L.srl_image_destroy(h)
