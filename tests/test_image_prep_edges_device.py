"""The camera image preparation on the GPU (srl_image_*) on the edge cases of image_prep_edge_cases, bit for bit: the device
maps, gray_image and rgb_image against the restatement (image_prep_reference) and, for every case whose outputs OpenCV
builds agree on, against tests/golden/image_prep_edges.npz (map2 at the unsaturated entries only), from host and device
inputs.  The overflow cameras hold k_img_map to OpenCV's saturating int16 pack; the tie-heavy map is held to the
restatement alone."""
import numpy as np
import pytest

import image_prep_edge_cases as EC
import image_prep_reference as R
from test_image_prep_edges_pin import GOLDEN, check_against_golden

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


@pytest.mark.parametrize("name", [c.name for c in EC.CASES])
def test_maps_and_images_equal_golden_and_restatement(ctx, golden, name):
    import torch
    from sr_livo_b200 import lio
    case = EC.BY_NAME[name]
    bgr = case.bgr()
    rgb_w, gray_w, m1_w, m2_w, s_w, K_w, t_w = R.prepare(bgr, **case.camera)
    ip = lio.ImageProcessing(ctx, **case.camera, cols=case.cols, rows=case.rows)
    try:
        assert ip.output_size() == (gray_w.shape[1], gray_w.shape[0])
        assert ip.tiles() == t_w and ip.scale_factor() == s_w
        m1, m2 = ip.maps()
        sat = R.saturated(m1_w)
        assert np.array_equal(m1, m1_w), (int((m1 != m1_w).any(-1).sum()), int(sat.sum()))
        assert np.array_equal(m2, m2_w), int((m2 != m2_w).sum())
        oc, orows = ip.output_size()
        d_img = torch.from_numpy(bgr).cuda()
        d_pad = torch.zeros((case.rows, case.cols * 3 + 29), dtype=torch.uint8, device="cuda")
        d_pad[:, :case.cols * 3] = d_img.reshape(case.rows, -1)
        d_pad = d_pad[:, :case.cols * 3].view(case.rows, case.cols, 3)
        outs = []
        for src in (bgr, d_img, d_pad):
            rgb, gray = ip.process(src)
            outs.append((rgb, gray))
            out = (torch.full((orows, oc, 3), 7, dtype=torch.uint8, device="cuda"), torch.full((orows, oc), 7, dtype=torch.uint8, device="cuda"))
            rgb_d, gray_d = ip.process(src, out=out)
            outs.append((rgb_d.cpu().numpy(), gray_d.cpu().numpy()))
        for rgb, gray in outs:
            assert np.array_equal(gray, gray_w), int((gray != gray_w).sum())
            assert np.array_equal(rgb, rgb_w), int((rgb != rgb_w).any(-1).sum())
            if case.opencv:
                check_against_golden(golden, case, rgb, gray, m1, m2)
    finally:
        ip.close()
