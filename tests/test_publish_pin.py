"""The published maps, the reference's own code against the oracle, every field bit for bit.

Left: oracle/_ref/libsrl_publish_ref.so, the reference's addPointsToMap / pubColorPoints / saveColorPoints compiled from its
sources with the clouds they hand to pcl::toROSMsg and pcl::io::savePCDFileBinary captured (oracle/publish.mk).  Right: the
oracle's restatement (orc_map_add_points_published, orc_color_export), which the GPU tests use as their yardstick.

CPU only; skipped when the reference library was not built.
"""
import numpy as np
import pytest

from oracle import publish_oracle as O

import publish_ref as PR
from color_map_cases import FINE, SIZE, camera, sweep
from publish_cases import CAP, MIN_DIST, lio_stream, render_images, small_color_points

pytestmark = pytest.mark.skipif(not PR.available(), reason="oracle/_ref/libsrl_publish_ref.so not built (needs the reference tree)")


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


@pytest.mark.parametrize("voxel_size", [1.0, 0.5])
@pytest.mark.parametrize("min_num_points", [0, 3])
def test_registered_cloud_reference_equals_oracle(voxel_size, min_num_points):
    ref, om = PR.PublishReference(), O.OracleMap()
    stream = lio_stream(seed=int(40 * voxel_size) + min_num_points, voxel_size=voxel_size)
    published = []
    for k, (pts, tz) in enumerate(stream):
        mnp = 0 if k == 0 else min_num_points                      # the first frame fills the map
        a_added, a = ref.add_points_to_map(pts, tz, voxel_size, CAP, MIN_DIST, mnp)
        b_added, b = om.add_points_published(pts, tz, voxel_size, CAP, MIN_DIST, mnp)
        assert a_added == b_added
        assert a.shape == b.shape and np.array_equal(bits(a), bits(b)), k
        published.append((a_added, a.shape[0]))
    # the stream does what it is meant to: points published, created voxels not, and with min_num_points = 3 nothing created
    assert published[0][1] > 0 and all(n_pub <= n_add for n_add, n_pub in published)
    if min_num_points == 0:
        assert any(n_pub < n_add for n_add, n_pub in published[1:])
    else:
        assert all(n_pub == n_add for n_add, n_pub in published[1:])
    keys, counts, _ = om.snapshot(CAP)
    assert (counts == CAP).any()
    # intensity is 50 * (z - tz) evaluated in FP64 and rounded once
    pts, tz = stream[-1]
    z = b[:, 2].astype(np.float64)
    assert np.array_equal(b[:, 3], (50.0 * (z - tz)).astype(np.float32))


def _color_pair(cap, sweeps, renders):
    ref = PR.PublishReference()
    oc = O.OracleColorMap(voxel_size=SIZE, max_num_points_in_voxel=cap, min_distance_points=FINE)
    for s, pts in enumerate(sweeps):
        t_end, t_proc = 1.0 + 0.1 * s, 1.0 * s
        ref.add_points_to_map(pts, 0.0, color_voxel_size=SIZE, color_max_points=cap, color_min_distance=FINE, add_point_step=1,
                              time_sweep_end=t_end, time_last_process=t_proc, to_rendering=True)
        oc.add_points(pts, add_point_step=1, time_sweep_end=t_end, time_last_process=t_proc, to_rendering=True)
        for k, img in enumerate(render_images(100 * cap + s, renders)):
            cam, obs = camera((0.02 * k, 0.0, 0.0)), t_end + 0.01 * (k + 1)
            assert ref.color_render(cam, img, obs) == oc.render(cam, img, obs)
    assert ref.num_rgb_points() == oc.num_rgb_points()
    return ref, oc


def _compare_exports(ref, oc, min_views_list):
    for order in (0, 1):
        for mv in min_views_list:
            a, b = ref.export(mv, order), oc.export(mv, order)
            assert np.array_equal(bits(a[0]), bits(b[0])) and np.array_equal(a[1], b[1]), (order, mv)


@pytest.mark.parametrize("cap", [50, 100])
def test_color_map_export_reference_equals_oracle(cap):
    rng = np.random.default_rng(cap)
    first = sweep(seed=11 * cap)
    ref, oc = _color_pair(cap, [first, first + rng.normal(0, 0.003, first.shape)], renders=2)
    top = oc.max_n_rgb()
    assert top >= 3
    _compare_exports(ref, oc, [-1, 0, 1, 3, top + 1])
    n = oc.num_rgb_points()
    assert len(oc.export(-1, 0)[0]) == n and len(oc.export(-1, 1)[0]) == n - 1      # save order skips index 0
    assert 0 < len(oc.export(1, 0)[0]) < n and len(oc.export(top + 1, 0)[0]) == 0
    # publish order is the reverse of the save order plus index 0
    p, s = oc.export(0, 0), oc.export(0, 1)
    assert np.array_equal(p[0][1:][::-1], s[0]) and np.array_equal(p[1][1:][::-1], s[1])


@pytest.mark.parametrize("k", [0, 1, 2])
def test_color_map_export_of_tiny_maps(k):
    """0, 1 and 2 rgb points: the save order never reaches index 0, so 0 or 1 point saves nothing."""
    ref, oc = _color_pair(50, [small_color_points(k)], renders=1)
    _compare_exports(ref, oc, [-1, 0, 1])
    assert len(oc.export(-1, 1)[0]) == max(k - 1, 0) and len(oc.export(-1, 0)[0]) == k
