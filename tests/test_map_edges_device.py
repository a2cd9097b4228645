"""The LIO voxel map at its edges on the GPU: for every case of tests/map_edge_cases.py and every source of points (host
array, device tensor, the resident sweep under a pose), the device map equals the plain restatement (tests/map_reference.py)
after every operation: stats, the downloaded contents and order inside each voxel, points stored, the published cloud bit
for bit and voxels evicted.  Eviction keeps the surviving voxels in their block order.  After the probe-chain, growth and
eviction cases, the scan-matching pass over keypoints in the chained voxels and next to voxels +-32765 and +-32766 equals
the oracle's, neighbour ids bit for bit.
"""
import numpy as np
import pytest

from oracle import oracle_py as O

import map_edge_cases as E
from map_reference import MapRef
from sweep_prep_reference import transform_point_fp64
from test_map_edges_pin import assert_same_map, bits, map_dict

pytestmark = pytest.mark.gpu
CASES = {c.name: c for c in E.all_cases()}
BIG = 2 ** 31 - 1
# the sweep source's pose.  The sweep holds world - POSE_T, and the restatement is fed what the restated transformPoint makes
# of it (equal to the crafted world points wherever the subtraction was exact)
POSE_Q = np.array([0.0, 0.0, 0.0, 1.0])
POSE_T = np.array([0.5, -0.25, 0.125])


def _insert(L, mode, xyz, md, mnp, tz):
    """(added, cloud, the world points the restatement is to be fed)"""
    import torch
    if mode == "host":
        added, cloud = L.addPointsToMapPublished(xyz, tz, md, mnp)
        return added, cloud, xyz, tz
    if mode == "device":
        added, cloud = L.addPointsToMapPublished(torch.from_numpy(np.ascontiguousarray(xyz)).cuda(), tz, md, mnp)
        assert cloud.is_cuda
        return added, cloud.cpu().numpy(), xyz, tz
    raw = xyz - POSE_T
    L.setKeypoints(raw)
    added, cloud = L.addSweepToMapPublished(POSE_Q, POSE_T, md, mnp)
    world = transform_point_fp64(raw, POSE_Q, POSE_T, np.eye(3), np.zeros(3))
    return added, cloud, world, float(POSE_T[2])


def _assert_pass_equal(g, o):
    assert o.num_fragile == 0
    assert np.array_equal(g.status, o.status)
    full = o.status >= 1
    assert np.array_equal(g.nbr[full], o.nbr[full])
    assert np.array_equal(g.nbr_dist[full], o.nbr_dist[full])
    assert g.num_residuals == o.num_residuals and g.num_full_neighborhoods == o.num_full_neighborhoods
    return int(full.sum())


@pytest.mark.parametrize("mode", ["host", "device", "sweep"])
@pytest.mark.parametrize("name", list(CASES))
def test_device_map_equals_restatement(name, mode):
    from sr_livo_b200 import lio
    case = CASES[name]
    L = lio.LioOptimization(max_voxels=1 << 14, sweep_capacity=1 << 13, size_voxel_map=case.size, max_num_points_in_voxel=case.cap,
                            initial_voxels=case.initial_voxels)
    m = MapRef(case.size, case.cap)
    try:
        for i, op in enumerate(case.ops):
            if op[0] == "upload":
                L.voxel_map.upload(*op[1:])
                m.load(*op[1:])
            elif op[0] == "insert":
                added, cloud, world, tz = _insert(L, mode, *op[1:])
                want_added, want_cloud = m.add_points(world, op[2], op[3], tz)
                assert added == want_added, (i, added, want_added)
                assert cloud.shape == want_cloud.shape and np.array_equal(bits(cloud), bits(want_cloud)), i
            else:
                before = [tuple(k) for k in L.voxel_map.download()[0].tolist()]
                assert L.removePointsFarFromLocation(op[1], op[2]) == m.remove_far(op[1], op[2]), i
                after = [tuple(k) for k in L.voxel_map.download()[0].tolist()]
                assert after == [k for k in before if k in m.vox], i     # survivors keep their block order
            assert L.voxel_map.stats() == (len(m.vox), m.num_points), i
            assert_same_map(map_dict(*L.voxel_map.download()), m.as_dict(), i)
        if case.probes is not None and mode == "host":
            om = O.OracleMap()
            keys = np.array(list(m.vox), np.int16).reshape(-1, 3)
            xyz = np.zeros((keys.shape[0], case.cap, 3), np.float32)
            for v, pts in enumerate(m.vox.values()):
                xyz[v, :len(pts)] = pts
            om.load(keys, np.array([len(p) for p in m.vox.values()], np.int32), xyz)
            L.setKeypoints(case.probes)
            q, t0 = np.array([0.0, 0.0, 0.0, 1.0]), np.zeros(3)
            n_full, edge_ids = 0, 0
            for kw in (dict(max_num_residuals=BIG), dict(max_num_residuals=BIG, frame_id=5)):   # nb = 1, then nb = 2
                g = L.buildPlaneResiduals(lio.r3live_params(**kw), q, t0, t0, debug=True)
                o = om.build_plane_residuals(case.probes, q, t0, t0, O.r3live_params(**kw), debug=True)
                n_full += _assert_pass_equal(g, o)
                edge_ids += int(np.isin(np.abs(o.nbr[o.status >= 1][..., 0].astype(np.int32)), (32765, 32766)).sum())
            assert n_full > 0 and edge_ids > 0       # neighbours found in voxels +-32765 and +-32766
    finally:
        L.close()
