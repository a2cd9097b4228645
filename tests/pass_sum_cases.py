"""Scenes and sizes for the pass-sum tests (tests/test_pass_sums_device.py).

Keypoints are small_world map points on the ground and the façades, seen from a pose in one corner of the 80 m map so
their ranges span 1.2 .. ~110 m and the rotational columns of J two decades.  Each base point is first moved onto the
plane the pass fits to its neighbourhood, then split into a twin pair at +-delta (2 .. 10 mm) along that plane's
normal: at the pose the keypoints were drawn from, the twins' J are equal and their h opposite, so J^T h cancels to
far below its terms.  Only pairs whose both members are accepted (status 2) at every pose and neighbourhood the tests
use, and whose twins share their neighbour lists, are kept; any resample of them is then accepted keypoint by keypoint.
"""
from __future__ import annotations

import numpy as np

from sr_livo_b200 import synth

BIG = 2 ** 31 - 1
MAP_EXTENT, MAP_DENSITY, MAP_SEED = 80.0, 60.0, 1       # the small_world map

POSE_Q = synth.quat_from_rotvec([0.01, -0.02, 0.7])      # the pose the keypoints are drawn from
POSE_T = np.array([-37.3, -36.1, 1.2])
OFFSET_Q = synth.quat_mul(POSE_Q, synth.quat_from_rotvec([3e-4, -2e-4, 4e-4]))   # ~0.03 deg, ~1.3 cm away
OFFSET_T = POSE_T + np.array([0.009, -0.007, 0.006])
T_LAST = POSE_T - synth.quat_to_rot(POSE_Q) @ np.array([1.0, 0.0, 0.0])

# k1_fit (split form): one group of 32 per warp, 4 warps per block, 32 blocks per chunk, 2048 blocks, grid-stride beyond
FIT_SIZES = [1, 31, 32, 33, 127, 128, 129,
             4095, 4096, 4097,            # 4097: the second chunk is one block holding one keypoint
             8193, 131072,                # 131072: 32 chunks
             262143, 262144, 262145,      # 262145: the second grid-stride round holds one keypoint
             266241,
             524289]                      # 64 chunks, two rounds
FAST_SIZES = [4097, 262145]


def assoc_sizes(sm_count: int) -> list[int]:
    """k1_assoc's grid is min(groups, sm_count * per_sm, 2048); per_sm is the library's occupancy query of the instance
    (1 to 4 blocks of 256 threads per SM), which a test cannot read, so every product p * per_sm for p = 1..4 and all
    four candidates is covered: one group short of, at, just past and one group past each grid-stride boundary."""
    mult = sorted({p * q for p in range(1, 5) for q in range(1, 5)})
    return sorted({1, 33} | {32 * sm_count * m + d for m in mult for d in (-1, 0, 1, 33)})


def map_points() -> np.ndarray:
    return synth.sample_map_points(MAP_EXTENT, MAP_DENSITY, seed=MAP_SEED)


def to_raw(world, q=POSE_Q, t=POSE_T) -> np.ndarray:
    """LiDAR-frame points of world points under pose (q, t) (R_il = I, t_il = 0)."""
    return np.ascontiguousarray((np.asarray(world) - t) @ synth.quat_to_rot(q))


def to_world(raw, q=POSE_Q, t=POSE_T) -> np.ndarray:
    return np.asarray(raw) @ synth.quat_to_rot(q).T + t


def surface_points(pts, rng, per_bin: int = 5000) -> np.ndarray:
    """Map points on the ground and the façades (away from edges and corners), moved by up to 1 cm along the surface
    normal, balanced over 8 logarithmic range bins from the pose."""
    x, y, z = pts[:, 0], pts[:, 1], pts[:, 2]
    fx, fy = np.mod(x, synth.PITCH), np.mod(y, synth.PITCH)
    gz = synth.ground_h(x, y)
    inside = lambda f: (f > synth.B_LO + 0.3) & (f < synth.B_HI - 0.3)   # noqa: E731
    foot = (fx > synth.B_LO - 0.3) & (fx < synth.B_HI + 0.3) & (fy > synth.B_LO - 0.3) & (fy < synth.B_HI + 0.3)
    ground = ~foot & (np.abs(z - gz) < 0.01)
    height = (z - gz > 0.3) & (z - gz < synth.B_H - 0.3)
    wall_x = height & inside(fy) & ((np.abs(fx - synth.B_LO) < 0.01) | (np.abs(fx - synth.B_HI) < 0.01))
    wall_y = height & inside(fx) & ((np.abs(fy - synth.B_LO) < 0.01) | (np.abs(fy - synth.B_HI) < 0.01))
    nrm = np.zeros_like(pts)
    nrm[ground] = np.stack([-0.006 * np.cos(0.3 * x[ground]), 0.004 * np.sin(0.2 * y[ground]), np.ones(ground.sum())], 1)
    nrm[wall_x, 0] = 1.0
    nrm[wall_y, 1] = 1.0
    keep = ground | wall_x | wall_y
    p = pts[keep] + rng.uniform(-0.01, 0.01, (int(keep.sum()), 1)) * (nrm[keep] / np.linalg.norm(nrm[keep], axis=1, keepdims=True))
    rng_m = np.linalg.norm(p - POSE_T, axis=1)
    edges = np.geomspace(1.0, 120.0, 9)
    out = []
    for lo, hi in zip(edges[:-1], edges[1:]):
        idx = np.flatnonzero((rng_m >= lo) & (rng_m < hi))
        out.append(p[rng.permutation(idx)[:per_bin]])
    return np.concatenate(out)


def twin_pool(L, seed: int = 5) -> np.ndarray:
    """(m, 2, 3) raw keypoints: twin pairs on their fitted planes, accepted at every pose / neighbourhood the tests use."""
    from sr_livo_b200 import lio
    rng = np.random.default_rng(seed)
    base = surface_points(map_points(), rng)
    prm1 = lio.r3live_params(max_num_residuals=BIG)
    L.setKeypoints(to_raw(base))
    g = L.buildPlaneResiduals(prm1, POSE_Q, POSE_T, T_LAST, debug=True)
    ok = g.status == 2
    base, plane = base[ok], g.plane[ok]
    nrm, dist = plane[:, 3:6], plane[:, 13]
    on_plane = base - dist[:, None] * nrm
    delta = rng.uniform(0.002, 0.01, (on_plane.shape[0], 1))
    twins = np.stack([on_plane + delta * nrm, on_plane - delta * nrm], 1)            # (m, 2, 3) world
    for _ in range(2):   # centre every pair on the plane its twins fit (their neighbourhood may differ from the base's)
        L.setKeypoints(to_raw(twins.reshape(-1, 3)))
        r = L.buildPlaneResiduals(prm1, POSE_Q, POSE_T, T_LAST, debug=True)
        pl = r.plane.reshape(-1, 2, 16)
        nbr = r.nbr.reshape(-1, 2, r.nbr.shape[1], 4)
        ok = (r.status.reshape(-1, 2) == 2).all(1) & (nbr[:, 0] == nbr[:, 1]).all(axis=(1, 2))
        twins, pl = twins[ok], pl[ok]
        mid = 0.5 * (pl[:, 0, 13] + pl[:, 1, 13])
        twins = twins - mid[:, None, None] * pl[:, :1, 3:6]
    raw = to_raw(twins.reshape(-1, 3)).reshape(-1, 2, 3)
    L.setKeypoints(raw.reshape(-1, 3))
    keep = np.ones(raw.shape[0], bool)
    for q, t, kw in ((POSE_Q, POSE_T, {}), (OFFSET_Q, OFFSET_T, {}), (POSE_Q, POSE_T, dict(frame_id=5)), (OFFSET_Q, OFFSET_T, dict(frame_id=5))):
        r = L.buildPlaneResiduals(lio.r3live_params(max_num_residuals=BIG, **kw), q, t, T_LAST, debug=True)
        keep &= (r.status.reshape(-1, 2) == 2).all(1)
        if not kw and q is POSE_Q:
            nbr = r.nbr.reshape(-1, 2, r.nbr.shape[1], 4)
            keep &= (nbr[:, 0] == nbr[:, 1]).all(axis=(1, 2))
    return np.ascontiguousarray(raw[keep])


def resample(pool, n: int, seed: int) -> np.ndarray:
    """n keypoints drawn with replacement from the twins (either member)."""
    rng = np.random.default_rng(seed)
    return np.ascontiguousarray(pool[rng.integers(0, pool.shape[0], n), rng.integers(0, 2, n)])


def cancelling(pool, pairs: int, seed: int) -> np.ndarray:
    """`pairs` twin pairs, both members, shuffled: at POSE their J^T h cancels."""
    rng = np.random.default_rng(seed)
    raw = pool[rng.integers(0, pool.shape[0], pairs)].reshape(-1, 3)
    return np.ascontiguousarray(raw[rng.permutation(raw.shape[0])])


def void_points(n: int, seed: int) -> np.ndarray:
    """Raw keypoints 60 m above the map: no voxel within reach, status 0."""
    rng = np.random.default_rng(seed)
    w = np.stack([rng.uniform(-35, 35, n), rng.uniform(-35, 35, n), rng.uniform(60, 70, n)], 1)
    return to_raw(w)


def capped_layout(pool, n: int, accepted_at, seed: int) -> np.ndarray:
    """n keypoints in their own order: twins at the indices `accepted_at`, points without a neighbourhood elsewhere."""
    raw = void_points(n, seed)
    acc = np.asarray(sorted(accepted_at))
    raw[acc] = resample(pool, acc.size, seed + 1)
    return raw
