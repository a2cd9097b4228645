"""Scenes for the colour map at the shipped map_options (0.1 m voxels, 50 / 100 points, 0.01 m fine cells).

Every scene is seeded and built from float64 world points:
  * dense surfaces: far more than 128 points per 0.1 m voxel, so every voxel fills up and later points are refused;
  * clusters at x = +-400 m, where the 0.01 m fine key wraps (|x / 0.01| > 32767);
  * pairs 655.36 m apart (2^16 fine cells: same fine key) and 6553.6 m apart (2^16 voxels: same voxel key);
  * points past +-3276.8 m, where the voxel key itself wraps.
The rule they pin: a key is static_cast<short>(q) as the reference compiles on x86-64, i.e. the low 16 bits of the int32
truncation of q = double(float(x)) / size (`wrap_key`).
"""
import numpy as np

SIZE, FINE = 0.1, 0.01


def wrap_key(xyz, size):
    """static_cast<short>(double(float(x)) / size) for |q| < 2^31: int32 truncation, then the low 16 bits."""
    q = np.asarray(xyz, np.float32).astype(np.float64) / size
    assert np.all(np.abs(q) < 2.0 ** 31)
    return (np.trunc(q).astype(np.int64) & 0xFFFF).astype(np.uint16).view(np.int16)


def patch(rng, n, center, half=0.35, thick=0.002):
    """a dense, nearly flat square facing the camera (z = depth)."""
    c = np.asarray(center, np.float64)
    return np.stack([rng.uniform(-half, half, n) + c[0], rng.uniform(-half, half, n) + c[1], rng.normal(0, thick, n) + c[2]], axis=1)


def sweep(seed, n_dense=20000):
    """one registered frame: the dense surfaces near the origin and at +-400 m, aliasing pairs and far points, shuffled."""
    rng = np.random.default_rng(seed)
    near = patch(rng, n_dense, (0.0, 0.0, 4.03))
    far_pos = patch(rng, n_dense // 2, (400.0, 0.0, 4.03))
    far_neg = patch(rng, n_dense // 4, (-400.0, 0.2, 4.03))
    base = patch(rng, 400, (0.1, -0.1, 4.03), half=0.2)
    fine_alias = base + [655.36, 0.0, 0.0]                  # same fine cell as `base` (2^16 cells of 0.01 m)
    vox_alias = base[:200] + [6553.6, 0.0, 0.0]            # same voxel as `base` (2^16 voxels of 0.1 m)
    beyond = np.concatenate([patch(rng, 300, (3300.0, -3400.0, 4.03), half=0.2), patch(rng, 300, (-5000.0, 4000.0, -3500.0), half=0.2),
                             patch(rng, 200, (-400.0, -1000.0, 9000.0), half=0.2)])
    pts = np.concatenate([near, far_pos, far_neg, base, fine_alias, vox_alias, beyond])
    return pts[rng.permutation(pts.shape[0])]


def voxel_exact_count(rng, cap, n_vox=24, center=(0.0, 0.0, 4.0)):
    """n_vox voxels on a row, each offered exactly cap points (even voxels) or cap + 1 points (odd voxels) on a grid inside
    the voxel, 4 mm clear of its faces."""
    out = []
    for v in range(n_vox):
        k = cap + (v & 1)
        g = int(np.ceil(np.sqrt(k)))
        ij = np.array([(i, j) for i in range(g) for j in range(g)][:k], np.float64)
        x0 = center[0] + 0.1 * v + 0.004
        p = np.stack([x0 + ij[:, 0] * (0.092 / g), center[1] + 0.004 + ij[:, 1] * (0.092 / g), np.full(k, center[2] + 0.05)], axis=1)
        out.append(p)
    pts = np.concatenate(out)
    return pts[rng.permutation(pts.shape[0])]


def camera(position, rows=480, cols=640):
    """identity rotation, camera at `position`, 640x480: the 15 doubles the oracle and the reference take."""
    pos = np.asarray(position, np.float64)
    q = np.array([0.0, 0.0, 0.0, 1.0])
    fx, fy, cx, cy, fov = 300.0, 300.0, cols / 2.0 + 0.25, rows / 2.0 - 0.25, 0.0001
    return np.concatenate([q, -pos, pos, [fx, fy, cx, cy, fov]])


def model_lists(sweeps_with_steps, cap):
    """addPointToColorMap's bookkeeping in plain Python with the `wrap_key` rule: voxel contents counts, rgb_points_vec as
    (voxel key, index in block) in order.  Agreement with the oracle pins the oracle's keys to the formula."""
    counts, fine, rgb = {}, set(), []
    for pts, step in sweeps_with_steps:
        sel = np.asarray(pts)[::step]
        vk, fk = wrap_key(sel, SIZE), wrap_key(sel, FINE)
        for v, f in zip(map(tuple, vk.tolist()), map(tuple, fk.tolist())):
            c = counts.get(v, 0)
            if c >= cap:
                continue
            counts[v] = c + 1
            if f not in fine:
                fine.add(f)
                rgb.append(v + (c,))
    return counts, np.array(rgb, np.int16).reshape(-1, 4)
