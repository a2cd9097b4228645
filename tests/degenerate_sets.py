"""Crafted neighbourhoods for the per-keypoint plane fit, and their truth in extended precision.

A map of isolated 20-point clusters, one per voxel and at least 4 voxels apart, so that a keypoint's 27-voxel search sees
exactly its own cluster.  Every cluster belongs to a class that stresses one branch of the symmetric 3x3 eigensolver
(exact planes, discs, poles, edges on both sides of the closed form's gap cut, near-isotropic sets, rank 1 / rank 0, a
spread of a few FP32 ulps, coordinates near the +-32767 key limit and inside the double-width cell 0).  The maps are
loaded with `voxel_map.upload` (keys / counts / FP32 xyz), the pose is the identity, so a keypoint's body and world
positions are its raw coordinates.

`truth()` restates computeNeighborhoodDistribution, the normal flip, the weight, the plane offset through the nearest
point, the signed distance and the Jacobian (src/optimize.cpp:42-101, 316-353) with mpmath at 50 digits, from the FP32
points as stored: barycenter and scatter are exact, the eigen-decomposition is accurate far beyond FP64.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import mpmath
import numpy as np

EPS = 2.0 ** -52
K = 20
# r3live.yaml values the pass uses (srl_icp_params_r3live)
DMAX = 0.3
LAMBDA_W, LAMBDA_N = 0.9, 0.1
IDENTITY_Q = np.array([0.0, 0.0, 0.0, 1.0])
ZERO_T = np.zeros(3)
# far along +z and off-axis: the flip of every normal that is not nearly horizontal is decided by a wide margin
T_LAST = np.array([137.0, -291.0, 2411.0])


@dataclass
class Cluster:
    name: str                   # class, e.g. "edge_gap_1.1e-3"
    key: tuple                  # voxel key
    pts: np.ndarray             # (20, 3) float32, as stored in the map
    kps: list = field(default_factory=list)   # keypoints (raw = world under the identity pose), float64 (3,)
    lam: tuple | None = None    # prescribed scatter eigenvalues (before FP32 rounding), if any


def random_rotation(rng) -> np.ndarray:
    q, r = np.linalg.qr(rng.normal(size=(3, 3)))
    q = q * np.sign(np.diag(r))
    if np.linalg.det(q) < 0:
        q[:, 0] = -q[:, 0]
    return q


def _whitened(rng, n=K) -> np.ndarray:
    """n x 3, columns centred and orthonormal: its scatter matrix is the identity."""
    while True:
        a = rng.normal(size=(n, 3))
        a -= a.mean(axis=0)
        q, _ = np.linalg.qr(a)
        if np.abs(q).max() < 0.62:
            return q


def _shaped(rng, lam, rot, centre) -> np.ndarray:
    """20 points whose scatter matrix is rot diag(lam) rot^T before rounding to FP32, around `centre`."""
    for _ in range(200):
        local = _whitened(rng) * np.sqrt(np.asarray(lam, np.float64))
        p = local @ rot.T
        if np.abs(p).max() < 0.45:
            return (p + centre).astype(np.float32)
    raise RuntimeError("could not fit the cluster inside its voxel")


def _centre(key):
    # voxel key -> centre; key 0 is the double-width cell (-1, 1) of trunc()
    return np.array([0.0 if k == 0 else k + (0.5 if k > 0 else -0.5) for k in key])


def _dyadic(rng, n, scale_bits=10, lo=-300, hi=300):
    return rng.integers(lo, hi, n).astype(np.float64) * 2.0 ** -scale_bits


def _pole_axis_aligned(rng, centre):
    """4-fold symmetric about the z axis with dyadic offsets: scatter diag(s, s, t) exactly, s << t (two smallest equal)."""
    pts = []
    zs = np.array([-0.375, -0.1875, 0.0, 0.1875, 0.375])
    for g in range(5):
        u, v = (rng.integers(1, 20, 2) * 2.0 ** -10)
        for (x, y) in ((u, v), (-v, u), (-u, -v), (v, -u)):
            pts.append((x, y, zs[g]))
    return (np.array(pts) + centre).astype(np.float32)


def _isotropic_axis_aligned(centre, a=0.25, c=0.125):
    """cube corners (+-a)^3 and the 12 edge midpoints: scatter (8a^2 + 8c^2) I exactly."""
    pts = [(sx * a, sy * a, sz * a) for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)]
    for i in range(3):
        for s1 in (-1, 1):
            for s2 in (-1, 1):
                p = [0.0, 0.0, 0.0]
                p[(i + 1) % 3] = s1 * c
                p[(i + 2) % 3] = s2 * c
                pts.append(tuple(p))
    return (np.array(pts) + centre).astype(np.float32)


def _zplane(rng, centre):
    x, y = _dyadic(rng, K, 10), _dyadic(rng, K, 10)
    return (np.stack([x, y, np.zeros(K)], 1) + centre).astype(np.float32)


def _rank1(rng, centre, rot=None):
    d = np.array([0.3125, 0.0, 0.0]) if rot is None else rot @ np.array([0.3, 0.0, 0.0])
    base = np.array([-0.0625, 0.0, 0.0]) if rot is None else rot @ np.array([-0.06, 0.01, 0.0])
    p = np.repeat((centre + base)[None], K, axis=0)
    p[7] = centre + base + d
    return p.astype(np.float32)


def _ulp_spread(rng, centre):
    c32 = centre.astype(np.float32)
    ulp = np.spacing(np.abs(c32)).astype(np.float64)
    steps = rng.integers(-3, 4, (K, 3)).astype(np.float64)
    steps[0] = [3, -2, 1]            # never all equal
    return (c32.astype(np.float64) + steps * ulp).astype(np.float32)


EDGE_GAPS = (0.5e-3, 0.9e-3, 1.1e-3, 2e-3)


def class_specs():
    """(name, builder(rng, centre) -> (pts, lam)) for every class; rotated variants draw a seeded rotation."""
    L = 0.25
    specs = [
        ("zplane", lambda rng, c: (_zplane(rng, c), None)),
        ("tilted_plane", lambda rng, c: (_shaped(rng, (0.0, 0.1, L), random_rotation(rng), c), (0.0, 0.1, L))),
        ("disc", lambda rng, c: (_shaped(rng, (0.002, L, L), np.eye(3), c), (0.002, L, L))),
        ("disc_rotated", lambda rng, c: (_shaped(rng, (0.002, L, L), random_rotation(rng), c), (0.002, L, L))),
        ("pole", lambda rng, c: (_pole_axis_aligned(rng, c), None)),
        ("pole_rotated", lambda rng, c: (_shaped(rng, (0.002, 0.002, L), random_rotation(rng), c), (0.002, 0.002, L))),
        ("isotropic", lambda rng, c: (_isotropic_axis_aligned(c), None)),
        ("isotropic_rotated", lambda rng, c: (_shaped(rng, (0.1, 0.1, 0.1), random_rotation(rng), c), (0.1, 0.1, 0.1))),
        ("rank1", lambda rng, c: (_rank1(rng, c), None)),
        ("rank1_rotated", lambda rng, c: (_rank1(rng, c, random_rotation(rng)), None)),
        ("ulp_spread", lambda rng, c: (_ulp_spread(rng, c), None)),
    ]
    for g in EDGE_GAPS:
        lmin = 0.002
        lam = (lmin, lmin + g * (L - lmin), L)
        specs.append((f"edge_gap_{g:.1e}", lambda rng, c, lam=lam: (_shaped(rng, lam, random_rotation(rng), c), lam)))
    for i in range(6):
        specs.append((f"random_{i}", lambda rng, c: (lambda lam: (_shaped(rng, lam, random_rotation(rng), c), lam))(
            tuple(np.sort(rng.uniform(0.02, L, 3))))))
    return specs


# classes whose normal is undefined or nearly so (exactly or numerically repeated smallest eigenvalue)
UNDEFINED_NORMAL = ("pole", "pole_rotated", "isotropic", "isotropic_rotated", "rank1", "rank1_rotated")


def nan_world(seed=7, n_good_clusters=30, kps_per_cluster=40):
    """Well-conditioned clusters with many keypoints each, plus one rank-0 cluster (20 copies of one point: zero scatter,
    a2D = 0 / 0 = NaN).  Returns (clusters, good keypoints, NaN keypoint within dmax of the point -- accepted whatever
    normal the zero matrix yields --, NaN keypoint 0.45 m from it along +x -- the normal the eigensolvers give the zero
    matrix, flipped towards T_LAST -- hence rejected)."""
    rng = np.random.default_rng(seed)
    clusters = []
    for i in range(n_good_clusters):
        key = (8 + 4 * (i % 6), 8 + 4 * (i // 6), 4)
        lam = tuple(np.sort(rng.uniform(0.02, 0.25, 3)))
        clusters.append(Cluster(f"random_{i}", key, _shaped(rng, lam, random_rotation(rng), _centre(key)), lam=lam))
    good = []
    for cl in clusters:
        cl.kps = [_keypoint(rng, cl, 0.12) for _ in range(kps_per_cluster)]
        good += cl.kps
    key0 = (60, 8, 4)
    p = (_centre(key0) + [0.0625, -0.125, 0.03125]).astype(np.float32)
    clusters.append(Cluster("rank0", key0, np.repeat(p[None], K, axis=0)))
    p = p.astype(np.float64)
    return clusters, np.array(good), p + [0.05, 0.03, -0.02], p + [0.45, 0.02, 0.03]


def build_clusters(seed=0, far=True, cell0=True, kps_per_cluster=6) -> list[Cluster]:
    """One cluster per (class, placement): placements at moderate coordinates, near the key limit and in cell 0."""
    rng = np.random.default_rng(seed)
    out = []
    grid = iter([(8 + 4 * a, 8 + 4 * b, 4 + 4 * c) for a in range(8) for b in range(8) for c in range(4)])
    specs = class_specs()
    for name, fn in specs:
        key = next(grid)
        pts, lam = fn(rng, _centre(key))
        out.append(Cluster(name, key, pts, lam=lam))
    by_name = dict(specs)
    if far:   # the key limit (+-32767) and a large FP32 ulp (2^-9 m)
        for key, name in (((31990, -31990, 17), "tilted_plane"), ((-31990, 100, 31990), "disc_rotated"),
                          ((31990, 31990, -31990), "random_0")):
            pts, lam = by_name[name](rng, _centre(key))
            out.append(Cluster(f"far_{name}", key, pts, lam=lam))
    if cell0:  # the double-width cell (-1, 1) on every axis, and on one axis
        for key, name in (((0, 0, 0), "tilted_plane"), ((0, 40, 0), "random_1"), ((40, 0, 44), "zplane")):
            pts, lam = by_name[name](rng, _centre(key))
            out.append(Cluster(f"cell0_{name}", key, pts, lam=lam))
    for cl in out:   # half of them close to the barycenter, half anywhere around it
        cl.kps = [_keypoint(rng, cl, 0.12 if i % 2 else 0.5) for i in range(kps_per_cluster)]
        _check_isolated(cl)
    return out


def _keypoint(rng, cl: Cluster, reach=0.5) -> np.ndarray:
    """A keypoint near the cluster, off the voxel faces, with no tie among its 20 squared distances (where the cluster
    has no duplicate points)."""
    c = cl.pts.astype(np.float64).mean(axis=0)
    for _ in range(1000):
        kp = c + rng.uniform(-reach, reach, 3)
        if np.any(np.abs(kp - np.round(kp)) < 1e-3):
            continue
        if np.any(np.trunc(kp).astype(np.int64) - np.asarray(cl.key) > 1) or np.any(np.trunc(kp).astype(np.int64) - np.asarray(cl.key) < -1):
            continue
        if not _has_ties(cl.pts, kp):
            return kp
    raise RuntimeError("no tie-free keypoint")


def _has_ties(pts32, kp) -> bool:
    uniq = np.unique(pts32, axis=0)
    d2 = sorted(exact_d2(p, kp) for p in uniq)
    return any(a == b for a, b in zip(d2, d2[1:]))


def _check_isolated(cl: Cluster):
    cells = np.trunc(cl.pts.astype(np.float64)).astype(np.int64)
    assert np.all(cells == np.asarray(cl.key)), (cl.name, cl.key)


def exact_d2(p, kp):
    """Squared distance of an FP32 map point to a FP64 keypoint, exactly (mpmath at 50 digits holds it)."""
    with mpmath.workdps(50):
        return sum((mpmath.mpf(float(a)) - mpmath.mpf(float(b))) ** 2 for a, b in zip(p, kp))


def map_arrays(clusters):
    keys = np.array([c.key for c in clusters], np.int16)
    counts = np.full(len(clusters), K, np.int32)
    xyz = np.stack([c.pts for c in clusters]).astype(np.float32)
    return keys, counts, xyz


def keypoints(clusters):
    """(n, 3) keypoints and, per keypoint, the index of its cluster."""
    kp = np.array([k for c in clusters for k in c.kps], np.float64)
    owner = np.array([i for i, c in enumerate(clusters) for _ in c.kps])
    return kp, owner


# ---- truth --------------------------------------------------------------------------------------------------------
@dataclass
class FitTruth:
    evals: tuple          # ascending, as floats
    evecs: object         # mpmath matrix, columns ascending
    centre: np.ndarray
    def gap_rel(self):
        lo, mid, hi = self.evals
        return (mid - lo) / (hi - lo) if hi > lo else 0.0
    def kappa(self):
        """lambda_max / (lambda_mid - lambda_min): the normal's condition number (inf when it is undefined)."""
        lo, mid, hi = self.evals
        return hi / (mid - lo) if mid > lo else float("inf")


def fit_truth(pts32) -> FitTruth:
    """Barycenter and scatter of the stored points exactly, eigen-decomposition at 50 digits."""
    with mpmath.workdps(50):
        P = [[mpmath.mpf(float(v)) for v in p] for p in np.asarray(pts32, np.float64)]
        m = [sum(p[a] for p in P) / len(P) for a in range(3)]
        S = mpmath.matrix(3, 3)
        for p in P:
            for a in range(3):
                for b in range(3):
                    S[a, b] += (p[a] - m[a]) * (p[b] - m[b])
        E, Q = mpmath.eigsy(S)
        order = sorted(range(3), key=lambda i: E[i])
        ev = tuple(float(E[i]) for i in order)
        Qs = mpmath.matrix(3, 3)
        for j, i in enumerate(order):
            for a in range(3):
                Qs[a, j] = Q[a, i]
        return FitTruth(ev, Qs, np.array([float(v) for v in m]))


@dataclass
class RowTruth:
    status: int           # 2 accepted, 1 rejected
    normal: np.ndarray    # flipped, unit
    a2D: float
    weight: float
    offset: float
    distance: float
    J: np.ndarray
    nearest: np.ndarray   # vector_neighbors[0]
    flip_margin: float    # |n . (t_last - b)| / |t_last - b|
    fit: FitTruth
    free_dim: int         # dimension of the eigenspace of the (numerically) smallest eigenvalue: 1 = the normal is defined
    free_radius: float    # |projection of (keypoint - nearest) on that eigenspace|: bounds |distance| for ANY normal in it
    fixed_dirs: np.ndarray  # (3 - free_dim, 3) eigenvectors outside it: every admissible normal is orthogonal to them


def row_truth(pts32, kp, fit: FitTruth | None = None, t_last=T_LAST, dmax=DMAX, power=2.0) -> RowTruth:
    fit = fit or fit_truth(pts32)
    with mpmath.workdps(50):
        lo, mid, hi = (mpmath.mpf(v) for v in fit.evals)
        s1, s2, s3 = mpmath.sqrt(abs(hi)), mpmath.sqrt(abs(mid)), mpmath.sqrt(abs(lo))
        a2D = (s2 - s3) / s1 if s1 != 0 else mpmath.nan
        n = [fit.evecs[a, 0] for a in range(3)]
        nn = mpmath.sqrt(sum(v * v for v in n))
        n = [v / nn for v in n]
        kpm = [mpmath.mpf(float(v)) for v in kp]
        tl = [mpmath.mpf(float(v)) for v in t_last]
        to_last = [tl[a] - kpm[a] for a in range(3)]
        side = sum(n[a] * to_last[a] for a in range(3))
        if side < 0:
            n = [-v for v in n]
        flip_margin = float(abs(side) / mpmath.sqrt(sum(v * v for v in to_last)))
        d2 = [exact_d2(p, kp) for p in pts32]
        j0 = int(np.argmin([float(v) for v in d2]))
        p0 = [mpmath.mpf(float(v)) for v in np.asarray(pts32[j0], np.float64)]
        dist0 = mpmath.sqrt(d2[j0])
        if a2D != a2D:
            w = mpmath.nan
        else:
            w = LAMBDA_W * (a2D ** power) + LAMBDA_N * mpmath.exp(-dist0 / (dmax * K))
        offset = -sum(n[a] * p0[a] for a in range(3))
        distance = sum(n[a] * kpm[a] for a in range(3)) + offset
        b = kpm
        bxn = [b[1] * n[2] - b[2] * n[1], b[2] * n[0] - b[0] * n[2], b[0] * n[1] - b[1] * n[0]]
        J = [w * v for v in n] + [w * v for v in bxn]
        free = [j for j in range(3) if fit.evals[j] - fit.evals[0] <= 1e-6 * abs(fit.evals[2])]
        V = np.array([[float(fit.evecs[a, j]) for a in range(3)] for j in range(3)])
        e = np.array([float(kpm[a] - p0[a]) for a in range(3)])
        return RowTruth(status=2 if distance < dmax else 1, normal=np.array([float(v) for v in n]), a2D=float(a2D),
                        weight=float(w), offset=float(offset), distance=float(distance), J=np.array([float(v) for v in J]),
                        nearest=np.array([float(v) for v in p0]), flip_margin=flip_margin, fit=fit, free_dim=len(free),
                        free_radius=float(np.linalg.norm(V[free] @ e)), fixed_dirs=V[[j for j in range(3) if j not in free]])


# ---- conditioning-aware error bounds (FP64 arithmetic on the stored points) ---------------------------------------
C_EIG = 1e3   # constant of the backward error of the scatter + eigensolver, in units of eps * lambda_max


def normal_bound(fit: FitTruth) -> float:
    """|n - n_true| for a backward-stable symmetric eigensolver: c eps lambda_max / (lambda_mid - lambda_min)."""
    return C_EIG * EPS * fit.kappa() + 64 * EPS


def _sqrt_err(lam, delta):
    return float(np.sqrt(abs(lam) + delta) - np.sqrt(max(abs(lam) - delta, 0.0)))


def a2d_bound(fit: FitTruth, a2D: float) -> float:
    """|a2D - a2D_true| when every eigenvalue carries an absolute error c eps lambda_max: the square roots of the two
    smallest lose up to half their digits when those are ~0 (an exact plane: sigma_3 ~ sqrt(eps) sigma_1)."""
    lo, mid, hi = fit.evals
    delta = C_EIG * EPS * abs(hi)
    s1 = np.sqrt(abs(hi))
    return (_sqrt_err(mid, delta) + _sqrt_err(lo, delta) + abs(a2D) * _sqrt_err(hi, delta)) / s1 + 1e-14
