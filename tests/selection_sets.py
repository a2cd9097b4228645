"""Crafted neighbourhoods for the FP32 neighbour selection of the scan-matching pass (k1_scan / k1_fit, k1_fast, k1_assoc).

Every keypoint gets a neighbourhood of its own: float32 map points around it, isolated from every other keypoint's
27-voxel search, loaded with `voxel_map.upload` / `OracleMap.load` / `Reference.load`.  The pose and the extrinsics are
the identity, so the world keypoints are the raw ones bit for bit.  The background of a neighbourhood is a plane
through the keypoint; the candidates whose order the selection has to decide lie off that plane on opposite sides, so
that picking the wrong one moves the fitted plane, `offset` and `distance` far beyond the 1e-5 of the parity tests.

Families (the window is W(T) = T 2^-11 + 2.5 eps32 with eps32 = 1e-4 size^2, DESIGN.md section 4):
  A  the (K+1)-th candidate r W(T) above the K-th, r in {0.05 .. 8}; zones of 1-3 extra slots (m = 21..23, resolved by
     k1_fit); a wide zone (j0 < 12) and a certifier inside the window (both flagged).
  B  2-6 candidates within W(key0) of the nearest, a few 1e-7 size^2 apart so that their keys tie and the packed
     candidate id orders them: b1 = 2..4 is resolved by k1_fit, b1 > 4 and a shell (b1 > j0) are flagged.
  C  the K nearest dealt to one lane: k1_scan gives a voxel's point i to lane i % LPK, so the near candidates sit at
     indices of one residue in four voxels; NLS - 1 of them in that lane is certified, NLS and more is flagged.
  D  ties that FP64 rounding decides: the keypoint is (X+e, Y+e, Z+e), a map point (X+s, Y+t, Z+w) and its partner
     (X+t, Y+s, Z+w) have the same exact distance; only pairs whose reference-order d^2 AND square roots differ are kept
     (the reference's answer is then fully determined), at the K-th boundary, at the nearest slot and mid-list.  A few
     pairs whose square roots tie are built apart (`sqrt_tie`): there the reference's heap decides.
  E  skip geometry: keypoints 1 ulp and 1e-3 size from a corner, an edge or a face of their voxel (both faces of the
     double-width cell 0 and the negative side included), the K-th neighbour in the corner voxel that c_off_fast visits
     last, and a two-point voxel inside the window that an occupancy threshold of 3 removes.
Every family runs at sizes 0.5, 0.7 (the division path of voxel_quotient), 1 and 2, near the origin on both sides, at
+-300 m, +-3000 m and at |q| ~ 32700 (family D where its pair search succeeds: near the origin and at +-300 m).

`measure()` records per keypoint what came out of the FP32 points: exact d^2 (fractions), the reference-order FP64 d^2,
the kernel's FP32 d2f with and without FMA contraction, the ratio of the K-th gap to W(T), and the verdict that
`select_model` predicts for every form of the pass.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from fractions import Fraction

import numpy as np

from test_selection_model import KF, scan_verdict

K = KF
CAP = 20
SIZES = (0.5, 0.7, 1.0, 2.0)
IDENTITY_Q = np.array([0.0, 0.0, 0.0, 1.0])
ZERO_T = np.zeros(3)
T_LAST = np.array([7.1e4, -9.2e4, 5.7e4])
_TL_DIR = T_LAST / np.linalg.norm(T_LAST)
# placement -> voxel key of the first neighbourhood and the step between neighbourhoods (6 voxels along y)
PLACEMENTS = ("origin+", "origin-", "p300", "m300", "p3000", "m3000", "qmax")
# every form of the pass: (name, options); the split form and k1_fast with their lane layouts
FORMS = {"split4": dict(k1_variant=3, split_lanes_per_keypoint=4), "split2": dict(k1_variant=3, split_lanes_per_keypoint=2),
         "fast1": dict(k1_variant=1, fast_lanes_per_keypoint=1), "fast2": dict(k1_variant=1, fast_lanes_per_keypoint=2),
         "fast4": dict(k1_variant=1, fast_lanes_per_keypoint=4), "assoc": dict(k1_variant=2), "exact": dict(force_exact_selection=1)}
MODEL_FORM = {"split4": dict(lpk=4, nls=14), "split2": dict(lpk=2, nls=20), "fast1": dict(lpk=1, fast=True),
              "fast2": dict(lpk=2, fast=True), "fast4": dict(lpk=4, fast=True)}
FAMILIES = ("A", "B", "C", "D", "E")


def window(T, size):
    """W(T) in m^2 (T in m^2)."""
    return T / 2048.0 + 2.5e-4 * size * size


def _base_key(place, size):
    q = {"origin+": (0, 2, 3), "origin-": (-2, -8, 0), "p300": (300, 300, 300), "m300": (-300, -300, -300),
         "p3000": (3000, 3000, 3000), "m3000": (-3000, -3000, -3000), "qmax": (32700, -32700, -32700)}[place]
    if place.startswith("origin") or place == "qmax":
        return np.array(q, np.int64)
    return np.array([int(v / size) for v in q], np.int64)


def _step(place):
    """Neighbourhoods 6 voxels apart; near the origin only the first one sits in the double-width cell 0."""
    return np.array({"origin+": (6, 0, 0), "origin-": (0, 0, -6)}.get(place, (0, 6, 0)), np.int64)


# ---- float helpers -----------------------------------------------------------------------------------------------
def exact_d2(p32, kp) -> Fraction:
    return sum((Fraction(float(a)) - Fraction(float(b))) ** 2 for a, b in zip(p32, kp))


def ref_d2(p32, kp):
    """The reference's squared distance: FP64, c0 + (c1 + c2), no FMA (src/optimize.cpp:394-395 through Eigen)."""
    d = np.asarray(p32, np.float64) - np.asarray(kp, np.float64)
    return d[..., 0] * d[..., 0] + (d[..., 1] * d[..., 1] + d[..., 2] * d[..., 2])


def packet_d2(p32, kp):
    d = np.asarray(p32, np.float64) - np.asarray(kp, np.float64)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def voxel_of(p, size):
    return np.trunc(np.asarray(p, np.float64) / size).astype(np.int64)


def _f32_corner(kp, size):
    k = voxel_of(kp, size)
    cx = k.astype(np.float64) * size
    of = cx.astype(np.float32)
    rf = (kp - of.astype(np.float64)).astype(np.float32)
    rel = (kp - cx).astype(np.float32)
    return k, of, rf, rel


def kernel_d2f(pts32, kp, size):
    """The kernels' FP32 d2f = |(m - of) - rf|^2 under the evaluation orders nvcc may emit: no contraction, and the two
    FMA chains.  (n, 3) -> dict of float32 arrays."""
    _, of, rf, _ = _f32_corner(kp, size)
    d = (np.asarray(pts32, np.float32) - of) - rf
    d0, d1, d2 = d[:, 0], d[:, 1], d[:, 2]
    f = np.float32
    nofma = (d0 * d0 + d1 * d1) + d2 * d2
    def fma(a, b, c):
        return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(f)
    fma_a = fma(d2, d2, fma(d1, d1, d0 * d0))
    fma_b = fma(d2, d2, fma(d0, d0, d1 * d1))
    return dict(nofma=nofma.astype(f), fma_a=fma_a, fma_b=fma_b)


def fast_offsets():
    """c_off_fast: the 27 offsets ordered by |offset|^2, centre first, then x, y, z ascending."""
    out = []
    for d2 in range(4):
        for x in (-1, 0, 1):
            for y in (-1, 0, 1):
                for z in (-1, 0, 1):
                    if x * x + y * y + z * z == d2:
                        out.append((x, y, z))
    return out


def lower_bound(kp, size, v):
    """k1_scan's conservative squared distance from the keypoint to voxel v, FP32, truncated as the kernel packs it."""
    k, _, _, rel = _f32_corner(kp, size)
    f = np.float32
    s = f(size)
    g = []
    for a in range(3):
        va, ka = int(v[a]), int(k[a])
        lo = f((va if va > 0 else va - 1) - ka) * s
        hi = f((va if va < 0 else va + 1) - ka) * s
        g.append(max(f(max(f(lo - rel[a]), f(rel[a] - hi)) - f(1e-5) * s), f(0.0)))
    lb = f(f(f(g[0] * g[0] + g[1] * g[1]) + g[2] * g[2]) * f(0.999999))
    return np.array([lb], np.float32).view(np.uint32)[0] & np.uint32(0xFFFFFF80)


# ---- neighbourhoods ----------------------------------------------------------------------------------------------
@dataclass
class Hood:
    family: str
    variant: str
    size: float
    place: str
    kp: np.ndarray                        # (3,) float64
    pts: np.ndarray                       # (n, 3) float32, in the order they are stored (per voxel)
    pair: tuple | None = None             # indices of the two candidates whose order the selection decides
    where: str = ""                       # "kth", "nearest", "mid" for a pair
    sqrt_tie: bool = False
    info: dict = field(default_factory=dict)


def _frame(rng, normal=None):
    if normal is None:
        while True:
            n = rng.normal(size=3)
            n /= np.linalg.norm(n)
            if abs(n @ _TL_DIR) > 0.4:
                break
    else:
        n = np.asarray(normal, np.float64) / np.linalg.norm(normal)
    a = np.cross(n, rng.normal(size=3))
    u1 = a / np.linalg.norm(a)
    return n, u1, np.cross(n, u1)


def _ulp32(x):
    return np.spacing(np.abs(np.float32(x))).astype(np.float64)


def _snap(kp, target, d2_target):
    """The float32 point near `target` whose squared distance to kp is closest to d2_target (searched over +-6 float32
    ulps per axis: where the float grid is coarse, a designed gap still lands where it was meant to)."""
    t32 = np.asarray(target, np.float32)
    u = np.spacing(np.abs(t32)).astype(np.float64)
    r = np.arange(-6, 7)
    g = np.stack(np.meshgrid(r, r, r, indexing="ij"), -1).reshape(-1, 3)
    cand = (t32.astype(np.float64) + g * u).astype(np.float32)
    d2 = ref_d2(cand, kp)
    return cand[int(np.argmin(np.abs(d2 - d2_target)))]


def _at(kp, size, frame, D2, theta, elev=0.0, snap=False):
    n, u1, u2 = frame
    d = np.sqrt(D2) * size
    dirv = np.cos(elev) * (np.cos(theta) * u1 + np.sin(theta) * u2) + np.sin(elev) * n
    p = kp + d * dirv
    return _snap(kp, p, D2 * size * size) if snap else p.astype(np.float32)


def _spread(rng, n):
    """n in-plane angles, spread around the circle"""
    return (np.arange(n) + rng.uniform(0, 1, n)) * (2 * np.pi / n) + rng.uniform(0, 2 * np.pi)


ELEV = np.deg2rad(25.0)


def _background(rng, kp, size, frame, D2s):
    th = _spread(rng, len(D2s))
    return [_at(kp, size, frame, D2, t) for D2, t in zip(D2s, th)]


def _std_rings(rng, n_core=12, n_mid=7, n_far=8, mid=(0.18, 0.30)):
    return (list(rng.uniform(0.04, 0.15, n_core)), list(rng.uniform(*mid, n_mid)), list(rng.uniform(0.5, 0.8, n_far)))


def _kp_in(rng, key, size):
    """A keypoint inside voxel `key`, 0.08 .. 0.2 size from one of its faces on every axis: its neighbourhood then
    spreads over the 8 voxels around a corner instead of crowding into one (a voxel holds 20 points)."""
    out = []
    for k in key:
        lo, hi = (k * size, (k + 1) * size) if k > 0 else ((k - 1) * size, k * size) if k < 0 else (-size, size)
        d = rng.uniform(0.08, 0.2) * size
        out.append(lo + d if rng.uniform() < 0.5 else hi - d)
    return np.array(out)


def fam_A(rng, keys, size):
    out = []
    T0 = 0.36
    W = window(T0 * size * size, size) / (size * size)
    variants = [("edge", r, 1) for r in (0.05, 0.5, 0.95, 1.05, 2.0, 8.0)] + [("zone2", 0.3, 2), ("zone3", 0.3, 3),
                                                                                ("wide", 0.3, 0), ("certifier", 0.2, 0)]
    for vi, (name, r, extra) in enumerate(variants):
        kp = _kp_in(rng, keys(vi), size)
        fr = _frame(rng)
        core, mid, far = _std_rings(rng)
        if name == "wide":           # slots 6..22 inside one window: j0 < 12 with m > K
            core, mid = core[:6], [T0 - 0.4 * W + 0.8 * W * i / 16 for i in range(16)]
        if name == "certifier":      # slots 20..23 inside the window of the K-th: the certifier is not outside it
            mid = mid + [T0 + W * x for x in (0.2, 0.35, 0.5, 0.65, 0.8)]
        pts = _background(rng, kp, size, fr, core + mid)
        th = rng.uniform(0, 2 * np.pi)
        pair = None
        if name in ("wide", "certifier"):
            pts += _background(rng, kp, size, fr, far)
        else:
            # the K-th and the (K+1)-th on opposite sides of the plane; the farther one is stored first
            hi = _at(kp, size, fr, T0 + r * W, th, -ELEV, snap=True)
            lo = _at(kp, size, fr, T0, th + np.pi * 0.9, ELEV, snap=True)
            zone = [_at(kp, size, fr, T0 + r * W + (i + 1) * 0.2 * W, th + 0.7 * (i + 1), 0.0, snap=True) for i in range(extra - 1)]
            pts += zone + [hi, lo]
            pair = (len(pts) - 1, len(pts) - 2)
            pts += _background(rng, kp, size, fr, far)
        out.append(Hood("A", f"{name}_{r}" if name == "edge" else name, size, "", kp, np.array(pts, np.float32), pair, "kth"))
    return out


def fam_B(rng, keys, size):
    out = []
    for vi, (n_tie, gap) in enumerate(((2, "tiny"), (3, "tiny"), (4, "tiny"), (2, "half"), (5, "tiny"), (6, "tiny"), (3, "shell"))):
        kp = _kp_in(rng, keys(vi), size)
        fr = _frame(rng)
        d0 = 0.02
        W0 = window(d0 * size * size, size) / (size * size)
        core, mid, far = _std_rings(rng)
        if gap == "shell":           # everything near one distance: nothing is certainly in, b1 > j0
            core, mid = [], [0.3 + W0 * 0.05 * i for i in range(21)]
        pts = _background(rng, kp, size, fr, core + mid)
        th = _spread(rng, n_tie)
        # tied candidates below the plane, the exactly nearest one above it and stored last
        step = 1e-7 if gap == "tiny" else 0.45 * W0 / n_tie
        ties = [_at(kp, size, fr, d0 + step * (n_tie - 1 - i), th[i], ELEV if i == n_tie - 1 else -ELEV, snap=True) for i in range(n_tie)]
        pts += ties
        pair = (len(pts) - 1, len(pts) - 2)
        pts += _background(rng, kp, size, fr, far)
        out.append(Hood("B", f"b{n_tie}_{gap}", size, "", kp, np.array(pts, np.float32), pair, "nearest"))
    return out


def fam_C(rng, keys, size):
    """Four voxels around a vertical edge of the keypoint's voxel, 20 points each: the K nearest sit at indices of one
    residue modulo LPK (in_lane of them) and at other indices (the rest), every other slot is far."""
    out = []
    for lpk, nls in ((4, 14), (2, 20)):
        for in_lane in (nls - 1, nls, nls + 1):
            if in_lane > K:
                continue
            key = keys(len(out))
            k = np.array(key)
            kp = np.array([(k[0] + 1) * size if k[0] >= 0 else (k[0] - 1) * size,
                           (k[1] + 1) * size if k[1] >= 0 else (k[1] - 1) * size, 0.0])
            sx = -1.0 if k[0] >= 0 else 1.0
            sy = -1.0 if k[1] >= 0 else 1.0
            kp[0] += sx * 0.1 * size
            kp[1] += sy * 0.1 * size
            kp[2] = _kp_in(rng, key, size)[2]
            near_d2 = np.sort(rng.uniform(0.03, 0.3, K))
            near_lane = rng.permutation(K)
            vox = []
            for dx in (0, 1):
                for dy in (0, 1):
                    vox.append(np.array([k[0] - sx * dx, k[1] - sy * dy, k[2]]))
            slots = [[None] * CAP for _ in vox]
            res = [(v, i) for i in range(0, CAP, lpk) for v in range(4)]
            oth = [(v, i) for i in range(CAP) if i % lpk for v in range(4)]
            rng.shuffle(res)
            rng.shuffle(oth)
            for j in range(K):
                v, i = res[j] if j < in_lane else oth[j - in_lane]
                slots[v][i] = ("near", near_d2[near_lane[j]])
            pts = []
            for v, sl in enumerate(slots):
                lo = np.array([vv * size if vv > 0 else (vv - 1) * size if vv < 0 else -size for vv in vox[v]], np.float64)
                hi = np.array([(vv + 1) * size if vv >= 0 else vv * size if vv < 0 else size for vv in vox[v]], np.float64)
                if vox[v][2] == 0:
                    lo[2], hi[2] = -size, size
                for s in sl:
                    want = s[1] if s else rng.uniform(0.55, 0.75)
                    for _ in range(2000):   # a point of this voxel at the wanted distance, in the keypoint's horizontal plane
                        th = rng.uniform(0, 2 * np.pi)
                        p = kp + np.sqrt(want) * size * np.array([np.cos(th), np.sin(th), rng.uniform(-0.02, 0.02)])
                        inset = 1e-3 * size
                        if np.all(p > lo + inset) and np.all(p < hi - inset):
                            break
                    else:
                        raise RuntimeError("family C: no point at that distance in the voxel")
                    pts.append(p.astype(np.float32))
            out.append(Hood("C", f"lpk{lpk}_in{in_lane}", size, "", kp, np.array(pts, np.float32), None, "",
                            info=dict(lpk=lpk, nls=nls, in_lane=in_lane)))
    return out


def _perm_pair(rng, kp_base, size, D2, tries=4000):
    """(keypoint, point, partner) with kp = (X+e, Y+e, Z+e), point (X+s, Y+t, Z+w), partner (X+t, Y+s, Z+w) at squared
    distance ~ D2 size^2, the reference-order d^2 and their square roots different.  None if the search fails."""
    X = np.asarray(kp_base, np.float32)
    u = float(max(_ulp32(x) for x in X))
    eg = u * 2.0 ** -14
    for _ in range(tries):
        e = rng.integers(-2 ** 12, 2 ** 12) * eg
        kp = X.astype(np.float64) + e
        dirv = rng.normal(size=3)
        dirv /= np.linalg.norm(dirv)
        off = np.round(dirv * np.sqrt(D2) * size / u) * u
        s, t, w = off
        if s == t:
            continue
        a = (X.astype(np.float64) + np.array([s, t, w])).astype(np.float32)
        b = (X.astype(np.float64) + np.array([t, s, w])).astype(np.float32)
        if not (np.all(a.astype(np.float64) == X + np.array([s, t, w])) and np.all(b.astype(np.float64) == X + np.array([t, s, w]))):
            continue
        da, db = ref_d2(a, kp), ref_d2(b, kp)
        if da != db and np.sqrt(da) != np.sqrt(db) and exact_d2(a, kp) == exact_d2(b, kp):
            return kp, a, b
    return None


def _sqrt_tie_pair(rng, kp_base, size, D2, tries=20000):
    X = np.asarray(kp_base, np.float32)
    u = float(max(_ulp32(x) for x in X))
    for _ in range(tries):
        e = rng.integers(-2 ** 12, 2 ** 12) * u * 2.0 ** -14
        kp = X.astype(np.float64) + e
        dirv = rng.normal(size=3)
        dirv /= np.linalg.norm(dirv)
        s, t, w = np.round(dirv * np.sqrt(D2) * size / u) * u
        if s == t:
            continue
        a = (X.astype(np.float64) + np.array([s, t, w])).astype(np.float32)
        b = (X.astype(np.float64) + np.array([t, s, w])).astype(np.float32)
        da, db = ref_d2(a, kp), ref_d2(b, kp)
        if da != db and np.sqrt(da) == np.sqrt(db):
            return kp, a, b
    return None


def fam_D(rng, keys, size, sqrt_ties=False):
    """Permutation pairs at the K-th boundary, at the nearest slot and mid-list.  The background plane has normal
    (1, -1, 0)/sqrt(2): swapping s and t puts the partner on the other side of it."""
    out = []
    wheres = ("kth", "kth", "nearest", "nearest", "mid") if not sqrt_ties else ("kth", "kth")
    for vi, where in enumerate(wheres):
        key = keys(vi)
        base = _kp_in(rng, key, size).astype(np.float32)
        D2 = {"kth": 0.36, "nearest": 0.02, "mid": 0.2}[where]
        got = (_sqrt_tie_pair if sqrt_ties else _perm_pair)(rng, base, size, D2)
        if got is None:
            continue
        kp, a, b = got
        n = np.array([1.0, -1.0, 0.0]) / np.sqrt(2.0)
        u1 = np.array([1.0, 1.0, 0.0]) / np.sqrt(2.0)
        fr = (n, u1, np.cross(n, u1))
        if where == "kth":
            core, mid, far = _std_rings(rng, n_mid=7)
        elif where == "nearest":
            core, mid, far = _std_rings(rng, n_core=12, n_mid=6)
        else:
            core, mid, far = _std_rings(rng, n_core=9, n_mid=9, mid=(0.22, 0.32))
        pts = _background(rng, kp, size, fr, core + mid)
        pts += [a, b]
        pair = (len(pts) - 2, len(pts) - 1)
        pts += _background(rng, kp, size, fr, far)
        out.append(Hood("D", f"{where}{'_sqrt_tie' if sqrt_ties else ''}", size, "", kp, np.array(pts, np.float32), pair,
                        where, sqrt_tie=sqrt_ties))
    return out


def fam_E(rng, keys, size):
    """Keypoints just inside a corner of their voxel (offsets 1 ulp / 1e-3 size / 0.3 size per axis); the K-th neighbour
    and the next one in the diagonal voxel past that corner (c_off_fast visits it last); two points in the voxel across
    the plane from the keypoint, inside the window (an occupancy threshold of 3 removes them)."""
    out = []
    for vi, (ox, oy, oz) in enumerate( (("ulp", "ulp", "ulp"), ("ulp", "ulp", "mid"), ("ulp", "mid", "mid"), ("milli", "milli", "milli"),
                         ("milli", "milli", "mid"), ("milli", "mid", "mid"))):
        k = np.array(keys(vi))
        sg = np.where(k >= 0, 1.0, -1.0)             # the corner away from 0 (for key 0: the +size faces of cell 0)
        if k[0] == 0 and rng.uniform() < 0.5:
            sg[0] = -1.0                              # and the -size face of cell 0
        corner = np.array([(kk + 1) * size if s > 0 and kk >= 0 else (kk - 1) * size if kk <= 0 else kk * size
                           for kk, s in zip(k, sg)])
        kp = corner.copy()
        for a, o in enumerate((ox, oy, oz)):
            if o == "ulp":
                kp[a] = np.nextafter(corner[a], corner[a] - sg[a] * np.inf)
            elif o == "milli":
                kp[a] = corner[a] - sg[a] * 1e-3 * size
            else:
                kp[a] = corner[a] - sg[a] * 0.3 * size
        n = sg * np.array([1.0, -1.0, 0.3])
        n /= np.linalg.norm(n)
        diag = sg * np.array([1.0, 1.3, 1.0])
        diag /= np.linalg.norm(diag)
        u2 = np.cross(n, diag)
        fr = (n, diag, u2)
        core = list(rng.uniform(0.04, 0.15, 12)) + list(rng.uniform(0.18, 0.3, 5))   # + the two corner points: 19
        pts = []
        for D2, th in zip(core, _spread(rng, len(core))):
            if abs(np.cos(th)) > 0.8 and np.cos(th) > 0:   # keep the far side of the corner for the K-th
                th += np.pi
            pts.append(_at(kp, size, fr, D2, th))
        T0 = 0.5
        W = window(T0 * size * size, size) / (size * size)
        hi = _at(kp, size, fr, T0 + 0.5 * W, 0.12, -np.deg2rad(12), snap=True)
        lo = _at(kp, size, fr, T0, -0.12, np.deg2rad(12), snap=True)
        pts += [hi, lo]
        pair = (len(pts) - 1, len(pts) - 2)
        pts += [_at(kp, size, fr, D2, th) for D2, th in zip(rng.uniform(0.75, 0.85, 6), _spread(rng, 6))]
        # two points off the plane on the side n points to, next to the corner
        for j in range(2):
            pts.append((corner + sg * np.array([0.15, -0.12, 0.15 + 0.05 * j]) * size).astype(np.float32))
        out.append(Hood("E", f"{ox}-{oy}-{oz}{'-neg0' if sg[0] < 0 and k[0] == 0 else ''}", size, "", kp,
                        np.array(pts, np.float32), pair, "kth"))
    return out


BUILDERS = {"A": fam_A, "B": fam_B, "C": fam_C, "D": fam_D, "E": fam_E}


# ---- batches -------------------------------------------------------------------------------------------------------
@dataclass
class Batch:
    family: str
    size: float
    hoods: list
    keys: np.ndarray
    counts: np.ndarray
    xyz: np.ndarray
    kp: np.ndarray
    slot: list            # per voxel: (hood index, index of each stored point in hood.pts)

    @property
    def map(self):
        return self.keys, self.counts, self.xyz


def assemble(hoods, size, family):
    vox = {}
    for h_i, h in enumerate(hoods):
        for p_i, p in enumerate(h.pts):
            v = tuple(int(x) for x in voxel_of(p.astype(np.float64), size))
            ent = vox.setdefault(v, (h_i, []))
            assert ent[0] == h_i, ("two neighbourhoods share a voxel", family, size, v)
            ent[1].append(p_i)
    for v, (h_i, idx) in vox.items():
        if len(idx) > CAP:
            raise ValueError(f"voxel {v} of {family} holds {len(idx)} points")
    # isolation: every voxel inside a keypoint's 27-voxel cube belongs to that keypoint's neighbourhood
    for h_i, h in enumerate(hoods):
        kk = voxel_of(h.kp, size)
        for dx in (-1, 0, 1):
            for dy in (-1, 0, 1):
                for dz in (-1, 0, 1):
                    v = (int(kk[0] + dx), int(kk[1] + dy), int(kk[2] + dz))
                    assert v not in vox or vox[v][0] == h_i, ("not isolated", family, size, h.variant, v)
        for p in h.pts:
            assert np.all(np.abs(voxel_of(p.astype(np.float64), size) - kk) <= 1), ("point outside the cube", family, h.variant)
    keys = np.array(list(vox.keys()), np.int16).reshape(-1, 3)
    counts = np.array([len(v[1]) for v in vox.values()], np.int32)
    xyz = np.zeros((len(vox), CAP, 3), np.float32)
    for j, (h_i, idx) in enumerate(vox.values()):
        xyz[j, :len(idx)] = hoods[h_i].pts[idx]
    kp = np.array([h.kp for h in hoods], np.float64)
    return Batch(family, size, hoods, keys, counts, xyz, kp, list(vox.values()))


def build_batch(family, size, seed=0, places=PLACEMENTS, sqrt_ties=False):
    """Every variant of one family at one voxel size, at every placement: one neighbourhood per keypoint, 6 voxels apart."""
    hoods = []
    for p_i, place in enumerate(places):
        base, step = _base_key(place, size), _step(place)
        for attempt in range(20):
            rng = np.random.default_rng([seed, FAMILIES.index(family), int(size * 10), p_i, attempt, int(sqrt_ties)])
            try:
                keys = lambda i: tuple(int(x) for x in base + step * i)
                got = fam_D(rng, keys, size, sqrt_ties) if family == "D" else BUILDERS[family](rng, keys, size)
                for h in got:
                    h.place = place
                assemble(hoods + got, size, family)
                break
            except (ValueError, RuntimeError, AssertionError):
                got = None
        assert got is not None, (family, size, place)
        hoods += got
    return assemble(hoods, size, family)


# ---- what came out ---------------------------------------------------------------------------------------------------
def candidates(batch, k, nb=1, thr=1):
    """The candidates of keypoint k in the kernels' order: present voxels (count >= thr) in c_off_fast order (nb = 1) and
    their points in stored order.  Returns (points (n,3) f32, packed ids e<<5|i, chunks, lower bounds, reference visit
    ids, voxel keys (n,3), index in voxel)."""
    size = batch.size
    kk = voxel_of(batch.kp[k], size)
    vmap = {tuple(map(int, key)): j for j, key in enumerate(batch.keys)}
    offs = fast_offsets() if nb == 1 else [(0, 0, 0)]
    W = 2 * nb + 1
    pts, ids, chunks, lbs, vis, vkeys, vidx = [], [], [], [], [], [], []
    e = 0
    for o in offs:
        v = (int(kk[0] + o[0]), int(kk[1] + o[1]), int(kk[2] + o[2]))
        j = vmap.get(v)
        if j is None or batch.counts[j] < thr:
            continue
        c = int(batch.counts[j])
        chunks.append(np.arange(len(pts), len(pts) + c))
        lbs.append(np.array([lower_bound(batch.kp[k], size, v)], np.uint32).view(np.float32)[0])
        r = ((o[0] + nb) * W + (o[1] + nb)) * W + (o[2] + nb)
        for i in range(c):
            pts.append(batch.xyz[j, i])
            ids.append((e << 5) | i)
            vis.append((r << 5) | i)
            vkeys.append(v)
            vidx.append(i)
        e += 1
    return (np.array(pts, np.float32).reshape(-1, 3), np.array(ids, np.uint32), chunks, np.array(lbs, np.float32),
            np.array(vis, np.int64), np.array(vkeys, np.int64).reshape(-1, 3), np.array(vidx, np.int64))


def brute_force(batch, k, K_=K, nb=1, thr=1):
    """The reference's answer by brute force: FP64 d^2 in its order, ranked by (d^2, visit index)."""
    size = batch.size
    kk = voxel_of(batch.kp[k], size)
    W = 2 * nb + 1
    rows = []
    vmap = {tuple(map(int, key)): j for j, key in enumerate(batch.keys)}
    for ox in range(-nb, nb + 1):
        for oy in range(-nb, nb + 1):
            for oz in range(-nb, nb + 1):
                v = (int(kk[0] + ox), int(kk[1] + oy), int(kk[2] + oz))
                j = vmap.get(v)
                if j is None or batch.counts[j] < thr:
                    continue
                r = ((ox + nb) * W + (oy + nb)) * W + (oz + nb)
                for i in range(int(batch.counts[j])):
                    rows.append((float(ref_d2(batch.xyz[j, i], batch.kp[k])), r, i, v))
    rows.sort(key=lambda t: (t[0], t[1], t[2]))
    return rows[:K_]


def measure(batch, k, forms=MODEL_FORM, thr=1):
    """Per keypoint: exact and reference-order d^2 of the candidates, the FP32 d2f variants, the K-th gap over W(T) and
    the model's verdict for every form and FP32 evaluation order."""
    size = batch.size
    kp = batch.kp[k]
    pts, ids, chunks, lbs, vis, _, _ = candidates(batch, k, thr=thr)
    d2r = ref_d2(pts, kp)
    ex = np.array([float(exact_d2(p, kp)) for p in pts])
    f32 = kernel_d2f(pts, kp, size)
    out = dict(n=len(pts), d2_ref=d2r, d2_exact=ex, d2f=f32, verdict={})
    order = np.lexsort((vis, d2r))
    if len(pts) > K:
        T, nxt = d2r[order[K - 1]], d2r[order[K]]
        out["gap_over_W"] = (nxt - T) / window(T, size)
    for name, kw in forms.items():
        out["verdict"][name] = {var: scan_verdict(d, size, chunks, lbs, ids=ids, **kw) for var, d in f32.items()}
    return out


def predicted_flags(meas, form):
    """(min, max) over the FP32 evaluation orders of whether the form flags the keypoint (0 / 1)."""
    if meas["n"] < K:
        return 0, 0
    v = [int(x["flagged"]) for x in meas["verdict"][form].values()]
    return min(v), max(v)


def branch(meas, form="split4"):
    """'flagged', 'zone' (m > K, resolved by k1_fit), 'nearest' (b1 > 1), 'zone+nearest' or 'plain' under the no-FMA order."""
    v = meas["verdict"][form]["nofma"]
    if meas["n"] < K:
        return "short"
    if v["flagged"]:
        return "flagged"
    z, b = v["m"] > K, v["b1"] > 1
    return "zone+nearest" if z and b else "zone" if z else "nearest" if b else "plain"


# family -> the least the model must predict over the whole family (every size, every placement) for split4
MINIMUMS = {"A": dict(zone=40, flagged=40), "B": dict(nearest=40, flagged=40), "C": dict(flagged=40, plain=20),
            "D": dict(zone=20, nearest=15), "E": dict(zone=15)}


def sum_scales(o):
    """Per component of HTH / HTh / loss_sum: the sum of the keypoints' absolute contributions (from debug rows).  The
    sums are compared relative to these, so that keypoints near the origin are not drowned by the Jacobians' lever arm
    of those at 65 km."""
    J = o.plane[:, 6:12]
    h = o.plane[:, 13] * o.plane[:, 14]
    acc = o.status == 2
    H = np.abs(J[acc, :, None] * J[acc, None, :]).sum(axis=0)
    g = np.abs(J[acc] * h[acc, None]).sum(axis=0)
    return np.maximum(H, 1e-300), np.maximum(g, 1e-300), max(float((o.plane[acc, 13] ** 2).sum()), 1e-300)
