"""Seeded cases at the edges of the LIO voxel map: distance ties, the 10 size^2 clamp, the cap and the min_num_points gate,
the key range, long and wrapping probe chains through growth and eviction, and the eviction rule itself.

A case is a sequence of operations on one map:
  ("upload", keys, counts, xyz)           srl_map_upload / the oracle's load
  ("insert", world_xyz, md, mnp, tz)      addPointsToMap(min_distance_points=md, min_num_points=mnp), intensity relative to tz
  ("remove", location, distance)          removePointsFarFromLocation
`probes` (when set) are keypoints whose scan-matching pass the device test compares with the oracle after the last operation.
`empty_voxels` marks states the compiled reference cannot take to eviction (it reads points[0] of an empty voxel).
"""
from __future__ import annotations

import functools
import math
from dataclasses import dataclass, field

import numpy as np

from map_reference import f32, hash_key, short_key, sq_dist, sq_dist_other_order

CAP = 20


@dataclass
class Case:
    name: str
    ops: list
    size: float = 1.0
    cap: int = CAP
    initial_voxels: int = 256
    probes: np.ndarray | None = None
    empty_voxels: bool = False
    # crafted pairs: dict(a, b, md, add = what the double evaluation decides for b against a, and what certifies it: exact
    # (the tie is exact in double), ulps (fl(sq) is that many doubles from fl(md^2)), split (the other reduction order
    # decides the opposite), clamp (the true squared distance exceeds 10 size^2))
    certs: list = field(default_factory=list)


def fnext(x: float, k: int = 1) -> float:
    """The float k steps from the float x (positive x, or crossing only within one sign)."""
    b = int(np.array([x], np.float32).view(np.int32)[0]) + k
    return float(np.array([b], np.int32).view(np.float32)[0])


def dnext(x: float, k: int = 1) -> float:
    for _ in range(abs(k)):
        x = math.nextafter(x, math.inf if k > 0 else -math.inf)
    return x


def _ins(xyz, md=0.15, mnp=0, tz=0.0):
    return ("insert", np.asarray(xyz, np.float64).reshape(-1, 3), float(md), int(mnp), float(tz))


def _shuffled(rng, *groups):
    pts = np.concatenate([np.asarray(g, np.float64).reshape(-1, 3) for g in groups])
    return pts[rng.permutation(pts.shape[0])]


# ---- distance ---------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def mine_near_tie(md: float, k: int, a=(0.25, 0.25, 0.0), start=0.08, dz_max=3e-6):
    """Two float positions whose double squared distance is k ulps from fl(md * md): y and x coarse, then z (tiny, so its
    square steps through single doubles) by bisection over the float bit patterns."""
    target = float(np.array([np.array([md * md]).view(np.int64)[0] + k]).view(np.float64)[0])
    ax, ay, az = a
    by = f32(ay + start)
    for _ in range(20000):
        by = fnext(by)
        dy = by - ay
        bx = f32(ax + math.sqrt(target - dy * dy))
        while (bx - ax) * (bx - ax) + dy * dy > target:
            bx = fnext(bx, -1)
        if target - ((bx - ax) * (bx - ax) + dy * dy) > dz_max * dz_max:
            continue

        def g(i):
            return sq_dist(a, (bx, by, az + float(np.array([i], np.int32).view(np.float32)[0])))
        lo, hi = 0, int(np.array([dz_max], np.float32).view(np.int32)[0])
        if g(hi) < target:
            continue
        while lo < hi:
            mid = (lo + hi) // 2
            lo, hi = (lo, mid) if g(mid) >= target else (mid + 1, hi)
        if g(lo) == target:
            return tuple(a), (bx, by, az + float(np.array([lo], np.int32).view(np.float32)[0]))
    raise RuntimeError("no near tie found")


def _fbits(x: float) -> int:
    return int(np.array([x], np.float32).view(np.int32)[0])


def _fval(i: int) -> float:
    return float(np.array([i], np.int32).view(np.float32)[0])


@functools.lru_cache(maxsize=None)
def mine_order_split(md: float, want_add: bool):
    """Two float positions where dx^2 + (dy^2 + dz^2) and (dx^2 + dy^2) + dz^2 fall on opposite sides of fl(md * md): the
    first (the reference's order) adds the point when want_add, the second would do the opposite.  Two coarse axes put the
    pair near the threshold, a tiny difference on the third (x for an add, z for a reject: where the two roundings part
    that way) is bisected to the crossing and searched around."""
    thr = md * md
    a = (0.0, 0.25, 0.25) if want_add else (0.25, 0.25, 0.0)   # 0 on the tiny axis: the tiny difference is itself a float
    for tiny, (c1, c2) in (((0, (2, 1)),) if want_add else ((2, (0, 1)),)):
        b2 = f32(a[c2] + 0.05)
        for _ in range(40000):
            b2 = fnext(b2)
            d2 = b2 - a[c2]
            if thr - d2 * d2 <= 0:
                break
            b1 = f32(a[c1] + math.sqrt(thr - d2 * d2))
            for b1k in (fnext(b1, -1), b1, fnext(b1, 1)):
                def at(i):
                    b = [0.0, 0.0, 0.0]
                    b[c1], b[c2], b[tiny] = b1k, b2, a[tiny] + _fval(i)
                    return tuple(b)
                lo, hi = 0, _fbits(1e-4)
                if sq_dist(a, at(hi)) <= thr or sq_dist(a, at(0)) > thr:
                    continue
                while lo < hi:
                    mid = (lo + hi) // 2
                    lo, hi = (lo, mid) if sq_dist(a, at(mid)) > thr else (mid + 1, hi)
                for i in range(max(lo - 64, 0), lo + 64):
                    b = at(i)
                    if (sq_dist(a, b) > thr) == want_add and (sq_dist_other_order(a, b) > thr) != want_add:
                        return tuple(a), b
    raise RuntimeError("no order split found")


def _mirror(pair, sgn):
    """The pair, or both points negated (every difference negates exactly, so the squared distance is the same)."""
    return tuple(tuple(sgn * c for c in p) for p in pair)


def distance_cases() -> list[Case]:
    rng = np.random.default_rng(101)
    out = []
    # dyadic 3-4-5 ties at md = 0.3125 (0.1875^2 + 0.25^2 = 0.3125^2 exactly), with the next float inward and outward, in
    # voxels of both signs; creators in one call with their tie partners, and again across calls
    md = 0.3125
    creators, partners, certs = [], [], []
    for v, (sx, sy) in enumerate([(1, 1), (-1, 1), (1, -1), (-1, -1)]):
        base = (sx * (2.25 + 3 * v), sy * 0.25, 0.5)
        creators.append(base)
        for k in (-1, 0, 1):   # inward, the tie, outward: x = base + 0.1875 moved by k floats away from base
            x = f32(base[0] + sx * 0.1875)
            x = fnext(x, k) if x > 0 else -fnext(-x, k)
            b = (x, base[1] + sy * 0.25, 0.5)
            partners.append(b)
            certs.append(dict(a=base, b=b, md=md, add=k > 0, exact=k == 0))
    one_call = np.concatenate([creators, partners])
    out.append(Case("dyadic_ties_one_call", [_ins(one_call, md)], certs=certs))
    out.append(Case("dyadic_ties_across_calls", [_ins(creators, md), _ins(partners[::-1], md)], certs=certs))
    # mined at the shipped 0.15 inside cell 0 (fine float steps): fl(dx^2 + (dy^2 + dz^2)) one ulp below, equal to and one
    # ulp above fl(0.15 * 0.15), on both signs; the pair again with its points swapped, and a third point at the same spot
    for k in (-1, 0, 1):
        for sgn in (1.0, -1.0):
            a, b = _mirror(mine_near_tie(0.15, k), sgn)
            cert = dict(a=a, b=b, md=0.15, add=k > 0, ulps=k)
            out.append(Case(f"mined_0p15_k{k}_{'pos' if sgn > 0 else 'neg'}", [_ins([a, b]), _ins([b, a, b])], certs=[cert]))
    # the reduction order decides: dx^2 + (dy^2 + dz^2) against (dx^2 + dy^2) + dz^2 on opposite sides of the threshold
    for want in (True, False):
        for sgn in (1.0, -1.0):
            a, b = _mirror(mine_order_split(0.15, want), sgn)
            cert = dict(a=a, b=b, md=0.15, add=want, split=True)
            out.append(Case(f"reduction_order_split_{'add' if want else 'reject'}_{'pos' if sgn > 0 else 'neg'}", [_ins([a, b])],
                            certs=[cert]))
    # md = 0: an exact duplicate is never added (0 > 0 fails), the next float is
    base = np.array([[0.5, 0.5, 0.5], [-3.25, 7.75, 1.5], [12.125, -0.5, -0.25]])
    dup = np.concatenate([base, base, base[:1], [[fnext(0.5), 0.5, 0.5]], base[::-1]])
    out.append(Case("zero_min_distance_duplicates", [_ins(dup, 0.0), _ins(base, 0.0), _ins(_shuffled(rng, base, base + 1e-3), 0.0)]))
    return out


# ---- clamp ------------------------------------------------------------------------------------------------------------
def clamp_cases() -> list[Case]:
    out = []
    for size in (1.0, 0.5):
        # opposite corners of the double-width cell 0: true squared distance up to 12 size^2, clamped to 10 size^2
        c = 0.99 * size
        corners = [(sx * c, sy * c, sz * c) for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)]
        # md just below and just above sqrt(10) size: fl(md^2) below / at-or-above fl(10 size^2)
        lim = 10 * size * size
        md_lo = math.sqrt(10) * size
        while md_lo * md_lo >= lim:
            md_lo = dnext(md_lo, -1)
        md_hi = dnext(md_lo, 1)
        while md_hi * md_hi < lim:
            md_hi = dnext(md_hi, 1)
        for name, md in (("below_sqrt10", md_lo), ("at_sqrt10", md_hi), ("3p3", 3.3 * size), ("3p0", 3.0 * size)):
            out.append(Case(f"clamp_cell0_size{size}_md_{name}", [_ins(corners, md), _ins(corners[::-1], md)], size=size,
                            certs=[dict(a=corners[0], b=corners[-1], md=md, add=lim > md * md, clamp=True)]))
    return out


# ---- cap and the min_num_points gate ------------------------------------------------------------------------------------
def _grid_in_voxel(v, n, size=1.0, offset=0.02):
    """n points of voxel v (non-negative key) on a grid of pitch >= 0.09 size: farther than 0.05 size from each other."""
    m = max(int(math.ceil(n ** (1 / 3) - 1e-9)), 1)
    step = min(0.09, 0.95 / m)
    idx = np.stack(np.unravel_index(np.arange(n), (m, m, m)), 1)
    return (np.asarray(v, np.float64) + offset + step * idx) * size


def cap_cases() -> list[Case]:
    rng = np.random.default_rng(7)
    out = []
    groups = [_grid_in_voxel((2 * j + 1, 3, 5), n) for j, n in enumerate((19, 20, 21, 33, 64, 1000))]
    others = [_grid_in_voxel((2 * j + 1, 9, 5), 3) for j in range(40)]
    out.append(Case("cap_offered_in_one_call", [_ins(_shuffled(rng, *groups, *others), 0.05)]))
    v = _grid_in_voxel((4, 4, 4), 24)
    out.append(Case("cap_filled_across_calls", [_ins(v[:CAP - 1], 0.05), _ins(v[CAP - 1:CAP + 2], 0.05), _ins(v[CAP + 2:], 0.05)]))
    keys = np.array([[4, 4, 4], [6, 6, 6]], np.int16)
    xyz = np.zeros((2, CAP, 3), np.float32)
    xyz[0, :CAP - 1] = v[:CAP - 1]
    xyz[1, :CAP] = _grid_in_voxel((6, 6, 6), CAP)
    out.append(Case("cap_uploaded_full_and_one_short", [("upload", keys, np.array([CAP - 1, CAP], np.int32), xyz),
                                                          _ins(_shuffled(rng, v[CAP - 1:], _grid_in_voxel((6, 6, 6), 30)[CAP:]), 0.05)]))
    # min_num_points -1, 0 and 3 against voxels holding exactly 2 and 3 points
    for mnp in (-1, 0, 3):
        two, three = _grid_in_voxel((1, 1, 1), 5), _grid_in_voxel((3, 1, 1), 6)
        keys = np.array([[1, 1, 1], [3, 1, 1]], np.int16)
        counts = np.array([2, 3], np.int32)
        xyz = np.zeros((2, CAP, 3), np.float32)
        xyz[0, :2], xyz[1, :3] = two[:2], three[:3]
        fresh = _grid_in_voxel((5, 1, 1), 4)
        out.append(Case(f"gate_mnp{mnp}_uploaded", [("upload", keys, counts, xyz), _ins(_shuffled(rng, two[2:], three[3:], fresh), 0.05, mnp)]))
        out.append(Case(f"gate_mnp{mnp}_inserted", [_ins(np.concatenate([two[:2], three[:3]]), 0.05),
                                                     _ins(_shuffled(rng, two[2:], three[3:], fresh), 0.05, mnp)]))
    return out


def empty_voxel_cases() -> list[Case]:
    """Voxels present with 0 points: found, so the first point offered meets sq_min = 10 size^2 (no point lowers it)."""
    out = []
    for size in (1.0, 0.5):
        keys = np.array([[2, 3, 4], [5, 5, 5], [-1, 0, 2]], np.int16)
        counts = np.array([0, 1, 0], np.int32)
        xyz = np.zeros((3, CAP, 3), np.float32)
        xyz[1, 0] = np.array([5.5, 5.5, 5.5]) * size
        pts = np.array([[2.5, 3.5, 4.5], [2.9, 3.1, 4.2], [5.1, 5.2, 5.3], [-1.5, 0.5, 2.5], [7.5, 7.5, 7.5]]) * size
        lim = 10 * size * size
        md_at = math.sqrt(lim)
        while md_at * md_at < lim:
            md_at = dnext(md_at, 1)
        md_below = dnext(md_at, -1)
        while md_below * md_below >= lim:
            md_below = dnext(md_below, -1)
        for md_name, md in (("at_sqrt10", md_at), ("4", 4.0 * size), ("below_sqrt10", md_below), ("0p15", 0.15)):
            for mnp in (0, -1, 1):
                out.append(Case(f"empty_voxel_size{size}_md_{md_name}_mnp{mnp}", [("upload", keys, counts, xyz), _ins(pts, md, mnp, 1.0)],
                                size=size, empty_voxels=True))
    return out


# ---- keys -------------------------------------------------------------------------------------------------------------
def key_cases() -> list[Case]:
    rng = np.random.default_rng(3)
    out = []
    # the double lies below a voxel face, its float rounding on it (and across), both signs; -0.0
    face = []
    for f in (1.0, 2.0, 7.0, 100.0):
        for s in (1, -1):
            face.append((s * dnext(f, -1), 0.5, 0.5))
            face.append((s * dnext(f, 1), 2.5, 0.5))
            face.append((s * fnext(f, -1), 4.5, 0.5))
    face += [(-0.0, 6.5, 0.5), (0.0, 6.5, 0.75), (-0.0, -0.0, -0.0), (0.5, -0.0, 0.25)]
    out.append(Case("key_float_rounding_at_faces", [_ins(face, 0.05)]))
    out.append(Case("key_float_rounding_at_faces_half", [_ins(face, 0.05)], size=0.5))
    # |q| at 32764.5, 32765, 32767.5, 32768 and 40000 on every axis and both signs: the wrap to int16
    big = []
    for q in (32764.5, 32765.0, 32765.5, 32766.5, 32767.5, 32768.0, 32768.5, 40000.0, 65535.5, 65536.5, 1e6 + 0.5, 2.0 ** 31 - 128):
        for s in (1, -1):
            big += [(s * q, 0.5, 0.5), (0.5, s * q, 0.5), (0.5, 0.5, s * q), (s * q, s * q, s * q)]
    out.append(Case("key_range_and_wrap", [_ins(big, 0.05), _ins(np.asarray(big) + 0.25, 0.05)]))
    # points 65536 voxels apart share a voxel (far apart, so 10 size^2 is the distance the second point meets)
    alias = [(5.5, 0.5, 0.5), (65541.5, 0.5, 0.5), (-65530.5, 0.5, 0.5), (5.5, 65536.5, 0.5), (5.25, 0.25, 131072.25)]
    out.append(Case("key_aliases_65536_apart", [_ins(alias, 0.05), _ins(alias[::-1], 0.05), _ins(alias, 3.2)]))
    # NaN, +-inf, |q| >= 2^31 and values past FLT_MAX in each axis: dropped, the finite points around them are not
    bad = []
    for v in (math.nan, math.inf, -math.inf, 2.0 ** 31, -2.0 ** 31, 1e300, 3.5e38, -1e39):
        for ax in range(3):
            p = [1.5, 2.5, 3.5]
            p[ax] = v
            bad.append(p)
    good = rng.uniform(-4, 4, (40, 3))
    out.append(Case("key_nan_inf_and_huge", [_ins(_shuffled(rng, bad, good), 0.05), _ins(bad, 0.05)]))
    return out


# ---- probe chains, growth and eviction of chained voxels ---------------------------------------------------------------
def chain_keys(n_near=100, n_far=100):
    """Voxel keys whose home slot under mask 2047 is one of the last four (so also under mask 1023): near ones within 30
    voxels of the origin on every axis, far ones 100-140 voxels out along x."""
    g = np.stack(np.meshgrid(np.arange(-140, 141), np.arange(-30, 31), np.arange(-30, 31), indexing="ij"), -1).reshape(-1, 3)
    h = np.array([hash_key(*k) for k in g[::997].tolist()], np.int64)          # spot check of the vectorised hash below
    u = g.astype(np.int64) & 0xFFFFFFFF
    v = ((u[:, 0] * 73856093) & 0xFFFFFFFF) ^ ((u[:, 1] * 19349669) & 0xFFFFFFFF) ^ ((u[:, 2] * 83492791) & 0xFFFFFFFF)
    v ^= v >> 16
    v = (v * 0x85EBCA6B) & 0xFFFFFFFF
    v ^= v >> 13
    assert np.array_equal(v[::997], h)
    hit = g[(v & 2047) >= 2044]
    near = [tuple(k) for k in hit[np.abs(hit[:, 0]) <= 30][:n_near].tolist()]
    far = [tuple(k) for k in hit[np.abs(hit[:, 0]) >= 100][:n_far].tolist()]
    assert len(near) == n_near and len(far) == n_far
    return near, far


def _voxel_points(keys, n, size=1.0, seed=0):
    """n points per voxel (sign-correct inside the voxel, so truncation keeps them there), spaced more than 0.05 apart."""
    rng = np.random.default_rng(seed)
    out = []
    for k in keys:
        base = _grid_in_voxel((0, 0, 0), n, offset=0.03) + rng.uniform(0.0, 0.004, (n, 3))   # off the lattice: no distance ties
        base = base[rng.permutation(n)]
        sgn = np.where(np.asarray(k) < 0, -1.0, 1.0)
        out.append((np.asarray(k, np.float64) + sgn * base) * size)
    return np.concatenate(out)


def chain_cases() -> list[Case]:
    rng = np.random.default_rng(17)
    near, far = chain_keys()
    chained = [k for pair in zip(near, far) for k in pair]          # every second chained voxel is a far one
    pts = _voxel_points(chained, 20, seed=1)
    others = [(x, y, 9) for x in range(-10, 10) for y in range(-10, 10)][:400]
    more = _voxel_points(others, 2, seed=2)
    wrap = [(32765, 0, 0), (32766, 0, 0), (-32765, 1, 0), (-32766, 1, 0)]
    wrap_pts = _voxel_points(wrap, 20, seed=3)
    probes_near = _voxel_points(near[:40], 2, seed=4) + np.random.default_rng(5).uniform(0.005, 0.02, (80, 3))
    probes_wrap = np.array([[32764.61, 0.43, 0.52], [32764.93, 0.21, 0.71], [-32764.57, 1.46, 0.53], [-32764.87, 1.91, 0.33]])
    probes = np.concatenate([probes_near, probes_wrap])
    out = []
    # 200 chained voxels on a 1024-slot table (the chain wraps to slot 0), then 400 more in one insert: the map grows past
    # 512 voxels and the table to 2048 slots, where the chained keys still collide
    grow = [_ins(_shuffled(rng, pts), 0.05), _ins(_shuffled(rng, more, wrap_pts), 0.05)]
    out.append(Case("chain_wraps_then_grows", grow, probes=probes))
    # every second chained voxel evicted (the far ones), then re-inserted; then the same through growth in one call
    evict = grow + [("remove", (0.0, 0.0, 0.0), 60.0), _ins(_shuffled(rng, pts, wrap_pts), 0.05)]
    out.append(Case("chain_evict_every_second_then_reinsert", evict, probes=probes))
    out.append(Case("chain_grow_inside_one_insert", [_ins(_shuffled(rng, pts, more, wrap_pts), 0.05), ("remove", (0.0, 0.0, 0.0), 60.0),
                                                      _ins(_shuffled(rng, pts[:2000], wrap_pts), 0.05)], probes=probes))
    return out


# ---- eviction ---------------------------------------------------------------------------------------------------------
def eviction_cases() -> list[Case]:
    rng = np.random.default_rng(23)
    out = []
    # first points at exactly 2.5 from the origin (1.5, 2, 0), the next float beyond it, and a far first point with near
    # points after it
    firsts = [(1.5, 2.0, 0.0), (fnext(1.5), 2.0, 0.0), (0.0, 1.5, 2.0), (0.0, -1.5, -fnext(2.0)), (-2.0, 0.0, 1.5)]
    later = [(1.25, 0.25, 0.25), (0.25, 1.25, 1.25), (0.25, -1.25, -1.25), (-1.25, 0.25, 1.25)]
    far_first = [(3.9, 0.5, 0.5), (3.1, 0.5, 0.5), (3.2, 0.25, 0.75)]
    fill = [_ins(firsts, 0.05), _ins(later, 0.05), _ins(far_first, 0.05)]
    for dist in (2.5, dnext(2.5, -1), dnext(2.5, 1), 3.5):
        out.append(Case(f"evict_at_distance_{dist!r}", fill + [("remove", (0.0, 0.0, 0.0), dist)]))
    cloud = rng.uniform(-6, 6, (3000, 3))
    out.append(Case("evict_zero_distance", [_ins(cloud, 0.05), _ins([(0.5, 0.5, 0.5)], 0.05), ("remove", (0.5, 0.5, 0.5), 0.0),
                                            ("remove", (0.5, 0.5, 0.5), 0.0)]))
    out.append(Case("evict_non_dyadic_location", [_ins(cloud, 0.05), ("remove", (0.1, 0.2, 0.3), 3.7), _ins(cloud[::-1], 0.05),
                                                  ("remove", (-1.3, 0.7, 2.9), 2.2)]))
    out.append(Case("evict_everything_then_insert", [_ins(cloud, 0.05), ("remove", (100.0, 0.0, 0.0), 1.0), _ins(cloud[:500], 0.05),
                                                     ("remove", (0.0, 0.0, 0.0), 1e9), _ins(cloud, 0.05)]))
    return out


@functools.lru_cache(maxsize=None)
def all_cases() -> list[Case]:
    return distance_cases() + clamp_cases() + cap_cases() + empty_voxel_cases() + key_cases() + chain_cases() + eviction_cases()


def defined(xyz, size: float) -> np.ndarray:
    """The rows whose key the reference's cast defines (|float(x) / size| < 2^31, not NaN): what the oracle may be fed."""
    f = np.asarray(xyz, np.float64).reshape(-1, 3)
    ok = [all(short_key(f32(c) / size) is not None for c in row) for row in f.tolist()]
    return f[np.asarray(ok, bool)] if len(ok) else f
