"""A plain restatement of the LIO voxel map: addPointToMap / addPointsToMap with the cloud addPointToPcl publishes
(src/lioOptimization.cpp:400-446,520-554,1346-1355) and removePointsFarFromLocation (:556-572), one point at a time.

Stored positions are numpy float32 (rgbPoint keeps position.cast<float>()); everything else is a Python float, one IEEE
double rounding per operation and nothing fused:
  * key: static_cast<short>(float(x) / size) as g++ compiles it for x86-64, (int16)(int32)trunc(q) for |q| < 2^31.  NaN,
    +-inf and larger quotients leave the reference's cast undefined; the point is dropped (DESIGN.md section 5);
  * squared distance: dx^2 + (dy^2 + dz^2) of the widened floats (Eigen's fixed-size reduction order);
  * a point goes into a found voxel when it is not full, min(10 size^2, distances) > min_distance_points^2 and
    (min_num_points <= 0 or the voxel holds at least min_num_points), and is then published; a point whose voxel is absent
    creates it (when min_num_points <= 0) and is not published.  An empty voxel that is present (a map uploaded with
    count 0) is found: no distance lowers 10 size^2;
  * eviction: a voxel goes when its first point is farther than `distance`, !(d^2 <= distance^2) evaluated as
    d2 > distance * distance; surviving voxels keep their order.  An empty voxel has no first point (the reference reads
    points[0]); it goes.

hash_key restates srl_device.cuh's slot hash in uint32 so that cases can mine colliding keys.  The Fraction helpers certify
crafted ties: the double evaluation is exact, or lies a stated number of ulps from the threshold.
"""
from __future__ import annotations

from fractions import Fraction

import numpy as np

I32 = 2.0 ** 31
M32 = 0xFFFFFFFF


def f32(x) -> float:
    """The float32 rounding of a double (rgbPoint's cast), as a Python float."""
    with np.errstate(over="ignore", invalid="ignore"):
        return float(np.float32(x))


def short_key(q: float):
    """static_cast<short>(q) on x86-64 for |q| < 2^31 (truncation to int32, low 16 bits); None where it is undefined."""
    if not abs(q) < I32:
        return None
    k = int(q)
    return ((k + 0x8000) & 0xFFFF) - 0x8000


def voxel_of(fpos, size: float):
    """The voxel key of a stored (float) position, or None when the point is dropped."""
    ks = tuple(short_key(c / size) for c in fpos)
    return None if None in ks else ks


def hash_key(x: int, y: int, z: int) -> int:
    """srl_device.cuh hash_key on the sign-extended int16 key, in uint32 arithmetic."""
    h = ((x & M32) * 73856093 & M32) ^ ((y & M32) * 19349669 & M32) ^ ((z & M32) * 83492791 & M32)
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & M32
    h ^= h >> 13
    return h


def sq_dist(a, b) -> float:
    """(a - b).squaredNorm() of two widened float positions: dx^2 + (dy^2 + dz^2)."""
    dx, dy, dz = a[0] - b[0], a[1] - b[1], a[2] - b[2]
    return dx * dx + (dy * dy + dz * dz)


def intensity(z: float, translation_z: float) -> float:
    """addPointToPcl's intensity: 50 * (cloudTemp.z - translation.z()) in double, rounded once to float."""
    return f32(50.0 * (z - translation_z))


class MapRef:
    """voxelHashMap + addPointsToMap + removePointsFarFromLocation, one point at a time."""

    def __init__(self, voxel_size: float = 1.0, cap: int = 20):
        self.size, self.cap = float(voxel_size), int(cap)
        self.vox: dict[tuple, list] = {}       # key -> stored (x, y, z) float positions, in insertion order

    def load(self, keys, counts, xyz):
        for k, c, p in zip(np.asarray(keys).tolist(), np.asarray(counts).tolist(), np.asarray(xyz, np.float32)):
            self.vox[tuple(k)] = [tuple(float(v) for v in p[i]) for i in range(c)]

    @property
    def num_points(self) -> int:
        return sum(len(v) for v in self.vox.values())

    def add_point(self, xyz, min_distance_points: float, min_num_points: int):
        """addPointToMap for one point: (stored, published, the stored position)."""
        p = tuple(f32(c) for c in xyz)
        key = voxel_of(p, self.size)
        if key is None:
            return False, False, p
        pts = self.vox.get(key)
        if pts is None:
            if min_num_points <= 0:
                self.vox[key] = [p]
                return True, False, p
            return False, False, p
        if len(pts) >= self.cap:
            return False, False, p
        sq_min = 10 * self.size * self.size
        for q in pts:
            d = sq_dist(q, p)
            if d < sq_min:
                sq_min = d
        if sq_min > min_distance_points * min_distance_points and (min_num_points <= 0 or len(pts) >= min_num_points):
            pts.append(p)
            return True, True, p
        return False, False, p

    def add_points(self, xyz, min_distance_points: float = 0.15, min_num_points: int = 0, translation_z: float = 0.0):
        """addPointsToMap: (points stored, (n_published, 4) float32 x, y, z, intensity in sweep order)."""
        added, cloud = 0, []
        for row in np.asarray(xyz, np.float64).reshape(-1, 3).tolist():
            stored, published, p = self.add_point(row, min_distance_points, min_num_points)
            added += stored
            if published:
                cloud.append((p[0], p[1], p[2], intensity(p[2], translation_z)))
        return added, np.array(cloud, np.float32).reshape(-1, 4)

    def remove_far(self, location, distance: float) -> int:
        lx, ly, lz = (float(v) for v in np.asarray(location, np.float64).reshape(3))
        lim = distance * distance
        gone = [k for k, pts in self.vox.items() if not pts or sq_dist(pts[0], (lx, ly, lz)) > lim]
        for k in gone:
            del self.vox[k]
        return len(gone)

    def as_dict(self):
        return {k: np.array(v, np.float32).reshape(-1, 3) for k, v in self.vox.items()}


# ---- certificates of crafted ties -------------------------------------------------------------------------------------
def exact_sq(a, b) -> Fraction:
    """The exact squared distance of two float positions."""
    return sum((Fraction(x) - Fraction(y)) ** 2 for x, y in zip(a, b))


def ulps_from(x: float, t: float) -> int:
    """The signed number of doubles from t to x; both non-negative and finite."""
    bits = np.array([x, t], np.float64).view(np.int64)
    return int(bits[0]) - int(bits[1])


def sq_dist_other_order(a, b) -> float:
    """(dx^2 + dy^2) + dz^2: the reduction order the device and the reference do not use."""
    dx, dy, dz = a[0] - b[0], a[1] - b[1], a[2] - b[2]
    return (dx * dx + dy * dy) + dz * dz


def certify_pair(a, b, min_distance_points: float) -> dict:
    """What the double evaluation decides for two stored positions against min_distance_points^2, with the exact values."""
    thr = min_distance_points * min_distance_points
    sq = sq_dist(a, b)
    return dict(sq=sq, thr=thr, ulps=ulps_from(sq, thr), sq_exact=Fraction(sq) == exact_sq(a, b),
                thr_exact=Fraction(thr) == Fraction(min_distance_points) ** 2, other_order=sq_dist_other_order(a, b))
