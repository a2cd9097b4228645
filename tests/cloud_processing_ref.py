"""Plain restatement of cloudProcessing (src/cloudProcessing.cpp) and of the point pops of getMeasurements
(src/lioOptimization.cpp:719-723, 759-763), with libstdc++'s std::sort restated as it runs.

  introsort(keys)            std::sort's permutation: __introsort_loop (depth limit 2*floor(log2 n), pivot by
                             __move_median_to_first(first, first+1, mid, last-1), __unguarded_partition), __partial_sort once the
                             depth limit is spent, __final_insertion_sort with threshold 16.  partition="scan" replaces the
                             sequential partition with the two-scan form the device runs (partition_scan).
  CloudProcessingRef         the four handlers, their carried state (last_end_time, given_offset_time, sweep_id) and the queue
  livox_records / cloud2     seeded wire-format messages: 19-byte packed Livox CustomPoint records, PointCloud2 data per lidar type
  SortProbe / ReferenceCP    ctypes bindings of oracle/_ref/libsrl_sort_probe.so and libsrl_cloud_processing_ref.so
"""
from __future__ import annotations

import ctypes as C
import math
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")

LIVOX, VELO, OUST, ROBO = 1, 2, 3, 4
SEC, MS, US, NS = 0, 1, 2, 3
THRESHOLD = 16


# ---------------------------------------------------------------------------------------------- libstdc++ std::sort
class _Sorter:
    """std::sort over a list of (key, index) pairs, comparing keys with <.  heapsorts counts __partial_sort calls."""

    def __init__(self, a, partition="seq"):
        self.a = a
        self.heapsorts = 0
        self.partition = self._partition_seq if partition == "seq" else self._partition_scan

    def lt(self, i, j):
        return self.a[i][0] < self.a[j][0]

    def swap(self, i, j):
        a = self.a
        a[i], a[j] = a[j], a[i]

    def move_median_to_first(self, result, a, b, c):
        if self.lt(a, b):
            if self.lt(b, c):
                self.swap(result, b)
            elif self.lt(a, c):
                self.swap(result, c)
            else:
                self.swap(result, a)
        elif self.lt(a, c):
            self.swap(result, a)
        elif self.lt(b, c):
            self.swap(result, c)
        else:
            self.swap(result, b)

    def _partition_seq(self, first, last, pivot):
        a, p = self.a, self.a[pivot][0]
        while True:
            while a[first][0] < p:
                first += 1
            last -= 1
            while p < a[last][0]:
                last -= 1
            if not first < last:
                return first
            a[first], a[last] = a[last], a[first]
            first += 1

    def _partition_scan(self, first, last, pivot):
        return partition_scan(self.a, first, last, self.a[pivot][0])

    # __adjust_heap / __push_heap / __make_heap / __sort_heap over a[first:first+len]
    def _push_heap(self, first, hole, top, value):
        a = self.a
        parent = (hole - 1) // 2
        while hole > top and a[first + parent][0] < value[0]:
            a[first + hole] = a[first + parent]
            hole = parent
            parent = (hole - 1) // 2
        a[first + hole] = value

    def _adjust_heap(self, first, hole, length, value):
        a = self.a
        top = hole
        second = hole
        while second < (length - 1) // 2:
            second = 2 * (second + 1)
            if a[first + second][0] < a[first + second - 1][0]:
                second -= 1
            a[first + hole] = a[first + second]
            hole = second
        if (length & 1) == 0 and second == (length - 2) // 2:
            second = 2 * (second + 1)
            a[first + hole] = a[first + second - 1]
            hole = second - 1
        self._push_heap(first, hole, top, value)

    def heapsort(self, first, last):
        """__partial_sort(first, last, last) = __heap_select (here only __make_heap) + __sort_heap"""
        self.heapsorts += 1
        a = self.a
        length = last - first
        if length >= 2:
            parent = (length - 2) // 2
            while True:
                self._adjust_heap(first, parent, length, a[first + parent])
                if parent == 0:
                    break
                parent -= 1
        while last - first > 1:
            last -= 1
            value = a[last]
            a[last] = a[first]
            self._adjust_heap(first, 0, last - first, value)

    def introsort_loop(self, first, last, depth):
        while last - first > THRESHOLD:
            if depth == 0:
                self.heapsort(first, last)
                return
            depth -= 1
            mid = first + (last - first) // 2
            self.move_median_to_first(first, first + 1, mid, last - 1)
            cut = self.partition(first + 1, last, first)
            self.introsort_loop(cut, last, depth)
            last = cut

    def insertion_sort(self, first, last):
        a = self.a
        for i in range(first + 1, last):
            v = a[i]
            j = i
            while j > first and v[0] < a[j - 1][0]:
                a[j] = a[j - 1]
                j -= 1
            a[j] = v

    def sort(self):
        n = len(self.a)
        if n == 0:
            return
        self.introsort_loop(0, n, 2 * (n.bit_length() - 1))
        # __final_insertion_sort: __insertion_sort on the first 16, __unguarded_linear_insert for the rest; both are the same
        # stable insertion, and the partitions put a sentinel in front of every element past the first 16
        self.insertion_sort(0, n)


def partition_scan(a, first, last, p):
    """__unguarded_partition(first, last, pivot p) in two scans and a scatter.  A = the positions in [first, last) whose key is
    >= p, left to right; B = those whose key is <= p, right to left.  The sequential loop swaps A[k] <-> B[k] for exactly the k
    below K, the first k where A[k] >= B[k] (or one list runs out), and returns min(A[K], B[K-1])."""
    A = [i for i in range(first, last) if not a[i][0] < p]
    B = [i for i in range(last - 1, first - 1, -1) if not p < a[i][0]]
    K = 0
    while K < len(A) and K < len(B) and A[K] < B[K]:
        K += 1
    for k in range(K):
        a[A[k]], a[B[k]] = a[B[k]], a[A[k]]
    cut_a = A[K] if K < len(A) else last
    cut_b = B[K - 1] if K > 0 else last
    return min(cut_a, cut_b)


def introsort(keys, partition="seq", return_heapsorts=False):
    """std::sort's permutation of `keys` (perm[p] = the index of the key that ends at p)."""
    s = _Sorter([(k, i) for i, k in enumerate(keys)], partition)
    s.sort()
    perm = np.array([i for _, i in s.a], np.int32)
    return (perm, s.heapsorts) if return_heapsorts else perm


def median_of_3_killer(n):
    """Keys that drive libstdc++'s median-of-3 quicksort to its depth limit, so the heapsort fallback runs: McIlroy's adversary
    ("A killer adversary for quicksort", 1999) played against the restated sort.  Every key starts as "gas" (above all others);
    when two gas keys meet, the one not last seen as the pivot candidate is frozen at the next solid value.  The frozen values,
    with the remaining gas numbered last, answer every comparison the sort made the same way, so the same sort reruns the
    same bad partitions."""
    gas = float(n)
    val = [gas] * n
    state = {"solid": 0, "cand": -1}

    def freeze(i):
        val[i] = float(state["solid"])
        state["solid"] += 1

    def lt(i, j):   # identities i, j
        if val[i] == gas and val[j] == gas:
            freeze(j if i == state["cand"] else i)
        if val[i] == gas:
            state["cand"] = i
        elif val[j] == gas:
            state["cand"] = j
        return val[i] < val[j]

    class _Stop(Exception):
        pass

    class _Adv(_Sorter):
        def lt(self, i, j):
            return lt(self.a[i][1], self.a[j][1])

        def _partition_seq(self, first, last, pivot):
            a, pk = self.a, self.a[pivot][1]
            while True:
                while lt(a[first][1], pk):
                    first += 1
                last -= 1
                while lt(pk, a[last][1]):
                    last -= 1
                if not first < last:
                    return first
                a[first], a[last] = a[last], a[first]
                first += 1

        def heapsort(self, first, last):
            raise _Stop

    try:
        _Adv([(0.0, i) for i in range(n)]).sort()
    except _Stop:
        pass
    out = np.array(val)
    rest = np.flatnonzero(out == gas)
    out[rest] = state["solid"] + np.arange(len(rest))
    return out


# ---------------------------------------------------------------------------------------------- wire formats
LIVOX_STRIDE = 19


def livox_dtype(stride=LIVOX_STRIDE):
    return np.dtype({"names": ["offset_time", "x", "y", "z", "reflectivity", "tag", "line"],
                     "formats": ["<u4", "<f4", "<f4", "<f4", "u1", "u1", "u1"],
                     "offsets": [0, 4, 8, 12, 16, 17, 18], "itemsize": stride})


# PointCloud2 layouts: (point_step, offsets of x, y, z, time field, ring), the time field's and ring's numpy types.  The velodyne
# and robosense drivers' packed layouts put the time field off its natural alignment.
CLOUD_LAYOUTS = {
    VELO: (22, (0, 4, 8, 18, 16), "<f4", "<u2"),
    OUST: (48, (0, 4, 8, 20, 26), "<u4", "u1"),
    ROBO: (26, (0, 4, 8, 18, 16), "<f8", "<u2"),
}


def cloud_dtype(lidar_type):
    step, off, tt, rt = CLOUD_LAYOUTS[lidar_type]
    return np.dtype({"names": ["x", "y", "z", "time", "ring"], "formats": ["<f4", "<f4", "<f4", tt, rt],
                     "offsets": list(off), "itemsize": step})


def time_unit_scale(time_unit):
    """setTimeUnit: a double holding the float literal"""
    return float(np.float32({SEC: 1.e3, MS: 1., US: 1.e-3, NS: 1.e-6}.get(time_unit, 1.)))


# ---------------------------------------------------------------------------------------------- the handlers
class CloudProcessingRef:
    """cloudProcessing with its point_buffer.  Queue entries: (x, y, z, relative_time, timestamp) as Python floats."""

    def __init__(self, lidar_type, n_scans, scan_rate, time_unit, blind, point_filter_num):
        self.lidar_type, self.N_SCANS, self.SCAN_RATE = lidar_type, n_scans, scan_rate
        self.scale = time_unit_scale(time_unit)
        self.blind, self.f = float(blind), int(point_filter_num)
        self.last_end_time = -1.0
        self.given_offset_time = False
        self.sweep_id = 0
        self.queue = []

    def getSweepInterval(self):
        return 1 / float(self.SCAN_RATE)

    def _outside_blind(self, x, y, z):
        return x * x + y * y + z * z > self.blind * self.blind

    def livoxHandler(self, rec, stamp):
        """rec: a livox_dtype() array.  Returns the number of points appended; an empty result appends nothing and leaves
        last_end_time (the reference reads back() of an empty vector there)."""
        sc = self.scale
        x, y, z = rec["x"], rec["y"], rec["z"]
        line, tag, ot = rec["line"].tolist(), rec["tag"].tolist(), rec["offset_time"].tolist()
        x64, y64, z64 = x.tolist(), y.tolist(), z.tolist()
        # float differences of each record and the raw record before it, widened as std::abs(float) > 1e-7 compares them
        dx, dy, dz = (np.abs(np.diff(c)).astype(np.float64).tolist() for c in (x, y, z))
        cand = []
        for i in range(1, len(rec)):
            xi, yi, zi = x64[i], y64[i], z64[i]
            # IS_VALID's unqualified abs resolves to the float overload (pinned against the compiled reference)
            if line[i] < self.N_SCANS and not abs(xi) > 1e8 and not abs(yi) > 1e8 and not abs(zi) > 1e8 and xi > 0.7:
                if xi > 2.0 and ((tag[i] & 0x03) != 0 or (tag[i] & 0x0C) != 0):
                    continue
                rel = float(ot[i]) * sc
                if dx[i - 1] > 1e-7 or dy[i - 1] > 1e-7 or dz[i - 1] > 1e-7:
                    cand.append((xi, yi, zi, rel, rel / 1000.0 + stamp))
        if not cand:
            return 0
        perm = introsort([c[3] for c in cand])
        pts = [cand[j] for j in perm]
        n0 = len(self.queue)
        for k, p in enumerate(pts):
            if (k + 1) % self.f != 0:
                continue
            if self._outside_blind(p[0], p[1], p[2]):
                self.queue.append(p)
        self.last_end_time = stamp + pts[-1][3] / 1000.0
        return len(self.queue) - n0

    def process(self, cloud, stamp):
        """cloud: a cloud_dtype(lidar_type) array.  Raises ValueError where the reference is undefined (a ring >= N_SCANS on the
        yaw path, a NaN sort key); nothing is appended then and no state changes."""
        n = len(cloud)
        if n == 0:
            self.sweep_id += 1
            return 0
        sc, robo = self.scale, self.lidar_type == ROBO
        t = cloud["time"]
        given = bool(t[n - 1] > 0)
        xs, ys, zs = (cloud[c].astype(np.float64) for c in ("x", "y", "z"))
        if given:
            if any(math.isnan(float(v)) for v in t):
                raise ValueError("NaN time field")
            perm = introsort([float(v) for v in t])
            dt_last = float(t[perm[-1]]) * sc
            front = float(t[perm[0]])
            out = []
            for i, j in enumerate(perm):
                if i % self.f != 0:
                    continue
                x, y, z = float(xs[j]), float(ys[j]), float(zs[j])
                rel = (float(t[j]) - front) * sc if robo else float(t[j]) * sc
                if self._outside_blind(x, y, z):
                    ts = rel / 1000.0 + stamp
                    if ts > self.last_end_time:
                        out.append((x, y, z, rel, ts))
        else:
            omega = 0.361 * self.SCAN_RATE
            rings = cloud["ring"]
            if n and int(rings.max()) >= self.N_SCANS:
                raise ValueError("ring >= N_SCANS")
            first = {}
            full = []
            for i in range(n):
                x, y, z = float(xs[i]), float(ys[i]), float(zs[i])
                layer = int(rings[i])
                yaw = math.atan2(y, x) * 57.2957
                if layer not in first:
                    first[layer] = yaw
                    full.append((x, y, z, 0.0, 0.0))
                    continue
                yf = first[layer]
                rel = (yf - yaw) / omega if yaw <= yf else (yf - yaw + 360.0) / omega
                full.append((x, y, z, rel, rel / 1000.0 + stamp))
            if any(math.isnan(p[3]) for p in full):
                raise ValueError("NaN relative_time")
            perm = introsort([p[3] for p in full])
            dt_last = full[perm[-1]][3]
            out = [full[j] for i, j in enumerate(perm) if i % self.f == 0 and full[j][4] > self.last_end_time]
        self.queue.extend(out)
        self.given_offset_time = given
        self.last_end_time = stamp + dt_last / 1000.0
        self.sweep_id += 1
        return len(out)

    def cut(self, t):
        """getMeasurements' pops: while the queue is not empty and front().timestamp < t.  Returns the popped entries."""
        k = 0
        while k < len(self.queue) and self.queue[k][4] < t:
            k += 1
        popped, self.queue = self.queue[:k], self.queue[k:]
        return popped


def as_arrays(entries):
    a = np.array(entries, np.float64).reshape(-1, 5)
    return np.ascontiguousarray(a[:, :3]), np.ascontiguousarray(a[:, 3]), np.ascontiguousarray(a[:, 4])


# ---------------------------------------------------------------------------------------------- seeded messages
def livox_records(seed, n, n_lines=6, stamp_ns_span=100_000_000, dup_every=9, ties=4, big=False, stride=LIVOX_STRIDE):
    """A Livox message: n records; offset_time in ns rising in groups of `ties` records (several lines fire together), every
    dup_every-th record repeats the one before it, some records fall to the x > 0.7, tag and line gates, x values sit on 0.7 and
    2.0, and with big=True some coordinates sit around 1e8 and past 2^31."""
    rng = np.random.default_rng(seed)
    r = np.zeros(n, livox_dtype(stride))
    base = np.sort(rng.integers(0, stamp_ns_span, (n + ties - 1) // ties, dtype=np.uint32))
    ot = np.repeat(base, ties)[:n]
    # shuffle groups a little so the input is not sorted
    sw = rng.integers(0, n, n // 10)
    ot[sw], ot[sw[::-1]] = ot[sw[::-1]], ot[sw]
    r["offset_time"] = ot
    r["x"] = rng.uniform(-2.0, 40.0, n).astype(np.float32)
    r["y"] = rng.uniform(-20.0, 20.0, n).astype(np.float32)
    r["z"] = rng.uniform(-3.0, 5.0, n).astype(np.float32)
    r["x"][rng.random(n) < 0.05] = np.float32(0.7)
    r["x"][rng.random(n) < 0.05] = np.float32(2.0)
    r["tag"] = rng.choice(np.array([0, 0, 0, 0x10, 0x01, 0x04, 0x02, 0x08], np.uint8), n)
    r["line"] = rng.integers(0, n_lines + 1, n).astype(np.uint8)
    r["reflectivity"] = rng.integers(0, 256, n).astype(np.uint8)
    for i in range(dup_every, n, dup_every):
        for c in ("x", "y", "z"):
            r[c][i] = r[c][i - 1]
    if big:
        m = rng.random(n) < 0.04
        r["y"][m] = rng.choice(np.array([1e8, -1e8, 1.00000008e8, 99999992.0, 2.2e9, -3e9], np.float32), int(m.sum()))
    return r


def cloud2(lidar_type, seed, rows, cols, given=True, scan_rate=10, ns=True, nan_time=False):
    """A rotating-lidar message of rows x cols points, column-major (every ring of a column in turn), as Ouster and Velodyne
    drivers emit: with given=True every ring of a column shares its time (rows-way ties); with given=False the time field is 0.
    Ranges vary from 0.5 m to 60 m so both blind settings cut.  Robosense times are absolute (s), the others relative."""
    rng = np.random.default_rng(seed)
    n = rows * cols
    c = np.zeros(n, cloud_dtype(lidar_type))
    az = np.repeat(np.linspace(0.0, 2 * np.pi, cols, endpoint=False), rows) + rng.normal(0, 1e-4, n)
    el = np.tile(np.linspace(-0.3, 0.3, rows), cols)
    rng_m = rng.uniform(0.5, 60.0, n)
    c["x"] = (rng_m * np.cos(el) * np.cos(az)).astype(np.float32)
    c["y"] = (rng_m * np.cos(el) * np.sin(az)).astype(np.float32)
    c["z"] = (rng_m * np.sin(el)).astype(np.float32)
    c["ring"] = np.tile(np.arange(rows), cols)
    col = np.repeat(np.arange(cols), rows)
    period = 1.0 / scan_rate
    if given:
        if lidar_type == OUST:
            c["time"] = (col * (period * 1e9 / cols)).astype(np.uint32) + 1   # ns
        elif lidar_type == VELO:
            c["time"] = (col * (period / cols)).astype(np.float32) * (1e9 if ns else 1.0)
        else:
            c["time"] = 1.7e9 + col * (period / cols)
        # a few columns out of order
        k = rng.integers(0, cols, max(1, cols // 20))
        for a, b in zip(k, k[::-1]):
            ia, ib = slice(a * rows, (a + 1) * rows), slice(b * rows, (b + 1) * rows)
            ta, tb = c["time"][ia].copy(), c["time"][ib].copy()
            c["time"][ia], c["time"][ib] = tb, ta
        if nan_time:
            c["time"][n // 2] = np.nan
    return c


def yaw_gap_ok(cloud, scan_rate, min_gap):
    """The yaw path's distinct keys (relative_time, ms) lie more than min_gap ms apart, so a device atan2 that moves each key by
    less than min_gap / 2 orders them as glibc's does: checked on the restated keys."""
    omega = 0.361 * scan_rate
    first = {}
    keys = []
    for p in cloud:
        x, y = float(p["x"]), float(p["y"])
        yaw = math.atan2(y, x) * 57.2957
        r = int(p["ring"])
        if r not in first:
            first[r] = yaw
            keys.append(0.0)
            continue
        yf = first[r]
        keys.append((yf - yaw) / omega if yaw <= yf else (yf - yaw + 360.0) / omega)
    k = np.unique(np.array(keys))
    if len(k) < 2:
        return True
    return bool(np.all(np.diff(k) > min_gap))


# ---------------------------------------------------------------------------------------------- compiled references
def _load(name):
    p = os.path.join(REF_DIR, name)
    return C.CDLL(p) if os.path.exists(p) else None


class SortProbe:
    def __init__(self):
        self.L = _load("libsrl_sort_probe.so")

    def perm(self, keys, dtype):
        k = np.ascontiguousarray(keys, dtype)
        out = np.empty(len(k), np.int32)
        fn = {np.float64: self.L.srl_sort_perm_f64, np.float32: self.L.srl_sort_perm_f32, np.uint32: self.L.srl_sort_perm_u32}[dtype]
        fn(C.c_void_p(k.ctypes.data), C.c_int64(len(k)), C.c_void_p(out.ctypes.data))
        return out


class ReferenceCP:
    """the reference's own cloudProcessing (oracle/_ref/libsrl_cloud_processing_ref.so)"""

    def __init__(self, lidar_type, n_scans, scan_rate, time_unit, blind, point_filter_num):
        L = self.L = _load("libsrl_cloud_processing_ref.so")
        L.srl_cp_create.restype = C.c_void_p
        L.srl_cp_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int]
        L.srl_cp_destroy.argtypes = [C.c_void_p]
        L.srl_cp_livox.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_double]
        L.srl_cp_process.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_double]
        L.srl_cp_queue_size.restype = C.c_int64
        L.srl_cp_queue_size.argtypes = [C.c_void_p]
        L.srl_cp_drain.restype = C.c_int64
        L.srl_cp_drain.argtypes = [C.c_void_p] * 4
        L.srl_cp_state.argtypes = [C.c_void_p] * 5
        self.lidar_type = lidar_type
        self.h = L.srl_cp_create(lidar_type, n_scans, scan_rate, time_unit, blind, point_filter_num)

    def close(self):
        if self.h:
            self.L.srl_cp_destroy(C.c_void_p(self.h))
            self.h = None

    def livox(self, rec, stamp):
        rec = np.ascontiguousarray(rec)
        self.L.srl_cp_livox(C.c_void_p(self.h), C.c_void_p(rec.ctypes.data), len(rec), rec.dtype.itemsize, stamp)

    def process(self, cloud, stamp):
        cloud = np.ascontiguousarray(cloud)
        off = np.array([cloud.dtype.fields[k][1] for k in ("x", "y", "z", "time", "ring")], np.int32)
        self.L.srl_cp_process(C.c_void_p(self.h), C.c_void_p(cloud.ctypes.data), len(cloud), cloud.dtype.itemsize,
                              C.c_void_p(off.ctypes.data), stamp)

    def drain(self):
        n = self.L.srl_cp_queue_size(C.c_void_p(self.h))
        xyz, rel, ts = np.empty((n, 3)), np.empty(n), np.empty(n)
        self.L.srl_cp_drain(C.c_void_p(self.h), C.c_void_p(xyz.ctypes.data), C.c_void_p(rel.ctypes.data), C.c_void_p(ts.ctypes.data))
        return xyz, rel, ts

    def state(self):
        le, g, s, si = C.c_double(), C.c_int32(), C.c_int32(), C.c_double()
        self.L.srl_cp_state(C.c_void_p(self.h), C.byref(le), C.byref(g), C.byref(s), C.byref(si))
        return le.value, bool(g.value), s.value, si.value


def have_probe():
    return os.path.exists(os.path.join(REF_DIR, "libsrl_sort_probe.so"))


def have_reference():
    return os.path.exists(os.path.join(REF_DIR, "libsrl_cloud_processing_ref.so"))


# ---------------------------------------------------------------------------------------------- seeded scenes
# name -> (lidar_type, n_scans, scan_rate, time_unit, blind, point_filter_num, messages); a message is regenerated from its
# arguments by scene_messages.  Five or more messages each, so last_end_time carries from one to the next.
def _cloud_msgs(lt, given, rows, cols, rate, k=5, seed0=0):
    return [("cloud", dict(lidar_type=lt, seed=seed0 + m, rows=rows, cols=cols, given=given, scan_rate=rate), 1.7e9 + m / rate)
            for m in range(k)]


def _livox_msgs(k=5, n=3000, seed0=0, big=True):
    return [("livox", dict(seed=seed0 + m, n=n, big=big), 1.7e9 + 0.1 * m) for m in range(k)]


SCENES = {
    "livox_r3live": (LIVOX, 6, 10, NS, 0.1, 4, _livox_msgs()),
    "livox_f1_blind4": (LIVOX, 6, 10, NS, 4.0, 1, _livox_msgs(seed0=10)),
    "velo_given": (VELO, 16, 10, NS, 4.0, 4, _cloud_msgs(VELO, True, 16, 200, 10)),
    "ouster_given_ntu": (OUST, 16, 20, NS, 4.0, 4, _cloud_msgs(OUST, True, 16, 256, 20, seed0=20)),
    "ouster_given_f1": (OUST, 16, 20, NS, 0.1, 1, _cloud_msgs(OUST, True, 16, 128, 20, seed0=30)),
    "robo_given": (ROBO, 16, 10, SEC, 4.0, 4, _cloud_msgs(ROBO, True, 16, 200, 10, seed0=40)),
    "velo_yaw": (VELO, 16, 10, NS, 4.0, 4, _cloud_msgs(VELO, False, 16, 200, 10, seed0=50)),
    "ouster_yaw_ntu": (OUST, 16, 20, NS, 4.0, 4, _cloud_msgs(OUST, False, 16, 256, 20, seed0=60)),
    "robo_yaw_f1": (ROBO, 16, 10, SEC, 0.1, 1, _cloud_msgs(ROBO, False, 16, 128, 10, seed0=70)),
}


def scene_messages(name):
    """[(kind, payload, stamp)]: kind "livox" with a livox_dtype() array, "cloud" with a cloud_dtype() array"""
    out = []
    for kind, kw, stamp in SCENES[name][6]:
        if kind == "livox":
            out.append((kind, livox_records(kw["seed"], kw["n"], big=kw["big"]), stamp))
        else:
            kw = dict(kw)
            lt = kw.pop("lidar_type")
            out.append((kind, cloud2(lt, **kw), stamp))
    return out


def cloud_layout(lidar_type):
    step, off, _, _ = CLOUD_LAYOUTS[lidar_type]
    return dict(point_step=step, x=off[0], y=off[1], z=off[2], time=off[3], ring=off[4])
