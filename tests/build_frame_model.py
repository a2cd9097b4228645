"""Models of lioOptimization::buildFrame (src/lioOptimization.cpp:786-893) for the tests.

- mt19937_64 and std::shuffle as libstdc++ draws (rule 0: Lemire's multiply-shift, libstdc++ with __int128; rule 1: the
  division downscale of libstdc++ without __int128 and libstdc++ <= 10), sequentially;
- the parallel resolution the device uses: every final position's source from the sorted steps (j_k, k);
- the oracle's buildFrame: makePointTimestamp in numpy, then the oracle's row N2 / N3 pieces in the reference's order;
- sweeps and IMU tracks for the cases.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

import sweep_prep_cases as SC
from oracle import oracle_py as O

REF_LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libsrl_build_frame_ref.so")
MASK = (1 << 64) - 1
_UM, _LM, _A = np.uint64(0xFFFFFFFF80000000), np.uint64(0x7FFFFFFF), np.uint64(0xB5026F5AA96619E9)


def mt19937_64(count: int) -> np.ndarray:
    """The first `count` outputs of a default-seeded std::mt19937_64."""
    mt = [5489]
    for i in range(1, 312):
        mt.append((6364136223846793005 * (mt[-1] ^ (mt[-1] >> 62)) + i) & MASK)
    mt = np.array(mt, np.uint64)
    out = []
    one = np.uint64(1)
    for _ in range((count + 311) // 312):
        x = (mt[:156] & _UM) | (mt[1:157] & _LM)
        mt[:156] = mt[156:312] ^ (x >> one) ^ np.where(x & one, _A, np.uint64(0))
        nxt = np.r_[mt[157:312], mt[:1]]
        x = (mt[156:312] & _UM) | (nxt & _LM)
        mt[156:312] = mt[0:156] ^ (x >> one) ^ np.where(x & one, _A, np.uint64(0))
        y = mt.copy()
        y ^= (y >> np.uint64(29)) & np.uint64(0x5555555555555555)
        y ^= (y << np.uint64(17)) & np.uint64(0x71D67FFFEDA60000)
        y ^= (y << np.uint64(37)) & np.uint64(0xFFF7EEE000000000)
        y ^= y >> np.uint64(43)
        out.append(y)
    return np.concatenate(out)[:count] if out else np.zeros(0, np.uint64)


def num_draws(n: int) -> int:
    return 0 if n <= 1 else (1 if n % 2 == 0 else 0) + (n - 1) // 2


def draw(words, pos: int, r: int, rule: int):
    """uniform_int_distribution<uint64>{0, r - 1} from words[pos...]: (value, next position)."""
    while True:
        w = int(words[pos]); pos += 1
        if rule == 0:
            p = w * r
            lo = p & MASK
            if lo < r and lo < ((1 << 64) - r) % r:
                continue
            return p >> 64, pos
        scaling = MASK // r
        if w >= r * scaling:
            continue
        return w // scaling, pos


def shuffle_targets(n: int, words, pos: int = 0, rule: int = 0):
    """std::shuffle's swap targets: j[k] for step k ("swap(a[k], a[j[k]])", k = 1..n-1), and the next word position."""
    j = np.zeros(max(n, 1), np.int64)
    if n <= 1:
        return j[:n], pos
    i = 1
    if n % 2 == 0:
        j[1], pos = draw(words, pos, 2, rule)
        i = 2
    while i < n:
        x, pos = draw(words, pos, (i + 1) * (i + 2), rule)
        j[i], j[i + 1] = x // (i + 2), x % (i + 2)
        i += 2
    return j, pos


def fisher_yates(j) -> np.ndarray:
    """The permutation the steps make, run sequentially: perm[p] = element that ends at position p."""
    a = np.arange(len(j))
    for k in range(1, len(j)):
        a[k], a[j[k]] = a[j[k]], a[k]
    return a


def resolve(j) -> np.ndarray:
    """The same permutation without running the steps: the last step k > p with j_k = p puts element k at p; without one,
    p holds what position j_p held just before step p, resolved the same way one level down."""
    n = len(j)
    if n == 0:
        return np.zeros(0, np.int64)
    k = np.arange(1, n, dtype=np.uint64)
    keys = np.sort((np.asarray(j[1:], np.uint64) << np.uint64(32)) | k)
    q = np.arange(n, dtype=np.uint64)
    t = np.full(n, n, np.uint64)
    src = np.full(n, -1, np.int64)
    todo = np.arange(n)
    while todo.size:
        qq, tt = q[todo], t[todo]
        at = np.searchsorted(keys, (qq << np.uint64(32)) | tt, "left") - 1
        kk = keys[np.maximum(at, 0)] if keys.size else np.zeros_like(qq)
        hit = (at >= 0) & ((kk >> np.uint64(32)) == qq) & ((kk & np.uint64(0xFFFFFFFF)) > qq)
        src[todo[hit]] = (kk[hit] & np.uint64(0xFFFFFFFF)).astype(np.int64)
        jq = np.asarray(j, np.int64)[qq.astype(np.int64)]
        stop = ~hit & ((qq == 0) | (jq == qq.astype(np.int64)))
        src[todo[stop]] = qq[stop].astype(np.int64)
        go = ~hit & ~stop
        t[todo[go]] = qq[go]
        q[todo[go]] = jq[go].astype(np.uint64)
        todo = todo[go]
    return src


def shuffle(n: int, words, pos: int = 0, rule: int = 0):
    j, pos = shuffle_targets(n, words, pos, rule)
    return fisher_yates(j), pos


def _mul128(w, r):
    """(high, low) 64-bit halves of w * r, uint64 arrays, from 32-bit limbs."""
    m32, s = np.uint64(0xFFFFFFFF), np.uint64(32)
    a1, a0, b1, b0 = w >> s, w & m32, r >> s, r & m32
    p00, p01, p10, p11 = a0 * b0, a0 * b1, a1 * b0, a1 * b1
    mid = (p00 >> s) + (p01 & m32) + (p10 & m32)
    return p11 + (p01 >> s) + (p10 >> s) + (mid >> s), (p00 & m32) | (mid << s)


def _draw_try(w, r, rule: int):
    """draw()'s one attempt on uint64 arrays: (accepted, value)."""
    if rule == 0:
        hi, lo = _mul128(w, r)
        return ~((lo < r) & (lo < (np.uint64(0) - r) % r)), hi
    scaling = np.uint64(MASK) // r
    return w < r * scaling, w // scaling


def shuffle_targets_fast(n: int, words, pos: int = 0, rule: int = 0):
    """shuffle_targets on arrays: every draw at once on the words it would take without a rejection, then from each
    rejected draw on again one word later.  (j, next word position, indices of the rejected draws; a draw rejected twice
    is listed twice)."""
    D = num_draws(n)
    j = np.zeros(max(n, 1), np.int64)
    if D == 0:
        return j[:n], pos, []
    d = np.arange(D, dtype=np.int64)
    i = 2 * d + (1 if n % 2 else 0)
    r = ((i + 1) * (i + 2)).astype(np.uint64)
    if n % 2 == 0:
        i[0], r[0] = 1, 2
    x = np.zeros(D, np.uint64)
    words = np.asarray(words, np.uint64)
    rejected, start = [], 0
    while start < D:
        w0 = pos + start + len(rejected)
        ok, val = _draw_try(words[w0:w0 + D - start], r[start:], rule)
        bad = np.flatnonzero(~ok)
        stop = D if bad.size == 0 else start + int(bad[0])
        x[start:stop] = val[:stop - start]
        if stop < D:
            rejected.append(stop)
        start = stop
    b = (i + 2).astype(np.uint64)
    pair = r != 2
    j[i[pair]] = (x[pair] // b[pair]).astype(np.int64)
    j[i[pair] + 1] = (x[pair] % b[pair]).astype(np.int64)
    if not pair[0]:
        j[1] = int(x[0])
    return j, pos + D + len(rejected), rejected


def shuffle_fast(n: int, words, pos: int = 0, rule: int = 0):
    """shuffle() for frames of millions of points: (perm, next word position, rejected draws)."""
    j, pos, rejected = shuffle_targets_fast(n, words, pos, rule)
    return resolve(j), pos, rejected


# ---- the oracle's buildFrame -------------------------------------------------------------------------------------------
def make_point_timestamp(ts, begin, end, point_time_enable):
    """makePointTimestamp (:786-819): (kept indices, relative_time ms, alpha_time)."""
    ts = np.asarray(ts, float)
    keep = np.arange(ts.shape[0]) if point_time_enable else np.flatnonzero(~(ts > end) & ~(ts < begin))
    delta_t = end - begin
    rel = ts[keep] - begin
    with np.errstate(divide="ignore", invalid="ignore"):   # delta_t 0: +-inf or NaN, as the reference divides
        alpha = rel / delta_t
    rel = rel * 1000.0
    if point_time_enable:
        alpha = np.where(alpha > 1.0, 1.0 - 1e-5, alpha)
    return keep, rel, alpha


def transform_point(raw, q, t, R_il, t_il):
    """transformPoint (src/utility.cpp:314-318): each 3-term sum as a0 b0 + (a1 b1 + a2 b2), as the reference evaluates it."""
    def mv(M, v):
        return np.stack([M[r, 0] * v[:, 0] + (M[r, 1] * v[:, 1] + M[r, 2] * v[:, 2]) for r in range(3)], axis=1)
    b = mv(np.asarray(R_il, float).reshape(3, 3), raw)
    b = b + np.asarray(t_il, float)[None, :]
    return mv(O.quat_to_rot(q), b) + np.asarray(t, float)[None, :]


def build_frame(c: dict, rule: int = 0) -> dict:
    """buildFrame over case c, composed of numpy and the oracle's row N2 / N3 pieces."""
    raw, ts = np.asarray(c["raw"], float).reshape(-1, 3), np.asarray(c["ts"], float)
    begin, end = c["begin"], c["begin"] + c["offset"]
    keep, rel, alpha = make_point_timestamp(ts, begin, end, c["point_time_enable"])
    raw1, ts1 = raw[keep], ts[keep]
    n1 = keep.shape[0]
    R_il, t_il = c["R_il"], c["t_il"]
    if c["motion_compensation"] == 1:
        imu = O.distort_frame_by_constant(raw1, rel, c["states"], begin, R_il, t_il) if n1 else np.zeros((0, 3))
    else:
        imu = O.distort_frame_by_imu(raw1, rel, c["states"], begin, R_il, t_il, imu_xyz_in=np.zeros((n1, 3)))[0] if n1 else np.zeros((0, 3))
    words = mt19937_64(2 * num_draws(n1) + 4096)
    order, pos, rej1 = shuffle_fast(n1, words, 0, rule)
    rej2 = []
    if c["voxel_size"] > 0:
        size = c["init_voxel_size"] if c["index_frame"] < c["init_num_frames"] else c["voxel_size"]
        sel = O.grid_sampling(raw1[order], size) if n1 else np.zeros(0, np.int64)
        order = order[sel]
        perm, pos, rej2 = shuffle_fast(order.shape[0], words, pos, rule)
        order = order[perm]
    imu_f = imu[order]
    raw_f = O.transform_all_imu_point(imu_f, c["states"][-1], R_il, t_il) if order.size else np.zeros((0, 3))
    if c["index_frame"] <= 2:
        point = transform_point(raw_f, [0.0, 0.0, 0.0, 1.0], np.zeros(3), R_il, t_il)
        alpha_f = np.ones(order.shape[0])
    else:
        point = transform_point(raw_f, c["q_pred"], c["t_pred"], R_il, t_il)
        alpha_f = alpha[order]
    return dict(raw_point=raw_f, point=point, imu_point=imu_f, relative_time=rel[order], alpha_time=alpha_f, timestamp=ts1[order],
                source_index=keep[order].astype(np.int32), engine_words=pos, n_timestamped=n1,
                rejected=(rej1, rej2))


# ---- cases --------------------------------------------------------------------------------------------------------------
def make_case(name, n=2000, seed=0, begin=1.7e9 + 0.25, offset=0.1, point_time_enable=True, motion_compensation=1, index_frame=5,
              init_num_frames=20, init_voxel_size=0.2, voxel_size=0.5, n_states=11, imu_span=None, edges=True, scale=40.0, early=0.05):
    """A cut sweep at Unix-epoch stamps: points in time order, a few exactly at begin / end and outside them, an IMU track
    over [begin, begin + imu_span] (imu_span < offset: the IMU walk stops early)."""
    rng = np.random.default_rng(seed)
    raw = SC.raw_points(rng, n, scale) if n else np.zeros((0, 3))
    ts = np.sort(begin + rng.uniform(-early * offset, 1.05 * offset, n)) if n else np.zeros(0)
    if edges and n >= 8:
        ts[:4] = [begin, begin, np.nextafter(begin, -np.inf), begin - 0.01]
        ts[-4:] = [begin + offset, np.nextafter(begin + offset, np.inf), begin + offset + 0.01, begin + offset]
        ts = np.sort(ts)
    span = offset if imu_span is None else imu_span
    stamps = [begin + span * k / (n_states - 1) for k in range(n_states)] if n_states > 1 else [begin]
    states = SC.track(rng, stamps, trans0=rng.uniform(-50, 50, 3))
    R_il, t_il = SC.extrinsic(rng)
    q_pred = SC._unit(rng.normal(size=4))
    return dict(name=name, raw=raw, ts=ts, begin=float(begin), offset=float(offset), point_time_enable=point_time_enable,
                motion_compensation=motion_compensation, index_frame=index_frame, init_num_frames=init_num_frames,
                init_voxel_size=init_voxel_size, voxel_size=voxel_size, states=states, R_il=R_il, t_il=t_il, q_pred=q_pred,
                t_pred=rng.uniform(-30, 30, 3), prev_time_sweep_end=float(begin - 0.003))


def cases() -> list[dict]:
    return [
        make_case("time_const_f5"),
        make_case("no_time_const_f5", point_time_enable=False, seed=1),
        make_case("time_imu_f5", motion_compensation=0, seed=2, edges=False, early=0.0, offset=0.105),
        make_case("no_time_imu_f3", point_time_enable=False, motion_compensation=0, index_frame=3, seed=3),
        make_case("imu_walk_stops_early", motion_compensation=0, imu_span=0.06, seed=4, point_time_enable=False),
        make_case("no_subsample", voxel_size=0.0, seed=5),
        make_case("no_subsample_negative", voxel_size=-1.0, index_frame=1, seed=6),
        make_case("frame1", index_frame=1, seed=7),
        make_case("frame2", index_frame=2, seed=8, point_time_enable=False),
        make_case("frame3_init_size", index_frame=3, seed=9),
        make_case("frame25_steady_size", index_frame=25, seed=10, n=5000),
        make_case("alpha_clamp", offset=0.05, seed=11),   # stamps run 5 % past the end: alpha > 1 clamped
        make_case("empty", n=0, seed=12),
        make_case("one_point", n=1, seed=13),
        make_case("two_points", n=2, seed=14, voxel_size=0.0),
        make_case("odd_small", n=7, seed=15, edges=False),
    ]


def imu_state_rows(states) -> np.ndarray:
    return O.imu_states_array(states)


def capi_imu_states(states) -> list:
    """The states as srl_imu_state structs for the library."""
    from sr_livo_b200 import capi
    out = []
    for s in states:
        st = capi.ImuState()
        st.timestamp = s["timestamp"]
        for name in ("quat", "trans", "vel", "un_acc", "un_gyr"):
            getattr(st, name)[:] = [float(v) for v in s[name]]
        out.append(st)
    return out


# ---- the reference's own buildFrame (oracle/srl_build_frame_harness.cpp, built by oracle/build_frame.mk) -----------------
_ref_lib = None


def reference_available() -> bool:
    return os.path.exists(REF_LIB)


class ReferenceBuildFrame:
    """One lioOptimization object of the reference whose buildFrame is called."""

    def __init__(self):
        global _ref_lib
        if _ref_lib is None:
            L = C.CDLL(REF_LIB)
            P, I64 = C.c_void_p, C.c_int64
            L.ref_bf_create.restype = P
            L.ref_bf_destroy.argtypes = [P]
            L.ref_build_frame.argtypes = [P, P, P, I64, P, I64] + [P] * 14
            L.ref_build_frame.restype = I64
            _ref_lib = L
        self._L = _ref_lib
        self._h = C.c_void_p(self._L.ref_bf_create())

    def __del__(self):
        try:
            if self._h:
                self._L.ref_bf_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def build_frame(self, c: dict) -> dict:
        """buildFrame over case c: the frame's fields in frame order (source_index = index in the cut sweep) + scalars."""
        f64 = lambda a: np.ascontiguousarray(a, np.float64)   # noqa: E731
        raw, ts, st = f64(c["raw"]).reshape(-1, 3), f64(c["ts"]).reshape(-1), f64(imu_state_rows(c["states"])).reshape(-1, 17)
        R, ti, qp, tp = f64(c["R_il"]).reshape(9), f64(c["t_il"]), f64(c["q_pred"]), f64(c["t_pred"])
        prm = f64([c["begin"], c["offset"], c["init_voxel_size"], c["voxel_size"], c["prev_time_sweep_end"]])
        cfg = np.ascontiguousarray([int(bool(c["point_time_enable"])), c["motion_compensation"], c["index_frame"], c["init_num_frames"]],
                                   np.int32)
        n = raw.shape[0]
        names = ("raw_point", "point", "imu_point", "relative_time", "alpha_time", "timestamp", "source_index")
        out = dict(raw_point=np.zeros((n, 3)), point=np.zeros((n, 3)), imu_point=np.zeros((n, 3)), relative_time=np.zeros(n),
                   alpha_time=np.zeros(n), timestamp=np.zeros(n), source_index=np.zeros(n, np.int32))
        sc = np.zeros(7)
        m = self._L.ref_build_frame(self._h, raw.ctypes.data, ts.ctypes.data, n, st.ctypes.data, st.shape[0], R.ctypes.data,
                                    ti.ctypes.data, qp.ctypes.data, tp.ctypes.data, prm.ctypes.data, cfg.ctypes.data,
                                    *[out[k].ctypes.data for k in names], sc.ctypes.data)
        out = {k: v[:m].copy() for k, v in out.items()}
        out["scalars"] = dict(zip(("time_sweep_begin", "time_sweep_end", "time_frame_begin", "time_frame_end", "offset_begin",
                                   "offset_end", "dt_offset"), sc.tolist()))
        return out
