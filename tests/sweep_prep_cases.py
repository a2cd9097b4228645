"""Seeded inputs for the sweep-preparation tests (tests/test_sweep_prep_truth.py on the CPU, tests/test_sweep_prep_device.py
on the GPU): the branch points of slerp and so3ToQuat, the interval walk at Unix-epoch timestamps, large magnitudes, and
the cell keys of gridSampling near their truncation points.

Every case is a dict with `kind` ("const", "imu", "end" or "grid"), its inputs, and `pins`: the decisions it exists to
place at (or within rounding of) their thresholds.  "time" = time_point, nudges and interval membership; "slerp" = absD >=
one; "so3" = theta < 1e-4; "clamp" = the alpha clamps; "grid" = the cell keys.  All other decisions of a case must lie
clear of their thresholds.
"""
from __future__ import annotations

import math

import numpy as np

T_EPOCH = 1.7e9        # Unix seconds: one ulp is 2.4e-7 s
HZ_DT = 0.005          # 200 Hz IMU
EPS = 2.0 ** -52


def _unit(q):
    q = np.asarray(q, float)
    return q / np.linalg.norm(q)


def qmul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                     aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz])


def qaxis(axis, angle):
    axis = np.asarray(axis, float) / np.linalg.norm(axis)
    return np.r_[axis * math.sin(angle / 2), math.cos(angle / 2)]


def extrinsic(rng):
    R = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    if np.linalg.det(R) < 0:
        R[:, 0] = -R[:, 0]
    return R, rng.normal(0, 0.3, 3)


def raw_points(rng, n, scale=200.0):
    """Raw LiDAR points out to `scale` metres, with some close ones."""
    r = rng.uniform(0.5, scale, n) * rng.choice([1.0, 0.01], n, p=[0.9, 0.1])
    d = rng.normal(size=(n, 3))
    return d / np.linalg.norm(d, axis=1)[:, None] * r[:, None]


def state(ts, q, trans, vel, acc, gyr):
    return dict(timestamp=float(ts), quat=np.asarray(q, float), trans=np.asarray(trans, float), vel=np.asarray(vel, float),
                un_acc=np.asarray(acc, float), un_gyr=np.asarray(gyr, float))


def track(rng, stamps, q0=None, trans0=None, gyr_scale=0.4, acc_scale=1.5, gyr=None):
    """A physically consistent track over the given stamps (quaternion and position integrated in FP64)."""
    q = _unit(rng.normal(size=4)) if q0 is None else np.asarray(q0, float)
    p = rng.uniform(-1e4, 1e4, 3) if trans0 is None else np.asarray(trans0, float)
    v = rng.normal(0, 3, 3)
    out = []
    for k, ts in enumerate(stamps):
        g = rng.normal(0, gyr_scale, 3) if gyr is None else np.asarray(gyr[k], float)
        a = rng.normal(0, acc_scale, 3)
        out.append(state(ts, q, p, v, a, g))
        dt = (stamps[k + 1] - ts) if k + 1 < len(stamps) else 0.0
        th = np.linalg.norm(g * dt)
        if th > 0:
            q = _unit(qmul(q, qaxis(g, th)))
        p = p + v * dt + 0.5 * a * dt * dt
        v = v + a * dt
    return out


def rel_for(t0: float, target: float) -> float:
    """A relative time (ms) for which t0 + rel / 1000 rounds to exactly `target`."""
    rel = (target - t0) * 1000.0
    for _ in range(64):
        tp = t0 + rel / 1000.0
        if tp == target:
            return rel
        rel = float(np.nextafter(rel, np.inf if tp < target else -np.inf))
    raise RuntimeError("no relative time hits the target")


# ---- distortFrameByConstant: slerp branch points -----------------------------------------------------------------
def _const_case(name, rng, qa, qb, t0=100.0, span=0.1, n=192, pins=(), n_states=5, trans_scale=1e4):
    stamps = [t0 + span * k / (n_states - 1) for k in range(n_states)] if n_states > 1 else [t0]
    st = track(rng, stamps)
    st[0]["quat"] = np.asarray(qa, float)
    st[-1]["quat"] = np.asarray(qb, float)
    st[-1]["trans"] = st[0]["trans"] + rng.normal(0, 1, 3) if trans_scale else st[-1]["trans"]
    rel = np.sort(rng.uniform(0.0, span * 1000.0, n))
    # the ends (both nudges), just outside them (clamps) and far outside (clamps)
    rel[:6] = [0.0, 1e-4, span * 1000.0, span * 1000.0 - 1e-4, -25.0, span * 1000.0 + 25.0]
    R, t = extrinsic(rng)
    return dict(name=name, kind="const", raw=raw_points(rng, n), rel=rel, states=st, t0=float(t0), R_il=R, t_il=t,
                pins=set(pins) | {"clamp"})


def const_cases():
    rng = np.random.default_rng(9101)
    out = []
    q = _unit(rng.normal(size=4))
    out.append(_const_case("still", rng, q, q.copy(), pins={"slerp"}))
    e_w = np.array([0.0, 0.0, 0.0, 1.0])
    # d exactly at one, one ulp above, one ulp below (qa = e_w: d = qb.w with no rounding at all)
    for tag, w in (("at_one", 1.0 - EPS), ("ulp_above", 1.0 - EPS / 2), ("ulp_below", 1.0 - 1.5 * EPS)):
        qb = np.array([math.sqrt(max(0.0, 1.0 - w * w)), 0.0, 0.0, w])
        out.append(_const_case(f"d_{tag}", rng, e_w, qb, pins={"slerp"}))
        out.append(_const_case(f"d_{tag}_neg", rng, e_w, -qb, pins={"slerp"}))
    # d in (1 - 1e-12, 1 - eps): slerp with theta between 2e-8 and 1.4e-6
    for k, delta in enumerate((3e-16, 1e-14, 1e-13, 5e-13, 9e-13)):
        qa = _unit(rng.normal(size=4))
        qb = qmul(qa, qaxis(rng.normal(size=3), 2 * math.sqrt(2 * delta)))
        out.append(_const_case(f"d_near_{k}", rng, qa, qb, pins={"slerp"} if k == 0 else ()))
    qa = _unit(rng.normal(size=4))
    out.append(_const_case("antipodal", rng, qa, -qa, pins={"slerp"}))
    out.append(_const_case("neg_dot", rng, qa, -qmul(qa, qaxis(rng.normal(size=3), 0.3))))
    for deg in (90.0, 170.0):
        qa = _unit(rng.normal(size=4))
        out.append(_const_case(f"rot{int(deg)}", rng, qa, qmul(qa, qaxis(rng.normal(size=3), math.radians(deg)))))
    for s in (0.9, 1.1):
        qa = _unit(rng.normal(size=4))
        out.append(_const_case(f"norm{s}", rng, s * qa, s * qmul(qa, qaxis(rng.normal(size=3), 0.2))))
    # a single IMU state: begin == end, the second nudge undoes the first and alpha = -1e-6 / 0 clamps to 0
    q = _unit(rng.normal(size=4))
    c = _const_case("one_state", rng, q, q, n_states=1, pins={"slerp"})
    out.append(c)
    c2 = _const_case("one_state_later", rng, q, qmul(q, qaxis([1, 2, 3], 0.1)), n_states=1, pins={"slerp"})
    c2["t0"] = c2["states"][0]["timestamp"] - 0.05
    out.append(c2)
    # Unix-epoch stamps
    qa = _unit(rng.normal(size=4))
    out.append(_const_case("epoch", rng, qa, qmul(qa, qaxis(rng.normal(size=3), 0.04)), t0=T_EPOCH, pins={"time"}))
    return out


# ---- distortFrameByImu: so3ToQuat branch points ----------------------------------------------------------------
def so3_cases():
    rng = np.random.default_rng(9202)
    out = []
    # one point per interval, in the middle; the interval's gyro puts |gyr dt| at 1e-4 (1 +- 2^-k)
    t0 = 100.0
    targets = [1e-4 * (1 + s * 2.0 ** -k) for k in (1, 4, 10, 20, 30, 40, 45) for s in (-1, 1)] + [1e-4 * 0.5, 1e-4 * 3, 5e-4]
    n_int = len(targets)
    stamps = [t0 + k * HZ_DT for k in range(n_int + 1)]
    rel = np.array([(stamps[k] + 0.0025 - t0) * 1000.0 for k in range(n_int)])
    tp = t0 + rel / 1000.0
    gyr = [np.zeros(3)]
    for k in range(n_int):
        d = _unit(rng.normal(size=3))
        gyr.append(d * targets[k] / (tp[k] - stamps[k]))
    st = track(rng, stamps, gyr=gyr)
    R, t = extrinsic(rng)
    out.append(dict(name="so3_threshold", kind="imu", raw=raw_points(rng, n_int), rel=rel, states=st, t0=t0, R_il=R, t_il=t,
                    pins={"so3"}))
    # zero gyro: every point on the small-angle branch (theta = 0)
    stamps = [t0 + k * HZ_DT for k in range(21)]
    st = track(rng, stamps, gyr=[np.zeros(3)] * 21)
    n = 600
    rel = np.sort(rng.uniform(0, 100.0, n))
    out.append(dict(name="zero_gyro", kind="imu", raw=raw_points(rng, n), rel=rel, states=st, t0=t0, R_il=R, t_il=t, pins=set()))
    # slow rotation: |gyr| < 0.02 rad/s keeps every point on the small-angle branch, time from 0 s
    st = track(rng, [k * HZ_DT for k in range(21)], gyr_scale=0.005)
    rel = np.sort(rng.uniform(0, 100.0, n))
    out.append(dict(name="slow_from_zero", kind="imu", raw=raw_points(rng, n), rel=rel, states=st, t0=0.0, R_il=R, t_il=t,
                    pins=set()))
    # 10 rad/s
    st = track(rng, stamps, gyr=[_unit(rng.normal(size=3)) * 10.0 for _ in range(21)])
    rel = np.sort(rng.uniform(0, 100.0, n))
    out.append(dict(name="gyro_10rad", kind="imu", raw=raw_points(rng, n), rel=rel, states=st, t0=t0, R_il=R, t_il=t, pins=set()))
    return out


# ---- distortFrameByImu: the walk at Unix-epoch stamps ------------------------------------------------------------
def _epoch_track(rng, n_states, repeat=()):
    stamps = [T_EPOCH + k * HZ_DT for k in range(n_states)]
    for k in repeat:
        stamps[k + 1] = stamps[k]
    return track(rng, stamps), stamps


def walk_cases():
    rng = np.random.default_rng(9303)
    R, t = extrinsic(rng)
    out = []
    st, stamps = _epoch_track(rng, 21)
    t0 = stamps[0]
    # points at every interior stamp +- k ulp, k = 0..6 (the nudge window is about 4.2 ulp wide)
    tps = []
    for s in stamps[1:-1]:
        u = np.spacing(s)
        tps += [s + j * u for j in range(-6, 7)]
    rel = np.array([rel_for(t0, x) for x in sorted(tps)])
    out.append(dict(name="stamp_ulps", kind="imu", raw=raw_points(rng, rel.size), rel=rel, states=st, t0=t0, R_il=R, t_il=t,
                    pins={"time"}))
    # repeated stamps: zero-length intervals
    st2, stamps2 = _epoch_track(rng, 21, repeat=(3, 4, 10))
    tps = sorted([s + j * np.spacing(s) for s in (stamps2[3], stamps2[10]) for j in range(-6, 7)] +
                 list(rng.uniform(stamps2[0], stamps2[-1], 200)))
    rel = np.array([rel_for(t0, x) for x in tps])
    out.append(dict(name="repeated_stamps", kind="imu", raw=raw_points(rng, rel.size), rel=rel, states=st2, t0=t0, R_il=R,
                    t_il=t, pins={"time"}))
    # points before the first stamp: the walk writes nothing
    rel = np.sort(rng.uniform(-50.0, -0.01, 40))
    out.append(dict(name="before_first", kind="imu", raw=raw_points(rng, 40), rel=rel, states=st, t0=t0, R_il=R, t_il=t,
                    pins={"time"}))
    # a NaN time stops the walk there
    rel = np.sort(rng.uniform(0, 100.0, 300))
    rel[137] = np.nan
    out.append(dict(name="nan_time", kind="imu", raw=raw_points(rng, 300), rel=rel, states=st, t0=t0, R_il=R, t_il=t,
                    pins={"time"}))
    # sizes around the 256-thread blocks, and a large sweep
    for n in (1, 255, 256, 257, 100000):
        rel = np.sort(rng.uniform(0, 100.0, n))
        out.append(dict(name=f"n{n}", kind="imu", raw=raw_points(rng, n), rel=rel, states=st, t0=t0, R_il=R, t_il=t,
                        pins={"time"}))
    # 4096 states (the shared-memory limit of the interval kernel) and 4097 (rejected by the device)
    for ns in (4096, 4097):
        stl, sl = _epoch_track(rng, ns)
        rel = np.sort(rng.uniform(0, (sl[-1] - sl[0]) * 1000.0, 3000))
        out.append(dict(name=f"states{ns}", kind="imu", raw=raw_points(rng, 3000), rel=rel, states=stl, t0=sl[0], R_il=R,
                        t_il=t, pins={"time"}))
    # time_point at epoch stamps where the rounding of rel / 1000 decides the rounding of begin + rel / 1000: the two
    # candidates rel / 1000 and rel * 1e-3 give time points one ulp (2.4e-7 s) apart
    stq = track(rng, stamps, gyr_scale=0.005)
    u = float(np.spacing(t0))
    rel = []
    for j in rng.choice(int(0.1 / u), 6000, replace=False):
        r0 = (j + 0.5) * u * 1000.0
        for d in range(-8, 9):
            r = r0 + d * float(np.spacing(r0))
            if t0 + r / 1000.0 != t0 + r * 1e-3:
                rel.append(r)
                break
        if len(rel) == 64:
            break
    rel = np.sort(rel)
    out.append(dict(name="time_rounding", kind="imu", raw=raw_points(rng, rel.size), rel=rel, states=stq, t0=t0, R_il=R,
                    t_il=t, pins={"time"}))
    # time_point = begin + rel / 1000 with begin = 0: the quotient is the time point, so its rounding shows
    stz = track(rng, [k * HZ_DT for k in range(21)], gyr_scale=0.005)
    rel = np.sort(rng.uniform(0, 100.0, 4000))
    out.append(dict(name="begin_zero", kind="imu", raw=raw_points(rng, 4000), rel=rel, states=stz, t0=0.0, R_il=R, t_il=t,
                    pins=set()))
    return out


# ---- transformAllImuPoint ----------------------------------------------------------------------------------------
def end_cases():
    rng = np.random.default_rng(9404)
    out = []
    R, t = extrinsic(rng)
    for tag, s in (("unit", 1.0), ("norm0.9", 0.9), ("norm1.1", 1.1), ("zero", 0.0)):
        q = s * _unit(rng.normal(size=4))
        trans = rng.uniform(-1e4, 1e4, 3)
        last = state(T_EPOCH, q, trans, np.zeros(3), np.zeros(3), np.zeros(3))
        # points near the end pose (the result cancels) and far from it
        imu = np.vstack([trans + rng.normal(0, 1e-3, (200, 3)), trans + raw_points(rng, 200), raw_points(rng, 100, 1e4)])
        out.append(dict(name=f"end_{tag}", kind="end", imu=imu, last=last, R_il=R, t_il=t, pins=set()))
    return out


# ---- gridSampling cell keys ---------------------------------------------------------------------------------------
def grid_cases():
    rng = np.random.default_rng(9505)
    out = []
    size = 0.1
    inv = 1.0 / size
    # coordinates whose correctly rounded x / size and x * (1 / size) truncate to different integers
    pts = []
    for k in range(1, 40000):
        for x0 in (k * size, -k * size):
            for x in (np.nextafter(x0, -np.inf), x0, np.nextafter(x0, np.inf)):
                x = float(x)
                if math.trunc(x / size) != math.trunc(x * inv):
                    pts.append(x)
        if len(pts) >= 96:
            break
    # each such point follows a partner in the middle of its cell (y and z cells of its own): the point must join the
    # partner's cell, so a key off by one keeps it as a new keypoint
    rows = []
    for j, x in enumerate(pts):
        kx = math.trunc(x / size)
        y = (3 * j + 0.5) * size
        rows += [[(kx + math.copysign(0.5, x)) * size, y, 0.05], [x, y, 0.05]]
    xyz = np.array(rows)
    out.append(dict(name="grid_quotient_ulp", kind="grid", xyz=xyz, size=size, pins={"grid"}))
    # -0.0, +0.0 and both halves of the two-cell-wide cell 0
    z = np.array([[-0.0, 0.0, 0.0], [0.0, -0.0, -0.0], [-0.07, 0.03, 0.0], [0.07, -0.03, -0.0], [-0.0999, 0.0999, 0.05],
                  [-0.1, 0.0, 0.0], [0.1, 0.0, 0.0], [-0.1000001, 0.0, 0.0]])
    out.append(dict(name="grid_cell0", kind="grid", xyz=z, size=size, pins={"grid"}))
    # |x / size| at 32764 and 32765 (the last key the device keeps is 32764)
    s1 = 1.0
    edge = np.array([[32764.5, 0, 0], [-32764.5, 0, 0], [0, 32764.999, 0], [0, 0, 32765.0], [32765.5, 0, 0],
                     [0, -32765.2, 0], [1.5, 2.5, 3.5]])
    out.append(dict(name="grid_key_range", kind="grid", xyz=edge, size=s1, pins={"grid"}))
    # NaN and +-inf: no cell
    nf = np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [1.2, 0.3, 0.4], [np.nan, np.nan, np.nan], [1.25, 0.3, 0.4]])
    out.append(dict(name="grid_nonfinite", kind="grid", xyz=nf, size=s1, pins={"grid"}))
    return out


def all_cases():
    return const_cases() + so3_cases() + walk_cases() + end_cases() + grid_cases()


# ---- running a case ----------------------------------------------------------------------------------------------
def sample(n: int, cap: int = 256, seed: int = 0) -> np.ndarray:
    """The points whose truth is evaluated: all of them up to `cap`, else the first and last 16 and a seeded draw."""
    if n <= cap:
        return np.arange(n)
    rng = np.random.default_rng(seed)
    return np.unique(np.r_[np.arange(16), np.arange(n - 16, n), rng.choice(n, cap - 32, replace=False)])


def run(impl, case, imu_in=None):
    """Run one case through an implementation with the oracle_py calling convention (oracle_py or reference_py).
    Returns (output, n_written or None)."""
    k = case["kind"]
    if k == "const":
        return impl.distort_frame_by_constant(case["raw"], case["rel"], case["states"], case["t0"], case["R_il"], case["t_il"]), None
    if k == "imu":
        keep = np.full_like(case["raw"], -7.0) if imu_in is None else imu_in
        r = impl.distort_frame_by_imu(case["raw"], case["rel"], case["states"], case["t0"], case["R_il"], case["t_il"],
                                      imu_xyz_in=keep)
        return (r if isinstance(r, tuple) else (r, None))
    if k == "end":
        return impl.transform_all_imu_point(case["imu"], case["last"], case["R_il"], case["t_il"]), None
    return impl.grid_sampling(case["xyz"], case["size"]), None


def truth(case):
    """The 50-digit truth of a case on its sampled points: dict(idx, val, err, info, n_written, k_of)."""
    import sweep_prep_reference as R
    k = case["kind"]
    out = dict(idx=np.zeros(0, np.int64), val=np.zeros((0, 3)), err=np.zeros((0, 3)), info=[], n_written=None, k_of=None)
    if k == "grid":
        return out
    if k == "imu":
        ts = [s["timestamp"] for s in case["states"]]
        nw, k_of = R.walk(case["t0"], case["rel"], ts)
        out["n_written"], out["k_of"] = nw, k_of
        idx = sample(nw)
        tps = R.time_points(case["t0"], case["rel"])
    else:
        idx = sample(case["raw"].shape[0] if k == "const" else case["imu"].shape[0])
    vals, errs, info = [], [], []
    for i in idx:
        if k == "const":
            p, inf = R.distort_constant_point(case["raw"][i], case["rel"][i], case["states"], case["t0"], case["R_il"], case["t_il"])
        elif k == "imu":
            kk = int(k_of[i])
            p, inf = R.distort_imu_point(case["raw"][i], float(tps[i]), case["states"][kk], case["states"][kk + 1], case["R_il"],
                                         case["t_il"])
            inf["k"] = kk
        else:
            p, inf = R.transform_all_imu_point(case["imu"][i], case["last"], case["R_il"], case["t_il"]), {}
        vals.append(R.vals(p))
        errs.append(R.errs(p))
        info.append(inf)
    out.update(idx=np.asarray(idx, np.int64), val=np.array(vals).reshape(-1, 3), err=np.array(errs).reshape(-1, 3), info=info)
    return out


def libm_free(case, tr):
    """Mask over tr['idx'] of the points whose path calls no libm function: every transformAllImuPoint point, points of
    distortFrameByImu on the small-angle branch, points of distortFrameByConstant on the lerp branch."""
    if case["kind"] == "end":
        return np.ones(tr["idx"].size, bool)
    if case["kind"] == "imu":
        return np.array([bool(i["small"]) for i in tr["info"]], bool)
    return np.array([bool(i["lerp"]) for i in tr["info"]], bool)
