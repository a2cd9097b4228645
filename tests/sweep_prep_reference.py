"""A 50-digit restatement of the sweep preparation (src/utility.cpp:167-332): the truth the oracle and the CUDA kernels of
srl_points.cu (row N3) and srl_grid_sampling (row N2) are measured against.

What is restated: distortFrameByConstant, distortFrameByImu ("distortion method 1"), transformAllImuPoint and the cell keys
of gridSampling, with the helpers they call: Eigen 3.3.7's QuaternionBase::slerp (its `one = 1 - eps` lerp branch and the
sign flip for d < 0), numType::so3ToQuat (the 1e-4 branch, then normalize), toRotationMatrix of the quaternion as given
(not normalised), Quaternion::inverse() (zero when n2 <= 0) and ((0.5 acc) dt) dt.

The reference's *decisions* are taken in FP64, exactly as it takes them: time_point = begin + rel / 1000, the two 1e-6
nudges, interval membership and the walk's stop, the alpha clamps, absD >= one, theta < 1e-4 and the cell keys.  Everything
after a decision is evaluated in mpmath at 50 digits on the FP64 inputs and returned with a first-order componentwise bound
of the error an FP64 evaluation in the reference's operation order may make (class `E`: every rounded operation adds
U |result|, every input error is carried through the operation's partial derivatives with absolute values).  The bounds
are built from the absolute values of the terms, so a coordinate that cancels (a point near the sweep's end pose in
transformAllImuPoint) keeps a bound of the size of its terms, not of its result.  libm calls (sin, cos, acos) add C_LIB U
|result|.  The slerp weights sin(w theta) / sin(theta) are bounded through their exact derivative in theta: theta's own
error grows like u / theta near the lerp threshold, the ratio does not.
"""
from __future__ import annotations

import math

import mpmath as mp
import numpy as np

mp.mp.dps = 50
U = 2.0 ** -53                       # unit roundoff of FP64
EPS = 2.0 ** -52                     # std::numeric_limits<double>::epsilon()
ONE = 1.0 - EPS                      # Eigen's `one` in slerp
K_THETA = 1e-4                       # THETA_THRESHOLD, include/utility.h:27
NUDGE = 1e-6                         # the 1e-6 s of src/utility.cpp:216-217,264,266-267
C_LIB = 4.0                          # sin / cos / acos: within 2 ulp (CUDA's documented bound; glibc is within 1)


# ---- values with a first-order error bound ---------------------------------------------------------------------------
class E:
    """An exact value (mpf) and a bound (float) of the error an FP64 evaluation of the same expression may carry."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=0.0):
        self.v = v if isinstance(v, mp.mpf) else mp.mpf(float(v))
        self.e = float(e)

    def __add__(a, b):
        b = _e(b)
        r = a.v + b.v
        return E(r, a.e + b.e + U * abs(float(r)))

    __radd__ = __add__

    def __sub__(a, b):
        b = _e(b)
        r = a.v - b.v
        return E(r, a.e + b.e + U * abs(float(r)))

    def __rsub__(a, b):
        return _e(b) - a

    def __neg__(a):
        return E(-a.v, a.e)

    def __mul__(a, b):
        b = _e(b)
        r = a.v * b.v
        return E(r, abs(float(b.v)) * a.e + abs(float(a.v)) * b.e + U * abs(float(r)))

    __rmul__ = __mul__

    def __truediv__(a, b):
        b = _e(b)
        r = a.v / b.v
        fb = abs(float(b.v))
        return E(r, a.e / fb + abs(float(r)) * b.e / fb + U * abs(float(r)))

    def __rtruediv__(a, b):
        return _e(b) / a


def _e(x):
    return x if isinstance(x, E) else E(x)


def esqrt(a: E) -> E:   # correctly rounded
    r = mp.sqrt(a.v)
    return E(r, (a.e / (2 * float(r)) if r > 0 else 0.0) + U * float(r))


def elib(fn, dfn, a: E) -> E:
    r = fn(a.v)
    return E(r, abs(float(dfn(a.v))) * a.e + C_LIB * U * abs(float(r)))


def vals(v):
    return np.array([float(x.v) for x in v])


def errs(v):
    return np.array([x.e for x in v])


def _vec(a):
    return [E(float(x)) for x in np.asarray(a, np.float64).reshape(-1)]


# ---- Eigen / numType helpers in the reference's operation order ------------------------------------------------------
def dot4(a, b):                       # coeffs (x,y,z,w), packet order (x+z)+(y+w)
    return (a[0] * b[0] + a[2] * b[2]) + (a[1] * b[1] + a[3] * b[3])


def qnormalized(q):
    n2 = dot4(q, q)
    if not n2.v > 0:
        return list(q)
    n = esqrt(n2)
    return [x / n for x in q]


def qmul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return [((aw * bx + ax * bw) + ay * bz) - az * by, ((aw * by + ay * bw) + az * bx) - ax * bz,
            ((aw * bz + az * bw) + ax * by) - ay * bx, ((aw * bw - ax * bx) - ay * by) - az * bz]


def qrot(q):                          # toRotationMatrix, quaternion as given
    x, y, z, w = q
    tx, ty, tz = 2.0 * x, 2.0 * y, 2.0 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return [1.0 - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1.0 - (txx + tzz), tyz - twx,
            txz - twy, tyz + twx, 1.0 - (txx + tyy)]


def mv3(M, v):                        # Matrix3d * Vector3d: a0 + (a1 + a2)
    return [M[3 * r] * v[0] + (M[3 * r + 1] * v[1] + M[3 * r + 2] * v[2]) for r in range(3)]


def qinverse(q):                      # conjugate / squaredNorm, zero when n2 <= 0 (the FP64 n2 decides)
    n2 = dot4(q, q)
    if not float(n2.v) > 0:
        return [E(0.0)] * 4
    return [-q[0] / n2, -q[1] / n2, -q[2] / n2, q[3] / n2]


def slerp_decision(a, b):
    """(d, absD >= one) of Eigen's slerp, in FP64."""
    d = (float(a[0]) * float(b[0]) + float(a[2]) * float(b[2])) + (float(a[1]) * float(b[1]) + float(a[3]) * float(b[3]))
    return d, abs(d) >= ONE


def slerp(a, t: E, b):
    """Eigen 3.3.7 QuaternionBase::slerp; a, b are FP64 quaternions (x,y,z,w), t an E.  Returns (quaternion, info)."""
    d_fp, lerp = slerp_decision(a, b)
    A, B = _vec(a), _vec(b)
    d = dot4(A, B)
    absD = E(abs(d.v), d.e)
    if lerp:
        s0, s1 = 1.0 - t, t
        theta = None
    else:
        x = absD.v
        if x >= 1:
            raise ValueError("slerp: the exact |d| is not below 1 on the acos branch")
        th = mp.acos(x)
        e_th = absD.e / float(mp.sqrt(1 - x * x)) + C_LIB * U * float(th)
        sth = mp.sin(th)
        theta = float(th)

        def weight(w: E):
            # sin(w theta) / sin(theta), its error through d/dtheta and d/dw, plus the roundings of w*theta, both sines
            # and the quotient
            wv = w.v
            s = mp.sin(wv * th)
            r = s / sth
            d_dth = (wv * mp.cos(wv * th) * sth - s * mp.cos(th)) / (sth * sth)
            d_dw = th * mp.cos(wv * th) / sth
            e = (abs(float(d_dth)) * e_th + abs(float(d_dw)) * w.e + U * abs(float(wv * th * mp.cos(wv * th) / sth))
                 + C_LIB * U * abs(float(r)) + C_LIB * U * abs(float(r)) + U * abs(float(r)))
            return E(r, e)
        s0, s1 = weight(1.0 - t), weight(t)
    if d_fp < 0:
        s1 = -s1
    q = [s0 * A[i] + s1 * B[i] for i in range(4)]
    return q, dict(d=d_fp, lerp=lerp, theta=theta, d_err=d.e)


def so3_to_quat(w, wf):
    """numType::so3ToQuat of an E 3-vector w; the branch is taken on theta of wf, the same vector as FP64 computes it.
    Returns (quaternion, FP64 theta)."""
    th_fp = math.sqrt(wf[0] * wf[0] + (wf[1] * wf[1] + wf[2] * wf[2]))
    n2 = w[0] * w[0] + (w[1] * w[1] + w[2] * w[2])
    if th_fp < K_THETA:
        return qnormalized([w[0] / 2.0, w[1] / 2.0, w[2] / 2.0, E(1.0)]), th_fp
    theta = esqrt(n2)
    u = [x / theta for x in w]                                         # Vector3d::normalized()
    half = 0.5 * theta
    s = elib(mp.sin, mp.cos, half)
    c = elib(mp.cos, lambda x: -mp.sin(x), half)
    return qnormalized([u[0] * s, u[1] * s, u[2] * s, c]), th_fp


def _point(R, R_il, t_il, raw, trans):
    b = mv3(R_il, raw)
    b = [b[i] + t_il[i] for i in range(3)]
    p = mv3(R, b)
    return [p[i] + trans[i] for i in range(3)]


def transform_point_fp64(raw_xyz, q, t, R_il, t_il) -> np.ndarray:
    """transformPoint (src/utility.cpp:314-318) in FP64, one IEEE rounding per operation: R(q) (R_il raw + t_il) + t, with
    toRotationMatrix of q as given and Eigen's a0 + (a1 + a2) products."""
    R = qrot([float(v) for v in np.asarray(q, np.float64).reshape(4)])
    Ril = [float(v) for v in np.asarray(R_il, np.float64).reshape(9)]
    til = [float(v) for v in np.asarray(t_il, np.float64).reshape(3)]
    tt = [float(v) for v in np.asarray(t, np.float64).reshape(3)]
    return np.array([_point(R, Ril, til, p, tt) for p in np.asarray(raw_xyz, np.float64).reshape(-1, 3).tolist()]).reshape(-1, 3)


# ---- FP64 decisions ------------------------------------------------------------------------------------------------
def time_points(t0: float, rel) -> np.ndarray:
    """time_point = time_frame_begin + relative_time / 1000.0 (numpy float64: one IEEE rounding per operation)."""
    return np.float64(t0) + np.asarray(rel, np.float64) / 1000.0


def nudge(tp: float, lo: float, hi: float) -> tuple[float, int]:
    """The two nudges of :216-217 / :266-267 in FP64; flags bit 0 / bit 1 when the first / second fires."""
    f = 0
    if abs(tp - lo) < NUDGE:
        tp = lo + NUDGE
        f |= 1
    if abs(tp - hi) < NUDGE:
        tp = hi - NUDGE
        f |= 2
    return tp, f


def walk(t0: float, rel, ts) -> tuple[int, np.ndarray]:
    """distortFrameByImu's one iterator over the points inside the loop over the IMU intervals, in FP64.
    Returns (number of points written, interval index per written point)."""
    tp = time_points(t0, rel).tolist()
    ts = [float(x) for x in ts]
    it, n = 0, len(tp)
    k_of = []
    for k in range(len(ts) - 1):
        lo, hi = ts[k] - NUDGE, ts[k + 1] + NUDGE
        while it != n and tp[it] > lo and tp[it] < hi:
            k_of.append(k)
            it += 1
    return it, np.array(k_of, np.int64)


def alpha_fp(tp: float, tb: float, te: float) -> tuple[float, int]:
    with np.errstate(divide="ignore", invalid="ignore"):     # IEEE: x / 0 = +-inf (one IMU state)
        a = float(np.float64(tp - tb) / np.float64(te - tb))
    c = 0
    if a > 1:
        a, c = 1.0, 1
    if a < 0:
        a, c = 0.0, -1
    return a, c


def grid_keys(xyz, size: float):
    """static_cast<short>(x / size) per axis in FP64, with the quotients.  Quotients with |q| >= 32765 or NaN leave the
    key undefined (the reference's cast is undefined there; srl_grid_sampling makes no cell): key row = None."""
    q = np.asarray(xyz, np.float64) / np.float64(size)
    keys = []
    for row in q:
        if np.all(np.abs(row) < 32765.0):
            keys.append(tuple(int(math.trunc(x)) for x in row))
        else:
            keys.append(None)
    return keys, q


def grid_sampling(xyz, size: float) -> list[int]:
    """First frame index of every cell, in frame order of first appearance (the set the reference keeps; its output
    ORDER is the hash container's and is checked against the oracle)."""
    keys, _ = grid_keys(xyz, size)
    seen, out = set(), []
    for i, k in enumerate(keys):
        if k is not None and k not in seen:
            seen.add(k)
            out.append(i)
    return out


# ---- the three functions -----------------------------------------------------------------------------------------
def distort_constant_point(raw, rel: float, states, t0: float, R_il, t_il):
    """One point of distortFrameByConstant: (imu_point as E[3], decisions)."""
    a, b = states[0], states[-1]
    tb, te = float(t0), float(b["timestamp"])
    tp = float(time_points(t0, [rel])[0])
    tp, f = nudge(tp, tb, te)
    al_fp, clamp = alpha_fp(tp, tb, te)
    alpha = E(al_fp) if clamp else (E(tp) - E(tb)) / (E(te) - E(tb))
    q, info = slerp(np.asarray(a["quat"], float), alpha, np.asarray(b["quat"], float))
    w0 = 1.0 - alpha
    ta, tb_ = _vec(a["trans"]), _vec(b["trans"])
    trans = [w0 * ta[i] + alpha * tb_[i] for i in range(3)]
    p = _point(qrot(q), _vec(R_il), _vec(t_il), _vec(raw), trans)
    return p, dict(tp=tp, nudge=f, alpha=al_fp, clamp=clamp, **info)


def distort_imu_point(raw, tp: float, sa, sb, R_il, t_il):
    """One point of distortFrameByImu inside interval (sa, sb), tp the FP64 time_point before the nudges."""
    ta, tb = float(sa["timestamp"]), float(sb["timestamp"])
    tp, f = nudge(tp, ta, tb)
    dt = E(tp) - E(ta)
    dt_fp = tp - ta
    gyr = _vec(sb["un_gyr"])
    dq, th = so3_to_quat([g * dt for g in gyr], [float(g.v) * dt_fp for g in gyr])
    q = qnormalized(qmul(_vec(sa["quat"]), dq))
    t, v, acc = _vec(sa["trans"]), _vec(sa["vel"]), _vec(sb["un_acc"])
    trans = [(t[i] + v[i] * dt) + ((0.5 * acc[i]) * dt) * dt for i in range(3)]
    p = _point(qrot(q), _vec(R_il), _vec(t_il), _vec(raw), trans)
    return p, dict(tp=tp, nudge=f, dt=dt_fp, theta=th, small=th < K_THETA)


def transform_all_imu_point(imu, last, R_il, t_il):
    """One point of transformAllImuPoint: R_il^T (R(q^-1) imu + t_inv) - R_il^T t_il."""
    qi = qinverse(_vec(last["quat"]))
    Rinv = qrot(qi)
    tinv = [-x for x in mv3(Rinv, _vec(last["trans"]))]
    R = np.asarray(R_il, float).reshape(3, 3)
    Rt = _vec(R.T)
    off = mv3(Rt, _vec(t_il))
    a = mv3(Rinv, _vec(imu))
    a = [a[i] + tinv[i] for i in range(3)]
    b = mv3(Rt, a)
    return [b[i] - off[i] for i in range(3)]
