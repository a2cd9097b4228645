"""A 50-digit restatement of one step of the iterated ESIKF update, the truth the host and device loops are measured against.

What is restated: lioOptimization::updateIEKF between two passes (src/optimize.cpp:172-310), eskfEstimator::observe
(src/eskfEstimator.cpp:219-230), the numType helpers it calls (include/utility.h:194-330) and AngularDistance
(src/utility.cpp:146-153).  It is evaluated in mpmath at 50 significant digits on the exact FP64 inputs (state,
prediction, covariance, HTH, HTh, laser_point_cov, thresholds), keeping every quirk of the reference: the two 17x17
inverses, acos without a clamp, the in-place column loops of the posterior covariance that read the partly updated P
(:287-297) and the K_x row projections (:299-303).  Only the arithmetic is exact; every branch is taken on the exact
value.  `step()` also returns the margins of every decision and the condition numbers the error bounds need.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import mpmath as mp
import numpy as np

DPS = 50
N = 17
K_THETA = mp.mpf("1e-4")           # THETA_THRESHOLD, include/utility.h:27


def _m(x):
    return mp.mpf(float(x))


def _vec(a):
    return [_m(x) for x in np.asarray(a, np.float64).reshape(-1)]


def _mat(a, r, c):
    a = np.asarray(a, np.float64).reshape(r, c)
    return [[_m(a[i, j]) for j in range(c)] for i in range(r)]


def _mm(A, B):
    return [[mp.fsum(A[i][k] * B[k][j] for k in range(len(B))) for j in range(len(B[0]))] for i in range(len(A))]


def _mv(A, v):
    return [mp.fsum(A[i][k] * v[k] for k in range(len(v))) for i in range(len(A))]


def _tr(A):
    return [list(r) for r in zip(*A)]


def _eye(n):
    return [[mp.mpf(1) if i == j else mp.mpf(0) for j in range(n)] for i in range(n)]


def _add(A, B, s=1):
    return [[A[i][j] + s * B[i][j] for j in range(len(A[0]))] for i in range(len(A))]


def _scale(s, A):
    return [[s * x for x in r] for r in A]


def _nrm(v):
    return mp.sqrt(mp.fsum(x * x for x in v))


def _unit(v):
    n = _nrm(v)
    return [x / n for x in v] if n > 0 else list(v)


def _hat(v):
    z = mp.mpf(0)
    return [[z, -v[2], v[1]], [v[2], z, -v[0]], [-v[1], v[0], z]]


def _acos(x):
    # acos is not clamped in the reference; in exact arithmetic its argument never leaves [-1, 1] by more than the
    # working precision, so the truth of the formula is the clamped value
    if x > 1 and x - 1 < mp.mpf("1e-40"):
        return mp.mpf(0)
    if x < -1 and -1 - x < mp.mpf("1e-40"):
        return mp.pi
    return mp.acos(x)


# ---- quaternions (x, y, z, w) ----------------------------------------------------------------------------------
def _qmul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return [aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
            aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz]


def _qinv(q):
    n2 = mp.fsum(x * x for x in q)
    return [-q[0] / n2, -q[1] / n2, -q[2] / n2, q[3] / n2]


def _qunit(q):
    n = _nrm(q)
    return [x / n for x in q]


def _qrot(q):   # Eigen's toRotationMatrix (not normalised)
    x, y, z, w = q
    tx, ty, tz = 2 * x, 2 * y, 2 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return [[1 - (tyy + tzz), txy - twz, txz + twy], [txy + twz, 1 - (txx + tzz), tyz - twx], [txz - twy, tyz + twx, 1 - (txx + tyy)]]


def _rot2q(m):   # Eigen's matrix -> quaternion
    t = m[0][0] + m[1][1] + m[2][2]
    q = [mp.mpf(0)] * 4
    if t > 0:
        t = mp.sqrt(t + 1)
        q[3] = t / 2
        t = mp.mpf(1) / (2 * t)
        q[0] = (m[2][1] - m[1][2]) * t
        q[1] = (m[0][2] - m[2][0]) * t
        q[2] = (m[1][0] - m[0][1]) * t
    else:
        i = 0
        if m[1][1] > m[0][0]:
            i = 1
        if m[2][2] > m[i][i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        t = mp.sqrt(m[i][i] - m[j][j] - m[k][k] + 1)
        q[i] = t / 2
        t = mp.mpf(1) / (2 * t)
        q[3] = (m[k][j] - m[j][k]) * t
        q[j] = (m[j][i] + m[i][j]) * t
        q[k] = (m[k][i] + m[i][k]) * t
    return q


# ---- numType helpers ----------------------------------------------------------------------------------------------
def log_so3(Rin):
    """numType::rotationToSo3: normalizeR, then acos without a clamp (include/utility.h:267-280)."""
    R = _qrot(_qunit(_rot2q(Rin)))
    th = _acos((R[0][0] + R[1][1] + R[2][2] - 1) / 2)
    a = [R[2][1] - R[1][2], R[0][2] - R[2][0], R[1][0] - R[0][1]]
    if th < K_THETA:
        return [x / 2 for x in a], th
    return [th * x / (2 * mp.sin(th)) for x in a], th


def exp_so3(w):
    """numType::so3ToRotation (include/utility.h:282-299)."""
    th = _nrm(w)
    if th < K_THETA:
        U = _hat(w)
        return _add(_add(_eye(3), U), _scale(mp.mpf("0.5"), _mm(U, U)))
    U = _hat(_unit(w))
    return _add(_add(_eye(3), _scale(mp.sin(th), U)), _scale(1 - mp.cos(th), _mm(U, U)))


def exp_quat(w):
    """numType::so3ToQuat (include/utility.h:301-324)."""
    th = _nrm(w)
    if th < K_THETA:
        return _qunit([w[0] / 2, w[1] / 2, w[2] / 2, mp.mpf(1)])
    u = _unit(w)
    s, c = mp.sin(th / 2), mp.cos(th / 2)
    return _qunit([u[0] * s, u[1] * s, u[2] * s, c])


def s2_basis(gin):
    """numType::derivativeS2 (include/utility.h:215-235), 3x2."""
    g = _unit(gin)
    b01 = -g[0] * g[1] / (1 + g[2])
    return [[1 - g[0] * g[0] / (1 + g[2]), b01], [b01, 1 - g[1] * g[1] / (1 + g[2])], [-g[0], -g[1]]]


def angular_distance(w):
    """AngularDistance (src/utility.cpp:146-153), degrees, acos not clamped."""
    R = exp_so3(w)
    return _acos((R[0][0] + R[1][1] + R[2][2] - 1) / 2) * 180 / mp.pi


# ---- one step ---------------------------------------------------------------------------------------------------
@dataclass
class StepResult:
    d_x: np.ndarray
    diverged: bool
    converged: bool
    final: bool
    state: dict                       # after observe (unchanged when diverged), cov = posterior when final
    margins: dict                     # |value - threshold| of every decision, in the decision's unit
    cond: dict                        # condition numbers and norms the error bounds need
    branches: dict = field(default_factory=dict)   # which side of each small-angle branch the exact values took
    mp_state: dict = field(default_factory=dict)


def _cond2(A):
    s = np.linalg.svd(np.asarray(A, np.float64), compute_uv=False)
    return float(s[0] / s[-1]) if s[-1] > 0 else float("inf")


def _to_np(A):
    return np.array([[float(x) for x in r] for r in A])


def step(cur: dict, pred: dict, HTH, HTh, laser_cov: float, thr_t: float, thr_r: float, frame_id: int,
         i_pass: int, max_iter: int) -> StepResult:
    """One pass of updateIEKF after buildPlaneResiduals (src/optimize.cpp:172-310) from the exact FP64 inputs.
    cur / pred: dicts with p q v ba bg g (and cov in cur).  i_pass: the loop index i of this pass (-1 first)."""
    with mp.workdps(DPS):
        p, q, v, ba, bg, g = (_vec(cur[k]) for k in ("p", "q", "v", "ba", "bg", "g"))
        pp, qp, vp, bap, bgp, gp = (_vec(pred[k]) for k in ("p", "q", "v", "ba", "bg", "g"))
        P0 = _mat(cur["cov"], N, N)
        H = _mat(HTH, 6, 6)
        h = _vec(HTh)
        c = _m(laser_cov)
        # boxminus (:172-211)
        d_p = [p[i] - pp[i] for i in range(3)]
        d_so3, th_so3 = log_so3(_qrot(_qmul(_qinv(qp), q)))
        d_v = [v[i] - vp[i] for i in range(3)]
        d_ba = [ba[i] - bap[i] for i in range(3)]
        d_bg = [bg[i] - bgp[i] for i in range(3)]
        gpn, gn = _unit(gp), _unit(g)
        cr = [gpn[1] * gn[2] - gpn[2] * gn[1], gpn[2] * gn[0] - gpn[0] * gn[2], gpn[0] * gn[1] - gpn[1] * gn[0]]
        dot = mp.fsum(gpn[i] * gn[i] for i in range(3))
        one_minus_dot = 1 - dot
        if abs(one_minus_dot) < mp.mpf("1e-6"):
            R_dg = _eye(3)
        else:
            sk = _hat(cr)
            den = mp.fsum(x * x for x in cr)
            R_dg = _add(_add(_eye(3), sk), _scale(one_minus_dot / den, _mm(sk, sk)))
        so3_dg, th_dg = log_so3(R_dg)
        Bp = s2_basis(gp)
        d_g = _mv(_tr(Bp), so3_dg)
        J_so3 = _add(_eye(3), _scale(mp.mpf("0.5"), _hat(d_so3)), -1)                     # :213
        J_s2 = _add(_eye(2), _scale(mp.mpf("0.5"), _mm(_tr(Bp), _mm(_hat(so3_dg), Bp))))     # :214
        dx = d_p + d_so3 + d_v + d_ba + d_bg + d_g
        dx_new = list(dx)
        dx_new[3:6] = _mv(J_so3, d_so3)                                                     # :217
        dx_new[15:17] = _mv(J_s2, d_g)                                                      # :218
        # covariance projection (:220-232)
        P = [list(r) for r in P0]
        for j in range(N):
            col = _mv(J_so3, [P[3][j], P[4][j], P[5][j]])
            P[3][j], P[4][j], P[5][j] = col
            col = _mv(J_s2, [P[15][j], P[16][j]])
            P[15][j], P[16][j] = col
        for j in range(N):
            row = _mv(J_so3, [P[j][3], P[j][4], P[j][5]])
            P[j][3], P[j][4], P[j][5] = row
            row = _mv(J_s2, [P[j][15], P[j][16]])
            P[j][15], P[j][16] = row
        # gain (:234-242): the reference's two 17x17 inverses
        A = mp.matrix([[x / c for x in r] for r in P])
        sing = False
        try:
            temp = A ** -1
        except ZeroDivisionError:
            sing = True
        if sing:
            raise ZeroDivisionError("P / laser_point_cov is singular")
        for r in range(6):
            for cc in range(6):
                temp[r, cc] += H[r][cc]
        temp_inv = temp ** -1
        T = [[temp_inv[r, a] for a in range(6)] for r in range(N)]
        K_h = _mv(T, h)
        K_x6 = _mm(T, H)                                                                    # columns >= 6 are zero
        d_x = [-K_h[r] + mp.fsum((K_x6[r][cc] - (1 if r == cc else 0)) * dx_new[cc] for cc in range(6))
               - (dx_new[r] if r >= 6 else 0) for r in range(N)]
        mats = dict(c=float(c), S=_to_np([[temp[r, cc] for cc in range(N)] for r in range(N)]),
                    Sinv=_to_np([[temp_inv[r, cc] for cc in range(N)] for r in range(N)]), P=_to_np(P), T=_to_np(T), H=_to_np(H), h=np.array([float(x) for x in h]),
                    dxn=np.array([float(x) for x in dx_new]), d_x=np.array([float(x) for x in d_x]))
        n_dp = _nrm(d_x[0:3])
        ang = angular_distance(d_x[3:6])
        th_dx = _nrm(d_x[3:6])
        diverged = bool(n_dp > 100 or ang > 100)                                            # :248-251
        converged = bool(not diverged and frame_id > 1 and n_dp < _m(thr_t) and ang < _m(thr_r))   # :265-270
        final = bool(not diverged and (converged or i_pass == max_iter - 1))               # :272
        st = dict(p=p, q=q, v=v, ba=ba, bg=bg, g=g, cov=P0)
        if not diverged:                                                                    # observe (:253)
            st = dict(st)
            st["p"] = [p[i] + d_x[i] for i in range(3)]
            st["q"] = _qunit(_qmul(q, exp_quat(d_x[3:6])))
            st["v"] = [v[i] + d_x[6 + i] for i in range(3)]
            st["ba"] = [ba[i] + d_x[9 + i] for i in range(3)]
            st["bg"] = [bg[i] + d_x[12 + i] for i in range(3)]
            B = s2_basis(g)
            st["g"] = _mv(exp_so3(_mv(B, d_x[15:17])), g)
        if final:                                                                           # :272-307
            Bb = s2_basis(g)
            J2so3 = _add(_eye(3), _scale(mp.mpf("0.5"), _hat(d_x[3:6])), -1)
            J2s2 = _add(_eye(2), _scale(mp.mpf("0.5"), _mm(_tr(Bb), _mm(_hat(_mv(Bb, d_x[15:17])), Bb))))
            Pn = [list(r) for r in P]
            for j in range(N):                                                              # :281-285 (read P)
                Pn[3][j], Pn[4][j], Pn[5][j] = _mv(J2so3, [P[3][j], P[4][j], P[5][j]])
                Pn[15][j], Pn[16][j] = _mv(J2s2, [P[15][j], P[16][j]])
            for j in range(N):                                                              # :287-291
                Pn[j][3], Pn[j][4], Pn[j][5] = _mv(J2so3, [P[j][3], P[j][4], P[j][5]])
                P[j][3], P[j][4], P[j][5] = _mv(J2so3, [P[j][3], P[j][4], P[j][5]])
            for j in range(N):                                                              # :293-297
                Pn[j][15], Pn[j][16] = _mv(J2s2, [P[j][15], P[j][16]])
                P[j][15], P[j][16] = _mv(J2s2, [P[j][15], P[j][16]])
            Kx = [list(r) for r in K_x6]                                                    # :299-303
            for cc in range(6):
                Kx[3][cc], Kx[4][cc], Kx[5][cc] = _mv(J2so3, [Kx[3][cc], Kx[4][cc], Kx[5][cc]])
                Kx[15][cc], Kx[16][cc] = _mv(J2s2, [Kx[15][cc], Kx[16][cc]])
            st["cov"] = [[Pn[r][cc] - mp.fsum(Kx[r][a] * P[a][cc] for a in range(6)) for cc in range(N)] for r in range(N)]
            mats.update(Pn=_to_np(Pn), Kx=_to_np(Kx), P6=_to_np(P[0:6]))
        # what the bounds need (float64 is enough for a condition number)
        Pn_np = _to_np(P0)
        A66 = _to_np([[x / c for x in r[0:6]] for r in P])[0:6]
        A6 = _to_np([[x / c for x in r[0:6]] for r in P])
        H_np = _to_np(H)
        M = np.eye(6) + H_np @ A66
        Minv = np.linalg.inv(M) if np.isfinite(M).all() and abs(np.linalg.det(M)) > 0 else np.full((6, 6), np.inf)
        cond = dict(kP=_cond2(_to_np(P)), kS=_cond2(_to_np([[temp[r, cc] for cc in range(N)] for r in range(N)])),
                    kM=_cond2(M), nT=float(np.linalg.norm(_to_np(T), 2)), nA6=float(np.linalg.norm(A6, 2)),
                    nMinv=float(np.linalg.norm(Minv, 2)), nH=float(np.linalg.norm(H_np, 2)),
                    nh=float(np.linalg.norm(_to_np([h]))), ndx=float(np.linalg.norm(_to_np([dx_new]))),
                    nP=float(np.linalg.norm(Pn_np, 2)), M=M, mats=mats)
        margins = dict(dp_100=abs(float(n_dp) - 100.0), ang_100=abs(float(ang) - 100.0),
                       dp_thr=abs(float(n_dp) - thr_t), ang_thr=abs(float(ang) - thr_r), thr_dp=thr_t, thr_ang=thr_r)
        branches = dict(th_dx=float(th_dx), th_so3=float(th_so3), th_dg=float(th_dg), one_minus_dot=float(one_minus_dot),
                        n_dp=float(n_dp), ang=float(ang))
        out_state = {k: (_to_np(v_) if k == "cov" else np.array([float(x) for x in v_])) for k, v_ in st.items()}
        return StepResult(d_x=np.array([float(x) for x in d_x]), diverged=diverged, converged=converged, final=final,
                          state=out_state, margins=margins, cond=cond, branches=branches, mp_state=st)
