"""A restatement of imageProcessing::vioEsikf (src/imageProcessing.cpp:220-380) and vioPhotometric (:402-552) in mpmath at 50
digits on the exact FP64 inputs, with every quirk of DESIGN.md section 5 kept: both iterations of vioEsikf, the photometric break
after iteration 0 when acc_residual / n < 10 (n counting the points skipped for N_rgb < 3), the Huber scale on both the residual
and the rows, acc_residual of the scaled photometric residual, R_mat_inv = 1 / cov_rgb, the extrinsic Jacobian -J_u_pc *
R_imu_cameraᵀ, the posterior covariance from the last iteration's K, H and solution.

cloudFrame::getRgb (src/lioOptimization.cpp:71-140) is restated exactly in numpy (get_rgb): each tap's four saturated products
cvRound(pixel * weight), their saturated sums, the float32 sums of the eight derivative taps divided by the float 20 in double,
evaluated at the FP64 rounding of the exact projection; taps are clamped to the nearest row and column as the device does.

The state is the 38-double layout of srl_vio_state: rotation (x, y, z, w), translation, R_imu_camera (row-major),
t_imu_camera, fx, fy, cx, cy, time_td, q_world_camera, t_world_camera, q_camera_world, t_camera_world.
"""
import numpy as np
from mpmath import mp, mpf

mp.dps = 50
THETA = mpf("0.0001")     # THETA_THRESHOLD
MIN_POINTS = 10


# ---- getRgb ------------------------------------------------------------------------------------------------------------
def _clamp(f, n):
    return n - 1 if f >= n - 1 else (int(f) if f > 0 else 0)


def sub_pixel(img, row, col):
    """getSubPixel<cv::Vec3b>(img, row, col) with the taps clamped to the image: 3 uint8 values."""
    rows, cols = img.shape[:2]
    fr, fc = np.floor(row), np.floor(col)
    frr, frc = row - fr, col - fc
    w = [(1.0 - frr) * (1.0 - frc), frr * (1.0 - frc), (1.0 - frr) * frc, frr * frc]
    r0, r1, c0, c1 = _clamp(fr, rows), _clamp(fr + 1.0, rows), _clamp(fc, cols), _clamp(fc + 1.0, cols)
    taps = [img[r0, c0], img[r1, c0], img[r0, c1], img[r1, c1]]
    out = np.zeros(3, np.int64)
    for ch in range(3):
        acc = 0
        for k in range(4):
            p = float(taps[k][ch]) * w[k]
            v = np.rint(p)
            v = 0 if not np.isfinite(v) or v < 0 else (255 if v > 255 else int(v))
            acc = min(acc + v, 255)
        out[ch] = acc
    return out


def get_rgb(img, u, v):
    """(value, dx, dy) of getRgb(u, v, 0, &dx, &dy) as float64 3-vectors."""
    c = sub_pixel(img, v, u).astype(np.float64)
    left, right = np.zeros(3, np.float32), np.zeros(3, np.float32)
    pd = np.float32(0)
    for b in range(1, 5):
        left = (left + sub_pixel(img, v, u - b).astype(np.float32)).astype(np.float32)
        right = (right + sub_pixel(img, v, u + b).astype(np.float32)).astype(np.float32)
        pd = np.float32(pd + np.float32(2 * b))
    dx = (right - left).astype(np.float32).astype(np.float64) / np.float64(pd)
    down, up = np.zeros(3, np.float32), np.zeros(3, np.float32)
    pd = np.float32(0)
    for b in range(1, 5):
        down = (down + sub_pixel(img, v - b, u).astype(np.float32)).astype(np.float32)
        up = (up + sub_pixel(img, v + b, u).astype(np.float32)).astype(np.float32)
        pd = np.float32(pd + np.float32(2 * b))
    dy = (up - down).astype(np.float32).astype(np.float64) / np.float64(pd)
    return c, dx, dy


# ---- rotations (exact) ---------------------------------------------------------------------------------------------------
def q_to_R(q):
    x, y, z, w = q
    return mp.matrix([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                      [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                      [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


# R_to_q's branch inputs: while a list is set here, each call appends (role, trace, m00, m11, m22), the values as float64
_BRANCH_LOG = None


def R_to_q(m, role=None):
    """Eigen's Quaterniond(Matrix3d) (the branch by the trace, then by the largest diagonal entry)."""
    q = [mpf(0)] * 4
    t = m[0, 0] + m[1, 1] + m[2, 2]
    if _BRANCH_LOG is not None:
        _BRANCH_LOG.append((role, float(t), float(m[0, 0]), float(m[1, 1]), float(m[2, 2])))
    if t > 0:
        t = mp.sqrt(t + 1); q[3] = t / 2; t = mpf(1) / (2 * t)
        q[0] = (m[2, 1] - m[1, 2]) * t; q[1] = (m[0, 2] - m[2, 0]) * t; q[2] = (m[1, 0] - m[0, 1]) * t
    else:
        i = 0
        if m[1, 1] > m[0, 0]:
            i = 1
        if m[2, 2] > m[i, i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        t = mp.sqrt(m[i, i] - m[j, j] - m[k, k] + 1); q[i] = t / 2; t = mpf(1) / (2 * t)
        q[3] = (m[k, j] - m[j, k]) * t; q[j] = (m[j, i] + m[i, j]) * t; q[k] = (m[k, i] + m[i, k]) * t
    return q


def qmul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return [aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
            aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz]


def qinv(q):
    n2 = sum(c * c for c in q)
    return [-q[0] / n2, -q[1] / n2, -q[2] / n2, q[3] / n2]


def qunit(q):
    n = mp.sqrt(sum(c * c for c in q))
    return [c / n for c in q]


def so3_to_quat(w):
    th = mp.sqrt(sum(c * c for c in w))
    if th < THETA:
        return qunit([w[0] / 2, w[1] / 2, w[2] / 2, mpf(1)])
    u = [c / th for c in w]
    s, c = mp.sin(th / 2), mp.cos(th / 2)
    return qunit([u[0] * s, u[1] * s, u[2] * s, c])


def rot2q_branch(t, m00, m11, m22):
    """the branch R_to_q takes on these inputs: "trace", or "i=0" / "i=1" / "i=2" (the largest diagonal entry)"""
    if t > 0:
        return "trace"
    d = [m00, m11, m22]
    i = 1 if d[1] > d[0] else 0
    return f"i={2 if d[2] > d[i] else i}"


def rotation_to_so3(R):
    R = q_to_R(qunit(R_to_q(R, "dq")))           # normalizeR
    th = mp.acos((R[0, 0] + R[1, 1] + R[2, 2] - 1) / 2)
    a = [R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]]
    if th < THETA:
        return [c / 2 for c in a]
    return [th * c / (2 * mp.sin(th)) for c in a]


def skew(v):
    return mp.matrix([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])


# ---- state -----------------------------------------------------------------------------------------------------------
class State:
    def __init__(self, s):
        s = [mpf(float(x)) for x in np.asarray(s, np.float64).reshape(38)]
        self.rotation = s[0:4]; self.translation = mp.matrix(s[4:7])
        self.Ric = mp.matrix([s[7:10], s[10:13], s[13:16]]); self.tic = mp.matrix(s[16:19])
        self.fx, self.fy, self.cx, self.cy, self.td = s[19:24]
        self.q_wc = s[24:28]; self.t_wc = mp.matrix(s[28:31]); self.q_cw = s[31:35]; self.t_cw = mp.matrix(s[35:38])

    def array(self):
        out = list(self.rotation) + list(self.translation) + [self.Ric[r, c] for r in range(3) for c in range(3)] + list(self.tic)
        out += [self.fx, self.fy, self.cx, self.cy, self.td] + list(self.q_wc) + list(self.t_wc) + list(self.q_cw) + list(self.t_cw)
        return np.array([float(x) for x in out])

    def update(self, d, esikf):
        """updateCameraParameters (:382-400 / :554-566) + refreshPoseForProjection"""
        o = 1 if esikf else 0
        if esikf:
            self.td += d[0]
        q = qunit(qmul(R_to_q(self.Ric, "Ric"), so3_to_quat([d[o], d[o + 1], d[o + 2]])))
        self.Ric = q_to_R(q)
        self.tic = self.tic + mp.matrix([d[o + 3], d[o + 4], d[o + 5]])
        if esikf:
            self.fx += d[7]; self.fy += d[8]; self.cx += d[9]; self.cy += d[10]
        Rw = q_to_R(self.rotation)
        self.q_wc = R_to_q(Rw * self.Ric, "Rwc")
        self.t_wc = Rw * self.tic + self.translation
        self.q_cw = qinv(self.q_wc)
        self.t_cw = -(q_to_R(self.q_cw) * self.t_wc)


def huber(r):
    return mpf(1) if r < 1 else (2 * mp.sqrt(r) - 1) / r


def weight(n_new_visited):
    w = 5.0 / n_new_visited if n_new_visited != 0 else float("inf")
    return mpf(max(0.001, min(w, 0.01)))


def _solve(S, g, P, Jz, dx, w, D):
    """K r, K H, solution of :361-362 / :528-529 with A⁻¹ = (I + Pw S)⁻¹ Pw (the same matrix as (S + Pw⁻¹)⁻¹)."""
    Pw = Jz * P * Jz.T * w
    M = mp.eye(D) + Pw * S
    cols = [mp.lu_solve(M, Pw.column(j)) for j in range(D)]
    Ainv = mp.matrix([[cols[j][i] for j in range(D)] for i in range(D)])
    KH = Ainv * S
    Kr = Ainv * g
    sol = -Kr - (mp.eye(D) - KH) * (Jz * dx)
    return KH, sol, M


def _f64(A):
    return np.array([[float(A[r, c]) for c in range(A.cols)] for r in range(A.rows)])


def vio_update(esikf, state, cov, xyz, uv, vel, rgb, cov_rgb, n_rgb, n_new_visited, img=None, mult=None):
    """One update on the exact inputs.  Returns dict(state (38 float64), cov (11 x 11 float64), result, iterations, used, acc,
    huber (per point, per iteration: True where the Huber branch scaled), residual_norms (per point, per iteration: what the Huber
    test compares with 1), projections (per iteration, float64 (n, 2)), acc_history (acc_residual per iteration, as the
    convergence tests read it), steps (the norm of each iteration's rotation step, which so3ToQuat compares with
    THETA_THRESHOLD), dx_rot (per iteration, the norm of d_x's rotation, whose rotationToSo3 compares its angle with
    THETA_THRESHOLD), systems (per iteration that solved: S, g and M = I + Pw S rounded to float64), rot2q (per R_to_q call in
    order: (role, trace, m00, m11, m22), role "Ric" for R_imu_camera, "Rwc" for R_world R_imu_camera, "dq" for the step
    rotation normalizeR converts)).

    mult (optional, one positive int per point): point i stands for mult[i] copies of itself in the list, its rows, acc_residual
    and used count added mult[i] times and n = sum(mult).  Exact here, so a list of repeated tiles costs what one tile costs."""
    global _BRANCH_LOG
    mult = None if mult is None else [int(m) for m in mult]
    n = len(xyz) if mult is None else sum(mult)
    D = 11 if esikf else 6
    cov_in = np.array(cov, np.float64).reshape(11, 11)
    out = dict(state=np.array(state, np.float64).reshape(38).copy(), cov=cov_in.copy(), result=0, iterations=0, used=0, acc=0.0,
               huber=[], projections=[], acc_history=[])
    if n < MIN_POINTS:
        return out
    out["result"] = 1
    _BRANCH_LOG = out["rot2q"] = []
    try:
        _iterate(out, esikf, state, cov_in, xyz, uv, vel, rgb, cov_rgb, n_rgb, n_new_visited, img, mult, n, D)
    finally:
        _BRANCH_LOG = None
    return out


def _iterate(out, esikf, state, cov_in, xyz, uv, vel, rgb, cov_rgb, n_rgb, n_new_visited, img, mult, n, D):
    st = State(state)
    o = 0 if esikf else 1
    P = mp.matrix([[mpf(float(cov_in[r + o, c + o])) for c in range(D)] for r in range(D)])
    w = weight(n_new_visited)
    pred = State(state)
    last = mpf("3e8")
    KH = sol = None
    for it in range(2):
        d_so3 = rotation_to_so3(q_to_R(qmul(qinv(R_to_q(pred.Ric, "Ric")), R_to_q(st.Ric, "Ric"))))
        d_p = st.tic - pred.tic
        if esikf:
            dx = mp.matrix([st.td - pred.td] + d_so3 + list(d_p) + [st.fx - pred.fx, st.fy - pred.fy, st.cx - pred.cx, st.cy - pred.cy])
        else:
            dx = mp.matrix(d_so3 + list(d_p))
        out.setdefault("dx_rot", []).append(float(mp.sqrt(sum(c * c for c in d_so3))))
        Rcw = q_to_R(st.q_cw)
        S = mp.zeros(D, D); g = mp.zeros(D, 1)
        acc = mpf(0); used = 0
        npt = len(xyz)
        hub = np.zeros(npt, bool); proj = np.full((npt, 2), np.nan); rn = np.full(npt, np.nan)
        for i in range(npt):
            if not esikf and n_rgb[i] < 3:
                continue
            m = 1 if mult is None else mult[i]
            pw = mp.matrix([mpf(float(np.float32(x))) for x in xyz[i]])
            pc = Rcw * pw + st.t_cw
            x, y, z = pc[0], pc[1], pc[2]
            v0, v1 = mpf(float(vel[i][0])), mpf(float(vel[i][1]))
            pu = st.fx * x / z + st.cx + st.td * v0
            pv = st.fy * y / z + st.cy + st.td * v1
            proj[i] = (float(pu), float(pv))
            J = mp.matrix([[st.fx / z, 0, -(st.fx * x) / (z * z)], [0, st.fy / z, -(st.fy * y) / (z * z)]])
            used += m
            if esikf:
                e = mp.matrix([pu - mpf(float(np.float32(uv[i][0]))), pv - mpf(float(np.float32(uv[i][1])))])
                res = mp.sqrt(e[0] ** 2 + e[1] ** 2)
                h = huber(res)
                hub[i] = res >= 1; rn[i] = float(res)
                acc += res * m
                H = mp.zeros(2, 11)
                JS = J * skew(pc); JR = -J * st.Ric.T
                for k in range(2):
                    H[k, 0] = (v0 if k == 0 else v1) * h
                    for j in range(3):
                        H[k, 1 + j] = JS[k, j] * h
                        H[k, 4 + j] = JR[k, j] * h
                H[0, 7] = x / z * h; H[0, 9] = h; H[1, 8] = y / z * h; H[1, 10] = h
                r = e * h
                S += H.T * H * m; g += H.T * r * m
            else:
                col, cdx, cdy = get_rgb(img, float(pu), float(pv))
                e = mp.matrix([mpf(float(col[c])) - int(rgb[i][c]) for c in range(3)])
                info = [1 / mpf(float(np.float32(cov_rgb[i][c]))) for c in range(3)]
                nrm = mp.sqrt(e[0] ** 2 + e[1] ** 2 + e[2] ** 2)
                h = huber(nrm)
                hub[i] = nrm >= 1; rn[i] = float(nrm)
                r = e * h
                acc += sum(r[c] * info[c] * r[c] for c in range(3)) * m
                Jcu = mp.matrix([[mpf(float(cdx[c])), mpf(float(cdy[c]))] for c in range(3)])
                Jc = Jcu * J
                A1 = Jc * skew(pc) * h; A2 = -Jc * st.Ric.T * h
                H = mp.zeros(3, 6)
                for k in range(3):
                    for j in range(3):
                        H[k, j] = A1[k, j]; H[k, 3 + j] = A2[k, j]
                Rinv = mp.diag(info)
                S += H.T * Rinv * H * m; g += H.T * Rinv * r * m
        if esikf:
            acc = acc / n
        out["huber"].append(hub); out["projections"].append(proj); out["acc_history"].append(acc)
        out.setdefault("residual_norms", []).append(rn)
        out["used"] = used
        if used < MIN_POINTS:
            break
        Jz = mp.eye(D)
        so = 1 if esikf else 0
        Js = mp.eye(3) - skew([dx[so], dx[so + 1], dx[so + 2]]) / 2
        for a in range(3):
            for b in range(3):
                Jz[so + a, so + b] = Js[a, b]
        KH, sol, M = _solve(S, g, P, Jz, dx, w, D)
        out.setdefault("systems", []).append(dict(S=_f64(S), g=_f64(g).reshape(D), M=_f64(M)))
        st.update([sol[k] for k in range(D)], esikf)
        out.setdefault("steps", []).append(float(mp.sqrt(sum(sol[so + k] ** 2 for k in range(3)))))
        out["iterations"] += 1
        out["acc"] = float(acc)
        if not esikf and acc / n < 10:
            break
        if abs(acc - last) < mpf("0.01"):
            break
        last = acc
    if KH is not None:
        so = 1 if esikf else 0
        Jk = mp.eye(D)
        Js = mp.eye(3) - skew([sol[so], sol[so + 1], sol[so + 2]]) / 2
        for a in range(3):
            for b in range(3):
                Jk[so + a, so + b] = Js[a, b]
        Pn = Jk * (mp.eye(D) - KH) * P * Jk.T
        cv = cov_in.copy()
        for r in range(D):
            for c in range(D):
                cv[r + o, c + o] = float(Pn[r, c])
        out["cov"] = cv
    out["state"] = st.array()
