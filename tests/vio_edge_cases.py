"""Edge cases of the two camera updates (srl_vio.cu, k_vio_update) where the kernel's own structure could go wrong while the
seeded scenes of vio_cases pass: chunk boundaries and short last chunks of the segment sums, the row swaps of the pivoted
Gauss-Jordan solve, steps below THETA_THRESHOLD, non-finite and gross measurements, and every branch of Quaterniond(Matrix3d).

Every builder takes a scene dict (vio_cases.device_scene's, or a host stand-in from stand_in() with the same keys) and asserts
its own premise where that needs no update; the premises that need the restated update (swap columns, step sizes, branches)
are checked by the tests on the restatement's outputs, with the helpers here.
"""
import numpy as np

import vio_cases as VC

# k_vio_update's layout: 256 threads, points in chunks of 128; E sums (the upper triangle of S, g, acc_residual, used) split
# into floor(256 / E) contiguous segments of each chunk's rows
THREADS, CHUNK = 256, 128
CHUNK_NS = (10, 127, 128, 129, 130, 255, 256, 257)


def dims(esikf):
    D = 11 if esikf else 6
    E = D * (D + 1) // 2 + D + 2
    return D, (2 if esikf else 3), E, THREADS // E


def chunk_shape(n, esikf):
    """(chunks, points in the last chunk, rows in the last chunk, segments, segments of the last chunk that hold rows)"""
    _, rpp, _, P = dims(esikf)
    chunks = -(-n // CHUNK)
    last = n - (chunks - 1) * CHUNK
    rows = last * rpp
    ln = -(-rows // P)
    return chunks, last, rows, P, -(-rows // ln)


# ---- scenes ------------------------------------------------------------------------------------------------------------
def stand_in(seed=501, camera="ntu", n=150, rotation=None, ric=None):
    """a host stand-in of device_scene: the same keys (ids are positions), colours drawn by make_case, N_rgb >= 3"""
    c = VC.make_case(seed, camera, n=n, zmin=3.0, zmax=12.0, rotation=rotation, ric=ric)
    return dict(c, ids=np.arange(n, dtype=np.uint32))


def exact_uv(sc, state, vel, noise_px, seed):
    """the matched points at the FP64 projections of the stored points from `state` (with time_td * velocity), plus Gaussian
    noise of noise_px: residuals far below the Huber threshold and rotation steps far below THETA_THRESHOLD"""
    from sr_livo_b200 import lio
    Rcw, tcw = lio._quat_to_rot(state[31:35]), state[35:38]
    fx, fy, cx, cy, td = state[19:24]
    pc = sc["xyz"].astype(np.float64) @ Rcw.T + tcw
    uv = np.stack([fx * pc[:, 0] / pc[:, 2] + cx + td * vel[:, 0], fy * pc[:, 1] / pc[:, 2] + cy + td * vel[:, 1]], 1)
    return (uv + np.random.default_rng(seed).normal(scale=noise_px, size=uv.shape)).astype(np.float32)


def small_step_variants(sc):
    """(name, state, uv, vel) with the matched points 1e-3 px from the projections: the scene's state and velocities, time_td
    set to 0, and all velocities 0"""
    out = []
    st0 = sc["state"].copy()
    st0[23] = 0.0
    for name, st, vel in (("small-steps", sc["state"], sc["vel"]), ("small-steps-td0", st0, sc["vel"]),
                          ("small-steps-vel0", sc["state"], np.zeros_like(sc["vel"]))):
        out.append((name, st, exact_uv(sc, st, vel, 1e-3, 17), np.ascontiguousarray(vel)))
    return out


def flat_image(sc, value=250):
    """a constant image: every getRgb derivative is 0, so S and g are 0 and (from an R_imu_camera whose quaternion has unit
    norm in FP64, and so a d_x of exactly 0) every rotation step is exactly 0, which only so3ToQuat's small-angle branch
    takes without dividing by it"""
    return np.full((sc["rows"], sc["cols"], 3), value, np.uint8)


# ---- rotation branches -------------------------------------------------------------------------------------------------
def _axis_angle(axis, angle):
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * K @ K


# a rotation per branch of Quaterniond(Matrix3d), far from every boundary: 0.5 rad (trace 2.75), and 160 degrees about an axis
# near x, y or z (trace -0.88, the largest diagonal entry 0.65 against -0.77)
BRANCH_ROTATIONS = {"trace": _axis_angle([1, 2, 3], 0.5), "i=0": _axis_angle([3, 1, 1], 2.8), "i=1": _axis_angle([1, 3, -1], 2.8),
                    "i=2": _axis_angle([-1, 1, 3], 2.8)}
# (R_imu_camera's branch, R_world R_imu_camera's branch) of the four branch scenes: each branch once for each matrix
BRANCH_PAIRS = (("trace", "i=0"), ("i=0", "i=1"), ("i=1", "i=2"), ("i=2", "trace"))


def branch_pose(ric_branch, rwc_branch):
    """(rotation (x, y, z, w), R_imu_camera) with R_imu_camera and rotation R_imu_camera in the given branches"""
    from sr_livo_b200 import lio
    ric = BRANCH_ROTATIONS[ric_branch]
    rw = BRANCH_ROTATIONS[rwc_branch] @ ric.T
    q = lio._rot_to_quat(rw)
    return q / np.linalg.norm(q), ric


def branches(truth):
    """{(role, branch)} of every Quaterniond(Matrix3d) the restated update evaluated"""
    import vio_reference as VR
    return {(r[0], VR.rot2q_branch(*r[1:])) for r in truth.get("rot2q", [])}


# ---- pivoting ----------------------------------------------------------------------------------------------------------
def pivot_replay(M):
    """the device's elimination order on M (largest |a| of the column from the diagonal down, the first index on ties):
    (columns where rows are swapped, smallest relative gap between a column's winning |a| and its runner-up)"""
    A = np.array(M, np.float64)
    D = len(A)
    swaps, gap = [], np.inf
    for k in range(D):
        col = np.abs(A[k:, k])
        p = k + int(np.argmax(col))
        if D - k > 1:
            s = np.sort(col)[::-1]
            gap = min(gap, (s[0] - s[1]) / s[0])
        if p != k:
            swaps.append(k)
            A[[k, p]] = A[[p, k]]
        rk = A[k] / A[k, k]
        f = A[:, k].copy()
        A[k] = rk
        for i in range(D):
            if i != k:
                A[i] = A[i] - f[i] * rk
    return swaps, gap


def system0(sc, esikf):
    """the iteration-0 S = Hᵀ R⁻¹ H of the scene in plain float64 (for choosing covariances; the premises use the restatement's)"""
    from sr_livo_b200 import lio
    import vio_reference as VR
    st = sc["state"]
    Rcw, tcw, Ric = lio._quat_to_rot(st[31:35]), st[35:38], st[7:16].reshape(3, 3)
    fx, fy, cx, cy, td = st[19:24]
    D = 11 if esikf else 6
    S = np.zeros((D, D))
    for i in range(len(sc["xyz"])):
        if not esikf and sc["n_rgb"][i] < 3:
            continue
        x, y, z = Rcw @ sc["xyz"][i].astype(np.float64) + tcw
        J = np.array([[fx / z, 0, -fx * x / z / z], [0, fy / z, -fy * y / z / z]])
        sk = np.array([[0, -z, y], [z, 0, -x], [-y, x, 0]])
        pu, pv = fx * x / z + cx + td * sc["vel"][i, 0], fy * y / z + cy + td * sc["vel"][i, 1]
        if esikf:
            e = np.array([pu - sc["uv"][i, 0], pv - sc["uv"][i, 1]])
            W = np.eye(2)
            H = np.zeros((2, 11))
            H[:, 0] = sc["vel"][i]; H[:, 1:4] = J @ sk; H[:, 4:7] = -J @ Ric.T
            H[0, 7], H[0, 9], H[1, 8], H[1, 10] = x / z, 1.0, y / z, 1.0
        else:
            col, dx, dy = VR.get_rgb(sc["img"], pu, pv)
            e = col - sc["rgb"][i]
            W = np.diag(1.0 / sc["cov_rgb"][i].astype(np.float64))
            Jc = np.stack([dx, dy], 1) @ J
            H = np.hstack([Jc @ sk, -Jc @ Ric.T])
        r = np.linalg.norm(e)
        h = 1.0 if r < 1 else (2 * np.sqrt(r) - 1) / r
        S += (H * h).T @ W @ (H * h)
    return S


# the swap columns each update's pivot cases force: early, middle and last (the last column has no row below it to swap)
PIVOT_TARGETS = {True: (1, 5, 9), False: (0, 2, 4)}


def pivot_covariance(sc, esikf, column, weight=0.01):
    """a diagonal covariance whose variances span six decades (seven or eight where six do not suffice; κ·ε is then 2.2e-10 to
    2.2e-8), chosen by a seeded search so that the device's elimination of I + Pw S swaps rows at `column` with every pivot 5 %
    clear of its runner-up (on the plain float64 iteration-0 system; the tests prove the premise on the restatement's systems of
    both iterations)"""
    D = 11 if esikf else 6
    S = system0(sc, esikf)
    for span in (6.0, 7.0, 8.0):
        for seed in range(3000):
            v = 10.0 ** np.random.default_rng(seed).uniform(-1.0 - span, -1.0, D)
            sw, gap = pivot_replay(np.eye(D) + np.diag(v * weight) @ S)
            if column in sw and gap > 0.05:
                cov = VC.initial_covariance()
                o = 0 if esikf else 1
                cov[o:o + D, o:o + D] = np.diag(v)
                return cov
    raise AssertionError(f"no covariance forces a swap at column {column}")


# ---- chunk layouts -----------------------------------------------------------------------------------------------------
def skipped_at_chunk_edges(sc):
    """a photometric list of three chunks: skipped points (N_rgb < 3) at slots 0 and 127 of every chunk, a whole chunk of skipped
    points in the middle, and a short last chunk"""
    usable, fresh = np.flatnonzero(sc["n_rgb"] >= 3), np.flatnonzero(sc["n_rgb"] < 3)
    assert len(usable) >= 126 + 40 and len(fresh) >= 132, (len(usable), len(fresh))
    idx = np.r_[fresh[0], usable[:126], fresh[1], fresh[2:130], fresh[130], usable[126:166], fresh[131]]
    assert len(idx) == 2 * CHUNK + 42
    for base in (0, CHUNK, 2 * CHUNK):
        assert sc["n_rgb"][idx[base]] < 3 and sc["n_rgb"][idx[min(base + CHUNK, len(idx)) - 1]] < 3
    assert np.all(sc["n_rgb"][idx[CHUNK:2 * CHUNK]] < 3)
    return idx


def scattered_usable(sc, k):
    """k usable points, one per chunk at a different slot of each, the rest of k chunks filled with skipped points"""
    usable, fresh = np.flatnonzero(sc["n_rgb"] >= 3), np.flatnonzero(sc["n_rgb"] < 3)
    n = k * CHUNK
    assert len(usable) >= k and len(fresh) >= n - k, (len(usable), len(fresh))
    idx = fresh[:n].copy()
    for j in range(k):
        idx[j * CHUNK + (37 * j + 5) % CHUNK] = usable[j]
    assert (sc["n_rgb"][idx] >= 3).sum() == k
    assert all(((sc["n_rgb"][idx[j * CHUNK:(j + 1) * CHUNK]] >= 3).sum() == 1) for j in range(k))
    return idx


def interleaved(usable, fresh):
    """usable and skipped points spread evenly through one list"""
    order = np.argsort(np.r_[np.arange(len(usable)) / max(len(usable), 1), (np.arange(len(fresh)) + 0.5) / max(len(fresh), 1)],
                       kind="stable")
    return np.r_[usable, fresh][order]


TILE, TILES = 397, 51   # 20 247 points: 159 chunks, the last of 23 points; 397 is prime, so a read one chunk off lands elsewhere


def tiled():
    """the tiled list's positions in its tile"""
    idx = np.tile(np.arange(TILE), TILES)
    assert chunk_shape(len(idx), True)[:2] == (159, 23)
    return idx
