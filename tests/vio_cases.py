"""Seeded cases of the two camera updates (vioEsikf, vioPhotometric): a camera state with the r3live or ntu intrinsics scaled
as process's first image scales them, points in front of the camera whose matched points and colour states are perturbed so
that residuals fall on both sides of the Huber threshold, a strongly textured image, non-zero time_td and velocities.

make_case(...) returns a dict of FP64 / FP32 inputs; the colour state is the one a colour map stores (BGR shorts, float
sigmas, N_rgb).  Projections are kept 6 pixels inside the image, so the reference's getRgb taps (+-4 and +1) stay in it.
"""
import numpy as np

from sr_livo_b200 import lio

CAMERAS = {"r3live": lio.r3live_camera_params(), "ntu": lio.ntu_camera_params()}


def _quat(rng, angle):
    ax = rng.normal(size=3)
    ax /= np.linalg.norm(ax)
    return np.r_[ax * np.sin(angle / 2), np.cos(angle / 2)]


def textured_image(rows, cols, seed):
    """A BGR8 image of random blobs plus pixel noise: strong gradients everywhere, so a wrong tap moves a result far."""
    rng = np.random.default_rng(seed)
    small = rng.integers(0, 256, size=(rows // 8 + 2, cols // 8 + 2, 3)).astype(np.float64)
    big = np.kron(small, np.ones((8, 8, 1)))[:rows, :cols]
    img = np.clip(big + rng.normal(0, 25, size=big.shape), 0, 255).astype(np.uint8)
    return np.ascontiguousarray(img)


def make_state(rng, cam, scale=1.0, td=0.0, ric_angle=0.02, rotation=None, ric=None):
    """rotation (x, y, z, w) and ric (3 x 3), when given, replace the seeded ones (the seeded draws are made either way)"""
    K = np.array(cam["camera_intrinsic"], np.float64).reshape(3, 3)
    fx, fy, cx, cy = K[0, 0] / scale, K[1, 1] / scale, K[0, 2] / scale, K[1, 2] / scale
    rot = _quat(rng, 0.7)
    r_ic = lio._quat_to_rot(_quat(rng, ric_angle)) @ np.array([[0.0, 0.0, 1.0], [-1.0, 0.0, 0.0], [0.0, -1.0, 0.0]])
    rot = rot if rotation is None else np.asarray(rotation, np.float64)
    r_ic = r_ic if ric is None else np.asarray(ric, np.float64)
    s = lio.CameraState(rot, rng.normal(size=3), r_ic, rng.normal(scale=0.05, size=3), fx, fy, cx, cy, td)
    return s


def state_array(s):
    c = s.c
    return np.r_[c.rotation[:], c.translation[:], c.R_imu_camera[:], c.t_imu_camera[:], c.fx, c.fy, c.cx, c.cy, c.time_td,
                 c.q_world_camera[:], c.t_world_camera[:], c.q_camera_world[:], c.t_camera_world[:]].astype(np.float64)


def make_case(seed, camera="r3live", n=300, scale=1.0, td=0.002, outlier_px=3.0, colour_noise=6.0, n_low=0, n_new_visited=40,
              pix_noise=0.6, margin=6.0, zmin=3.0, zmax=25.0, colour_at_projection=False, rotation=None, ric=None):
    rng = np.random.default_rng(seed)
    cam = CAMERAS[camera]
    cols, rows = int(cam["image_width"] / scale), int(cam["image_height"] / scale)
    s = make_state(rng, cam, scale, td, rotation=rotation, ric=ric)
    st = state_array(s)
    Rcw = lio._quat_to_rot(st[31:35])
    tcw = st[35:38]
    fx, fy, cx, cy = st[19:23]
    # points: pixels inside the window, depths 3..25 m, back to the world
    u = rng.uniform(margin + 4, cols - margin - 4, n)
    v = rng.uniform(margin + 4, rows - margin - 4, n)
    z = rng.uniform(zmin, zmax, n)
    pc = np.stack([(u - cx) / fx * z, (v - cy) / fy * z, z], 1)
    pw = (pc - tcw) @ Rcw            # Rcwᵀ (pc - tcw)
    xyz = pw.astype(np.float32)
    vel = rng.normal(scale=20.0, size=(n, 2))
    noise = rng.normal(scale=pix_noise, size=(n, 2))
    out = rng.random(n) < 0.2
    noise[out] *= outlier_px / pix_noise
    uv = (np.stack([u, v], 1) + td * vel + noise).astype(np.float32)
    img = textured_image(rows, cols, seed + 1)
    # colour state: the image's colour at a slightly moved pixel, plus noise
    uu = np.clip(np.rint(u + rng.normal(scale=0.5, size=n)), 0, cols - 1).astype(int)
    vv = np.clip(np.rint(v + rng.normal(scale=0.5, size=n)), 0, rows - 1).astype(int)
    base = img[vv, uu].astype(np.float64)
    if colour_at_projection:   # the colour the update samples at the point's projection: small photometric residuals
        import vio_reference as VR
        pu, pv = u + td * vel[:, 0], v + td * vel[:, 1]
        base = np.array([VR.sub_pixel(img, pv[i], pu[i]) for i in range(n)], np.float64)
    rgb = np.clip(base + rng.normal(scale=colour_noise, size=(n, 3)), 0, 255).astype(np.int16)
    cov_rgb = rng.uniform(2.0, 12.0, size=(n, 3)).astype(np.float32)
    n_rgb = rng.integers(3, 40, size=n).astype(np.int16)
    if n_low:
        n_rgb[rng.choice(n, size=n_low, replace=False)] = rng.integers(0, 3, size=n_low)
    return dict(seed=seed, camera=camera, cols=cols, rows=rows, state=st, xyz=xyz, uv=uv, vel=vel, rgb=rgb, cov_rgb=cov_rgb,
                n_rgb=n_rgb, img=img, n_new_visited=n_new_visited)


def initial_covariance():
    c = np.eye(11) * 1e-4
    c[0, 0] = 1e-5
    for i in range(1, 11):
        c[i, i] = 1e-3
    return c


def ill_conditioned_covariance(seed, kappa=1e8):
    rng = np.random.default_rng(seed)
    q, _ = np.linalg.qr(rng.normal(size=(11, 11)))
    ev = np.logspace(-3, -3 - np.log10(kappa), 11)
    return (q * ev) @ q.T


def singular_covariance():
    """setInitialCov with the fx variance set to zero: the reference's (J P Jᵀ w).inverse() is not finite"""
    c = initial_covariance()
    c[7, 7] = 0.0
    return c


def suite():
    """(name, case, covariance) of the CPU pin tests"""
    cs = []
    for cam in ("r3live", "ntu"):
        for n in (9, 10, 30, 300):
            cs.append((f"{cam}-n{n}", make_case(100 + n, cam, n=n, scale=1.0 if cam == "ntu" else 2.0), initial_covariance()))
    cs.append(("r3live-n2000", make_case(7, "r3live", n=2000, scale=2.0), initial_covariance()))
    cs.append(("photometric-9-usable", make_case(11, "ntu", n=20, n_low=11), initial_covariance()))
    cs.append(("photometric-10-usable", make_case(12, "ntu", n=20, n_low=10), initial_covariance()))
    for nv in (0, -3, 1, 100000):
        cs.append((f"n_new_visited{nv}", make_case(20 + abs(nv) % 7, "ntu", n=60, n_new_visited=nv), initial_covariance()))
    cs.append(("td-zero", make_case(31, "ntu", n=60, td=0.0), initial_covariance()))
    cs.append(("photometric-break", make_case(32, "ntu", n=60, colour_noise=0.3, colour_at_projection=True), initial_covariance()))
    cs.append(("photometric-no-break", make_case(33, "ntu", n=60, colour_noise=30.0), initial_covariance()))
    cs.append(("ill-conditioned", make_case(34, "ntu", n=80), ill_conditioned_covariance(5)))
    cs.append(("small-steps", make_case(35, "ntu", n=60, pix_noise=0.01, outlier_px=0.02, td=0.0), initial_covariance()))
    return cs


# ---- decisions near their thresholds ----------------------------------------------------------------------------------
# Relative margin a case keeps from every threshold its discrete decisions compare with: far above the FP64 rounding of any
# of the compared forms (the device, the compiled reference, the restatement differ by < 1e-12 relative on this suite).
MARGIN = 1e-6


def fragile(truth, esikf, n):
    """The decisions of one restated update that lie within MARGIN of their thresholds: the Huber test (residual norm vs 1),
    so3ToQuat's small-angle branch (rotation step vs THETA_THRESHOLD), rotationToSo3's (d_x's rotation vs THETA_THRESHOLD),
    the photometric break (acc_residual / n vs 10), and the branches of Quaterniond(Matrix3d) (the trace vs 0, then the
    diagonal comparisons), two of which give q and -q for the same rotation."""
    out = []
    # photometric residuals are differences of integers (a sampled BGR value and the short state): the squared norm is an
    # integer every form computes exactly, so that Huber test cannot round differently
    for it, rn in enumerate(truth.get("residual_norms", []) if esikf else []):
        near = np.abs(rn[np.isfinite(rn)] - 1.0) < MARGIN
        if near.any():
            out.append(("huber", it, int(near.sum())))
    for it, st in enumerate(truth.get("steps", [])):
        if abs(st - 1e-4) < MARGIN * 1e-4:
            out.append(("theta", it, st))
    for it, st in enumerate(truth.get("dx_rot", [])):
        if abs(st - 1e-4) < MARGIN * 1e-4:
            out.append(("dtheta", it, st))
    if not esikf and truth["acc_history"]:
        r = float(truth["acc_history"][0]) / n
        if abs(r - 10.0) < MARGIN * 10.0:
            out.append(("break", 0, r))
    for k, (role, t, m00, m11, m22) in enumerate(truth.get("rot2q", [])):
        if abs(t) < MARGIN:
            out.append(("rot2q trace", k, role, t))
        elif t <= 0 and (abs(m22 - max(m00, m11)) < MARGIN or (m22 < max(m00, m11) and abs(m11 - m00) < MARGIN)):
            out.append(("rot2q diagonal", k, role, (m00, m11, m22)))   # the comparison that picks the largest entry
    return out


# ---- device scenes -----------------------------------------------------------------------------------------------------
def device_scene(lio, ctx, camera="ntu", seed=501, n_usable=400, n_fresh=0, photometric_seed=950, rotation=None, ric=None):
    """A colour map filled and coloured on the device as process fills it: n_usable points (depths 3-12 m) added and rendered
    three times (N_rgb = 3), then n_fresh points (depths 14-25 m, so in other voxels) added and rendered once (N_rgb = 1).
    Returns the handles, the state, and per selected point its id, gathered colour state, matched uv and velocity; img is the
    image the photometric update samples (half the rendered scene, half an unrelated texture).  rotation (the IMU's, x, y, z,
    w) and ric (R_imu_camera), when given, replace the seeded ones."""
    cam = CAMERAS[camera]
    c = make_case(seed, camera, n=n_usable, zmin=3.0, zmax=12.0, rotation=rotation, ric=ric)
    ip = lio.ImageProcessing(ctx, **cam)
    cols, rows = ip.output_size()
    cm = lio.ColorVoxelMap(ctx, 1.0, 20, 1 << 15, 0.05)
    st = lio.CameraState(c["state"][0:4], c["state"][4:7], c["state"][7:16].reshape(3, 3), c["state"][16:19], *c["state"][19:24])
    cam_c = st.camera(cols, rows, 0.005)
    base = c["img"][:rows, :cols]
    cm.addPoints(c["xyz"].astype(np.float64), time_sweep_end=1.0)
    for k in range(3):
        cm.renderPointsInRecentVoxel(cam_c, np.ascontiguousarray(textured_image(rows, cols, 900 + k) // 2 + base // 2), 1.0 + k)
    if n_fresh:
        # the same camera state, so the fresh points are projected from the same pose
        rng = np.random.default_rng(seed + 2)
        Rcw, tcw = lio._quat_to_rot(c["state"][31:35]), c["state"][35:38]
        fx, fy, cx, cy = c["state"][19:23]
        u = rng.uniform(12, cols - 12, n_fresh); v = rng.uniform(12, rows - 12, n_fresh); z = rng.uniform(14.0, 25.0, n_fresh)
        pc = np.stack([(u - cx) / fx * z, (v - cy) / fy * z, z], 1)
        cm.addPoints((pc - tcw) @ Rcw, time_sweep_end=5.0, time_last_process=4.0)
        cm.renderPointsInRecentVoxel(cam_c, np.ascontiguousarray(textured_image(rows, cols, 903) // 2 + base // 2), 5.0)
    ids, xyz, uv = cm.selectPointsForProjection(cam_c, minimum_dis=2.0, use_all_points=True)
    g = cm.gatherPoints(ids)
    rng = np.random.default_rng(seed + 3)
    n = len(ids)
    vel = rng.normal(scale=20.0, size=(n, 2))
    uvm = (uv.astype(np.float64) + 0.002 * vel + rng.normal(scale=0.7, size=(n, 2))).astype(np.float32)
    img = np.ascontiguousarray(textured_image(rows, cols, photometric_seed) // 2 + base // 2)
    return dict(ip=ip, cm=cm, state=state_array(st), ids=np.ascontiguousarray(ids, np.uint32), xyz=g["xyz"], rgb=g["rgb"],
                cov_rgb=g["cov"], n_rgb=g["n_rgb"], uv=uvm, vel=vel, img=img, cols=cols, rows=rows, camera=camera)


def subset(sc, idx):
    """the scene restricted to the selected points idx (in that order)"""
    out = dict(sc)
    for k in ("ids", "xyz", "rgb", "cov_rgb", "n_rgb", "uv", "vel"):
        out[k] = np.ascontiguousarray(sc[k][idx])
    return out


def image_digest(img) -> bytes:
    """SHA-256 of an image's bytes: the golden file records the images it was made with by digest, not by value"""
    import hashlib
    return hashlib.sha256(np.ascontiguousarray(img).tobytes()).digest()
