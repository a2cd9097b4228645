"""The two camera updates on the device (srl_image_vio_esikf / srl_image_vio_photometric, row N8) against the 50-digit
restatement (tests/vio_reference.py), the reference's own compiled vioEsikf / vioPhotometric where oracle/_ref was built, and
its outputs recorded in tests/golden/vio_updates.npz where it was not.

Scenes are made on the device as process makes them (tests/vio_cases.py: device_scene): the colour map is filled by addPoints
and coloured by the renderer (three renderings give N_rgb = 3, one gives N_rgb = 1), the tracked ids come from
selectPointsForProjection, and the colour state the updates read is gathered back by id for the restatement and the
reference.  Which points are passed, the image and the covariance steer each decision of the updates."""
import os

import numpy as np
import pytest

import vio_cases as VC
import vio_ref as RF
import vio_reference as VR

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vio_updates.npz")
# |device - truth| <= max(TOL, κ(Pw)·ε) * (1 + |truth|) componentwise for the state and max(TOL_COV, κ(Pw)·ε) * max|cov| for
# the covariance.  On the well-conditioned scenes the device lies within 1e-14 of the truth (the reference within 2e-15
# and 2e-14); κ(Pw)·ε is the first-order effect of the prior covariance's conditioning on any FP64 solve.
TOL, TOL_COV = 1e-11, 1e-10
EPS = 2.0 ** -52


def _bounds(cov, esikf):
    k = np.linalg.cond(cov if esikf else cov[1:7, 1:7]) * EPS
    return max(TOL, k), max(TOL_COV, k)


@pytest.fixture(scope="module")
def env():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from sr_livo_b200 import lio
    ctx = lio.Context(0)
    scenes = {}
    yield dict(lio=lio, ctx=ctx, torch=torch, scenes=scenes)
    for sc in scenes.values():
        sc["cm"].close(); sc["ip"].close()
    ctx.close()


def _scene(env, name):
    if name not in env["scenes"]:
        kw = dict(base_ntu=dict(camera="ntu"), base_r3live=dict(camera="r3live", seed=502),
                  mixed=dict(camera="ntu", seed=503, n_usable=200, n_fresh=300))[name]
        env["scenes"][name] = VC.device_scene(env["lio"], env["ctx"], **kw)
    return env["scenes"][name]


def _state(s, lio):
    st = lio.CameraState(s[0:4], s[4:7], s[7:16].reshape(3, 3), s[16:19], *s[19:24])
    st.c.q_world_camera[:] = s[24:28].tolist(); st.c.t_world_camera[:] = s[28:31].tolist()
    st.c.q_camera_world[:] = s[31:35].tolist(); st.c.t_camera_world[:] = s[35:38].tolist()
    return st


def _run(env, sc, esikf, state, cov, ids=None, uv=None, vel=None, img=None, n_new=40):
    sc["ip"].setCovariance(cov)
    st = _state(state, env["lio"])
    ids = sc["ids"] if ids is None else ids
    vel = sc["vel"] if vel is None else vel
    if esikf:
        r = sc["ip"].vioEsikf(sc["cm"], st, ids, sc["uv"] if uv is None else uv, vel, n_new)
    else:
        r = sc["ip"].vioPhotometric(sc["cm"], st, ids, vel, n_new, sc["img"] if img is None else img)
    return VC.state_array(st), sc["ip"].covariance(), r


def _truth(sc, esikf, state, cov, n_new=40):
    return VR.vio_update(esikf, state, cov, sc["xyz"], sc["uv"], sc["vel"], sc["rgb"], sc["cov_rgb"], sc["n_rgb"], n_new, sc["img"])


def _check(env, sc, esikf, state, cov, n_new=40, moved=True):
    """the device's update against the truth (decisions equal, results within the bounds) and against the reference"""
    s, c, r = _run(env, sc, esikf, state, cov, n_new=n_new)
    t = _truth(sc, esikf, state, cov, n_new)
    assert not VC.fragile(t, esikf, len(sc["ids"])), "a decision of this scene is too close to its threshold to pin"
    assert int(r) == t["result"]
    it, used, _ = sc["ip"].vio_last_summary(0 if esikf else 1)
    assert (it, used) == (t["iterations"], t["used"])
    if moved:
        assert np.abs(t["state"] - state).max() > 1e-6, "the update moved nothing: the case tests nothing"
    tol, tol_cov = _bounds(cov, esikf)
    assert np.all(np.abs(s - t["state"]) <= tol * (1 + np.abs(t["state"]))), np.abs(s - t["state"]).max()
    assert np.abs(c - t["cov"]).max() <= tol_cov * np.abs(t["cov"]).max(), np.abs(c - t["cov"]).max()
    if RF.available():
        rs, rc, rr, _ = RF.update(0 if esikf else 1, state, cov, sc["xyz"], sc["uv"], sc["vel"], sc["rgb"], sc["cov_rgb"], sc["n_rgb"],
                                  n_new, sc["img"])
        assert rr[0 if esikf else 1] == int(r)
        if np.all(np.isfinite(rs)):
            assert np.all(np.abs(rs - t["state"]) <= tol * (1 + np.abs(t["state"])))
    return s, c, r, t


@pytest.mark.parametrize("name", ["base_ntu", "base_r3live"])
@pytest.mark.parametrize("esikf", [True, False], ids=["esikf", "photometric"])
def test_device_update_against_the_truth_and_the_reference(env, name, esikf):
    sc = _scene(env, name)
    _check(env, sc, esikf, sc["state"], VC.initial_covariance())


@pytest.mark.parametrize("esikf", [True, False], ids=["esikf", "photometric"])
def test_device_update_against_the_golden_reference_outputs(env, esikf):
    """the reference's outcomes recorded by tests/golden/make_vio_golden.py on the same device scenes"""
    g = np.load(GOLDEN)
    for name in ("base_ntu", "base_r3live", "mixed"):
        sc = _scene(env, name)
        for k in ("ids", "xyz", "rgb", "cov_rgb", "n_rgb", "uv", "vel", "state"):
            assert np.array_equal(sc[k], g[f"{name}.{k}"]), (name, k)
        assert np.array_equal(np.frombuffer(VC.image_digest(sc["img"]), np.uint8), g[f"{name}.img_digest"])
        w = "esikf" if esikf else "photometric"
        cov = VC.initial_covariance()
        s, c, r = _run(env, sc, esikf, sc["state"], cov)
        assert int(r) == int(g[f"{name}.{w}.result"])
        assert np.all(np.abs(s - g[f"{name}.{w}.state"]) <= 2 * TOL * (1 + np.abs(g[f"{name}.{w}.state"])))
        assert np.abs(c - g[f"{name}.{w}.cov"]).max() <= 2 * TOL_COV * np.abs(g[f"{name}.{w}.cov"]).max()


@pytest.mark.parametrize("n_new", [0, -5, 1, 100000])
@pytest.mark.parametrize("esikf", [True, False], ids=["esikf", "photometric"])
def test_measurement_weight_edges(env, n_new, esikf):
    """5.0 / 0 = inf gives 0.01, a negative count 0.001, 1 gives 0.01, a large count 0.001"""
    sc = _scene(env, "base_ntu")
    _check(env, sc, esikf, sc["state"], VC.initial_covariance(), n_new=n_new)


def test_photometric_with_nine_usable_points_returns_true_and_changes_nothing(env):
    sc = _scene(env, "mixed")
    usable = np.flatnonzero(sc["n_rgb"] >= 3)
    fresh = np.flatnonzero(sc["n_rgb"] < 3)
    assert len(usable) >= 9 and len(fresh) >= 20
    sub = VC.subset(sc, np.r_[usable[:9], fresh[:20]])
    cov = VC.initial_covariance()
    s, c, r = _run(env, sub, False, sub["state"], cov)
    assert r is True and np.array_equal(s, sub["state"]) and np.array_equal(c, cov)
    assert sub["ip"].vio_last_summary(1)[:2] == (0, 9)
    _check(env, sub, False, sub["state"], cov, moved=False)
    # ten usable points: it iterates
    sub10 = VC.subset(sc, np.r_[usable[:10], fresh[:20]])
    _check(env, sub10, False, sub10["state"], cov)


def test_photometric_break_counts_the_skipped_points(env):
    """acc_residual / n < 10 with n counting the N_rgb < 3 points: choose how many of them to pass so that acc / n < 10 while
    acc / (points used) > 10; the break must be taken (one iteration), and without the skipped points it must not."""
    sc = _scene(env, "mixed")
    usable = np.flatnonzero(sc["n_rgb"] >= 3)[:60]
    fresh = np.flatnonzero(sc["n_rgb"] < 3)
    cov = VC.initial_covariance()
    only = VC.subset(sc, usable)
    t0 = _truth(only, False, only["state"], cov)
    acc0 = float(t0["acc_history"][0])
    assert acc0 / len(usable) > 10.5 and t0["iterations"] == 2, acc0 / len(usable)
    m = int(np.ceil(acc0 / 9.0)) - len(usable)          # acc0 / (used + m) <= 9
    assert 0 < m <= len(fresh)
    mix = VC.subset(sc, np.r_[usable, fresh[:m]])
    _, _, _, t = _check(env, mix, False, mix["state"], cov)
    assert t["iterations"] == 1 and mix["ip"].vio_last_summary(1)[0] == 1
    _check(env, only, False, only["state"], cov)


def test_ill_conditioned_covariance_carried_over_frames(env):
    sc = _scene(env, "base_ntu")
    cov = VC.ill_conditioned_covariance(5)
    sc["ip"].setCovariance(cov)
    s, ts, tc = sc["state"], sc["state"], cov
    for frame in range(3):
        for esikf in (True, False):
            st = _state(s, env["lio"])
            if esikf:
                sc["ip"].vioEsikf(sc["cm"], st, sc["ids"], sc["uv"], sc["vel"], 40)
            else:
                sc["ip"].vioPhotometric(sc["cm"], st, sc["ids"], sc["vel"], 40, sc["img"])
            s = VC.state_array(st)
            t = _truth(sc, esikf, ts, tc)
            ts, tc = t["state"], t["cov"]
    tol, tol_cov = _bounds(cov, True)
    dc = sc["ip"].covariance()
    assert np.abs(dc - tc).max() <= 10 * tol_cov * np.abs(tc).max(), np.abs(dc - tc).max() / np.abs(tc).max()
    assert np.all(np.abs(s - ts) <= 10 * tol * (1 + np.abs(ts))), np.abs(s - ts).max()


def test_covariance_persists_across_frames(env):
    sc = _scene(env, "base_r3live")
    cov = VC.initial_covariance()
    sc["ip"].setCovariance(cov)
    s, ts, tc = sc["state"], sc["state"], cov
    for frame in range(3):
        for esikf in (True, False):
            st = _state(s, env["lio"])
            if esikf:
                sc["ip"].vioEsikf(sc["cm"], st, sc["ids"], sc["uv"], sc["vel"], 40)
            else:
                sc["ip"].vioPhotometric(sc["cm"], st, sc["ids"], sc["vel"], 40, sc["img"])
            s = VC.state_array(st)
            t = _truth(sc, esikf, ts, tc)
            ts, tc = t["state"], t["cov"]
    assert np.abs(sc["ip"].covariance() - tc).max() <= TOL_COV * np.abs(tc).max()
    assert np.all(np.abs(s - ts) <= 1e-9 * (1 + np.abs(ts)))


def test_singular_covariance_gives_the_finite_limit(env):
    """a zero fx variance: the reference's (J P Jᵀ w).inverse() is not finite (test_vio_pin.py); the device returns the finite
    Woodbury update, the restatement's, with the zero row and column of the posterior kept exactly zero"""
    sc = _scene(env, "base_ntu")
    cov = VC.singular_covariance()
    s, c, r = _run(env, sc, True, sc["state"], cov)
    t = _truth(sc, True, sc["state"], cov)
    assert r is True and np.all(np.isfinite(s)) and np.all(np.isfinite(c))
    assert np.all(c[7] == 0.0) and np.all(c[:, 7] == 0.0)
    assert np.all(np.abs(s - t["state"]) <= TOL * (1 + np.abs(t["state"])))
    assert np.abs(c - t["cov"]).max() <= TOL_COV * np.abs(t["cov"]).max()


def test_projections_at_the_image_edge_are_clamped(env):
    """velocities that move some projections to within 4 pixels of each border, onto it and past it: the taps are clamped to
    the nearest row and column (the reference would read outside the image there), checked against the restatement only"""
    sc = _scene(env, "base_ntu")
    vel = sc["vel"].copy()
    td = sc["state"][23]
    fx, fy, cx, cy = sc["state"][19:23]
    proj = VR.vio_update(False, sc["state"], VC.initial_covariance(), sc["xyz"], sc["uv"], np.zeros_like(vel), sc["rgb"],
                         sc["cov_rgb"], sc["n_rgb"], 40, sc["img"])["projections"][0]
    targets = [(1.5, None), (-2.25, None), (sc["cols"] - 1.0, None), (sc["cols"] + 3.5, None), (None, 0.5), (None, sc["rows"] - 2.5),
               (None, sc["rows"] + 1.0), (2.0, 3.0)]
    for k, (tu, tv) in enumerate(targets):
        if tu is not None:
            vel[k, 0] = (tu - proj[k, 0]) / td
        if tv is not None:
            vel[k, 1] = (tv - proj[k, 1]) / td
    edge = dict(sc, vel=vel)
    cov = VC.initial_covariance()
    s, c, r = _run(env, edge, False, edge["state"], cov)
    t = _truth(edge, False, edge["state"], cov)
    p0 = t["projections"][0]
    assert (p0[:len(targets), 0].min() < 0 and p0[:len(targets), 0].max() > sc["cols"] and p0[:len(targets), 1].max() > sc["rows"])
    assert int(r) == t["result"] and edge["ip"].vio_last_summary(1)[:2] == (t["iterations"], t["used"])
    assert np.all(np.abs(s - t["state"]) <= TOL * (1 + np.abs(t["state"])))
    assert np.abs(c - t["cov"]).max() <= TOL_COV * np.abs(t["cov"]).max()


def test_host_and_device_inputs_and_repeats_give_identical_bits(env):
    torch = env["torch"]
    sc = _scene(env, "base_ntu")
    cov = VC.initial_covariance()
    for esikf in (True, False):
        a = _run(env, sc, esikf, sc["state"], cov)
        b = _run(env, sc, esikf, sc["state"], cov)
        d_ids = torch.from_numpy(sc["ids"].view(np.int32)).cuda()
        d_uv = torch.from_numpy(sc["uv"]).cuda()
        d_vel = torch.from_numpy(sc["vel"]).cuda()
        # a padded device image: 64 bytes of pitch beyond the pixels
        pad = torch.zeros((sc["rows"], sc["cols"] * 3 + 64), dtype=torch.uint8, device="cuda")
        pad[:, :sc["cols"] * 3] = torch.from_numpy(sc["img"].reshape(sc["rows"], -1)).cuda()
        d_img = pad[:, :sc["cols"] * 3].view(sc["rows"], sc["cols"], 3)
        c = _run(env, sc, esikf, sc["state"], cov, ids=d_ids, uv=d_uv, vel=d_vel, img=d_img)
        for x, y in ((a, b), (a, c)):
            assert np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) and x[2] == y[2]


def test_chained_frame_without_host_copies(env):
    """process -> selectPointsForProjection -> trackImage -> vioEsikf -> vioPhotometric -> renderPointsInRecentVoxel, every
    image, point list and velocity in device memory; the same calls on host copies of the same inputs give the same bits"""
    torch, lio = env["torch"], env["lio"]
    cam = VC.CAMERAS["ntu"]
    c = VC.make_case(601, "ntu", n=500, zmin=3.0, zmax=12.0)
    ip = lio.ImageProcessing(env["ctx"], **cam)
    cols, rows = ip.output_size()
    cm = lio.ColorVoxelMap(env["ctx"], 1.0, 20, 1 << 15, 0.05)
    lk = lio.LKOpticalFlowKernel(env["ctx"], **lio.tracker_lk_params())
    try:
        st0 = lio.CameraState(c["state"][0:4], c["state"][4:7], c["state"][7:16].reshape(3, 3), c["state"][16:19], *c["state"][19:24])
        raw1 = torch.from_numpy(VC.textured_image(cam["image_height"], cam["image_width"], 610)).cuda()
        raw2 = torch.roll(raw1, shifts=(1, 2), dims=(0, 1)).contiguous()
        rgb1 = torch.empty((rows, cols, 3), dtype=torch.uint8, device="cuda"); gray1 = torch.empty((rows, cols), dtype=torch.uint8, device="cuda")
        rgb2 = torch.empty_like(rgb1); gray2 = torch.empty_like(gray1)
        ip.process(raw1, out=(rgb1, gray1))
        cm.addPoints(torch.from_numpy(c["xyz"].astype(np.float64)).cuda(), time_sweep_end=1.0)
        camera = st0.camera(cols, rows, 0.005)
        for k in range(3):
            cm.renderPointsInRecentVoxel(camera, rgb1, 1.0 + k)
        n = cm.countPointsForProjection(camera, minimum_dis=10.0)
        ids = torch.empty(n, dtype=torch.int32, device="cuda")
        uv = torch.empty((n, 2), dtype=torch.float32, device="cuda")
        cm.selectPointsForProjection(camera, minimum_dis=10.0, out=(ids, None, uv))
        lk.trackImage(gray1, uv)                                   # first image: the pyramid only
        ip.process(raw2, out=(rgb2, gray2))
        curr, status, _ = lk.trackImage(gray2, uv)
        vel = ((curr - uv).double() / 0.1).contiguous()              # image_velocity as the tracker forms it, on the device
        st = _state(VC.state_array(st0), lio)
        ip.setCovariance(VC.initial_covariance())
        r1 = ip.vioEsikf(cm, st, ids, curr, vel, 40)
        r2 = ip.vioPhotometric(cm, st, ids, vel, 40, rgb2)
        dev_state, dev_cov = VC.state_array(st), ip.covariance()
        assert r1 and r2 and n >= 10
        assert np.abs(dev_state - VC.state_array(st0)).max() > 1e-9
        # the same two updates from host copies (before the render, which changes the colour state they read)
        h = dict(ids=ids.cpu().numpy().view(np.uint32), uv=curr.cpu().numpy(), vel=vel.cpu().numpy(), img=rgb2.cpu().numpy())
        st_h = _state(VC.state_array(st0), lio)
        ip.setCovariance(VC.initial_covariance())
        ip.vioEsikf(cm, st_h, h["ids"], h["uv"], h["vel"], 40)
        ip.vioPhotometric(cm, st_h, h["ids"], h["vel"], 40, h["img"])
        assert np.array_equal(VC.state_array(st_h), dev_state) and np.array_equal(ip.covariance(), dev_cov)
        assert cm.renderPointsInRecentVoxel(st.camera(cols, rows, 0.005), rgb2, 5.0) > 0   # process:155 with the updated camera
    finally:
        cm.close(); ip.close(); lk.close()


def test_fewer_than_ten_points_change_nothing(env):
    sc = _scene(env, "base_ntu")
    cov = VC.initial_covariance()
    for esikf in (True, False):
        s, c, r = _run(env, sc, esikf, sc["state"], cov, ids=sc["ids"][:9], uv=sc["uv"][:9], vel=sc["vel"][:9])
        assert r is False and np.array_equal(s, sc["state"]) and np.array_equal(c, cov)


def test_bad_id_and_singular_pivot_write_nothing(env):
    lio = env["lio"]
    sc = _scene(env, "base_ntu")
    cov = VC.initial_covariance()
    ids = sc["ids"].copy()
    ids[5] = 0xfffffff0
    for esikf in (True, False):
        with pytest.raises(lio.SrlError) as e:
            _run(env, sc, esikf, sc["state"], cov, ids=ids)
        assert e.value.code == 4   # SRL_BAD_ARG
        assert np.array_equal(sc["ip"].covariance(), cov)
    bad = cov.copy()
    bad[3, 3] = np.nan
    for esikf in (True, False):
        st = _state(sc["state"], lio)
        sc["ip"].setCovariance(bad)
        with pytest.raises(lio.SrlError) as e:
            if esikf:
                sc["ip"].vioEsikf(sc["cm"], st, sc["ids"], sc["uv"], sc["vel"], 40)
            else:
                sc["ip"].vioPhotometric(sc["cm"], st, sc["ids"], sc["vel"], 40, sc["img"])
        assert e.value.code == 6   # SRL_SINGULAR
        assert np.array_equal(VC.state_array(st), sc["state"])
        assert np.array_equal(sc["ip"].covariance(), bad, equal_nan=True)
    with pytest.raises(lio.SrlError):
        sc["ip"].vioPhotometric(sc["cm"], _state(sc["state"], lio), sc["ids"], sc["vel"], 40, sc["img"][:-1])
