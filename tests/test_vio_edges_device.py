"""The two camera updates on the device (k_vio_update) at their edges (tests/vio_edge_cases.py) against the 50-digit
restatement (tests/vio_reference.py), the compiled reference where oracle/_ref was built, and tests/golden/vio_edges.npz:
chunk boundaries and short last chunks, skipped points at chunk edges and in whole chunks, the photometric decisions spread
over chunks, 20 247 and 2 000 points, row swaps at early, middle and last columns, steps below THETA_THRESHOLD (and exactly 0),
non-finite and gross measurements, and every branch of Quaterniond(Matrix3d) for R_imu_camera and R_world R_imu_camera.

Bounds are test_vio_device's: max(TOL, κ(Pw)·ε) for the state and the covariance, equal decisions and (iterations, used)."""
import os

import numpy as np
import pytest

import vio_cases as VC
import vio_edge_cases as EC
import vio_ref as RF
import vio_reference as VR
from test_vio_device import TOL, TOL_COV, _bounds, _run, _state

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vio_edges.npz")
SCENES = {"base": dict(camera="ntu"), "many_fresh": dict(camera="ntu", seed=504, n_usable=200, n_fresh=1500),
          "big": dict(camera="ntu", seed=505, n_usable=2300), "ric_identity": dict(camera="ntu", seed=506, ric=np.eye(3))}
for _a, _b in EC.BRANCH_PAIRS:
    _q, _r = EC.branch_pose(_a, _b)
    SCENES[f"branch_{_a}_{_b}"] = dict(camera="ntu", seed=507, rotation=_q, ric=_r)


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
        env["scenes"][name] = VC.device_scene(env["lio"], env["ctx"], **SCENES[name])
    return env["scenes"][name]


def _truth(sc, esikf, state, cov, mult=None):
    return VR.vio_update(esikf, state, cov, sc["xyz"], sc["uv"], sc["vel"], sc["rgb"], sc["cov_rgb"], sc["n_rgb"], 40, sc["img"],
                         mult=mult)


def _check(env, sc, esikf, cov=None, state=None, truth=None, moved=True, reference=True):
    """the device against the truth: equal result, (iterations, used), no fragile decision, state and covariance within bounds;
    and the compiled reference within the same bounds of the truth where it is built and defined"""
    cov = VC.initial_covariance() if cov is None else cov
    state = sc["state"] if state is None else state
    t = _truth(sc, esikf, state, cov) if truth is None else truth
    n = len(sc["ids"])
    s, c, r = _run(env, sc, esikf, state, cov)
    assert not VC.fragile(t, esikf, n), VC.fragile(t, esikf, n)
    assert int(r) == t["result"]
    assert sc["ip"].vio_last_summary(0 if esikf else 1)[:2] == (t["iterations"], t["used"])
    if moved:
        assert np.abs(t["state"] - state).max() > 1e-6, "the update moved nothing: the case tests nothing"
    tol, tol_cov = _bounds(cov, esikf)
    assert np.all(np.isfinite(s)) and np.all(np.isfinite(c))
    assert np.all(np.abs(s - t["state"]) <= tol * (1 + np.abs(t["state"]))), np.abs(s - t["state"]).max()
    assert np.abs(c - t["cov"]).max() <= tol_cov * np.abs(t["cov"]).max(), np.abs(c - t["cov"]).max()
    if reference and RF.available():
        rs, _, rr, _ = RF.update(0 if esikf else 1, state, cov, sc["xyz"], sc["uv"], sc["vel"], sc["rgb"], sc["cov_rgb"], sc["n_rgb"],
                                 40, sc["img"])
        assert rr[0 if esikf else 1] == int(r)
        assert np.all(np.abs(rs - t["state"]) <= tol * (1 + np.abs(t["state"])))
    return s, c, t


# ---- chunks --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", EC.CHUNK_NS)
@pytest.mark.parametrize("esikf", [True, False], ids=["esikf", "photometric"])
def test_chunk_boundaries(env, n, esikf):
    """the first n points of one scene: n = 128k and 128k + 1, short last chunks; at n = 129 the last chunk is one point, 2 or 3
    rows against 3 or 8 segments"""
    if n == 129:
        assert EC.chunk_shape(n, esikf)[1:] == ((1, 2, 3, 2) if esikf else (1, 3, 8, 3))
    sc = _scene(env, "base")
    assert len(sc["ids"]) >= max(EC.CHUNK_NS)
    _check(env, VC.subset(sc, np.arange(n)), esikf)


def test_skipped_points_at_chunk_edges_and_a_whole_skipped_chunk(env):
    sc = _scene(env, "many_fresh")
    sub = VC.subset(sc, EC.skipped_at_chunk_edges(sc))
    _, _, t = _check(env, sub, False)
    assert t["used"] == 166


def test_nine_and_ten_usable_points_one_per_chunk(env):
    """nine usable points, one in each of 9 chunks of otherwise skipped points: true, nothing changes, 9 used; ten: it iterates"""
    sc = _scene(env, "many_fresh")
    sub = VC.subset(sc, EC.scattered_usable(sc, 9))
    cov = VC.initial_covariance()
    s, c, r = _run(env, sub, False, sub["state"], cov)
    assert r is True and np.array_equal(s, sub["state"]) and np.array_equal(c, cov)
    assert sub["ip"].vio_last_summary(1)[:2] == (0, 9)
    sub10 = VC.subset(sc, EC.scattered_usable(sc, 10))
    _, _, t = _check(env, sub10, False)
    assert t["iterations"] >= 1 and t["used"] == 10


def test_photometric_break_on_both_sides_over_several_chunks(env):
    """acc_residual / n against 10 with n counting skipped points interleaved through several chunks: m skipped points that
    bring the ratio to <= 9 (break after one iteration) and m' that keep it >= 11 (two iterations)"""
    sc = _scene(env, "many_fresh")
    usable, fresh = np.flatnonzero(sc["n_rgb"] >= 3), np.flatnonzero(sc["n_rgb"] < 3)
    cov = VC.initial_covariance()
    acc0 = float(_truth(VC.subset(sc, usable), False, sc["state"], cov)["acc_history"][0])
    m_break, m_keep = int(np.ceil(acc0 / 9.0)) - len(usable), int(np.floor(acc0 / 11.0)) - len(usable)
    assert 0 <= m_keep < m_break <= len(fresh), (acc0 / len(usable), m_keep, m_break)
    for m, its in ((m_break, 1), (m_keep, 2)):
        idx = EC.interleaved(usable, fresh[:m])
        assert len(idx) > EC.CHUNK
        _, _, t = _check(env, VC.subset(sc, idx), False)
        assert t["iterations"] == its, (m, t["iterations"], float(t["acc_history"][0]) / len(idx))


# ---- size ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("esikf", [True, False], ids=["esikf", "photometric"])
def test_twenty_thousand_points_as_a_tiled_list(env, esikf):
    """397 distinct points repeated 51 times (159 chunks, a 23-point last chunk) against the restatement with mult = 51; vioEsikf
    against the compiled reference on the whole list too (the reference's photometric update would need two dense 60 741 x 60 741
    matrices)"""
    sc = _scene(env, "base")
    tile = VC.subset(sc, np.arange(EC.TILE))
    big = VC.subset(tile, EC.tiled())
    cov = VC.initial_covariance()
    t = _truth(tile, esikf, sc["state"], cov, mult=[EC.TILES] * EC.TILE)
    assert t["used"] == (EC.TILE * EC.TILES if esikf else int((tile["n_rgb"] >= 3).sum()) * EC.TILES)
    s, c, r = _run(env, big, esikf, sc["state"], cov)
    assert not VC.fragile(t, esikf, len(big["ids"]))
    assert int(r) == t["result"] and big["ip"].vio_last_summary(0 if esikf else 1)[:2] == (t["iterations"], t["used"])
    tol, tol_cov = _bounds(cov, esikf)
    assert np.all(np.abs(s - t["state"]) <= tol * (1 + np.abs(t["state"]))), np.abs(s - t["state"]).max()
    assert np.abs(c - t["cov"]).max() <= tol_cov * np.abs(t["cov"]).max(), np.abs(c - t["cov"]).max()
    if esikf:
        g = np.load(GOLDEN)
        assert np.all(np.abs(s - g["tiled.esikf.state"]) <= 2 * tol * (1 + np.abs(t["state"])))
        if RF.available():
            rs, rc, rr, _ = RF.update(0, sc["state"], cov, big["xyz"], big["uv"], big["vel"], big["rgb"], big["cov_rgb"], big["n_rgb"], 40)
            assert rr[0] == 1 and np.all(np.abs(rs - t["state"]) <= tol * (1 + np.abs(t["state"])))


@pytest.mark.parametrize("esikf", [True, False], ids=["esikf", "photometric"])
def test_two_thousand_distinct_points(env, esikf):
    sc = _scene(env, "big")
    assert len(sc["ids"]) >= 2000
    _check(env, VC.subset(sc, np.arange(2000)), esikf, reference=esikf)


# ---- pivoting ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", [0, 1, 2], ids=["early", "middle", "last"])
@pytest.mark.parametrize("esikf", [True, False], ids=["esikf", "photometric"])
def test_row_swaps_at_early_middle_and_last_columns(env, which, esikf):
    """a diagonal covariance over six decades that makes the elimination of I + Pw S swap rows at the target column in both
    iterations; the premise replays the device's pivot rule on the restatement's systems, each winner clear of its runner-up"""
    sc = _scene(env, "base")
    col = EC.PIVOT_TARGETS[esikf][which]
    cov = EC.pivot_covariance(sc, esikf, col)
    t = _truth(sc, esikf, sc["state"], cov)
    assert len(t["systems"]) == 2
    for sy in t["systems"]:
        swaps, gap = EC.pivot_replay(sy["M"])
        assert col in swaps and gap > VC.MARGIN, (swaps, gap)
    s, c, _ = _check(env, sc, esikf, cov=cov, truth=t)
    g = np.load(GOLDEN)
    key = f"pivot.{'esikf' if esikf else 'photometric'}.{col}"
    assert np.array_equal(cov, g[key + ".cov"])
    tol, _ = _bounds(cov, esikf)
    assert np.all(np.abs(s - g[key + ".state"]) <= 2 * tol * (1 + np.abs(g[key + ".state"])))


# ---- small steps ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["small-steps", "small-steps-td0", "small-steps-vel0"])
def test_small_steps(env, variant):
    """matched points 1e-3 px from the projections: the rotation step is below THETA_THRESHOLD in iteration 0 and d_x's rotation
    below it in iteration 1 (so3ToQuat's and rotationToSo3's small-angle branches)"""
    sc = _scene(env, "base")
    name, st, uv, vel = [v for v in EC.small_step_variants(sc) if v[0] == variant][0]
    edge = dict(sc, uv=uv, vel=vel)
    t = _truth(edge, True, st, VC.initial_covariance())
    assert t["steps"][0] < 1e-4 and t["dx_rot"][1] < 1e-4, (t["steps"], t["dx_rot"])
    _check(env, edge, True, state=st, truth=t)


# Bound on R_imu_camera and the two camera quaternions after one step below THETA_THRESHOLD: the step itself is off by about
# κ(I + Pw S)·ε·|step| < 1e-16, and rot2q, qmul, qunit and qrot round about fifteen times at 1.1e-16 each on entries of
# magnitude <= 1, below 2e-15; the bound leaves a factor 5.  so3ToQuat's large-angle
# form differs from the small-angle one by θ³/24 in the quaternion (about twice that in the matrix), 3e-14 at θ = 9e-5.
TOL_ROT = 1e-14


def test_step_just_below_theta_takes_the_small_angle_branch(env):
    """a photometric update that breaks after iteration 0 (skipped points bring acc_residual / n below 10), so that its state is
    that one step's, which no second iteration re-solves; the covariance is scaled so that the rotation step lies just below
    THETA_THRESHOLD (the step grows monotonically with the scale), where the two forms of so3ToQuat differ by θ³/24"""
    sc = _scene(env, "many_fresh")
    usable, fresh = np.flatnonzero(sc["n_rgb"] >= 3), np.flatnonzero(sc["n_rgb"] < 3)
    acc0 = float(_truth(VC.subset(sc, usable), False, sc["state"], VC.initial_covariance())["acc_history"][0])
    m = int(np.ceil(acc0 / 9.0)) - len(usable)
    assert 0 < m <= len(fresh)
    sub = VC.subset(sc, EC.interleaved(usable, fresh[:m]))
    def at(log_beta):
        cov = VC.initial_covariance() * 10.0 ** log_beta
        return cov, _truth(sub, False, sub["state"], cov)
    lo, hi = -6.0, 2.0                       # bisect log10 of the scale for a step in [9.4e-5, 9.9e-5]
    for _ in range(30):
        mid = (lo + hi) / 2
        cov, t = at(mid)
        if 9.4e-5 <= t["steps"][0] <= 9.9e-5:
            break
        lo, hi = (mid, hi) if t["steps"][0] < 9.4e-5 else (lo, mid)
    assert t["iterations"] == 1 and 9e-5 < t["steps"][0] < 1e-4 * (1 - 1e-3), (t["iterations"], t["steps"])
    assert t["steps"][0] ** 3 / 24 > 2.5 * TOL_ROT
    s, _, _ = _check(env, sub, False, cov=cov, truth=t)
    err = max(np.abs(s[k] - t["state"][k]).max() for k in (slice(7, 16), slice(24, 28), slice(31, 35)))
    print(f"step {t['steps'][0]:.6e}: R_imu_camera and camera quaternions within {err:.2e} of the truth")
    assert err <= TOL_ROT, err


def test_flat_image_gives_exactly_zero_steps(env):
    """a constant image and an R_imu_camera whose quaternion has unit norm in FP64: S = 0, g = 0, d_x = 0 and every rotation step
    exactly 0; the state keeps its pose and the covariance its bits"""
    sc = _scene(env, "ric_identity")
    flat = dict(sc, img=EC.flat_image(sc))
    cov = VC.initial_covariance()
    t = _truth(flat, False, sc["state"], cov)
    assert t["iterations"] == 2 and max(t["steps"]) < 1e-40
    s, c, _ = _check(env, flat, False, truth=t, moved=False)
    assert np.array_equal(c, cov)
    assert np.array_equal(s[7:16], sc["state"][7:16])


# ---- non-finite and gross measurements -----------------------------------------------------------------------------------
@pytest.mark.parametrize("slot", [0, 127])
@pytest.mark.parametrize("field", ["uv", "vel"])
@pytest.mark.parametrize("value", [np.nan, np.inf, -np.inf], ids=["nan", "inf", "-inf"])
def test_esikf_non_finite_measurement_is_singular_and_writes_nothing(env, slot, field, value):
    """one non-finite uv or velocity component makes every row of S non-finite: SRL_SINGULAR, state and covariance untouched
    (the reference writes a NaN state and covariance and returns true; test_vio_edges_pin pins that)"""
    lio = env["lio"]
    sc = _scene(env, "base")
    arr = sc[field].copy()
    arr[slot, slot % 2] = value
    cov = VC.initial_covariance()
    sc["ip"].setCovariance(cov)
    st = _state(sc["state"], lio)
    with pytest.raises(lio.SrlError) as e:
        sc["ip"].vioEsikf(sc["cm"], st, sc["ids"], arr if field == "uv" else sc["uv"], arr if field == "vel" else sc["vel"], 40)
    assert e.value.code == 6   # SRL_SINGULAR
    assert np.array_equal(VC.state_array(st), sc["state"]) and np.array_equal(sc["ip"].covariance(), cov)


def test_photometric_nan_velocity_samples_zero(env):
    """a NaN velocity makes that point's projection NaN: the sampler gives colour 0 and zero derivatives, and the update stays
    finite and equal to the restatement's (the reference's read is undefined there: restatement only)"""
    sc = _scene(env, "base")
    vel = sc["vel"].copy()
    vel[3, 0] = np.nan
    vel[130, 1] = np.nan
    edge = dict(sc, vel=vel)
    _, _, t = _check(env, edge, False, reference=False)
    assert np.isnan(t["projections"][0][3, 0]) and np.isnan(t["projections"][0][130, 1])


@pytest.mark.parametrize("offset", [1e6, 3.4028234663852886e38, -3.4028234663852886e38], ids=["1e6", "flt_max", "-flt_max"])
def test_gross_uv_outliers_stay_bounded(env, offset):
    """a few matched points 1e6 px or at FLT_MAX from their projections (vioEsikf: vioPhotometric reads no uv): the Huber scale
    bounds each one's share of g, and the update stays finite and within the bounds of the restatement"""
    sc = _scene(env, "base")
    uv = sc["uv"].astype(np.float64)
    for k in (0, 127, 128, 300):
        uv[k, k % 2] = uv[k, k % 2] + offset
    edge = dict(sc, uv=np.clip(uv, -3.4028234663852886e38, 3.4028234663852886e38).astype(np.float32))
    assert np.all(np.isfinite(edge["uv"]))
    _, _, t = _check(env, edge, True)
    assert all(t["residual_norms"][0][k] > 0.9 * min(abs(offset), 1e38) for k in (0, 127, 128, 300))


# ---- rotation branches ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pair", EC.BRANCH_PAIRS, ids=lambda p: f"{p[0]}_{p[1]}")
@pytest.mark.parametrize("esikf", [True, False], ids=["esikf", "photometric"])
def test_rotation_branches(env, pair, esikf):
    """R_imu_camera and R_world R_imu_camera in the given branches of Quaterniond(Matrix3d), far from every boundary (two of the
    branches give q and -q, so a different branch would flip the stored quaternions); against the golden reference outputs too"""
    name = f"branch_{pair[0]}_{pair[1]}"
    sc = _scene(env, name)
    t = _truth(sc, esikf, sc["state"], VC.initial_covariance())
    b = EC.branches(t)
    assert ("Ric", pair[0]) in b and ("Rwc", pair[1]) in b, b
    s, c, _ = _check(env, sc, esikf, truth=t)
    g = np.load(GOLDEN)
    for k in ("ids", "xyz", "rgb", "cov_rgb", "n_rgb", "uv", "vel", "state"):
        assert np.array_equal(sc[k], g[f"{name}.{k}"]), (name, k)
    assert np.array_equal(np.frombuffer(VC.image_digest(sc["img"]), np.uint8), g[f"{name}.img_digest"])
    w = "esikf" if esikf else "photometric"
    tol, tol_cov = _bounds(VC.initial_covariance(), esikf)
    assert np.all(np.abs(s - g[f"{name}.{w}.state"]) <= 2 * tol * (1 + np.abs(g[f"{name}.{w}.state"])))
    assert np.abs(c - g[f"{name}.{w}.cov"]).max() <= 2 * tol_cov * np.abs(g[f"{name}.{w}.cov"]).max()
