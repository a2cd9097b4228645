"""Generates the reference vectors with THE REFERENCE'S OWN CODE: oracle/_ref/libsrl_reference.so, i.e. the reference's
src/{optimize,utility,eskfEstimator,cloudMap,state,lioOptimization,rgbMapTracker}.cpp compiled unmodified by oracle/Makefile
over the stand-in headers of oracle/shim/ (DESIGN.md section 2).

  reference_outputs.npz     outputs on the inputs of scan_matching.npz / sweep_prep.npz / map_insert.npz (the fixture holds
                            only outputs); they pin the oracle (tests/test_golden.py, CPU) and the CUDA path (GPU).
  reference_small_world.npz outputs on the small_world fixture of tests/conftest.py and on the seeded plane-fit / observe
                            inputs of tests/test_host_logic.py (see small_world() below).

Both travel to machines where the reference sources are absent.  The arithmetic inside Eigen calls is the shim's restatement
(unpinned, see DESIGN.md).  Run from the repository root where oracle/Makefile could build oracle/_ref:
python tests/golden/make_reference_golden.py
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import oracle_py as O          # noqa: E402  (parameter structs only)
from oracle import reference_py as Rf      # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
BIG = 2 ** 31 - 1
PASS_CASES = {"nb1": dict(max_num_residuals=BIG, frame_id=100), "nb2": dict(max_num_residuals=BIG, frame_id=5),
              "cap": dict(max_num_residuals=100, frame_id=100), "cap600": dict(max_num_residuals=600, frame_id=100),
              "dflt": dict(max_num_residuals=-1, frame_id=100)}
IEKF_CASES = {"steady": dict(max_num_residuals=BIG), "cap600": dict(max_num_residuals=600), "init": dict(max_num_residuals=BIG, frame_id=5)}


def main():
    sm = np.load(os.path.join(HERE, "scan_matching.npz"))
    sp = np.load(os.path.join(HERE, "sweep_prep.npz"))
    mi = np.load(os.path.join(HERE, "map_insert.npz"))
    out = {}
    ref = Rf.Reference()
    ref.load(sm["map_keys"], sm["map_counts"], sm["map_xyz"])
    for tag, kw in PASS_CASES.items():                                  # lioOptimization::buildPlaneResiduals
        r = ref.build_plane_residuals(sm["raw_xyz"], sm["q_init"], sm["t_init"], sm["t_last"], O.r3live_params(**kw))
        assert not r["threw"]
        out.update({f"pass_{tag}_rows": r["rows"], f"pass_{tag}_world": r["world_xyz"], f"pass_{tag}_loss": np.array(r["loss_sum"]),
                    f"pass_{tag}_success": np.array(r["success"]), f"pass_{tag}_num_residuals": np.array(r["num_residuals_used"])})
    for tag, kw in IEKF_CASES.items():                                  # lioOptimization::updateIEKF
        e0 = O.Eskf(p=sm["t_init"].copy(), q=sm["q_init"].copy(), cov=sm["prior_cov"].copy())
        r = ref.update_iekf(sm["raw_xyz"], e0, sm["t_last"], O.r3live_params(**kw))
        assert not r["threw"] and r["success"]
        e = r["eskf"]
        out.update({f"iekf_{tag}_p": e.p, f"iekf_{tag}_q": e.q, f"iekf_{tag}_v": e.v, f"iekf_{tag}_ba": e.ba, f"iekf_{tag}_bg": e.bg,
                    f"iekf_{tag}_g": e.g, f"iekf_{tag}_cov": e.cov, f"iekf_{tag}_frame_q": r["frame_q"], f"iekf_{tag}_frame_t": r["frame_t"],
                    f"iekf_{tag}_num_residuals": np.array(r["num_residuals_used"])})
    # gridSampling, distortFrameBy*, transformAllImuPoint (src/utility.cpp)
    st = [dict(timestamp=r[0], quat=r[1:5], trans=r[5:8], vel=r[8:11], un_acc=r[11:14], un_gyr=r[14:17]) for r in sp["imu_states"]]
    t0 = float(sp["t0"])
    out["by_const"] = Rf.distort_frame_by_constant(sp["raw"], sp["rel"], st, t0, sp["R_il"], sp["t_il"])
    out["by_imu"] = Rf.distort_frame_by_imu(sp["raw"], sp["rel"], st, t0, sp["R_il"], sp["t_il"])
    out["by_imu_cut"] = Rf.distort_frame_by_imu(sp["raw"], sp["rel_cut"], st, t0, sp["R_il"], sp["t_il"], imu_xyz_in=np.full_like(sp["raw"], 9.0))
    out["end_frame"] = Rf.transform_all_imu_point(out["by_imu"], st[-1], sp["R_il"], sp["t_il"])
    out["grid_keep"] = Rf.grid_sampling(out["by_imu"], float(sp["grid_size"]))
    # addPointsToMap (src/lioOptimization.cpp:520-554), two batches
    m = Rf.Reference()
    out["added_a"] = np.array(m.add_points_to_map(mi["batch_a"]))
    s = m.snapshot()
    out.update(keys_a=s["keys"], counts_a=s["counts"], xyz_a=s["xyz"])
    out["added_b"] = np.array(m.add_points_to_map(mi["batch_b"]))
    s = m.snapshot()
    out.update(keys_b=s["keys"], counts_b=s["counts"], xyz_b=s["xyz"])
    np.savez_compressed(os.path.join(HERE, "reference_outputs.npz"), **out)
    print("reference_outputs.npz:", {k: v.shape for k, v in out.items() if k.startswith("pass_") and k.endswith("rows")},
          os.path.getsize(os.path.join(HERE, "reference_outputs.npz")) // 1024, "KiB")


def sha256(a) -> str:
    """Digest of a float64 array: stands for reference outputs too large to store, which the oracle reproduces bit for bit."""
    return hashlib.sha256(np.ascontiguousarray(a, np.float64).tobytes()).hexdigest()


# the parameter sets of the tests that compare with the reference on the `small_world` fixture (tests/conftest.py)
SMALL_PASS = [dict(max_num_residuals=BIG), dict(max_num_residuals=BIG, frame_id=5), dict(max_num_residuals=600)]
SMALL_UPDATE = [dict(max_num_residuals=BIG), dict(max_num_residuals=600)]
SMALL_HOST_ALGEBRA = [dict(max_num_residuals=BIG), dict(max_num_residuals=BIG, threshold_translation_norm=0.0), dict(max_num_residuals=600)]


def _state(out, prefix, r):
    e = r["eskf"]
    out.update({f"{prefix}_{f}": getattr(e, f) for f in ("p", "q", "v", "ba", "bg", "g", "cov")})
    out.update({f"{prefix}_frame_q": r["frame_q"], f"{prefix}_frame_t": r["frame_t"], f"{prefix}_success": np.array(r["success"]),
                f"{prefix}_num_residuals": np.array(r["num_residuals_used"])})


def small_world():
    """tests/golden/reference_small_world.npz: the reference's outputs on the `small_world` fixture (80 m map, 4000-point sweep) and
    on the seeded plane-fit / observe inputs of tests/test_host_logic.py.  Pass rows and transformed keypoints are stored as
    SHA-256 digests; the tests check that the oracle reproduces them and then compare the CUDA path with the oracle's arrays."""
    from sr_livo_b200 import synth
    pts = synth.sample_map_points(80.0, 60.0, seed=1)
    sw = synth.make_sweep(4000, seed=1000, yaw=0.5)
    om = O.OracleMap()
    om.add_points(pts)
    ref = Rf.Reference()
    ref.load(*om.snapshot())
    P = synth.prior_covariance()
    out = {}
    for i, kw in enumerate(SMALL_PASS):                                  # lioOptimization::buildPlaneResiduals
        r = ref.build_plane_residuals(sw.raw_xyz, sw.q_init, sw.t_init, sw.t_last, O.r3live_params(**kw))
        assert not r["threw"]
        out.update({f"pass{i}_success": np.array(r["success"]), f"pass{i}_num_residuals": np.array(r["num_residuals_used"]),
                    f"pass{i}_loss": np.array(r["loss_sum"]), f"pass{i}_rows_sha256": np.array(sha256(r["rows"])),
                    f"pass{i}_world_sha256": np.array(sha256(r["world_xyz"]))})
    v0 = np.array([0.3, 0.0, 0.0])
    for i, kw in enumerate(SMALL_UPDATE):                                # lioOptimization::updateIEKF, with a velocity in the prior
        r = ref.update_iekf(sw.raw_xyz, O.Eskf(p=sw.t_init.copy(), q=sw.q_init.copy(), v=v0.copy(), cov=P.copy()), sw.t_last, O.r3live_params(**kw))
        assert not r["threw"]
        _state(out, f"update{i}", r)
    for i, kw in enumerate(SMALL_HOST_ALGEBRA):
        r = ref.update_iekf(sw.raw_xyz, O.Eskf(p=sw.t_init.copy(), q=sw.q_init.copy(), cov=P.copy()), sw.t_last, O.r3live_params(**kw))
        assert not r["threw"]
        _state(out, f"host{i}", r)
    # computeNeighborhoodDistribution and eskfEstimator::observe on the seeded draws of
    # test_host_plane_fit_and_observe_match_the_compiled_reference (same generator, same order of draws)
    rng = np.random.default_rng(19)
    normals, a2d = np.zeros((200, 3)), np.zeros(200)
    for trial in range(200):
        Pn = rng.normal(size=(20, 3)) * np.array([0.5, 0.4, 0.01 * (1 + trial % 5)])
        Pn = (Pn @ np.linalg.qr(rng.normal(size=(3, 3)))[0].T + rng.normal(size=3) * 30).astype(np.float32).astype(np.float64)
        rc, nh = ref.neighborhood(Pn)
        assert rc == 0
        normals[trial], a2d[trial] = nh["normal"], nh["a2D"]
    observed = np.zeros((30, 19))
    for trial in range(30):
        scale = [0.05, 1e-6, 0.5][trial % 3]
        kw = dict(p=rng.normal(size=3), q=synth.quat_from_rotvec(rng.normal(size=3)), v=rng.normal(size=3), ba=rng.normal(size=3) * 0.01,
                  bg=rng.normal(size=3) * 0.01, g=np.array([0.3, -0.2, 9.7]) + rng.normal(size=3) * 0.1)
        dx = rng.normal(size=17) * scale
        b = Rf.eskf_observe(O.Eskf(**kw), dx)
        observed[trial] = np.concatenate([b.p, b.q, b.v, b.ba, b.bg, b.g])
    out.update(neighborhood_normal=normals, neighborhood_a2D=a2d, observe_p_q_v_ba_bg_g=observed)
    path = os.path.join(HERE, "reference_small_world.npz")
    np.savez_compressed(path, **out)
    print("reference_small_world.npz:", os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
    small_world()
