"""The oracle's sweep preparation (distortFrameByConstant, distortFrameByImu, transformAllImuPoint, gridSampling) against a
50-digit restatement (tests/sweep_prep_reference.py) on the inputs of tests/sweep_prep_cases.py, and against the
reference's own compiled sources when oracle/_ref is built.  CPU only.

The truth takes the reference's decisions in FP64 and evaluates everything after them exactly; each output carries a
first-order componentwise bound of the FP64 evaluation's error (`E` in the reference module).  The oracle calls glibc,
which is within 1 ulp, so it must lie within the bound itself (constant 1).
"""
from __future__ import annotations

import math
import os

import numpy as np
import pytest

import sweep_prep_cases as SC
import sweep_prep_reference as R
from oracle import oracle_py as O

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = {c["name"]: c for c in SC.all_cases()}
VALUED = [n for n, c in CASES.items() if c["kind"] != "grid"]
_TRUTH = {}


def truth(name):
    if name not in _TRUTH:
        _TRUTH[name] = SC.truth(CASES[name])
    return _TRUTH[name]


def _states(sp):
    return [dict(timestamp=r[0], quat=r[1:5], trans=r[5:8], vel=r[8:11], un_acc=r[11:14], un_gyr=r[14:17]) for r in sp["imu_states"]]


def test_truth_restates_the_oracle_on_the_golden_sweep():
    sp = np.load(os.path.join(HERE, "golden", "sweep_prep.npz"))
    st, t0 = _states(sp), float(sp["t0"])
    oc = O.distort_frame_by_constant(sp["raw"], sp["rel"], st, t0, sp["R_il"], sp["t_il"])
    oi, n = O.distort_frame_by_imu(sp["raw"], sp["rel"], st, t0, sp["R_il"], sp["t_il"])
    ot = O.transform_all_imu_point(oi, st[-1], sp["R_il"], sp["t_il"])
    nw, k_of = R.walk(t0, sp["rel"], [s["timestamp"] for s in st])
    assert nw == n == int(sp["n_imu"])
    tps = R.time_points(t0, sp["rel"])
    for i in SC.sample(len(sp["rel"]), 64, seed=1):
        p, _ = R.distort_constant_point(sp["raw"][i], sp["rel"][i], st, t0, sp["R_il"], sp["t_il"])
        q, _ = R.distort_imu_point(sp["raw"][i], float(tps[i]), st[k_of[i]], st[k_of[i] + 1], sp["R_il"], sp["t_il"])
        e = R.transform_all_imu_point(oi[i], st[-1], sp["R_il"], sp["t_il"])
        for got, v in ((oc[i], p), (oi[i], q), (ot[i], e)):
            assert np.all(np.abs(got - R.vals(v)) <= 1e-12 * np.abs(R.vals(v)).max())
            assert np.all(np.abs(got - R.vals(v)) <= R.errs(v))


@pytest.mark.parametrize("name", VALUED)
def test_oracle_within_the_truth_bounds(name):
    c, tr = CASES[name], truth(name)
    out, n_written = SC.run(O, c)
    if c["kind"] == "imu":
        assert n_written == tr["n_written"]
        assert np.all(out[n_written:] == -7.0)          # the points the walk never reaches keep the caller's values
        assert np.array_equal(np.diff(tr["k_of"]) >= 0, np.ones(max(0, n_written - 1), bool))
    got = out[tr["idx"]]
    err = np.abs(got - tr["val"])
    bad = ~(err <= tr["err"])
    assert not bad.any(), (name, tr["idx"][bad.any(axis=1)][:5], err[bad][:5], tr["err"][bad][:5])


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_the_compiled_reference_bit_for_bit(name):
    from oracle import reference_py as Rf
    if not Rf.available():
        pytest.skip("the compiled reference (oracle/_ref) is not built here")
    c = CASES[name]
    if c["kind"] == "grid" and name in ("grid_nonfinite", "grid_key_range"):
        # the reference's (short) cast of a NaN or out-of-range quotient is undefined: only the defined rows are compared
        keys, _ = R.grid_keys(c["xyz"], c["size"])
        c = dict(c, xyz=c["xyz"][[k is not None for k in keys]])
    o, _ = SC.run(O, c)
    r, _ = SC.run(Rf, c)
    assert o.shape == r.shape and o.tobytes() == r.tobytes()


def test_bounds_are_not_vacuous():
    """Every bound is far below the quantity's scale (raw points to 200 m, translations to 1e4 m), and the oracle's error
    reaches a sizeable fraction of its bound somewhere: the bound is neither empty nor loose by orders of magnitude."""
    worst_ratio, worst_bound = 0.0, 0.0
    for name in VALUED:
        c, tr = CASES[name], truth(name)
        if tr["idx"].size == 0:
            continue
        out, _ = SC.run(O, c)
        err = np.abs(out[tr["idx"]] - tr["val"])
        scale = np.abs(tr["val"]).max(axis=1, keepdims=True) + 1.0
        assert np.all(tr["err"] <= 1e-12 * np.maximum(scale, 1e4)), name
        worst_bound = max(worst_bound, float(tr["err"].max()))
        pos = tr["err"] > 0
        worst_ratio = max(worst_ratio, float((err[pos] / tr["err"][pos]).max()))
    print(f"largest bound {worst_bound:.3g} m; largest oracle error / bound {worst_ratio:.3g}")
    assert worst_bound < 1e-8
    assert worst_ratio > 0.05


def _ulp(x):
    return float(np.spacing(abs(x)))


@pytest.mark.parametrize("name", VALUED)
def test_no_decision_within_a_bound_of_its_threshold(name):
    """Unless the case exists to pin it, every FP64 decision is clear of its threshold by more than the error of the
    quantity it tests, so a correct kernel cannot take the other branch."""
    c, tr = CASES[name], truth(name)
    pins = c["pins"]
    for inf in tr["info"]:
        if "d" in inf and "slerp" not in pins:
            # |d| against one: the FP64 dot carries at most its bound; `one` is exact
            assert abs(abs(inf["d"]) - R.ONE) > 2 * inf["d_err"] + 1e-300, (name, inf["d"])
        if "theta" in inf and c["kind"] == "imu" and "so3" not in pins:
            assert abs(inf["theta"] - R.K_THETA) > 8 * R.U * max(inf["theta"], R.K_THETA), (name, inf["theta"])
        if "alpha" in inf and "clamp" not in pins and inf["clamp"] == 0:
            assert min(abs(inf["alpha"]), abs(inf["alpha"] - 1)) > 4 * R.U, (name, inf["alpha"])
    if "time" in pins or c["kind"] == "end":
        return
    # time_point against every threshold the walk and the nudges compare it with: clear by more than two ulps
    tp = R.time_points(c["t0"], c["rel"])
    ts = np.array([s["timestamp"] for s in c["states"]])
    thr = np.r_[ts - R.NUDGE, ts + R.NUDGE]
    for x in tp[np.isfinite(tp)]:
        assert np.abs(thr - x).min() > 2 * _ulp(x), (name, x)


def test_cases_reach_the_branches_they_pin():
    def lerp_of(name):
        return {bool(i["lerp"]) for i in truth(name)["info"]}
    assert lerp_of("d_at_one") == {True} and lerp_of("d_ulp_above") == {True} and lerp_of("d_ulp_below") == {False}
    assert lerp_of("d_at_one_neg") == {True} and lerp_of("d_ulp_below_neg") == {False} and lerp_of("antipodal") == {True}
    for k in range(5):
        assert lerp_of(f"d_near_{k}") == {False}
        assert all(1 - abs(i["d"]) < 1e-12 for i in truth(f"d_near_{k}")["info"])
    assert lerp_of("rot90") == lerp_of("rot170") == lerp_of("neg_dot") == {False}
    assert all(i["d"] < 0 for i in truth("neg_dot")["info"])
    # the clamps fire at both ends
    assert {i["clamp"] for i in truth("rot90")["info"]} == {-1, 0, 1}
    # so3: both branches, including 2^-45 on either side of 1e-4
    th = [(i["theta"], i["small"]) for i in truth("so3_threshold")["info"]]
    assert any(s for _, s in th) and any(not s for _, s in th)
    assert min(abs(t - R.K_THETA) for t, _ in th) < 1e-4 * 2.0 ** -40
    assert all(i["small"] for n in ("zero_gyro", "slow_from_zero", "begin_zero") for i in truth(n)["info"])
    big = [not i["small"] for i in truth("gyro_10rad")["info"]]
    assert sum(big) > 0.95 * len(big)          # all but the points nudged to 1e-6 s after an interval's start
    # the walk: stamps +- k ulp give both nudges, points before the first stamp and a NaN stop it
    assert truth("stamp_ulps")["n_written"] == CASES["stamp_ulps"]["rel"].size
    assert {i["nudge"] for i in truth("stamp_ulps")["info"]} >= {1, 2}
    assert truth("before_first")["n_written"] == 0 and truth("nan_time")["n_written"] == 137
    # time_point = rel / 1000 differs from rel * 1e-3 on some points of begin_zero
    c = CASES["time_rounding"]
    assert c["rel"].size >= 32 and np.all(c["t0"] + c["rel"] / 1000.0 != c["t0"] + c["rel"] * 1e-3)
    assert all(i["small"] for i in truth("time_rounding")["info"])
    rel = CASES["begin_zero"]["rel"]
    assert np.count_nonzero(rel / 1000.0 != rel * 1e-3) > 100


def test_grid_keys_against_the_truth():
    for name in ("grid_quotient_ulp", "grid_cell0"):
        c = CASES[name]
        assert sorted(O.grid_sampling(c["xyz"], c["size"]).tolist()) == R.grid_sampling(c["xyz"], c["size"])
    c = CASES["grid_quotient_ulp"]
    q = c["xyz"][1::2, 0] / c["size"]
    assert np.all(np.trunc(q) != np.trunc(c["xyz"][1::2, 0] * (1.0 / c["size"])))
    assert len(R.grid_sampling(c["xyz"], c["size"])) == q.size          # every such point joins its partner's cell
    # -0.0 and +0.0 and both halves of (-1, 1) share cell 0; -0.1 / 0.1 are the neighbours; -0.1000001 too (trunc)
    keys, _ = R.grid_keys(CASES["grid_cell0"]["xyz"], 0.1)
    assert keys[0] == keys[1] == keys[2] == keys[3] == keys[4] == (0, 0, 0)
    assert keys[5] == (-1, 0, 0) and keys[6] == (1, 0, 0) and keys[7] == (-1, 0, 0)
    # |x / size| >= 32765 makes no cell here (the reference's cast is undefined there); 32764.x does
    keys, _ = R.grid_keys(CASES["grid_key_range"]["xyz"], 1.0)
    assert [k is None for k in keys] == [False, False, False, True, True, True, False]
    keys, _ = R.grid_keys(CASES["grid_nonfinite"]["xyz"], 1.0)
    assert [k is None for k in keys] == [True, True, True, False, True, False]


def test_point_transforms_are_compiled_without_contraction():
    """srl_points.cu rounds every product and sum separately (--fmad=false): the end-of-sweep transform has no DFMA, and
    the source calls no fma itself, so the DFMAs left in the other kernels belong to division, sqrt and libm."""
    import shutil
    import subprocess
    root = os.path.dirname(HERE)
    src = open(os.path.join(root, "sr_livo_b200", "csrc", "srl_points.cu")).read()
    assert "fma" not in src.replace("--fmad", "")
    obj = os.path.join(root, "sr_livo_b200", "csrc", "build", "srl_points.o")
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not (os.path.exists(obj) and os.path.exists(tool)):
        pytest.skip("no srl_points object or cuobjdump here")
    sass = subprocess.run([tool, "-sass", obj], capture_output=True, text=True, check=True).stdout
    fn, count = None, {}
    for line in sass.splitlines():
        if "Function :" in line:
            fn = line.split("Function :")[1].strip()
        elif "DFMA" in line:
            count[fn] = count.get(fn, 0) + 1
    assert "k_imu_to_lidar_end" in sass
    assert not [f for f in count if "k_imu_to_lidar_end" in f], count
