"""The edge cases of the camera updates (tests/vio_edge_cases.py) on the host: the chunk arithmetic the device tests rely on,
the restatement's multiplicity against an explicitly tiled list, the compiled reference within rounding of the restatement on
host stand-ins of the device edge scenes (and its NaN outcome for a non-finite measurement, where the device deviates), and
that the edge set reaches every branch, swap column, chunk shape and small-angle branch it is there for."""
import numpy as np
import pytest

import vio_cases as VC
import vio_edge_cases as EC
import vio_ref as RF
import vio_reference as VR

EPS = 2.0 ** -52
TOL, TOL_COV = 1e-13, 1e-12   # test_vio_pin's bounds of the compiled reference against the truth
needs_ref = pytest.mark.skipif(not RF.available(), reason="oracle/_ref/libsrl_vio_ref.so not built (needs the reference tree)")


def _truth(sc, esikf, cov, state=None, img=None, mult=None):
    return VR.vio_update(esikf, sc["state"] if state is None else state, cov, sc["xyz"], sc["uv"], sc["vel"], sc["rgb"], sc["cov_rgb"],
                         sc["n_rgb"], 40, sc["img"] if img is None else img, mult=mult)


def _stand_ins():
    """(name, esikf, scene, covariance, state, image) of the host stand-ins"""
    out = []
    base = EC.stand_in()
    for esikf in (True, False):
        for col in EC.PIVOT_TARGETS[esikf]:
            out.append((f"pivot-{col}", esikf, base, EC.pivot_covariance(base, esikf, col), None, None))
        for a, b in EC.BRANCH_PAIRS:
            out.append((f"branch-{a}-{b}", esikf, EC.stand_in(507, rotation=EC.branch_pose(a, b)[0], ric=EC.branch_pose(a, b)[1]),
                        VC.initial_covariance(), None, None))
    for name, st, uv, vel in EC.small_step_variants(base):
        out.append((name, True, dict(base, uv=uv, vel=vel), VC.initial_covariance(), st, None))
    flat = EC.stand_in(506, ric=np.eye(3))
    out.append(("flat-image", False, flat, VC.initial_covariance(), None, EC.flat_image(flat)))
    return out


STAND_INS = _stand_ins()


def test_chunk_shapes():
    """E = 79 / 29 sums in 3 / 8 segments; n = 129 leaves a last chunk of one point, fewer rows than segments; the tiled list has
    159 chunks and a 23-point last chunk"""
    assert EC.dims(True)[2:] == (79, 3) and EC.dims(False)[2:] == (29, 8)
    assert EC.chunk_shape(129, True) == (2, 1, 2, 3, 2) and EC.chunk_shape(129, False) == (2, 1, 3, 8, 3)
    assert EC.chunk_shape(128, True)[:2] == (1, 128) and EC.chunk_shape(256, False)[:2] == (2, 128)
    assert EC.chunk_shape(10, True) == (1, 10, 20, 3, 3) and EC.chunk_shape(10, False) == (1, 10, 30, 8, 8)
    assert EC.chunk_shape(len(EC.tiled()), True)[:2] == (159, 23)


@pytest.mark.parametrize("esikf", [True, False], ids=["esikf", "photometric"])
def test_multiplicity_equals_the_tiled_list(esikf):
    c = EC.stand_in(n=23)
    c["n_rgb"][[0, 5]] = 1
    idx = np.tile(np.arange(23), 3)
    a = _truth(c, esikf, VC.initial_covariance(), mult=[3] * 23)
    b = _truth(VC.subset(c, idx), esikf, VC.initial_covariance())
    assert (a["iterations"], a["used"], a["result"]) == (b["iterations"], b["used"], b["result"])
    assert np.array_equal(a["state"], b["state"]) and np.array_equal(a["cov"], b["cov"])


@needs_ref
@pytest.mark.parametrize("name,esikf,sc,cov,state,img", STAND_INS, ids=[f"{s[0]}-{'esikf' if s[1] else 'photometric'}" for s in STAND_INS])
def test_reference_within_rounding_of_the_truth(name, esikf, sc, cov, state, img):
    state = sc["state"] if state is None else state
    img = sc["img"] if img is None else img
    t = _truth(sc, esikf, cov, state, img)
    assert not VC.fragile(t, esikf, len(sc["xyz"])), VC.fragile(t, esikf, len(sc["xyz"]))
    rs, rc, rr, _ = RF.update(0 if esikf else 1, state, cov, sc["xyz"], sc["uv"], sc["vel"], sc["rgb"], sc["cov_rgb"], sc["n_rgb"], 40, img)
    assert rr[0 if esikf else 1] == t["result"]
    kap = np.linalg.cond(cov if esikf else cov[1:7, 1:7]) * EPS
    assert np.all(np.abs(rs - t["state"]) <= max(TOL, kap) * (1 + np.abs(t["state"]))), np.abs(rs - t["state"]).max()
    assert np.abs(rc - t["cov"]).max() <= max(TOL_COV, kap) * np.abs(t["cov"]).max()


@needs_ref
@pytest.mark.parametrize("field", ["uv", "vel"])
def test_reference_writes_nan_for_a_non_finite_measurement(field):
    """the reference's vioEsikf with one NaN uv or velocity returns true with a non-finite state and covariance; the device
    returns SRL_SINGULAR and writes nothing (DESIGN.md section 5, test_vio_edges_device)"""
    c = EC.stand_in(n=40)
    arr = c[field].copy()
    arr[0, 0] = np.nan
    rs, rc, rr, _ = RF.update(0, c["state"], VC.initial_covariance(), c["xyz"], arr if field == "uv" else c["uv"],
                              arr if field == "vel" else c["vel"], c["rgb"], c["cov_rgb"], c["n_rgb"], 40)
    assert rr[0] == 1 and not np.all(np.isfinite(rs)) and not np.all(np.isfinite(rc))


def test_the_edge_set_reaches_every_branch_swap_column_chunk_shape_and_small_angle_branch():
    seen = set()
    for name, esikf, sc, cov, state, img in STAND_INS:
        t = _truth(sc, esikf, cov, state, img)
        for role, br in EC.branches(t):
            seen.add(("rot2q", role, br))
        for sy in t.get("systems", []):
            seen.update(("swap", esikf, k) for k in EC.pivot_replay(sy["M"])[0])
        seen.update(("exp_quat small", s < 1e-4) for s in t.get("steps", []))
        seen.update(("log_so3 small", s < 1e-4) for s in t.get("dx_rot", [])[1:])
        if name == "flat-image":
            assert t["iterations"] == 2 and max(t["steps"]) < 1e-40
            seen.add(("zero step",))
    for n in EC.CHUNK_NS:
        for esikf in (True, False):
            chunks, last, rows, segs, filled = EC.chunk_shape(n, esikf)
            seen.add(("chunk", esikf, "full" if last == EC.CHUNK else ("one point" if last == 1 else "partial")))
            if filled < segs:
                seen.add(("chunk", esikf, "empty segments"))
    for role in ("Ric", "Rwc"):
        assert {("rot2q", role, b) for b in ("trace", "i=0", "i=1", "i=2")} <= seen, sorted(s for s in seen if s[0] == "rot2q")
    for esikf in (True, False):
        assert {("swap", esikf, k) for k in EC.PIVOT_TARGETS[esikf]} <= seen
        assert {("chunk", esikf, k) for k in ("full", "one point", "partial", "empty segments")} <= seen
    assert {("exp_quat small", True), ("exp_quat small", False), ("log_so3 small", True), ("log_so3 small", False), ("zero step",)} <= seen
