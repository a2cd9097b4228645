"""The 50-digit restatement of vioEsikf / vioPhotometric (tests/vio_reference.py) pinned to the reference's own compiled code
(oracle/_ref/libsrl_vio_ref.so) on the seeded cases of tests/vio_cases.py: the same return values, and states and covariances
within rounding of each other; and the restatement's getRgb bit for bit the reference's cloudFrame::getRgb."""
import numpy as np
import pytest

import vio_cases as VC
import vio_ref as RF
import vio_reference as VR

pytestmark = pytest.mark.skipif(not RF.available(), reason="oracle/_ref/libsrl_vio_ref.so not built (needs the reference tree)")

# The compiled reference lies within 2e-15 (state, componentwise, relative to 1 + |x|) and 2e-14 (covariance, relative to its
# largest entry) of the truth on the well-conditioned cases; the bounds leave a factor of about 50.  The reference inverts
# Pw = (J P Jᵀ) w and then the sum S + Pw⁻¹: to first order the first inverse carries κ(Pw)·ε of relative error into the
# update, so the bound is max(TOL, κ(Pw)·ε) (ε = 2⁻⁵², κ measured by numpy in the 2-norm).  On the ill-conditioned case
# (κ = 1e8) that is 2.2e-8, and the reference is 6.6e-10 off in the covariance.
TOL, TOL_COV = 1e-13, 1e-12
EPS = 2.0 ** -52
CASES = VC.suite()
SINGULAR = [c for c in CASES if c[0] == "ill-conditioned"][0][1]


@pytest.mark.parametrize("name,case,cov", CASES, ids=lambda v: v if isinstance(v, str) else "")
@pytest.mark.parametrize("esikf", [True, False], ids=["esikf", "photometric"])
def test_reference_within_rounding_of_the_truth(name, case, cov, esikf):
    c = case
    rs, rc, rr, _ = RF.update(0 if esikf else 1, c["state"], cov, c["xyz"], c["uv"], c["vel"], c["rgb"], c["cov_rgb"], c["n_rgb"],
                              c["n_new_visited"], c["img"])
    t = VR.vio_update(esikf, c["state"], cov, c["xyz"], c["uv"], c["vel"], c["rgb"], c["cov_rgb"], c["n_rgb"], c["n_new_visited"],
                      c["img"])
    assert rr[0 if esikf else 1] == t["result"]
    kap = np.linalg.cond(cov[1:7, 1:7] if not esikf else cov) * EPS
    assert np.all(np.abs(rs - t["state"]) <= max(TOL, kap) * (1 + np.abs(t["state"]))), np.abs(rs - t["state"]).max()
    assert np.abs(rc - t["cov"]).max() <= max(TOL_COV, kap) * np.abs(t["cov"]).max()
    assert not VC.fragile(t, esikf, len(c["xyz"])), VC.fragile(t, esikf, len(c["xyz"]))


def test_the_suite_takes_both_sides_of_each_decision():
    seen = set()
    for name, c, cov in CASES:
        if c["xyz"].shape[0] > 300:
            continue
        if name == "photometric-break" or name == "photometric-no-break":
            t = VR.vio_update(False, c["state"], cov, c["xyz"], c["uv"], c["vel"], c["rgb"], c["cov_rgb"], c["n_rgb"], c["n_new_visited"],
                              c["img"])
            assert t["iterations"] == (1 if name == "photometric-break" else 2), (name, t["iterations"])
        te = VR.vio_update(True, c["state"], cov, c["xyz"], c["uv"], c["vel"], c["rgb"], c["cov_rgb"], c["n_rgb"], c["n_new_visited"])
        seen.update(("theta small", s < 1e-4) for s in te.get("steps", []))
        t = VR.vio_update(False, c["state"], cov, c["xyz"], c["uv"], c["vel"], c["rgb"], c["cov_rgb"], c["n_rgb"], c["n_new_visited"],
                          c["img"])
        seen.add(("photometric iterations", t["iterations"]))
        for h in t["huber"]:
            seen.update(("huber", bool(b)) for b in h)
    assert {("photometric iterations", 0), ("photometric iterations", 1), ("photometric iterations", 2)} <= seen
    assert {("huber", True), ("huber", False)} <= seen
    assert {("theta small", True), ("theta small", False)} <= seen


def test_singular_covariance_in_the_compiled_reference():
    """A zero fx variance: the reference's (J P Jᵀ w).inverse() makes vioEsikf's state and covariance non-finite.  The
    restatement (and the device) use (I + Pw S)⁻¹ Pw, the finite limit of the same formula (DESIGN.md section 5)."""
    c, cov = SINGULAR, VC.singular_covariance()
    rs, rc, rr, _ = RF.update(0, c["state"], cov, c["xyz"], c["uv"], c["vel"], c["rgb"], c["cov_rgb"], c["n_rgb"], c["n_new_visited"])
    assert rr[0] == 1
    assert not (np.all(np.isfinite(rs)) and np.all(np.isfinite(rc)))
    t = VR.vio_update(True, c["state"], cov, c["xyz"], c["uv"], c["vel"], c["rgb"], c["cov_rgb"], c["n_rgb"], c["n_new_visited"])
    assert np.all(np.isfinite(t["state"])) and np.all(np.isfinite(t["cov"]))
    assert t["cov"][7, 7] == 0.0 and np.all(t["cov"][7] == 0.0)


def test_get_rgb_bit_for_bit():
    rng = np.random.default_rng(3)
    img = VC.textured_image(64, 80, 5)
    for _ in range(400):
        u, v = rng.uniform(5, 74), rng.uniform(5, 58)
        if rng.random() < 0.2:
            u = float(np.floor(u)) + rng.choice([0.0, 0.5])
        ref = RF.get_rgb(img, u, v)
        mine = VR.get_rgb(img, u, v)
        for a, b in zip(ref, mine):
            assert np.array_equal(a.view(np.uint64), b.view(np.uint64)), (u, v, ref, mine)
