"""The colour renderer on crafted scenes (render_cases): the plain restatement (render_reference), the oracle
(OracleColorMap.render) and the reference's own compiled code (Reference.color_render) agree after every rendering on the
return count and every stored field: rgb, N_rgb, the bits of cov, observe_distance and last_observe_time.  Beside them the
exact layers: a first observation's colour lies within 2 of the exact bilinear value, and the covariance follows the exact
recursion within a first-order bound.

The oracle gets each image inside a buffer two rows taller than the image, and the reference harness copies it into one:
a point at v == rows - 1 exactly reads row `rows` with weight 0 (and at u == cols - 1 also the pixel after it), which then
stays in memory the caller owns.

CPU only; the reference comparisons are skipped when oracle/_ref/libsrl_reference.so was not built.
"""
from fractions import Fraction

import numpy as np
import pytest

from oracle import oracle_py as O
from oracle import reference_py as Rf

import render_cases as RC
import render_reference as RR
from render_cases import assert_state, padded

needs_ref = pytest.mark.skipif(not Rf.available(), reason="oracle/_ref/libsrl_reference.so not built (needs the reference tree)")


@pytest.mark.parametrize("name", list(RC.SCENES))
def test_oracle_equals_the_restatement(name):
    sc = RC.scene(name)
    oc = O.OracleColorMap(voxel_size=RC.VOXEL, max_num_points_in_voxel=RC.CAP, min_distance_points=RC.FINE)
    assert oc.add_points(sc.points, 1, 1.0, 0.0, True) == sc.points.shape[0]
    assert oc.counts()["recent"] == oc.counts()["voxels"]
    for k, r in enumerate(sc.renders):
        assert oc.render(r.cam.cam15, padded(r.img), r.obs_time, rows=r.cam.rows) == sc.counts[k], (name, k)
        assert_state(oc.snapshot(), sc, k, "oracle")


@needs_ref
@pytest.mark.parametrize("name", list(RC.SCENES))
def test_reference_equals_the_restatement(name):
    sc = RC.scene(name)
    ref = Rf.Reference()
    ref.add_points_to_map(sc.points, 1.0, 20, 0.15, 0, color_voxel_size=RC.VOXEL, color_max_points=RC.CAP, color_min_distance=RC.FINE,
                          add_point_step=1, time_sweep_end=1.0, time_last_process=0.0, to_rendering=True)
    assert ref.num_points(1) == sc.points.shape[0]
    for k, r in enumerate(sc.renders):
        assert ref.color_render(r.cam.cam15, r.img, r.obs_time) == sc.counts[k], (name, k)
        assert_state(ref.snapshot(which=1, cap=RC.CAP, color=True), sc, k, "reference")


@pytest.mark.parametrize("name", list(RC.SCENES))
def test_first_observation_colour_is_within_2_of_the_exact_bilinear_value(name):
    """four products each rounded by at most 1/2: the colour is within 2 of the exact value, unless the sum saturated"""
    sc = RC.scene(name)
    n_first = n_saturated = 0
    for k, r in enumerate(sc.renders):
        for o in sc.observations[k]:
            if not o.first:
                continue
            n_first += 1
            exact = RR.exact_bilinear(r.img, *o.uv)
            for ch in range(3):
                if o.sample.raw_sums[ch] > 255:
                    n_saturated += 1
                    assert o.sample.color[ch] == 255.0 and exact[ch] > 253
                else:
                    assert abs(Fraction(o.sample.color[ch]) - exact[ch]) <= 2, (name, k, ch, o.uv, o.sample.color, float(exact[ch]))
    assert n_first > 0
    if name == "saturation":
        assert n_saturated > 0


@pytest.mark.parametrize("name", list(RC.SCENES))
def test_covariance_follows_the_exact_recursion(name):
    """cov_rgb after each rendering against updateRgb's recursion at 80 digits (render_reference.exact_cov_chain).

    Bound (an estimate, which the restatement confirms): a fusion rounds cov to float twice (the process-noise sum and the
    posterior, 2^-24 relative each) and squares it in float once (2^-24 relative, halved by the square root); the double
    operations add ~1e-16.  The posterior map c -> sqrt(1 / (1 / c^2 + 1 / 15^2)) has derivative (new / c)^3 <= 1, so an
    earlier error does not grow.  After m fusions |cov - exact| <= 3 * m * 2^-24 * max(15, |cov|)."""
    sc = RC.scene(name)
    worst = 0.0
    for i in range(sc.points.shape[0]):
        times, flags = [], []
        for k, r in enumerate(sc.renders):
            o = sc.observations[k][i]
            times.append(r.obs_time)
            flags.append("first" if o.first else bool(o.fused))
        exact = RR.exact_cov_chain(times, flags)
        m = 0
        for k, (e, f) in enumerate(zip(exact, flags)):
            m += f is True
            if e is None:
                continue
            got = sc.states[k][i].cov
            assert got[0] == got[1] == got[2]
            bound = 3 * m * 2.0 ** -24 * max(15.0, abs(float(got[0])))
            err = abs(float(got[0]) - e)
            assert err <= bound, (name, i, k, float(got[0]), e, m)
            if m:
                worst = max(worst, err / bound)
    if name == "chain":
        assert max(s.n_rgb for s in sc.states[-1]) >= 30 and worst > 0.0
