"""The kernel choice is per context: which compiled instance of each pass kernel a context launches (lanes per keypoint,
resident blocks per SM) and how it orders a sweep (cluster_order).  Options set on one context leave every other context
as it was; the environment variables set a context's choice when it is created; a choice other than the default gives the
same pass, on the host-driven and on the device-resident loop, when it is set before the context's first pass."""
import os
import subprocess
import sys

import numpy as np
import pytest

from sr_livo_b200 import capi, lio, synth

pytestmark = pytest.mark.gpu
BIG = 2 ** 31 - 1
DEFAULTS = dict(split_lanes_per_keypoint=4, scan_min_blocks=8, fit_min_blocks=6, fast_lanes_per_keypoint=1,
                fast_min_blocks=5, k1_min_blocks=3, cluster_order=1)
OTHERS = dict(split_lanes_per_keypoint=2, scan_min_blocks=6, fit_min_blocks=4, fast_lanes_per_keypoint=4,
              fast_min_blocks=8, k1_min_blocks=2, cluster_order=0)
INVALID = dict(split_lanes_per_keypoint=[1, 3, 8], scan_min_blocks=[4, 7], fit_min_blocks=[3, 7], fast_lanes_per_keypoint=[0, 3, 8],
               fast_min_blocks=[3, 7, 9], k1_min_blocks=[1, 5], cluster_order=[-1, 4], k1_variant=[-1, 4], shuffle_rule=[2])


def _close(a, b, rel=1e-12):   # the tolerance of test_gpu_parity.py for sums summed in a different order
    return np.abs(a - b).max() <= rel * np.abs(b).max()


def _choice(ctx):
    return {k: ctx.counter(k) for k in DEFAULTS}


def test_options_apply_to_the_context_they_are_set_on():
    a, b = lio.Context(0), lio.Context(0)
    try:
        assert _choice(a) == _choice(b) == DEFAULTS
        for k, v in OTHERS.items():
            a.set_option(k, v)
        assert _choice(a) == OTHERS and _choice(b) == DEFAULTS
        assert a.counter("cluster_order_active") == 0 and b.counter("cluster_order_active") == -1
    finally:
        a.close(); b.close()


def test_invalid_values_are_rejected_and_change_nothing():
    ctx = lio.Context(0)
    try:
        for k, bad in INVALID.items():
            before = ctx.counter(k)
            for v in bad:
                with pytest.raises(capi.SrlError) as ei:
                    ctx.set_option(k, v)
                assert ei.value.code == capi.SRL_BAD_ARG, (k, v)
                assert ctx.counter(k) == before, (k, v)
    finally:
        ctx.close()


_ENV_WORKER = r"""
import sys
sys.path.insert(0, sys.argv[1])
from sr_livo_b200 import lio
ctx = lio.Context(0)
print(ctx.counter("k1_min_blocks"), ctx.counter("fast_lanes_per_keypoint"), ctx.counter("fit_min_blocks"))
ctx.close()
"""


def test_environment_sets_the_choice_at_creation(tmp_path):
    """SRL_FIT_MINB=7 is not a compiled instance: the context keeps the default, 6."""
    script = tmp_path / "env_worker.py"
    script.write_text(_ENV_WORKER)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, SRL_K1_MINB="2", SRL_FAST_LPK="4", SRL_FIT_MINB="7")
    r = subprocess.run([sys.executable, str(script), root], capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    assert r.stdout.split() == ["2", "4", "6"]


def _load(L, world):
    L.voxel_map.upload(*world["omap"].snapshot())
    return world["sweep"]


def test_sweep_order_per_context(small_world):
    """A orders its sweeps with CUB, B with the cluster sort, verified against CUB in its own first four uses.  The pass
    sums are summed in sweep order, so both contexts' sums are bit-identical."""
    A = lio.LioOptimization(max_voxels=1 << 18, sweep_capacity=1 << 13)
    B = lio.LioOptimization(max_voxels=1 << 18, sweep_capacity=1 << 13)
    try:
        A.ctx.set_option("cluster_order", 0)
        prm = lio.r3live_params(max_num_residuals=BIG)
        out = {}
        for name, L in (("A", A), ("B", B)):
            sw = _load(L, small_world)
            for use in range(4):
                L.setKeypoints(sw.raw_xyz)
                assert L.ctx.counter("cluster_order_active") == {"A": 0, "B": -1 if use < 3 else 1}[name], (name, use)
            out[name] = L.buildPlaneResiduals(prm, sw.q_init, sw.t_init, sw.t_last)
        assert np.array_equal(out["A"].HTH, out["B"].HTH) and np.array_equal(out["A"].HTh, out["B"].HTh)
        assert out["A"].num_residuals == out["B"].num_residuals
    finally:
        A.close(); B.close()


def _run(world, options, iekf_kw):
    """A fresh context with `options` set before its first pass: the debug pass's neighbour ids, the product pass's sums
    and the updateIEKF result of the host-driven loop (0) and of the device-resident loop (1)."""
    L = lio.LioOptimization(max_voxels=1 << 18, sweep_capacity=1 << 13)
    try:
        for k, v in options.items():
            L.ctx.set_option(k, v)
        sw = _load(L, world)
        L.setKeypoints(sw.raw_xyz)
        prm = lio.r3live_params(max_num_residuals=BIG, **iekf_kw)
        out = dict(dbg=L.buildPlaneResiduals(prm, sw.q_init, sw.t_init, sw.t_last, debug=True),
                   sums=L.buildPlaneResiduals(prm, sw.q_init, sw.t_init, sw.t_last))
        for mode in (0, 1):
            L.ctx.set_option("device_loop", mode)
            L.eskf_pro = lio.EskfEstimator(p=sw.t_init.copy(), q=sw.q_init.copy(), cov=synth.prior_covariance())
            summ, fq, ft = L.updateIEKF(prm, sw.t_last)
            assert mode == 0 or L.ctx.counter("device_loop_active") == 1
            out[mode] = (summ, fq, ft, L.eskf_pro)
        return out
    finally:
        L.close()


FORMS = {
    "split": dict(k1_variant=3, split_lanes_per_keypoint=2, scan_min_blocks=6, fit_min_blocks=4, k1_min_blocks=4),
    "fast": dict(k1_variant=1, fast_lanes_per_keypoint=2, fast_min_blocks=8, k1_min_blocks=2),
    "assoc": dict(k1_variant=2, k1_min_blocks=2),
    "assoc_nb2": dict(k1_variant=2, k1_min_blocks=4),
}


@pytest.mark.parametrize("form", list(FORMS))
def test_non_default_choice_on_a_fresh_context(small_world, form):
    iekf_kw = dict(frame_id=5, num_iters_icp=3) if form == "assoc_nb2" else dict(threshold_translation_norm=0.0)
    ref = _run(small_world, {}, iekf_kw)
    got = _run(small_world, FORMS[form], iekf_kw)
    assert np.array_equal(got["dbg"].status, ref["dbg"].status) and np.array_equal(got["dbg"].nbr, ref["dbg"].nbr)
    g, r = got["sums"], ref["sums"]
    assert g.num_residuals == r.num_residuals and _close(g.HTH, r.HTH) and _close(g.HTh, r.HTh)
    for mode in (0, 1):
        (sg, qg, tg, eg), (sr, qr, tr, er) = got[mode], ref[mode]
        assert (sg.success, sg.passes_run, sg.num_residuals_used) == (sr.success, sr.passes_run, sr.num_residuals_used), mode
        assert np.allclose(sg.trace[:sg.passes_run], sr.trace[:sr.passes_run], rtol=1e-7, atol=1e-11), mode
        for f in ("p", "q"):
            assert np.allclose(getattr(eg, f), getattr(er, f), rtol=1e-9, atol=1e-11), (mode, f)
        assert np.allclose(qg, qr, atol=1e-11) and np.allclose(tg, tr, atol=1e-11), mode
