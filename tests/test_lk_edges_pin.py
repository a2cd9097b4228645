"""CPU pins of the pyramidal Lucas-Kanade at its edges (no GPU):
  - the numpy restatement (tests/lk_track_reference.py) equals the compiled reference (oracle/_ref/libsrl_lk_ref.so) on every
    crafted family of tests/lk_edge_cases.py: point bits (NaN payloads included), status, return value, level count and every
    padded level; and equals tests/golden/lk_track.npz on every golden run;
  - every family reaches the edge it is there for, read from the restatement's trace;
  - an exact layer independent of the reference: each float chain of A and b lies within gamma_n * sum |terms| of its int64
    sum, and well-conditioned points recover a whole-pixel shift.
"""
import os

import numpy as np
import pytest

import lk_cases as K
import lk_edge_cases as E
import lk_ref as R
import lk_track_reference as T

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lk_track.npz")
needs_ref = pytest.mark.skipif(not R.available(), reason="oracle/_ref/libsrl_lk_ref.so not built (needs the reference tree)")
pytestmark = pytest.mark.filterwarnings("ignore:invalid value encountered:RuntimeWarning")


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def test_cumsum_is_a_sequential_float32_chain():
    """The restatement's chains rely on np.cumsum being a left-to-right float32 accumulate (np.sum is pairwise)."""
    rng = np.random.default_rng(1)
    v = np.concatenate([[3e7, -3e7], rng.integers(-66585600, 66585601, 4000)]).astype(np.float32)
    acc = np.float32(0)
    for x in v:
        acc = np.float32(acc + x)
    got = np.cumsum(v[None, :, None], axis=1, dtype=np.float32)[0, -1, 0]
    assert bits(got) == bits(acc)


@needs_ref
@pytest.mark.parametrize("family", list(E.FAMILIES))
def test_restatement_matches_reference(family):
    for case in E.FAMILIES[family]():
        curr, st, ret, _, res = E.restate(case)
        ref = R.LKReference(**case.kw)
        ref.track(case.frames[0], case.pts)
        c_ref, s_ref, r_ref = ref.track(case.frames[1], case.pts)
        assert np.array_equal(bits(curr), bits(c_ref)), (case.name, np.flatnonzero((bits(curr) != bits(c_ref)).any(1))[:8])
        assert np.array_equal(st, s_ref) and ret == r_ref, case.name
        assert res.max_level == ref.info()["max_level"] and res.info()["max_count"] == ref.info()["max_count"], case.name
        assert res.info()["epsilon"] == ref.info()["epsilon"], case.name
        for which in (0, 1):
            for l in range(res.max_level + 1):
                for a, b in zip(res.level(which, l), ref.level(which, l)):
                    assert np.array_equal(a, b), (case.name, which, l)


@pytest.mark.parametrize("run", K.GOLDEN_RUNS, ids=[r[0] for r in K.GOLDEN_RUNS])
def test_restatement_matches_golden(run):
    g = np.load(GOLDEN)
    frames, pts, kw = K.run_inputs(run)
    res = T.LKRestated(**kw)
    key, last = run[0] + "/", pts
    for k, f in enumerate(frames):
        curr, st, ret = res.track(f, last)
        assert np.array_equal(bits(curr), bits(g[key + f"pts{k}"])), k
        assert np.array_equal(st, g[key + f"status{k}"]) and ret == int(g[key + f"ret{k}"]), k
        assert K.level_digest([res.level(0, l) for l in range(res.max_level + 1)]) == str(g[key + f"levels{k}"]), k
        last = curr
    assert res.max_level == int(g[key + "max_level"])


# ---- coverage: each family reaches its edge ---------------------------------------------------------------------------------

def _fold(cases, key, fn=max):
    out = 0
    for c in cases:
        _, _, _, tr, _ = E.restate(c)
        out = fn([out] + [int(l[key].max(initial=0)) for l in tr])
    return out


def test_saturation_reaches_the_extremes():
    cases = E.saturation()
    assert _fold(cases, "scharr") == 4080
    assert _fold(cases, "diff") == 8160
    assert _fold(cases, "madd") == 2 * 8160 * 4080 > 1 << 24


def test_min_eig_threshold_at_a_points_min_eig():
    cases = E.min_eig_cases()
    assert len(cases) == 6
    for c in cases:
        _, st, _, tr, res = E.restate(c)
        t = c.expect["target"]
        assert tr[0]["min_eig"][t] == res.min_eig or c.expect["rejected"], c.name     # exactly on the threshold
        assert (tr[0]["exit"][t] == T.MIN_EIG) == c.expect["rejected"], c.name
        assert st[t] == (0 if c.expect["rejected"] else 1), c.name


def test_faint_textures_straddle_flt_epsilon():
    by_thr = {}
    for c in E.faint_cases():
        _, _, _, tr, _ = E.restate(c)
        by_thr[c.kw["min_eig_threshold"]] = tr[0]
    lo = by_thr[-1.0]
    D, eps = lo["D"].astype(np.float64), float(T.FLT_EPSILON)
    below = D[(lo["exit"] == T.DET) & (D > 0)]
    above = D[(D >= eps) & (lo["exit"] != T.DET) & (lo["exit"] != T.MIN_EIG)]
    assert len(below) and len(above)
    # measured: 0.11 % below and 0.29 % above FLT_EPSILON
    assert (eps - below.max()) / eps < 0.01 and (above.min() - eps) / eps < 0.01
    neg = lo["min_eig"] < 0
    assert neg.sum() >= 3
    assert (lo["exit"][neg] != T.MIN_EIG).all()                     # threshold -1 lets them through to the D rule
    assert (by_thr[0.0]["exit"][neg] == T.MIN_EIG).all()            # threshold 0 stops them


def test_epsilon_at_an_iterations_ddot():
    cases = E.eps_cases()
    assert len(cases) >= 8
    for c in cases:
        _, _, _, tr, _ = E.restate(c)
        t, j = c.expect["target"], c.expect["j"]
        assert tr[0]["ddot"][t, j] >= c.kw["criteria"][2], c.name
        if c.expect["stops"]:
            assert tr[0]["exit"][t] == T.EPS and tr[0]["iters"][t] == j + 1, c.name
        else:
            assert tr[0]["iters"][t] > j + 1, c.name


def test_criteria_clamps():
    for c in E.criteria_cases():
        _, _, _, tr, res = E.restate(c)
        assert (res.max_count, res.epsilon) == c.expect["term"], c.name
        iters = np.concatenate([l["iters"] for l in tr])
        exits = np.concatenate([l["exit"] for l in tr])
        assert iters.max() <= res.max_count, c.name
        if res.max_count == 0:
            assert (exits == T.COUNT).any() and iters.max() == 0
        if res.epsilon == 10.0:
            assert ((exits == T.EPS) & (iters == 1)).sum() > 10
        if res.max_count in (1, 5):
            assert ((exits == T.COUNT) & (iters == res.max_count)).any(), c.name


def test_oscillation_rule_near_its_bound():
    (c,) = E.osc_cases()
    _, _, _, tr, _ = E.restate(c)
    m = E.osc_margins(tr[0])
    miss, hit = np.nanmin(np.where(m >= 0, m, np.nan)), np.nanmax(np.where(m < 0, m, np.nan))
    # the closest the scene gets to |dx + pdx| = 0.01 without firing and while firing (measured 2.4e-5 and -7.7e-6)
    assert 0 <= miss < 1e-4 and -1e-4 < hit < 0, (miss, hit)
    assert (tr[0]["exit"] == T.OSC).sum() >= 10


def test_borders_reach_every_limit():
    iter_out_levels, whole, partial = set(), 0, 0
    for c in E.borders():
        _, _, _, tr, _ = E.restate(c)
        for i, (level, side, axis, v, inside) in enumerate(c.expect["tags"]):
            assert tr[level]["ipx" if axis == 0 else "ipy"][i] == v, (c.name, level, side)
            assert (tr[level]["exit"][i] == T.OUTSIDE) != inside, (c.name, level, side)
            if v == -c.kw["win_size"][axis]:
                # on the low limit the patch sees the level's first column (row) and the zero border only, and REFLECT_101
                # makes that column's Ix (row's Iy) zero: A is rank one at most, D = 0, and the point is rejected whatever
                # its fraction.  So the first check's `< -W` and `<= -W` give the same outputs; only this trace tells them apart.
                l = tr[level]
                assert l["A12"][i] == 0 and l["A11" if axis == 0 else "A22"][i] == 0 and l["D"][i] == 0, (c.name, level, side)
                assert l["exit"][i] in (T.MIN_EIG, T.DET), (c.name, level, side)
        for level, l in enumerate(tr):
            if (l["exit"] == T.OUTSIDE_ITER).any():
                iter_out_levels.add(level)
            done = np.isfinite(l["A11"])
            whole += int(((l["A11"] == 0) & (l["A12"] == 0) & (l["A22"] == 0)).sum())
            partial += int((done & (l["ipx"] < 0) & (l["A11"] > 0)).sum())
    assert 0 in iter_out_levels and max(iter_out_levels) >= 1, iter_out_levels
    assert whole > 0 and partial > 0


def test_non_finite_points_come_back_quietened():
    for c in E.non_finite():
        curr, st, _, tr, _ = E.restate(c)
        p = c.pts
        nan = np.isnan(p)
        assert nan.sum() >= 3 * len(E.NAN_BITS)
        assert np.array_equal(bits(curr)[nan], bits(p)[nan] | 0x00400000)
        huge = ~np.isfinite(p) | (np.abs(p) >= 2.0 ** 31 - 128)
        assert (st[huge.any(1)] == 0).all()
        assert (np.asarray([l["exit"] for l in tr])[:, huge.any(1)] == T.OUTSIDE).all()
        assert np.array_equal(bits(curr)[huge & ~nan], bits(p)[huge & ~nan])   # only scaled by powers of two
        sub = (np.abs(p) < 1.2e-38) & (p != 0)
        assert sub.any(1).sum() >= 4 and st[sub.any(1) & ~huge.any(1)].any()


def test_shapes_reach_their_level_counts():
    seen = set()
    for c in E.shapes():
        _, _, _, _, res = E.restate(c)
        if c.expect["levels"] is not None:
            assert res.max_level == c.expect["levels"], c.name
        seen.add(len(c.pts))
        seen.add(res.max_level)
    assert {1, 2, 3, 5, 4097, 8} <= seen


# ---- the exact layer --------------------------------------------------------------------------------------------------------

def _gamma(n):
    u = 2.0 ** -24
    return n * u / (1 - n * u)


@pytest.mark.parametrize("pick", ["saturation", "shapes", "thresholds"])
def test_chains_within_gamma_bound_of_exact_sums(pick):
    """Each float chain (serial adds, lane folds, rounded int -> float terms) is within gamma_(n + 2) * sum |terms| of the exact
    int64 sum, n the number of terms: a bound that does not care about the order the reference picked."""
    cases = E.FAMILIES[pick]()[::3]
    checked = 0
    for c in cases:
        _, _, _, tr, _ = E.restate(c, exact=True)
        for l in tr:
            if "A_terms" not in l:
                continue
            done = np.isfinite(l["A_sum"][:, 0])
            err = np.abs(l["A_sum"][done].astype(np.float64) - l["A_exact"][done])
            assert (err <= _gamma(l["A_terms"] + 2) * l["A_abs"][done]).all(), c.name
            ran = np.isfinite(l["b_sum"][..., 0])
            err = np.abs(l["b_sum"][ran].astype(np.float64) - l["b_exact"][ran])
            assert (err <= _gamma(l["b_terms"] + 2) * l["b_abs"][ran]).all(), c.name
            checked += int(done.sum() + ran.sum())
    assert checked > 100


# measured largest error over these three scenes: 2.44e-4 px (about 1/4096 px, in every one); the tolerance keeps a 4x margin
SHIFT_TOL = 1e-3


@pytest.mark.parametrize("shift", [(3, -2), (-5, 1), (0, 7)])
def test_whole_pixel_shift_recovered(shift):
    dx, dy = shift
    w = E._texture(320, 240, 901 + dx)
    I, J = K.sample(w, 320, 240), K.sample(w, 320, 240, dx * 256, dy * 256)      # J(x) = I(x + d): content moves by -d
    rng = np.random.default_rng(902)
    pts = (rng.integers(40 * 256, 280 * 256, (400, 2)) / 256.0).astype(np.float32)
    pts[:, 1] = np.clip(pts[:, 1], 40, 200)
    res = T.LKRestated(**E.kw_with(criteria=(3, 30, 1e-6)))
    res.track(I, pts)
    curr, st, _ = res.track(J, pts)
    l0 = res.trace[0]
    good = (st == 1) & (l0["min_eig"] > 0.05) & (l0["exit"] == T.EPS)
    assert good.sum() > 40
    err = np.abs(curr[good].astype(np.float64) - (pts[good].astype(np.float64) - (dx, dy))).max()
    assert err < SHIFT_TOL, err
