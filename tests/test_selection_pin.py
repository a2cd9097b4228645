"""The crafted near-tie sets of tests/selection_sets.py on the CPU: the sets themselves, the oracle against a numpy brute
force, the compiled reference against the oracle, and proof that the sets tell the two plausible orders of the 3-term
distance reduction apart.

  * the generator's own properties: isolated neighbourhoods, every kept permutation pair exactly tied with different
    reference-order d^2 and different square roots, every family reaching its branches in the model;
  * oracle == brute force: FP64 d^2 in the reference's order c0 + (c1 + c2), ranked by (d^2, visit index);
  * every pair decided at the K-th boundary or at the nearest slot moves its batch's sums by >= 100x the tolerance the
    GPU test compares them with (the oracle with the winner moved just behind the loser);
  * compiled reference == oracle: buildPlaneResiduals rows bit for bit, searchNeighbors lists and voxels in order
    (skipped without oracle/_ref/libsrl_reference.so);
  * teeth: the reference compiled with (c0 + c1) + c2 disagrees with the oracle on family D, the default build on none.
"""
import numpy as np
import pytest

import selection_sets as S
from oracle import oracle_py as O
from oracle import reference_py as Rf

BIG = 2 ** 31 - 1
SUM_REL = 1e-6      # what test_selection_device.py allows between the device's sums and the oracle's


@pytest.fixture(scope="module")
def batches():
    return {(f, s): S.build_batch(f, s) for f in S.FAMILIES for s in S.SIZES}


def _oracle(b, debug=True, **kw):
    om = O.OracleMap()
    om.load(*b.map)
    return om.build_plane_residuals(b.kp, S.IDENTITY_Q, S.ZERO_T, S.T_LAST,
                                    O.r3live_params(size_voxel_map=b.size, max_num_residuals=BIG, **kw), debug=debug)


def test_generator_properties(batches):
    counts = {f: {} for f in S.FAMILIES}
    places = {f: set() for f in S.FAMILIES}
    for (f, s), b in batches.items():
        for k, h in enumerate(b.hoods):
            br = S.branch(S.measure(b, k))
            counts[f][br] = counts[f].get(br, 0) + 1
            places[f].add(h.place)
            if f == "D":
                a, c = (h.pts[i] for i in h.pair)
                assert S.exact_d2(a, h.kp) == S.exact_d2(c, h.kp)
                da, dc = S.ref_d2(a, h.kp), S.ref_d2(c, h.kp)
                assert da != dc and np.sqrt(da) != np.sqrt(dc)
    print({f: dict(c) for f, c in counts.items()})
    for f, mins in S.MINIMUMS.items():
        for br, n in mins.items():
            assert counts[f].get(br, 0) + counts[f].get("zone+nearest", 0) * (br in ("zone", "nearest")) >= n, (f, br, counts[f])
    assert all(len(p) >= (4 if f == "D" else 7) for f, p in places.items()), places


def test_oracle_equals_the_brute_force(batches):
    n_full = 0
    for (f, s), b in batches.items():
        o = _oracle(b)
        for k in range(len(b.hoods)):
            bf = S.brute_force(b, k)
            if o.status[k] == 0:
                assert len(bf) < S.K
                continue
            n_full += 1
            want = np.array([[*v, i] for _, _, i, v in bf], np.int16)
            assert np.array_equal(o.nbr[k], want), (f, s, b.hoods[k].variant)
            assert np.array_equal(o.nbr_dist[k], np.sqrt([d for d, *_ in bf])), (f, s, b.hoods[k].variant)
    assert n_full > 800


def _contrib(o):
    J = o.plane[:, 6:12]
    h = o.plane[:, 13] * o.plane[:, 14]
    acc = (o.status == 2)[:, None]
    return np.where(acc[:, :, None], J[:, :, None] * J[:, None, :], 0.0), np.where(acc, J * h[:, None], 0.0)


def test_every_decided_pair_moves_the_sums(batches):
    """Moving the reference's choice of each pair just behind the other candidate changes that keypoint's neighbourhood;
    its change of HTH / HTh relative to the batch's sums is the margin the GPU sum comparison has on that keypoint."""
    margins = []
    for (f, s), b in batches.items():
        pairs = [k for k, h in enumerate(b.hoods) if h.pair is not None and h.where in ("kth", "nearest")]
        if not pairs:
            continue
        o = _oracle(b)
        moved = b.xyz.copy()
        where = {}
        for j, (h_i, idx) in enumerate(b.slot):
            for i, p_i in enumerate(idx):
                where[(h_i, p_i)] = (j, i)
        for k in pairs:
            h = b.hoods[k]
            x, y = h.pair
            w, l = (x, y) if (S.ref_d2(h.pts[x], h.kp), x) < (S.ref_d2(h.pts[y], h.kp), y) else (y, x)
            jw, iw = where[(k, w)]
            d2l = float(S.ref_d2(h.pts[l], h.kp))
            tgt = h.kp + (h.pts[w] - h.kp) * np.sqrt((d2l + S.window(d2l, s) * 0.01) / float(S.ref_d2(h.pts[w], h.kp)))
            moved[jw, iw] = S._snap(h.kp, tgt, d2l + S.window(d2l, s) * 0.01)
        om = O.OracleMap()
        om.load(b.keys, b.counts, moved)
        o2 = om.build_plane_residuals(b.kp, S.IDENTITY_Q, S.ZERO_T, S.T_LAST,
                                      O.r3live_params(size_voxel_map=s, max_num_residuals=BIG), debug=True)
        H1, h1 = _contrib(o)
        H2, h2 = _contrib(o2)
        sH, sh, _ = S.sum_scales(o)
        for k in pairs:
            if not np.array_equal(o.nbr[k], o2.nbr[k]) or o.status[k] != o2.status[k]:
                margins.append(max((np.abs(H1[k] - H2[k]) / sH).max(), (np.abs(h1[k] - h2[k]) / sh).max()))
    m = np.array(margins)
    print(f"{m.size} decided pairs; change of the sums / tolerance: median {np.median(m) / SUM_REL:.0f}, "
          f"{int((m < 100 * SUM_REL).sum())} below 100")
    assert m.size >= 200 and (m >= 100 * SUM_REL).mean() >= 0.9


needs_ref = pytest.mark.skipif(not Rf.available(), reason="oracle/_ref/libsrl_reference.so not built (needs /root/reference)")


@needs_ref
@pytest.mark.parametrize("family", S.FAMILIES)
def test_compiled_reference_equals_the_oracle(batches, family):
    for s in S.SIZES:
        b = batches[(family, s)]
        ref = Rf.Reference()
        ref.load(*b.map)
        prm = O.r3live_params(size_voxel_map=s, max_num_residuals=BIG)
        r = ref.build_plane_residuals(b.kp, S.IDENTITY_Q, S.ZERO_T, S.T_LAST, prm)
        o = _oracle(b)
        assert not r["threw"] and r["num_residuals_used"] == o.num_residuals
        assert np.array_equal(r["world_xyz"], o.world_xyz) and np.array_equal(r["world_xyz"], b.kp)
        assert np.array_equal(r["rows"], o.plane[o.status == 2][:, :15])
        blocks = {tuple(k): x for k, x in zip(b.keys.tolist(), b.xyz)}
        for k in range(len(b.hoods)):
            xyz, vox = ref.search_neighbors(b.kp[k], nb=1, size=s, K=20, thr=1)
            if o.status[k] == 0:
                continue
            want = np.array([blocks[tuple(v[:3])][v[3]] for v in o.nbr[k].tolist()], np.float64)
            assert np.array_equal(xyz, want) and np.array_equal(vox, o.nbr[k][:, :3]), (family, s, b.hoods[k].variant)


@needs_ref
@pytest.mark.skipif(not Rf.available("packet"), reason="oracle/_ref/libsrl_reference_packet.so not built")
def test_the_sets_tell_the_two_reduction_orders_apart(batches):
    """Family D: the (c0 + c1) + c2 build picks another neighbour list (or another nearest point) than the oracle at many
    keypoints; the default build at none."""
    differ = same = 0
    for s in S.SIZES:
        b = batches[("D", s)]
        a, p = Rf.Reference(), Rf.Reference("packet")
        a.load(*b.map)
        p.load(*b.map)
        o = _oracle(b)
        blocks = {tuple(k): x for k, x in zip(b.keys.tolist(), b.xyz)}
        for k in range(len(b.hoods)):
            if o.status[k] == 0:
                continue
            want = np.array([blocks[tuple(v[:3])][v[3]] for v in o.nbr[k].tolist()], np.float64)
            xa, _ = a.search_neighbors(b.kp[k], nb=1, size=s)
            xp, _ = p.search_neighbors(b.kp[k], nb=1, size=s)
            assert np.array_equal(xa, want), (s, b.hoods[k].variant)
            if b.hoods[k].where in ("kth", "nearest"):
                differ += int(not np.array_equal(xp, want))
                same += int(np.array_equal(xp, want))
    print(f"family D: the (c0 + c1) + c2 build differs from the oracle at {differ} of {differ + same} decided keypoints")
    assert differ >= 10
