"""Inputs of the NaN-planarity checks on the capped pass (max_num_residuals < n), shared by the capped-loop tests.

The map is degenerate_sets.nan_world(): isolated clusters, one of which makes the plane fit of a keypoint next to it NaN
(the reference throws std::runtime_error("error") when its loop reaches such a keypoint, src/optimize.cpp:348).  Each
case places that keypoint before, at or after k*, the keypoint at which the reference's loop breaks (src/optimize.cpp:107);
keypoints moved FAR away have no neighbourhood, so a prefix of them moves k* and the NaN keypoint into a later chunk of the
capped pass's schedule without changing which of them the loop reaches."""
import numpy as np

import degenerate_sets as D
from oracle import oracle_py as O

BIG = 2 ** 31 - 1
FAR = np.array([5000.0, 0.0, 0.0])


def nan_world():
    """The map, its oracle, the keypoints the oracle accepts (they decide k*) and the two NaN-planarity keypoints (one the
    gate would accept, one it rejects)."""
    clusters, good, n_acc, n_rej = D.nan_world()
    keys, counts, xyz = D.map_arrays(clusters)
    om = O.OracleMap()
    om.load(keys, counts, xyz)
    o = om.build_plane_residuals(good, D.IDENTITY_Q, D.ZERO_T, D.T_LAST, O.r3live_params(max_num_residuals=BIG), debug=True)
    acc = good[o.status == 2]
    assert acc.shape[0] >= 720
    return dict(map=(keys, counts, xyz), om=om, acc=acc, n_acc=n_acc, n_rej=n_rej)


def far_prefix(w, m):
    """m keypoints without a neighbourhood (never full, never counted toward the cap)."""
    return w["acc"][np.arange(m) % w["acc"].shape[0]] + FAR


def capped_nan_cases(w, m=0):
    """(cap, where, keypoints): the NaN keypoint before, at and after k* (cap >= 1: the cap-th accepted keypoint;
    cap <= 0: the first with a full neighbourhood), behind m keypoints without a neighbourhood."""
    acc, n_acc, n_rej = w["acc"], w["n_acc"][None], w["n_rej"][None]
    cat = np.concatenate
    cases = [
        (600, "before", cat([acc[:10], n_acc, acc[10:700]])),
        (600, "at", cat([acc[:599], n_acc, acc[599:700]])),
        (600, "after", cat([acc[:650], n_acc, acc[650:700]])),
        (1, "before", cat([n_rej, acc[:50]])),
        (1, "at", cat([n_acc, acc[:50]])),
        (1, "after", cat([acc[:1], n_acc, acc[1:50]])),
        (-1, "at", cat([n_acc, acc[:50]])),
        (-1, "after", cat([acc[:1], n_rej, n_acc, acc[1:50]])),
    ]
    if m:
        pre = far_prefix(w, m)
        cases = [(cap, where, cat([pre, kp])) for cap, where, kp in cases]
    return cases
