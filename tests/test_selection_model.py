"""CPU model of the FP32 neighbour selection of k1_scan / k1_fit (sr_livo_b200/csrc/srl_fast.cu) and property tests of the
exactness argument in DESIGN.md §4 ("Why the FP32 selection is exact").

The kernels select the K = 20 nearest map points of a keypoint from packed 32-bit keys (FP32 squared distance with the
low 10 mantissa bits replaced by a candidate id), four lanes per keypoint with 14-entry lists, and certify the result
with a handful of window tests; anything not certified is flagged and redone with FP64 keys.  The association has to
be bit-exact, so the certificate must never pass a wrong answer.  This file restates that logic in numpy (same
constants, same formulas) and attacks it with adversarial candidate sets: near ties at the K-th distance, clusters,
duplicates, FP32 errors at the assumed bound.  It also checks the bound itself on the kernel's FP32 distance formula.
No GPU, no product code: a model of the math, complementing the GPU parity tests.

Second part: the parallel formulations used by rows N2 / N3 (srl_grid_sampling's dedupe-then-replay, the max-scan form
of distortFrameByImu's one-iterator walk) against the sequential originals, on random and degenerate inputs.
"""
import numpy as np
import pytest

KF, NG = 20, 3
NS = KF + NG          # candidate slots that can end up in the neighbourhood
NL = NS + 1           # + the certifier
LPK, NLS = 4, 14      # lanes per keypoint, keys tracked per lane
K_REL = np.float32(1.0 / 2048.0)
K_ZONE0, K_BEST_MAX = 12, 4
INF_KEY = np.uint32(0xFFFFFFFF)


def key_value(k):
    k = np.asarray(k, np.uint32)
    v = (k & np.uint32(0xFFFFFC00)).view(np.float32).copy()
    v[k == INF_KEY] = np.inf
    return v


def scan_verdict(d2f, size=1.0, chunks=None, lbs=None, lpk=LPK, nls=NLS, fast=False, ids=None):
    """The FP32 stage of one keypoint: lane lists, voxel skip, merge and verdict.  fast=False models k1_scan<lpk, nls>
    (skip bound = the largest of the lanes' ceil(K/lpk)-th keys, lane certificate, j0 / b1 rules); fast=True models
    k1_fast with lpk lanes of NL keys (skip bound = the smallest of the lanes' K-th keys, certifier only).  ids: the
    10-bit candidate id packed into each key (default: the candidate's index).  Returns a dict with flagged, m, j0, b1,
    the merged keys and, per slot, the candidate index it holds."""
    n = d2f.shape[0]
    eps_abs = np.float32(1e-4) * np.float32(size) * np.float32(size)
    ids = np.arange(n, dtype=np.uint32) if ids is None else np.asarray(ids, np.uint32)
    assert n <= 1024 and int(ids.max(initial=0)) < 1024
    keys = (d2f.astype(np.float32).view(np.uint32) & np.uint32(0xFFFFFC00)) | ids
    if chunks is None:
        chunks, lbs = [np.arange(n)], np.zeros(1, np.float32)
    width = NL if fast else nls
    lane_lists = [np.full(width, INF_KEY, np.uint32) for _ in range(lpk)]
    q = (KF + lpk - 1) // lpk
    for ch, lb in zip(chunks, lbs):
        if fast:
            T = min(key_value([l[KF - 1]])[0] for l in lane_lists)   # every lane's K-th key bounds the K-th from above
        else:
            T = key_value([max(l[q - 1] for l in lane_lists)])[0]   # the largest of the lanes' q-th keys bounds the K-th
        with np.errstate(invalid="ignore", over="ignore"):
            if np.float32(lb) > np.float32(T + T * K_REL + np.float32(3.0) * eps_abs):
                continue                                         # the voxel cannot matter any more
        ch = np.asarray(ch)
        for lane in range(lpk):
            mine = keys[ch[lane::lpk]]                            # dealt round-robin inside the voxel
            merged = np.sort(np.concatenate([lane_lists[lane], mine]))
            lane_lists[lane] = merged[:width]
    own_last = [l[width - 1] for l in lane_lists]
    merged = np.sort(np.concatenate(lane_lists + [np.full(32, INF_KEY, np.uint32)]))[:32]
    kv = key_value(merged)
    pos = {int(k): i for i, k in enumerate(keys)}
    slot_cand = np.array([pos.get(int(k), -1) for k in merged])
    out = dict(keys=merged, slot_cand=slot_cand, m=0, j0=0, b1=0)
    if not np.isfinite(kv[KF - 1]):
        out["flagged"] = True                                     # fewer than K tracked: the kernel never gets here (total < Kmin)
        return out
    T = kv[KF - 1]
    lim = np.float32(T + T * K_REL + np.float32(2.5) * eps_abs)
    kvK, v0 = kv[KF], kv[0]
    lim0 = np.float32(v0 + v0 * K_REL + np.float32(2.5) * eps_abs)
    m = int((kv[:NS] <= lim).sum())
    b1 = int((kv[:NS] <= lim0).sum())
    with np.errstate(invalid="ignore"):
        j0 = int(((kv[:KF] + kv[:KF] * K_REL + np.float32(2.5) * eps_abs) < kvK).sum())
    if fast:   # k1_fast resolves every slot inside the window exactly: only the certifier
        flagged = not kv[NS] > lim
        j0, b1 = 0, m
    else:
        flagged = (not kv[NS] > lim) or any(not key_value([o])[0] > lim for o in own_last) or \
                  (m > KF and j0 < K_ZONE0) or b1 > K_BEST_MAX or b1 > j0
    out.update(flagged=bool(flagged), m=m, j0=j0, b1=b1,
               lane_full=any(not key_value([o])[0] > lim for o in own_last) and not fast)
    return out


def select_model(d2_exact, d2f, size=1.0, chunks=None, lbs=None, lpk=LPK, nls=NLS, fast=False, ids=None):
    """Returns (flagged, chosen candidate indices (set), nearest candidate index).  d2_exact: float64 exact squared
    distances; d2f: float32 values the kernel would have computed; chunks: list of index arrays visited in order
    ("voxels") with lower bounds lbs (float32) used for the skip rule; default: one chunk, no skipping.  lpk / nls:
    lanes per keypoint and keys per lane of k1_scan (4 / 14 and 2 / 20 are compiled); fast=True: k1_fast."""
    v = scan_verdict(d2f, size, chunks, lbs, lpk, nls, fast, ids)
    if v["flagged"]:
        return True, None, None
    m, j0, b1 = v["m"], v["j0"], v["b1"]
    slot_ids = v["slot_cand"].astype(np.int64)
    chosen = list(slot_ids[:j0])
    zone = slot_ids[j0:m]
    if m > KF:
        order = sorted(zone, key=lambda i: (d2_exact[i], i))      # exact (distance^2, visit id)
        chosen += order[:KF - j0]
    else:
        chosen += list(zone)
    near = min(slot_ids[:b1], key=lambda i: (d2_exact[i], i))
    return False, set(int(c) for c in chosen), int(near)


def exact_answer(d2_exact):
    order = sorted(range(d2_exact.shape[0]), key=lambda i: (d2_exact[i], i))
    return set(order[:KF]), order[0]


def adversarial_set(rng, kind, n):
    """Squared distances (float64, units of size^2 with size = 1) with trouble around the K-th."""
    base = np.sort(rng.uniform(0.01, 2.0, n))
    if kind == "near_ties":                       # candidates 15..30 within 1e-7 .. 1e-3 of each other
        gap = 10.0 ** rng.uniform(-8, -3)
        base[15:30] = base[15] + gap * np.arange(15)
    elif kind == "cluster":                       # many points at (almost) the same distance as the K-th
        w = 10.0 ** rng.uniform(-9, -4)
        k = rng.integers(10, 40)
        base[KF - 5:KF - 5 + k] = base[KF - 5] + rng.uniform(0, w, k)
    elif kind == "duplicates":                    # exact ties in the exact distance
        base[18:24] = base[18]
        base[0:3] = base[0]
    elif kind == "tiny":                          # all very close to the keypoint: relative window dominates nothing
        base *= 1e-4
    elif kind == "nearest_tie":
        base[0:6] = base[0] + 10.0 ** rng.uniform(-9, -5) * np.arange(6)
    return rng.permutation(base)


@pytest.mark.parametrize("kind", ["random", "near_ties", "cluster", "duplicates", "tiny", "nearest_tie"])
def test_certified_answers_are_exact(kind):
    rng = np.random.default_rng(sum(map(ord, kind)))
    eps = 1e-4
    certified = 0
    for trial in range(400):
        n = int(rng.integers(64, 400))
        d2 = adversarial_set(rng, kind, n)
        # FP32 values at the assumed error bound (DESIGN: |d2f - d2| <= 1e-4 size^2), adversarial sign pattern
        noise = rng.choice([-1.0, 1.0, 0.0], n) * eps * rng.choice([1.0, 0.999, 0.5, 0.0], n)
        d2f = np.maximum(d2 + noise, 0.0).astype(np.float32)
        flagged, chosen, near = select_model(d2, d2f)
        want_set, want_near = exact_answer(d2)
        if not flagged:
            certified += 1
            assert chosen == want_set, (kind, trial)
            assert near == want_near, (kind, trial)
    if kind == "random":
        assert certified >= 300                    # the certificate is not vacuous: ordinary inputs pass it
    if kind == "tiny":
        assert certified == 0                      # distances of the order of the FP32 error: everything goes the exact way


FORMS = {"scan4": dict(lpk=4, nls=14), "scan2": dict(lpk=2, nls=20), "fast1": dict(lpk=1, fast=True),
         "fast2": dict(lpk=2, fast=True), "fast4": dict(lpk=4, fast=True)}


@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("kind", ["random", "near_ties", "cluster", "nearest_tie"])
def test_certified_answers_are_exact_on_every_form(kind, form):
    """The same attack on every compiled lane layout: k1_scan with 2 lanes of 20 keys, k1_fast with 1, 2 or 4 lanes of
    NL keys and the certifier alone."""
    rng = np.random.default_rng(sum(map(ord, kind + form)))
    certified = 0
    for trial in range(200):
        n = int(rng.integers(64, 400))
        d2 = adversarial_set(rng, kind, n)
        noise = rng.choice([-1.0, 1.0, 0.0], n) * 1e-4 * rng.choice([1.0, 0.999, 0.5, 0.0], n)
        d2f = np.maximum(d2 + noise, 0.0).astype(np.float32)
        flagged, chosen, near = select_model(d2, d2f, **FORMS[form])
        want_set, want_near = exact_answer(d2)
        if not flagged:
            certified += 1
            assert chosen == want_set and near == want_near, (kind, form, trial)
    if kind == "random":
        assert certified >= 150


def test_lane_certificate_counts_what_one_lane_holds():
    """k1_scan deals a voxel's point i to lane i % LPK: when the K nearest crowd into one lane, that lane's list of NLS keys
    is full inside the window and the keypoint is flagged (it cannot tell whether it dropped one), one fewer and it is
    certified."""
    for lpk, nls in ((4, 14), (2, 20)):
        for in_lane in (nls - 1, nls, nls + 1):
            if in_lane > KF:
                continue
            near = np.linspace(0.05, 0.3, KF)                     # the K nearest; everything else lies far outside the window
            order = np.random.default_rng(in_lane).permutation(KF)
            d2 = np.full(80, 0.8) + np.arange(80) * 1e-3
            lane0 = np.arange(0, 80, lpk)
            others = np.setdiff1d(np.arange(80), lane0)
            d2[lane0[:in_lane]] = near[order[:in_lane]]
            d2[others[:KF - in_lane]] = near[order[in_lane:]]
            v = scan_verdict(d2.astype(np.float32), lpk=lpk, nls=nls, chunks=np.split(np.arange(80), 4),
                             lbs=np.zeros(4, np.float32))
            assert v["lane_full"] == (in_lane >= nls) and v["flagged"] == (in_lane >= nls), (lpk, nls, in_lane)


def test_voxel_skip_never_drops_a_true_neighbour():
    """Candidates arrive voxel by voxel with a lower bound per voxel; voxels are skipped once the bound exceeds the
    group's threshold.  Whatever is certified must still be the exact answer."""
    rng = np.random.default_rng(99)
    eps = 1e-4
    certified = skipped_any = 0
    for trial in range(400):
        n_vox = int(rng.integers(3, 20))
        sizes = rng.integers(1, 21, n_vox)
        lo = np.sort(rng.uniform(0.0, 3.0, n_vox))               # voxels come nearest first, roughly
        d2_parts = [lo[v] + rng.uniform(0, 0.6, sizes[v]) for v in range(n_vox)]
        d2 = np.concatenate(d2_parts)
        if d2.shape[0] < KF + 2:
            continue
        idx = np.split(np.arange(d2.shape[0]), np.cumsum(sizes)[:-1])
        lbs = np.array([max(min(p) * 0.999999 - 1e-5, 0.0) for p in d2_parts], np.float32)   # conservative, like the kernel's
        noise = rng.uniform(-eps, eps, d2.shape[0])
        d2f = np.maximum(d2 + noise, 0.0).astype(np.float32)
        flagged, chosen, near = select_model(d2, d2f, chunks=idx, lbs=lbs)
        flagged0, chosen0, _ = select_model(d2, d2f)
        want_set, want_near = exact_answer(d2)
        if not flagged:
            certified += 1
            assert chosen == want_set and near == want_near, trial
        if not flagged and not flagged0 and chosen0 == chosen:
            skipped_any += 1
    assert certified > 200


def test_fp32_distance_error_stays_inside_the_assumed_bound():
    """The kernel computes d2f = sum(((m - of) - rf)^2) in FP32 with of = float(corner of the keypoint's voxel),
    rf = float(p - of).  DESIGN.md bounds |d2f - d2| by 1e-4 size^2 for candidates up to nb = 2 voxels away."""
    rng = np.random.default_rng(5)
    for size in (0.5, 1.0, 2.0):
        worst = 0.0
        for _ in range(200):
            k = rng.integers(-300, 300, 3).astype(np.float64)
            corner = k * size
            p = corner + rng.uniform(0, size, 3) * np.sign(k + 0.5)          # inside its (truncation) voxel
            m32 = (corner[None, :] + rng.uniform(-2.0 * size, 3.0 * size, (500, 3))).astype(np.float32)
            of = corner.astype(np.float32)
            rf = (p - of.astype(np.float64)).astype(np.float32)
            d = (m32 - of[None, :]) - rf[None, :]
            d2f = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]).astype(np.float32) + d[:, 2] * d[:, 2]
            dd = m32.astype(np.float64) - p[None, :]
            d2 = dd[:, 0] ** 2 + (dd[:, 1] ** 2 + dd[:, 2] ** 2)
            worst = max(worst, float(np.abs(d2f.astype(np.float64) - d2).max()))
        assert worst <= 1e-4 * size * size, (size, worst)
        assert worst <= 0.5e-4 * size * size                                  # in fact with a margin of 2


# ---- distortFrameByImu: the parallel formulation of the reference's one-iterator walk (srl_points.cu) ---------------
def _imu_walk_parallel(tp, ts):
    """What srl_distort_frame_by_imu computes: f_i / l_i = first / last interval holding point i (the reference's
    comparisons), n_i = max(f_0..f_i), valid while n_i <= l_i; returns (interval per point, number of points written)."""
    n, ns = tp.shape[0], ts.shape[0]
    inside = (tp[:, None] > ts[None, :-1] - 1e-6) & (tp[:, None] < ts[None, 1:] + 1e-6)
    any_in = inside.any(axis=1)
    f = np.where(any_in, inside.argmax(axis=1), ns)
    l = np.where(any_in, ns - 2 - inside[:, ::-1].argmax(axis=1), -1)
    m = np.maximum.accumulate(f)
    bad = (m >= ns) | (m > l)
    v = int(np.argmax(bad)) if bad.any() else n
    return m, v


def _imu_walk_reference(tp, ts):
    """The loop of src/utility.cpp:238-312 reduced to its control flow."""
    n, ns = tp.shape[0], ts.shape[0]
    used = np.full(n, -1)
    it = 0
    for k in range(ns - 1):
        while it != n:
            if tp[it] > ts[k] - 1e-6 and tp[it] < ts[k + 1] + 1e-6:
                used[it] = k
                it += 1
            else:
                break
    return used, it


def test_imu_interval_walk_parallel_form_equals_the_iterator():
    rng = np.random.default_rng(17)
    for trial in range(600):
        ns = int(rng.integers(2, 30))
        ts = 100.0 + np.cumsum(rng.choice([0.005, 0.005, 0.0049, 0.0, 0.01], ns))       # non-decreasing, repeated stamps allowed
        n = int(rng.integers(1, 200))
        tp = np.sort(rng.uniform(ts[0] - 0.002, ts[-1] + 0.002, n))
        mode = trial % 4
        if mode == 1:        # points exactly on / within the 1e-6 tolerance of IMU stamps
            j = rng.integers(0, n, min(n, 10))
            tp[j] = ts[rng.integers(0, ns, j.shape[0])] + rng.choice([0.0, 5e-7, -5e-7, 1e-6, -1e-6], j.shape[0])
            tp = np.sort(tp)
        elif mode == 2:      # locally unsorted
            j = rng.integers(0, n, 3)
            tp[j] = rng.uniform(ts[0] - 0.002, ts[-1] + 0.002, 3)
        elif mode == 3:      # everything inside
            tp = np.sort(rng.uniform(ts[0], ts[-1], n))
        used, it = _imu_walk_reference(tp, ts)
        m, v = _imu_walk_parallel(tp, ts)
        assert v == it, (trial, v, it)
        assert np.array_equal(m[:v], used[:it]), trial


def test_grid_sampling_order_survives_the_dedupe():
    """srl_grid_sampling keeps the first point of every cell on the GPU and replays only those through the reference's
    std::tr1::unordered_map: duplicates never change the container's structure, so the iteration order is the same."""
    from oracle import oracle_py as O
    rng = np.random.default_rng(23)
    for size, spread, n in ((0.5, 6.0, 20000), (1.5, 40.0, 30000), (0.2, 1.0, 5000)):
        pts = rng.normal(0, spread, (n, 3))
        keep_all = O.grid_sampling(pts, size)
        cells = np.trunc(pts / size).astype(np.int64)          # static_cast<short>(x / size): truncation toward zero
        _, first = np.unique(cells, axis=0, return_index=True)
        first = np.sort(first)                                 # first occurrence of every cell, frame order
        keep_u = O.grid_sampling(pts[first], size)
        assert np.array_equal(first[keep_u], keep_all)
