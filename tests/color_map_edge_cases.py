"""Seeded cases at the edges of the colour map's insertion (addPointToColorMap and its driver loop): keys at voxel and
fine-cell faces, cell 0, the int16 wrap, aliases and the int32 limit; block capacity and the fine set; add_point_step; the
two time gates at their 1e-5 tolerance; the recent lists over rendering and non-rendering calls; a long run of sweeps
without an image; and the fine set's probe chains across its growth.

A case is a sequence of calls on one colour map, each (world_xyz, kw) with kw the arguments of addPoints: add_point_step,
time_sweep_end, time_last_process, to_rendering.  Every builder asserts the property that defines its case while it builds
it, mostly by replaying the plain restatement (tests/color_map_reference.py); `expect` names the restatement's events the
case must reach.  Ties in double arithmetic are certified with Fraction.
"""
from __future__ import annotations

import functools
import math
from dataclasses import dataclass
from fractions import Fraction

import numpy as np

from color_map_reference import TIME_GATE, ColorMapRef
from map_edge_cases import chain_keys
from map_reference import f32, hash_key, short_key, voxel_of

SIZE, FINE = 0.1, 0.01
I32 = 2.0 ** 31
BIG_STEP = 2 ** 31 - 1


@dataclass
class Case:
    name: str
    calls: list
    size: float = SIZE
    fine: float = FINE
    cap: int = 50
    max_voxels: int = 4096
    initial_voxels: int = 1          # the growable map's start; the fixed map commits max_voxels
    expect: tuple = ()               # restatement events the case reaches


def call(xyz, t_end=1.0, t_last=0.0, render=True, step=1):
    return (np.asarray(xyz, np.float64).reshape(-1, 3),
            dict(add_point_step=int(step), time_sweep_end=float(t_end), time_last_process=float(t_last), to_rendering=bool(render)))


def replay(case: Case) -> ColorMapRef:
    m = ColorMapRef(case.size, case.cap, case.fine)
    for xyz, kw in case.calls:
        m.add_points(xyz, **kw)
    return m


def wrap16(k: int) -> int:
    return ((k + 0x8000) & 0xFFFF) - 0x8000


def dnext(x: float, k: int = 1) -> float:
    for _ in range(abs(k)):
        x = math.nextafter(x, math.inf if k > 0 else -math.inf)
    return x


def fstep(x: float, toward: float) -> float:
    return float(np.nextafter(np.float32(x), np.float32(toward)))


def face_pair(k: int, size: float):
    """The two adjacent floats around the face where double(float(x)) / size reaches the integer k > 0: trunc gives k - 1
    at the first and k at the second."""
    assert k > 0
    x = f32(k * size)
    while x / size >= k:
        x = fstep(x, 0.0)
    while fstep(x, math.inf) / size < k:
        x = fstep(x, math.inf)
    hi = fstep(x, math.inf)
    assert short_key(x / size) == wrap16(k - 1) and short_key(hi / size) == wrap16(k), (k, size)
    return x, hi


def cell_point(key, size: float):
    """A position inside the cell `key` of a grid of `size` (truncation: cell 0 is (-size, size))."""
    p = tuple((k + (0.5 if k >= 0 else -0.5)) * size for k in key)
    assert voxel_of(tuple(f32(c) for c in p), size) == tuple(key), (key, size)
    return p


# ---- cells ------------------------------------------------------------------------------------------------------------
def _face_points(size: float, ks, inner):
    """For every face k (and -k) of a grid and every axis: the floats either side of it, the other axes at `inner`."""
    out = []
    for k in ks:
        lo, hi = face_pair(k, size)
        for sgn in (1.0, -1.0):
            for axis in range(3):
                for v in (lo, hi):
                    p = list(inner)
                    p[axis] = sgn * v
                    out.append(p)
    return out


def cell_cases() -> list[Case]:
    out = []
    for md in (0.01, 0.1, 0.03, 0.15):
        rng = np.random.default_rng(int(md * 1000))
        inner = (0.0433, -0.0271, 0.0617)
        pts = _face_points(SIZE, (1, 2, 7), inner) + _face_points(md, (1, 3, 10), inner)
        pts += [[s * 0.3 * md, s * 0.7 * SIZE, 0.0] for s in (1.0, -1.0)] + [[-0.0, 1e-30, -1e-30], [0.7 * SIZE, -0.7 * SIZE, 0.45 * md]]
        wrap = _face_points(SIZE, (32767, 32768, 32769), inner) + _face_points(md, (32767, 32768, 32769), inner)
        # aliases: 2^16 cells apart share a key (655.36 m of 0.01 m cells, 6553.6 m of 0.1 m voxels)
        base = [0.2345, 0.4567, 0.1234]
        alias = [base, [base[0] + 6553.6, base[1], base[2]], [base[0], base[1] + 65536 * md, base[2]]]
        a = [tuple(f32(c) for c in p) for p in alias]
        assert voxel_of(a[0], SIZE) == voxel_of(a[1], SIZE) and a[0] != a[1]
        assert voxel_of(a[0], md) == voxel_of(a[2], md) and (md == SIZE or voxel_of(a[0], SIZE) != voxel_of(a[2], SIZE))
        groups = [np.array(pts), np.array(wrap), np.array(alias)]
        expect = ["stored_in_claimed_cell"]
        if md in (0.03, 0.15):
            # fine cells that straddle a voxel face: x in [3 md, 4 md) spans voxels 0 and 1 at md 0.03, [md, 2 md) spans 1
            # and 2 at 0.15.  The later point (another voxel) is stored but its cell is taken.
            x0, x1 = (0.105, 0.095) if md == 0.03 else (0.25, 0.17)
            s = [(x0, 0.01, 0.01), (x1, 0.012, 0.011)]
            fs = [tuple(f32(c) for c in p) for p in s]
            assert voxel_of(fs[0], md) == voxel_of(fs[1], md) and voxel_of(fs[0], SIZE) != voxel_of(fs[1], SIZE)
            groups.append(np.array(s))
        xyz = np.concatenate(groups)
        first = xyz[rng.permutation(xyz.shape[0])]
        second = xyz[rng.permutation(xyz.shape[0])]
        out.append(Case(f"cells_md{md}", [call(first, 1.0, 0.0), call(second, 2.0, 1.0)], fine=md, cap=20, expect=tuple(expect)))
    return out


def _size_for_quotient(x: float, q: float) -> float:
    """A double size with fl(x / size) == q exactly (searched around x / q)."""
    s = x / q
    for k in range(-8, 9):
        c = dnext(s, k)
        if x / c == q:
            return c
    raise AssertionError((x, q))


def int32_cases() -> list[Case]:
    below = dnext(I32, -1)                             # the last double below 2^31
    x = 2147483520.0                                   # the last float below 2^31
    assert f32(x) == x and f32(dnext(x, 1)) != dnext(x, 1)
    s = _size_for_quotient(x, below)
    kept = [[x, 0.5, 0.5], [-x, 0.5, 0.5], [0.5, x, -x]]
    for p in kept:
        for c in p:
            assert abs(c / s) < I32
    assert x / s == below and short_key(x / s) == -1 and short_key(-x / s) == 1
    # q = 2^31 exactly (size 1, x = +-2^31) and beyond: dropped, like NaN and +-inf
    assert I32 / 1.0 == I32 and short_key(I32) is None and short_key(-I32) is None and short_key(below) == -1
    ok = [[0.25, 0.5, 4.0], [1.5, -2.5, 4.0], [-3.5, 0.5, 4.0]]
    bad1 = [[I32, 0.5, 4.0], [0.5, -I32, 4.0], [float("nan"), 0.5, 4.0], [0.5, float("inf"), 4.0], [0.5, 0.5, -float("inf")]]
    one = np.array(ok + bad1 + [[below, 0.5, 4.0]])      # below rounds to the float 2^31: dropped too
    assert f32(below) == I32
    return [Case("int32_last_below_2p31", [call(np.array(kept + ok)), call(np.array(kept), 2.0, 1.0)], size=s, fine=s, cap=4),
            Case("int32_at_2p31_nan_inf", [call(one), call(one[::-1], 2.0, 1.0)], size=1.0, fine=1.0, cap=4, expect=("dropped",))]


# ---- capacity and the fine set -----------------------------------------------------------------------------------------
def _distinct_cells(vkey, n, rng, md=FINE, size=SIZE):
    """n points of voxel vkey in n distinct fine cells (md divides the voxel into at least n cells)."""
    per = int(round(size / md))
    cells = rng.permutation(per ** 3)[:n]
    sgn = np.where(np.asarray(vkey) < 0, -1.0, 1.0)
    out = []
    for c in cells.tolist():
        i, j, k = c // (per * per), (c // per) % per, c % per
        local = (np.array([i, j, k]) + 0.3 + 0.4 * rng.random(3)) * md
        out.append(np.asarray(vkey) * size + sgn * local)
    pts = np.array(out)
    fp = [tuple(f32(c) for c in p) for p in pts]
    assert all(voxel_of(p, size) == tuple(vkey) for p in fp) and len({voxel_of(p, md) for p in fp}) == n
    return pts


def cap_cases() -> list[Case]:
    out = []
    for cap in (1, 2, 20, 21, 50, 100, 128):
        rng = np.random.default_rng(100 + cap)
        A, B = (3, 2, 40), (4, 2, 40)
        a = _distinct_cells(A, cap + 2, rng)
        b = _distinct_cells(B, cap + 2, rng)
        first = np.concatenate([a[:cap - 1], b])                # A one short of full, B fills mid-call
        first = first[rng.permutation(first.shape[0])]
        second = np.concatenate([a[cap - 1:], b[cap:], first[:3]])   # A's last slot, then refusals; re-offered cells
        c = Case(f"cap_{cap}", [call(first, 1.0, 0.0), call(second, 2.0, 1.0)], cap=cap,
                 expect=("refused", "index_cap_minus_1", "listed_without_a_stored_point"))
        m = replay(c)
        assert len(m.vox[A].pts) == cap and len(m.vox[B].pts) == cap
        assert any(r[:3] == A and r[3] == cap - 1 for r in m.rgb)
        out.append(c)
    # 200 points in one fine cell
    rng = np.random.default_rng(7)
    one = np.array([0.0412, 0.0523, 4.0347]) + rng.uniform(0.0, 0.0006, (200, 3))
    assert len({voxel_of(tuple(f32(v) for v in p), FINE) for p in one}) == 1
    c = Case("cap_128_one_cell_200_points", [call(one)], cap=128, expect=("refused", "stored_in_claimed_cell"))
    m = replay(c)
    assert m.num_points == 128 and len(m.rgb) == 1
    out.append(c)
    # a full voxel refuses a point in a free cell that straddles a voxel face; a later point in the same cell but in the
    # next voxel claims it, in the same call; a cell claimed in an earlier call stays claimed
    for md, fill, refused, claim in ((0.03, (0.02, 0.05), 0.095, 0.105), (0.15, (0.11, 0.14), 0.17, 0.25)):
        y, z = 0.0137, 0.0219
        fp = lambda x: tuple(f32(v) for v in (x, y, z))
        assert voxel_of(fp(refused), md) == voxel_of(fp(claim), md) and voxel_of(fp(refused), SIZE) != voxel_of(fp(claim), SIZE)
        assert voxel_of(fp(refused), md) not in {voxel_of(fp(f), md) for f in fill}
        calls = [call([(f, y, z) for f in fill], 1.0, 0.0),
                 call([(refused, y, z), (claim, y, z), (claim + 0.004, y, z)], 2.0, 1.0),
                 call([(claim + 0.002, y + 0.001, z), (fill[0] + 0.001, y, z)], 3.0, 2.0)]
        c = Case(f"refused_cell_claimed_across_voxels_md{md}", calls, fine=md, cap=2,
                 expect=("cell_claimed_after_refusal", "cell_won_across_voxels", "stored_in_claimed_cell", "listed_without_a_stored_point"))
        m = replay(c)
        assert m.rgb[-1] == voxel_of(fp(claim), SIZE) + (0,) and len(m.vox[voxel_of(fp(refused), SIZE)].pts) == 2
        out.append(c)
    return out


# ---- add_point_step ----------------------------------------------------------------------------------------------------
def step_cases() -> list[Case]:
    out = []
    n = 50
    rng = np.random.default_rng(11)
    pts = np.concatenate([_distinct_cells(k, n // 2, rng) for k in ((0, 0, 40), (1, 0, 40))])
    pts = pts[rng.permutation(n)]
    dirty = pts.copy()
    dirty[0] = [np.nan, 0.0, 4.0]                    # selected by every step
    dirty[1] = [0.0, np.inf, 4.0]                    # selected by step 1 only
    dirty[14] = [3e9, 0.0, 4.0]                      # |q| >= 2^31; selected by steps 1, 2 and 7
    for step in (1, 2, 3, 7, n - 1, n, n + 1, BIG_STEP):
        c = Case(f"step_{step}", [call(dirty, 1.0, 0.0, step=step), call(pts[::-1], 2.0, 1.0, step=step)], expect=("dropped",))
        m = replay(c)
        assert m.events["dropped"] == sum(1 for i in (0, 1, 14) if i % step == 0)
        out.append(c)
    tiny = [call(np.zeros((0, 3)), 1.0, 0.0), call(pts[:1], 2.0, 1.0), call(pts[:2], 3.0, 2.0, render=False, step=2),
            call(pts[2:4], 4.0, 3.0), call(np.zeros((0, 3)), 5.0, 4.0, render=False), call(pts[4:5], 6.0, 5.0, step=3),
            call(np.zeros((0, 3)), 7.0, 6.0)]
    out.append(Case("calls_of_0_1_2_points", tiny))
    return out


# ---- time gates and the lists ------------------------------------------------------------------------------------------
def _voxels(rng, keys, per=2):
    return np.concatenate([_distinct_cells(k, per, rng) for k in keys])


def _exact_tie(lo_start: float) -> tuple[float, float]:
    """(a, a + 1e-5) with the sum exact in double, a searched upward from lo_start."""
    a = lo_start
    for _ in range(64):
        b = a + TIME_GATE
        if Fraction(b) - Fraction(a) == Fraction(TIME_GATE):
            return a, b
        a = dnext(a)
    raise AssertionError(lo_start)


def time_cases() -> list[Case]:
    out = []
    rng = np.random.default_rng(21)
    old = [(i, 0, 40) for i in range(4)]
    new = lambda c: [(i, 5 + c, 40) for i in range(2)]
    # fabs(t_end - t_last_process) at 1e-5: the tie and one double either side, on the same voxels and on new ones
    t_last, tie = _exact_tie(2.0 ** -20)
    assert tie - t_last == TIME_GATE and tie > TIME_GATE                     # new voxels pass the other gate
    below, above = dnext(tie, -1), dnext(tie, 1)
    assert below - t_last == dnext(TIME_GATE, -1) and above - t_last == dnext(TIME_GATE, 1)
    calls = [call(_voxels(rng, old + new(0)), tie, t_last), call(_voxels(rng, old + new(1)), below, t_last),
             call(_voxels(rng, old + new(2)), above, t_last)]
    c = Case("gate_process_time_at_1e-5", calls, expect=("gate_within_one_double",))
    m = replay(c)
    assert m.events["listed"] == len(m.recent) == len(old) + 2                          # only the last call lists
    out.append(c)
    # fabs(last_visited - t_end) at 1e-5 across calls: three groups of voxels visited at a - 1 ulp, a and a + 1 ulp (one
    # double of 1e-5's binade each), then all three at t_end = a + 1e-5
    a, b = _exact_tie(1.2e-5)
    assert a > TIME_GATE and b - a == TIME_GATE
    assert Fraction(b) - Fraction(dnext(a, -1)) == Fraction(dnext(TIME_GATE, 1))
    assert Fraction(b) - Fraction(dnext(a, 1)) == Fraction(dnext(TIME_GATE, -1))
    groups = [[(i, g, 40) for i in range(3)] for g in range(3)]
    calls = [call(_voxels(rng, groups[0]), dnext(a, -1), -1.0, render=False), call(_voxels(rng, groups[1]), a, -1.0),
             call(_voxels(rng, groups[2]), dnext(a, 1), -1.0), call(_voxels(rng, sum(groups, [])), b, -1.0)]
    c = Case("gate_last_visited_at_1e-5", calls, cap=20, expect=("gate_within_one_double",))
    m = replay(c)
    assert m.recent == groups[0] and m.vox[groups[0][0]].last_visited == b and m.vox[groups[1][0]].last_visited == a
    out.append(c)
    # t_end within 1e-5 of 0: new voxels start at last_visited 0.0 and are never listed; exactly 1e-5 neither; one above is
    calls = [call(_voxels(rng, old), 5e-6, -1.0), call(_voxels(rng, old + new(0)), TIME_GATE, -1.0),
             call(_voxels(rng, new(1)), dnext(TIME_GATE, -1), -1.0), call(_voxels(rng, new(2)), dnext(TIME_GATE, 1), -1.0),
             call(_voxels(rng, old), -5e-6, -1.0)]
    c = Case("sweep_end_near_zero", calls, expect=("gate_within_one_double",))
    m = replay(c)
    assert m.events["listed"] == 2 and len(m.recent) == 0
    out.append(c)
    # negative, NaN and infinite times
    seq = [(-2.5, -3.0), (float("nan"), 0.0), (1.0, float("nan")), (float("inf"), 0.0), (float("inf"), 1.0), (-float("inf"), 0.0),
           (5.0, float("inf")), (5.0, 0.0), (-5.0, -5.0)]
    calls = [call(_voxels(rng, old + new(i)), te, tl) for i, (te, tl) in enumerate(seq)]
    c = Case("times_negative_nan_inf", calls)
    m = replay(c)
    assert any(blk.last_visited == -math.inf for blk in m.vox.values()) and any(blk.last_visited == 5.0 for blk in m.vox.values())
    out.append(c)
    return out


def sequence_cases() -> list[Case]:
    """R = a rendering call, N = one without; every call offers points in old voxels and in new ones, and the sweep's last
    point is alone in a new voxel, which is therefore listed last."""
    out = []
    old = [(i, 1, 40) for i in range(5)]
    for name, seq in (("R", [(1.0, "R")]), ("RR_same_end", [(1.0, "R"), (1.0, "R")]), ("NR_same_end", [(1.0, "N"), (1.0, "R")]),
                      ("RNN", [(1.0, "R"), (2.0, "N"), (3.0, "N")]), ("NNNNR", [(1.0, "N"), (2.0, "N"), (3.0, "N"), (4.0, "N"), (5.0, "R")]),
                      ("NRNR", [(1.0, "N"), (2.0, "R"), (3.0, "N"), (3.0, "R")])):
        rng = np.random.default_rng(len(out) + 31)
        calls = []
        for i, (t, kind) in enumerate(seq):
            body = _voxels(rng, old + [(i, 6, 40), (i + 1, 6, 40)], per=3)
            body = body[rng.permutation(body.shape[0])]
            last = _distinct_cells((i, 9, 40), 1, rng)
            calls.append(call(np.concatenate([body, last]), t, t - 0.5, render=kind == "R"))
        c = Case(f"sequence_{name}", calls, cap=8)
        m = ColorMapRef(c.size, c.cap, c.fine)
        published = None
        for i, (xyz, kw) in enumerate(calls):
            m.add_points(xyz, **kw)
            if kw["to_rendering"]:
                published = (list(m.recent), m.new_recent)
                if m.recent:
                    assert m.recent[-1] == (i, 9, 40)          # the voxel of the sweep's last point comes last
            else:
                assert published is None or (m.recent, m.new_recent) == published   # N changes nothing that is published
        out.append(c)
    return out


# ---- the no-image run --------------------------------------------------------------------------------------------------
NO_IMAGE_VOXELS = 1024
NO_IMAGE_CALLS = 12


def no_image_cases() -> list[Case]:
    """1024 voxels (the map's limit) visited by every call, distinct sweep ends, twelve calls without rendering and then one
    with.  Before a call without rendering stopped appending to the recent list, the list (4 * 1024 + 1024 entries) was
    exactly full after five such calls and the sixth failed with SRL_MAP_FULL."""
    rng = np.random.default_rng(41)
    keys = [(i, j, 40) for i in range(32) for j in range(32)]
    calls = []
    for c in range(NO_IMAGE_CALLS + 1):
        pts = np.concatenate([_distinct_cells(k, 1, rng) for k in keys])
        pts = pts[rng.permutation(pts.shape[0])]
        t = 1.0 + 0.1 * c
        calls.append(call(pts, t, t - 0.05, render=c == NO_IMAGE_CALLS))
    case = Case("no_image_run", calls, cap=1, max_voxels=NO_IMAGE_VOXELS, expect=("listed_without_a_stored_point",))
    m = ColorMapRef(case.size, case.cap, case.fine)
    for c, (xyz, kw) in enumerate(calls):
        m.add_points(xyz, **kw)
        if c == 4:
            assert len(m.recent_temp) == 4 * NO_IMAGE_VOXELS + 1024
        if c == 5:
            assert len(m.recent_temp) > 4 * NO_IMAGE_VOXELS + 1024
    assert len(m.vox) == NO_IMAGE_VOXELS and len(m.recent) == NO_IMAGE_VOXELS == m.new_recent
    return [case]


# ---- growth ------------------------------------------------------------------------------------------------------------
def growth_cases() -> list[Case]:
    """Fine cells whose home slot is one of the last four under both mask 1023 and 2047, claimed while the fine table has
    1024 slots (rgb points committed <= 512) and after it has doubled; fillers in distinct cells push the rgb count past
    512 in the second call.  The growable map starts from one voxel (50 committed rgb points)."""
    near, far = chain_keys()
    assert all(chained(k) for k in near + far)
    near_pts = np.array([cell_point(k, FINE) for k in near])
    far_pts = np.array([cell_point(k, FINE) for k in far])
    fill = lambda z: np.array([cell_point((5 * i, 5 * j, z), FINE) for i in range(25) for j in range(10)])
    rng = np.random.default_rng(51)
    first = np.concatenate([near_pts, fill(-200)])
    second = np.concatenate([far_pts, fill(-300)])
    c = Case("fine_chain_across_growth", [call(first[rng.permutation(first.shape[0])], 1.0, 0.0),
                                          call(second[rng.permutation(second.shape[0])], 2.0, 1.0)])
    m = ColorMapRef(c.size, c.cap, c.fine)
    m.add_points(*c.calls[0][:1], **c.calls[0][1])
    assert 256 < len(m.rgb) <= 512
    m.add_points(*c.calls[1][:1], **c.calls[1][1])
    assert len(m.rgb) > 512 and len(m.rgb) == 700
    # the chained cells are the ones the points fall in, and each claims its cell: 100 on either side of the growth
    for (xyz, _), keys in zip(c.calls, (near, far)):
        cells = {voxel_of(tuple(f32(v) for v in p), FINE) for p in xyz}
        assert set(keys) <= cells and sum(chained(k) for k in cells) >= len(keys) == 100
    claimed = {voxel_of(tuple(f32(v) for v in m.vox[r[:3]].pts[r[3]]), FINE) for r in m.rgb}
    assert set(near + far) <= claimed
    return [c]


def chained(cell) -> bool:
    """The cell's home slot is one of the last four of a 1024-slot and of a 2048-slot table: its probe chain wraps."""
    h = hash_key(*cell)
    return h & 1023 >= 1020 and h & 2047 >= 2044


@functools.lru_cache(maxsize=None)
def _all() -> tuple:
    return tuple(cell_cases() + int32_cases() + cap_cases() + step_cases() + time_cases() + sequence_cases() + no_image_cases()
                 + growth_cases())


def all_cases() -> list[Case]:
    return list(_all())


def feed_for_reference(xyz, kw, case: Case):
    """(points, kw) for the oracle and the compiled reference: their static_cast<short> is undefined for NaN, +-inf and
    |q| >= 2^31, so the call's selected points go without those and with step 1, which selects the same points."""
    f = np.asarray(xyz, np.float64).reshape(-1, 3)
    ok = [all(voxel_of(tuple(f32(c) for c in row), s) is not None for s in (case.size, case.fine)) for row in f.tolist()]
    if all(ok):
        return f, kw
    sel = np.zeros(f.shape[0], bool)
    sel[::kw["add_point_step"]] = True
    return f[sel & np.asarray(ok, bool)], dict(kw, add_point_step=1)
