"""Seeded inputs of the iterated ESIKF update that no pass over a rich street scene produces: dense correlated covariances
(kappa(P) = 1e3 ... 1e12), a covariance carried through 20 corridor updates, an exactly singular covariance, normal
equations of rank 6 / 5 (corridor) / 3 (ground plane) at magnitudes 1e0 ... 1e10, 6x6 systems that force the device's
Gauss-Jordan inverse off the diagonal pivot order, updates aimed at the branch points of the manifold helpers and the
divergence guard, and multi-pass sequences whose later passes see a real offset from the prediction (gravity included,
with 1 - dot on both sides of 1e-6).

A case is given the way the loop receives it: a start state and one block of 32 sums per pass (DESIGN §3 layout).
`host_loop()` runs the product's host algebra (srl_iekf_begin / srl_iekf_step) on those blocks with the status checks
srl_update_iekf makes before every step, and records the exact FP64 input of every step.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from sr_livo_b200 import capi, synth

N = 17
LASER_COV = 0.001


@dataclass
class Case:
    name: str
    state: dict                           # p q v ba bg g cov
    blocks: np.ndarray                    # (n_pass, 32)
    prm: dict = field(default_factory=dict)   # srl_icp_params overrides
    kappa_class: str = "diag"


# ---- sums ---------------------------------------------------------------------------------------------------------------
def pack32(HTH, HTh, n_res=1000, nan_count=0):
    b = np.zeros(32)
    HTH = np.asarray(HTH, np.float64)
    k = 0
    for a in range(6):
        for c in range(a, 6):
            b[k] = HTH[a, c]
            k += 1
    b[21:27] = HTh
    b[27] = 0.0
    b[28] = n_res
    b[29] = n_res
    b[31] = nan_count
    return b


def unpack32(b):
    ne = capi.NormalEq()
    blk = np.ascontiguousarray(b, np.float64)
    assert capi.lib().srl_normal_eq_unpack(capi.ptr(blk), C.byref(ne)) == 0
    return ne


def jacobian_rows(kind: str, rng, n=400):
    """Rows [n, x cross n] of point-to-plane residuals (the Jacobian of src/optimize.cpp:57-61 up to the rotation)."""
    if kind == "rank6":
        nrm = rng.normal(size=(n, 3))
        x = rng.uniform(-20, 20, size=(n, 3))
    elif kind == "corridor":   # walls y = +-2, floor z = 0, ceiling z = 3: no normal has an x component
        side = rng.integers(0, 4, n)
        nrm = np.zeros((n, 3))
        nrm[side == 0, 1] = 1; nrm[side == 1, 1] = -1; nrm[side == 2, 2] = 1; nrm[side == 3, 2] = -1
        x = np.stack([rng.uniform(-100, 100, n), np.where(side < 2, np.where(side == 0, -2.0, 2.0), rng.uniform(-2, 2, n)),
                      np.where(side >= 2, np.where(side == 2, 0.0, 3.0), rng.uniform(0, 3, n))], 1)
    elif kind == "plane":      # open field: ground only
        nrm = np.tile([0.0, 0.0, 1.0], (n, 1))
        x = np.stack([rng.uniform(-30, 30, n), rng.uniform(-30, 30, n), np.zeros(n)], 1)
    else:
        raise ValueError(kind)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    return np.concatenate([nrm, np.cross(x, nrm)], 1)


def normal_eq(kind: str, rng, scale=1.0):
    J = jacobian_rows(kind, rng)
    H = (J.T @ J) * scale
    return 0.5 * (H + H.T)


RANKS = {"rank6": 6, "corridor": 5, "plane": 3}


# ---- covariances ------------------------------------------------------------------------------------------------------
def dense_spd(kappa: float, rng, top=1e-2):
    Q, _ = np.linalg.qr(rng.normal(size=(N, N)))
    ev = top * np.logspace(0.0, -np.log10(kappa), N)
    P = (Q * ev) @ Q.T
    return 0.5 * (P + P.T)


def singular_gravity():
    P = synth.prior_covariance()
    P[15:17, :] = 0.0
    P[:, 15:17] = 0.0
    return P


def base_state(rng, cov):
    return dict(p=rng.normal(size=3), q=synth.quat_from_rotvec(rng.normal(size=3) * 0.5), v=rng.normal(size=3),
                ba=rng.normal(size=3) * 0.01, bg=rng.normal(size=3) * 0.001, g=np.array([0.1, -0.2, 9.79]), cov=np.array(cov))


# ---- what the device loop computes at pass 0, in float64 (Woodbury) ------------------------------------------------------
def gain_T6(P, HTH, laser_cov=LASER_COV):
    A6 = P[:, 0:6] / laser_cov
    M = np.eye(6) + HTH @ A6[0:6]
    return A6 @ np.linalg.inv(M)


def aim_HTh(P, HTH, target6, laser_cov=LASER_COV):
    """Pass 0 has dx_new = 0, so d_x[0:6] = -T6[0:6] HTh: the HTh that makes d_x[0:6] = target6."""
    return -np.linalg.solve(gain_T6(P, HTH, laser_cov)[0:6], target6)


def pivot_order(M):
    """numpy model of inverse6_warp's pivot rule: the unused row with the largest high word of |a[r][k]| (the first such
    row on ties), rows never swapped.  Returns the pivot row of every column."""
    a = np.concatenate([np.array(M, np.float64), np.eye(6)], 1)
    used = np.zeros(6, bool)
    order = []
    for k in range(6):
        hi = np.abs(a[:, k]).view(np.uint64) >> np.uint64(32)
        hi = np.where(used, np.uint64(0), hi)
        top = hi.max()
        who = int(np.nonzero((hi == top) & ~used)[0][0])
        order.append(who)
        a[who] /= a[who, k]
        for r in range(6):
            if r != who:
                a[r] -= a[r, k] * a[who]
        used[who] = True
    return order


# ---- the product's host loop on given sums ------------------------------------------------------------------------------
def icp_params(**kw):
    base = dict(max_num_residuals=2 ** 31 - 1, num_iters_icp=0, frame_id=100, init_num_frames=20,
                threshold_translation_norm=0.01, threshold_orientation_norm=0.1, laser_point_cov=LASER_COV)
    base.update(kw)
    return capi.r3live_params(**base)


def host_loop(case: Case):
    """srl_update_iekf's host-driven loop with the case's blocks in place of passes.  Returns the status, passes run,
    converged flag, trace rows, final state, and the exact FP64 input (state, prediction, i_pass) of every step."""
    prm = icp_params(**case.prm)
    st = capi.eskf_to_c(**case.state)
    it = capi.IekfIter()
    assert capi.lib().srl_iekf_begin(C.byref(st), C.byref(prm), C.byref(it)) == 0
    pred = capi.eskf_from_c(it.predict)
    fq, ft = np.array(case.state["q"], np.float64), np.array(case.state["p"], np.float64)
    trace, inputs = [], []
    status, converged = capi.SRL_OK, 0
    for b in case.blocks:
        if b[31] > 0:
            status = capi.SRL_NAN_PLANARITY
            trace.append(None)
            break
        if int(np.rint(b[28])) < prm.min_number_neighbors:
            status = capi.SRL_TOO_FEW_RESIDUALS
            trace.append(None)
            break
        ne = unpack32(b)
        inputs.append(dict(cur=capi.eskf_from_c(st), pred=pred, HTH=np.array(ne.HTH).reshape(6, 6), HTh=np.array(ne.HTh),
                           i_pass=int(it.pass_index), max_iter=int(it.max_num_iter)))
        dx = np.zeros(17)
        done, div = C.c_int32(0), C.c_int32(0)
        rc = capi.lib().srl_iekf_step(C.byref(it), C.byref(ne), C.byref(prm), C.byref(st), capi.ptr(fq), capi.ptr(ft),
                                      capi.ptr(dx), C.byref(done), C.byref(div))
        if rc != capi.SRL_OK:
            status = rc
            trace.append(None)
            break
        trace.append(np.concatenate([dx, ft, fq]))
        if done.value:
            converged = 1 if done.value == 2 else 0
            break
    return dict(status=status, passes=len(trace), converged=converged, trace=trace, state=capi.eskf_from_c(st),
                inputs=inputs, frame_q=fq, frame_t=ft, max_iter=int(it.max_num_iter))


# ---- the case list --------------------------------------------------------------------------------------------------------
KAPPAS = {"k1e3": 1e3, "k1e6": 1e6, "k1e9": 1e9, "k1e12": 1e12}
AIM_ROT = [0.5e-4, 0.99e-4, 1.01e-4, 5e-3, 1e-2, 1.0, 1.7, np.deg2rad(100.0) * 1.002]
AIM_DP = [99.0, 101.0]


def _unit(v):
    return v / np.linalg.norm(v)


def carried_covariance(seed=7, sweeps=20, dt=0.1):
    """The posterior of `sweeps` updates of the product's host loop (srl_iekf_step, not the oracle) on corridor normal equations, propagated between sweeps by a constant-velocity
    F P F^T + Q: real p-v-theta correlations and a nearly unobservable axis."""
    rng = np.random.default_rng(seed)
    P = synth.prior_covariance()
    F = np.eye(N)
    F[0:3, 6:9] = np.eye(3) * dt
    Q = np.diag([1e-6] * 3 + [1e-6] * 3 + [1e-4] * 3 + [1e-8] * 6 + [1e-9] * 2)
    for s in range(sweeps):
        H = normal_eq("corridor", rng, 1e-2)
        st = base_state(rng, P)
        case = Case("carry", st, np.array([pack32(H, H @ rng.normal(size=6) * 1e-3)]), dict(num_iters_icp=0))
        P = host_loop(case)["state"]["cov"]
        P = F @ P @ F.T + Q
        P = 0.5 * (P + P.T)
    return P


def single_step_cases():
    """One pass, always the final one (num_iters_icp = 0, frame_id >= init_num_frames)."""
    rng = np.random.default_rng(2024)
    covs = {"diag": synth.prior_covariance(), **{k: dense_spd(v, rng) for k, v in KAPPAS.items()}, "carried": carried_covariance()}
    out = []
    for cname, P in covs.items():
        for kind in ("rank6", "corridor", "plane"):
            for mag in (1e0, 1e5, 1e10):
                H = normal_eq(kind, rng, mag)
                st = base_state(rng, P)
                tgt = np.concatenate([rng.normal(size=3) * 0.05, _unit(rng.normal(size=3)) * 0.01])
                out.append(Case(f"{cname}-{kind}-{mag:.0e}", st, np.array([pack32(H, aim_HTh(P, H, tgt))]), kappa_class=cname))
    # aimed rotations and translations (dense, well-conditioned prior so that the aim is exact)
    P = dense_spd(1e3, rng)
    for th in AIM_ROT:
        H = normal_eq("rank6", rng, 1e3)
        tgt = np.concatenate([rng.normal(size=3) * 0.01, _unit(rng.normal(size=3)) * th])
        out.append(Case(f"aim-rot-{th:.4g}", base_state(rng, P), np.array([pack32(H, aim_HTh(P, H, tgt))]), kappa_class="k1e3"))
    for dp in AIM_DP:
        H = normal_eq("rank6", rng, 1e3)
        tgt = np.concatenate([_unit(rng.normal(size=3)) * dp, _unit(rng.normal(size=3)) * 1e-3])
        out.append(Case(f"aim-dp-{dp:g}", base_state(rng, P), np.array([pack32(H, aim_HTh(P, H, tgt))]), kappa_class="k1e3"))
    out += pivot_cases(rng)
    return out


def pivot_cases(rng):
    """A66 correlated so that M = I + HTH A66 has a zero (or 1e-9) diagonal entry while M itself is well conditioned:
    with A[a,a] = 1, A[a,b] = 2, A[b,b] = 5 and HTH = s v v^T on (a, b), v = (1, -1): M[a,a] = 1 - s."""
    out = []
    lc = 0.5                     # a power of two: P / laser_point_cov is exact
    for (a, b) in ((0, 1), (2, 4), (3, 5)):
        for s in (1.0, 1.0 - 1e-9):
            A = np.eye(N) * 1.0
            A[a, a], A[a, b], A[b, a], A[b, b] = 1.0, 2.0, 2.0, 5.0
            P = A * lc
            P[9:12, 9:12] *= 0.001; P[12:15, 12:15] *= 0.0001; P[15:17, 15:17] *= 0.00001
            H = np.diag([2.0] * 6)
            H[a, a] = H[b, b] = s
            H[a, b] = H[b, a] = -s
            others = [i for i in range(6) if i not in (a, b)]
            for i in others:
                H[i, i] = 3.0
            tgt = np.concatenate([rng.normal(size=3) * 0.02, _unit(rng.normal(size=3)) * 0.01])
            out.append(Case(f"pivot-{a}{b}-s{s:.12g}", base_state(rng, P), np.array([pack32(H, aim_HTh(P, H, tgt, lc))]),
                            dict(laser_point_cov=lc), kappa_class="pivot"))
    return out


def linear_model_blocks(case0: Case, H, HTh0, n_pass):
    """Sums of a linear measurement model relinearised at every pass: HTh_p = HTh_0 + HTH d6(x_p), d6 = (p - p0,
    Log(q0^-1 q)) of the state before pass p.  That state comes from the host loop on the blocks so far; once the loop
    has ended, the remaining blocks repeat the last one."""
    import mpmath as mp
    from iekf_reference import _qinv, _qmul, _qrot, _vec, log_so3
    p0, q0 = np.array(case0.state["p"]), np.array(case0.state["q"])
    blocks = [pack32(H, HTh0)]
    while len(blocks) < n_pass:
        pad = [blocks[-1]] * (n_pass - len(blocks))
        r = host_loop(Case(case0.name, case0.state, np.array(blocks + pad), case0.prm))
        p = len(blocks)
        if len(r["inputs"]) <= p:
            blocks += pad
            break
        st = r["inputs"][p]["cur"]
        with mp.workdps(30):
            dth, _ = log_so3(_qrot(_qmul(_qinv(_vec(q0)), _vec(st["q"]))))
        blocks.append(pack32(H, HTh0 + H @ np.concatenate([st["p"] - p0, [float(x) for x in dth]])))
    return np.array(blocks)


def multi_pass_cases():
    """num_iters_icp 0 ... 5 at frame_id 100, and frame_id 5 < init_num_frames (at least 15 iterations); the later passes see
    an offset from the prediction in every block of the state, gravity included (1 - dot just below / above 1e-6)."""
    rng = np.random.default_rng(99)
    out = []
    for n_iter, frame_id, g_omd in [(0, 100, None), (1, 100, None), (2, 100, 0.999e-6), (3, 100, 1.001e-6), (4, 100, None),
                                    (5, 100, 0.5e-6), (5, 100, 2e-6), (3, 5, None)]:
        P = synth.prior_covariance()
        P[15:17, 15:17] = np.eye(2) * 1e-3
        C6 = rng.normal(size=(11, 6)) * 1e-3            # cross-covariance of v, ba, bg, g with the pose
        P[6:17, 0:6] += C6; P[0:6, 6:17] += C6.T
        H = normal_eq("rank6", rng, 1e2)
        tgt = np.concatenate([rng.normal(size=3) * 0.3, _unit(rng.normal(size=3)) * 0.02])
        if g_omd is not None:   # scale the gravity cross-covariance so that pass 0 moves gravity by acos(1 - g_omd)
            T6 = gain_T6(P, H)
            HTh = aim_HTh(P, H, tgt)
            dg = -(T6 @ HTh)[15:17]
            want = np.arccos(1.0 - g_omd)
            P[15:17, 0:6] *= want / np.linalg.norm(dg); P[0:6, 15:17] = P[15:17, 0:6].T
            assert np.linalg.eigvalsh(P).min() > 0
        assert np.linalg.eigvalsh(P).min() > 0
        st = base_state(rng, P)
        prm = dict(num_iters_icp=n_iter, frame_id=frame_id)
        if n_iter == 5:   # no convergence exit: every pass runs
            prm["threshold_translation_norm"] = 0.0
        c0 = Case(f"multi-{n_iter}-f{frame_id}-g{g_omd}", st, np.zeros((1, 32)), prm, kappa_class="multi")
        n_pass = (max(15, n_iter) if frame_id < 20 else n_iter) + 1
        c0.blocks = linear_model_blocks(c0, H, aim_HTh(P, H, tgt), n_pass)
        out.append(c0)
    # weak measurements (HTH far below (P / c)^-1): the prior term (T HTH - I) dx_new ~ -dx_new dominates the later passes, so
    # the boxminus of a large rotation offset reaches d_x undamped
    rng = np.random.default_rng(123)
    for n_iter, th in ((2, 0.3), (3, 1.2)):
        P = synth.prior_covariance()
        H = normal_eq("rank6", rng, 1e-10)
        tgt = np.concatenate([rng.normal(size=3) * 0.1, _unit(rng.normal(size=3)) * th])
        c0 = Case(f"weak-{n_iter}-rot{th:g}", base_state(rng, P), np.zeros((1, 32)),
                  dict(num_iters_icp=n_iter, threshold_translation_norm=0.0), kappa_class="multi")
        c0.blocks = linear_model_blocks(c0, H, aim_HTh(P, H, tgt), n_iter + 1)
        out.append(c0)
    return out
