"""CPU model of the device's closed-form symmetric 3x3 eigensolver (srl_math.cuh: eig3_sym_closed).

On the device the plane fit first tries the closed form (trigonometric cubic + cross-product eigenvector) and hands the
matrix to the QR iteration (eig3_sym, the reference's algorithm) when it declines: a (numerically) isotropic matrix, two
smallest eigenvalues closer than 1e-3 of the spread, or a degenerate cross product.  The closed form is compiled for
the device only, so this test builds srl_math.cuh for the host (g++ -ffp-contract=off; 1/x and 1/sqrt(x) stand in for
the device's reciprocal and reciprocal square root) and runs it on 20k adversarial scatter matrices:

- every class reaches the branch the device relies on (planes, discs, edges with gap ratio >= 1.1e-3 and random
  well-conditioned sets take the closed form; poles, edges with gap ratio <= 0.9e-3, isotropic, rank 1 and rank 0
  matrices go to the QR iteration);
- where the closed form answers, its normal is within 5e-11 of the QR iteration's and of the 50-digit truth, and its
  planarity a2D within 3e-8 of the QR iteration's.

This is a model of the device code; the GPU tests in test_degenerate_planes.py are the authority.
"""
import ctypes as C
import os
import subprocess

import mpmath
import numpy as np
import pytest

import degenerate_sets as D

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "sr_livo_b200", "csrc")

SHIM = r"""
#include "srl_math.cuh"
extern "C" void eig_batch(const double* s, long n, int* ok, double* ev_c, double* n_c, double* ev_q, double* n_q) {
    for (long i = 0; i < n; ++i) {
        const double* m = s + 6 * i;   // s00 s10 s11 s20 s21 s22
        ok[i] = srl::eig3_sym_closed(m[0], m[1], m[2], m[3], m[4], m[5], ev_c + 3 * i, n_c[3 * i], n_c[3 * i + 1], n_c[3 * i + 2]) ? 1 : 0;
        srl::eig3_sym(m[0], m[1], m[2], m[3], m[4], m[5], ev_q + 3 * i, n_q[3 * i], n_q[3 * i + 1], n_q[3 * i + 2]);
    }
}
"""

# the branch each class must take: True = closed form, False = QR iteration, None = either
EXPECT = {"plane": True, "disc": True, "edge_gap_1.1e-03": True, "edge_gap_2.0e-03": True, "random": True,
          "pole": False, "edge_gap_5.0e-04": False, "edge_gap_9.0e-04": False, "isotropic": False,
          "isotropic_rotated": False, "rank1": False, "rank0": False,
          # the same classes as FP32 point sets, scatter accumulated like the reference
          "pts_zplane": True, "pts_tilted_plane": True, "pts_disc": True, "pts_disc_rotated": True, "pts_pole": False,
          "pts_pole_rotated": False, "pts_isotropic": False, "pts_isotropic_rotated": None, "pts_rank1": False,
          "pts_rank1_rotated": False, "pts_ulp_spread": None, "pts_edge_gap_5.0e-04": False, "pts_edge_gap_9.0e-04": False,
          "pts_edge_gap_1.1e-03": True, "pts_edge_gap_2.0e-03": True, "pts_random": True}


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("eig_shim")
    src, so = d / "eig_shim.cpp", d / "eig_shim.so"
    src.write_text(SHIM)
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I", CSRC, str(src), "-o", str(so)])
    lib = C.CDLL(str(so))
    lib.eig_batch.argtypes = [C.c_void_p, C.c_long] + [C.c_void_p] * 5
    lib.eig_batch.restype = None

    def run(S):
        S = np.ascontiguousarray(S, np.float64)
        n = S.shape[0]
        out = dict(ok=np.zeros(n, np.int32), ev_c=np.zeros((n, 3)), n_c=np.zeros((n, 3)), ev_q=np.zeros((n, 3)), n_q=np.zeros((n, 3)))
        lib.eig_batch(S.ctypes.data, n, *[out[k].ctypes.data for k in ("ok", "ev_c", "n_c", "ev_q", "n_q")])
        return out
    return run


def _lower(M):
    return np.stack([M[:, 0, 0], M[:, 1, 0], M[:, 1, 1], M[:, 2, 0], M[:, 2, 1], M[:, 2, 2]], axis=1)


def _scatter(pts32):
    """The reference's accumulation (src/optimize.cpp:320-338): sequential barycenter, then the upper triangle."""
    P = np.asarray(pts32, np.float64)
    m = np.zeros(3)
    for p in P:
        m = m + p
    m = m / P.shape[0]
    S = np.zeros((3, 3))
    for p in P:
        d = p - m
        for k in range(3):
            for l in range(k, 3):
                S[k, l] += d[k] * d[l]
    return np.triu(S) + np.triu(S, 1).T


def _matrices(rng, n_per_class=1600):
    """Scatter matrices R diag(lambda) R^T at scales 1e-6 .. 1e6, by class, plus matrices of the FP32 point sets."""
    names, mats = [], []

    def add(name, lam_fn, rotate=True):
        for _ in range(n_per_class):
            lam = np.asarray(lam_fn(), np.float64) * 10.0 ** rng.uniform(-6, 6)
            R = D.random_rotation(rng) if rotate else np.eye(3)
            mats.append((R * lam) @ R.T)
            names.append(name)
    u = rng.uniform
    add("plane", lambda: (0.0, u(0.05, 1.0), 1.0))
    add("disc", lambda: (u(1e-4, 1e-2), 1.0, 1.0))
    add("pole", lambda: (lambda a: (a, a, 1.0))(u(1e-4, 0.1)))
    for g in D.EDGE_GAPS:
        add(f"edge_gap_{g:.1e}", lambda g=g: (lambda lo: (lo, lo + g * (1.0 - lo), 1.0))(u(1e-5, 1e-2)))
    add("isotropic", lambda: (1.0, 1.0, 1.0), rotate=False)
    add("isotropic_rotated", lambda: (1.0, 1.0, 1.0))
    add("rank1", lambda: (0.0, 0.0, 1.0))
    add("rank0", lambda: (0.0, 0.0, 0.0), rotate=False)
    add("random", lambda: np.sort(u(0.01, 1.0, 3)))
    specs = D.class_specs()
    for i in range(40):                                          # the FP32 point sets of the GPU test, many seeds
        for name, fn in specs:
            pts, _ = fn(rng, np.array([8.5, 12.5, 4.5]) + 4 * rng.integers(-3, 4, 3))
            mats.append(_scatter(pts))
            names.append("pts_" + ("random" if name.startswith("random") else name))
    return np.array(names), np.array(mats)


def _truth_normal(M):
    with mpmath.workdps(50):
        E, Q = mpmath.eigsy(mpmath.matrix(M.tolist()))
        j = min(range(3), key=lambda i: E[i])
        v = np.array([float(Q[a, j]) for a in range(3)])
    return v / np.linalg.norm(v)


def _a2d(ev):
    return (np.sqrt(np.abs(ev[:, 1])) - np.sqrt(np.abs(ev[:, 0]))) / np.sqrt(np.abs(ev[:, 2]))


def test_closed_form_branch_and_accuracy_on_adversarial_scatter_matrices(shim):
    rng = np.random.default_rng(2024)
    names, mats = _matrices(rng)
    assert len(names) >= 20000
    r = shim(_lower(mats))
    ok = r["ok"].astype(bool)
    for name, want in EXPECT.items():
        sel = names == name
        assert sel.any(), name
        if want is not None:
            assert np.all(ok[sel] == want), (name, int(ok[sel].sum()), int(sel.sum()))
    # where the closed form answers: normal and planarity against the QR iteration and the truth
    sign = lambda a, b: np.where(np.sum(a * b, axis=1, keepdims=True) < 0, -1.0, 1.0)
    d_qr = np.abs(r["n_c"][ok] - sign(r["n_c"][ok], r["n_q"][ok]) * r["n_q"][ok]).max(axis=1)
    assert d_qr.max() <= 5e-11, (names[ok][np.argmax(d_qr)], d_qr.max())
    da = np.abs(_a2d(r["ev_c"][ok]) - _a2d(r["ev_q"][ok]))
    assert da.max() <= 3e-8, (names[ok][np.argmax(da)], da.max())
    idx = np.nonzero(ok)[0]
    nt = np.array([_truth_normal(mats[i]) for i in idx])
    d_t = np.abs(r["n_c"][idx] - sign(r["n_c"][idx], nt) * nt).max(axis=1)
    assert d_t.max() <= 5e-11, (names[idx][np.argmax(d_t)], d_t.max())
    print(f"{len(names)} matrices, closed form answered {int(ok.sum())}: normal vs QR <= {d_qr.max():.1e}, vs truth <= "
          f"{d_t.max():.1e}, a2D vs QR <= {da.max():.1e}")
