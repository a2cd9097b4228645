"""Exact pass sums and the rounding bound of each grid reduction that forms them.

Every scan-matching pass ends in 32 sums (srl_api.cu unpack32): components 0..20 are the upper triangle of J^T J,
21..26 are J^T h, 27 is sum d^2, 28 the accepted count, 29 the full-neighbourhood count, 30 the candidates scanned
and 31 the NaN-planarity count.  Each accepted keypoint contributes one product per component 0..27: J_i J_j, J_i h
with h = fl(distance * weight) (the device rounds h on its own before it multiplies), and distance^2.

The exact sum of those products is formed here with TwoProduct (Dekker / Veltkamp: p + e == a * b exactly, no FMA
needed) and math.fsum over all p and e, which returns the correctly rounded value of the exact sum.  The pass kernels
are compiled with FMA contraction, so a product may be rounded on its own or fused into the first add that consumes it;
both are covered, because the reference is the exact product.

Bound (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., §4.2): a sum formed by any tree whose every
leaf passes through at most h roundings (its own product's, then one per add on its way to the root) satisfies
    |computed - exact| <= gamma_h * sum_k |x_k|,      gamma_h = h u / (1 - h u),  u = 2^-53.
A fused first add removes one rounding from that leaf's path, so the same h bounds it.  The h of each form is derived
next to its function below from the code of the reduction.
"""
from __future__ import annotations

import math

import numpy as np

U = 2.0 ** -53
_SPLITTER = 134217729.0   # 2^27 + 1 (Veltkamp)

# (i, j) of components 0..20: the upper triangle of J^T J, row by row (srl_api.cu unpack32)
PAIRS = [(i, j) for i in range(6) for j in range(i, 6)]
N_TERM_COMPONENTS = 28    # 0..27 are sums of products; 28..31 are counts


def gamma(h: int) -> float:
    return h * U / (1.0 - h * U)


# ---- exact products and sums ---------------------------------------------------------------------------------------
def _split(a):
    c = _SPLITTER * a
    hi = c - (c - a)
    return hi, a - hi


def two_product(a, b):
    """p = fl(a b) and e with p + e == a b exactly (no overflow, no underflow below 2^-969 in the product)."""
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    e = ((ah * bh - p) + ah * bl + al * bh) + al * bl
    return p, e


def exact_sum_of_products(a, b) -> tuple[float, float]:
    """(correctly rounded sum_k a_k b_k, an upper bound of sum_k |a_k b_k|)."""
    p, e = two_product(a, b)
    s = math.fsum(np.concatenate([p, e]).tolist())
    mag = math.fsum(np.abs(p).tolist()) + math.fsum(np.abs(e).tolist())
    return s, mag


def term_factors(plane, status):
    """The per-keypoint factors of components 0..27 from a debug pass: plane[:, 6:12] = J, plane[:, 13] = distance,
    plane[:, 14] = weight; only accepted keypoints (status 2) contribute.  Returns a list of 28 (a, b) pairs."""
    acc = np.asarray(status) == 2
    J = np.asarray(plane, np.float64)[acc, 6:12]
    d = np.asarray(plane, np.float64)[acc, 13]
    h = d * np.asarray(plane, np.float64)[acc, 14]          # fl(distance * weight), as the device rounds it
    fac = [(J[:, i], J[:, j]) for i, j in PAIRS]
    fac += [(J[:, i], h) for i in range(6)]
    fac.append((d, d))
    return fac


def exact_sums(plane, status, members=None):
    """Exact components 0..29 of a pass (30 has no per-keypoint reference; 31 is the NaN-planarity count, 0 here) and
    sum |x_k| per component.  `members`: boolean mask of the keypoints that belong to the sum (a shard, k <= k*)."""
    status = np.asarray(status)
    plane = np.asarray(plane, np.float64)
    if members is not None:
        status = np.where(members, status, 0)
    ref = np.zeros(32)
    mag = np.zeros(32)
    for c, (a, b) in enumerate(term_factors(plane, status)):
        ref[c], mag[c] = exact_sum_of_products(a, b)
    ref[28] = float(np.count_nonzero(status == 2))
    ref[29] = float(np.count_nonzero(status >= 1))
    return ref, mag


def term_values(plane, status):
    """The rounded products x_k of components 0..27 (rows = components), for the non-vacuity check."""
    return np.stack([a * b for a, b in term_factors(plane, status)])


def bound(mag, h: int):
    return gamma(h) * np.asarray(mag)


# ---- h per form ----------------------------------------------------------------------------------------------------
MAX_GRID = 2048           # srl_api.cu: ctx->max_grid, the rows of the block-partials buffer
FAST_WARPS = 4            # kFastWarps (srl_internal.h): k1_fast / k1_fit blocks of 4 warps
CHUNK_BLOCKS = 32         # kChunkBlocks (srl_fast.cu)
K1_WARPS = 8              # kK1Warps (srl_internal.h): k1_assoc blocks of 8 warps


def _cdiv(a: int, b: int) -> int:
    return -(-a // b)


def fit_grid(n: int) -> int:
    """launch_k1_split: one 32-keypoint group per warp, 4 warps per block, at most MAX_GRID blocks (grid-stride beyond)."""
    return max(1, min(_cdiv(_cdiv(n, 32), FAST_WARPS), MAX_GRID))


def h_fit(n: int) -> int:
    """k1_fit (srl_fast.cu), one leaf's roundings:
      1  its product (or none, fused into the first add below)
      5  reduce8_over_warp: 3 halving steps over the 8-lane groups, then the xor-8 and xor-16 butterflies
      g  acc += over the warp's groups, g = ceil(groups / (4 G)): the grid-stride rounds (the first add is to 0.0)
      4  the block row: s += s_acc[w] over the 4 warps
      8  the chunk-closing block: r[u] summed over its 8 rows per warp (rows w, w + 4, ...)
      4  cs += over the 4 warps -> chunk_sums
      ceil(n_chunks / 4)  the last block: chunks ch = w, w + 4, ... per warp
      4  tot += over the 4 warps
      1  lane 30 adds k1_scan's scan_count (component 30 only; counted for every component)"""
    G = fit_grid(n)
    g = _cdiv(_cdiv(n, 32), FAST_WARPS * G)
    n_chunks = _cdiv(G, CHUNK_BLOCKS)
    return 1 + 5 + g + 4 + 8 + 4 + _cdiv(n_chunks, 4) + 4 + 1


def assoc_grid(n: int, sm_count: int, per_sm: int) -> int:
    """launch_k1: min(groups, sm_count * per_sm, MAX_GRID); per_sm is the occupancy of the product instance (1 for the
    fallback launch)."""
    return max(1, min(_cdiv(n, 32), sm_count * per_sm, MAX_GRID))


def h_assoc(n: int, sm_count: int, per_sm: int, fallback: bool = False) -> int:
    """k1_assoc (srl_assoc.cu):
      1  the product
      5  transpose_reduce32: xor 16, 8, 4, 2, 1
      g  acc += over the warp's groups, g = ceil(groups / (8 G))
      8  the block row: s += s_acc[w] over the 8 warps
      ceil(G / 8)  the last block: rows b = w, w + 8, ... per warp
      8  tot += over the 8 warps
      1  (fallback launch) tot += prev_out32[lane], the first launch's sums"""
    G = assoc_grid(n, sm_count, per_sm)
    g = _cdiv(_cdiv(n, 32), K1_WARPS * G)
    return 1 + 5 + g + 8 + _cdiv(G, 8) + 8 + (1 if fallback else 0)


def h_assoc_any(n: int, sm_count: int, fallback: bool = False) -> int:
    """per_sm is an occupancy query of the library (1..4 blocks of 256 threads fit an SM): the largest h over all four."""
    return max(h_assoc(n, sm_count, p, fallback) for p in (1, 2, 3, 4))


def fast_grid(n: int, lpk: int) -> int:
    return max(1, min(_cdiv(_cdiv(n, 32 // lpk), FAST_WARPS), MAX_GRID))


def h_fast(n: int, lpk: int) -> int:
    """k1_fast (srl_fast.cu, variant 1):
      1  the product
      5  transpose_reduce32f
      g  acc += over the warp's groups of 32 / lpk keypoints, g = ceil(groups / (4 G))
      4  the block row over the 4 warps
      ceil(G / 32) + 7  the last block: warp w's rows in 8 accumulators, the remainder (< 8 rows) into sacc[0]
      3  the pairwise sum of the 8 accumulators
      4  tot += over the 4 warps"""
    G = fast_grid(n, lpk)
    g = _cdiv(_cdiv(n, 32 // lpk), FAST_WARPS * G)
    return 1 + 5 + g + 4 + _cdiv(G, 32) + 7 + 3 + 4


def h_fallback(first_h: int, n_sweep: int, sm_count: int) -> int:
    """The fallback launch (k1_assoc over the flagged keypoints, one block per SM) adds the first launch's sums last:
    a leaf takes the longer of the two paths, plus that one add."""
    return max(first_h, h_assoc(n_sweep, sm_count, 1)) + 1


def cap_chunk_bounds(n: int, cap: int) -> list[int]:
    """srl_api.cu cap_chunk_bounds: chunk 0 is [0, max(4096, 2 max(cap, 1))), every later chunk twice as long."""
    b = [0]
    chunk = max(4096, 2 * max(cap, 1))
    while b[-1] < n:
        b.append(min(n, b[-1] + chunk))
        chunk *= 2
    return b


def h_cap(bounds: list[int], chunks_run: int) -> int:
    """k2_cap_reduce (srl_assoc.cu), one 1024-thread block per chunk:
      1  the product (fused into acc += r[p] * r[q] or not)
      r  acc += over the thread's rounds k = base + tid, r = ceil(longest chunk run / 1024)
      5  the xor butterflies over the warp
      32 tot += s_red[w] over the 32 warps
      c  v = out32 + tot: the chunks run so far, in order"""
    longest = max(bounds[j + 1] - bounds[j] for j in range(chunks_run))
    return 1 + _cdiv(longest, 1024) + 5 + 32 + chunks_run
