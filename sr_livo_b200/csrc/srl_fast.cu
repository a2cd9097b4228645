// srl_fast.cu — k1_fast: the thread-per-keypoint form of the fused scan-matching pass (sm_90a),
// and the spatial ordering of a sweep's keypoints that makes it coalesce.
//
// Why a second form of K1: the warp-per-keypoint kernel (srl_assoc.cu) is a serial chain of warp shuffles per
// keypoint (long dependent chains, few working warps per SM on a 100k-point sweep).  Here one THREAD owns one keypoint:
//   * keypoints are processed in Morton order of their LiDAR-frame cell (sorted once per sweep), so the 32 lanes
//     of a warp sit in the same few voxels and their 16-byte point loads hit the same L1 lines;
//   * each thread probes its 27 voxels (16 B slot loads), keeps the present ones in a private list, and walks the
//     candidates with ONE float4 load + 9 FP32 ops each;
//   * the K+1 = 21 best candidates live in registers as packed 32-bit keys (FP32 distance^2 with the low 10
//     mantissa bits replaced by the candidate's id) and every candidate goes through a 21-stage min/max chain:
//     no shuffles, no shared memory, no divergence inside the chain;
//   * the 21st key is the guard: if it is farther than the 20th by more than the total error bound (FP32 rounding +
//     the 10 truncated bits), the 20 keys are exactly the reference's 20 nearest points (as a set) and the thread
//     finishes in FP64: exact distances (reference operation order), nearest neighbour, plane fit, residual,
//     Jacobian, 32-component reduction — identical to srl_assoc.cu from there on;
//   * otherwise the keypoint is flagged and redone by k1_assoc's exact selection (launched right after, on the
//     flagged keypoints only), whose final step adds this kernel's sums.
// Handles voxel_neighborhood <= 1 and max/min_number_neighbors == 20 (every reference config outside the first
// 20 init frames); anything else goes to k1_assoc alone.
#include <algorithm>

#include <cooperative_groups.h>
#include <cub/cub.cuh>

#include "srl_internal.h"

namespace srl {

__constant__ VoxelOffsets<27> c_off_fast = voxel_offsets<27>();   // the 27 offsets of the nb<=1 cube ordered by |offset|^2 (centre first)

constexpr unsigned FULLM = 0xffffffffu;
constexpr int KF = 20;            // neighbours kept by the fast path
constexpr int NG = 3;             // guard entries beyond the K-th: boundary candidates are resolved exactly in the finish
constexpr int NS = KF + NG;       // slots that can end up in the neighbourhood
constexpr int NL = NS + 1;        // tracked keys; the last one certifies that nothing untracked can matter
typedef unsigned long long u64;

__device__ __forceinline__ double transpose_reduce32f(double (&v)[32], int lane) {
#pragma unroll
    for (int s = 16; s >= 1; s >>= 1) {
        const bool upper = (lane & s) != 0;
#pragma unroll
        for (int i = 0; i < s; ++i) {
            const double send = upper ? v[i] : v[i + s];
            const double keep = upper ? v[i + s] : v[i];
            v[i] = keep + __shfl_xor_sync(FULLM, send, s);
        }
    }
    return v[0];
}

// Sum over the 32 lanes of 8 per-lane values w[0..7]: on return every lane holds the total of w[lane & 7].  Three halving
// steps (4 + 2 + 1 exchanges) leave one value per lane summed over its 8-lane group, two butterflies sum the four groups:
// 9 exchanges for 8 components, and only 8 values live at a time (the 32-wide transpose needs all 32 in registers).
__device__ __forceinline__ double reduce8_over_warp(double (&w)[8], int lane) {
#pragma unroll
    for (int s = 4; s >= 1; s >>= 1) {
        const bool upper = (lane & s) != 0;
#pragma unroll
        for (int i = 0; i < s; ++i) {
            const double send = upper ? w[i] : w[i + s];
            const double keep = upper ? w[i + s] : w[i];
            w[i] = keep + __shfl_xor_sync(FULLM, send, s);
        }
    }
    double x = w[0];
    x += __shfl_xor_sync(FULLM, x, 8);
    x += __shfl_xor_sync(FULLM, x, 16);
    return x;
}

struct SelNb {   // the K selected points: float indices into the block pool (thread-private array)
    const float* blocks;
    const unsigned* pt;
    __device__ __forceinline__ bool use(int) const { return true; }
    __device__ __forceinline__ void get(int j, float& x, float& y, float& z) const {
        const float4 p = __ldg(reinterpret_cast<const float4*>(blocks + pt[j]));
        x = p.x; y = p.y; z = p.z;
    }
};

__device__ __forceinline__ float key_value(unsigned key) {   // packed key -> (truncated) FP32 distance^2
    return key == 0xffffffffu ? __int_as_float(0x7f800000) : __uint_as_float(key & ~1023u);
}

// NU = candidates per round through the min/max grid; LPK = lanes per keypoint (1, 2 or 4): the candidates of every
// voxel are dealt round-robin to the LPK lanes, each keeps its own top-NL list, the lists are merged with a bitonic
// network over shuffles and lane 0 of the group finishes.  More lanes per keypoint = shorter dependent chain per
// thread and more warps in flight (a 100k-point sweep is only 21 warps per SM at LPK = 1).
template <bool DEBUG, int MINB, int NU, int LPK>
__global__ void __launch_bounds__(kFastThreads, MINB) k1_fast(const __grid_constant__ PassArgs A) {
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    constexpr int KPW = 32 / LPK;                 // keypoints per warp
    const int sub = lane % LPK;                   // this lane's share of every voxel's candidates
    const unsigned gmask = (LPK == 1) ? (1u << lane) : (((1u << LPK) - 1u) << (lane & ~(LPK - 1)));   // lanes of my keypoint
    __shared__ PassConst s_c;
    if (!load_pass_const(A.link, A.c, s_c)) return;   // device-resident loop already ended: nothing to do
    const PassConst& c = s_c;
    const int nb = c.nb;
    const int W = 2 * nb + 1;
    const int V = W * W * W;
    const float size_f = (float)c.size;
    const float lb_margin = 1e-5f * size_f;
    const float eps_abs = 1e-4f * size_f * size_f;   // FP32 rounding of d2f (DESIGN.md); the key truncation adds T * 2^-13
    const float kRel = 1.0f / 2048.0f;

    double acc = 0.0;
    unsigned long long scanned = 0;
    const long long n = A.k_end - A.k_begin;
    const long long n_groups = (n + KPW - 1) / KPW;
    const long long G = gridDim.x;

    for (long long g = (long long)blockIdx.x + (long long)warp * G; g < n_groups; g += G * kFastWarps) {
        const long long s = A.k_begin + g * KPW + lane / LPK;
        const bool valid = s < A.k_end;
        const long long k = valid ? (long long)(A.order ? A.order[s] : (unsigned)s) : 0;
        double bx = 0, by = 0, bz = 0, pwx = 0, pwy = 0, pwz = 0;
        int kx = 0, ky = 0, kz = 0;
        float relx = 0, rely = 0, relz = 0, ofx = 0, ofy = 0, ofz = 0, rfx = 0, rfy = 0, rfz = 0;
        bool in_range = false;
        if (valid) {
            const double rx = A.raw[3 * k], ry = A.raw[3 * k + 1], rz = A.raw[3 * k + 2];
            double tx, ty, tz;
            matvec3_exact(c.R_il, rx, ry, rz, tx, ty, tz);
            bx = SRL_ADD(tx, c.t_il[0]); by = SRL_ADD(ty, c.t_il[1]); bz = SRL_ADD(tz, c.t_il[2]);      // src/optimize.cpp:83
            matvec3_exact(c.Rn, bx, by, bz, tx, ty, tz);
            pwx = SRL_ADD(tx, c.t[0]); pwy = SRL_ADD(ty, c.t[1]); pwz = SRL_ADD(tz, c.t[2]);            // :38
            const double qx = voxel_quotient(pwx, c), qy = voxel_quotient(pwy, c), qz = voxel_quotient(pwz, c);   // :372-374
            in_range = fabs(qx) < 32765.0 && fabs(qy) < 32765.0 && fabs(qz) < 32765.0;
            if (in_range) {
                kx = (int)qx; ky = (int)qy; kz = (int)qz;
                const double cx = (double)kx * c.size, cy = (double)ky * c.size, cz = (double)kz * c.size;
                relx = (float)(pwx - cx); rely = (float)(pwy - cy); relz = (float)(pwz - cz);
                ofx = (float)cx; ofy = (float)cy; ofz = (float)cz;
                rfx = (float)(pwx - (double)ofx); rfy = (float)(pwy - (double)ofy); rfz = (float)(pwz - (double)ofz);
            }
            if (DEBUG && A.out.dbg_world && sub == 0) { A.out.dbg_world[3 * k] = pwx; A.out.dbg_world[3 * k + 1] = pwy; A.out.dbg_world[3 * k + 2] = pwz; }
        }

        // ---- probes: this thread's 27 voxels; present ones go to a private list (blk<<5|cnt , lower bound|offset)
        unsigned ent[27], lbo[27];
        int n_e = 0, total = 0;
        if (in_range) {
            for (int o = 0; o < V; ++o) {
                const int ox = c_off_fast[4 * o], oy = c_off_fast[4 * o + 1], oz = c_off_fast[4 * o + 2];
                const int vx = kx + ox, vy = ky + oy, vz = kz + oz;
                unsigned b, cn;
                if (map_find(A.map.slots, A.map.mask, vx, vy, vz, b, cn) && (int)cn >= c.thr_occ) {            // :386-390
                    const float lox = (float)((vx > 0 ? vx : vx - 1) - kx) * size_f, hix = (float)((vx < 0 ? vx : vx + 1) - kx) * size_f;
                    const float loy = (float)((vy > 0 ? vy : vy - 1) - ky) * size_f, hiy = (float)((vy < 0 ? vy : vy + 1) - ky) * size_f;
                    const float loz = (float)((vz > 0 ? vz : vz - 1) - kz) * size_f, hiz = (float)((vz < 0 ? vz : vz + 1) - kz) * size_f;
                    const float gx = fmaxf(fmaxf(lox - relx, relx - hix) - lb_margin, 0.f);
                    const float gy = fmaxf(fmaxf(loy - rely, rely - hiy) - lb_margin, 0.f);
                    const float gz = fmaxf(fmaxf(loz - relz, relz - hiz) - lb_margin, 0.f);
                    const float lb = (gx * gx + gy * gy + gz * gz) * 0.999999f;
                    ent[n_e] = (b << 5) | cn;
                    lbo[n_e] = (__float_as_uint(lb) & ~127u) | (unsigned)o;   // truncated downward: still a lower bound
                    ++n_e;
                    total += (int)cn;
                }
            }
        }
        const bool full_cand = in_range && total >= c.Kmin;   // else src/optimize.cpp:78 skips the keypoint

        // ---- scan: candidates go through the NL-stage min/max grid on packed keys, NU at a time (the NU x NL grid has
        //      a critical path of NU + NL dependent ops instead of NU * NL: instruction-level parallelism for a thread
        //      that has few sibling warps to hide latency behind)
        unsigned lst[NL];
#pragma unroll
        for (int j = 0; j < NL; ++j) lst[j] = 0xffffffffu;
        if (full_cand) {
            for (int e = 0; e < n_e; ++e) {
                float T = key_value(lst[KF - 1]);
                if (LPK > 1) {   // every lane's K-th key bounds the true K-th distance from above: share the tightest
#pragma unroll
                    for (int d = 1; d < LPK; d <<= 1) T = fminf(T, __shfl_xor_sync(gmask, T, d));
                }
                if (__uint_as_float(lbo[e] & ~127u) > T + T * kRel + 3.f * eps_abs) continue;   // voxel cannot matter any more
                const int cnt = (int)(ent[e] & 31u);
                const float4* bp = reinterpret_cast<const float4*>(A.map.blocks + (size_t)(ent[e] >> 5) * kBlockFloats);
                if (sub == 0) scanned += (unsigned)cnt;
                for (int i0 = sub * NU; i0 < cnt; i0 += NU * LPK) {
                    unsigned key[NU];
#pragma unroll
                    for (int u = 0; u < NU; ++u) {
                        key[u] = 0xffffffffu;
                        if (i0 + u < cnt) {
                            const float4 mp = __ldg(bp + i0 + u);
                            const float dx = (mp.x - ofx) - rfx, dy = (mp.y - ofy) - rfy, dz = (mp.z - ofz) - rfz;
                            const float d2f = dx * dx + dy * dy + dz * dz;
                            key[u] = (__float_as_uint(d2f) & ~1023u) | ((unsigned)e << 5) | (unsigned)(i0 + u);
                        }
                    }
#pragma unroll
                    for (int j = 0; j < NL; ++j) {
#pragma unroll
                        for (int u = 0; u < NU; ++u) {
                            const unsigned lo = min(lst[j], key[u]);
                            key[u] = max(lst[j], key[u]);
                            lst[j] = lo;
                        }
                    }
                }
                if (LPK > 1) __syncwarp(gmask);
            }
        }
        if (LPK > 1) {
            // ---- merge the LPK sorted lists: min(a[j], b[31-j]) over 32 padded slots is a bitonic sequence holding the 32
            //      smallest of both; a 5-stage bitonic merge sorts it; the first NL are the merged list
            __syncwarp(gmask);
#pragma unroll
            for (int d = 1; d < LPK; d <<= 1) {
                unsigned cmb[32];
#pragma unroll
                for (int j = 0; j < 32; ++j) {
                    const unsigned mine = (j < NL) ? lst[j] : 0xffffffffu;
                    const int r = 31 - j;
                    const unsigned theirs_src = (r < NL) ? lst[r] : 0xffffffffu;   // what I send for the partner's slot j
                    const unsigned theirs = __shfl_xor_sync(gmask, theirs_src, d);
                    cmb[j] = min(mine, theirs);
                }
#pragma unroll
                for (int st = 16; st >= 1; st >>= 1) {
#pragma unroll
                    for (int j = 0; j < 32; ++j) {
                        if ((j & st) == 0) {
                            const unsigned lo = min(cmb[j], cmb[j + st]), hi = max(cmb[j], cmb[j + st]);
                            cmb[j] = lo; cmb[j + st] = hi;
                        }
                    }
                }
#pragma unroll
                for (int j = 0; j < NL; ++j) lst[j] = cmb[j];
            }
        }
        const bool leader = (sub == 0);

        // ---- verdict: the slots whose key is within the error window of the K-th can be among the true K nearest; if the
        //      certifier (last tracked key) is outside the window, the true K nearest are among the first m <= NS slots
        bool ambiguous = false;
        int m = 0;
        if (full_cand && leader) {
            const float T = key_value(lst[KF - 1]);
            const float lim = T + T * kRel + 2.5f * eps_abs;
#pragma unroll
            for (int j = 0; j < NS; ++j) m += (key_value(lst[j]) <= lim) ? 1 : 0;   // keys are sorted: the first m slots
            ambiguous = !(key_value(lst[NS]) > lim);
            if (A.force_amb_mod > 0 && (k % A.force_amb_mod) == 0) ambiguous = true;   // test knob: exercise the hand-over
        }
        if (valid && leader && A.flags) A.flags[k] = ambiguous ? 1 : 0;
        const bool do_fit = full_cand && leader && !ambiguous;

        double v[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = 0.0;
        int status = 0;
        if (do_fit) {
            // ---- FP64 finish: exact distances (reference operation order) of the m boundary-inclusive candidates; the
            //      K smallest (distance^2, visit index) are the neighbourhood, the smallest is vector_neighbors[0]
            // (compact code on purpose: thread-private arrays and rolled loops keep this section small in the I-cache;
            //  it runs once per keypoint, the scan above is where the time goes)
            unsigned cand[NS];
#pragma unroll
            for (int j = 0; j < NS; ++j) cand[j] = lst[j];
            u64 xk[NS];
            unsigned xi[NS], xp[NS];
            for (int j = 0; j < m; ++j) {
                const unsigned e = (cand[j] >> 5) & 31u, i = cand[j] & 31u;
                const unsigned pt = (ent[e] >> 5) * kBlockFloats + 4u * i;
                const float4 mp = __ldg(reinterpret_cast<const float4*>(A.map.blocks + pt));
                const double dx = SRL_SUB((double)mp.x, pwx), dy = SRL_SUB((double)mp.y, pwy), dz = SRL_SUB((double)mp.z, pwz);   // :394-395
                const int o = (int)(lbo[e] & 127u);
                const int vis = ((c_off_fast[4 * o] + nb) * W + (c_off_fast[4 * o + 1] + nb)) * W + (c_off_fast[4 * o + 2] + nb);
                xk[j] = (u64)__double_as_longlong(SRL_ADD(SRL_MUL(dx, dx), SRL_ADD(SRL_MUL(dy, dy), SRL_MUL(dz, dz))));
                xi[j] = ((unsigned)vis << 5) | i;   // reference visit order: breaks exact distance ties
                xp[j] = pt;
            }
            unsigned mask = (1u << m) - 1u;
            for (int drop = m - KF; drop > 0; --drop) {   // rare: more candidates than K inside the window: drop the farthest
                u64 wk = 0; unsigned wi = 0; int wj = -1;
                for (int j = 0; j < m; ++j) {
                    const bool in = (mask >> j) & 1u;
                    if (in && (wj < 0 || xk[j] > wk || (xk[j] == wk && xi[j] > wi))) { wk = xk[j]; wi = xi[j]; wj = j; }
                }
                mask &= ~(1u << wj);
            }
            u64 best = ~0ull;
            unsigned best_id = 0xffffffffu, best_pt = 0;
            unsigned sel[KF];
            int ns = 0;
            u64 dkey[DEBUG ? KF : 1];
            unsigned did[DEBUG ? KF : 1];
            for (int j = 0; j < m; ++j) {
                if (!((mask >> j) & 1u)) continue;
                if (xk[j] < best || (xk[j] == best && xi[j] < best_id)) { best = xk[j]; best_id = xi[j]; best_pt = xp[j]; }
                if (DEBUG) { dkey[ns] = xk[j]; did[ns] = xi[j]; }
                sel[ns++] = xp[j];
            }
            const float4 n0 = __ldg(reinterpret_cast<const float4*>(A.map.blocks + best_pt));
            PlaneRow row;
            SelNb nbv{A.map.blocks, sel};
            plane_residual<0>(nbv, KF, (double)n0.x, (double)n0.y, (double)n0.z, c, pwx, pwy, pwz, bx, by, bz, row);
            status = row.accepted ? 2 : 1;
            v[29] = 1.0;
            v[31] = (double)row.nan_planarity;
            const double h = row.distance * row.weight;                                                        // :169
            if (row.accepted) {
                v[0] = row.J[0] * row.J[0]; v[1] = row.J[0] * row.J[1]; v[2] = row.J[0] * row.J[2];
                v[3] = row.J[0] * row.J[3]; v[4] = row.J[0] * row.J[4]; v[5] = row.J[0] * row.J[5];
                v[6] = row.J[1] * row.J[1]; v[7] = row.J[1] * row.J[2]; v[8] = row.J[1] * row.J[3];
                v[9] = row.J[1] * row.J[4]; v[10] = row.J[1] * row.J[5];
                v[11] = row.J[2] * row.J[2]; v[12] = row.J[2] * row.J[3]; v[13] = row.J[2] * row.J[4];
                v[14] = row.J[2] * row.J[5];
                v[15] = row.J[3] * row.J[3]; v[16] = row.J[3] * row.J[4]; v[17] = row.J[3] * row.J[5];
                v[18] = row.J[4] * row.J[4]; v[19] = row.J[4] * row.J[5];
                v[20] = row.J[5] * row.J[5];
                v[21] = row.J[0] * h; v[22] = row.J[1] * h; v[23] = row.J[2] * h;
                v[24] = row.J[3] * h; v[25] = row.J[4] * h; v[26] = row.J[5] * h;
                v[27] = row.distance * row.distance;                                                          // :104
                v[28] = 1.0;
            }
            if (DEBUG) {
                if (A.out.dbg_plane) {
                    double* d = A.out.dbg_plane + 16 * k;
                    d[0] = bx; d[1] = by; d[2] = bz; d[3] = row.nx; d[4] = row.ny; d[5] = row.nz;
#pragma unroll
                    for (int i = 0; i < 6; ++i) d[6 + i] = row.accepted ? row.J[i] : 0.0;
                    d[12] = row.offset; d[13] = row.distance; d[14] = row.weight; d[15] = row.a2D;
                }
                // neighbour list in the reference's order: ascending (distance^2, visit index); dropped slots sort last
                for (int a = 1; a < KF; ++a) {
                    const u64 kd = dkey[a]; const unsigned ki = did[a];
                    int b = a - 1;
                    while (b >= 0 && (dkey[b] > kd || (dkey[b] == kd && did[b] > ki))) { dkey[b + 1] = dkey[b]; did[b + 1] = did[b]; --b; }
                    dkey[b + 1] = kd; did[b + 1] = ki;
                }
                for (int j = 0; j < KF; ++j) {
                    const int vis = (int)(did[j] >> 5), i = (int)(did[j] & 31u);
                    if (A.out.dbg_nbr) {
                        short* d = A.out.dbg_nbr + (k * KF + j) * 4;
                        d[0] = (short)(kx + vis / (W * W) - nb);
                        d[1] = (short)(ky + (vis / W) % W - nb);
                        d[2] = (short)(kz + vis % W - nb);
                        d[3] = (short)i;
                    }
                    if (A.out.dbg_nbr_dist) A.out.dbg_nbr_dist[k * KF + j] = sqrt(__longlong_as_double((long long)dkey[j]));
                }
            }
        }
        if (valid && leader && A.out.status && !ambiguous) A.out.status[k] = status;
        if (ambiguous) { atomicAdd(&A.stats->fast_ambiguous, 1ull); atomicAdd(&A.stats->flagged, 1ull); }
        __syncwarp();
        acc += transpose_reduce32f(v, lane);
    }
    // per-thread scanned counts -> component 30
    {
        double sc = (double)scanned;
#pragma unroll
        for (int s = 16; s >= 1; s >>= 1) sc += __shfl_xor_sync(FULLM, sc, s);
        if (lane == 30) acc += sc;
    }

    __shared__ double s_acc[kFastWarps][32];
    __shared__ bool s_last;
    s_acc[warp][lane] = acc;
    __syncthreads();
    if (warp == 0) {
        double s = 0.0;
#pragma unroll
        for (int w = 0; w < kFastWarps; ++w) s += s_acc[w][lane];
        A.partials[(size_t)blockIdx.x * 32 + lane] = s;
        __threadfence();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned t = atomicAdd(A.ticket, 1u);
        s_last = (t == gridDim.x - 1);
    }
    __syncthreads();
    if (s_last) {
        __threadfence();
        // fixed-order sum of the block partials, 8 independent accumulators per thread to pipeline the loads
        double sacc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        int b = warp;
        for (; b + 7 * kFastWarps < (int)gridDim.x; b += 8 * kFastWarps) {
#pragma unroll
            for (int u = 0; u < 8; ++u) sacc[u] += __ldcg(A.partials + (size_t)(b + u * kFastWarps) * 32 + lane);
        }
        for (; b < (int)gridDim.x; b += kFastWarps) sacc[0] += __ldcg(A.partials + (size_t)b * 32 + lane);
        const double s = ((sacc[0] + sacc[1]) + (sacc[2] + sacc[3])) + ((sacc[4] + sacc[5]) + (sacc[6] + sacc[7]));
        s_acc[warp][lane] = s;
        __syncthreads();
        if (warp == 0) {
            double tot = 0.0;
#pragma unroll
            for (int w = 0; w < kFastWarps; ++w) tot += s_acc[w][lane];
            A.sink.out32[lane] = tot;
            if (lane == 0) *A.ticket = 0u;
        }
    }
}

// =========================================================================================================
// Split form of the pass: k1_scan (LPK lanes per keypoint, FP32 selection) -> k1_fit (thread per keypoint, FP64).
//
// k1_fast is bound by the length of ONE thread's dependent chain (a 100k-point sweep is a single wave of 21 warps per
// SM: time = latency of a warp that probes, scans its candidates, finishes and fits).  The split
// form cuts that chain where it can be cut:
//   * k1_scan gives every keypoint LPK lanes: the 27 probes are dealt to the lanes (results shared through shared
//     memory), every voxel's candidates are dealt round-robin, each lane keeps only its NLS best packed keys (NLS < NL:
//     a lane that could have dropped a relevant key flags the keypoint instead), with all NLS stages of an insertion
//     independent of each other.  The group's bound for the voxel skip is the largest of the lanes' ceil(K/LPK)-th
//     keys (LPK * ceil(K/LPK) >= K tracked candidates are at least that close).  The lanes' lists are merged with an
//     in-register bitonic network over shuffles, the verdict is the one of k1_fast, and the boundary-inclusive
//     candidates go to HBM/L2 as (block * 20 + index, offset id) per sorted position (coalesced for k1_fit).
//   * k1_fit is k1_fast's exact FP64 finish + plane fit + residual + reduction, one thread per keypoint.
// Four times as many, four times shorter warps in the scan; no idle lanes in the fit.
// =========================================================================================================
constexpr int kScanThreads = 128;
constexpr int kChunkBlocks = 32;   // k1_fit's grid reduction: blocks per chunk (a multiple of kFastWarps)
constexpr unsigned KINF = 0xffffffffu;
constexpr int kZone0 = 12;     // k1_fit resolves the K-th boundary among slots >= kZone0 (k1_scan flags anything wider)
constexpr int kRowWords = 24;  // candidate row of a keypoint: NS point ids + header word
constexpr int kBestMax = 4;    // ... and the nearest neighbour among the first kBestMax slots
static_assert(NS == kSplitSlots, "srl_internal.h: kSplitSlots must equal NS");

// the 32 smallest (sorted) of my sorted list and the partner lane's (xor distance d); only the first NV entries of the
// inputs can be finite.  min(a[j], b[31-j]) is a bitonic sequence of the 32 smallest; 5 half-cleaner stages sort it.
template <int NV>
__device__ __forceinline__ void merge_with_partner(unsigned (&l)[32], unsigned gmask, int d) {
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const int r = 31 - j;
        const unsigned a = l[j], b = l[r];
        unsigned ta = KINF, tb = KINF;
        if (r < NV) ta = __shfl_xor_sync(gmask, b, d);   // partner's l[31-j] meets my l[j]
        if (j < NV) tb = __shfl_xor_sync(gmask, a, d);   // partner's l[j] meets my l[31-j]
        l[j] = min(a, ta);
        l[r] = min(b, tb);
    }
#pragma unroll
    for (int st = 16; st >= 1; st >>= 1) {
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            if ((j & st) == 0) {
                const unsigned lo = min(l[j], l[j + st]), hi = max(l[j], l[j + st]);
                l[j] = lo; l[j + st] = hi;
            }
        }
    }
}

// sorts a bitonic 16-sequence held in registers (4 half-cleaner stages)
__device__ __forceinline__ void sort_bitonic16(unsigned (&x)[16]) {
#pragma unroll
    for (int st = 8; st >= 1; st >>= 1) {
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            if ((j & st) == 0) {
                const unsigned lo = min(x[j], x[j + st]), hi = max(x[j], x[j + st]);
                x[j] = lo; x[j + st] = hi;
            }
        }
    }
}

template <int LPK, int NLS, int MINB>
__global__ void __launch_bounds__(kScanThreads, MINB) k1_scan(const __grid_constant__ PassArgs A) {
    static_assert(LPK == 2 || LPK == 4, "lanes per keypoint");
    constexpr int KPW = 32 / LPK;                 // keypoints per warp
    constexpr int KPB = kScanThreads / LPK;       // keypoints per block
    constexpr int Q = (KF + LPK - 1) / LPK;       // the largest of the lanes' Q-th keys bounds the K-th overall from above
    static_assert(NLS >= Q && NLS <= NL, "per-lane list length");
    __shared__ unsigned s_ent[KPB][27];           // (block << 5 | count) of the voxel at offset o, 0 = absent / too few points
    __shared__ unsigned s_lb[KPB][27];            // lower bound of the squared distance to that voxel (FP32 bits)
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int sub = lane % LPK;
    const int kp = threadIdx.x / LPK;
    const int gshift = lane & ~(LPK - 1);          // first lane of my group
    // (all warp-level primitives below run with the full mask at warp-uniform points: a per-group member mask would make
    //  the compiler serialise them over the 32 / LPK distinct masks)
    __shared__ PassConst s_c;
    if (!load_pass_const(A.link, A.c, s_c)) return;   // device-resident loop already ended: nothing to do
    if (cap_chunk_done(A.link)) return;   // capped pass: k* is in an earlier chunk
    const PassConst& c = s_c;
    const int nb = c.nb;
    const int W = 2 * nb + 1;
    const int V = W * W * W;
    const float size_f = (float)c.size;
    const float lb_margin = 1e-5f * size_f;
    const float eps_abs = 1e-4f * size_f * size_f;
    const float kRel = 1.0f / 2048.0f;

    unsigned long long scanned = 0;
    const long long n = A.k_end - A.k_begin;
    const long long n_groups = (n + KPW - 1) / KPW;
    const long long G = gridDim.x;

    for (long long g = (long long)blockIdx.x + (long long)warp * G; g < n_groups; g += G * (kScanThreads / 32)) {
        const long long s = A.k_begin + g * KPW + lane / LPK;
        const bool valid = s < A.k_end;
        const long long k = valid ? (long long)(A.order ? A.order[s] : (unsigned)s) : 0;
        int kx = 0, ky = 0, kz = 0;
        float relx = 0, rely = 0, relz = 0, ofx = 0, ofy = 0, ofz = 0, rfx = 0, rfy = 0, rfz = 0;
        bool in_range = false;
        if (valid) {
            const double rx = A.raw[3 * k], ry = A.raw[3 * k + 1], rz = A.raw[3 * k + 2];
            double tx, ty, tz;
            matvec3_exact(c.R_il, rx, ry, rz, tx, ty, tz);
            const double bx = SRL_ADD(tx, c.t_il[0]), by = SRL_ADD(ty, c.t_il[1]), bz = SRL_ADD(tz, c.t_il[2]);   // src/optimize.cpp:83
            matvec3_exact(c.Rn, bx, by, bz, tx, ty, tz);
            const double pwx = SRL_ADD(tx, c.t[0]), pwy = SRL_ADD(ty, c.t[1]), pwz = SRL_ADD(tz, c.t[2]);         // :38
            const double qx = voxel_quotient(pwx, c), qy = voxel_quotient(pwy, c), qz = voxel_quotient(pwz, c);        // :372-374
            in_range = fabs(qx) < 32765.0 && fabs(qy) < 32765.0 && fabs(qz) < 32765.0;
            if (in_range) {
                kx = (int)qx; ky = (int)qy; kz = (int)qz;
                const double cx = (double)kx * c.size, cy = (double)ky * c.size, cz = (double)kz * c.size;
                relx = (float)(pwx - cx); rely = (float)(pwy - cy); relz = (float)(pwz - cz);
                ofx = (float)cx; ofy = (float)cy; ofz = (float)cz;
                rfx = (float)(pwx - (double)ofx); rfy = (float)(pwy - (double)ofy); rfz = (float)(pwz - (double)ofz);
            }
        }

        // ---- probes: the group's 27 voxels dealt to its lanes; the present ones are packed (in offset order: nearest
        //      voxels first) into the group's shared-memory rows
        int total = 0, n_e = 0;
        for (int o0 = 0; o0 < V; o0 += LPK) {
            const int o = o0 + sub;
            unsigned e_out = 0, l_out = 0;
            if (in_range && o < V) {
                const int ox = c_off_fast[4 * o], oy = c_off_fast[4 * o + 1], oz = c_off_fast[4 * o + 2];
                const int vx = kx + ox, vy = ky + oy, vz = kz + oz;
                unsigned b, cn;
                if (map_find(A.map.slots, A.map.mask, vx, vy, vz, b, cn) && (int)cn >= c.thr_occ) {            // :386-390
                    const float lox = (float)((vx > 0 ? vx : vx - 1) - kx) * size_f, hix = (float)((vx < 0 ? vx : vx + 1) - kx) * size_f;
                    const float loy = (float)((vy > 0 ? vy : vy - 1) - ky) * size_f, hiy = (float)((vy < 0 ? vy : vy + 1) - ky) * size_f;
                    const float loz = (float)((vz > 0 ? vz : vz - 1) - kz) * size_f, hiz = (float)((vz < 0 ? vz : vz + 1) - kz) * size_f;
                    const float gx = fmaxf(fmaxf(lox - relx, relx - hix) - lb_margin, 0.f);
                    const float gy = fmaxf(fmaxf(loy - rely, rely - hiy) - lb_margin, 0.f);
                    const float gz = fmaxf(fmaxf(loz - relz, relz - hiz) - lb_margin, 0.f);
                    e_out = (b << 5) | cn;
                    l_out = (__float_as_uint((gx * gx + gy * gy + gz * gz) * 0.999999f) & ~127u) | (unsigned)o;   // truncated downward: still a lower bound
                    total += (int)cn;
                }
            }
            const unsigned present = (__ballot_sync(FULLM, e_out != 0u) >> gshift) & ((1u << LPK) - 1u);
            if (e_out != 0u) {
                const int pos = n_e + __popc(present & ((1u << sub) - 1u));
                s_ent[kp][pos] = e_out;
                s_lb[kp][pos] = l_out;
            }
            n_e += __popc(present);
        }
#pragma unroll
        for (int d = 1; d < LPK; d <<= 1) total += __shfl_xor_sync(FULLM, total, d);
        __syncwarp();
        const bool full_cand = in_range && total >= c.Kmin;   // else src/optimize.cpp:78 skips the keypoint

        // ---- scan: this lane's share of every voxel's candidates through its own NLS-entry sorted list
        unsigned lst[NLS];
#pragma unroll
        for (int j = 0; j < NLS; ++j) lst[j] = KINF;
        // Every group walks its own voxel list: per step the group's bound T is refreshed, voxels that cannot matter any
        // more are stepped over, and the next one is scanned; the warp leaves when no group has a voxel left.
        int e = full_cand ? 0 : n_e;
        for (;;) {
            unsigned tq = lst[Q - 1];
#pragma unroll
            for (int d = 1; d < LPK; d <<= 1) tq = max(tq, __shfl_xor_sync(FULLM, tq, d));
            const float T = key_value(tq);
            const float Tlim = T + T * kRel + 3.f * eps_abs;
            unsigned lbo = 0;
            while (e < n_e && __uint_as_float((lbo = s_lb[kp][e]) & ~127u) > Tlim) ++e;
            const bool active = e < n_e;
            if (!__any_sync(FULLM, active)) break;
            if (active) {
                const unsigned ent = s_ent[kp][e];
                const int cnt = (int)(ent & 31u);
                const float4* bp = reinterpret_cast<const float4*>(A.map.blocks + (size_t)(ent >> 5) * kBlockFloats);
                if (sub == 0) scanned += (unsigned)cnt;
                int i = sub;
                // two candidates per step while the lane has two left: for a sorted pair (lo, hi) the merged list is
                // l'[j] = min(l[j], max(l[j-1], lo), max(l[j-2], hi)) — 3 ops per stage for 2 candidates (VIMNMX3)
                for (; i + LPK < cnt; i += 2 * LPK) {
                    const float4 ma = __ldg(bp + i), mb = __ldg(bp + i + LPK);
                    const float ax = (ma.x - ofx) - rfx, ay = (ma.y - ofy) - rfy, az = (ma.z - ofz) - rfz;
                    const float bx_ = (mb.x - ofx) - rfx, by_ = (mb.y - ofy) - rfy, bz_ = (mb.z - ofz) - rfz;
                    const unsigned ka = (__float_as_uint(ax * ax + ay * ay + az * az) & ~1023u) | ((unsigned)e << 5) | (unsigned)i;
                    const unsigned kb = (__float_as_uint(bx_ * bx_ + by_ * by_ + bz_ * bz_) & ~1023u) | ((unsigned)e << 5) | (unsigned)(i + LPK);
                    const unsigned lo = min(ka, kb), hi = max(ka, kb);
#pragma unroll
                    for (int j = NLS - 1; j >= 2; --j) lst[j] = min(min(lst[j], max(lst[j - 1], lo)), max(lst[j - 2], hi));
                    lst[1] = min(min(lst[1], max(lst[0], lo)), hi);
                    lst[0] = min(lst[0], lo);
                }
                if (i < cnt) {
                    const float4 mp = __ldg(bp + i);
                    const float dx = (mp.x - ofx) - rfx, dy = (mp.y - ofy) - rfy, dz = (mp.z - ofz) - rfz;
                    const float d2f = dx * dx + dy * dy + dz * dz;
                    const unsigned key = (__float_as_uint(d2f) & ~1023u) | ((unsigned)e << 5) | (unsigned)i;
#pragma unroll
                    for (int j = NLS - 1; j >= 1; --j) lst[j] = min(lst[j], max(lst[j - 1], key));   // stages independent of each other
                    lst[0] = min(lst[0], key);
                }
                ++e;
            }
            __syncwarp();
        }

        const unsigned own_last = lst[NLS - 1];
        bool ambiguous = false;
        int m = 0, j0 = 0, b1 = 0;
        if constexpr (LPK == 4) {
            // ---- merge, result left distributed: the group's sorted best 32 end up as slots 0..15 in lane 0 and 16..31
            //      in lane 1 (lanes 2, 3 compute along and are ignored).  Level 1, lane pairs: the even lane keeps
            //      min(a[j], b[15-j]) = the 16 smallest of both lists, the odd lane max(...) = the 16 largest, each a
            //      bitonic sequence that 4 half-cleaner stages sort.  Level 2, pair against pair: min(P[j], Q[31-j])
            //      over the 32 slots is bitonic and holds the 32 smallest; its first half-cleaner stage runs across
            //      lanes 0/1, the other 4 inside each lane.
            static_assert(NLS <= 16, "per-lane list must fit 16 slots");
            unsigned x[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) x[j] = (j < NLS) ? lst[j] : KINF;
            const bool odd = (sub & 1) != 0;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int r = 15 - j;
                const unsigned va = x[j], vb = x[r];
                unsigned ta = KINF, tb = KINF;
                if (r < NLS) ta = __shfl_xor_sync(FULLM, vb, 1);   // partner's x[15-j] meets my x[j]
                if (j < NLS) tb = __shfl_xor_sync(FULLM, va, 1);   // partner's x[j] meets my x[15-j]
                x[j] = odd ? max(va, ta) : min(va, ta);
                x[r] = odd ? max(vb, tb) : min(vb, tb);
            }
            sort_bitonic16(x);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int r = 15 - j;
                const unsigned va = x[j], vb = x[r];
                const unsigned ta = __shfl_xor_sync(FULLM, vb, 3), tb = __shfl_xor_sync(FULLM, va, 3);
                x[j] = min(va, ta);
                x[r] = min(vb, tb);
            }
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const unsigned t = __shfl_xor_sync(FULLM, x[j], 1);
                x[j] = odd ? max(x[j], t) : min(x[j], t);
            }
            sort_bitonic16(x);

            // ---- verdict (k1_fast's) + the lane certificate: what a lane dropped is not below its last tracked key.
            //      j0 = leading slots that are certainly among the K nearest (even their upper bound is below the (K+1)-th
            //      key), b1 = leading slots that can be THE nearest; k1_fit computes exact distances only for [j0, m), [0, b1)
            static_assert(KF - 1 >= 16 && NS < 32, "slots K-1, K and NS live in the odd lane");
            const unsigned k0 = __shfl_sync(FULLM, x[0], gshift);
            const unsigned kT = __shfl_sync(FULLM, x[KF - 1 - 16], gshift + 1);
            const unsigned kK = __shfl_sync(FULLM, x[KF - 16], gshift + 1);
            const unsigned kC = __shfl_sync(FULLM, x[NS - 16], gshift + 1);
            const float T = key_value(kT);
            const float lim = T + T * kRel + 2.5f * eps_abs;
            const float kvK = key_value(kK);
            const float v0 = key_value(k0);
            const float lim0 = v0 + v0 * kRel + 2.5f * eps_abs;
            const int n_ns = odd ? NS - 16 : 16, n_kf = odd ? KF - 16 : 16;   // my slots below NS / below K
            int cm = 0, cb = 0, cj = 0;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const float kv = key_value(x[j]);
                if (j < n_ns) { cm += (kv <= lim) ? 1 : 0; cb += (kv <= lim0) ? 1 : 0; }
                if (j < n_kf) cj += (kv + kv * kRel + 2.5f * eps_abs < kvK) ? 1 : 0;
            }
            m = cm + __shfl_xor_sync(FULLM, cm, 1);
            b1 = cb + __shfl_xor_sync(FULLM, cb, 1);
            j0 = cj + __shfl_xor_sync(FULLM, cj, 1);
            if (full_cand)
                ambiguous = !(key_value(own_last) > lim) ||
                            (sub < 2 && (!(key_value(kC) > lim) || (m > KF && j0 < kZone0) || b1 > kBestMax || b1 > j0));
            ambiguous = ((__ballot_sync(FULLM, ambiguous) >> gshift) & ((1u << LPK) - 1u)) != 0u;
            if (full_cand && A.force_amb_mod > 0 && (k % A.force_amb_mod) == 0) ambiguous = true;   // test knob
            if (valid) {
                // one 96-byte row per sorted position: 23 x u32 (block * 20 + index in block) + header word
                unsigned* row = A.cand_rows + (size_t)s * kRowWords;
                if (sub == 0) {
                    row[NS] = (full_cand ? (ambiguous ? 255u : (unsigned)m) : 0u) | ((unsigned)j0 << 8) | ((unsigned)b1 << 16);
                    A.flags[k] = ambiguous ? 1 : 0;   // every keypoint of the range: no separate clear of the flags
                    if (ambiguous) { atomicAdd(&A.stats->fast_ambiguous, 1ull); atomicAdd(&A.stats->flagged, 1ull); }
                }
                if (full_cand && !ambiguous && sub < 2) {
                    unsigned* rw = row + (odd ? 16 : 0);
                    const int mine = m - (odd ? 16 : 0);   // how many of my slots are inside the window
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        if (j < n_ns && j < mine) {
                            const unsigned key = x[j];
                            rw[j] = (s_ent[kp][(key >> 5) & 31u] >> 5) * (unsigned)kBlockCap + (key & 31u);
                        }
                    }
                }
            }
        } else {
            // ---- merge the lanes' lists (every lane ends up with the group's sorted best 32)
            unsigned l32[32];
    #pragma unroll
            for (int j = 0; j < 32; ++j) l32[j] = (j < NLS) ? lst[j] : KINF;
            merge_with_partner<NLS>(l32, FULLM, 1);
            if (LPK == 4) merge_with_partner<(2 * NLS < NL ? 2 * NLS : NL)>(l32, FULLM, 2);

            // ---- verdict (k1_fast's) + the lane certificate: what a lane dropped is not below its last tracked key
            //      j0 = leading slots that are certainly among the K nearest (even their upper bound is below the (K+1)-th
            //      key), b1 = leading slots that can be THE nearest; k1_fit computes exact distances only for [j0, m) and [0, b1)
            if (full_cand) {
                const float T = key_value(l32[KF - 1]);
                const float lim = T + T * kRel + 2.5f * eps_abs;
                const float kvK = key_value(l32[KF]);
                const float v0 = key_value(l32[0]);
                const float lim0 = v0 + v0 * kRel + 2.5f * eps_abs;
    #pragma unroll
                for (int j = 0; j < NS; ++j) {
                    const float kv = key_value(l32[j]);
                    m += (kv <= lim) ? 1 : 0;
                    b1 += (kv <= lim0) ? 1 : 0;
                    if (j < KF) j0 += (kv + kv * kRel + 2.5f * eps_abs < kvK) ? 1 : 0;
                }
                ambiguous = !(key_value(l32[NS]) > lim) || !(key_value(own_last) > lim) ||
                            (m > KF && j0 < kZone0) || b1 > kBestMax || b1 > j0;
            }
            ambiguous = ((__ballot_sync(FULLM, ambiguous) >> gshift) & ((1u << LPK) - 1u)) != 0u;
            if (full_cand && A.force_amb_mod > 0 && (k % A.force_amb_mod) == 0) ambiguous = true;   // test knob
            if (valid) {
                // one 96-byte row per sorted position: 23 x u32 (block * 20 + index in block) + header word
                unsigned* row = A.cand_rows + (size_t)s * kRowWords;
                if (sub == 0) {
                    row[NS] = (full_cand ? (ambiguous ? 255u : (unsigned)m) : 0u) | ((unsigned)j0 << 8) | ((unsigned)b1 << 16);
                    A.flags[k] = ambiguous ? 1 : 0;   // every keypoint of the range: no separate clear of the flags
                    if (ambiguous) { atomicAdd(&A.stats->fast_ambiguous, 1ull); atomicAdd(&A.stats->flagged, 1ull); }
                }
                if (full_cand && !ambiguous) {
    #pragma unroll
                    for (int j = 0; j < NS; ++j) {
                        if ((j % LPK) == sub && j < m) {
                            const unsigned key = l32[j];
                            row[j] = (s_ent[kp][(key >> 5) & 31u] >> 5) * (unsigned)kBlockCap + (key & 31u);
                        }
                    }
                }
            }
        }
        __syncwarp();   // the group's shared-memory rows are rewritten by the next group
    }
#pragma unroll
    for (int sft = 16; sft >= 1; sft >>= 1) scanned += __shfl_xor_sync(FULLM, scanned, sft);
    if (lane == 0 && scanned) atomicAdd(A.scan_count, scanned);
}

// neighbour slots of one candidate row: point id (block * 20 + index) per slot and the mask of the K selected slots
struct RowNb {
    const float* blocks;
    const unsigned (&cp)[24];
    unsigned mask;
    __device__ __forceinline__ bool use(int j) const { return (mask >> j) & 1u; }
    __device__ __forceinline__ void get(int j, float& x, float& y, float& z) const {
        const float4 p = __ldg(reinterpret_cast<const float4*>(blocks + (size_t)cp[j] * 4u));
        x = p.x; y = p.y; z = p.z;
    }
};

// exact squared distance (reference operation order, src/optimize.cpp:394-395) as sortable bits
__device__ __forceinline__ u64 exact_d2_bits(const float* blocks, unsigned cp, double pwx, double pwy, double pwz) {
    const float4 mp = __ldg(reinterpret_cast<const float4*>(blocks + (size_t)cp * 4u));
    const double dx = SRL_SUB((double)mp.x, pwx), dy = SRL_SUB((double)mp.y, pwy), dz = SRL_SUB((double)mp.z, pwz);
    return (u64)__double_as_longlong(SRL_ADD(SRL_MUL(dx, dx), SRL_ADD(SRL_MUL(dy, dy), SRL_MUL(dz, dz))));
}
// (visit index of the point's voxel in the reference's loop order) << 5 | index in block: breaks exact distance ties.
// The voxel comes from the key kept in the block's spare w lanes (srl_device.cuh); only rare paths need it.
__device__ __forceinline__ unsigned visit_id(const float* blocks, unsigned cp, double pwx, double pwy, double pwz, double size, int nb, int W) {
    const unsigned blk = cp / (unsigned)kBlockCap;
    const unsigned* meta = reinterpret_cast<const unsigned*>(blocks + (size_t)blk * kBlockFloats);
    short vx, vy, vz;
    unpack_key((unsigned long long)__ldg(meta + kMetaKeyLo) | ((unsigned long long)__ldg(meta + kMetaKeyHi) << 32), vx, vy, vz);
    const int kx = (int)SRL_DIV(pwx, size), ky = (int)SRL_DIV(pwy, size), kz = (int)SRL_DIV(pwz, size);   // src/optimize.cpp:372-374
    const int vis = (((int)vx - kx + nb) * W + ((int)vy - ky + nb)) * W + ((int)vz - kz + nb);
    return ((unsigned)vis << 5) | (cp - blk * (unsigned)kBlockCap);
}

template <bool DEBUG, int MINB>
__global__ void __launch_bounds__(kFastThreads, MINB) k1_fit(const __grid_constant__ PassArgs A) {
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    __shared__ PassConst s_c;
    if (!load_pass_const(A.link, A.c, s_c)) return;   // device-resident loop already ended: nothing to do
    if (cap_chunk_done(A.link)) return;   // capped pass: k* is in an earlier chunk
    const PassConst& c = s_c;
    const int nb = c.nb;
    const int W = 2 * nb + 1;

    double acc = 0.0;
    const long long n = A.k_end - A.k_begin;
    const long long n_groups = (n + 31) / 32;
    const long long G = gridDim.x;

    for (long long g = (long long)blockIdx.x + (long long)warp * G; g < n_groups; g += G * kFastWarps) {
        const long long s = A.k_begin + g * 32 + lane;
        const bool valid = s < A.k_end;
        const long long k = valid ? (long long)(A.order ? A.order[s] : (unsigned)s) : 0;
        unsigned cp[24];
#pragma unroll
        for (int q = 0; q < 24; ++q) cp[q] = 0;
        if (valid) {   // the keypoint's row, written by k1_scan just before: L2, all 6 loads in flight
            const uint4* rp = reinterpret_cast<const uint4*>(A.cand_rows + (size_t)s * kRowWords);
#pragma unroll
            for (int q = 0; q < 6; ++q) {
                const uint4 w = __ldcg(rp + q);
                cp[4 * q] = w.x; cp[4 * q + 1] = w.y; cp[4 * q + 2] = w.z; cp[4 * q + 3] = w.w;
            }
        }
        const unsigned head = cp[NS];
        const int vd = (int)(head & 255u);
        const bool ambiguous = vd == 255;
        const bool do_fit = vd >= KF && vd <= NS;
        const int m = do_fit ? vd : 0;
        const int j0 = (int)((head >> 8) & 255u), b1 = (int)((head >> 16) & 255u);
        double bx = 0, by = 0, bz = 0, pwx = 0, pwy = 0, pwz = 0;
        int kx = 0, ky = 0, kz = 0;
        if (valid) {
            const double rx = A.raw[3 * k], ry = A.raw[3 * k + 1], rz = A.raw[3 * k + 2];
            double tx, ty, tz;
            matvec3_exact(c.R_il, rx, ry, rz, tx, ty, tz);
            bx = SRL_ADD(tx, c.t_il[0]); by = SRL_ADD(ty, c.t_il[1]); bz = SRL_ADD(tz, c.t_il[2]);      // src/optimize.cpp:83
            matvec3_exact(c.Rn, bx, by, bz, tx, ty, tz);
            pwx = SRL_ADD(tx, c.t[0]); pwy = SRL_ADD(ty, c.t[1]); pwz = SRL_ADD(tz, c.t[2]);            // :38
            if (DEBUG) {
                if (do_fit) { kx = (int)SRL_DIV(pwx, c.size); ky = (int)SRL_DIV(pwy, c.size); kz = (int)SRL_DIV(pwz, c.size); }
                if (A.out.dbg_world) { A.out.dbg_world[3 * k] = pwx; A.out.dbg_world[3 * k + 1] = pwy; A.out.dbg_world[3 * k + 2] = pwz; }
            }
        }

        // the keypoint's contribution: J (6), h, d^2 and three flags; the 32 products are formed group by group in the
        // reduction below so that they never all live in registers
        double Jr[6] = {0, 0, 0, 0, 0, 0}, hr = 0.0, d2r = 0.0, acc_f = 0.0, full_f = 0.0, nan_f = 0.0;
        int status = 0;
        if (do_fit) {
            // ---- the K-th boundary: slots [0, j0) are in; of the uncertain slots [j0, m) the m - K farthest by exact
            //      (distance^2, visit index) are out.  Usually m == K and there is nothing to decide.
            unsigned mask = (1u << m) - 1u;
            if (m > KF) {
                u64 zk[NS - kZone0];
                unsigned zi[NS - kZone0];
#pragma unroll
                for (int j = kZone0; j < NS; ++j) {
                    zk[j - kZone0] = 0ull; zi[j - kZone0] = 0u;
                    if (j >= j0 && j < m) {
                        zk[j - kZone0] = exact_d2_bits(A.map.blocks, cp[j], pwx, pwy, pwz);
                        zi[j - kZone0] = visit_id(A.map.blocks, cp[j], pwx, pwy, pwz, c.size, nb, W);
                    }
                }
                for (int drop = m - KF; drop > 0; --drop) {
                    u64 wk = 0; unsigned wi = 0; int wj = -1;
#pragma unroll
                    for (int j = kZone0; j < NS; ++j) {
                        const bool in = j >= j0 && j < m && ((mask >> j) & 1u);
                        if (in && (wj < 0 || zk[j - kZone0] > wk || (zk[j - kZone0] == wk && zi[j - kZone0] > wi))) {
                            wk = zk[j - kZone0]; wi = zi[j - kZone0]; wj = j;
                        }
                    }
                    mask &= ~(1u << wj);
                }
            }
            // ---- vector_neighbors[0]: the exact nearest among the first b1 slots (usually b1 == 1)
            unsigned best_cp = cp[0];
            if (b1 > 1) {
                u64 best = ~0ull;
                unsigned best_id = 0xffffffffu;
#pragma unroll
                for (int j = 0; j < kBestMax; ++j) {
                    if (j < b1) {
                        const u64 d = exact_d2_bits(A.map.blocks, cp[j], pwx, pwy, pwz);
                        const unsigned id = visit_id(A.map.blocks, cp[j], pwx, pwy, pwz, c.size, nb, W);
                        if (d < best || (d == best && id < best_id)) { best = d; best_id = id; best_cp = cp[j]; }
                    }
                }
            }
            const float4 n0 = __ldg(reinterpret_cast<const float4*>(A.map.blocks + (size_t)best_cp * 4u));
            PlaneRow row;
            RowNb nbv{A.map.blocks, cp, mask};
            plane_residual<NS>(nbv, KF, (double)n0.x, (double)n0.y, (double)n0.z, c, pwx, pwy, pwz, bx, by, bz, row);
            status = row.accepted ? 2 : 1;
            full_f = 1.0;
            nan_f = (double)row.nan_planarity;
            const double h = row.distance * row.weight;                                                        // :169
            if (row.accepted) {
#pragma unroll
                for (int i = 0; i < 6; ++i) Jr[i] = row.J[i];
                hr = h; d2r = row.distance * row.distance;                                                     // :104
                acc_f = 1.0;
            }
            if (A.out.rows) {   // per-keypoint rows for the ordered max_num_residuals cap (src/optimize.cpp:107)
                double* rr = A.out.rows + 8 * k;
#pragma unroll
                for (int i = 0; i < 6; ++i) rr[i] = row.J[i];
                rr[6] = h; rr[7] = row.distance * row.distance;
                if (row.nan_planarity) rr[0] = __longlong_as_double(0x7ff8000000000000ll);   // the flag k2_cap_reduce reads
            }
            if (DEBUG) {
                if (A.out.dbg_plane) {
                    double* d = A.out.dbg_plane + 16 * k;
                    d[0] = bx; d[1] = by; d[2] = bz; d[3] = row.nx; d[4] = row.ny; d[5] = row.nz;
#pragma unroll
                    for (int i = 0; i < 6; ++i) d[6 + i] = row.accepted ? row.J[i] : 0.0;
                    d[12] = row.offset; d[13] = row.distance; d[14] = row.weight; d[15] = row.a2D;
                }
                // neighbour list in the reference's order: ascending (distance^2, visit index)
                u64 dkey[KF];
                unsigned did[KF];
                int ns = 0;
#pragma unroll
                for (int j = 0; j < NS; ++j) {
                    if (((mask >> j) & 1u) && ns < KF) {
                        dkey[ns] = exact_d2_bits(A.map.blocks, cp[j], pwx, pwy, pwz);
                        did[ns] = visit_id(A.map.blocks, cp[j], pwx, pwy, pwz, c.size, nb, W);
                        ++ns;
                    }
                }
                for (int a = 1; a < KF; ++a) {
                    const u64 kd = dkey[a]; const unsigned ki = did[a];
                    int b = a - 1;
                    while (b >= 0 && (dkey[b] > kd || (dkey[b] == kd && did[b] > ki))) { dkey[b + 1] = dkey[b]; did[b + 1] = did[b]; --b; }
                    dkey[b + 1] = kd; did[b + 1] = ki;
                }
                for (int j = 0; j < KF; ++j) {
                    const int vis = (int)(did[j] >> 5), i = (int)(did[j] & 31u);
                    if (A.out.dbg_nbr) {
                        short* d = A.out.dbg_nbr + (k * KF + j) * 4;
                        d[0] = (short)(kx + vis / (W * W) - nb);
                        d[1] = (short)(ky + (vis / W) % W - nb);
                        d[2] = (short)(kz + vis % W - nb);
                        d[3] = (short)i;
                    }
                    if (A.out.dbg_nbr_dist) A.out.dbg_nbr_dist[k * KF + j] = sqrt(__longlong_as_double((long long)dkey[j]));
                }
            }
        }
        if (valid && A.out.status && !ambiguous) A.out.status[k] = status;   // the fallback launch writes the flagged (ambiguous) ones
        __syncwarp();
        // components 0..20 = upper triangle of J^T J, 21..26 = J^T h, 27 d^2, 28 residuals, 29 full, 30 (scan count), 31 NaN
        {
            double w[8];
            w[0] = Jr[0] * Jr[0]; w[1] = Jr[0] * Jr[1]; w[2] = Jr[0] * Jr[2]; w[3] = Jr[0] * Jr[3];
            w[4] = Jr[0] * Jr[4]; w[5] = Jr[0] * Jr[5]; w[6] = Jr[1] * Jr[1]; w[7] = Jr[1] * Jr[2];
            const double t0 = reduce8_over_warp(w, lane);
            w[0] = Jr[1] * Jr[3]; w[1] = Jr[1] * Jr[4]; w[2] = Jr[1] * Jr[5]; w[3] = Jr[2] * Jr[2];
            w[4] = Jr[2] * Jr[3]; w[5] = Jr[2] * Jr[4]; w[6] = Jr[2] * Jr[5]; w[7] = Jr[3] * Jr[3];
            const double t1 = reduce8_over_warp(w, lane);
            w[0] = Jr[3] * Jr[4]; w[1] = Jr[3] * Jr[5]; w[2] = Jr[4] * Jr[4]; w[3] = Jr[4] * Jr[5];
            w[4] = Jr[5] * Jr[5]; w[5] = Jr[0] * hr; w[6] = Jr[1] * hr; w[7] = Jr[2] * hr;
            const double t2 = reduce8_over_warp(w, lane);
            w[0] = Jr[3] * hr; w[1] = Jr[4] * hr; w[2] = Jr[5] * hr; w[3] = d2r;
            w[4] = acc_f; w[5] = full_f; w[6] = 0.0; w[7] = nan_f;
            const double t3 = reduce8_over_warp(w, lane);
            const int grp = lane >> 3;
            acc += grp == 0 ? t0 : (grp == 1 ? t1 : (grp == 2 ? t2 : t3));
        }
    }

    // ---- block sum -> chunk sum (the last block of every 32-block chunk) -> total (the block that closes the last chunk).
    //      Fixed summation order at every level (run-to-run bitwise deterministic); two short levels instead of one block
    //      walking all gridDim.x partial rows (for 782 blocks that walk was ~9 us of single-block tail).
    __shared__ double s_acc[kFastWarps][32];
    __shared__ int s_role;
    s_acc[warp][lane] = acc;
    __syncthreads();
    const unsigned chunk = blockIdx.x / kChunkBlocks, n_chunks = (gridDim.x + kChunkBlocks - 1) / kChunkBlocks;
    const unsigned in_chunk = min((unsigned)kChunkBlocks, gridDim.x - chunk * kChunkBlocks);
    if (warp == 0) {
        double s = 0.0;
#pragma unroll
        for (int w = 0; w < kFastWarps; ++w) s += s_acc[w][lane];
        A.partials[(size_t)blockIdx.x * 32 + lane] = s;
    }
    __syncthreads();
    if (threadIdx.x == 0) {   // release (the block's row, through the barrier) - ticket - acquire (the other blocks' rows): one thread fences
        fence_acq_rel_gpu();
        const unsigned t = atomicAdd(A.chunk_tickets + chunk, 1u);
        fence_acq_rel_gpu();
        s_role = (t == in_chunk - 1) ? 1 : 0;
    }
    __syncthreads();
    if (!s_role) return;
    {   // this block closes its chunk: sum the chunk's rows (warp w takes rows w, w + 4, ...: 8 independent loads each)
        double r[kChunkBlocks / kFastWarps];
#pragma unroll
        for (int u = 0; u < kChunkBlocks / kFastWarps; ++u) {
            const unsigned row = (unsigned)(warp + u * kFastWarps);
            r[u] = row < in_chunk ? __ldcg(A.partials + (size_t)(chunk * kChunkBlocks + row) * 32 + lane) : 0.0;
        }
        double s = 0.0;
#pragma unroll
        for (int u = 0; u < kChunkBlocks / kFastWarps; ++u) s += r[u];
        __syncthreads();
        s_acc[warp][lane] = s;
        __syncthreads();
        if (warp == 0) {
            double cs = 0.0;
#pragma unroll
            for (int w = 0; w < kFastWarps; ++w) cs += s_acc[w][lane];
            A.chunk_sums[(size_t)chunk * 32 + lane] = cs;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            A.chunk_tickets[chunk] = 0u;
            fence_acq_rel_gpu();
            const unsigned t = atomicAdd(A.ticket, 1u);
            fence_acq_rel_gpu();
            s_role = (t == n_chunks - 1) ? 2 : 0;
        }
        __syncthreads();
        if (s_role != 2) return;
    }
    {   // this block closes the last chunk: the pass's totals
        double s = 0.0;
        for (unsigned ch = (unsigned)warp; ch < n_chunks; ch += kFastWarps) s += __ldcg(A.chunk_sums + (size_t)ch * 32 + lane);
        __syncthreads();
        s_acc[warp][lane] = s;
        __syncthreads();
        if (warp == 0) {
            double tot = 0.0;
#pragma unroll
            for (int w = 0; w < kFastWarps; ++w) tot += s_acc[w][lane];
            if (lane == 30) { tot += (double)__ldcg(A.scan_count); *A.scan_count = 0ull; }   // k1_scan's visit count
            if (lane == 0) *A.ticket = 0u;
            // nothing flagged in this pass on this rank (the usual case): these ARE the rank's sums, finalised here.  The
            // fallback launch that follows then only forwards them again (same values, same sequence number).
            if (__ldcg(&A.stats->flagged) == 0ull) {
                if (lane == 0) A.stats->finalised = 1ull;
                finalise_pass(A, false, tot, lane);
            } else {
                A.sink.out32[lane] = tot;   // the fallback launch adds its own sums to these and finalises
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// sweep ordering: Morton code of the LiDAR-frame 1 m cell of every keypoint, stable radix sort -> order[]
// (a rigid transform keeps neighbours neighbours, so the order is pose independent and computed once per sweep)
// ---------------------------------------------------------------------------------------------------------
// 8 bits per axis (1 m cells within +-128 m of the sensor; farther points are clamped, which only costs locality):
// 24-bit Morton keys -> 3 radix passes (the sort of a 100k-point sweep is launch-latency bound: ~11 us per pass)
__device__ __forceinline__ unsigned spread8(unsigned x) {
    x &= 0xffu;
    x = (x | (x << 8)) & 0x00f00fu;
    x = (x | (x << 4)) & 0x0c30c3u;
    x = (x | (x << 2)) & 0x249249u;
    return x;
}
__global__ void k_sweep_keys(const double* __restrict__ raw, long long n, double cell, unsigned* keys, unsigned* idx) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double fx = fmin(fmax(floor(raw[3 * i] / cell) + 128.0, 0.0), 255.0);
    const double fy = fmin(fmax(floor(raw[3 * i + 1] / cell) + 128.0, 0.0), 255.0);
    const double fz = fmin(fmax(floor(raw[3 * i + 2] / cell) + 128.0, 0.0), 255.0);
    keys[i] = spread8((unsigned)fx) | (spread8((unsigned)fy) << 1) | (spread8((unsigned)fz) << 2);
    idx[i] = (unsigned)i;
}

// ---- the same order in ONE launch: a thread-block cluster sorts the sweep's keys with a stable LSD radix sort (3 passes of
// 8 bits over the 24-bit Morton keys).  The CUB path above is six launch-latency-bound kernels (~45 us of GPU time for
// 100k keys plus the gaps between them); here the CTAs of one cluster (16 where the device allows it, else the portable 8)
// own consecutive chunks of the sequence, every warp a consecutive sub-chunk of at most 8 x 32 keys that it keeps in
// REGISTERS for the whole pass.  Per pass: load (pass 0 derives the keys from the raw points, so no key array is written
// first) -> warp-private digit counts in shared memory, remembering each key's rank among the warp's keys of that digit ->
// a shuffle scan over the 32 warps per digit -> CTA totals, which the other CTAs read through distributed shared memory ->
// every CTA derives the global position of its first key of every digit -> scatter straight from the registers -> cluster
// barrier (release/acquire at cluster scope orders the global stores; the next pass reads them with ld.global.cg).
// A stable sort has exactly one result, so the order is identical to the CUB one (checked once per process at first use).
namespace cg = cooperative_groups;
constexpr int kSortThreads = 1024, kSortWarps = kSortThreads / 32, kSortRounds = 8;
constexpr int kSortKeysPerCta = kSortWarps * kSortRounds * 32;   // 8192

template <bool LOCAL_SORT>
__global__ void __launch_bounds__(kSortThreads, 1)
k_sweep_order_cluster(const double* __restrict__ raw, int n, double cell, unsigned* keys_a, unsigned* idx_a, unsigned* keys_b, unsigned* order_out) {
    cg::cluster_group cluster = cg::this_cluster();
    const unsigned cta = cluster.block_rank(), n_cta = cluster.num_blocks();
    __shared__ unsigned s_cnt[kSortWarps][257];   // per-warp digit counts, then the warp's offset inside the CTA's run of that digit (padded: the scan reads columns)
    __shared__ unsigned s_block[256];             // this CTA's digit totals (the other CTAs read them through DSMEM)
    __shared__ unsigned s_part[2][4][256];        // partial sums over a quarter of the CTAs: [all | the CTAs before this one]
    __shared__ unsigned s_base[256];              // keys with that digit in the CTAs before this one
    __shared__ unsigned s_scan[256];              // keys with a smaller digit in the whole sequence
    __shared__ unsigned s_start[256];             // keys with a smaller digit in this CTA
    extern __shared__ unsigned s_stage[];         // LOCAL_SORT: the CTA's keys [0, 8192) and indices [8192, 16384) in digit order
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n_warps = (int)n_cta * kSortWarps;
    const int per = ((n + n_warps - 1) / n_warps + 31) / 32 * 32;   // keys per warp: consecutive, a multiple of 32, <= 256 (host)
    const int gw = (int)cta * kSortWarps + warp;
    const int begin = min(n, gw * per), end = min(n, begin + per);
    const int cta_n = min(n, ((int)cta + 1) * kSortWarps * per) - min(n, (int)cta * kSortWarps * per);
    const unsigned lt = (1u << lane) - 1u;

    const unsigned* kin = nullptr;
    const unsigned* iin = nullptr;
    unsigned* kout = keys_b;
    unsigned* iout = order_out;
    unsigned key[kSortRounds], idx[kSortRounds], lrk[kSortRounds];
#pragma unroll 1
    for (int pass = 0; pass < 3; ++pass) {
        const int shift = 8 * pass;
        for (int d = lane; d < 256; d += 32) s_cnt[warp][d] = 0u;
#pragma unroll
        for (int r = 0; r < kSortRounds; ++r) {
            const int j = begin + r * 32 + lane;
            key[r] = 0u; idx[r] = 0u;
            if (j < end) {
                if (pass == 0) {
                    const double x = raw[3 * (long long)j], y = raw[3 * (long long)j + 1], z = raw[3 * (long long)j + 2];
                    const double fx = fmin(fmax(floor(cell == 1.0 ? x : x / cell) + 128.0, 0.0), 255.0);
                    const double fy = fmin(fmax(floor(cell == 1.0 ? y : y / cell) + 128.0, 0.0), 255.0);
                    const double fz = fmin(fmax(floor(cell == 1.0 ? z : z / cell) + 128.0, 0.0), 255.0);
                    key[r] = spread8((unsigned)fx) | (spread8((unsigned)fy) << 1) | (spread8((unsigned)fz) << 2);
                    idx[r] = (unsigned)j;
                } else {
                    key[r] = __ldcg(kin + j);
                    idx[r] = __ldcg(iin + j);
                }
            }
        }
        __syncwarp();
#pragma unroll
        for (int r = 0; r < kSortRounds; ++r) {   // every round runs on the full warp: lanes past the end match nobody
            const bool valid = begin + r * 32 + lane < end;
            const unsigned d = (key[r] >> shift) & 255u;
            const unsigned peers = __match_any_sync(FULLM, valid ? d : (256u + (unsigned)lane));
            const unsigned rank = __popc(peers & lt);
            const unsigned prior = valid ? s_cnt[warp][d] : 0u;
            __syncwarp();
            if (valid && rank == 0u) s_cnt[warp][d] = prior + (unsigned)__popc(peers);
            __syncwarp();
            lrk[r] = prior + rank;   // rank among the warp's keys of this digit
        }
        __syncthreads();
#pragma unroll
        for (int q = 0; q < 8; ++q) {   // exclusive prefix over the CTA's warps, and the CTA's total: warp w scans digits 8w..8w+7
            const int dig = warp * 8 + q;
            const unsigned c = s_cnt[lane][dig];
            unsigned incl = c;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const unsigned t = __shfl_up_sync(FULLM, incl, o); if (lane >= o) incl += t; }
            s_cnt[lane][dig] = incl - c;
            if (lane == 31) s_block[dig] = incl;
        }
        cluster.sync();    // every CTA's s_block is complete (and this CTA's s_cnt offsets are)
        {
            const int dig = tid & 255, part = tid >> 8;
            unsigned tot = 0, before = 0;
            for (unsigned c = (unsigned)part; c < n_cta; c += 4u) {
                const unsigned v = *cluster.map_shared_rank(&s_block[dig], c);
                tot += v;
                if (c < cta) before += v;
            }
            s_part[0][part][dig] = tot;
            s_part[1][part][dig] = before;
        }
        __syncthreads();
        {   // exclusive scans over the 256 digits of the cluster's totals and of this CTA's: 8 digits per lane, then a warp scan
            // of the lane sums (every warp computes them -- no shuffle under a branch --, warp 0 stores)
            unsigned v[8], w[8], sum = 0, sum_l = 0;
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const int dig = lane * 8 + q;
                v[q] = s_part[0][0][dig] + s_part[0][1][dig] + s_part[0][2][dig] + s_part[0][3][dig];
                w[q] = s_block[dig];
                sum += v[q]; sum_l += w[q];
            }
            unsigned incl = sum, incl_l = sum_l;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned t = __shfl_up_sync(FULLM, incl, o), u = __shfl_up_sync(FULLM, incl_l, o);
                if (lane >= o) { incl += t; incl_l += u; }
            }
            unsigned run = incl - sum, run_l = incl_l - sum_l;
            if (warp == 0) {
#pragma unroll
                for (int q = 0; q < 8; ++q) { s_scan[lane * 8 + q] = run; run += v[q]; s_start[lane * 8 + q] = run_l; run_l += w[q]; }
            }
        }
        if (tid < 256) s_base[tid] = s_part[1][0][tid] + s_part[1][1][tid] + s_part[1][2][tid] + s_part[1][3][tid];
        __syncthreads();
        if (LOCAL_SORT) {
            // a scattered 4-byte store costs a full L2 transaction, and 16 SMs issue all of them: order the CTA's keys by digit
            // in shared memory first, then every run of equal digits leaves as consecutive addresses
#pragma unroll
            for (int r = 0; r < kSortRounds; ++r) {
                if (begin + r * 32 + lane < end) {
                    const unsigned d = (key[r] >> shift) & 255u;
                    const unsigned li = s_start[d] + s_cnt[warp][d] + lrk[r];
                    s_stage[li] = key[r];
                    s_stage[kSortKeysPerCta + li] = idx[r];
                }
            }
            __syncthreads();
            if (tid < 256) s_base[tid] += s_scan[tid] - s_start[tid];   // global position of local slot i with this digit: s_base[d] + i
            __syncthreads();
#pragma unroll
            for (int k = 0; k < kSortRounds; ++k) {
                const int i = k * kSortThreads + tid;
                if (i < cta_n) {
                    const unsigned ky = s_stage[i];
                    const unsigned pos = s_base[(ky >> shift) & 255u] + (unsigned)i;
                    if (pass < 2) kout[pos] = ky;
                    iout[pos] = s_stage[kSortKeysPerCta + i];
                }
            }
        } else {
#pragma unroll
            for (int r = 0; r < kSortRounds; ++r) {
                if (begin + r * 32 + lane < end) {
                    const unsigned d = (key[r] >> shift) & 255u;
                    const unsigned pos = s_scan[d] + s_base[d] + s_cnt[warp][d] + lrk[r];
                    if (pass < 2) kout[pos] = key[r];
                    iout[pos] = idx[r];
                }
            }
        }
        cluster.sync();    // all keys of the pass are placed, and nobody reads this pass's s_block any more
        // regs -> (b, order) -> (a, idx_a) -> order: the third pass leaves the sorted indices in order_out
        if (pass == 0) { kin = keys_b; iin = order_out; kout = keys_a; iout = idx_a; }
        else { kin = keys_a; iin = idx_a; kout = keys_b; iout = order_out; }
    }
}

// first version, kept selectable for A/B runs (keys re-read from HBM in the scatter phase)
__global__ void __launch_bounds__(kSortThreads, 1)
k_sweep_order_cluster_v1(const double* __restrict__ raw, long long n, double cell, unsigned* keys_a, unsigned* idx_a, unsigned* keys_b, unsigned* order_out) {
    cg::cluster_group cluster = cg::this_cluster();
    const unsigned cta = cluster.block_rank(), n_cta = cluster.num_blocks();
    __shared__ unsigned s_cnt[kSortWarps][256];   // per-warp digit counts, then the warp's running offset inside the CTA's run of that digit
    __shared__ unsigned s_block[256];             // this CTA's digit totals (the other CTAs read them through DSMEM)
    __shared__ unsigned s_base[256];              // global position of this CTA's first key with that digit
    __shared__ unsigned s_scan[256];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const long long n_warps = (long long)n_cta * kSortWarps;
    const long long per = ((n + n_warps - 1) / n_warps + 31) / 32 * 32;   // keys per warp: consecutive, a multiple of 32
    const long long gw = (long long)cta * kSortWarps + warp;
    const long long begin = min(n, gw * per), end = min(n, begin + per);

    for (long long i = (long long)cta * kSortThreads + tid; i < n; i += (long long)n_cta * kSortThreads) {
        const double fx = fmin(fmax(floor(raw[3 * i] / cell) + 128.0, 0.0), 255.0);
        const double fy = fmin(fmax(floor(raw[3 * i + 1] / cell) + 128.0, 0.0), 255.0);
        const double fz = fmin(fmax(floor(raw[3 * i + 2] / cell) + 128.0, 0.0), 255.0);
        keys_a[i] = spread8((unsigned)fx) | (spread8((unsigned)fy) << 1) | (spread8((unsigned)fz) << 2);
        idx_a[i] = (unsigned)i;
    }
    __threadfence();
    cluster.sync();

    const unsigned* kin = keys_a;
    const unsigned* iin = idx_a;
    unsigned* kout = keys_b;
    unsigned* iout = order_out;
    for (int pass = 0; pass < 3; ++pass) {
        const int shift = 8 * pass;
        for (int d = lane; d < 256; d += 32) s_cnt[warp][d] = 0u;
        __syncwarp();
        for (long long j = begin + lane; j < end; j += 32) atomicAdd(&s_cnt[warp][(kin[j] >> shift) & 255u], 1u);
        __syncthreads();
        if (tid < 256) {   // exclusive prefix over the CTA's warps, and the CTA's total, per digit
            unsigned run = 0;
            for (int w = 0; w < kSortWarps; ++w) { const unsigned c = s_cnt[w][tid]; s_cnt[w][tid] = run; run += c; }
            s_block[tid] = run;
        }
        cluster.sync();    // every CTA's s_block is complete
        if (tid < 256) {
            unsigned tot = 0, before = 0;
            for (unsigned c = 0; c < n_cta; ++c) {
                const unsigned v = *cluster.map_shared_rank(&s_block[tid], c);
                tot += v;
                if (c < cta) before += v;
            }
            s_scan[tid] = tot;
            s_base[tid] = before;
        }
        __syncthreads();
        if (warp == 0) {   // exclusive scan of the 256 digit totals: 8 per lane, then a warp scan of the lane sums
            unsigned v[8], sum = 0;
#pragma unroll
            for (int q = 0; q < 8; ++q) { v[q] = s_scan[lane * 8 + q]; sum += v[q]; }
            unsigned incl = sum;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const unsigned t = __shfl_up_sync(FULLM, incl, o); if (lane >= o) incl += t; }
            unsigned run = incl - sum;
#pragma unroll
            for (int q = 0; q < 8; ++q) { s_scan[lane * 8 + q] = run; run += v[q]; }
        }
        __syncthreads();
        if (tid < 256) s_base[tid] += s_scan[tid];
        __syncthreads();
        for (long long j0 = begin; j0 < end; j0 += 32) {   // rounds of 32 consecutive keys, in order
            const long long j = j0 + lane;
            const bool valid = j < end;
            const unsigned key = valid ? kin[j] : 0u;
            const unsigned d = (key >> shift) & 255u;
            const unsigned peers = __match_any_sync(FULLM, valid ? d : (256u + (unsigned)lane));   // lanes past the end match nobody
            const unsigned rank = __popc(peers & ((1u << lane) - 1u));
            if (valid) {
                const unsigned pos = s_base[d] + s_cnt[warp][d] + rank;
                kout[pos] = key;
                iout[pos] = iin[j];
            }
            __syncwarp();
            if (valid && rank + 1u == (unsigned)__popc(peers)) s_cnt[warp][d] += (unsigned)__popc(peers);   // the last peer moves the running offset
            __syncwarp();
        }
        __threadfence();
        cluster.sync();    // all keys of the pass are placed, and nobody reads this pass's s_block any more
        // a -> (b, order) -> (a, idx_a) -> (b, order): the third pass leaves the sorted indices in order_out
        if (pass == 0) { kin = keys_b; iin = order_out; kout = keys_a; iout = idx_a; }
        else { kin = keys_a; iin = idx_a; kout = keys_b; iout = order_out; }
    }
}

__global__ void k_order_mismatch(const unsigned* __restrict__ a, const unsigned* __restrict__ b, long long n, unsigned* count) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && a[i] != b[i]) atomicAdd(count, 1u);
}

// scratch needs 3 * n * 4 bytes (aligned); returns cudaErrorNotSupported when no cluster size is launchable or n exceeds
// what the cluster holds in registers (16 CTAs: 131072 keys, 8 CTAs: 65536) -- the caller then uses CUB
static long long sweep_cluster_capacity(const KernelChoice& ch) {
    return ch.cluster_size < 0 ? 0 : (long long)(ch.cluster_size > 0 ? ch.cluster_size : 16) * kSortKeysPerCta;
}
static cudaError_t sweep_order_cluster(KernelChoice& ch, const double* d_raw, long long n, unsigned* d_order, void* scratch, cudaStream_t stream) {
    auto al = [](size_t x) { return (x + 255) / 256 * 256; };
    char* p = static_cast<char*>(scratch);
    unsigned* ka = reinterpret_cast<unsigned*>(p); p += al(n * 4);
    unsigned* kb = reinterpret_cast<unsigned*>(p); p += al(n * 4);
    unsigned* ia = reinterpret_cast<unsigned*>(p);
    if (ch.cluster_size < 0) return cudaErrorNotSupported;
    const int sizes[2] = {16, 8};
    for (int t = 0; t < 2; ++t) {
        const int cs = ch.cluster_size > 0 ? ch.cluster_size : sizes[t];
        if (n > (long long)cs * kSortKeysPerCta) {
            if (ch.cluster_size > 0) return cudaErrorNotSupported;   // this sweep is too long; the kernel stays in use for shorter ones
            continue;
        }
        if (ch.cluster_size == 0) {   // first launch: opt in to the 16-CTA cluster and to the staging buffer
            if (cs > 8 && (cudaFuncSetAttribute(k_sweep_order_cluster<true>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess ||
                           cudaFuncSetAttribute(k_sweep_order_cluster<false>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess ||
                           cudaFuncSetAttribute(k_sweep_order_cluster_v1, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess)) { cudaGetLastError(); continue; }
            if (cudaFuncSetAttribute(k_sweep_order_cluster<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * kSortKeysPerCta * (int)sizeof(unsigned)) != cudaSuccess) { cudaGetLastError(); break; }
        }
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3((unsigned)cs); cfg.blockDim = dim3(kSortThreads); cfg.dynamicSmemBytes = 0; cfg.stream = stream;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = (unsigned)cs; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        cudaError_t e;
        if (ch.order_mode == 3) e = cudaLaunchKernelEx(&cfg, k_sweep_order_cluster_v1, d_raw, n, 1.0, ka, ia, kb, d_order);
        else if (ch.order_mode == 2) e = cudaLaunchKernelEx(&cfg, k_sweep_order_cluster<false>, d_raw, (int)n, 1.0, ka, ia, kb, d_order);
        else {   // keys in registers + CTA-local digit order before the stores
            cfg.dynamicSmemBytes = 2 * kSortKeysPerCta * sizeof(unsigned);
            e = cudaLaunchKernelEx(&cfg, k_sweep_order_cluster<true>, d_raw, (int)n, 1.0, ka, ia, kb, d_order);
        }
        if (e == cudaSuccess) { ch.cluster_size = cs; return cudaSuccess; }
        cudaGetLastError();
        if (ch.cluster_size > 0) break;
    }
    ch.cluster_size = -1;
    return cudaErrorNotSupported;
}

// CUB's radix sort of the keys; scratch: three n-word arrays, then CUB's `tmp` bytes
static cudaError_t sweep_order_cub(const double* d_raw, long long n, unsigned* d_order, void* scratch, size_t tmp, cudaStream_t stream) {
    auto al = [](size_t x) { return (x + 255) / 256 * 256; };
    char* p = static_cast<char*>(scratch);
    unsigned* ka = reinterpret_cast<unsigned*>(p); p += al(n * 4);
    unsigned* kb = reinterpret_cast<unsigned*>(p); p += al(n * 4);
    unsigned* ia = reinterpret_cast<unsigned*>(p); p += al(n * 4);
    const int T = 256;
    k_sweep_keys<<<(unsigned)((n + T - 1) / T), T, 0, stream>>>(d_raw, n, 1.0, ka, ia);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    return cub::DeviceRadixSort::SortPairs(p, tmp, ka, kb, ia, d_order, (int)n, 0, 24, stream);
}

cudaError_t sweep_compute_order(KernelChoice& ch, const double* d_raw, long long n, unsigned* d_order, void* scratch,
                                size_t scratch_bytes, size_t* needed, cudaStream_t stream) {
    auto al = [](size_t x) { return (x + 255) / 256 * 256; };
    size_t tmp = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tmp, (unsigned*)nullptr, (unsigned*)nullptr, (unsigned*)nullptr, (unsigned*)nullptr, (int)n, 0, 24, stream);
    const size_t need = al(n * 4) * 4 + al(tmp) + 256;
    if (needed) *needed = need;
    if (!scratch || scratch_bytes < need) return cudaSuccess;
    if (ch.order_state != 0 && n <= sweep_cluster_capacity(ch)) {
        if (ch.order_state == 1) {
            if (sweep_order_cluster(ch, d_raw, n, d_order, scratch, stream) == cudaSuccess) return cudaSuccess;
            if (ch.cluster_size < 0) ch.order_state = 0;   // else: only this sweep is too long for the cluster
        } else {
            // first uses: run both, compare on the device, keep the cluster kernel only if the orders are identical
            char* q = static_cast<char*>(scratch) + al(n * 4) * 3 + al(tmp);
            unsigned* ref = reinterpret_cast<unsigned*>(q);                      // the 4th n-word array
            unsigned* cnt = reinterpret_cast<unsigned*>(q + al(n * 4));
            ch.order_state = 0;
            cudaError_t e = sweep_order_cub(d_raw, n, ref, scratch, tmp, stream);
            if (e != cudaSuccess) return e;
            unsigned mism = 1u;
            if (sweep_order_cluster(ch, d_raw, n, d_order, scratch, stream) == cudaSuccess) {
                cudaMemsetAsync(cnt, 0, 4, stream);
                k_order_mismatch<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(d_order, ref, n, cnt);
                if (cudaMemcpyAsync(&mism, cnt, 4, cudaMemcpyDeviceToHost, stream) != cudaSuccess || cudaStreamSynchronize(stream) != cudaSuccess) { cudaGetLastError(); mism = 1u; }
            }
            if (mism == 0u) { ch.order_state = --ch.order_checks_left > 0 ? -1 : 1; return cudaSuccess; }
            return cudaMemcpyAsync(d_order, ref, (size_t)n * 4, cudaMemcpyDeviceToDevice, stream);   // keep CUB's order, and CUB from now on
        }
    }
    return sweep_order_cub(d_raw, n, d_order, scratch, tmp, stream);
}

// ---------------------------------------------------------------------------------------------------------
// The compiled instances of the fast and split forms, keyed by the KernelChoice fields that select them.  Debug instances
// are loaded lazily at their first launch: only srl_build_plane_residuals asks for debug outputs, and it drives its pass
// from the host, so no persistent ESIKF block can be spinning while one loads.
typedef void (*FastFn)(const PassArgs);
struct FastInstance { int minb, lpk; FastFn fn, dbg; };
static const FastInstance kFast[] = {
    {4, 1, k1_fast<false, 4, 2, 1>, k1_fast<true, 4, 2, 1>}, {4, 2, k1_fast<false, 4, 2, 2>, k1_fast<true, 4, 2, 2>},
    {4, 4, k1_fast<false, 4, 2, 4>, k1_fast<true, 4, 2, 4>}, {5, 1, k1_fast<false, 5, 2, 1>, k1_fast<true, 5, 2, 1>},
    {5, 2, k1_fast<false, 5, 2, 2>, k1_fast<true, 5, 2, 2>}, {5, 4, k1_fast<false, 5, 2, 4>, k1_fast<true, 5, 2, 4>},
    {6, 1, k1_fast<false, 6, 2, 1>, k1_fast<true, 6, 2, 1>}, {6, 2, k1_fast<false, 6, 2, 2>, k1_fast<true, 6, 2, 2>},
    {6, 4, k1_fast<false, 6, 2, 4>, k1_fast<true, 6, 2, 4>}, {8, 1, k1_fast<false, 8, 2, 1>, k1_fast<true, 8, 2, 1>},
    {8, 2, k1_fast<false, 8, 2, 2>, k1_fast<true, 8, 2, 2>}, {8, 4, k1_fast<false, 8, 2, 4>, k1_fast<true, 8, 2, 4>}};
struct ScanInstance { int lpk, minb; FastFn fn; };
static const ScanInstance kScan[] = {
    {4, 8, k1_scan<4, 14, 8>}, {4, 6, k1_scan<4, 14, 6>}, {2, 8, k1_scan<2, 20, 8>}, {2, 6, k1_scan<2, 20, 6>}};
struct FitInstance { int minb; FastFn fn; };
static const FitInstance kFit[] = {{4, k1_fit<false, 4>}, {5, k1_fit<false, 5>}, {6, k1_fit<false, 6>}};
static const FastFn kFitDebug = k1_fit<true, 4>;

static FastFn pick_fast(const KernelChoice& ch, bool debug) {
    for (const FastInstance& i : kFast)
        if (i.minb == ch.fast_minb && i.lpk == ch.fast_lpk) return debug ? i.dbg : i.fn;
    return nullptr;
}
static FastFn pick_scan(const KernelChoice& ch) {
    for (const ScanInstance& i : kScan)
        if (i.lpk == ch.split_lpk && i.minb == ch.scan_minb) return i.fn;
    return nullptr;
}
static FastFn pick_fit(const KernelChoice& ch, bool debug) {
    if (debug) return kFitDebug;
    for (const FitInstance& i : kFit)
        if (i.minb == ch.fit_minb) return i.fn;
    return nullptr;
}

// one group of 32 / lanes-per-keypoint keypoints per warp when it fits (the block scheduler then balances the waves),
// grid-stride beyond that
cudaError_t launch_k1_fast(const srl_ctx* ctx, const PassArgs& a, long long n, bool debug) {
    const FastFn fn = pick_fast(ctx->choice, debug);
    if (!fn) return cudaErrorInvalidDeviceFunction;
    const long long kpw = 32 / ctx->choice.fast_lpk;
    const long long n_groups = (n + kpw - 1) / kpw;
    const long long grid = std::max<long long>(1, std::min<long long>((n_groups + kFastWarps - 1) / kFastWarps, ctx->max_grid));
    fn<<<(unsigned)grid, kFastThreads, 0, ctx->stream>>>(a);
    return cudaGetLastError();
}

// k1_scan then k1_fit on the same stream
cudaError_t launch_k1_split(const srl_ctx* ctx, const PassArgs& a, long long n, bool debug, bool pdl) {
    const FastFn scan = pick_scan(ctx->choice), fit = pick_fit(ctx->choice, debug);
    if (!scan || !fit) return cudaErrorInvalidDeviceFunction;
    const long long kpw = 32 / ctx->choice.split_lpk;
    const long long n_groups = (n + kpw - 1) / kpw;
    const long long grid_a = std::max<long long>(1, std::min<long long>((n_groups + 3) / 4, 1 << 20));
    cudaError_t e = launch_pass_kernel(scan, a, (unsigned)grid_a, kScanThreads, 0, ctx->stream, pdl);
    if (e != cudaSuccess) return e;
    const long long grid_b = std::max<long long>(1, std::min<long long>(((n + 31) / 32 + kFastWarps - 1) / kFastWarps, ctx->max_grid));
    return launch_pass_kernel(fit, a, (unsigned)grid_b, kFastThreads, 0, ctx->stream, pdl);
}

cudaError_t preload_fast_kernels(const KernelChoice& ch, size_t* max_local) {
    for (const FastFn fn : {pick_scan(ch), pick_fit(ch, false), pick_fast(ch, false)}) {
        const cudaError_t e = preload_kernel((const void*)fn, max_local);
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

}  // namespace srl
