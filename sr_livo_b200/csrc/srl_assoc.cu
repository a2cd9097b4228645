// srl_assoc.cu — K1: the fused scan-matching pass for sm_90a.
//
// One launch = one ESIKF pass over this rank's keypoint shard, replacing the body of
// lioOptimization::buildPlaneResiduals (src/optimize.cpp:18-131) plus the H_x/h assembly and the
// HTH / H^T h products (src/optimize.cpp:160-170,235,239):
//
//   prologue (thread per keypoint)  raw -> body -> world (FP64, same operation order as the reference,
//                                    no FMA contraction) -> voxel key by truncation (:38,:372-374)
//   phase 1 (warp per keypoint)     27/125 hash probes by 27/125 lanes (16 B slot loads), voxels ordered by
//                                    a conservative point-to-cell lower bound, candidate distances in FP64
//                                    from the FP32 map points, K-best list kept sorted across lanes with
//                                    warp shuffles; a voxel whose lower bound exceeds the current K-th
//                                    distance ends the scan (the reference visits all of them: :379-405).
//                                    Order = (distance^2, reference visit index): equal to the reference's
//                                    heap walk whenever no exact tie exists.
//   phase 2 (thread per keypoint)   plane fit, weight, signed distance, gate, 1x6 Jacobian (srl_math.cuh)
//   reduction                       32-component register transpose-reduce per group of 32 keypoints ->
//                                    per-warp -> per-block -> last block sums block partials in fixed order
//                                    (no FP64 atomics on the result: run-to-run deterministic).
//
// The 32-double result block: [0..20] HTH upper triangle (row-major a<=b), [21..26] H^T h, [27] sum d^2,
// [28] residuals, [29] keypoints with a full neighbourhood, [30] map points scanned, [31] NaN-planarity count.
#include <cstdlib>

#include "srl_internal.h"

namespace srl {

__constant__ signed char c_off[125 * 4];   // voxel offsets ordered by |offset|^2; first 27 = the nb=1 cube

constexpr unsigned FULL = 0xffffffffu;
constexpr int NBS = 33;   // padded stride of the per-warp neighbour tile (bank-conflict free both ways)
typedef unsigned long long u64;

// (distance^2 bits, reference visit index) lexicographic order on integers: distances are non-negative doubles, so
// their bit patterns order like the values; no FP64 compares, no branches.
__device__ __forceinline__ bool key_less(u64 da, unsigned ia, u64 db, unsigned ib) {
    return (da < db) | ((da == db) & (ia < ib));
}
__device__ __forceinline__ float warp_min_pos(float x) {   // x >= 0 (or +inf): uint order == float order
    return __uint_as_float(__reduce_min_sync(FULL, __float_as_uint(x)));
}

// the K neighbours of this lane's keypoint: float indices into the block pool, gathered from L1/L2 in phase 2
struct TileNb {
    const float* blocks; const unsigned* tile; int lane;
    __device__ __forceinline__ bool use(int) const { return true; }
    __device__ __forceinline__ void get(int j, float& x, float& y, float& z) const {
        const float4 p = __ldg(reinterpret_cast<const float4*>(blocks + tile[j * NBS + lane]));
        x = p.x; y = p.y; z = p.z;
    }
};

// 32x32 transpose-reduce: on return lane l holds sum over lanes of v[l] (31 shuffles instead of 160).
__device__ __forceinline__ double transpose_reduce32(double (&v)[32], int lane) {
#pragma unroll
    for (int s = 16; s >= 1; s >>= 1) {
        const bool upper = (lane & s) != 0;
#pragma unroll
        for (int i = 0; i < s; ++i) {
            const double send = upper ? v[i] : v[i + s];
            const double keep = upper ? v[i + s] : v[i];
            v[i] = keep + __shfl_xor_sync(FULL, send, s);
        }
    }
    return v[0];
}

// one chunk (<= 32 voxels) of the probed neighbourhood, sorted by lower bound: lane r holds the r-th nearest voxel
struct ChunkView {
    unsigned cnt, blk;
    int vis;
    float lb;
    int n_present;
};

__device__ __forceinline__ ChunkView sort_chunk(unsigned cnt, unsigned blk, int vis, float lb, int lane) {
    unsigned key = cnt ? ((__float_as_uint(lb) & ~31u) | (unsigned)lane) : 0xffffffffu;
#pragma unroll
    for (int kk = 2; kk <= 32; kk <<= 1) {
#pragma unroll
        for (int j = kk >> 1; j > 0; j >>= 1) {
            const unsigned other = __shfl_xor_sync(FULL, key, j);
            const bool up = (lane & kk) == 0, lower = (lane & j) == 0;
            key = (lower == up) ? min(key, other) : max(key, other);
        }
    }
    const int src = (int)(key & 31u);
    ChunkView v;
    v.cnt = __shfl_sync(FULL, cnt, src);
    v.blk = __shfl_sync(FULL, blk, src);
    v.vis = __shfl_sync(FULL, vis, src);
    v.lb = __uint_as_float(key & ~31u);   // mantissa truncated downward: still a lower bound
    v.n_present = __popc(__ballot_sync(FULL, key != 0xffffffffu));
    return v;
}

struct KpQuery {          // warp-uniform description of the keypoint being associated
    double px, py, pz;    // world position (FP64, reference operation order)
    float ofx, ofy, ofz;  // float origin (the keypoint's voxel corner)
    float rfx, rfy, rfz;  // p - origin, rounded to float
};

// ---------------------------------------------------------------------------------------------------------
// Fast selection: FP32 distances with a proven error bound.
//   d2f differs from the exact FP64 d2 by at most eps (see DESIGN.md "K1 selection"): if the (K+1)-th smallest
//   d2f over everything that could matter exceeds the K-th by more than 2*eps, the K lanes hold exactly the K
//   nearest points (as a set); the exact FP64 finish then orders them.  Otherwise the caller falls back to
//   select_exact.  Voxels are skipped only when their lower bound exceeds kth + 3*eps.
// ---------------------------------------------------------------------------------------------------------
template <int NCH>
__device__ __forceinline__ bool select_fast(const float* __restrict__ blocks, const ChunkView (&cv)[NCH], const KpQuery& q, int K,
                                            float eps, int lane, float& bf, unsigned& bid, int& nfound, long long& scanned) {
    const float INF = __int_as_float(0x7f800000);
    bf = INF; bid = 0xffffffffu;
    float kth = INF, rej = INF, r_ev = INF;
    bool empty = true;
#pragma unroll
    for (int ch = 0; ch < NCH; ++ch) {
        for (int r = 0; r < cv[ch].n_present; ++r) {
            const float lb_r = __shfl_sync(FULL, cv[ch].lb, r);
            if (lb_r > kth + 3.f * eps) break;   // every remaining voxel of this chunk is farther still
            const unsigned b = __shfl_sync(FULL, cv[ch].blk, r);
            const int cn = (int)__shfl_sync(FULL, cv[ch].cnt, r);
            const int v = __shfl_sync(FULL, cv[ch].vis, r);
            scanned += cn;
            float d2f = INF;
            unsigned id = 0xffffffffu;
            if (lane < cn) {
                const float4 mp = __ldg(reinterpret_cast<const float4*>(blocks + (size_t)b * kBlockFloats) + lane);
                const float dx = (mp.x - q.ofx) - q.rfx;
                const float dy = (mp.y - q.ofy) - q.rfy;
                const float dz = (mp.z - q.ofz) - q.rfz;
                d2f = dx * dx + dy * dy + dz * dz;
                id = ((unsigned)v << 5) | (unsigned)lane;
            }
            if (empty) {
                // first voxel: a bitonic sort of the 32 lanes initialises the list
#pragma unroll
                for (int kk = 2; kk <= 32; kk <<= 1) {
#pragma unroll
                    for (int j = kk >> 1; j > 0; j >>= 1) {
                        const float od = __shfl_xor_sync(FULL, d2f, j);
                        const unsigned oi = __shfl_xor_sync(FULL, id, j);
                        const bool up = (lane & kk) == 0, lower = (lane & j) == 0;
                        const bool take = (lower == up) ? (od < d2f) : (d2f < od);
                        d2f = take ? od : d2f;
                        id = take ? oi : id;
                    }
                }
                rej = fminf(rej, lane >= K ? d2f : INF);   // sorted entries beyond K are rejections
                if (lane < K) { bf = d2f; bid = id; }
                empty = false;
                kth = __shfl_sync(FULL, bf, K - 1);
            } else {
                const bool pass = d2f < kth;
                rej = fminf(rej, pass ? INF : d2f);
                unsigned m = __ballot_sync(FULL, pass);
                while (m) {
                    const int j = __ffs(m) - 1;
                    m &= m - 1;
                    const float nv = __shfl_sync(FULL, d2f, j);
                    const unsigned ni = __shfl_sync(FULL, id, j);
                    if (nv < kth) {
                        const int pos = __popc(__ballot_sync(FULL, bf <= nv));
                        const float uf = __shfl_up_sync(FULL, bf, 1);
                        const unsigned ui = __shfl_up_sync(FULL, bid, 1);
                        r_ev = fminf(r_ev, kth);            // the old K-th entry leaves the list
                        if (lane < K) {
                            bf = (lane > pos) ? uf : ((lane == pos) ? nv : bf);
                            bid = (lane > pos) ? ui : ((lane == pos) ? ni : bid);
                        }
                        kth = __shfl_sync(FULL, bf, K - 1);
                    } else {
                        r_ev = fminf(r_ev, nv);             // threshold tightened meanwhile
                    }
                }
            }
        }
    }
    nfound = __popc(__ballot_sync(FULL, lane < K && bf < INF));
    if (nfound < K) return true;   // every candidate seen is in the list, nothing was skipped (kth stayed +inf)
    const float rmin = fminf(warp_min_pos(rej), r_ev);
    return rmin > kth + 2.f * eps;
}

// ---------------------------------------------------------------------------------------------------------
// Exact selection (fallback for ambiguous keypoints): FP64 distances in the reference's operation order
// (src/optimize.cpp:394-395), K-best list ordered by (distance^2 bits, reference visit index).
// ---------------------------------------------------------------------------------------------------------
template <int NCH>
__device__ __forceinline__ void select_exact(const float* __restrict__ blocks, const ChunkView (&cv)[NCH], const KpQuery& q, int K,
                                             int lane, u64& bd, unsigned& bid, int& nfound, long long& scanned) {
    const u64 KINF = 0x7ff0000000000000ull;
    bd = KINF; bid = 0xffffffffu;
    u64 kth_d = KINF;
    unsigned kth_id = 0xffffffffu;
    bool empty = true;
#pragma unroll
    for (int ch = 0; ch < NCH; ++ch) {
        for (int r = 0; r < cv[ch].n_present; ++r) {
            const float lb_r = __shfl_sync(FULL, cv[ch].lb, r);
            if ((u64)__double_as_longlong((double)lb_r) > kth_d) break;
            const unsigned b = __shfl_sync(FULL, cv[ch].blk, r);
            const int cn = (int)__shfl_sync(FULL, cv[ch].cnt, r);
            const int v = __shfl_sync(FULL, cv[ch].vis, r);
            scanned += cn;
            u64 d = KINF;
            unsigned id = 0xffffffffu;
            if (lane < cn) {
                const float4 mp = __ldg(reinterpret_cast<const float4*>(blocks + (size_t)b * kBlockFloats) + lane);
                const double mx = (double)mp.x, my = (double)mp.y, mz = (double)mp.z;
                const double dx = SRL_SUB(mx, q.px), dy = SRL_SUB(my, q.py), dz = SRL_SUB(mz, q.pz);
                d = (u64)__double_as_longlong(SRL_ADD(SRL_MUL(dx, dx), SRL_ADD(SRL_MUL(dy, dy), SRL_MUL(dz, dz))));
                id = ((unsigned)v << 5) | (unsigned)lane;
            }
            if (empty) {
#pragma unroll
                for (int kk = 2; kk <= 32; kk <<= 1) {
#pragma unroll
                    for (int j = kk >> 1; j > 0; j >>= 1) {
                        const u64 od = __shfl_xor_sync(FULL, d, j);
                        const unsigned oi = __shfl_xor_sync(FULL, id, j);
                        const bool up = (lane & kk) == 0, lower = (lane & j) == 0;
                        const bool take = (lower == up) ? key_less(od, oi, d, id) : key_less(d, id, od, oi);
                        d = take ? od : d;
                        id = take ? oi : id;
                    }
                }
                if (lane < K) { bd = d; bid = id; }
                empty = false;
            } else {
                unsigned m = __ballot_sync(FULL, key_less(d, id, kth_d, kth_id));
                while (m) {
                    const int j = __ffs(m) - 1;
                    m &= m - 1;
                    const u64 nd = __shfl_sync(FULL, d, j);
                    const unsigned ni = __shfl_sync(FULL, id, j);
                    if (key_less(nd, ni, kth_d, kth_id)) {
                        const int pos = __popc(__ballot_sync(FULL, key_less(bd, bid, nd, ni)));
                        const u64 ud = __shfl_up_sync(FULL, bd, 1);
                        const unsigned ui = __shfl_up_sync(FULL, bid, 1);
                        if (lane < K) {
                            bd = (lane > pos) ? ud : ((lane == pos) ? nd : bd);
                            bid = (lane > pos) ? ui : ((lane == pos) ? ni : bid);
                        }
                        kth_d = __shfl_sync(FULL, bd, K - 1);
                        kth_id = __shfl_sync(FULL, bid, K - 1);
                    }
                }
                continue;
            }
            kth_d = __shfl_sync(FULL, bd, K - 1);
            kth_id = __shfl_sync(FULL, bid, K - 1);
        }
    }
    nfound = __popc(__ballot_sync(FULL, lane < K && bd < KINF));
}

// The pass's result straight into mapped pinned host memory (one warp): 32 sums, system fence, sequence flag.  The host
// spins on the flag (srl_api.cu: wait_host_result) — no D2H copy, no stream synchronize on the critical path.
__device__ __forceinline__ void publish_to_host(const K1Args& A, double tot, int lane) {
    if (!A.host_out) return;
    A.host_out[lane] = tot;
    __syncwarp();
    if (lane == 0) st_release_sys(reinterpret_cast<unsigned long long*>(A.host_out + 32), A.host_seq);
}

template <int NCH, bool DEBUG, int MINB>
__global__ void __launch_bounds__(kK1Threads, MINB) k1_assoc(const __grid_constant__ K1Args A) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    __shared__ PassConst s_c;
    if (!load_pass_const(A.dev, A.wait_pose, A.pose_ticket, A.end_ticket, A.c, s_c)) return;   // device-resident loop already ended: nothing to do
    const PassConst& c = s_c;
    const int K = c.K;
    const int nb = c.nb;
    const int W = 2 * nb + 1;
    const int V = W * W * W;

    // per-warp shared memory: K x 33 point indices (into the block pool), then block index per visited voxel
    const size_t warp_bytes = (size_t)(K * NBS) * sizeof(unsigned) + 128 * sizeof(int);
    unsigned* tile = reinterpret_cast<unsigned*>(smem_raw + warp * warp_bytes);
    int* sblk = reinterpret_cast<int*>(tile + K * NBS);

    const float size_f = (float)c.size;
    const float lb_margin = 1e-5f * size_f;
    const float eps = 1e-4f * size_f * size_f * A.eps_scale;   // bound on |d2f - d2| (DESIGN.md), with margin

    double acc = 0.0;                 // lane i accumulates component i of the 32-double result
    long long scanned = 0;            // warp-uniform: map points whose distance was evaluated
    unsigned fallbacks = 0;           // warp-uniform: keypoints that needed the exact selection

    // fallback launch with nothing flagged in this pass (the usual case): one warp forwards the fast form's sums
    if (A.only_flagged && A.stats && __ldcg(A.stats + 2) == 0ull) {
        if (blockIdx.x == 0 && warp == 0) {
            double tot = A.prev_out32 ? A.prev_out32[lane] : 0.0;
            const bool finalised = __ldcg(A.stats + 3) != 0ull;   // k1_fit already finalised the pass (exchange, publication)
            __syncwarp();
            if (A.comm.world > 1 && !finalised) tot = comm_exchange(A.comm, tot, lane);
            if (lane == 0 && finalised) A.stats[3] = 0ull;
            A.out32[lane] = tot;
            publish_to_host(A, tot, lane);
            if (!finalised) publish_sums_to_loop(A.dev, A.pose_ticket, tot, lane);
        }
        return;
    }

    const long long n = A.k_end - A.k_begin;
    const long long n_groups = (n + 31) / 32;
    // block-minor assignment: consecutive groups go to different blocks (SMs), so every SM gets ~the same share
    const long long G = gridDim.x;

    for (long long g = (long long)blockIdx.x + (long long)warp * G; g < n_groups; g += G * kK1Warps) {
        // ------------------------------------------------------------------ prologue: thread per keypoint
        const long long k = A.k_begin + g * 32 + lane;
        const bool in_shard = k < A.k_end;
        // fallback launch: only the keypoints k1_fast flagged are ours
        const bool valid = in_shard && (!A.only_flagged || A.only_flagged[k] != 0);
        if (A.only_flagged && !__any_sync(FULL, valid)) continue;
        double bx = 0, by = 0, bz = 0, pwx = 0, pwy = 0, pwz = 0;
        int kx = 0, ky = 0, kz = 0;
        float relx = 0, rely = 0, relz = 0;       // p - exact voxel corner (for the cell lower bounds)
        float ofx = 0, ofy = 0, ofz = 0, rfx = 0, rfy = 0, rfz = 0;   // float origin and p - origin
        bool in_range = false;
        if (valid) {
            const double rx = A.raw[3 * k], ry = A.raw[3 * k + 1], rz = A.raw[3 * k + 2];
            double tx, ty, tz;
            matvec3_exact(c.R_il, rx, ry, rz, tx, ty, tz);                 // R_il * raw
            bx = SRL_ADD(tx, c.t_il[0]); by = SRL_ADD(ty, c.t_il[1]); bz = SRL_ADD(tz, c.t_il[2]);   // + t_il  (:83)
            matvec3_exact(c.Rn, bx, by, bz, tx, ty, tz);                   // R * (...)
            pwx = SRL_ADD(tx, c.t[0]); pwy = SRL_ADD(ty, c.t[1]); pwz = SRL_ADD(tz, c.t[2]);         // + t     (:38)
            const double qx = voxel_quotient(pwx, c), qy = voxel_quotient(pwy, c), qz = voxel_quotient(pwz, c);   // :372-374
            in_range = fabs(qx) < 32765.0 && fabs(qy) < 32765.0 && fabs(qz) < 32765.0;   // (short) cast is UB beyond
            if (in_range) {
                kx = (int)qx; ky = (int)qy; kz = (int)qz;   // truncation toward zero, like static_cast<short>
                const double cx = (double)kx * c.size, cy = (double)ky * c.size, cz = (double)kz * c.size;
                relx = (float)(pwx - cx); rely = (float)(pwy - cy); relz = (float)(pwz - cz);
                ofx = (float)cx; ofy = (float)cy; ofz = (float)cz;
                rfx = (float)(pwx - (double)ofx); rfy = (float)(pwy - (double)ofy); rfz = (float)(pwz - (double)ofz);
            }
            if (DEBUG && A.dbg_world) { A.dbg_world[3 * k] = pwx; A.dbg_world[3 * k + 1] = pwy; A.dbg_world[3 * k + 2] = pwz; }
        }
        int my_count = 0;   // neighbours found for this lane's keypoint (0 = not a full neighbourhood)

        // ------------------------------------------------------------------ phase 1: warp per keypoint
        const int n_in_group = (int)min((long long)32, n - g * 32);
        for (int kp = 0; kp < n_in_group; ++kp) {
            if (!__shfl_sync(FULL, (int)in_range, kp)) continue;
            KpQuery q;
            q.px = __shfl_sync(FULL, pwx, kp); q.py = __shfl_sync(FULL, pwy, kp); q.pz = __shfl_sync(FULL, pwz, kp);
            q.ofx = __shfl_sync(FULL, ofx, kp); q.ofy = __shfl_sync(FULL, ofy, kp); q.ofz = __shfl_sync(FULL, ofz, kp);
            q.rfx = __shfl_sync(FULL, rfx, kp); q.rfy = __shfl_sync(FULL, rfy, kp); q.rfz = __shfl_sync(FULL, rfz, kp);
            const int ckx = __shfl_sync(FULL, kx, kp), cky = __shfl_sync(FULL, ky, kp), ckz = __shfl_sync(FULL, kz, kp);
            const float rlx = __shfl_sync(FULL, relx, kp), rly = __shfl_sync(FULL, rely, kp), rlz = __shfl_sync(FULL, relz, kp);

            // ---- probes: lane o handles voxel offset o of the chunk; then order each chunk by lower bound
            ChunkView cv[NCH];
            int total = 0;
#pragma unroll
            for (int ch = 0; ch < NCH; ++ch) {
                unsigned cnt = 0, blk = 0;
                int vis = 0;
                float lb = 0.f;
                const int o = ch * 32 + lane;
                if (o < V) {
                    const int ox = c_off[4 * o], oy = c_off[4 * o + 1], oz = c_off[4 * o + 2];
                    const int vx = ckx + ox, vy = cky + oy, vz = ckz + oz;
                    vis = ((ox + nb) * W + (oy + nb)) * W + (oz + nb);   // reference scan order (:379-381)
                    unsigned b, cn;
                    if (map_find(A.slots, A.mask, vx, vy, vz, b, cn) && (int)cn >= c.thr_occ) {   // :386-390
                        cnt = cn; blk = b;
                        sblk[vis] = (int)b;
                        // conservative lower bound of the distance to any point stored under key (vx,vy,vz):
                        // cell k>0 spans [k,k+1), k<0 spans (k-1,k], k=0 spans (-1,1) (truncation toward zero)
                        const float lox = (float)((vx > 0 ? vx : vx - 1) - ckx) * size_f, hix = (float)((vx < 0 ? vx : vx + 1) - ckx) * size_f;
                        const float loy = (float)((vy > 0 ? vy : vy - 1) - cky) * size_f, hiy = (float)((vy < 0 ? vy : vy + 1) - cky) * size_f;
                        const float loz = (float)((vz > 0 ? vz : vz - 1) - ckz) * size_f, hiz = (float)((vz < 0 ? vz : vz + 1) - ckz) * size_f;
                        const float gx = fmaxf(fmaxf(lox - rlx, rlx - hix) - lb_margin, 0.f);
                        const float gy = fmaxf(fmaxf(loy - rly, rly - hiy) - lb_margin, 0.f);
                        const float gz = fmaxf(fmaxf(loz - rlz, rlz - hiz) - lb_margin, 0.f);
                        lb = (gx * gx + gy * gy + gz * gz) * 0.999999f;
                    }
                }
                total += (int)cnt;
                cv[ch] = sort_chunk(cnt, blk, vis, lb, lane);
            }
            total = __reduce_add_sync(FULL, total);
            if (total < c.Kmin) continue;   // fewer candidates than min_number_neighbors: :78 will skip it
            __syncwarp();                   // sblk[] visible to the whole warp

            // ---- K nearest: FP32 selection with exact FP64 finish, or the exact selection when ambiguous
            float bf;
            unsigned bid;
            int nfound;
            u64 key = ~0ull;
            const bool sure = select_fast<NCH>(A.blocks, cv, q, K, eps, lane, bf, bid, nfound, scanned);
            if (!sure) { select_exact<NCH>(A.blocks, cv, q, K, lane, key, bid, nfound, scanned); ++fallbacks; }

            if (nfound >= c.Kmin) {
                unsigned pt = 0;
                if (lane < nfound) {
                    pt = (unsigned)sblk[bid >> 5] * kBlockFloats + 4u * (bid & 31u);
                    if (sure) {   // exact distance of the selected points, reference operation order (:394-395)
                        const float4 mp = __ldg(reinterpret_cast<const float4*>(A.blocks + pt));
                        const double mx = (double)mp.x, my = (double)mp.y, mz = (double)mp.z;
                        const double dx = SRL_SUB(mx, q.px), dy = SRL_SUB(my, q.py), dz = SRL_SUB(mz, q.pz);
                        key = (u64)__double_as_longlong(SRL_ADD(SRL_MUL(dx, dx), SRL_ADD(SRL_MUL(dy, dy), SRL_MUL(dz, dz))));
                    }
                } else {
                    key = ~0ull; bid = 0xffffffffu;
                }
                if (sure) {
                    // the FP32 order is almost always the exact order; sort exactly only if an inversion shows up
                    const u64 pk = __shfl_up_sync(FULL, key, 1);
                    const unsigned pi = __shfl_up_sync(FULL, bid, 1);
                    const bool inv = lane > 0 && lane < nfound && key_less(key, bid, pk, pi);
                    if (__any_sync(FULL, inv)) {
#pragma unroll
                        for (int kk = 2; kk <= 32; kk <<= 1) {
#pragma unroll
                            for (int j = kk >> 1; j > 0; j >>= 1) {
                                const u64 od = __shfl_xor_sync(FULL, key, j);
                                const unsigned oi = __shfl_xor_sync(FULL, bid, j);
                                const bool up = (lane & kk) == 0, lower = (lane & j) == 0;
                                const bool take = (lower == up) ? key_less(od, oi, key, bid) : key_less(key, bid, od, oi);
                                key = take ? od : key;
                                bid = take ? oi : bid;
                            }
                        }
                        if (lane < nfound) pt = (unsigned)sblk[bid >> 5] * kBlockFloats + 4u * (bid & 31u);
                    }
                }
                if (lane < nfound) {
                    tile[lane * NBS + kp] = pt;
                    if (DEBUG) {
                        const long long kk = A.k_begin + g * 32 + kp;
                        const int v = (int)(bid >> 5), i = (int)(bid & 31u);
                        if (A.dbg_nbr) {
                            short* d = A.dbg_nbr + (kk * K + lane) * 4;
                            d[0] = (short)(ckx + v / (W * W) - nb);
                            d[1] = (short)(cky + (v / W) % W - nb);
                            d[2] = (short)(ckz + v % W - nb);
                            d[3] = (short)i;
                        }
                        if (A.dbg_nbr_dist) A.dbg_nbr_dist[kk * K + lane] = sqrt(__longlong_as_double((long long)key));
                    }
                }
                if (lane == kp) my_count = nfound;
            }
            __syncwarp();   // sblk[] is rewritten by the next keypoint's probes
        }
        __syncwarp();

        // ------------------------------------------------------------------ phase 2: thread per keypoint
        double v[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = 0.0;
        int status = 0;
        if (valid && my_count > 0) {
            PlaneRow row;
            TileNb acc_nb{A.blocks, tile, lane};
            float n0x, n0y, n0z;
            acc_nb.get(0, n0x, n0y, n0z);
            plane_residual<0>(acc_nb, my_count, (double)n0x, (double)n0y, (double)n0z, c, pwx, pwy, pwz, bx, by, bz, row);
            status = row.accepted ? 2 : 1;
            v[29] = 1.0;
            v[31] = (double)row.nan_planarity;
            const double h = row.distance * row.weight;   // :169
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
                v[27] = row.distance * row.distance;   // :104
                v[28] = 1.0;
            }
            if (A.rows) {   // per-keypoint rows for the ordered max_num_residuals cap (:107)
                double* rr = A.rows + 8 * k;
#pragma unroll
                for (int i = 0; i < 6; ++i) rr[i] = row.J[i];
                rr[6] = h; rr[7] = row.distance * row.distance;
            }
            if (DEBUG && A.dbg_plane) {
                double* d = A.dbg_plane + 16 * k;
                d[0] = bx; d[1] = by; d[2] = bz; d[3] = row.nx; d[4] = row.ny; d[5] = row.nz;
#pragma unroll
                for (int i = 0; i < 6; ++i) d[6 + i] = row.accepted ? row.J[i] : 0.0;
                d[12] = row.offset; d[13] = row.distance; d[14] = row.weight; d[15] = row.a2D;
            }
        }
        if (valid && A.status) A.status[k] = status;
        acc += transpose_reduce32(v, lane);
        __syncwarp();   // the neighbour tile is rewritten by the next group
    }
    if (lane == 30) acc += (double)scanned;
    if (A.stats && lane == 0 && fallbacks) atomicAdd(A.stats, (unsigned long long)fallbacks);

    // ---------------------------------------------------------------------- block + grid reduction
    __shared__ double s_acc[kK1Warps][32];
    __shared__ bool s_last;
    s_acc[warp][lane] = acc;
    __syncthreads();
    if (warp == 0) {
        double s = 0.0;
#pragma unroll
        for (int w = 0; w < kK1Warps; ++w) s += s_acc[w][lane];
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
        double s = 0.0;
        for (int b = warp; b < (int)gridDim.x; b += kK1Warps) s += __ldcg(A.partials + (size_t)b * 32 + lane);
        s_acc[warp][lane] = s;
        __syncthreads();
        if (warp == 0) {
            double tot = 0.0;
#pragma unroll
            for (int w = 0; w < kK1Warps; ++w) tot += s_acc[w][lane];
            if (A.prev_out32) tot += A.prev_out32[lane];   // fallback launch: add k1_fast's sums (fixed order)
            if (A.comm.world > 1) tot = comm_exchange(A.comm, tot, lane);
            A.out32[lane] = tot;
            if (lane == 0) { *A.ticket = 0u; if (A.only_flagged && A.stats) A.stats[2] = 0ull; }
            publish_to_host(A, tot, lane);
            publish_sums_to_loop(A.dev, A.pose_ticket, tot, lane);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// K2: ordered residual cap (src/optimize.cpp:99,107).  Single block.  The reference loop stops after
// the first full-neighbourhood keypoint k* at which the running count of accepted residuals is >= cap,
// so the rows that count are the accepted ones with k <= k*.  cap >= 1: k* = the cap-th accepted
// keypoint; cap <= 0 (the compiled default -1): k* = the first keypoint with a full neighbourhood.
// state[0] = running accepted count, state[1] = k* found flag, state[2] = k*
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024, 1) k2_cap_reduce(const double* __restrict__ rows, int* __restrict__ status,
                                                          long long k_begin, long long k_end, int cap,
                                                          long long* __restrict__ state, double* __restrict__ out32,
                                                          int mark_unvisited) {
    __shared__ int s_scan[1024];
    __shared__ double s_red[32][33];
    __shared__ long long s_kstar;
    __shared__ int s_found;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    long long run_acc = state[0];
    if (tid == 0) { s_found = (int)state[1]; s_kstar = state[2]; }
    __syncthreads();
    double acc[29];
#pragma unroll
    for (int i = 0; i < 29; ++i) acc[i] = 0.0;
    double n_full = 0.0, n_nan = 0.0;
    for (long long base = k_begin; base < k_end && !s_found; base += 1024) {
        const long long k = base + tid;
        const int st = (k < k_end) ? status[k] : 0;
        const int a = (st == 2) ? 1 : 0;
        // inclusive block scan of accepted flags
        s_scan[tid] = a;
        __syncthreads();
        for (int off = 1; off < 1024; off <<= 1) {
            int t = (tid >= off) ? s_scan[tid - off] : 0;
            __syncthreads();
            s_scan[tid] += t;
            __syncthreads();
        }
        const long long incl = run_acc + s_scan[tid];
        // k* candidate: full neighbourhood and running count >= cap
        const bool is_kstar_cand = (st >= 1) && (incl >= (long long)cap);
        // first such k in this chunk
        unsigned long long cand = is_kstar_cand ? (unsigned long long)k : ~0ull;
        // block min via shared
        __shared__ unsigned long long s_min[32];
        for (int s = 16; s >= 1; s >>= 1) { unsigned long long o = __shfl_xor_sync(0xffffffffu, cand, s); cand = o < cand ? o : cand; }
        if (lane == 0) s_min[warp] = cand;
        __syncthreads();
        if (warp == 0) {
            unsigned long long m = s_min[lane];
            for (int s = 16; s >= 1; s >>= 1) { unsigned long long o = __shfl_xor_sync(0xffffffffu, m, s); m = o < m ? o : m; }
            if (lane == 0 && m != ~0ull) { s_found = 1; s_kstar = (long long)m; }
        }
        __syncthreads();
        const long long kstar = s_found ? s_kstar : (long long)0x7fffffffffffffffLL;
        if (k < k_end && k <= kstar) {
            if (st >= 1) n_full += 1.0;
            if (st >= 1 && rows[8 * k] != rows[8 * k]) n_nan += 1.0;   // NaN planarity -> NaN weight -> NaN Jacobian (the reference throws, :348)
            if (a) {
                const double* r = rows + 8 * k;
                int idx = 0;
#pragma unroll
                for (int p = 0; p < 6; ++p)
#pragma unroll
                    for (int q = p; q < 6; ++q) acc[idx++] += r[p] * r[q];
#pragma unroll
                for (int p = 0; p < 6; ++p) acc[21 + p] += r[p] * r[6];
                acc[27] += r[7];
                acc[28] += 1.0;
            }
        }
        run_acc += s_scan[1023];
        __syncthreads();
    }
    // keypoints after k* were never visited by the reference loop
    if (mark_unvisited && s_found)
        for (long long k = s_kstar + 1 + tid; k < k_end; k += 1024) status[k] = -1;
    // fixed-order block reduction of the 30 components
    double comps[31];
#pragma unroll
    for (int i = 0; i < 29; ++i) comps[i] = acc[i];
    comps[29] = n_full;
    comps[30] = n_nan;
    for (int i = 0; i < 31; ++i) {
        double x = comps[i];
        for (int s = 16; s >= 1; s >>= 1) x += __shfl_xor_sync(0xffffffffu, x, s);
        if (lane == 0) s_red[warp][i] = x;
    }
    __syncthreads();
    if (warp == 0 && lane < 31) {
        double tot = 0.0;
        for (int w = 0; w < 32; ++w) tot += s_red[w][lane];
        out32[lane == 30 ? 31 : lane] += tot;   // chunks append; [31] = NaN-planarity keypoints the reference loop reached
    }
    if (tid == 0) { state[0] = run_acc; state[1] = s_found; state[2] = s_kstar; }
}

// transformPoint over a sweep (src/utility.cpp:314-318): world = R(q) * (R_il * raw + t_il) + t
__global__ void k_transform(const double* __restrict__ raw, long long n, PassConst c, double* __restrict__ out) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    double tx, ty, tz;
    matvec3_exact(c.R_il, raw[3 * k], raw[3 * k + 1], raw[3 * k + 2], tx, ty, tz);
    const double bx = SRL_ADD(tx, c.t_il[0]), by = SRL_ADD(ty, c.t_il[1]), bz = SRL_ADD(tz, c.t_il[2]);
    matvec3_exact(c.Rq, bx, by, bz, tx, ty, tz);
    out[3 * k] = SRL_ADD(tx, c.t[0]); out[3 * k + 1] = SRL_ADD(ty, c.t[1]); out[3 * k + 2] = SRL_ADD(tz, c.t[2]);
}

// ---------------------------------------------------------------------------------------------
// host launchers
// ---------------------------------------------------------------------------------------------
static bool g_off_uploaded[64] = {false};

static void upload_offsets(int device) {
    if (device >= 0 && device < 64 && g_off_uploaded[device]) return;
    // all 125 offsets of the 5x5x5 cube ordered by squared norm; the 27 with |.|inf <= 1 come first
    signed char tab[125 * 4];
    int n = 0;
    for (int pass = 0; pass < 2; ++pass)
        for (int d2 = 0; d2 <= 12; ++d2)
            for (int x = -2; x <= 2; ++x)
                for (int y = -2; y <= 2; ++y)
                    for (int z = -2; z <= 2; ++z) {
                        const bool inner = x >= -1 && x <= 1 && y >= -1 && y <= 1 && z >= -1 && z <= 1;
                        if ((pass == 0) != inner) continue;
                        if (x * x + y * y + z * z != d2) continue;
                        tab[4 * n] = (signed char)x; tab[4 * n + 1] = (signed char)y; tab[4 * n + 2] = (signed char)z; tab[4 * n + 3] = 0;
                        ++n;
                    }
    cudaMemcpyToSymbol(c_off, tab, sizeof(tab));
    if (device >= 0 && device < 64) g_off_uploaded[device] = true;
}

size_t k1_smem_bytes(int K) { return (size_t)kK1Warps * ((size_t)(K * NBS) * sizeof(unsigned) + 128 * sizeof(int)); }

typedef void (*K1Fn)(const K1Args);
static int g_minb = -1;
void k1_set_min_blocks(int v) { if (v == 2 || v == 3 || v == 4) g_minb = v; }
int k1_min_blocks() {   // resident blocks per SM the kernel is compiled for; SRL_K1_MINB=2|3|4 selects the variant
    if (g_minb < 0) {
        const char* e = getenv("SRL_K1_MINB");
        int v = e ? atoi(e) : 3;
        g_minb = (v == 2 || v == 3 || v == 4) ? v : 3;
    }
    return g_minb;
}
template <int NCH, bool DBG>
static K1Fn pick_minb() {
    switch (k1_min_blocks()) {
        case 2: return k1_assoc<NCH, DBG, 2>;
        case 4: return k1_assoc<NCH, DBG, 4>;
        default: return k1_assoc<NCH, DBG, 3>;
    }
}
static K1Fn pick_k1(int nb, bool debug) {
    if (nb <= 1) return debug ? pick_minb<1, true>() : pick_minb<1, false>();
    return debug ? pick_minb<4, true>() : pick_minb<4, false>();
}

cudaError_t launch_k1(const K1Args& a, int grid, bool debug, int device, cudaStream_t stream, bool pdl) {
    upload_offsets(device);
    const size_t smem = k1_smem_bytes(a.c.K);
    K1Fn fn = pick_k1(a.c.nb, debug);
    cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    return launch_pass_kernel(fn, a, (unsigned)grid, kK1Threads, smem, stream, pdl);
}

cudaError_t preload_assoc_kernels(int device, int K, size_t* max_local) {
    upload_offsets(device);
    cudaFuncAttributes at;
    const size_t smem = k1_smem_bytes(K > 0 ? K : 20);
    for (int nb = 1; nb <= 2; ++nb) {
        K1Fn fn = pick_k1(nb, false);
        cudaError_t e = cudaFuncGetAttributes(&at, fn);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        if (at.localSizeBytes > *max_local) *max_local = at.localSizeBytes;
    }
    return cudaSuccess;
}

int k1_max_blocks_per_sm(int K, int nb) {
    int nblk = 0;
    K1Fn fn = pick_k1(nb, false);
    const size_t smem = k1_smem_bytes(K);
    cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nblk, fn, kK1Threads, smem) != cudaSuccess) return 1;
    return nblk < 1 ? 1 : nblk;
}

cudaError_t launch_k2(const double* rows, int* status, long long k_begin, long long k_end, int cap, long long* state,
                      double* out32, int mark_unvisited, cudaStream_t stream) {
    k2_cap_reduce<<<1, 1024, 0, stream>>>(rows, status, k_begin, k_end, cap, state, out32, mark_unvisited);
    return cudaGetLastError();
}

cudaError_t launch_transform(const double* raw, long long n, const PassConst& c, double* out, cudaStream_t stream) {
    if (n <= 0) return cudaSuccess;
    const int threads = 256;
    const long long blocks = (n + threads - 1) / threads;
    k_transform<<<(unsigned)blocks, threads, 0, stream>>>(raw, n, c, out);
    return cudaGetLastError();
}

}  // namespace srl
