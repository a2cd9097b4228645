// srl_api.cu — C-ABI glue: context, sweep residency, one ESIKF pass, the iterated update.
#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>

#include "srl_internal.h"

namespace srl {

int set_err(srl_ctx* ctx, int code, const std::string& msg) {
    if (ctx) ctx->err = msg;
    return code;
}
int cuda_fail(srl_ctx* ctx, cudaError_t e, const char* where) {
    if (ctx) ctx->err = std::string(where) + ": " + cudaGetErrorString(e);
    cudaGetLastError();   // clear sticky-less errors
    return SRL_CUDA_ERROR;
}
int ensure_scratch(srl_ctx* ctx, size_t bytes) {
    if (bytes <= ctx->scratch_bytes) return SRL_OK;
    if (ctx->d_scratch) { cudaStreamSynchronize(ctx->stream); cudaFree(ctx->d_scratch); ctx->d_scratch = nullptr; ctx->scratch_bytes = 0; }
    size_t want = bytes + bytes / 4;
    cudaError_t e = cudaMalloc(&ctx->d_scratch, want);
    if (e != cudaSuccess) return cuda_fail(ctx, e, "ensure_scratch/cudaMalloc");
    ctx->scratch_bytes = want;
    return SRL_OK;
}
int ensure_pinned(srl_ctx* ctx, size_t bytes) {
    if (bytes <= ctx->pinned_bytes) return SRL_OK;
    if (ctx->h_pinned) { cudaStreamSynchronize(ctx->stream); cudaFreeHost(ctx->h_pinned); ctx->h_pinned = nullptr; ctx->pinned_bytes = 0; }
    size_t want = bytes + bytes / 4;
    cudaError_t e = cudaMallocHost(&ctx->h_pinned, want);
    if (e != cudaSuccess) return cuda_fail(ctx, e, "ensure_pinned/cudaMallocHost");
    ctx->pinned_bytes = want;
    return SRL_OK;
}

// fold a finished event pair into the running totals.  Pairs alternate between passes and the pair of the PREVIOUS pass is
// collected when the next one starts: its last kernel (the fallback launch, which on one GPU is off the host's critical
// path) has long finished by then, so timing never makes the host wait for the device.
static void timing_collect_pair(srl_ctx* ctx, int i) {
    if (!ctx->ev_pending[i]) return;
    float ms = 0.f;
    cudaEventSynchronize(ctx->ev1[i]);
    if (cudaEventElapsedTime(&ms, ctx->ev0[i], ctx->ev1[i]) == cudaSuccess) { ctx->k1_ms += ms; ctx->k1_launches += 1; }
    else cudaGetLastError();
    ctx->ev_pending[i] = false;
}
void timing_collect(srl_ctx* ctx) { timing_collect_pair(ctx, 0); timing_collect_pair(ctx, 1); }

// the per-pass constants of buildPlaneResiduals (src/optimize.cpp:21-28,35,55-61,95)
void make_pass_const(const srl_frame& f, const srl_icp_params& p, PassConst& c) {
    const double* q = f.q_cur;
    // Eigen normalized() on the 4 coefficients (SSE2 pairing (x^2+z^2)+(y^2+w^2))
    double n2 = (q[0] * q[0] + q[2] * q[2]) + (q[1] * q[1] + q[3] * q[3]);
    double qn[4] = {q[0], q[1], q[2], q[3]};
    if (n2 > 0.0) { const double n = std::sqrt(n2); for (int i = 0; i < 4; ++i) qn[i] = q[i] / n; }
    quat_to_rot(qn, c.Rn);
    quat_to_rot(q, c.Rq);
    for (int i = 0; i < 3; ++i) { c.t[i] = f.t_cur[i]; c.t_last[i] = f.t_last[i]; c.t_il[i] = f.t_il[i]; }
    for (int i = 0; i < 9; ++i) c.R_il[i] = f.R_il[i];
    c.size = p.size_voxel_map;
    { int e = 0; c.inv_size = std::frexp(c.size, &e) == 0.5 ? 1.0 / c.size : 0.0; c.pad_ = 0.0; }   // exact reciprocal only for 2^k
    double lw = std::fabs(p.weight_alpha), ln = std::fabs(p.weight_neighborhood);
    const double sum = lw + ln;
    c.lambda_w = lw / sum; c.lambda_n = ln / sum;
    c.power = p.power_planarity;
    c.dmax = p.max_dist_to_plane_icp;
    c.exp_den = p.max_dist_to_plane_icp * p.min_number_neighbors;
    c.K = p.max_number_neighbors;
    c.Kmin = p.min_number_neighbors;
    const bool init = p.frame_id < p.init_num_frames;
    c.nb = init ? 2 : p.voxel_neighborhood;
    c.thr_occ = init ? 1 : p.threshold_voxel_occupancy;
}

static int check_params(srl_ctx* ctx, const srl_icp_params* p) {
    if (!p) return set_err(ctx, SRL_BAD_ARG, "null srl_icp_params");
    if (!(p->size_voxel_map > 0)) return set_err(ctx, SRL_BAD_ARG, "size_voxel_map must be > 0");
    if (p->max_number_neighbors < 1 || p->max_number_neighbors > 32) return set_err(ctx, SRL_BAD_ARG, "max_number_neighbors must be in [1,32]");
    if (p->min_number_neighbors < 1) return set_err(ctx, SRL_BAD_ARG, "min_number_neighbors must be >= 1");
    const int nb = p->frame_id < p->init_num_frames ? 2 : p->voxel_neighborhood;
    if (nb < 0 || nb > 2) return set_err(ctx, SRL_BAD_ARG, "voxel_neighborhood must be 0, 1 or 2");
    return SRL_OK;
}

static void unpack32(const double* o, srl_normal_eq* out, long long n_keypoints) {
    int idx = 0;
    for (int a = 0; a < 6; ++a)
        for (int b = a; b < 6; ++b) { out->HTH[a * 6 + b] = o[idx]; out->HTH[b * 6 + a] = o[idx]; ++idx; }
    for (int a = 0; a < 6; ++a) out->HTh[a] = o[21 + a];
    out->loss_sum = o[27];
    out->num_residuals = (int64_t)llround(o[28]);
    out->num_full_neighborhoods = (int64_t)llround(o[29]);
    out->num_candidates_scanned = (int64_t)llround(o[30]);
    out->nan_planarity = o[31] > 0.0 ? 1 : 0;
    out->num_keypoints = n_keypoints;
    out->reserved = 0;
}

constexpr bool kDefaultSplit = true;    // variant 0 (auto): k1_scan + k1_fit (H100, 100k-point sweep: 0.46 vs 0.75 ms per sweep for k1_fast in the same run, BASELINE.md)

static int pass_grid(srl_ctx* ctx, long long n, int K, int nb) {
    const long long n_groups = (n + 31) / 32;
    long long want = n_groups;   // block-minor group assignment: one group per block first, then per warp
    const long long resident = (long long)ctx->sm_count * k1_max_blocks_per_sm(K, nb);
    if (want > resident) want = resident;
    if (want < 1) want = 1;
    if (want > ctx->max_grid) want = ctx->max_grid;
    return (int)want;
}

}  // namespace srl

using namespace srl;

// The device-resident loop needs the persistent ESIKF block and the pass kernels to run at the same time.  Tools that
// serialise kernels (ncu, CUDA_LAUNCH_BLOCKING=1) make that impossible: probe once per ctx and fall back to the
// host-driven loop (same kernels, srl_iekf_step on the host) instead of timing out.
static bool device_loop_usable(srl_ctx* ctx) {
    if (!ctx->device_loop) return false;
    if (ctx->concurrent_kernels < 0) {
        bool ok = false;
        cudaSetDevice(ctx->device);
        int* d_probe = reinterpret_cast<int*>(ctx->d_stats + 4);   // two spare words behind the counters
        if (probe_concurrent_kernels(ctx->loop_stream, ctx->stream, d_probe, &ok) != cudaSuccess) { cudaGetLastError(); ok = false; }
        ctx->concurrent_kernels = ok ? 1 : 0;
    }
    return ctx->concurrent_kernels == 1;
}


template <typename T>
static int ensure_buf(srl_ctx* ctx, T** p, size_t count) {
    if (*p) return SRL_OK;
    cudaError_t e = cudaMalloc(p, count * sizeof(T));
    if (e != cudaSuccess) return cuda_fail(ctx, e, "cudaMalloc(debug/rows)");
    return SRL_OK;
}

// Result of a pass through the mapped host buffer: arm_host_result() before the launch, wait_host_result() after it.
static void arm_host_result(srl_ctx* ctx, K1Args& a) {
    if (!ctx->mapped_result) { a.host_out = nullptr; a.host_seq = 0; return; }
    a.host_out = ctx->d_h_out32;
    a.host_seq = ++ctx->host_seq;
}
// Spins on the sequence flag the pass's last kernel writes after its 32 sums; falls back to the stream's status so a
// failed launch or a device fault is reported instead of spinning forever.
static int wait_host_result(srl_ctx* ctx, const K1Args& a) {
    if (!a.host_out) {
        SRL_CUDA(ctx, cudaMemcpyAsync(ctx->h_out32, ctx->d_out32, 32 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        return SRL_OK;
    }
    volatile unsigned long long* flag = reinterpret_cast<volatile unsigned long long*>(ctx->h_out32 + 32);
    for (unsigned long long spins = 1;; ++spins) {
        if (*flag == a.host_seq) break;
        if ((spins & 0x3fffull) == 0) {
            const cudaError_t q = cudaStreamQuery(ctx->stream);
            if (q == cudaSuccess) {   // everything ran: the flag must be there (or the kernel never published)
                if (*flag == a.host_seq) break;
                return set_err(ctx, SRL_CUDA_ERROR, "the pass finished without publishing its result");
            }
            if (q != cudaErrorNotReady) return cuda_fail(ctx, q, "cudaStreamQuery while waiting for a pass");
        }
    }
    std::atomic_thread_fence(std::memory_order_acquire);
    return SRL_OK;
}

// One pass on the ctx stream.  Fast form (k1_fast + k1_assoc on the flagged keypoints) when the configuration allows
// it, k1_assoc alone otherwise (nb = 2, K != 20, residual cap, forced exact selection).
// The Morton order of the sweep's keypoints (srl_fast.cu), computed once per upload: eagerly right behind the copy that
// brings the keypoints to HBM (so it is off the critical path of the first pass), lazily here otherwise.
static int ensure_order(srl_ctx* ctx, srl_sweep* sw) {
    int rc;
    if ((rc = ensure_buf(ctx, &sw->d_order, sw->capacity)) != SRL_OK) return rc;
    if (!sw->order_valid && sw->n > 0) {
        size_t need = 0;
        sweep_compute_order(sw->d_raw, (long long)sw->n, sw->d_order, nullptr, 0, &need, ctx->stream);
        if ((rc = ensure_scratch(ctx, need)) != SRL_OK) return rc;
        SRL_CUDA(ctx, sweep_compute_order(sw->d_raw, (long long)sw->n, sw->d_order, ctx->d_scratch, ctx->scratch_bytes, &need, ctx->stream));
        sw->order_valid = true;
        ctx->launches += 1;
    }
    return SRL_OK;
}

static bool pass_is_fast(const srl_ctx* ctx, const K1Args& a) {
    // (rows = the ordered residual cap: the split form handles it, in keypoint order instead of Morton order)
    const bool split = ctx->variant == 3 || (ctx->variant == 0 && kDefaultSplit);
    return !ctx->force_exact && ctx->variant != 2 && a.c.nb <= 1 && a.c.K == 20 && a.c.Kmin == 20 && (!a.rows || split);
}
// Everything a pass needs besides its kernel launches: buffers, the sweep's Morton order, cleared flags / candidate rows,
// constant tables and (once per ctx) the kernels themselves.  Idempotent.  The device-resident loop calls it BEFORE it
// launches the persistent ESIKF block: an allocation, a module load (CUDA loads kernels lazily, and loading waits for
// running kernels) or a synchronous copy issued while that block spins would deadlock against it.
static int prepare_pass(srl_ctx* ctx, srl_sweep* sw, const K1Args& a) {
    if (!ctx->kernels_preloaded) {
        size_t max_local = 0;
        SRL_CUDA(ctx, preload_fast_kernels(ctx->device, &max_local));
        SRL_CUDA(ctx, preload_assoc_kernels(ctx->device, a.c.K, &max_local));
        // The first launch of a kernel whose local memory (spills) exceeds the context's reservation makes the driver
        // grow that reservation, and the driver waits for the device to go idle to do it.  Launched behind the persistent
        // ESIKF block, which spins until the pass finishes, that wait never ends (k1_fast keeps a ~1.6 KB spill frame on
        // sm_90a).  So the reservation is grown here, while nothing spins, to fit every pass kernel.
        size_t stack = 0;
        SRL_CUDA(ctx, cudaDeviceGetLimit(&stack, cudaLimitStackSize));
        if (max_local > stack) SRL_CUDA(ctx, cudaDeviceSetLimit(cudaLimitStackSize, max_local));
        ctx->kernels_preloaded = true;
    }
    if (!pass_is_fast(ctx, a)) return SRL_OK;
    int rc;
    if ((rc = ensure_order(ctx, sw)) != SRL_OK) return rc;
    if ((rc = ensure_buf(ctx, &sw->d_flags, sw->capacity)) != SRL_OK) return rc;
    // k1_scan / k1_fast write the flag of every keypoint of their range in every pass; the fallback launch walks the
    // flags of the whole sweep, so the keypoints outside this rank's range need zeros once per (upload, shard)
    if (!sw->flags_clean) {
        if (sw->n) SRL_CUDA(ctx, cudaMemsetAsync(sw->d_flags, 0, sw->n, ctx->stream));
        sw->flags_clean = true;
    }
    const bool split = ctx->variant == 3 || (ctx->variant == 0 && kDefaultSplit);
    if (split && !sw->d_cand_rows) {   // k1_fit loads whole rows and uses only the slots k1_scan filled: start from defined memory
        if ((rc = ensure_buf(ctx, &sw->d_cand_rows, sw->capacity * (size_t)24 + 8)) != SRL_OK) return rc;
        SRL_CUDA(ctx, cudaMemsetAsync(sw->d_cand_rows, 0, (sw->capacity * (size_t)24 + 8) * sizeof(unsigned), ctx->stream));
    }
    return SRL_OK;
}

static int launch_pass(srl_ctx* ctx, srl_sweep* sw, const K1Args& a, bool debug, bool own_timing = true, bool pdl = false) {
    const long long n = a.k_end - a.k_begin;
    const bool fast = pass_is_fast(ctx, a);
    const bool timing = ctx->timing && own_timing;
    {
        const int rc = prepare_pass(ctx, sw, a);
        if (rc != SRL_OK) return rc;
    }
    if (timing) {
        ctx->ev_cur ^= 1;
        timing_collect_pair(ctx, ctx->ev_cur);   // the pair used two passes ago
        cudaEventRecord(ctx->ev0[ctx->ev_cur], ctx->stream);
    }
    if (!fast) {
        SRL_CUDA(ctx, launch_k1(a, pass_grid(ctx, n, a.c.K, a.c.nb), debug, ctx->device, ctx->stream, pdl));
        ctx->launches += 1;
    } else {
        FastArgs f;
        std::memset(&f, 0, sizeof(f));
        f.c = a.c; f.slots = a.slots; f.mask = a.mask; f.blocks = a.blocks; f.raw = a.raw;
        f.order = a.rows ? nullptr : sw->d_order;   // the residual cap consumes keypoints in their own order (src/optimize.cpp:68,107)
        f.rows = a.rows;
        f.s_begin = a.k_begin; f.s_end = a.k_end;   // the shard is a range of SORTED positions in this form
        f.chunk_tickets = ctx->d_chunk_tickets; f.chunk_sums = ctx->d_chunk_sums;
        f.partials = a.partials; f.ticket = a.ticket; f.out32 = ctx->d_fast_out; f.flags = sw->d_flags; f.status = a.status;
        f.dbg_world = a.dbg_world; f.dbg_nbr = a.dbg_nbr; f.dbg_nbr_dist = a.dbg_nbr_dist; f.dbg_plane = a.dbg_plane; f.stats = a.stats;
        f.force_amb_mod = ctx->force_amb_mod;
        f.dev = a.dev; f.pose_ticket = a.pose_ticket; f.end_ticket = a.end_ticket; f.wait_pose = a.wait_pose;
        const bool split = ctx->variant == 3 || (ctx->variant == 0 && kDefaultSplit);
        if (split) {
            f.cand_rows = sw->d_cand_rows; f.scan_count = ctx->d_scan_count;
            // k1_fit publishes the result itself when nothing was flagged (multi-GPU: after running the exchange, option
            // exchange_in_fit); the fallback launch then runs off the host's critical path and republishes the same values
            f.comm = a.comm; f.exchange_in_fit = ctx->exchange_in_fit ? 1 : 0;
            if (a.comm.world <= 1 || ctx->exchange_in_fit) { f.host_out = a.host_out; f.host_seq = a.host_seq; }
            SRL_CUDA(ctx, launch_k1_split(f, n, ctx->max_grid, debug, ctx->device, ctx->stream, pdl));
            ctx->launches += 1;
        } else {
            const long long kpw = 32 / k1_fast_lanes_per_keypoint();
            const long long n_groups = (n + kpw - 1) / kpw;
            // one group per warp when it fits (the block scheduler then balances the waves), grid-stride beyond that
            long long grid = std::min<long long>((n_groups + kFastWarps - 1) / kFastWarps, (long long)ctx->max_grid);
            grid = std::max<long long>(1, std::min<long long>(grid, ctx->max_grid));
            SRL_CUDA(ctx, launch_k1_fast(f, (int)grid, debug, ctx->device, ctx->stream));
        }
        K1Args b = a;   // exact selection for the keypoints k1_fast could not decide; its last block adds k1_fast's sums
        b.only_flagged = sw->d_flags; b.prev_out32 = ctx->d_fast_out;
        if (!a.rows) { b.k_begin = 0; b.k_end = (long long)sw->n; }   // Morton order: the range's keypoints are scattered over the sweep
        // almost always nothing is flagged: a one-block-per-SM grid walks the flags (32 per warp step) and leaves
        const int fb_grid = (int)std::min<long long>(ctx->sm_count, std::max<long long>(1, ((long long)sw->n + 31) / 32));
        SRL_CUDA(ctx, launch_k1(b, fb_grid, debug, ctx->device, ctx->stream, pdl));
        ctx->launches += 2;
    }
    if (timing) { cudaEventRecord(ctx->ev1[ctx->ev_cur], ctx->stream); ctx->ev_pending[ctx->ev_cur] = true; }
    return SRL_OK;
}

extern "C" {

int srl_abi_version(void) { return SRL_ABI_VERSION; }
const char* srl_build_info(void) { return "srlivo_b200 sm_90a, CUDA " __DATE__; }

int srl_ctx_create(int device, void* cuda_stream, srl_ctx** out) {
    if (!out) return SRL_BAD_ARG;
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0 || device < 0 || device >= ndev) { cudaGetLastError(); return SRL_CUDA_ERROR; }   // no CPU fallback
    if (cudaSetDevice(device) != cudaSuccess) return SRL_CUDA_ERROR;
    srl_ctx* ctx = new srl_ctx();
    ctx->device = device;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) ctx->sm_count = prop.multiProcessorCount;
    if (cuda_stream) { ctx->stream = static_cast<cudaStream_t>(cuda_stream); ctx->own_stream = false; }
    else {
        if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) { delete ctx; return SRL_CUDA_ERROR; }
        ctx->own_stream = true;
    }
    ctx->max_grid = 2048;   // rows of the block-partials buffer (>= any grid we launch)
    bool ok = cudaMalloc(&ctx->d_partials, (size_t)ctx->max_grid * 32 * sizeof(double)) == cudaSuccess &&
              cudaMalloc(&ctx->d_ticket, sizeof(unsigned int)) == cudaSuccess &&
              cudaMalloc(&ctx->d_chunk_tickets, (size_t)(ctx->max_grid / 32 + 1) * sizeof(unsigned int)) == cudaSuccess &&
              cudaMemset(ctx->d_chunk_tickets, 0, (size_t)(ctx->max_grid / 32 + 1) * sizeof(unsigned int)) == cudaSuccess &&
              cudaMalloc(&ctx->d_chunk_sums, (size_t)(ctx->max_grid / 32 + 1) * 32 * sizeof(double)) == cudaSuccess &&
              cudaMalloc(&ctx->d_out32, 64 * sizeof(double)) == cudaSuccess &&
              cudaMalloc(&ctx->d_k2_state, 4 * sizeof(long long)) == cudaSuccess &&
              cudaMalloc(&ctx->d_stats, 6 * sizeof(unsigned long long)) == cudaSuccess &&
              cudaMalloc(&ctx->d_fast_out, 32 * sizeof(double)) == cudaSuccess &&
              cudaMalloc(&ctx->d_scan_count, sizeof(unsigned long long)) == cudaSuccess &&
              cudaMemset(ctx->d_scan_count, 0, sizeof(unsigned long long)) == cudaSuccess &&
              cudaMemset(ctx->d_stats, 0, 6 * sizeof(unsigned long long)) == cudaSuccess &&
              cudaHostAlloc(&ctx->h_out32, 64 * sizeof(double), cudaHostAllocMapped) == cudaSuccess &&
              cudaHostGetDevicePointer(&ctx->d_h_out32, ctx->h_out32, 0) == cudaSuccess &&
              cudaStreamCreateWithFlags(&ctx->loop_stream, cudaStreamNonBlocking) == cudaSuccess &&
              cudaMalloc(&ctx->d_iekf, sizeof(IekfDev)) == cudaSuccess &&
              cudaMemset(ctx->d_iekf, 0, sizeof(IekfDev)) == cudaSuccess &&
              cudaHostAlloc(&ctx->h_iekf, sizeof(IekfHostOut), cudaHostAllocMapped) == cudaSuccess &&
              cudaHostGetDevicePointer(&ctx->d_h_iekf, ctx->h_iekf, 0) == cudaSuccess &&
              cudaMemset(ctx->d_ticket, 0, sizeof(unsigned int)) == cudaSuccess;
    if (!ok) { srl_ctx_destroy(ctx); cudaGetLastError(); return SRL_CUDA_ERROR; }
    std::memset(ctx->h_out32, 0, 64 * sizeof(double));
    std::memset(ctx->h_iekf, 0, sizeof(IekfHostOut));
    if (const char* e = getenv("SRL_DEVICE_LOOP")) ctx->device_loop = atoi(e) != 0;
    if (const char* e = getenv("SRL_PDL")) ctx->pdl = atoi(e) != 0;
    if (const char* e = getenv("SRL_CLUSTER_ORDER")) sweep_order_set_impl(atoi(e));
    if (const char* e = getenv("SRL_MAPPED_RESULT")) ctx->mapped_result = atoi(e) != 0;   // A/B switch (bench runs)
    if (const char* e = getenv("SRL_EXCHANGE_IN_FIT")) ctx->exchange_in_fit = atoi(e) != 0;
    *out = ctx;
    return SRL_OK;
}

void srl_ctx_destroy(srl_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    if (ctx->loop_stream) { cudaStreamSynchronize(ctx->loop_stream); cudaStreamDestroy(ctx->loop_stream); }
    cudaFree(ctx->d_partials); cudaFree(ctx->d_ticket); cudaFree(ctx->d_chunk_tickets); cudaFree(ctx->d_chunk_sums); cudaFree(ctx->d_out32); cudaFree(ctx->d_k2_state); cudaFree(ctx->d_stats); cudaFree(ctx->d_fast_out); cudaFree(ctx->d_scan_count);
    cudaFree(ctx->d_scratch); cudaFree(ctx->d_iekf);
    if (ctx->h_iekf) cudaFreeHost(ctx->h_iekf);
    for (auto& e : ctx->loop_ev0) if (e) cudaEventDestroy(e);
    for (auto& e : ctx->loop_ev1) if (e) cudaEventDestroy(e);
    if (ctx->h_out32) cudaFreeHost(ctx->h_out32);
    if (ctx->h_pinned) cudaFreeHost(ctx->h_pinned);
    for (int i = 0; i < 2; ++i) { if (ctx->ev0[i]) cudaEventDestroy(ctx->ev0[i]); if (ctx->ev1[i]) cudaEventDestroy(ctx->ev1[i]); }
    if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

const char* srl_last_error(const srl_ctx* ctx) { return ctx ? ctx->err.c_str() : "null ctx"; }
int srl_ctx_synchronize(srl_ctx* ctx) {
    if (!ctx) return SRL_BAD_ARG;
    SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return SRL_OK;
}
int64_t srl_ctx_kernel_launches(const srl_ctx* ctx) { return ctx ? ctx->launches : 0; }
int srl_ctx_set_option(srl_ctx* ctx, const char* name, int64_t value) {
    if (!ctx || !name) return SRL_BAD_ARG;
    const std::string n(name);
    if (n == "force_exact_selection") { ctx->force_exact = value != 0; return SRL_OK; }
    if (n == "fast_force_ambiguous_mod") { ctx->force_amb_mod = (int)value; return SRL_OK; }
    if (n == "fast_lanes_per_keypoint") {
        if (value != 1 && value != 2 && value != 4) return set_err(ctx, SRL_BAD_ARG, "fast_lanes_per_keypoint must be 1, 2 or 4");
        k1_fast_set_lanes_per_keypoint((int)value);
        return SRL_OK;
    }
    if (n == "mapped_result") { ctx->mapped_result = value != 0; return SRL_OK; }
    if (n == "device_loop") { ctx->device_loop = value != 0; return SRL_OK; }
    if (n == "eager_order") { ctx->eager_order = value != 0; return SRL_OK; }
    if (n == "pdl") { ctx->pdl = value != 0; return SRL_OK; }
    if (n == "cluster_order") { sweep_order_set_impl((int)value); return SRL_OK; }   // process-wide
    if (n == "exchange_in_fit") { ctx->exchange_in_fit = value != 0; return SRL_OK; }
    if (n == "split_lanes_per_keypoint") {
        if (value != 2 && value != 4) return set_err(ctx, SRL_BAD_ARG, "split_lanes_per_keypoint must be 2 or 4");
        k1_split_set_lanes_per_keypoint((int)value);
        return SRL_OK;
    }
    if (n == "fast_min_blocks") {
        if (value != 4 && value != 5 && value != 6 && value != 8) return set_err(ctx, SRL_BAD_ARG, "fast_min_blocks must be 4, 5, 6 or 8");
        k1_fast_set_min_blocks((int)value);
        return SRL_OK;
    }
    if (n == "k1_variant") {
        if (value < 0 || value > 3) return set_err(ctx, SRL_BAD_ARG, "k1_variant must be 0 (auto), 1 (k1_fast), 2 (k1_assoc only) or 3 (k1_scan + k1_fit)");
        ctx->variant = (int)value;
        return SRL_OK;
    }
    if (n == "k1_min_blocks") {
        if (value != 2 && value != 3 && value != 4) return set_err(ctx, SRL_BAD_ARG, "k1_min_blocks must be 2, 3 or 4");
        k1_set_min_blocks((int)value);
        return SRL_OK;
    }
    return set_err(ctx, SRL_BAD_ARG, "unknown option " + n);
}
int srl_ctx_get_counter(srl_ctx* ctx, const char* name, int64_t* value) {
    if (!ctx || !name || !value) return SRL_BAD_ARG;
    const std::string n(name);
    if (n == "exact_fallbacks") {
        unsigned long long v = 0;
        SRL_CUDA(ctx, cudaMemcpyAsync(&v, ctx->d_stats, sizeof(v), cudaMemcpyDeviceToHost, ctx->stream));
        SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        *value = (int64_t)v;
        return SRL_OK;
    }
    if (n == "fast_ambiguous") {
        unsigned long long v = 0;
        SRL_CUDA(ctx, cudaMemcpyAsync(&v, ctx->d_stats + 1, sizeof(v), cudaMemcpyDeviceToHost, ctx->stream));
        SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        *value = (int64_t)v;
        return SRL_OK;
    }
    if (n == "kernel_launches") { *value = ctx->launches; return SRL_OK; }
    if (n.rfind("iekf_stage_", 0) == 0 && n.size() == 12 && n[11] >= '0' && n[11] <= '7') { *value = ctx->h_iekf->stage_cycles[n[11] - '0']; return SRL_OK; }
    if (n == "cluster_order_active") { *value = sweep_order_impl(); return SRL_OK; }
    if (n == "device_loop_active") { *value = device_loop_usable(ctx) ? 1 : 0; return SRL_OK; }
    if (n == "iekf_step_cycles_avg") {   // device-resident loop: average SM clock ticks of one ESIKF step (resets on read)
        *value = ctx->step_cycles_n ? (int64_t)(ctx->step_cycles_sum / (double)ctx->step_cycles_n) : 0;
        ctx->step_cycles_sum = 0.0; ctx->step_cycles_n = 0;
        return SRL_OK;
    }
    return set_err(ctx, SRL_BAD_ARG, "unknown counter " + n);
}
int srl_ctx_set_timing(srl_ctx* ctx, int enable) {
    if (!ctx) return SRL_BAD_ARG;
    if (enable && !ctx->ev0[0]) {
        SRL_CUDA(ctx, cudaSetDevice(ctx->device));
        for (int i = 0; i < 2; ++i) {
            SRL_CUDA(ctx, cudaEventCreate(&ctx->ev0[i]));
            SRL_CUDA(ctx, cudaEventCreate(&ctx->ev1[i]));
        }
    }
    ctx->timing = enable != 0;
    return SRL_OK;
}
int srl_ctx_pass_time(srl_ctx* ctx, double* total_ms, int64_t* launches, int reset) {
    if (!ctx) return SRL_BAD_ARG;
    SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    timing_collect(ctx);
    if (total_ms) *total_ms = ctx->k1_ms;
    if (launches) *launches = ctx->k1_launches;
    if (reset) { ctx->k1_ms = 0.0; ctx->k1_launches = 0; }
    return SRL_OK;
}

// ---- sweep -------------------------------------------------------------------------------------------------
int srl_sweep_create(srl_ctx* ctx, size_t capacity, srl_sweep** out) {
    if (!ctx || !out || capacity == 0) return SRL_BAD_ARG;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    srl_sweep* s = new srl_sweep();
    s->ctx = ctx; s->capacity = capacity;
    cudaError_t e = cudaMalloc(&s->d_raw, capacity * 3 * sizeof(double));
    if (e != cudaSuccess) { delete s; return cuda_fail(ctx, e, "srl_sweep_create/cudaMalloc"); }
    *out = s;
    return SRL_OK;
}
void srl_sweep_destroy(srl_sweep* s) {
    if (!s) return;
    cudaFree(s->d_raw); cudaFree(s->d_rows); cudaFree(s->d_status); cudaFree(s->d_order); cudaFree(s->d_flags); cudaFree(s->d_cand_rows);
    cudaFree(s->d_dbg_world); cudaFree(s->d_dbg_nbr); cudaFree(s->d_dbg_nbr_dist); cudaFree(s->d_dbg_plane);
    delete s;
}
int srl_sweep_upload(srl_sweep* s, const double* raw_xyz, size_t n) {
    if (!s || (n && !raw_xyz)) return SRL_BAD_ARG;
    srl_ctx* ctx = s->ctx;
    if (n > s->capacity) return set_err(ctx, SRL_BAD_ARG, "srl_sweep_upload: n exceeds capacity");
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    if (n) {
        // pinned caller memory goes straight to the DMA engine; pageable memory is staged through a pinned buffer
        cudaPointerAttributes attr;
        const bool pinned = cudaPointerGetAttributes(&attr, raw_xyz) == cudaSuccess && attr.type == cudaMemoryTypeHost;
        if (!pinned) {
            cudaGetLastError();
            int rc = ensure_pinned(ctx, n * 3 * sizeof(double));
            if (rc != SRL_OK) return rc;
            std::memcpy(ctx->h_pinned, raw_xyz, n * 3 * sizeof(double));
        }
        SRL_CUDA(ctx, cudaMemcpyAsync(s->d_raw, pinned ? raw_xyz : static_cast<const double*>(ctx->h_pinned), n * 3 * sizeof(double),
                                      cudaMemcpyHostToDevice, ctx->stream));
        // the staging buffer is shared by every upload of the ctx: it must not be refilled while the DMA still reads it
        // (pinned caller memory is read asynchronously: the caller keeps it unchanged until the next synchronising call)
        if (!pinned) SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    s->n = n; s->shard_begin = 0; s->shard_end = n; s->order_valid = false; s->flags_clean = false;
    return ctx->eager_order ? ensure_order(ctx, s) : SRL_OK;
}
int srl_sweep_set_device(srl_sweep* s, const double* d_raw_xyz, size_t n) {
    if (!s || (n && !d_raw_xyz)) return SRL_BAD_ARG;
    srl_ctx* ctx = s->ctx;
    if (n > s->capacity) return set_err(ctx, SRL_BAD_ARG, "srl_sweep_set_device: n exceeds capacity");
    SRL_CUDA(ctx, cudaMemcpyAsync(s->d_raw, d_raw_xyz, n * 3 * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
    s->n = n; s->shard_begin = 0; s->shard_end = n; s->order_valid = false; s->flags_clean = false;
    return ctx->eager_order ? ensure_order(ctx, s) : SRL_OK;
}
int srl_sweep_set_shard(srl_sweep* s, size_t begin, size_t end) {
    if (!s || begin > end || end > s->n) return SRL_BAD_ARG;
    s->shard_begin = begin; s->shard_end = end; s->flags_clean = false;
    return SRL_OK;
}

// ---- one pass ----------------------------------------------------------------------------------------------
static int fill_k1_args(srl_ctx* ctx, srl_map* map, srl_sweep* sw, const srl_frame* frame, const srl_icp_params* prm, K1Args& a) {
    int rc = check_params(ctx, prm);
    if (rc != SRL_OK) return rc;
    if (!map || !sw || !frame) return set_err(ctx, SRL_BAD_ARG, "null map/sweep/frame");
    if (map->ctx != ctx || sw->ctx != ctx) return set_err(ctx, SRL_BAD_ARG, "map/sweep belong to another ctx");
    if (std::fabs(prm->size_voxel_map - map->voxel_size) > 0) return set_err(ctx, SRL_BAD_ARG, "icp size_voxel_map differs from the map's voxel size");
    std::memset(&a, 0, sizeof(a));
    make_pass_const(*frame, *prm, a.c);
    a.slots = map->d_slots; a.mask = (unsigned)(map->capacity - 1); a.blocks = map->d_blocks;
    a.raw = sw->d_raw; a.k_begin = (long long)sw->shard_begin; a.k_end = (long long)sw->shard_end;
    a.partials = ctx->d_partials; a.ticket = ctx->d_ticket; a.out32 = ctx->d_out32;
    a.stats = ctx->d_stats;
    a.eps_scale = ctx->force_exact ? std::numeric_limits<float>::infinity() : 1.0f;
    return SRL_OK;
}

int srl_build_plane_residuals_async(srl_ctx* ctx, srl_map* map, srl_sweep* sw, const srl_frame* frame, const srl_icp_params* prm,
                                    double* d_out32) {
    if (!ctx || !d_out32) return SRL_BAD_ARG;
    K1Args a;
    int rc = fill_k1_args(ctx, map, sw, frame, prm, a);
    if (rc != SRL_OK) return rc;
    const long long n = a.k_end - a.k_begin;
    if ((long long)prm->max_num_residuals < n) return set_err(ctx, SRL_BAD_ARG, "async pass does not implement the max_num_residuals cap");
    a.out32 = d_out32;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    if (n <= 0) { SRL_CUDA(ctx, cudaMemsetAsync(d_out32, 0, 32 * sizeof(double), ctx->stream)); return SRL_OK; }
    return launch_pass(ctx, sw, a, false);
}

int srl_normal_eq_unpack(const double* h_out32, srl_normal_eq* out) {
    if (!h_out32 || !out) return SRL_BAD_ARG;
    unpack32(h_out32, out, 0);
    return SRL_OK;
}

int srl_build_plane_residuals(srl_ctx* ctx, srl_map* map, srl_sweep* sw, const srl_frame* frame, const srl_icp_params* prm,
                              srl_normal_eq* out, srl_debug_out* dbg) {
    if (!ctx || !out) return SRL_BAD_ARG;
    K1Args a;
    int rc = fill_k1_args(ctx, map, sw, frame, prm, a);
    if (rc != SRL_OK) return rc;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    std::memset(out, 0, sizeof(*out));
    const long long n = a.k_end - a.k_begin;
    const int K = a.c.K;
    const bool cap_mode = (long long)prm->max_num_residuals < n;
    if (cap_mode && (sw->shard_begin != 0 || sw->shard_end != sw->n))
        return set_err(ctx, SRL_BAD_ARG, "max_num_residuals < shard size is only supported on an unsharded sweep");
    const bool debug = dbg != nullptr;
    if (debug) {
        if (sw->dbg_K != K) {   // neighbour arrays depend on K
            cudaFree(sw->d_dbg_nbr); cudaFree(sw->d_dbg_nbr_dist); sw->d_dbg_nbr = nullptr; sw->d_dbg_nbr_dist = nullptr; sw->dbg_K = K;
        }
        if ((rc = ensure_buf(ctx, &sw->d_dbg_world, sw->capacity * 3)) != SRL_OK) return rc;
        if ((rc = ensure_buf(ctx, &sw->d_dbg_nbr, sw->capacity * K * 4)) != SRL_OK) return rc;
        if ((rc = ensure_buf(ctx, &sw->d_dbg_nbr_dist, sw->capacity * K)) != SRL_OK) return rc;
        if ((rc = ensure_buf(ctx, &sw->d_dbg_plane, sw->capacity * 16)) != SRL_OK) return rc;
        SRL_CUDA(ctx, cudaMemsetAsync(sw->d_dbg_world, 0, sw->capacity * 3 * sizeof(double), ctx->stream));
        SRL_CUDA(ctx, cudaMemsetAsync(sw->d_dbg_nbr, 0xff, sw->capacity * K * 4 * sizeof(short), ctx->stream));
        SRL_CUDA(ctx, cudaMemsetAsync(sw->d_dbg_nbr_dist, 0, sw->capacity * K * sizeof(double), ctx->stream));
        SRL_CUDA(ctx, cudaMemsetAsync(sw->d_dbg_plane, 0, sw->capacity * 16 * sizeof(double), ctx->stream));
        a.dbg_world = sw->d_dbg_world; a.dbg_nbr = sw->d_dbg_nbr; a.dbg_nbr_dist = sw->d_dbg_nbr_dist; a.dbg_plane = sw->d_dbg_plane;
    }
    if (debug || cap_mode) {
        if ((rc = ensure_buf(ctx, &sw->d_status, sw->capacity)) != SRL_OK) return rc;
        SRL_CUDA(ctx, cudaMemsetAsync(sw->d_status, 0, sw->capacity * sizeof(int), ctx->stream));
        a.status = sw->d_status;
    }
    double* h = ctx->h_out32;
    double zero32[32];
    if (n <= 0) {   // an empty shard sums to zero; the mapped buffer may still be written by the previous pass's fallback launch
        std::memset(zero32, 0, sizeof(zero32));
        h = zero32;
    } else if (!cap_mode) {
        arm_host_result(ctx, a);
        if ((rc = launch_pass(ctx, sw, a, debug)) != SRL_OK) return rc;
        if ((rc = wait_host_result(ctx, a)) != SRL_OK) return rc;
    } else {
        // ordered cap (src/optimize.cpp:107): process keypoints in order, chunk by chunk, until k* is found
        if ((rc = ensure_buf(ctx, &sw->d_rows, sw->capacity * 8)) != SRL_OK) return rc;
        a.rows = sw->d_rows;
        double* d_cap_out = ctx->d_out32 + 32;
        SRL_CUDA(ctx, cudaMemsetAsync(d_cap_out, 0, 32 * sizeof(double), ctx->stream));
        SRL_CUDA(ctx, cudaMemsetAsync(ctx->d_k2_state, 0, 4 * sizeof(long long), ctx->stream));
        const long long cap = prm->max_num_residuals;
        long long chunk = std::max<long long>(4096, 2 * std::max<long long>(cap, 1));
        double scanned = 0, nanf = 0;
        long long begin = 0;
        long long st[4] = {0, 0, 0, 0};
        while (begin < n) {
            const long long end = std::min(n, begin + chunk);
            K1Args c = a;
            c.k_begin = begin; c.k_end = end;
            if ((rc = launch_pass(ctx, sw, c, debug)) != SRL_OK) return rc;
            SRL_CUDA(ctx, launch_k2(sw->d_rows, sw->d_status, begin, end, (int)cap, ctx->d_k2_state, d_cap_out, 0, ctx->stream));
            ctx->launches += 1;
            SRL_CUDA(ctx, cudaMemcpyAsync(h, ctx->d_out32, 32 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
            SRL_CUDA(ctx, cudaMemcpyAsync(st, ctx->d_k2_state, sizeof(st), cudaMemcpyDeviceToHost, ctx->stream));
            SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            scanned += h[30]; nanf += h[31];
            begin = end;
            if (st[1]) break;   // k* found: the reference loop has hit its `break`
            chunk *= 2;
        }
        // keypoints after k* were never visited
        if (st[1] && st[2] + 1 < n) {
            const long long first = st[2] + 1;
            std::vector<int> neg((size_t)(n - first), -1);
            SRL_CUDA(ctx, cudaMemcpyAsync(sw->d_status + first, neg.data(), neg.size() * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
        }
        SRL_CUDA(ctx, cudaMemcpyAsync(h, d_cap_out, 32 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        // [31] comes from k2_cap_reduce: NaN planarity counts only where the reference loop got to (k <= k*)
        (void)nanf;
        h[30] = scanned;   // candidates scanned in the chunks processed (an upper bound of the reference's count up to k*)
    }
    unpack32(h, out, n);
    if (debug) {
        const size_t N = sw->n;
        if (dbg->world_xyz) SRL_CUDA(ctx, cudaMemcpyAsync(dbg->world_xyz, sw->d_dbg_world, N * 3 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        if (dbg->status) SRL_CUDA(ctx, cudaMemcpyAsync(dbg->status, sw->d_status, N * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        if (dbg->nbr) SRL_CUDA(ctx, cudaMemcpyAsync(dbg->nbr, sw->d_dbg_nbr, N * K * 4 * sizeof(short), cudaMemcpyDeviceToHost, ctx->stream));
        if (dbg->nbr_dist) SRL_CUDA(ctx, cudaMemcpyAsync(dbg->nbr_dist, sw->d_dbg_nbr_dist, N * K * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        if (dbg->plane) SRL_CUDA(ctx, cudaMemcpyAsync(dbg->plane, sw->d_dbg_plane, N * 16 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    if (out->nan_planarity) return set_err(ctx, SRL_NAN_PLANARITY, "NaN planarity (the reference throws at src/optimize.cpp:348)");
    if (out->num_residuals < prm->min_number_neighbors)
        return set_err(ctx, SRL_TOO_FEW_RESIDUALS, "[Optimization] Error : not enough keypoints selected in ct-icp !");
    return SRL_OK;
}

// ---- iterated update ---------------------------------------------------------------------------------------
// Row N1: the whole updateIEKF loop enqueued at once.  Pass 0 takes its pose by value; every later pass reads the pose
// the persistent ESIKF block (k_iekf_loop) left in HBM and leaves immediately once the loop has ended on the device.  One host wait at the end, on
// the sequence flag the finishing step writes into mapped pinned memory after the state, the trace and the summary.
static int update_iekf_device(srl_ctx* ctx, srl_comm* comm, srl_map* map, srl_sweep* sw, srl_eskf_state* eskf, double frame_q[4],
                              double frame_t[3], const double t_last[3], const double R_il[9], const double t_il[3],
                              const srl_icp_params* prm, srl_iekf_summary* summary) {
    srl_frame fr;
    std::memcpy(fr.q_cur, frame_q, sizeof(fr.q_cur));
    std::memcpy(fr.t_cur, frame_t, sizeof(fr.t_cur));
    std::memcpy(fr.t_last, t_last, sizeof(fr.t_last));
    std::memcpy(fr.R_il, R_il, sizeof(fr.R_il));
    std::memcpy(fr.t_il, t_il, sizeof(fr.t_il));
    K1Args a;
    int rc = fill_k1_args(ctx, map, sw, &fr, prm, a);
    if (rc != SRL_OK) return rc;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    srl_iekf_iter it;
    if ((rc = srl_iekf_begin(eskf, prm, &it)) != SRL_OK) return rc;
    const int n_pass = it.max_num_iter + 1;                          // i = -1 .. max_iter - 1 (src/optimize.cpp:147)
    if (n_pass > kLoopMaxPasses) return set_err(ctx, SRL_BAD_ARG, "num_iters_icp > 39 is not supported by the device-resident loop");
    if (comm) {
        a.comm.world = comm->world; a.comm.rank = comm->rank; a.comm.seq = comm->d_seq;
        for (int r = 0; r < comm->world; ++r) a.comm.mail[r] = comm->peer[r];
    }
    static_assert(sizeof(IekfLoopArgs) <= 4000, "the loop kernel's arguments must fit the 4 KB kernel parameter space");
    IekfLoopArgs la;
    std::memset(&la, 0, sizeof(la));
    IekfInit& init = la.init;
    init.eskf = *eskf;
    std::memcpy(init.frame_q, frame_q, sizeof(init.frame_q));
    std::memcpy(init.frame_t, frame_t, sizeof(init.frame_t));
    init.pc0 = a.c;
    init.laser_cov = prm->laser_point_cov; init.thr_t = prm->threshold_translation_norm; init.thr_r = prm->threshold_orientation_norm;
    init.max_iter = it.max_num_iter; init.frame_id = prm->frame_id; init.min_neighbors = prm->min_number_neighbors;
    la.dev = ctx->d_iekf; la.host_out = ctx->d_h_iekf; la.host_seq = ++ctx->iekf_seq;
    la.base = ctx->loop_base; ctx->loop_base += 64;
    la.world = comm ? comm->world : 1; la.n_pass = n_pass;
    const IekfLoopArgs& st = la;
    if ((rc = prepare_pass(ctx, sw, a)) != SRL_OK) return rc;
    if (ctx->timing && !ctx->loop_ev0[0])
        for (int i = 0; i < kLoopMaxPasses; ++i) { SRL_CUDA(ctx, cudaEventCreate(&ctx->loop_ev0[i])); SRL_CUDA(ctx, cudaEventCreate(&ctx->loop_ev1[i])); }
    // the persistent ESIKF block first (side stream): it is resident before any pass kernel can wait for it
    SRL_CUDA(ctx, launch_iekf_loop(la, ctx->loop_stream));
    ctx->launches += 1;
    for (int p = 0; p < n_pass; ++p) {
        K1Args ap = a;
        ap.dev = ctx->d_iekf;
        ap.pose_ticket = la.base + (unsigned long long)p;
        ap.end_ticket = la.base + 63ull;
        ap.wait_pose = p ? 1 : 0;                                    // pass 0: pose by value
        if (ctx->timing) cudaEventRecord(ctx->loop_ev0[p], ctx->stream);
        if ((rc = launch_pass(ctx, sw, ap, false, false, ctx->pdl && !ctx->timing)) != SRL_OK) {
            // the persistent block is waiting for a pass that will never come: tell it, wait for it to leave, report the launch error
            const std::string why = ctx->err;
            launch_iekf_abort(ctx->d_iekf, ctx->stream);
            cudaStreamSynchronize(ctx->loop_stream);
            cudaGetLastError();
            return set_err(ctx, rc, why);
        }
        if (ctx->timing) cudaEventRecord(ctx->loop_ev1[p], ctx->stream);
    }
    // the one host wait of the sweep
    volatile unsigned long long* flag = &ctx->h_iekf->seq;
    for (unsigned long long spins = 1;; ++spins) {
        if (*flag == st.host_seq) break;
        if ((spins & 0x3fffull) == 0) {
            const cudaError_t q = cudaStreamQuery(ctx->loop_stream);   // the ESIKF block leaves right after publishing
            if (q == cudaSuccess) {
                if (*flag == st.host_seq) break;
                return set_err(ctx, SRL_CUDA_ERROR, "the device-resident updateIEKF loop finished without publishing its result");
            }
            if (q != cudaErrorNotReady) return cuda_fail(ctx, q, "cudaStreamQuery while waiting for the updateIEKF loop");
        }
    }
    std::atomic_thread_fence(std::memory_order_acquire);
    const IekfHostOut* h = ctx->h_iekf;
    const int passes = h->passes_run;
    if (ctx->timing) {   // the passes that ran have finished (their events precede the step that published)
        for (int p = 0; p < passes && p < n_pass; ++p) {
            float ms = 0.f;
            if (cudaEventElapsedTime(&ms, ctx->loop_ev0[p], ctx->loop_ev1[p]) == cudaSuccess) { ctx->k1_ms += ms; ctx->k1_launches += 1; }
            else cudaGetLastError();
        }
    }
    *eskf = h->eskf;
    std::memcpy(frame_q, h->frame_q, sizeof(h->frame_q));
    std::memcpy(frame_t, h->frame_t, sizeof(h->frame_t));
    std::memcpy(ctx->h_out32, h->sums, 32 * sizeof(double));
    if (summary) {
        std::memset(summary, 0, sizeof(*summary));
        summary->success = h->status == SRL_TOO_FEW_RESIDUALS ? 0 : 1;
        summary->passes_run = passes;
        summary->num_residuals_used = h->num_residuals_used;
        summary->converged = h->converged;
        std::memcpy(summary->trace, h->trace, sizeof(double) * 24 * (size_t)std::min(passes, 32));
    }
    for (int p = 0; p < passes && p < kLoopMaxPasses; ++p) { ctx->step_cycles_sum += (double)h->step_cycles[p]; ctx->step_cycles_n += 1; }
    switch (h->status) {
        case SRL_OK: return SRL_OK;
        case SRL_TOO_FEW_RESIDUALS: return set_err(ctx, SRL_TOO_FEW_RESIDUALS, "[Optimization] Error : not enough keypoints selected in ct-icp !");
        case SRL_NAN_PLANARITY: return set_err(ctx, SRL_NAN_PLANARITY, "NaN planarity (the reference throws at src/optimize.cpp:348)");
        case SRL_SINGULAR: return set_err(ctx, SRL_SINGULAR, "the 6x6 system of the ESIKF gain is singular (src/optimize.cpp:234,237)");
        case SRL_COMM_ERROR: return set_err(ctx, SRL_COMM_ERROR, "peer exchange timed out (a rank did not reach this pass)");
        default: return set_err(ctx, h->status, "device-resident updateIEKF loop failed");
    }
}

int srl_update_iekf(srl_ctx* ctx, srl_map* map, srl_sweep* sw, srl_eskf_state* eskf, double frame_q[4], double frame_t[3],
                    const double t_last[3], const double R_il[9], const double t_il[3], const srl_icp_params* prm,
                    srl_iekf_summary* summary) {
    if (!ctx || !eskf || !frame_q || !frame_t || !t_last || !R_il || !t_il || !prm) return SRL_BAD_ARG;
    if (device_loop_usable(ctx) && map && sw && !((long long)prm->max_num_residuals < (long long)(sw->shard_end - sw->shard_begin)))
        return update_iekf_device(ctx, nullptr, map, sw, eskf, frame_q, frame_t, t_last, R_il, t_il, prm, summary);
    srl_iekf_iter it;
    int rc = srl_iekf_begin(eskf, prm, &it);
    if (rc != SRL_OK) return rc;
    if (summary) { std::memset(summary, 0, sizeof(*summary)); summary->success = 1; }
    srl_frame fr;
    std::memcpy(fr.t_last, t_last, sizeof(fr.t_last));
    std::memcpy(fr.R_il, R_il, sizeof(fr.R_il));
    std::memcpy(fr.t_il, t_il, sizeof(fr.t_il));
    int passes = 0;
    for (;;) {
        std::memcpy(fr.q_cur, frame_q, sizeof(fr.q_cur));
        std::memcpy(fr.t_cur, frame_t, sizeof(fr.t_cur));
        srl_normal_eq ne;
        rc = srl_build_plane_residuals(ctx, map, sw, &fr, prm, &ne, nullptr);       // src/optimize.cpp:153
        ++passes;
        if (summary) { summary->passes_run = passes; summary->num_residuals_used = (int32_t)ne.num_residuals; }
        if (rc == SRL_TOO_FEW_RESIDUALS) { if (summary) summary->success = 0; return rc; }   // :155
        if (rc != SRL_OK) return rc;
        double d_x[17];
        int32_t done = 0, diverged = 0;
        rc = srl_iekf_step(&it, &ne, prm, eskf, frame_q, frame_t, d_x, &done, &diverged);
        if (rc != SRL_OK) return set_err(ctx, rc, "srl_iekf_step failed (singular 17x17)");
        if (summary && passes <= 32) {
            double* tr = summary->trace[passes - 1];
            std::memcpy(tr, d_x, 17 * sizeof(double));
            std::memcpy(tr + 17, frame_t, 3 * sizeof(double));
            std::memcpy(tr + 20, frame_q, 4 * sizeof(double));
        }
        if (done) { if (summary) summary->converged = (done == 2); break; }
    }
    return SRL_OK;
}

// ---- multi-GPU -------------------------------------------------------------------------------------------------
int srl_comm_create(srl_ctx* ctx, int rank, int world, srl_comm** out) {
    if (!ctx || !out || world < 1 || world > kMaxRanks || rank < 0 || rank >= world) return SRL_BAD_ARG;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    srl_comm* c = new srl_comm();
    c->ctx = ctx; c->rank = rank; c->world = world;
    cudaError_t e = cudaMalloc(&c->d_mail, sizeof(Mailbox));
    if (e != cudaSuccess) { delete c; return cuda_fail(ctx, e, "srl_comm_create/cudaMalloc"); }
    e = cudaMemset(c->d_mail, 0, sizeof(Mailbox));
    if (e == cudaSuccess) e = cudaMalloc(&c->d_seq, sizeof(unsigned long long));
    if (e == cudaSuccess) e = cudaMemset(c->d_seq, 0, sizeof(unsigned long long));
    if (e != cudaSuccess) { cudaFree(c->d_mail); cudaFree(c->d_seq); delete c; return cuda_fail(ctx, e, "srl_comm_create/cudaMemset"); }
    c->peer[rank] = c->d_mail;
    c->connected = (world == 1);
    *out = c;
    return SRL_OK;
}
void srl_comm_destroy(srl_comm* c) {
    if (!c) return;
    cudaSetDevice(c->ctx->device);
    cudaStreamSynchronize(c->ctx->stream);
    for (int r = 0; r < c->world; ++r) if (c->opened[r]) cudaIpcCloseMemHandle(c->peer[r]);
    cudaFree(c->d_mail); cudaFree(c->d_seq);
    delete c;
}
int srl_comm_export(srl_comm* c, void* handle64) {
    if (!c || !handle64) return SRL_BAD_ARG;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle is 64 bytes");
    cudaIpcMemHandle_t h;
    SRL_CUDA(c->ctx, cudaIpcGetMemHandle(&h, c->d_mail));
    std::memcpy(handle64, &h, 64);
    return SRL_OK;
}
int srl_comm_connect(srl_comm* c, const void* handles) {
    if (!c || !handles) return SRL_BAD_ARG;
    srl_ctx* ctx = c->ctx;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    for (int r = 0; r < c->world; ++r) {
        if (r == c->rank || c->opened[r]) continue;
        cudaIpcMemHandle_t h;
        std::memcpy(&h, static_cast<const char*>(handles) + 64 * r, 64);
        void* p = nullptr;
        cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) { cuda_fail(ctx, e, "cudaIpcOpenMemHandle (peer mailbox)"); return SRL_COMM_ERROR; }
        c->peer[r] = static_cast<Mailbox*>(p);
        c->opened[r] = true;
    }
    c->connected = true;
    return SRL_OK;
}

int srl_update_iekf_dist(srl_ctx* ctx, srl_comm* comm, srl_map* map, srl_sweep* sw, srl_eskf_state* eskf, double frame_q[4],
                         double frame_t[3], const double t_last[3], const double R_il[9], const double t_il[3],
                         const srl_icp_params* prm, srl_iekf_summary* summary) {
    if (!ctx || !comm || !eskf || !frame_q || !frame_t || !t_last || !R_il || !t_il || !prm) return SRL_BAD_ARG;
    if (comm->ctx != ctx || !comm->connected) return set_err(ctx, SRL_COMM_ERROR, "srl_comm is not connected");
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    if (map && sw && (long long)prm->max_num_residuals < (long long)sw->n)
        return set_err(ctx, SRL_BAD_ARG, "the sharded update does not implement the max_num_residuals cap");
    if (device_loop_usable(ctx) && map && sw)
        return update_iekf_device(ctx, comm, map, sw, eskf, frame_q, frame_t, t_last, R_il, t_il, prm, summary);
    srl_iekf_iter it;
    int rc = srl_iekf_begin(eskf, prm, &it);
    if (rc != SRL_OK) return rc;
    if (summary) { std::memset(summary, 0, sizeof(*summary)); summary->success = 1; }
    srl_frame fr;
    std::memcpy(fr.t_last, t_last, sizeof(fr.t_last));
    std::memcpy(fr.R_il, R_il, sizeof(fr.R_il));
    std::memcpy(fr.t_il, t_il, sizeof(fr.t_il));
    int passes = 0;
    for (;;) {
        std::memcpy(fr.q_cur, frame_q, sizeof(fr.q_cur));
        std::memcpy(fr.t_cur, frame_t, sizeof(fr.t_cur));
        K1Args a;
        rc = fill_k1_args(ctx, map, sw, &fr, prm, a);
        if (rc != SRL_OK) return rc;
        const long long n = a.k_end - a.k_begin;
        if ((long long)prm->max_num_residuals < (long long)sw->n)
            return set_err(ctx, SRL_BAD_ARG, "the sharded update does not implement the max_num_residuals cap");
        a.comm.world = comm->world; a.comm.rank = comm->rank; a.comm.seq = comm->d_seq;
        for (int r = 0; r < comm->world; ++r) a.comm.mail[r] = comm->peer[r];
        (void)n;
        arm_host_result(ctx, a);
        if ((rc = launch_pass(ctx, sw, a, false)) != SRL_OK) return rc;     // also valid for an empty shard
        double* h = ctx->h_out32;
        if ((rc = wait_host_result(ctx, a)) != SRL_OK) return rc;
        if (h[0] != h[0]) return set_err(ctx, SRL_COMM_ERROR, "peer exchange timed out (a rank did not reach this pass)");
        srl_normal_eq ne;
        unpack32(h, &ne, (long long)sw->n);
        ++passes;
        if (summary) { summary->passes_run = passes; summary->num_residuals_used = (int32_t)ne.num_residuals; }
        if (ne.nan_planarity) return set_err(ctx, SRL_NAN_PLANARITY, "NaN planarity (the reference throws at src/optimize.cpp:348)");
        if (ne.num_residuals < prm->min_number_neighbors) {
            if (summary) summary->success = 0;
            return set_err(ctx, SRL_TOO_FEW_RESIDUALS, "[Optimization] Error : not enough keypoints selected in ct-icp !");
        }
        double d_x[17];
        int32_t done = 0, diverged = 0;
        rc = srl_iekf_step(&it, &ne, prm, eskf, frame_q, frame_t, d_x, &done, &diverged);
        if (rc != SRL_OK) return set_err(ctx, rc, "srl_iekf_step failed (singular 17x17)");
        if (summary && passes <= 32) {
            double* tr = summary->trace[passes - 1];
            std::memcpy(tr, d_x, 17 * sizeof(double));
            std::memcpy(tr + 17, frame_t, 3 * sizeof(double));
            std::memcpy(tr + 20, frame_q, 4 * sizeof(double));
        }
        if (done) { if (summary) summary->converged = (done == 2); break; }
    }
    return SRL_OK;
}

int srl_sweep_transform_device(srl_ctx* ctx, srl_sweep* sw, const double q[4], const double t[3], const double R_il[9],
                               const double t_il[3], double* d_world_xyz) {
    if (!ctx || !sw || !q || !t || !R_il || !t_il || !d_world_xyz) return SRL_BAD_ARG;
    PassConst c;
    std::memset(&c, 0, sizeof(c));
    quat_to_rot(q, c.Rq);   // transformPoint uses q_end.toRotationMatrix() un-normalised (src/utility.cpp:317)
    for (int i = 0; i < 3; ++i) { c.t[i] = t[i]; c.t_il[i] = t_il[i]; }
    for (int i = 0; i < 9; ++i) c.R_il[i] = R_il[i];
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    SRL_CUDA(ctx, launch_transform(sw->d_raw, (long long)sw->n, c, d_world_xyz, ctx->stream));
    ctx->launches += 1;
    return SRL_OK;
}

int srl_optimize_host(srl_ctx* ctx, srl_map* map, srl_sweep* sw, const double* raw_xyz, size_t n, srl_eskf_state* eskf,
                      double frame_q[4], double frame_t[3], const double t_last[3], const double R_il[9], const double t_il[3],
                      const srl_icp_params* prm, srl_iekf_summary* summary, double* world_xyz_out) {
    if (!ctx || !sw) return SRL_BAD_ARG;
    int rc = srl_sweep_upload(sw, raw_xyz, n);                                   // H2D of the keypoints
    if (rc != SRL_OK) return rc;
    rc = srl_update_iekf(ctx, map, sw, eskf, frame_q, frame_t, t_last, R_il, t_il, prm, summary);   // src/optimize.cpp:435
    if (rc != SRL_OK) return rc;                                                 // :437-439
    if (world_xyz_out && n) {                                                    // :441-445
        int r2 = ensure_scratch(ctx, n * 3 * sizeof(double));
        if (r2 != SRL_OK) return r2;
        r2 = srl_sweep_transform_device(ctx, sw, frame_q, frame_t, R_il, t_il, static_cast<double*>(ctx->d_scratch));
        if (r2 != SRL_OK) return r2;
        SRL_CUDA(ctx, cudaMemcpyAsync(world_xyz_out, ctx->d_scratch, n * 3 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    return SRL_OK;
}

void srl_shard_range(size_t n, int rank, int world, size_t* begin, size_t* end) {
    // contiguous keypoint ranges on multiples of 32 (whole warp groups), in rank order (SURVEY.md §8(e))
    const size_t groups = (n + 31) / 32;
    size_t b = world > 0 ? (groups * (size_t)rank) / (size_t)world * 32 : 0;
    size_t e = world > 0 ? (groups * (size_t)(rank + 1)) / (size_t)world * 32 : n;
    if (b > n) b = n;
    if (e > n) e = n;
    if (begin) *begin = b;
    if (end) *end = e;
}

int srl_optimize_host_dist(srl_ctx* ctx, srl_comm* comm, srl_map* map, srl_sweep* sw, const double* raw_xyz, size_t n,
                           srl_eskf_state* eskf, double frame_q[4], double frame_t[3], const double t_last[3], const double R_il[9],
                           const double t_il[3], const srl_icp_params* prm, srl_iekf_summary* summary, double* world_xyz_out,
                           size_t* shard_begin, size_t* shard_end) {
    if (!ctx || !comm || !sw || (n && !raw_xyz)) return SRL_BAD_ARG;
    size_t b = 0, e = 0;
    srl_shard_range(n, comm->rank, comm->world, &b, &e);
    if (shard_begin) *shard_begin = b;
    if (shard_end) *shard_end = e;
    // this rank's keypoints only: H2D of (e - b) points, the local sweep is sorted and registered as a whole, the 32 sums
    // of every pass are exchanged inside the pass (srl_update_iekf_dist), so every rank ends with the same state
    int rc = srl_sweep_upload(sw, raw_xyz + 3 * b, e - b);
    if (rc != SRL_OK) return rc;
    rc = srl_update_iekf_dist(ctx, comm, map, sw, eskf, frame_q, frame_t, t_last, R_il, t_il, prm, summary);
    if (rc != SRL_OK) return rc;
    if (world_xyz_out && e > b) {                                                // src/optimize.cpp:441-445, this rank's rows
        int r2 = ensure_scratch(ctx, (e - b) * 3 * sizeof(double));
        if (r2 != SRL_OK) return r2;
        r2 = srl_sweep_transform_device(ctx, sw, frame_q, frame_t, R_il, t_il, static_cast<double*>(ctx->d_scratch));
        if (r2 != SRL_OK) return r2;
        SRL_CUDA(ctx, cudaMemcpyAsync(world_xyz_out + 3 * b, ctx->d_scratch, (e - b) * 3 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    return SRL_OK;
}

// ---- host unit hook for the per-keypoint math (same source as the kernel's phase 2) -------------------------
struct HostNb {
    const double* p;
    SRL_HD bool use(int) const { return true; }
    SRL_HD void get(int j, float& x, float& y, float& z) const { x = (float)p[3 * j]; y = (float)p[3 * j + 1]; z = (float)p[3 * j + 2]; }
};
int srl_host_plane_fit(const double* nbr_xyz, int32_t K, double normal[3], double* a2D, double evals[3]) {
    if (!nbr_xyz || K < 1 || !normal || !a2D || !evals) return SRL_BAD_ARG;
    HostNb nb{nbr_xyz};
    // run the same plane_residual the kernel runs, with an identity pose, and read normal / a2D back
    PassConst c;
    std::memset(&c, 0, sizeof(c));
    c.Rq[0] = c.Rq[4] = c.Rq[8] = 1.0; c.Rn[0] = c.Rn[4] = c.Rn[8] = 1.0; c.R_il[0] = c.R_il[4] = c.R_il[8] = 1.0;
    c.size = 1.0; c.lambda_w = 0.9; c.lambda_n = 0.1; c.power = 2.0; c.dmax = 0.3; c.exp_den = 6.0; c.K = K; c.Kmin = K; c.nb = 1; c.thr_occ = 1;
    PlaneRow row;
    plane_residual<0>(nb, K, nbr_xyz[0], nbr_xyz[1], nbr_xyz[2], c, nbr_xyz[0], nbr_xyz[1], nbr_xyz[2], 0.0, 0.0, 0.0, row);
    normal[0] = row.nx; normal[1] = row.ny; normal[2] = row.nz;
    // eigenvalues from the same solver
    double mx = 0, my = 0, mz = 0;
    for (int j = 0; j < K; ++j) { mx += (double)(float)nbr_xyz[3 * j]; my += (double)(float)nbr_xyz[3 * j + 1]; mz += (double)(float)nbr_xyz[3 * j + 2]; }
    mx /= K; my /= K; mz /= K;
    double c00 = 0, c01 = 0, c02 = 0, c11 = 0, c12 = 0, c22 = 0;
    for (int j = 0; j < K; ++j) {
        double dx = (double)(float)nbr_xyz[3 * j] - mx, dy = (double)(float)nbr_xyz[3 * j + 1] - my, dz = (double)(float)nbr_xyz[3 * j + 2] - mz;
        c00 += dx * dx; c01 += dx * dy; c02 += dx * dz; c11 += dy * dy; c12 += dy * dz; c22 += dz * dz;
    }
    double n0, n1, n2;
    eig3_sym(c00, c01, c11, c02, c12, c22, evals, n0, n1, n2);
    *a2D = (std::sqrt(std::fabs(evals[1])) - std::sqrt(std::fabs(evals[0]))) / std::sqrt(std::fabs(evals[2]));
    return SRL_OK;
}

}  // extern "C"
