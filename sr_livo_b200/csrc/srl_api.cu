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
    if (ctx->d_scratch) cudaStreamSynchronize(ctx->stream);
    const size_t want = bytes + bytes / 4;
    SRL_CUDA(ctx, ctx->d_scratch.alloc(want));
    ctx->scratch_bytes = want;
    return SRL_OK;
}
int ensure_pinned(srl_ctx* ctx, size_t bytes) {
    if (bytes <= ctx->pinned_bytes) return SRL_OK;
    if (ctx->h_pinned) cudaStreamSynchronize(ctx->stream);
    const size_t want = bytes + bytes / 4;
    SRL_CUDA(ctx, ctx->h_pinned.alloc(want));
    ctx->pinned_bytes = want;
    return SRL_OK;
}
MemKind mem_kind(const void* p) {
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, p) != cudaSuccess) { cudaGetLastError(); return MemKind::Pageable; }
    if (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged) return MemKind::Device;
    return attr.type == cudaMemoryTypeHost ? MemKind::Pinned : MemKind::Pageable;
}
int copy_to_host(srl_ctx* ctx, void* dst, const void* d_src, size_t bytes) {
    if (bytes == 0) return SRL_OK;
    if (mem_kind(dst) == MemKind::Pinned) {
        SRL_CUDA(ctx, cudaMemcpyAsync(dst, d_src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
        SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        return SRL_OK;
    }
    const size_t chunk = std::min(bytes, size_t(64) << 20);   // no host temporary the size of the output
    int rc = ensure_pinned(ctx, chunk);
    if (rc != SRL_OK) return rc;
    for (size_t off = 0; off < bytes; off += chunk) {
        const size_t len = std::min(chunk, bytes - off);
        SRL_CUDA(ctx, cudaMemcpyAsync(ctx->h_pinned, static_cast<const char*>(d_src) + off, len, cudaMemcpyDeviceToHost, ctx->stream));
        SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        std::memcpy(static_cast<char*>(dst) + off, ctx->h_pinned, len);
    }
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

// Chunk schedule of the ordered residual cap, shared by the host-driven and the device-resident loop: chunk 0 is
// [0, max(4096, 2 max(cap, 1))), each later chunk twice as long, the last one clipped to n.  Returns the n_chunks + 1
// boundaries.  k2_cap_reduce adds each chunk's block sum to the pass's sums, so the boundaries fix the summation order:
// with the same schedule both loops' capped sums are bitwise equal whenever the pass constants are.
static std::vector<long long> cap_chunk_bounds(long long n, long long cap) {
    std::vector<long long> b(1, 0);
    long long chunk = std::max<long long>(4096, 2 * std::max<long long>(cap, 1));
    while (b.back() < n) {
        b.push_back(std::min(n, b.back() + chunk));
        chunk *= 2;
    }
    return b;
}

constexpr bool kDefaultSplit = true;    // variant 0 (auto): k1_scan + k1_fit (H100, 100k-point sweep: 0.46 vs 0.75 ms per sweep for k1_fast in the same run, BASELINE.md)

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
        if (probe_concurrent_kernels(ctx->loop_stream, ctx->stream, ctx->d_stats->probe, &ok) != cudaSuccess) { cudaGetLastError(); ok = false; }
        ctx->concurrent_kernels = ok ? 1 : 0;
    }
    return ctx->concurrent_kernels == 1;
}


// Spins until the mapped sequence word *p holds `seq`, which the device writes behind its result; falls back to the status
// of stream `s` so that a failed launch or a device fault is reported instead of spinning forever.
static int wait_host_seq(srl_ctx* ctx, const volatile unsigned long long* p, unsigned long long seq, cudaStream_t s,
                         const char* unpublished, const char* query_failed) {
    for (unsigned long long spins = 1;; ++spins) {
        if (*p == seq) break;
        if ((spins & 0x3fffull) == 0) {
            const cudaError_t q = cudaStreamQuery(s);
            if (q == cudaSuccess) {   // everything ran: the word must be there (or the kernel never published)
                if (*p == seq) break;
                return set_err(ctx, SRL_CUDA_ERROR, unpublished);
            }
            if (q != cudaErrorNotReady) return cuda_fail(ctx, q, query_failed);
        }
    }
    std::atomic_thread_fence(std::memory_order_acquire);
    return SRL_OK;
}
// Result of a pass through the mapped host buffer: arm_host_result() before the launch, wait_host_result() after it.
static void arm_host_result(srl_ctx* ctx, PassArgs& a) {
    a.sink.host_out = ctx->h_out32.dev();
    a.sink.host_seq = ++ctx->host_seq;
}
static int wait_host_result(srl_ctx* ctx, const PassArgs& a) {
    return wait_host_seq(ctx, reinterpret_cast<volatile unsigned long long*>(ctx->h_out32 + 32), a.sink.host_seq, ctx->stream,
                         "the pass finished without publishing its result", "cudaStreamQuery while waiting for a pass");
}

// The Morton order of the sweep's keypoints (srl_fast.cu), computed once per upload, right behind the copy that brings
// the keypoints to HBM (so it is off the critical path of the first pass); a pass computes it only if that failed.
static int ensure_order(srl_ctx* ctx, srl_sweep* sw) {
    SRL_CUDA(ctx, sw->d_order.ensure(sw->capacity));
    if (!sw->order_valid && sw->n > 0) {
        int rc;
        size_t need = 0;
        sweep_compute_order(ctx->choice, sw->d_raw, (long long)sw->n, sw->d_order, nullptr, 0, &need, ctx->stream);
        if ((rc = ensure_scratch(ctx, need)) != SRL_OK) return rc;
        SRL_CUDA(ctx, sweep_compute_order(ctx->choice, sw->d_raw, (long long)sw->n, sw->d_order, ctx->d_scratch, ctx->scratch_bytes, &need, ctx->stream));
        sw->order_valid = true;
        ctx->launches += 1;
    }
    return SRL_OK;
}

// assoc: k1_assoc alone (nb = 2, K != 20, forced exact selection, option); fast / split: k1_fast or k1_scan + k1_fit, then
// k1_assoc on the keypoints they flagged.  The ordered residual cap (rows) needs keypoint order, which only split offers.
enum class PassForm { assoc, fast, split };
static PassForm pass_form(const srl_ctx* ctx, const PassArgs& a) {
    const bool split = ctx->variant == 3 || (ctx->variant == 0 && kDefaultSplit);
    if (ctx->force_exact || ctx->variant == 2 || a.c.nb > 1 || a.c.K != 20 || a.c.Kmin != 20 || (a.out.rows && !split)) return PassForm::assoc;
    return split ? PassForm::split : PassForm::fast;
}
// Everything a pass needs besides its kernel launches: buffers, the sweep's Morton order, cleared flags / candidate rows,
// and (once per kernel choice) the kernels themselves; binds the sweep's buffers of the pass's form into `a`.
// Idempotent.  The device-resident loop calls it BEFORE it launches the persistent ESIKF block: an allocation, a module
// load (CUDA loads kernels lazily, and loading waits for running kernels) or a synchronous copy issued while that block
// spins would deadlock against it.
static int prepare_pass(srl_ctx* ctx, srl_sweep* sw, PassArgs& a) {
    if (!ctx->kernels_preloaded) {
        size_t max_local = 0;
        SRL_CUDA(ctx, preload_fast_kernels(ctx->choice, &max_local));
        SRL_CUDA(ctx, preload_assoc_kernels(ctx->choice, a.c.K, &max_local));
        // The first launch of a kernel whose local memory (spills) exceeds the context's reservation makes the driver
        // grow that reservation, and the driver waits for the device to go idle to do it.  Launched behind the persistent
        // ESIKF block, which spins until the pass finishes, that wait never ends (k1_fast keeps a ~1.6 KB spill frame on
        // sm_90a).  So the reservation is grown here, while nothing spins, to fit every pass kernel.
        size_t stack = 0;
        SRL_CUDA(ctx, cudaDeviceGetLimit(&stack, cudaLimitStackSize));
        if (max_local > stack) SRL_CUDA(ctx, cudaDeviceSetLimit(cudaLimitStackSize, max_local));
        ctx->kernels_preloaded = true;
    }
    const PassForm form = pass_form(ctx, a);
    if (form == PassForm::assoc) return SRL_OK;
    int rc;
    if ((rc = ensure_order(ctx, sw)) != SRL_OK) return rc;
    SRL_CUDA(ctx, sw->d_flags.ensure(sw->capacity));
    // k1_scan / k1_fast write the flag of every keypoint of their range in every pass; the fallback launch walks the
    // flags of the whole sweep, so the keypoints outside this rank's range need zeros once per (upload, shard)
    if (!sw->flags_clean) {
        if (sw->n) SRL_CUDA(ctx, cudaMemsetAsync(sw->d_flags, 0, sw->n, ctx->stream));
        sw->flags_clean = true;
    }
    if (form == PassForm::split && !sw->d_cand_rows) {   // k1_fit loads whole rows and uses only the slots k1_scan filled: start from defined memory
        SRL_CUDA(ctx, sw->d_cand_rows.ensure(sw->capacity * (size_t)24 + 8));
        SRL_CUDA(ctx, cudaMemsetAsync(sw->d_cand_rows, 0, (sw->capacity * (size_t)24 + 8) * sizeof(unsigned), ctx->stream));
    }
    a.order = a.out.rows ? nullptr : sw->d_order.get();   // the residual cap consumes keypoints in their own order (src/optimize.cpp:68,107)
    a.flags = sw->d_flags; a.cand_rows = sw->d_cand_rows;
    return SRL_OK;
}

static int launch_pass(srl_ctx* ctx, srl_sweep* sw, PassArgs a, bool debug, bool pdl = false) {
    const long long n = a.k_end - a.k_begin;
    const bool timing = ctx->timing && !a.link.dev;   // the device-resident loop brackets its passes with events of its own
    {
        const int rc = prepare_pass(ctx, sw, a);
        if (rc != SRL_OK) return rc;
    }
    if (timing) {
        ctx->ev_cur ^= 1;
        timing_collect_pair(ctx, ctx->ev_cur);   // the pair used two passes ago
        cudaEventRecord(ctx->ev0[ctx->ev_cur], ctx->stream);
    }
    const PassForm form = pass_form(ctx, a);
    if (form == PassForm::assoc) {
        SRL_CUDA(ctx, launch_k1(ctx, a, n, debug, pdl));
        ctx->launches += 1;
    } else {
        PassArgs first = a;   // its sums go to d_fast_out; the range is one of SORTED positions unless the pass is capped
        first.sink.out32 = ctx->d_fast_out;
        if (form == PassForm::split) {
            // k1_fit finalises the pass itself when nothing was flagged (multi-GPU: after running the exchange); the
            // fallback launch then runs off the host's critical path and republishes the same values
            SRL_CUDA(ctx, launch_k1_split(ctx, first, n, debug, pdl));
            ctx->launches += 1;
        } else {
            SRL_CUDA(ctx, launch_k1_fast(ctx, first, n, debug));
        }
        // exact selection for the keypoints the first launch could not decide; its last block adds the first launch's sums
        a.only_flagged = a.flags; a.prev_out32 = ctx->d_fast_out;
        if (a.order) { a.k_begin = 0; a.k_end = (long long)sw->n; }   // Morton order: the range's keypoints are scattered over the sweep
        SRL_CUDA(ctx, launch_k1(ctx, a, (long long)sw->n, debug, pdl));   // its grid covers the flags of the whole sweep
        ctx->launches += 2;
    }
    if (timing) { cudaEventRecord(ctx->ev1[ctx->ev_cur], ctx->stream); ctx->ev_pending[ctx->ev_cur] = true; }
    return SRL_OK;
}

// The integer options of srl_ctx_set_option: the values each accepts, where the ctx keeps it, and the environment variable
// srl_ctx_create reads it from (a value outside the set leaves the default).  srl_ctx_get_counter reads each one back.
struct IntOption {
    const char* name;
    std::vector<int> allowed;
    int& (*field)(srl_ctx&);
    const char* env;
    const char* must_be;
};
static const IntOption kIntOptions[] = {
    {"k1_variant", {0, 1, 2, 3}, [](srl_ctx& c) -> int& { return c.variant; }, nullptr,
     "k1_variant must be 0 (auto), 1 (k1_fast), 2 (k1_assoc only) or 3 (k1_scan + k1_fit)"},
    {"shuffle_rule", {0, 1}, [](srl_ctx& c) -> int& { return c.shuffle_rule; }, nullptr, "shuffle_rule must be 0 (Lemire) or 1 (division)"},
    {"split_lanes_per_keypoint", {2, 4}, [](srl_ctx& c) -> int& { return c.choice.split_lpk; }, "SRL_SPLIT_LPK", "split_lanes_per_keypoint must be 2 or 4"},
    {"scan_min_blocks", {6, 8}, [](srl_ctx& c) -> int& { return c.choice.scan_minb; }, "SRL_SCAN_MINB", "scan_min_blocks must be 6 or 8"},
    {"fit_min_blocks", {4, 5, 6}, [](srl_ctx& c) -> int& { return c.choice.fit_minb; }, "SRL_FIT_MINB", "fit_min_blocks must be 4, 5 or 6"},
    {"fast_lanes_per_keypoint", {1, 2, 4}, [](srl_ctx& c) -> int& { return c.choice.fast_lpk; }, "SRL_FAST_LPK", "fast_lanes_per_keypoint must be 1, 2 or 4"},
    {"fast_min_blocks", {4, 5, 6, 8}, [](srl_ctx& c) -> int& { return c.choice.fast_minb; }, "SRL_FAST_MINB", "fast_min_blocks must be 4, 5, 6 or 8"},
    {"k1_min_blocks", {2, 3, 4}, [](srl_ctx& c) -> int& { return c.choice.k1_minb; }, "SRL_K1_MINB", "k1_min_blocks must be 2, 3 or 4"},
    {"cluster_order", {0, 1, 2, 3}, [](srl_ctx& c) -> int& { return c.choice.order_mode; }, "SRL_CLUSTER_ORDER", "cluster_order must be 0, 1, 2 or 3"},
};
static bool allowed(const IntOption& o, int64_t v) { return std::find(o.allowed.begin(), o.allowed.end(), v) != o.allowed.end(); }

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
    std::unique_ptr<srl_ctx> ctx(new srl_ctx());
    ctx->device = device;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) ctx->sm_count = prop.multiProcessorCount;
    if (cuda_stream) { ctx->stream = static_cast<cudaStream_t>(cuda_stream); ctx->own_stream = false; }
    else {
        if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) return SRL_CUDA_ERROR;
        ctx->own_stream = true;
    }
    ctx->max_grid = 2048;   // rows of the block-partials buffer (>= any grid we launch)
    const size_t n_chunks = (size_t)(ctx->max_grid / 32 + 1);
    bool ok = ctx->d_partials.alloc((size_t)ctx->max_grid * 32) == cudaSuccess &&
              ctx->d_ticket.alloc(1) == cudaSuccess &&
              ctx->d_chunk_tickets.alloc(n_chunks) == cudaSuccess &&
              cudaMemset(ctx->d_chunk_tickets, 0, n_chunks * sizeof(unsigned int)) == cudaSuccess &&
              ctx->d_chunk_sums.alloc(n_chunks * 32) == cudaSuccess &&
              ctx->d_out32.alloc(64) == cudaSuccess &&
              ctx->d_k2_state.alloc(4) == cudaSuccess &&
              ctx->d_cap_chunks.alloc(1) == cudaSuccess &&
              cudaMemset(ctx->d_cap_chunks, 0, sizeof(unsigned long long)) == cudaSuccess &&
              ctx->d_stats.alloc(1) == cudaSuccess &&
              ctx->d_fast_out.alloc(32) == cudaSuccess &&
              ctx->d_scan_count.alloc(1) == cudaSuccess &&
              cudaMemset(ctx->d_scan_count, 0, sizeof(unsigned long long)) == cudaSuccess &&
              cudaMemset(ctx->d_stats, 0, sizeof(PassStats)) == cudaSuccess &&
              ctx->h_out32.alloc(64) == cudaSuccess &&
              cudaStreamCreateWithFlags(&ctx->loop_stream, cudaStreamNonBlocking) == cudaSuccess &&
              ctx->d_iekf.alloc(1) == cudaSuccess &&
              cudaMemset(ctx->d_iekf, 0, sizeof(IekfDev)) == cudaSuccess &&
              ctx->h_iekf.alloc(1) == cudaSuccess &&
              cudaMemset(ctx->d_ticket, 0, sizeof(unsigned int)) == cudaSuccess;
    if (!ok) { cudaGetLastError(); return SRL_CUDA_ERROR; }
    std::memset(ctx->h_out32, 0, 64 * sizeof(double));
    std::memset(ctx->h_iekf, 0, sizeof(IekfHostOut));
    if (const char* e = getenv("SRL_DEVICE_LOOP")) ctx->device_loop = atoi(e) != 0;
    for (const IntOption& o : kIntOptions) {
        const char* e = o.env ? getenv(o.env) : nullptr;
        if (e && allowed(o, atoi(e))) o.field(*ctx) = atoi(e);
    }
    ctx->choice.restart_order_checks();
    *out = ctx.release();
    return SRL_OK;
}

void srl_ctx_destroy(srl_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    if (ctx->loop_stream) cudaStreamSynchronize(ctx->loop_stream);
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
    if (n == "device_loop") { ctx->device_loop = value != 0; return SRL_OK; }
    if (n == "shuffle_on_host") { ctx->shuffle_on_host = value != 0; return SRL_OK; }
    for (const IntOption& o : kIntOptions) {
        if (n != o.name) continue;
        if (!allowed(o, value)) return set_err(ctx, SRL_BAD_ARG, o.must_be);
        o.field(*ctx) = (int)value;
        if (n == "cluster_order") ctx->choice.restart_order_checks();
        ctx->kernels_preloaded = false;   // the next pass loads the instances of the choice (before any persistent block spins)
        return SRL_OK;
    }
    return set_err(ctx, SRL_BAD_ARG, "unknown option " + n);
}
int srl_ctx_get_counter(srl_ctx* ctx, const char* name, int64_t* value) {
    if (!ctx || !name || !value) return SRL_BAD_ARG;
    const std::string n(name);
    if (n == "exact_fallbacks") {
        unsigned long long v = 0;
        SRL_CUDA(ctx, cudaMemcpyAsync(&v, &ctx->d_stats->exact_fallbacks, sizeof(v), cudaMemcpyDeviceToHost, ctx->stream));
        SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        *value = (int64_t)v;
        return SRL_OK;
    }
    if (n == "fast_ambiguous") {
        unsigned long long v = 0;
        SRL_CUDA(ctx, cudaMemcpyAsync(&v, &ctx->d_stats->fast_ambiguous, sizeof(v), cudaMemcpyDeviceToHost, ctx->stream));
        SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        *value = (int64_t)v;
        return SRL_OK;
    }
    if (n == "cap_chunks_run") {   // capped chunks whose kernels did work in the last update (all its passes) or pass call
        if (ctx->cap_chunks_on_device) {
            unsigned long long v = 0;
            SRL_CUDA(ctx, cudaMemcpyAsync(&v, ctx->d_cap_chunks, sizeof(v), cudaMemcpyDeviceToHost, ctx->stream));
            SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            ctx->cap_chunks_run = (int64_t)v;
            ctx->cap_chunks_on_device = false;
        }
        *value = ctx->cap_chunks_run;
        return SRL_OK;
    }
    if (n == "kernel_launches") { *value = ctx->launches; return SRL_OK; }
    if (n.rfind("iekf_stage_", 0) == 0 && n.size() == 12 && n[11] >= '0' && n[11] <= '7') { *value = ctx->h_iekf->stage_cycles[n[11] - '0']; return SRL_OK; }
    if (n == "cluster_order_active") { *value = ctx->choice.order_state; return SRL_OK; }
    for (const IntOption& o : kIntOptions)
        if (n == o.name) { *value = o.field(*ctx); return SRL_OK; }
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
            SRL_CUDA(ctx, ctx->ev0[i].create());
            SRL_CUDA(ctx, ctx->ev1[i].create());
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
    std::unique_ptr<srl_sweep> s(new srl_sweep());
    s->ctx = ctx; s->device = ctx->device; s->capacity = capacity;
    SRL_CUDA(ctx, s->d_raw.alloc(capacity * 3));
    *out = s.release();
    return SRL_OK;
}
void srl_sweep_destroy(srl_sweep* s) {
    if (!s) return;
    cudaSetDevice(s->device);
    delete s;
}
int srl_sweep_upload(srl_sweep* s, const double* raw_xyz, size_t n) {
    if (!s || (n && !raw_xyz)) return SRL_BAD_ARG;
    srl_ctx* ctx = s->ctx;
    if (n > s->capacity) return set_err(ctx, SRL_BAD_ARG, "srl_sweep_upload: n exceeds capacity");
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    if (n) {
        // pinned caller memory goes straight to the DMA engine; pageable memory is staged through a pinned buffer
        const bool pinned = mem_kind(raw_xyz) == MemKind::Pinned;
        if (!pinned) {
            int rc = ensure_pinned(ctx, n * 3 * sizeof(double));
            if (rc != SRL_OK) return rc;
            std::memcpy(ctx->h_pinned, raw_xyz, n * 3 * sizeof(double));
        }
        SRL_CUDA(ctx, cudaMemcpyAsync(s->d_raw, pinned ? raw_xyz : static_cast<const double*>(ctx->h_pinned.get()), n * 3 * sizeof(double),
                                      cudaMemcpyHostToDevice, ctx->stream));
        // the staging buffer is shared by every upload of the ctx: it must not be refilled while the DMA still reads it
        // (pinned caller memory is read asynchronously: the caller keeps it unchanged until the next synchronising call)
        if (!pinned) SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    s->n = n; s->shard_begin = 0; s->shard_end = n; s->order_valid = false; s->flags_clean = false;
    return ensure_order(ctx, s);
}
int srl_sweep_set_device(srl_sweep* s, const double* d_raw_xyz, size_t n) {
    if (!s || (n && !d_raw_xyz)) return SRL_BAD_ARG;
    srl_ctx* ctx = s->ctx;
    if (n > s->capacity) return set_err(ctx, SRL_BAD_ARG, "srl_sweep_set_device: n exceeds capacity");
    SRL_CUDA(ctx, cudaMemcpyAsync(s->d_raw, d_raw_xyz, n * 3 * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
    s->n = n; s->shard_begin = 0; s->shard_end = n; s->order_valid = false; s->flags_clean = false;
    return ensure_order(ctx, s);
}
int srl_sweep_set_shard(srl_sweep* s, size_t begin, size_t end) {
    if (!s || begin > end || end > s->n) return SRL_BAD_ARG;
    s->shard_begin = begin; s->shard_end = end; s->flags_clean = false;
    return SRL_OK;
}
int srl_sweep_download_order(srl_sweep* s, uint32_t* order, size_t max_n, int64_t* n_out) {
    if (!s) return SRL_BAD_ARG;
    srl_ctx* ctx = s->ctx;
    if (n_out) *n_out = (int64_t)s->n;
    if (!order || s->n == 0) return SRL_OK;
    if (max_n < s->n) return set_err(ctx, SRL_BAD_ARG, "srl_sweep_download_order: output too small");
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    int rc;
    if ((rc = ensure_order(ctx, s)) != SRL_OK) return rc;
    SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return copy_to_host(ctx, order, s->d_order, s->n * sizeof(unsigned));
}

// ---- one pass ----------------------------------------------------------------------------------------------
// The srl_last_error text of a failed pass or of a failed device-resident loop, the same on every entry point.
static int status_error(srl_ctx* ctx, int code) {
    switch (code) {
        case SRL_TOO_FEW_RESIDUALS: return set_err(ctx, code, "[Optimization] Error : not enough keypoints selected in ct-icp !");
        case SRL_NAN_PLANARITY: return set_err(ctx, code, "NaN planarity (the reference throws at src/optimize.cpp:348)");
        case SRL_COMM_ERROR: return set_err(ctx, code, "peer exchange timed out (a rank did not reach this pass)");
        case SRL_SINGULAR: return set_err(ctx, code, "the 6x6 system of the ESIKF gain is singular (src/optimize.cpp:234,237)");
        default: return set_err(ctx, code, "device-resident updateIEKF loop failed");
    }
}

// The ordered residual cap (src/optimize.cpp:107) applies when max_num_residuals is below the keypoints of the pass.  It is
// implemented on an unsharded sweep of one GPU only: `rejected` sets the error, and the caller returns SRL_BAD_ARG.
enum class Cap { none, capped, rejected };
static Cap cap_mode(srl_ctx* ctx, const srl_icp_params* prm, const srl_sweep* sw, const srl_comm* comm) {
    const long long cap = prm->max_num_residuals;
    if (comm) {   // the whole sweep is the sum of every rank's local sweep
        if (cap >= (long long)sw->n) return Cap::none;
        set_err(ctx, SRL_BAD_ARG, "the sharded update does not implement the max_num_residuals cap");
        return Cap::rejected;
    }
    if (cap >= (long long)(sw->shard_end - sw->shard_begin)) return Cap::none;
    if (sw->shard_begin == 0 && sw->shard_end == sw->n) return Cap::capped;
    set_err(ctx, SRL_BAD_ARG, "max_num_residuals < shard size is only supported on an unsharded sweep");
    return Cap::rejected;
}

static srl_frame make_frame(const double q[4], const double t[3], const double t_last[3], const double R_il[9], const double t_il[3]) {
    srl_frame f;
    std::memcpy(f.q_cur, q, sizeof(f.q_cur));
    std::memcpy(f.t_cur, t, sizeof(f.t_cur));
    std::memcpy(f.t_last, t_last, sizeof(f.t_last));
    std::memcpy(f.R_il, R_il, sizeof(f.R_il));
    std::memcpy(f.t_il, t_il, sizeof(f.t_il));
    return f;
}

static MapView map_view(const srl_map& m) { return {m.d_slots, (unsigned)(m.capacity - 1), m.d_blocks}; }

// Describes a pass; launch_pass and launch_cap_chunk only adjust the range, the sink and the link of what they launch.
// `comm`: the pass's last kernel exchanges the 32 sums with the peers, so every rank gets the whole sweep's.
static int fill_pass_args(srl_ctx* ctx, const srl_comm* comm, srl_map* map, srl_sweep* sw, const srl_frame* frame, const srl_icp_params* prm,
                          PassArgs& a) {
    int rc = check_params(ctx, prm);
    if (rc != SRL_OK) return rc;
    if (!map || !sw || !frame) return set_err(ctx, SRL_BAD_ARG, "null map/sweep/frame");
    if (map->ctx != ctx || sw->ctx != ctx) return set_err(ctx, SRL_BAD_ARG, "map/sweep belong to another ctx");
    if ((rc = check_lio_map(ctx, map)) != SRL_OK) return rc;
    if (std::fabs(prm->size_voxel_map - map->voxel_size) > 0) return set_err(ctx, SRL_BAD_ARG, "icp size_voxel_map differs from the map's voxel size");
    std::memset(&a, 0, sizeof(a));
    make_pass_const(*frame, *prm, a.c);
    a.map = map_view(*map);
    a.raw = sw->d_raw; a.k_begin = (long long)sw->shard_begin; a.k_end = (long long)sw->shard_end;
    a.partials = ctx->d_partials; a.ticket = ctx->d_ticket; a.sink.out32 = ctx->d_out32;
    a.stats = ctx->d_stats;
    a.force_amb_mod = ctx->force_amb_mod;
    a.scan_count = ctx->d_scan_count; a.chunk_tickets = ctx->d_chunk_tickets; a.chunk_sums = ctx->d_chunk_sums;
    a.eps_scale = ctx->force_exact ? std::numeric_limits<float>::infinity() : 1.0f;
    if (comm) {
        CommDev& cm = a.sink.comm;
        cm.world = comm->world; cm.rank = comm->rank; cm.seq = comm->d_seq;
        for (int r = 0; r < comm->world; ++r) cm.mail[r] = comm->peer[r];
    }
    return SRL_OK;
}

// Chunk j of a capped pass over the keypoints [bounds[j], bounds[j + 1]): the pass kernels, then k2_cap_reduce.  In the
// device-resident loop (a.link.dev set) all chunks are enqueued at once: a chunk after the one that found k* leaves at once,
// and k2_cap_reduce of the chunk that found k* (or of the last one) hands the pass's sums to the ESIKF block.
static int launch_cap_chunk(srl_ctx* ctx, srl_sweep* sw, PassArgs a, const std::vector<long long>& bounds, size_t j, int cap,
                            bool debug, bool pdl) {
    a.k_begin = bounds[j]; a.k_end = bounds[j + 1];
    if (a.link.dev && j) a.link.cap_state = ctx->d_k2_state;
    const int rc = launch_pass(ctx, sw, a, debug, pdl);
    if (rc != SRL_OK) return rc;
    K2Args k2;
    std::memset(&k2, 0, sizeof(k2));
    k2.rows = sw->d_rows; k2.status = sw->d_status; k2.k_begin = a.k_begin; k2.k_end = a.k_end; k2.cap = cap;
    k2.chunk = (int)j; k2.state = ctx->d_k2_state; k2.out32 = ctx->d_out32 + 32;
    if (a.link.dev) {
        k2.last = j + 2 == bounds.size() ? 1 : 0;
        k2.pass_out32 = ctx->d_out32; k2.chunks_run = ctx->d_cap_chunks;
        k2.link = a.link;
    }
    const cudaError_t e = launch_k2(k2, ctx->stream, pdl);
    if (e != cudaSuccess) return cuda_fail(ctx, e, "launch_k2");
    ctx->launches += 1;
    return SRL_OK;
}

int srl_build_plane_residuals_async(srl_ctx* ctx, srl_map* map, srl_sweep* sw, const srl_frame* frame, const srl_icp_params* prm,
                                    double* d_out32) {
    if (!ctx || !d_out32) return SRL_BAD_ARG;
    PassArgs a;
    int rc = fill_pass_args(ctx, nullptr, map, sw, frame, prm, a);
    if (rc != SRL_OK) return rc;
    const long long n = a.k_end - a.k_begin;
    if ((long long)prm->max_num_residuals < n) return set_err(ctx, SRL_BAD_ARG, "async pass does not implement the max_num_residuals cap");
    a.sink.out32 = d_out32;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    if (n <= 0) { SRL_CUDA(ctx, cudaMemsetAsync(d_out32, 0, 32 * sizeof(double), ctx->stream)); return SRL_OK; }
    return launch_pass(ctx, sw, a, false);
}

int srl_normal_eq_unpack(const double* h_out32, srl_normal_eq* out) {
    if (!h_out32 || !out) return SRL_BAD_ARG;
    unpack32(h_out32, out, 0);
    return SRL_OK;
}

// One pass (buildPlaneResiduals, src/optimize.cpp:153) with the host waiting for its sums, unpacked into `out`.  Adds the
// capped chunks it runs to the counter "cap_chunks_run".  `comm`: the pass exchanges its sums with the peers (see fill_pass_args).
static int run_pass(srl_ctx* ctx, srl_comm* comm, srl_map* map, srl_sweep* sw, const srl_frame* frame, const srl_icp_params* prm,
                    srl_normal_eq* out, srl_debug_out* dbg) {
    PassArgs a;
    int rc = fill_pass_args(ctx, comm, map, sw, frame, prm, a);
    if (rc != SRL_OK) return rc;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    std::memset(out, 0, sizeof(*out));
    const long long n = a.k_end - a.k_begin;
    const int K = a.c.K;
    const Cap cap = cap_mode(ctx, prm, sw, comm);
    if (cap == Cap::rejected) return SRL_BAD_ARG;
    const bool capped = cap == Cap::capped;
    const bool debug = dbg != nullptr;
    if (debug) {
        if (sw->dbg_K != K) {   // neighbour arrays depend on K
            sw->d_dbg_nbr.reset(); sw->d_dbg_nbr_dist.reset(); sw->dbg_K = K;
        }
        SRL_CUDA(ctx, sw->d_dbg_world.ensure(sw->capacity * 3));
        SRL_CUDA(ctx, sw->d_dbg_nbr.ensure(sw->capacity * K * 4));
        SRL_CUDA(ctx, sw->d_dbg_nbr_dist.ensure(sw->capacity * K));
        SRL_CUDA(ctx, sw->d_dbg_plane.ensure(sw->capacity * 16));
        SRL_CUDA(ctx, cudaMemsetAsync(sw->d_dbg_world, 0, sw->capacity * 3 * sizeof(double), ctx->stream));
        SRL_CUDA(ctx, cudaMemsetAsync(sw->d_dbg_nbr, 0xff, sw->capacity * K * 4 * sizeof(short), ctx->stream));
        SRL_CUDA(ctx, cudaMemsetAsync(sw->d_dbg_nbr_dist, 0, sw->capacity * K * sizeof(double), ctx->stream));
        SRL_CUDA(ctx, cudaMemsetAsync(sw->d_dbg_plane, 0, sw->capacity * 16 * sizeof(double), ctx->stream));
        a.out.dbg_world = sw->d_dbg_world; a.out.dbg_nbr = sw->d_dbg_nbr; a.out.dbg_nbr_dist = sw->d_dbg_nbr_dist; a.out.dbg_plane = sw->d_dbg_plane;
    }
    if (debug || capped) {
        SRL_CUDA(ctx, sw->d_status.ensure(sw->capacity));
        SRL_CUDA(ctx, cudaMemsetAsync(sw->d_status, 0, sw->capacity * sizeof(int), ctx->stream));
        a.out.status = sw->d_status;
    }
    double* h = ctx->h_out32;
    double zero32[32];
    if (n <= 0 && !comm) {
        // an empty shard sums to zero (the mapped buffer may still be written by the previous pass's fallback launch); with
        // a comm it runs its pass all the same: the peers wait for its part of the exchange
        std::memset(zero32, 0, sizeof(zero32));
        h = zero32;
    } else if (!capped) {
        arm_host_result(ctx, a);
        if ((rc = launch_pass(ctx, sw, a, debug)) != SRL_OK) return rc;
        if ((rc = wait_host_result(ctx, a)) != SRL_OK) return rc;
    } else {
        // ordered cap (src/optimize.cpp:107): process keypoints in order, chunk by chunk, until k* is found
        SRL_CUDA(ctx, sw->d_rows.ensure(sw->capacity * 8));
        a.out.rows = sw->d_rows;
        double* d_cap_out = ctx->d_out32 + 32;
        SRL_CUDA(ctx, cudaMemsetAsync(d_cap_out, 0, 32 * sizeof(double), ctx->stream));
        SRL_CUDA(ctx, cudaMemsetAsync(ctx->d_k2_state, 0, 4 * sizeof(long long), ctx->stream));
        const std::vector<long long> bounds = cap_chunk_bounds(n, prm->max_num_residuals);
        double scanned = 0;
        long long st[4] = {0, 0, 0, 0};
        for (size_t j = 0; j + 1 < bounds.size(); ++j) {
            if ((rc = launch_cap_chunk(ctx, sw, a, bounds, j, (int)prm->max_num_residuals, debug, false)) != SRL_OK) return rc;
            ctx->cap_chunks_run += 1;
            SRL_CUDA(ctx, cudaMemcpyAsync(h, ctx->d_out32, 32 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
            SRL_CUDA(ctx, cudaMemcpyAsync(st, ctx->d_k2_state, sizeof(st), cudaMemcpyDeviceToHost, ctx->stream));
            SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            scanned += h[30];
            if (st[1]) break;   // k* found: the reference loop has hit its `break`
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
        h[30] = scanned;   // candidates scanned in the chunks processed (an upper bound of the reference's count up to k*)
    }
    // a failed exchange makes all 32 sums NaN; [31] is a count, which a NaN Jacobian (NaN planarity) never turns into NaN
    if (h[31] != h[31]) return status_error(ctx, SRL_COMM_ERROR);
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
    if (out->nan_planarity) return status_error(ctx, SRL_NAN_PLANARITY);
    if (out->num_residuals < prm->min_number_neighbors) return status_error(ctx, SRL_TOO_FEW_RESIDUALS);
    return SRL_OK;
}

int srl_build_plane_residuals(srl_ctx* ctx, srl_map* map, srl_sweep* sw, const srl_frame* frame, const srl_icp_params* prm,
                              srl_normal_eq* out, srl_debug_out* dbg) {
    if (!ctx || !out) return SRL_BAD_ARG;
    ctx->cap_chunks_run = 0; ctx->cap_chunks_on_device = false;   // counter "cap_chunks_run": this call's chunks
    return run_pass(ctx, nullptr, map, sw, frame, prm, out, dbg);
}

// ---- iterated update ---------------------------------------------------------------------------------------
// Row N1: the whole updateIEKF loop enqueued at once.  Pass 0 takes its pose by value; every later pass reads the pose
// the persistent ESIKF block (k_iekf_loop) left in HBM and leaves immediately once the loop has ended on the device.  One host wait at the end, on
// the sequence flag the finishing step writes into mapped pinned memory after the state, the trace and the summary.
// The loop kernel's arguments for one sweep: updateIEKF's state, frame pose and thresholds, pass 0's constants, a fresh
// ticket base (so nothing on the device has to be reset) and a fresh host sequence number.
static int iekf_loop_args(srl_ctx* ctx, const srl_eskf_state* eskf, const double frame_q[4], const double frame_t[3],
                          const PassConst& pc0, const srl_icp_params* prm, int world, IekfLoopArgs& la) {
    srl_iekf_iter it;
    int rc;
    if ((rc = srl_iekf_begin(eskf, prm, &it)) != SRL_OK) return rc;
    const int n_pass = it.max_num_iter + 1;                          // i = -1 .. max_iter - 1 (src/optimize.cpp:147)
    if (n_pass > kLoopMaxPasses) return set_err(ctx, SRL_BAD_ARG, "num_iters_icp > 39 is not supported by the device-resident loop");
    static_assert(sizeof(IekfLoopArgs) <= 4000, "the loop kernel's arguments must fit the 4 KB kernel parameter space");
    std::memset(&la, 0, sizeof(la));
    IekfInit& init = la.init;
    init.eskf = *eskf;
    std::memcpy(init.frame_q, frame_q, sizeof(init.frame_q));
    std::memcpy(init.frame_t, frame_t, sizeof(init.frame_t));
    init.pc0 = pc0;
    init.laser_cov = prm->laser_point_cov; init.thr_t = prm->threshold_translation_norm; init.thr_r = prm->threshold_orientation_norm;
    init.max_iter = it.max_num_iter; init.frame_id = prm->frame_id; init.min_neighbors = prm->min_number_neighbors;
    la.dev = ctx->d_iekf; la.host_out = ctx->h_iekf.dev(); la.host_seq = ++ctx->iekf_seq;
    la.base = ctx->loop_base; ctx->loop_base += 64;
    la.world = world; la.n_pass = n_pass;
    return SRL_OK;
}

// A pass could not be enqueued: the persistent block is waiting for it.  Tell it, wait for it to leave, report `rc`.
static int iekf_loop_abort(srl_ctx* ctx, int rc) {
    const std::string why = ctx->err;
    launch_iekf_abort(ctx->d_iekf, ctx->stream);
    cudaStreamSynchronize(ctx->loop_stream);
    cudaGetLastError();
    return set_err(ctx, rc, why);
}

// The one host wait of the sweep (on the sequence word the finishing step writes into mapped pinned memory after the
// state, the trace and the summary), then the result.  `timed`: the passes were bracketed by ctx->loop_ev0/1.
static int iekf_loop_finish(srl_ctx* ctx, const IekfLoopArgs& st, bool timed, srl_eskf_state* eskf, double frame_q[4],
                            double frame_t[3], srl_iekf_summary* summary) {
    const int rc = wait_host_seq(ctx, &ctx->h_iekf->seq, st.host_seq, ctx->loop_stream,   // the ESIKF block leaves right after publishing
                                 "the device-resident updateIEKF loop finished without publishing its result",
                                 "cudaStreamQuery while waiting for the updateIEKF loop");
    if (rc != SRL_OK) return rc;
    const IekfHostOut* h = ctx->h_iekf;
    const int passes = h->passes_run;
    const int n_pass = st.n_pass;
    if (timed) {   // the passes that ran have finished (their events precede the step that published)
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
    return h->status == SRL_OK ? SRL_OK : status_error(ctx, h->status);
}

// `capped`: the ordered residual cap on an unsharded, non-empty sweep (cap_mode).
static int update_iekf_device(srl_ctx* ctx, srl_comm* comm, srl_map* map, srl_sweep* sw, srl_eskf_state* eskf, double frame_q[4],
                              double frame_t[3], const double t_last[3], const double R_il[9], const double t_il[3],
                              const srl_icp_params* prm, bool capped, srl_iekf_summary* summary) {
    const srl_frame fr = make_frame(frame_q, frame_t, t_last, R_il, t_il);
    PassArgs a;
    int rc = fill_pass_args(ctx, comm, map, sw, &fr, prm, a);
    if (rc != SRL_OK) return rc;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    IekfLoopArgs la;
    if ((rc = iekf_loop_args(ctx, eskf, frame_q, frame_t, a.c, prm, comm ? comm->world : 1, la)) != SRL_OK) return rc;
    // ordered residual cap (src/optimize.cpp:107): every pass is the chunk schedule of the host-driven loop, each chunk's
    // pass kernels followed by k2_cap_reduce; the chunks after k* leave at once
    std::vector<long long> bounds;
    if (capped) {
        SRL_CUDA(ctx, sw->d_rows.ensure(sw->capacity * 8));
        SRL_CUDA(ctx, sw->d_status.ensure(sw->capacity));
        a.out.rows = sw->d_rows; a.out.status = sw->d_status;
        bounds = cap_chunk_bounds(a.k_end - a.k_begin, prm->max_num_residuals);
        SRL_CUDA(ctx, cudaMemsetAsync(ctx->d_cap_chunks, 0, sizeof(unsigned long long), ctx->stream));
        ctx->cap_chunks_on_device = true;
    }
    if ((rc = prepare_pass(ctx, sw, a)) != SRL_OK) return rc;   // (with rows set: the same pass form the chunks launch)
    if (ctx->timing && !ctx->loop_ev0[0])
        for (int i = 0; i < kLoopMaxPasses; ++i) { SRL_CUDA(ctx, ctx->loop_ev0[i].create()); SRL_CUDA(ctx, ctx->loop_ev1[i].create()); }
    // the persistent ESIKF block first (side stream): it is resident before any pass kernel can wait for it
    SRL_CUDA(ctx, launch_iekf_loop(la, ctx->loop_stream));
    ctx->launches += 1;
    const bool pdl = !ctx->timing;   // programmatic dependent launch, except between the events that bracket each pass in timing mode
    for (int p = 0; p < la.n_pass; ++p) {
        PassArgs ap = a;
        ap.link.dev = ctx->d_iekf; ap.link.pose_ticket = la.base + (unsigned long long)p; ap.link.end_ticket = la.base + 63ull;
        ap.link.wait_pose = p ? 1 : 0;                               // pass 0: pose by value
        if (ctx->timing) cudaEventRecord(ctx->loop_ev0[p], ctx->stream);
        if (!capped) {
            rc = launch_pass(ctx, sw, ap, false, pdl);
        } else {
            for (size_t j = 0; rc == SRL_OK && j + 1 < bounds.size(); ++j)
                rc = launch_cap_chunk(ctx, sw, ap, bounds, j, (int)prm->max_num_residuals, false, pdl);
        }
        if (rc != SRL_OK) return iekf_loop_abort(ctx, rc);
        if (ctx->timing) cudaEventRecord(ctx->loop_ev1[p], ctx->stream);
    }
    return iekf_loop_finish(ctx, la, ctx->timing, eskf, frame_q, frame_t, summary);
}

int srl_iekf_replay(srl_ctx* ctx, srl_eskf_state* eskf, double frame_q[4], double frame_t[3], const srl_icp_params* prm,
                    const double* sums, int32_t n_blocks, int64_t first_delay_cycles, srl_iekf_summary* summary) {
    if (!ctx) return SRL_BAD_ARG;
    if (!eskf || !frame_q || !frame_t || !prm || !sums) return set_err(ctx, SRL_BAD_ARG, "srl_iekf_replay: null argument");
    if (n_blocks < 1 || n_blocks > kLoopMaxPasses) return set_err(ctx, SRL_BAD_ARG, "srl_iekf_replay: n_blocks outside [1, 40]");
    if (first_delay_cycles > (1ll << 32)) return set_err(ctx, SRL_BAD_ARG, "srl_iekf_replay: first_delay_cycles > 2^32");
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!device_loop_usable(ctx))
        return set_err(ctx, SRL_CUDA_ERROR, "srl_iekf_replay needs the device-resident loop (option device_loop = 0, or kernels are serialised)");
    PassConst none;
    std::memset(&none, 0, sizeof(none));
    IekfLoopArgs la;
    int rc;
    if ((rc = iekf_loop_args(ctx, eskf, frame_q, frame_t, none, prm, 1, la)) != SRL_OK) return rc;
    if (n_blocks < la.n_pass) return set_err(ctx, SRL_BAD_ARG, "srl_iekf_replay: fewer blocks of sums than the loop has passes");
    // everything the feeders need exists before the persistent block spins: buffer, copy, the feeder kernel's module
    if ((rc = ensure_scratch(ctx, (size_t)n_blocks * 32 * sizeof(double))) != SRL_OK) return rc;
    double* d_sums = static_cast<double*>(ctx->d_scratch.get());
    SRL_CUDA(ctx, cudaMemcpyAsync(d_sums, sums, (size_t)n_blocks * 32 * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    SRL_CUDA(ctx, preload_iekf_feed());
    IekfFeedArgs f;
    std::memset(&f, 0, sizeof(f));
    f.link.dev = ctx->d_iekf; f.link.end_ticket = la.base + 63ull; f.c = none;
    const int first_after = first_delay_cycles < 0 ? 1 : 0;
    if (first_delay_cycles < 0) {   // pass 0's sums are there before the loop starts: it skips its warm-up step
        f.sums = d_sums; f.link.pose_ticket = la.base; f.link.wait_pose = 0;
        SRL_CUDA(ctx, launch_iekf_feed(f, ctx->stream));
        SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        ctx->launches += 1;
    }
    SRL_CUDA(ctx, launch_iekf_loop(la, ctx->loop_stream));
    ctx->launches += 1;
    for (int p = first_after; p < la.n_pass; ++p) {
        f.sums = d_sums + (size_t)p * 32;
        f.link.pose_ticket = la.base + (unsigned long long)p;
        f.link.wait_pose = p ? 1 : 0;
        f.delay_cycles = p == 0 ? first_delay_cycles : 0;
        const cudaError_t e = launch_iekf_feed(f, ctx->stream);
        if (e != cudaSuccess) return iekf_loop_abort(ctx, cuda_fail(ctx, e, "launch_iekf_feed"));
        ctx->launches += 1;
    }
    return iekf_loop_finish(ctx, la, false, eskf, frame_q, frame_t, summary);
}

// The host-driven loop: one pass at a time, srl_iekf_step on the host between them.
static int update_iekf_host(srl_ctx* ctx, srl_comm* comm, srl_map* map, srl_sweep* sw, srl_eskf_state* eskf, double frame_q[4],
                            double frame_t[3], const double t_last[3], const double R_il[9], const double t_il[3],
                            const srl_icp_params* prm, srl_iekf_summary* summary) {
    srl_iekf_iter it;
    int rc = srl_iekf_begin(eskf, prm, &it);
    if (rc != SRL_OK) return rc;
    if (summary) { std::memset(summary, 0, sizeof(*summary)); summary->success = 1; }
    for (int passes = 1;; ++passes) {
        const srl_frame fr = make_frame(frame_q, frame_t, t_last, R_il, t_il);
        srl_normal_eq ne{};
        rc = run_pass(ctx, comm, map, sw, &fr, prm, &ne, nullptr);                   // src/optimize.cpp:153
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
        if (done) { if (summary) summary->converged = (done == 2); return SRL_OK; }
    }
}

// updateIEKF (src/optimize.cpp:133-314) on one GPU or, with `comm`, on this rank's shard of a sweep: the device-resident
// loop where it is usable, the host-driven loop otherwise.
static int update_iekf(srl_ctx* ctx, srl_comm* comm, srl_map* map, srl_sweep* sw, srl_eskf_state* eskf, double frame_q[4],
                       double frame_t[3], const double t_last[3], const double R_il[9], const double t_il[3],
                       const srl_icp_params* prm, srl_iekf_summary* summary) {
    if (!ctx || !eskf || !frame_q || !frame_t || !t_last || !R_il || !t_il || !prm) return SRL_BAD_ARG;
    if (comm && (comm->ctx != ctx || !comm->connected)) return set_err(ctx, SRL_COMM_ERROR, "srl_comm is not connected");
    if (map && check_lio_map(ctx, map) != SRL_OK) return SRL_BAD_ARG;
    ctx->cap_chunks_run = 0; ctx->cap_chunks_on_device = false;
    const Cap cap = map && sw ? cap_mode(ctx, prm, sw, comm) : Cap::none;   // (the pass reports a null map or sweep)
    if (cap == Cap::rejected) return SRL_BAD_ARG;
    // an empty capped sweep takes the host loop: its pass sums to zero without launching anything
    if (map && sw && device_loop_usable(ctx) && (cap == Cap::none || sw->n > 0))
        return update_iekf_device(ctx, comm, map, sw, eskf, frame_q, frame_t, t_last, R_il, t_il, prm, cap == Cap::capped, summary);
    return update_iekf_host(ctx, comm, map, sw, eskf, frame_q, frame_t, t_last, R_il, t_il, prm, summary);
}

int srl_update_iekf(srl_ctx* ctx, srl_map* map, srl_sweep* sw, srl_eskf_state* eskf, double frame_q[4], double frame_t[3],
                    const double t_last[3], const double R_il[9], const double t_il[3], const srl_icp_params* prm,
                    srl_iekf_summary* summary) {
    return update_iekf(ctx, nullptr, map, sw, eskf, frame_q, frame_t, t_last, R_il, t_il, prm, summary);
}

// ---- multi-GPU -------------------------------------------------------------------------------------------------
int srl_comm_create(srl_ctx* ctx, int rank, int world, srl_comm** out) {
    if (!ctx || !out || world < 1 || world > kMaxRanks || rank < 0 || rank >= world) return SRL_BAD_ARG;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    std::unique_ptr<srl_comm> c(new srl_comm());
    c->ctx = ctx; c->device = ctx->device; c->rank = rank; c->world = world;
    SRL_CUDA(ctx, c->d_mail.alloc(1));
    SRL_CUDA(ctx, cudaMemset(c->d_mail, 0, sizeof(Mailbox)));
    SRL_CUDA(ctx, c->d_seq.alloc(1));
    SRL_CUDA(ctx, cudaMemset(c->d_seq, 0, sizeof(unsigned long long)));
    c->peer[rank] = c->d_mail;
    c->connected = (world == 1);
    *out = c.release();
    return SRL_OK;
}
void srl_comm_destroy(srl_comm* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();   // the ctx's passes that exchange through the mailboxes have finished
    for (int r = 0; r < c->world; ++r) if (c->opened[r]) cudaIpcCloseMemHandle(c->peer[r]);
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
    if (!comm) return SRL_BAD_ARG;
    return update_iekf(ctx, comm, map, sw, eskf, frame_q, frame_t, t_last, R_il, t_il, prm, summary);
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

// optimize() from host buffers (src/optimize.cpp:428-448) on the keypoints [b, e) of raw_xyz: H2D of those keypoints, the
// iterated update, the final re-transform and D2H into world_xyz_out[b, e).
static int optimize_host(srl_ctx* ctx, srl_comm* comm, srl_map* map, srl_sweep* sw, const double* raw_xyz, size_t b, size_t e,
                         srl_eskf_state* eskf, double frame_q[4], double frame_t[3], const double t_last[3], const double R_il[9],
                         const double t_il[3], const srl_icp_params* prm, srl_iekf_summary* summary, double* world_xyz_out) {
    if (map && check_lio_map(ctx, map) != SRL_OK) return SRL_BAD_ARG;
    int rc = srl_sweep_upload(sw, raw_xyz + 3 * b, e - b);
    if (rc != SRL_OK) return rc;
    rc = update_iekf(ctx, comm, map, sw, eskf, frame_q, frame_t, t_last, R_il, t_il, prm, summary);   // src/optimize.cpp:435
    if (rc != SRL_OK) return rc;                                                 // :437-439
    if (world_xyz_out && e > b) {                                                // :441-445
        if ((rc = ensure_scratch(ctx, (e - b) * 3 * sizeof(double))) != SRL_OK) return rc;
        rc = srl_sweep_transform_device(ctx, sw, frame_q, frame_t, R_il, t_il, static_cast<double*>(ctx->d_scratch.get()));
        if (rc != SRL_OK) return rc;
        SRL_CUDA(ctx, cudaMemcpyAsync(world_xyz_out + 3 * b, ctx->d_scratch, (e - b) * 3 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    return SRL_OK;
}

int srl_optimize_host(srl_ctx* ctx, srl_map* map, srl_sweep* sw, const double* raw_xyz, size_t n, srl_eskf_state* eskf,
                      double frame_q[4], double frame_t[3], const double t_last[3], const double R_il[9], const double t_il[3],
                      const srl_icp_params* prm, srl_iekf_summary* summary, double* world_xyz_out) {
    if (!ctx || !sw) return SRL_BAD_ARG;
    return optimize_host(ctx, nullptr, map, sw, raw_xyz, 0, n, eskf, frame_q, frame_t, t_last, R_il, t_il, prm, summary, world_xyz_out);
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
    // of every pass are exchanged inside the pass, so every rank ends with the same state
    return optimize_host(ctx, comm, map, sw, raw_xyz, b, e, eskf, frame_q, frame_t, t_last, R_il, t_il, prm, summary, world_xyz_out);
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
