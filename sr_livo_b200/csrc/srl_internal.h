// srl_internal.h — internal declarations shared by the .cu/.cpp translation units of libsrlivo_b200.so
#pragma once

#include <cuda_runtime.h>
#include <math_constants.h>

#include <cstdint>
#include <string>
#include <vector>

#include "../../include/srlivo_b200.h"
#include "srl_device.cuh"
#include "srl_math.cuh"

namespace srl {

constexpr int kK1Warps = 8;
constexpr int kK1Threads = kK1Warps * 32;

constexpr int kMaxRanks = 8;
// One mailbox per rank (device memory, exported over CUDA IPC): peers write their 32 sums of a pass into
// data[parity][their rank] and then set flag[parity][their rank] = pass sequence number.
struct Mailbox {
    double data[2][kMaxRanks][32];
    unsigned long long flag[2][kMaxRanks];
};
struct CommDev {              // by-value kernel argument; world <= 1 disables the exchange
    int world, rank;
    unsigned long long* seq;  // device counter of the exchanges this rank has run (same on every rank: all ranks run the
                              // same passes); the exchange of a pass uses *seq + 1 and stores it back.  Kept on the device
                              // because the device-resident loop skips enqueued passes the host cannot know about.
    Mailbox* mail[kMaxRanks]; // mail[r] = rank r's mailbox as mapped in THIS process (mail[rank] is local memory)
};

// ---- device-resident updateIEKF loop (srl_iekf.cu, row N1) ------------------------------------------------------
// One persistent 128-thread block per sweep (k_iekf_loop, on the ctx's side stream) runs the ESIKF algebra of every
// pass; the pass kernels on the main stream and that block hand data to each other through HBM and three tickets:
//   alive_seq : set by the block when it starts (diagnostics: the block is launched before any pass kernel that waits for it)
//   sums_seq  : ticket + 1 once the sums of the pass with that ticket are in `sums` (written by the pass's last block)
//   pose_seq  : >= ticket once the constants of the pass with that ticket are in `pc` (written by the ESIKF block); the
//               block stores a ticket beyond every pass of the sweep when the loop has ended (`done`)
// ticket = base + pass number; base grows by 64 per sweep, so tickets never repeat and nothing has to be reset.
constexpr int kLoopMaxPasses = 40;
struct IekfDev {              // one per ctx, in HBM
    PassConst pc;             // constants of the NEXT pass: the ESIKF block rewrites Rn, Rq, t after every observe()
    unsigned long long alive_seq, sums_seq, pose_seq;
    int done;                 // != 0: the loop has ended (break :309 / return :155); kernels still enqueued leave at once
    int status;               // srl_status of the loop
    int pass_index;           // i of the next step, starts at -1 (src/optimize.cpp:147)
    int max_iter;
    int passes_run, converged, num_residuals_used, frame_id;
    int min_neighbors;
    int abort;                // set by k_iekf_abort when the host could not enqueue a pass: the block stops waiting and ends the loop
    double laser_cov, thr_t, thr_r;
    double sums[32];          // the (all-reduced) sums of the pass in flight
    srl_eskf_state cur, predict;   // eskf_pro now / the snapshot of :138-143
    double frame_q[4], frame_t[3]; // p_frame->p_state (:255-256)
    double trace[32][24];
    long long step_cycles[kLoopMaxPasses];   // clock64 ticks from "sums seen" to "pose published" per pass (tuning)
    long long stage_cycles[8];               // ... and to the stages inside the last step
};
struct IekfInit {             // by-value argument of the loop kernel (whole argument block < 4 KB)
    srl_eskf_state eskf;
    double frame_q[4], frame_t[3];
    PassConst pc0;            // pass 0 constants (also given by value to pass 0's kernels)
    double laser_cov, thr_t, thr_r;
    int max_iter, frame_id, min_neighbors, pad0;
};
struct IekfHostOut {          // mapped pinned host memory: what the loop hands back, then the sequence flag
    srl_eskf_state eskf;
    double frame_q[4], frame_t[3];
    double sums[32];          // the last pass's (all-reduced) sums
    int status, passes_run, num_residuals_used, converged;
    double trace[32][24];
    long long step_cycles[kLoopMaxPasses];
    long long stage_cycles[8];
    unsigned long long seq;
};
struct IekfLoopArgs {
    IekfDev* dev;
    IekfHostOut* host_out;    // device-side address of the mapped buffer
    unsigned long long host_seq;
    unsigned long long base;  // ticket of this sweep's pass 0
    int world, n_pass;
    IekfInit init;
};
cudaError_t launch_iekf_loop(const IekfLoopArgs& a, cudaStream_t stream);
cudaError_t launch_iekf_abort(IekfDev* dev, cudaStream_t stream);
cudaError_t probe_concurrent_kernels(cudaStream_t side, cudaStream_t main_stream, int* d_two_ints, bool* concurrent);

#if defined(__CUDACC__)
// Message passing between kernels / GPUs / the host: payload stores, then a RELEASE store of the ticket; the reader polls
// the ticket (relaxed) and ends with one ACQUIRE load.  __threadfence() is fence.sc (MEMBAR.SC + an L1 invalidate) executed
// by every calling thread; the release store is one MEMBAR.ALL by one thread, the acquire load only invalidates L1 — and
// the release is cumulative over the stores of the threads that reached it through __syncthreads() / __syncwarp().
__device__ __forceinline__ void st_release_gpu(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.gpu.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.sys.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_gpu(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.gpu.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long ld_relaxed_gpu(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long ld_relaxed_sys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.sys.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void fence_acq_rel_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }

// Fused exchange over NVLink peer memory (one warp): publish this rank's 32 sums into every rank's mailbox, wait for the
// others' sums of the same pass, add all of them in rank order (bitwise identical everywhere).  NaN marks a failed exchange.
__device__ __forceinline__ double comm_exchange(const CommDev& cm, double tot, int lane) {
    const unsigned long long seq = *reinterpret_cast<volatile unsigned long long*>(cm.seq) + 1ull;
    __syncwarp();
    if (lane == 0) *reinterpret_cast<volatile unsigned long long*>(cm.seq) = seq;
    const int par = (int)(seq & 1ull);
    for (int p = 0; p < cm.world; ++p) cm.mail[p]->data[par][cm.rank][lane] = tot;
    __syncwarp();
    if (lane < cm.world) st_release_sys(&cm.mail[lane]->flag[par][cm.rank], seq);   // covers the warp's 32 stores to that peer
    bool ok = true;
    if (lane < cm.world) {
        const unsigned long long* f = &cm.mail[cm.rank]->flag[par][lane];
        long long spins = 0;
        while (ld_relaxed_sys(f) < seq) { if (++spins > (1ll << 27)) { ok = false; break; } }   // a peer died: give up, do not hang
        (void)ld_acquire_sys(f);
    }
    ok = __all_sync(0xffffffffu, ok);
    double sum = 0.0;
    for (int r = 0; r < cm.world; ++r) {
        const volatile double* d = &cm.mail[cm.rank]->data[par][r][lane];
        sum += *d;
    }
    return ok ? sum : __longlong_as_double(0x7ff8000000000000ll);
}
#endif

struct K1Args {
    PassConst c;
    const Slot* slots;
    unsigned int mask;
    const float* blocks;
    const double* raw;        // sweep, n*3 (device)
    long long k_begin, k_end; // this rank's shard
    double* partials;         // [grid][32]
    unsigned int* ticket;
    double* out32;            // device, 32 doubles
    double* rows;             // optional n*8 (J6, h, d^2)
    int* status;              // optional n
    double* dbg_world;        // optional debug outputs (device)
    short* dbg_nbr;
    double* dbg_nbr_dist;
    double* dbg_plane;
    const unsigned char* only_flagged;   // optional: process only keypoints whose flag is set (k1_fast's ambiguous ones)
    const double* prev_out32;            // optional: 32 doubles added to the final sums
    unsigned long long* stats;   // optional device counters: [0] keypoints that took the exact-selection fallback
    float eps_scale;             // 1 normally; +inf forces the exact selection for every keypoint (tests)
    CommDev comm;                // multi-GPU: the last block exchanges the 32 sums with the peers over NVLink
    double* host_out;            // optional mapped pinned host buffer: the final 32 sums are also written there, then
    unsigned long long host_seq; // host_out[32] (as u64) = host_seq after a system fence: the host spins on it instead of
                                 // a D2H copy + stream synchronize
    IekfDev* dev;                // device-resident loop: the pass's last block leaves its sums in dev->sums and bumps sums_seq;
    unsigned long long pose_ticket;   // with wait_pose the kernel first waits for pose_seq >= pose_ticket and takes its constants from
    unsigned long long end_ticket;   // dev->pc; pose_seq >= end_ticket says the loop has ended: the kernel leaves at once
    int wait_pose;
};

constexpr int kFastWarps = 4;
constexpr int kFastThreads = kFastWarps * 32;

struct FastArgs {               // k1_fast (srl_fast.cu)
    PassConst c;
    const Slot* slots;
    unsigned int mask;
    const float* blocks;
    const double* raw;          // sweep, n*3 (device)
    const unsigned* order;      // sorted position -> keypoint index (nullptr: identity)
    long long s_begin, s_end;   // this rank's range of sorted positions
    double* partials;
    unsigned int* ticket;
    double* out32;
    unsigned char* flags;       // per keypoint: 1 = ambiguous, redo with k1_assoc's exact selection
    int* status;
    double* dbg_world;
    short* dbg_nbr;
    double* dbg_nbr_dist;
    double* dbg_plane;
    unsigned long long* stats;  // [1] += ambiguous keypoints
    int force_amb_mod;          // test knob: > 0 flags every keypoint whose index is a multiple of it
    // split form (k1_scan -> k1_fit): per sorted position, the NS boundary-inclusive candidates of the keypoint
    unsigned* cand_rows;        // one 96-byte row per sorted position: 23 x u32 (block * 20 + index in block) + header word
                                // (byte 0: 0 = < K candidates, K..NS = candidates inside the window, 255 = ambiguous;
                                //  byte 1: slots certainly among the K nearest; byte 2: slots that can be the nearest)
    unsigned long long* scan_count;   // candidates visited by k1_scan, folded into component 30 by k1_fit's last block
    double* host_out;                 // optional: mapped host buffer; k1_fit publishes the final sums there when no keypoint
    unsigned long long host_seq;      // was flagged in this pass (see K1Args::host_out)
    CommDev comm;                     // multi-GPU with exchange_in_fit: k1_fit's last block runs the exchange in that case
    int exchange_in_fit;
    IekfDev* dev;                     // device-resident loop (see K1Args::dev)
    unsigned long long pose_ticket, end_ticket;
    int wait_pose;
    double* rows;                     // optional n*8 per-keypoint rows (J6, h, d^2) for the ordered residual cap (k2_cap_reduce)
    unsigned int* chunk_tickets;      // k1_fit's two-level grid reduction: one ticket and one 32-double sum per chunk of 32 blocks
    double* chunk_sums;
};

#if defined(__CUDACC__)
// Programmatic dependent launch (sm_90+): the pass kernels of a sweep are launched with the programmatic-stream-
// serialization attribute; each lets its successor become resident at once (trigger) and waits for its predecessor's
// completion and memory flush before touching anything (wait) — stream order with the launch latency hidden.  Both are
// no-ops for a kernel launched without the attribute.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
// Every pass kernel reads its constants from shared memory: filled from the by-value argument (host-driven pass, pass 0
// of the device-resident loop) or from the loop state once the ESIKF block has published them.  Returns false when the
// loop has already ended (the whole grid leaves).
__device__ __forceinline__ bool load_pass_const(const IekfDev* dev, int wait_pose, unsigned long long ticket, unsigned long long end_ticket,
                                                const PassConst& by_value, PassConst& s_c) {
    constexpr int ND = (int)(sizeof(PassConst) / sizeof(double));
    static_assert(sizeof(PassConst) % sizeof(double) == 0, "PassConst is copied as doubles");
    pdl_trigger();
    pdl_wait();
    if (dev && wait_pose) {
        __shared__ int s_go;
        if (threadIdx.x == 0) {
            const unsigned long long* ps = &dev->pose_seq;
            long long spins = 0;
            unsigned long long v;
            while ((v = ld_relaxed_gpu(ps)) < ticket) { if (++spins > (1ll << 26)) { v = ~0ull; break; } }   // the ESIKF block died: leave, do not hang
            if (v != ~0ull) v = ld_acquire_gpu(ps);
            s_go = v < end_ticket ? 1 : 0;   // a ticket beyond the sweep's passes = the loop has ended (also a later sweep's)
        }
        __syncthreads();
        if (!s_go) return false;
        if (threadIdx.x < ND) reinterpret_cast<double*>(&s_c)[threadIdx.x] = __ldcg(reinterpret_cast<const double*>(&dev->pc) + threadIdx.x);
    } else if (threadIdx.x < ND) {   // by value: the kernel argument is __grid_constant__, so it can be indexed like memory (a
        // copy by thread 0 alone kept every warp of the block at the barrier below for ~10 % of k1_fit's duration)
        reinterpret_cast<double*>(&s_c)[threadIdx.x] = reinterpret_cast<const double*>(&by_value)[threadIdx.x];
    }
    __syncthreads();
    return true;
}
// the pass's last block (one warp) hands the final sums to the ESIKF block
__device__ __forceinline__ void publish_sums_to_loop(IekfDev* dev, unsigned long long ticket, double tot, int lane) {
    if (!dev) return;
    dev->sums[lane] = tot;
    __syncwarp();
    if (lane == 0) st_release_gpu(&dev->sums_seq, ticket + 1ull);
}
#endif

cudaError_t launch_k1_fast(const FastArgs& a, int grid, bool debug, int device, cudaStream_t stream);
// load every pass kernel (CUDA loads lazily at first launch, and a load waits for running kernels) and the offset tables;
// *max_local is raised to the largest per-thread local memory (spill frame) of the kernels loaded
cudaError_t preload_fast_kernels(int device, size_t* max_local);
cudaError_t preload_assoc_kernels(int device, int K, size_t* max_local);
constexpr int kSplitSlots = 23;   // = NS of srl_fast.cu: candidate slots k1_scan hands to k1_fit per keypoint
cudaError_t launch_k1_split(const FastArgs& a, long long n, int max_grid, bool debug, int device, cudaStream_t stream, bool pdl);
// <<<>>> with the programmatic-stream-serialization attribute when pdl is set
template <typename Args>
inline cudaError_t launch_pass_kernel(void (*fn)(const Args), const Args& a, unsigned grid, unsigned block, size_t smem, cudaStream_t stream, bool pdl) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(block); cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, fn, a);
}
void k1_split_set_lanes_per_keypoint(int v);
int k1_fast_max_blocks_per_sm();
void k1_fast_set_min_blocks(int v);
void k1_fast_set_lanes_per_keypoint(int v);
int k1_fast_lanes_per_keypoint();
cudaError_t sweep_compute_order(const double* d_raw, long long n, unsigned* d_order, void* scratch, size_t scratch_bytes,
                                size_t* needed, cudaStream_t stream);
void sweep_order_set_impl(int v);   // 1: the single-launch cluster sort (verified against the CUB order at first use), 0: CUB
int sweep_order_impl();             // -1 cluster kernel not verified yet, 1 verified and in use, 0 CUB

size_t k1_smem_bytes(int K);
int k1_max_blocks_per_sm(int K, int nb);
void k1_set_min_blocks(int v);
cudaError_t launch_k1(const K1Args& a, int grid, bool debug, int device, cudaStream_t stream, bool pdl = false);
cudaError_t launch_k2(const double* rows, int* status, long long k_begin, long long k_end, int cap, long long* state,
                      double* out32, int mark_unvisited, cudaStream_t stream);
cudaError_t launch_transform(const double* raw, long long n, const PassConst& c, double* out, cudaStream_t stream);

// host-side pass constants from the reference's per-pass inputs (src/optimize.cpp:21-28,55-61)
void make_pass_const(const srl_frame& f, const srl_icp_params& p, PassConst& c);

}  // namespace srl

// ---- opaque handle definitions ------------------------------------------------------------------
struct srl_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    int sm_count = 132;
    std::string err;
    int64_t launches = 0;
    // optional CUDA-event timing of k1_assoc
    bool timing = false;
    cudaEvent_t ev0[2] = {nullptr, nullptr}, ev1[2] = {nullptr, nullptr};   // two pairs: the pass in flight and the one before
    bool ev_pending[2] = {false, false};
    int ev_cur = 0;
    double k1_ms = 0.0;
    int64_t k1_launches = 0;
    // per-pass scratch
    double* d_partials = nullptr;   // [max_grid][32]
    int max_grid = 0;
    unsigned int* d_ticket = nullptr;
    unsigned int* d_chunk_tickets = nullptr;   // [max_grid / 32 + 1], zero between passes
    double* d_chunk_sums = nullptr;            // [max_grid / 32 + 1][32]
    double* d_out32 = nullptr;
    double* h_out32 = nullptr;      // pinned + mapped: [0,32) sums, [32] sequence flag written by the pass's last kernel, [33..64) scratch
    double* d_h_out32 = nullptr;    // device-side address of h_out32
    unsigned long long host_seq = 0;
    bool exchange_in_fit = true;    // option "exchange_in_fit" / SRL_EXCHANGE_IN_FIT: multi-GPU, k1_fit runs the exchange when it flagged nothing
    bool mapped_result = true;      // option "mapped_result": read a pass's sums through the mapped buffer (default) or by memcpy + sync
    long long* d_k2_state = nullptr;
    unsigned long long* d_stats = nullptr;   // 4 counters
    double* d_fast_out = nullptr;            // k1_fast's 32 sums, added by the exact-fallback launch
    bool force_exact = false;
    int force_amb_mod = 0;                   // test knob for the k1_fast -> k1_assoc hand-over
    int variant = 0;                         // 0 auto, 1 = k1_fast, 2 = k1_assoc only, 3 = k1_scan + k1_fit (1 and 3 with the exact fallback)
    unsigned long long* d_scan_count = nullptr;
    // device-resident updateIEKF loop (row N1)
    bool kernels_preloaded = false;
    bool pdl = true;                         // option "pdl" / SRL_PDL: programmatic dependent launch of the pass kernels
    bool eager_order = true;                 // option "eager_order": Morton-order a sweep right behind its upload (default) or at its first pass
    int concurrent_kernels = -1;             // -1 not probed yet; 0: kernels of this process are serialised (profiler): host loop
    bool device_loop = true;                 // option "device_loop" / SRL_DEVICE_LOOP: 0 = the host-driven loop of round 1
    srl::IekfDev* d_iekf = nullptr;
    srl::IekfHostOut* h_iekf = nullptr;      // pinned + mapped
    srl::IekfHostOut* d_h_iekf = nullptr;    // its device-side address
    unsigned long long iekf_seq = 0;
    unsigned long long loop_base = 64;       // ticket of the next sweep's pass 0 (grows by 64 per sweep)
    cudaStream_t loop_stream = nullptr;      // side stream of the persistent ESIKF block
    double step_cycles_sum = 0.0;            // counter "iekf_step_cycles_avg": clock ticks from "sums seen" to "pose published"
    long long step_cycles_n = 0;
    cudaEvent_t loop_ev0[srl::kLoopMaxPasses] = {nullptr}, loop_ev1[srl::kLoopMaxPasses] = {nullptr};   // timing mode: one pair per enqueued pass
    // generic scratch (map insert)
    void* d_scratch = nullptr;
    size_t scratch_bytes = 0;
    void* h_pinned = nullptr;
    size_t pinned_bytes = 0;
};

struct srl_map {
    srl_ctx* ctx = nullptr;
    double voxel_size = 1.0;
    int cap = 20;
    size_t max_voxels = 0;
    size_t capacity = 0;            // slots (power of two)
    srl::Slot* d_slots = nullptr;
    float* d_blocks = nullptr;
    int64_t n_voxels = 0;           // host mirror of the block count
    long long* d_counters = nullptr;   // [0] n_points, [1] scratch
};

struct srl_comm {
    srl_ctx* ctx = nullptr;
    int rank = 0, world = 1;
    unsigned long long* d_seq = nullptr;            // device counter of the exchanges run (CommDev::seq)
    srl::Mailbox* d_mail = nullptr;                 // this rank's mailbox
    srl::Mailbox* peer[srl::kMaxRanks] = {nullptr}; // mapped peers (peer[rank] == d_mail)
    bool opened[srl::kMaxRanks] = {false};
    bool connected = false;
};

struct srl_sweep {
    srl_ctx* ctx = nullptr;
    size_t capacity = 0;
    size_t n = 0;
    size_t shard_begin = 0, shard_end = 0;
    double* d_raw = nullptr;        // capacity*3
    unsigned* d_order = nullptr;    // capacity: Morton order of the keypoints (lazily computed per upload)
    bool order_valid = false;
    bool flags_clean = false;       // d_flags holds zeros outside the range the current shard rewrites every pass
    unsigned char* d_flags = nullptr;   // capacity
    unsigned* d_cand_rows = nullptr;    // split form: 24 words per keypoint (k1_scan -> k1_fit)
    double* d_rows = nullptr;       // capacity*8, lazily allocated (cap mode)
    int* d_status = nullptr;        // capacity, lazily allocated
    // debug buffers, lazily allocated
    double* d_dbg_world = nullptr;
    short* d_dbg_nbr = nullptr;
    double* d_dbg_nbr_dist = nullptr;
    double* d_dbg_plane = nullptr;
    int dbg_K = 0;
};

namespace srl {
int set_err(srl_ctx* ctx, int code, const std::string& msg);
int cuda_fail(srl_ctx* ctx, cudaError_t e, const char* where);
int ensure_scratch(srl_ctx* ctx, size_t bytes);
int ensure_pinned(srl_ctx* ctx, size_t bytes);
void timing_collect(srl_ctx* ctx);
}  // namespace srl

#define SRL_CUDA(ctx, call)                                             \
    do {                                                                \
        cudaError_t e__ = (call);                                       \
        if (e__ != cudaSuccess) return srl::cuda_fail((ctx), e__, #call); \
    } while (0)
