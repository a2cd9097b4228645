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
// How a pass kernel is tied to the device-resident loop (dev == nullptr: a host-driven pass).  The pass's last block leaves
// its sums in dev->sums and bumps sums_seq to pose_ticket + 1.
struct PassLink {
    IekfDev* dev;
    unsigned long long pose_ticket;   // with wait_pose the kernel first waits for pose_seq >= pose_ticket and takes its constants from
    unsigned long long end_ticket;    // dev->pc; pose_seq >= end_ticket says the loop has ended: the kernel leaves at once
    int wait_pose;
    const long long* cap_state;  // chunk j >= 1 of a capped pass: k2_cap_reduce's state; the grid leaves when k* is already found
};
struct IekfFeedArgs {         // srl_iekf_replay: a one-warp stand-in for pass `link.pose_ticket - base` (k_iekf_feed)
    PassLink link;
    const double* sums;       // device, the 32 sums this pass hands to the loop
    long long delay_cycles;   // > 0: spin this many SM clock ticks before publishing
    PassConst c;              // by-value constants of load_pass_const (unused)
};
cudaError_t preload_iekf_feed();
cudaError_t launch_iekf_feed(const IekfFeedArgs& a, cudaStream_t stream);
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

// ---- arguments of the pass kernels ------------------------------------------------------------------------------
struct PassSink {             // where a pass's final 32 sums go (finalise_pass)
    double* out32;            // device, 32 doubles
    double* host_out;            // optional mapped pinned host buffer: the sums are also written there, then host_out[32] (as u64) =
    unsigned long long host_seq; // host_seq with a system-scope release: the host spins on it instead of a D2H copy + synchronize
    CommDev comm;             // multi-GPU: the sums are first exchanged with the peers over NVLink
};
struct KeypointOut {          // optional per-keypoint outputs (device)
    int* status;              // n
    double* rows;             // n*8 (J6, h, d^2) for the ordered residual cap (k2_cap_reduce), in keypoint order
    double* dbg_world;
    short* dbg_nbr;
    double* dbg_nbr_dist;
    double* dbg_plane;
};
struct PassStats {            // one per ctx, in HBM, zero between passes except the two counters
    unsigned long long exact_fallbacks;   // counter: keypoints that took k1_assoc's exact selection
    unsigned long long fast_ambiguous;    // counter: keypoints k1_fast / k1_scan flagged as ambiguous
    unsigned long long flagged;     // keypoints flagged in the pass in flight; the fallback launch's last block resets it
    unsigned long long finalised;   // k1_fit finalised the pass in flight (nothing was flagged); the fallback launch, which then
                                    // only forwards the sums, resets it
    int probe[2];                   // scratch of probe_concurrent_kernels
};

struct PassArgs {             // k1_scan, k1_fit, k1_fast and k1_assoc
    PassConst c;
    MapView map;
    const double* raw;        // sweep, n*3 (device)
    long long k_begin, k_end; // this rank's range: of sorted positions when `order` is set, of keypoint indices otherwise
    double* partials;         // [grid][32]
    unsigned int* ticket;
    PassSink sink;
    KeypointOut out;
    PassStats* stats;
    PassLink link;
    // fast and split forms (k1_fast, k1_scan -> k1_fit)
    const unsigned* order;    // sorted position -> keypoint index (nullptr: identity)
    unsigned char* flags;     // per keypoint: 1 = ambiguous, redo with k1_assoc's exact selection
    int force_amb_mod;        // test knob: > 0 flags every keypoint whose index is a multiple of it
    unsigned* cand_rows;      // k1_scan -> k1_fit, one 96-byte row per sorted position: 23 x u32 (block * 20 + index in block) +
                              // header word (byte 0: 0 = < K candidates, K..NS = candidates inside the window, 255 = ambiguous;
                              //  byte 1: slots certainly among the K nearest; byte 2: slots that can be the nearest)
    unsigned long long* scan_count;   // candidates visited by k1_scan, folded into component 30 by k1_fit's last block
    unsigned int* chunk_tickets;      // k1_fit's two-level grid reduction: one ticket and one 32-double sum per chunk of 32 blocks
    double* chunk_sums;
    // k1_assoc
    const unsigned char* only_flagged;   // fallback launch: process only keypoints whose flag is set
    const double* prev_out32;            // fallback launch: the first launch's 32 sums, added to the final sums
    float eps_scale;             // 1 normally; +inf forces the exact selection for every keypoint (tests)
};
static_assert(sizeof(PassArgs) <= 1024, "the pass kernels' argument block stays far below the 4 KB kernel parameter space");

constexpr int kFastWarps = 4;
constexpr int kFastThreads = kFastWarps * 32;

struct K2Args {                 // k2_cap_reduce: one chunk of the ordered residual cap (srl_assoc.cu)
    const double* rows;         // n*8 per-keypoint rows (J6, h, d^2) written by the chunk's pass kernels
    int* status;                // n: 0 no full neighbourhood, 1 full, 2 accepted
    long long k_begin, k_end;   // the chunk
    int cap;
    int chunk;                  // index of the chunk in its pass: chunk 0 starts from a zero state, so nothing is reset between passes
    long long* state;           // [0] accepted so far, [1] k* found, [2] k*
    double* out32;              // the pass's capped sums: chunk 0 writes them, later chunks add to them
    int mark_unvisited;         // status -1 for the chunk's keypoints after k*
    int last;                   // the pass's last chunk: it publishes even when k* was not found
    const double* pass_out32;   // optional: the chunk's pass sums; their [30] (candidates scanned) is added to out32[30]
    unsigned long long* chunks_run;   // optional device counter of the chunks that did work
    PassLink link;              // device-resident loop: the chunk that finds k*, or the last one, publishes out32
};

#if defined(__CUDACC__)
// Programmatic dependent launch (sm_90+): the pass kernels of a sweep are launched with the programmatic-stream-
// serialization attribute; each lets its successor become resident at once (trigger) and waits for its predecessor's
// completion and memory flush before touching anything (wait) — stream order with the launch latency hidden.  Both are
// no-ops for a kernel launched without the attribute.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
// The ticket half of load_pass_const: lets the successor launch, waits for the predecessor, then (wait_pose) for the pose
// of pass `pose_ticket`.  Returns false when the loop has already ended (the whole grid leaves).
__device__ __forceinline__ bool wait_pass_ticket(const PassLink link) {
    pdl_trigger();
    pdl_wait();
    if (link.dev && link.wait_pose) {
        __shared__ int s_go;
        if (threadIdx.x == 0) {
            const unsigned long long* ps = &link.dev->pose_seq;
            long long spins = 0;
            unsigned long long v;
            while ((v = ld_relaxed_gpu(ps)) < link.pose_ticket) { if (++spins > (1ll << 26)) { v = ~0ull; break; } }   // the ESIKF block died: leave, do not hang
            if (v != ~0ull) v = ld_acquire_gpu(ps);
            s_go = v < link.end_ticket ? 1 : 0;   // a ticket beyond the sweep's passes = the loop has ended (also a later sweep's)
        }
        __syncthreads();
        if (!s_go) return false;
    }
    return true;
}
// Chunk j >= 1 of a capped pass (device-resident loop): k* was found by an earlier chunk's k2_cap_reduce, which completed
// before this kernel passed pdl_wait, so every thread reads the same word and the whole grid leaves together.
__device__ __forceinline__ bool cap_chunk_done(const PassLink& link) {
    return link.cap_state && __ldcg(link.cap_state + 1) != 0;
}
// Every pass kernel reads its constants from shared memory: filled from the by-value argument (host-driven pass, pass 0
// of the device-resident loop) or from the loop state once the ESIKF block has published them.  Returns false when the
// loop has already ended (the whole grid leaves).
__device__ __forceinline__ bool load_pass_const(const PassLink link, const PassConst& by_value, PassConst& s_c) {
    constexpr int ND = (int)(sizeof(PassConst) / sizeof(double));
    static_assert(sizeof(PassConst) % sizeof(double) == 0, "PassConst is copied as doubles");
    if (!wait_pass_ticket(link)) return false;
    if (link.dev && link.wait_pose) {
        if (threadIdx.x < ND) reinterpret_cast<double*>(&s_c)[threadIdx.x] = __ldcg(reinterpret_cast<const double*>(&link.dev->pc) + threadIdx.x);
    } else if (threadIdx.x < ND) {   // by value: the kernel argument is __grid_constant__, so it can be indexed like memory (a
        // copy by thread 0 alone kept every warp of the block at the barrier below for ~10 % of k1_fit's duration)
        reinterpret_cast<double*>(&s_c)[threadIdx.x] = reinterpret_cast<const double*>(&by_value)[threadIdx.x];
    }
    __syncthreads();
    return true;
}
// the pass's last block (one warp) hands the final sums to the ESIKF block
__device__ __forceinline__ void publish_sums_to_loop(const PassLink& link, double tot, int lane) {
    if (!link.dev) return;
    link.dev->sums[lane] = tot;
    __syncwarp();
    if (lane == 0) st_release_gpu(&link.dev->sums_seq, link.pose_ticket + 1ull);
}
// The pass's result straight into mapped pinned host memory (one warp): 32 sums, then the sequence word with a system-scope
// release.  The host spins on that word (srl_api.cu: wait_host_seq) — no D2H copy, no stream synchronize on the critical path.
__device__ __forceinline__ void publish_to_host(const PassSink& sink, double tot, int lane) {
    if (!sink.host_out) return;
    sink.host_out[lane] = tot;
    __syncwarp();
    if (lane == 0) st_release_sys(reinterpret_cast<unsigned long long*>(sink.host_out + 32), sink.host_seq);
}
// These are the pass's final sums: called by exactly one warp of the launch that holds them, `tot` in lane order.  Exchange
// with the peers, out32, the host, the ESIKF block.  `forward`: an earlier launch of the pass (k1_fit) has already run the
// exchange and handed the sums to the loop; this launch only writes the same values to out32 and to the host again.  A
// capped pass (rows set) is handed to the loop by k2_cap_reduce alone.  A pass is published either to the host
// (host-driven: link.dev is null) or to the loop, never both, so the order of those two steps decides nothing.
__device__ __forceinline__ void finalise_pass(const PassArgs& A, bool forward, double tot, int lane) {
    if (A.sink.comm.world > 1 && !forward) tot = comm_exchange(A.sink.comm, tot, lane);
    A.sink.out32[lane] = tot;
    publish_to_host(A.sink, tot, lane);
    if (!forward && !A.out.rows) publish_sums_to_loop(A.link, tot, lane);
}
#endif

#if defined(__CUDACC__)
__device__ __forceinline__ unsigned char sat_u8(double v) {       // cv::saturate_cast<uchar>(double): cvRound (half to even), clamp
    const long long r = __double2ll_rn(v);
    return (unsigned char)(r < 0 ? 0 : (r > 255 ? 255 : r));
}
__device__ __forceinline__ unsigned char sat_add_u8(unsigned char a, unsigned char b) { const int r = (int)a + (int)b; return (unsigned char)(r > 255 ? 255 : r); }
// an image index from a floored coordinate, clamped to [0, n - 1] (NaN to 0): every tap stays inside the image
__device__ __forceinline__ int clamp_tap(double f, int n) { return f >= (double)(n - 1) ? n - 1 : (f > 0.0 ? (int)f : 0); }
// getSubPixel<cv::Vec3b>(mat, row, col) (src/lioOptimization.cpp:71-98) of a BGR8 image: four saturated products and three
// saturated sums per channel, the taps (floor | floor + 1) clamped to the nearest row and column.  Inside the image (row, col
// >= 0 and floor + 1 within it, or a zero weight on the +1 tap) the values are the reference's.  The renderer and the
// photometric camera update sample through it.
__device__ __forceinline__ void sub_pixel_bgr(const unsigned char* __restrict__ img, size_t pitch, int cols, int rows, double row, double col,
                                              unsigned char out[3]) {
    const double fr = floor(row), fc = floor(col);
    const double frac_r = __dsub_rn(row, fr), frac_c = __dsub_rn(col, fc);
    const double w00 = __dmul_rn(__dsub_rn(1.0, frac_r), __dsub_rn(1.0, frac_c)), w10 = __dmul_rn(frac_r, __dsub_rn(1.0, frac_c));
    const double w01 = __dmul_rn(__dsub_rn(1.0, frac_r), frac_c), w11 = __dmul_rn(frac_r, frac_c);
    const int r0 = clamp_tap(fr, rows), r1 = clamp_tap(__dadd_rn(fr, 1.0), rows);
    const int c0 = clamp_tap(fc, cols), c1 = clamp_tap(__dadd_rn(fc, 1.0), cols);
    const unsigned char* p00 = img + (size_t)r0 * pitch + (size_t)c0 * 3;
    const unsigned char* p10 = img + (size_t)r1 * pitch + (size_t)c0 * 3;
    const unsigned char* p01 = img + (size_t)r0 * pitch + (size_t)c1 * 3;
    const unsigned char* p11 = img + (size_t)r1 * pitch + (size_t)c1 * 3;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        const unsigned char a = sat_u8(__dmul_rn((double)p00[ch], w00));
        const unsigned char b = sat_u8(__dmul_rn((double)p10[ch], w10));
        const unsigned char cc = sat_u8(__dmul_rn((double)p01[ch], w01));
        const unsigned char d = sat_u8(__dmul_rn((double)p11[ch], w11));
        out[ch] = sat_add_u8(sat_add_u8(sat_add_u8(a, b), cc), d);
    }
}
#endif

// An srl_camera as the projection kernels read it (camera_constants)
struct CamConst { double R[9], t_cw[3], t_wc[3], fx, fy, cx, cy, fov; int cols, rows; };
CamConst camera_constants(const srl_camera* cam);
// The cell coordinates of one image axis for cells of min_dis pixels over the FoV window of `fov`: the axis offset and its
// bit count (srl_map.cu).  False when they do not fit an int.
bool cell_axis(double fov, int size, double min_dis, int& offset, int& bits);
#if defined(__CUDACC__)
// cloudFrame::project3dPointInThisImage with scale 1 (src/lioOptimization.cpp:142-198) of a stored position widened to double:
// project3dTo2d (reject pcz < 0.001), then if2dPointsAvailable with the frame's own fov_margin.  Products and sums rounded one
// by one like the host code.  The renderer, the tracker's selection and the optical-flow tracker project through it.
// *z_ok (may be null) tells whether project3dTo2d got as far as writing u and v.
__device__ __forceinline__ bool project_in_image(const CamConst& c, double px, double py, double pz, double& u, double& v,
                                                 bool* z_ok = nullptr) {
    double cxm, cym, czm;
    matvec3_exact(c.R, px, py, pz, cxm, cym, czm);
    const double pcx = __dadd_rn(cxm, c.t_cw[0]), pcy = __dadd_rn(cym, c.t_cw[1]), pcz = __dadd_rn(czm, c.t_cw[2]);
    if (z_ok) *z_ok = !(pcz < 0.001);
    if (pcz < 0.001) return false;
    u = __dadd_rn(__ddiv_rn(__dmul_rn(pcx, c.fx), pcz), c.cx);
    v = __dadd_rn(__ddiv_rn(__dmul_rn(pcy, c.fy), pcz), c.cy);
    return (u >= __dadd_rn(__dmul_rn(c.fov, (double)c.cols), 1.0)) && (ceil(u) < __dmul_rn(__dsub_rn(1.0, c.fov), (double)c.cols)) &&
           (v >= __dadd_rn(__dmul_rn(c.fov, (double)c.rows), 1.0)) && (ceil(v) < __dmul_rn(__dsub_rn(1.0, c.fov), (double)c.rows));
}
// The pixel cell of a projected coordinate (src/rgbMapTracker.cpp:116-117, src/opticalFlowTracker.cpp:29-30): std::round (half
// away from zero), times min_dis, the double truncated to int
__device__ __forceinline__ int projection_cell(double x, double min_dis) { return (int)__dmul_rn(round(__ddiv_rn(x, min_dis)), min_dis); }
#endif

// A colour map's stored points as the camera updates read them (srl_map.cu owns the map): position of point id in
// blocks[(id / block_pts) * 4 * block_pts + 4 * (id % block_pts)], colour state in cpts[id]; an id is valid when its block is
// below n_voxels and its index below the block's count.
struct ColorMapView {
    const float* blocks;
    const ColorPoint* cpts;
    int block_pts;
    long long n_voxels;
};
ColorMapView color_map_view(const srl_color_map* cm);
srl_ctx* color_map_ctx(const srl_color_map* cm);
// The colour states of a colour map for the one writer outside srl_map.cu: the optical-flow tracker's is_out_lier_count
ColorPoint* color_map_states(srl_color_map* cm);
srl_ctx* lk_ctx(const srl_lk* lk);

// Which compiled instance of each pass kernel a ctx launches, and the state of its sweep-order sort.  Filled once by
// srl_ctx_create (defaults, then the SRL_* environment variables), changed by srl_ctx_set_option.
struct KernelChoice {
    int split_lpk = 4, scan_minb = 8, fit_minb = 6;   // k1_scan lanes per keypoint and blocks per SM, k1_fit blocks per SM
    int fast_lpk = 1, fast_minb = 5;                  // k1_fast
    int k1_minb = 3;                                  // k1_assoc
    int order_mode = 1;          // option "cluster_order": 0 CUB; 1, 2, 3 the cluster kernel (default, direct scatter, first version)
    int order_state = -1;        // -1 the cluster kernel is being verified against CUB, 1 verified and in use, 0 CUB
    int order_checks_left = 4;   // the first uses after the mode is set run both sorts and compare the orders on the device
    int cluster_size = 0;        // 0 not decided yet (first launch), -1 no cluster size is launchable, else the size in use
    void restart_order_checks() { order_state = order_mode ? -1 : 0; order_checks_left = 4; }
};
// Load the instances a non-debug pass of `ch` can launch, of every pass form (CUDA loads lazily at first launch, and a
// load waits for running kernels); *max_local is raised to their largest per-thread local memory (spill frame).
cudaError_t preload_fast_kernels(const KernelChoice& ch, size_t* max_local);
cudaError_t preload_assoc_kernels(const KernelChoice& ch, int K, size_t* max_local);
inline cudaError_t preload_kernel(const void* fn, size_t* max_local) {
    cudaFuncAttributes at;
    const cudaError_t e = cudaFuncGetAttributes(&at, fn);
    if (e == cudaSuccess && at.localSizeBytes > *max_local) *max_local = at.localSizeBytes;
    return e;
}
constexpr int kSplitSlots = 23;   // = NS of srl_fast.cu: candidate slots k1_scan hands to k1_fit per keypoint
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
// The Morton order of a sweep's n keypoints into d_order, by the sort ch.order_state selects.  With scratch == nullptr
// (or too small) only *needed is set.
cudaError_t sweep_compute_order(KernelChoice& ch, const double* d_raw, long long n, unsigned* d_order, void* scratch,
                                size_t scratch_bytes, size_t* needed, cudaStream_t stream);

// The pass launchers, on ctx->stream with the instance of ctx->choice; each computes its own grid for the pass's n keypoints.
// k1_assoc (the assoc form, or with a.only_flagged set the fallback launch of the fast and split forms)
cudaError_t launch_k1(const srl_ctx* ctx, const PassArgs& a, long long n, bool debug, bool pdl = false);
cudaError_t launch_k1_fast(const srl_ctx* ctx, const PassArgs& a, long long n, bool debug);
cudaError_t launch_k1_split(const srl_ctx* ctx, const PassArgs& a, long long n, bool debug, bool pdl);
cudaError_t launch_k2(const K2Args& a, cudaStream_t stream, bool pdl = false);
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
    long long* d_k2_state = nullptr;
    unsigned long long* d_cap_chunks = nullptr;   // device-resident loop: k2_cap_reduce counts the capped chunks that did work
    int64_t cap_chunks_run = 0;              // counter "cap_chunks_run": capped chunks processed by the last update's passes
    bool cap_chunks_on_device = false;       // ... still to be read from d_cap_chunks
    srl::PassStats* d_stats = nullptr;
    double* d_fast_out = nullptr;            // k1_fast's 32 sums, added by the exact-fallback launch
    bool force_exact = false;
    int force_amb_mod = 0;                   // test knob for the k1_fast -> k1_assoc hand-over
    int variant = 0;                         // 0 auto, 1 = k1_fast, 2 = k1_assoc only, 3 = k1_scan + k1_fit (1 and 3 with the exact fallback)
    srl::KernelChoice choice;
    unsigned long long* d_scan_count = nullptr;
    // device-resident updateIEKF loop (row N1)
    bool kernels_preloaded = false;          // the instances `choice` can launch are loaded; setting an integer option clears it
    int shuffle_rule = 0;                    // option "shuffle_rule": srl_build_frame's draws, 0 Lemire (libstdc++ with __int128), 1 division
    bool shuffle_on_host = false;            // option "shuffle_on_host": srl_build_frame's shuffles as a host Fisher-Yates + upload
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

namespace srl {
// What one launch of a camera update (srl_vio.cu) hands back in one device-to-host copy
struct VioOut {
    srl_vio_state state;
    double cov[121];               // the whole 11 x 11 covariance (the photometric update rewrites its 6 x 6 block)
    double acc_residual;           // of the last iteration run
    int status;                    // SRL_OK, SRL_BAD_ARG (an id names no stored point), SRL_SINGULAR
    int result;                    // the reference's return value
    int iterations, points_used;
};
// imageProcessing::setInitialCov (src/imageProcessing.cpp:65-72)
void vio_initial_covariance(double cov[121]);
}  // namespace srl

struct srl_image {
    srl_ctx* ctx = nullptr;
    int device = 0;
    int in_cols = 0, in_rows = 0;      // the input size fixed at creation
    int cols = 0, rows = 0;            // the output size
    int tiles = 0, tw = 0, th = 0;     // CLAHE's grid and its tile size
    double scale = 1.;                 // image_scale_factor
    double K[9] = {0};                 // the scaled intrinsics
    short2* map1 = nullptr;
    uint16_t* map2 = nullptr;
    uint8_t* planes = nullptr;
    uint8_t* lut = nullptr;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};   // call start, image uploaded, remapped, equalised
    bool timed = false;
    // the camera updates (srl_vio.cu)
    double cov[121] = {0};             // imageProcessing::covariance
    srl::VioOut* d_vio_out = nullptr;  // device
    cudaEvent_t vio_ev[4] = {nullptr, nullptr, nullptr, nullptr};   // before / after the esikf kernel, the photometric kernel
    bool vio_ran[2] = {false, false}, vio_timed[2] = {false, false};
    int vio_iterations[2] = {0, 0}, vio_points[2] = {0, 0};
    double vio_acc[2] = {0., 0.};
};

namespace srl {
// Device array that grows in place: virtual address space for its limit is reserved once, and physical memory is mapped
// behind it on demand (CUDA VMM), so its address never changes and growing copies nothing.  Newly mapped bytes are zero.
struct VmArray {
    unsigned long long base = 0;    // CUdeviceptr
    size_t granularity = 0, reserved = 0, mapped = 0;
    std::vector<std::pair<unsigned long long, size_t>> chunks;   // (CUmemGenericAllocationHandle, bytes), in address order
};
}  // namespace srl

struct srl_map {
    srl_ctx* ctx = nullptr;
    double voxel_size = 1.0;
    int cap = 20;
    int block_pts = srl::kBlockCap; // points per block of the pool (block stride = 4 * block_pts floats): kBlockCap for
                                    // every map the LIO path accepts; cap for a colour map of cap > kBlockCap
    size_t max_voxels = 0;          // hard limit (SRL_MAP_FULL beyond it)
    size_t committed_voxels = 0;    // blocks backed by memory; grows inside the insert / upload entry points only
    size_t capacity = 0;            // slots (power of two, >= 2 x committed_voxels): rebuilt when the map grows, so the
                                    // pass kernels take d_slots / capacity from the map at every call
    srl::Slot* d_slots = nullptr;
    srl::VmArray blocks_mem;
    float* d_blocks = nullptr;      // == blocks_mem.base
    int64_t n_voxels = 0;           // host mirror of the block count
    long long* d_counters = nullptr;   // [0] n_points, [1] scratch
    srl_color_map* owner = nullptr; // the colour map whose voxel map this is: its per-voxel arrays grow with the blocks
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
// SRL_OK for a map laid out with kBlockCap points per block (the layout every LIO kernel addresses), else SRL_BAD_ARG
int check_lio_map(srl_ctx* ctx, const srl_map* m);

// Where a caller's buffer lives.  Device covers device and managed memory: a kernel can use it in place.  Pinned is
// page-locked host memory, which the copy engine reads and writes directly.
enum class MemKind { Pageable, Pinned, Device };
MemKind mem_kind(const void* p);
// device -> host: a pinned destination is written by the copy engine directly, any other through the ctx's pinned staging
// buffer in chunks of at most 64 MB.  Returns when the bytes are in dst.
int copy_to_host(srl_ctx* ctx, void* dst, const void* d_src, size_t bytes);

inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

// Bump allocation of 256-byte-aligned arrays from one region; with base == nullptr it only measures (take returns null).
struct Carve {
    char* base = nullptr;
    size_t used = 0;
    template <class T> T* take(size_t count) {
        T* p = base ? reinterpret_cast<T*>(base + used) : nullptr;
        used += align_up(count * sizeof(T));
        return p;
    }
};
// An entry point's scratch: layout(Carve&) runs once to measure, the ctx scratch grows to that size, and layout runs again
// over it.  The layout must take the same arrays both times.
template <class Layout> int carve_scratch(srl_ctx* ctx, Layout&& layout) {
    Carve probe;
    layout(probe);
    const int rc = ensure_scratch(ctx, probe.used);
    if (rc != SRL_OK) return rc;
    Carve c{static_cast<char*>(ctx->d_scratch), 0};
    layout(c);
    return SRL_OK;
}

// A caller's buffer of T, host or device (detected per pointer), as the kernels see it: the buffer itself when it is on the
// device, else scratch placed by place().  upload() fills the scratch from an input; hand_back() returns an output.  A null
// buffer stays null.
template <class T> struct Staged {
    T* user;
    bool dev;
    T* d = nullptr;
    explicit Staged(T* p) : user(p), dev(p && mem_kind(p) == MemKind::Device) {}
    void place(Carve& c, size_t count) { d = (dev || !user) ? user : c.take<T>(count); }
    int upload(srl_ctx* ctx, size_t count) const;
    // elements [0, count) of the scratch into the caller's buffer at element `offset`
    int hand_back(srl_ctx* ctx, size_t count, size_t offset = 0) const {
        return (dev || !user) ? SRL_OK : copy_to_host(ctx, user + offset, d, count * sizeof(T));
    }
};
}  // namespace srl

#define SRL_CUDA(ctx, call)                                             \
    do {                                                                \
        cudaError_t e__ = (call);                                       \
        if (e__ != cudaSuccess) return srl::cuda_fail((ctx), e__, #call); \
    } while (0)

template <class T> int srl::Staged<T>::upload(srl_ctx* ctx, size_t count) const {
    if (!dev && user && count)
        SRL_CUDA(ctx, cudaMemcpyAsync(const_cast<void*>(static_cast<const void*>(d)), user, count * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
    return SRL_OK;
}
