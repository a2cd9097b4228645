// srl_iekf.cu — row N1 of SURVEY.md §8(f): the iterated ESIKF update on the device.
//
// k_iekf_loop is what lioOptimization::updateIEKF does between two calls of buildPlaneResiduals
// (src/optimize.cpp:172-310) plus eskfEstimator::observe (src/eskfEstimator.cpp:219-230), as ONE persistent 128-thread
// block per sweep on the ctx's side stream.  It consumes each pass's 32 sums where the pass's last block leaves them in
// HBM and hands the next pass's constants (pose) back through HBM; the pass kernels of all max_iter + 1 passes are
// enqueued on the main stream at once, wait for their pose ticket on the device and leave at once when the loop has
// ended (`break` at :309, early return at :155).  The host waits once per sweep.
//
// Why a persistent block and not a kernel per pass: the step is ~4000 instructions of straight-line FP64 code run by a
// few threads.  Launched per pass it lands on an arbitrary SM with a cold instruction cache and takes ~50 us (ncu:
// stall_no_instruction dominant); the host does the same algebra in 3 us.  A block that stays resident keeps its code
// in the SM's instruction cache, splits the step into the part that needs the sums (post) and the part that only needs
// the state (pre: boxminus, covariance projection — run in the shadow of the next pass's kernels), and runs one dry
// post step at the start of the sweep (in the shadow of pass 0) so that even the first real step finds warm code.
//
// Algebra.  The reference forms temp = (P/c)^-1, adds HTH to its top-left 6x6, inverts again and uses only the first six
// columns of the result (:234-242).  With A = P/c and M = I6 + HTH * A[0:6,0:6] the Woodbury identity gives
//     ((A^-1 + E HTH E^T)^-1)[:, 0:6] = A[:, 0:6] * M^-1        (E = first six columns of I17)
// exactly, so the step needs one 6x6 Gauss-Jordan inverse (one warp, a row per lane) instead of two 17x17 inverses; the
// result differs from the reference's double inversion by rounding only.  Against a 50-digit evaluation of the reference's
// formula (tests/test_iekf_device.py, DESIGN §4 "Algebra") the error of this form grows with cond(M), that of the double
// inversion with cond(P) + cond(P^-1 + HTH): on ill-conditioned covariances the device sits closer to the exact result
// than the host loop and the reference do.  Everything else keeps the reference's operation order, including the in-place
// column loops of the posterior covariance that read the pre-update matrix (:287-297).  The 3x3 / quaternion chains that
// do not depend on each other run on different warps.
#include "srl_eskf_math.cuh"
#include "srl_internal.h"

namespace srl {

using namespace ekf;

constexpr int kIekfThreads = 128;

__device__ __forceinline__ void copy_doubles(double* dst, const double* src, int n, int tid) {
    for (int i = tid; i < n; i += kIekfThreads) dst[i] = src[i];
}

// One warp inverts the 6x6 matrix in sM (row-major 6x12 with the identity appended) by Gauss-Jordan elimination with
// partial pivoting: lane r < 6 holds row r.  Rows are never swapped: the pivot of column k is the largest |a[r][k]| among
// the rows that have not been a pivot row yet, and the lane that pivoted column k ends up holding row k of the inverse.
// One reciprocal per column (a FP64 division is a ~40-instruction subroutine).  Returns false on a zero / NaN pivot.
__device__ __forceinline__ bool inverse6_warp(const double* sM, double* sMinv, int lane, bool store) {
    constexpr unsigned FULLM = 0xffffffffu;
    double row[12];
#pragma unroll
    for (int c = 0; c < 12; ++c) row[c] = lane < 6 ? sM[lane * 12 + c] : 0.0;
    bool ok = true, used = false;
    int my_k = 0;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        // pivot = the unused row with the largest |a[r][k]|, compared on the high word of the magnitude (monotonic for
        // non-negative doubles; 2^-20 relative resolution is plenty for choosing a pivot): one REDUX + one ballot
        const unsigned mag = (lane < 6 && !used) ? (unsigned)__double2hiint(fabs(row[k])) : 0u;
        const unsigned top = __reduce_max_sync(FULLM, mag);
        const int who = __ffs(__ballot_sync(FULLM, lane < 6 && !used && mag == top)) - 1;
        const double piv = __shfl_sync(FULLM, row[k], who < 0 ? 0 : who);
        if (who < 0 || !(fabs(piv) > 0.0)) ok = false;   // also catches NaN
        const double inv = __drcp_rn(piv);
        if (lane == who) {
#pragma unroll
            for (int c = 0; c < 12; ++c) row[c] *= inv;
            used = true; my_k = k;
        }
        const int src = who < 0 ? 0 : who;
        const double f = row[k];
#pragma unroll
        for (int c = 0; c < 12; ++c) {
            if (c > k) {   // columns <= k of the left half are already unit vectors (or become one now)
                const double pk = __shfl_sync(FULLM, row[c], src);
                if (lane != who && lane < 6) row[c] -= f * pk;
            }
        }
    }
    if (store && lane < 6) {
#pragma unroll
        for (int c = 0; c < 6; ++c) sMinv[my_k * 6 + c] = row[6 + c];
    }
    return ok;
}

struct IekfShared {
    double P0[N * N];       // eskf covariance as given (it only changes at the final pass)
    double P[N * N];        // projected prior covariance (:220-232), later updated in place by the posterior column loops
    double Pn[N * N];       // P_new of the posterior (:274)
    double A6[N * 6];       // (P / laser_point_cov)[:, 0:6]
    double sums[32];
    double H[36], HTh[6];
    double M[6 * 12], Minv[36];
    double T6[N * 6];       // temp_inv[:, 0:6]
    double Kx[N * 6], Kh[N];
    double cur[19], pred[19];   // p3 q4 v3 ba3 bg3 g3
    double dx_new[N], d_x[N];
    double Jso3[9], Js2[4];
    double q_new[4], g_new[3], Rn[9], Rq[9];
    double J2so3[9], J2s2[4];
    double n_dp, ang;
    int singular;
    int go;
    long long stamp[8];     // clock64 at the stages of the last post step (tuning)
};

__device__ __forceinline__ void rows_project(double* dst, const double* src, const double* Jso3, const double* Js2, int j) {
    // dst(3:6, j) = Jso3 * src(3:6, j); dst(15:17, j) = Js2 * src(15:17, j)      (:222-226, :281-285)
    const double c0 = src[3 * N + j], c1 = src[4 * N + j], c2 = src[5 * N + j];
#pragma unroll
    for (int r = 0; r < 3; ++r) dst[(3 + r) * N + j] = Jso3[r * 3] * c0 + (Jso3[r * 3 + 1] * c1 + Jso3[r * 3 + 2] * c2);
    const double e0 = src[15 * N + j], e1 = src[16 * N + j];
    dst[15 * N + j] = Js2[0] * e0 + Js2[1] * e1;
    dst[16 * N + j] = Js2[2] * e0 + Js2[3] * e1;
}
__device__ __forceinline__ void cols_project(double* dst, const double* src, const double* Jso3, const double* Js2, int j) {
    // dst(j, 3:6) = src(j, 3:6) * Jso3^T; dst(j, 15:17) = src(j, 15:17) * Js2^T   (:228-232, :287-297)
    const double c0 = src[j * N + 3], c1 = src[j * N + 4], c2 = src[j * N + 5];
    const double e0 = src[j * N + 15], e1 = src[j * N + 16];
#pragma unroll
    for (int r = 0; r < 3; ++r) dst[j * N + 3 + r] = Jso3[r * 3] * c0 + (Jso3[r * 3 + 1] * c1 + Jso3[r * 3 + 2] * c2);
    dst[j * N + 15] = Js2[0] * e0 + Js2[1] * e1;
    dst[j * N + 16] = Js2[2] * e0 + Js2[3] * e1;
}

// ---- pre: everything of a step that needs only the state (src/optimize.cpp:172-232): boxminus against the prediction,
//      its Jacobians, the projected prior covariance and A[:, 0:6] = (P / laser_point_cov)[:, 0:6]
__device__ __noinline__ void iekf_pre(IekfShared& S, double laser_cov) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (warp == 0 && lane == 0) {
        V3 d_so3; M3 J;
        boxminus_so3(S.pred + 3, S.cur + 3, d_so3, J);
        V3 t = J * d_so3;                                                                  // :217
        for (int i = 0; i < 3; ++i) S.dx_new[3 + i] = t.a[i];
        for (int i = 0; i < 9; ++i) S.Jso3[i] = J.a[i];
    } else if (warp == 1 && lane == 0) {
        Mat<2, 1> d_g; Mat<2, 2> J;
        boxminus_s2(S.pred + 16, S.cur + 16, d_g, J);
        Mat<2, 1> t = J * d_g;                                                             // :218
        S.dx_new[15] = t.a[0]; S.dx_new[16] = t.a[1];
        for (int i = 0; i < 4; ++i) S.Js2[i] = J.a[i];
    } else if (warp == 2 && lane < 12) {
        const int i = lane < 3 ? lane : lane + 3;            // rows 0..2 (p), 6..14 (v, ba, bg)
        const int s = lane < 3 ? lane : lane + 4;            // same entries in the packed p3 q4 v3 ba3 bg3 layout
        S.dx_new[i] = S.cur[s] - S.pred[s];
    }
    __syncthreads();
    if (tid < N) rows_project(S.P, S.P0, S.Jso3, S.Js2, tid);   // rows 3:6, 15:17 from P0 ...
    else if (tid >= 32) {                                      // ... the other rows are copies
        for (int e = tid - 32; e < N * N; e += kIekfThreads - 32) {
            const int r = e / N;
            if (!((r >= 3 && r < 6) || r >= 15)) S.P[e] = S.P0[e];
        }
    }
    __syncthreads();
    if (tid < N) cols_project(S.P, S.P, S.Jso3, S.Js2, tid);
    __syncthreads();
    if (tid < N * 6) S.A6[tid] = S.P[(tid / 6) * N + (tid % 6)] / laser_cov;              // :234 (the scaling)
    __syncthreads();
}

// ---- post: what needs the pass's sums (:234-253 up to the new state), no global memory traffic.  On return S holds
//      d_x, the observed quaternion / gravity, the next pass's rotations, |dp|, the angular distance, the posterior
//      Jacobians.  `dry` replaces d_x by typical values so that the warm-up run takes the large-angle branches.
__device__ __noinline__ void iekf_post(IekfShared& S, bool dry) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < 36) {   // HTH from its upper triangle; M = I + HTH * A66 with the identity appended
        const int r = tid / 6, c = tid % 6;
        double s = 0.0;
#pragma unroll
        for (int k = 0; k < 6; ++k) {
            const int a = r < k ? r : k, b = r < k ? k : r;
            s += S.sums[a * 6 - a * (a - 1) / 2 + (b - a)] * S.A6[k * 6 + c];
        }
        S.M[r * 12 + c] = s + (r == c ? 1.0 : 0.0);
        S.M[r * 12 + 6 + c] = (r == c ? 1.0 : 0.0);
        const int a = r < c ? r : c, b = r < c ? c : r;
        S.H[tid] = S.sums[a * 6 - a * (a - 1) / 2 + (b - a)];
    } else if (tid < 42) S.HTh[tid - 36] = S.sums[21 + tid - 36];
    __syncthreads();
    if (tid == 0) S.stamp[1] = clock64();
    {   // every warp runs the (warp-synchronous) inverse, warp 0 keeps the result: called under `if (warp == 0)` the compiler
        // cannot prove the warp converged and emits the slow collective form of every shuffle (measured: 47k cycles vs 3k)
        const bool ok = inverse6_warp(S.M, S.Minv, lane, warp == 0);
        if (tid == 0) S.singular = ok ? 0 : 1;
    }
    __syncthreads();
    if (tid == 0) S.stamp[2] = clock64();
    if (tid < N * 6) {
        const int r = tid / 6, c = tid % 6;
        double s = 0.0;
#pragma unroll
        for (int k = 0; k < 6; ++k) s += S.A6[r * 6 + k] * S.Minv[k * 6 + c];
        S.T6[tid] = s;
    }
    __syncthreads();
    if (tid < N * 6) {                                                                     // K_x (:241-242)
        const int r = tid / 6, c = tid % 6;
        double t = 0.0;
#pragma unroll
        for (int a = 0; a < 6; ++a) t += S.T6[r * 6 + a] * S.H[a * 6 + c];
        S.Kx[tid] = t;
    } else if (tid < N * 6 + N) {                                                          // K_h (:239)
        const int r = tid - N * 6;
        double s = 0.0;
#pragma unroll
        for (int a = 0; a < 6; ++a) s += S.T6[r * 6 + a] * S.HTh[a];
        S.Kh[r] = s;
    }
    __syncthreads();
    if (tid < N) {                                                                         // d_x (:244)
        const int r = tid;
        double s = 0.0;
#pragma unroll
        for (int c = 0; c < 6; ++c) s += (S.Kx[r * 6 + c] - (r == c ? 1.0 : 0.0)) * S.dx_new[c];
        if (r >= 6) s += (0.0 - 1.0) * S.dx_new[r];          // columns >= 6 of K_x are zero: only the -I term remains
        S.d_x[r] = dry ? 0.004 * (double)(r + 1) : -S.Kh[r] + s;
    }
    __syncthreads();
    if (tid == 0) S.stamp[3] = clock64();
    // guard (:248), observe (:253), posterior Jacobians (:278-279): independent chains on different warps
    if (warp == 0 && lane == 0) {
        S.n_dp = nrm(v3(S.d_x));
        S.ang = angular_distance(v3(S.d_x + 3));
    } else if (warp == 1 && lane == 0) {
        observe_quat(S.cur + 3, S.d_x + 3, S.q_new);
        // the next pass's rotations (src/optimize.cpp:35 normalised, :95,:101 as stored)
        const double* q = S.q_new;
        const double n2 = (q[0] * q[0] + q[2] * q[2]) + (q[1] * q[1] + q[3] * q[3]);
        double qn[4] = {q[0], q[1], q[2], q[3]};
        if (n2 > 0.0) { const double rn = rsqrt(n2); for (int i = 0; i < 4; ++i) qn[i] = q[i] * rn; }   // (q_new is already unit to 1 ulp)
        quat_to_rot(qn, S.Rn);
        quat_to_rot(q, S.Rq);
    } else if (warp == 2 && lane == 0) {
        observe_gravity(S.cur + 16, S.d_x[15], S.d_x[16], S.g_new);
    } else if (warp == 3 && lane == 0) {
        M3 J; Mat<2, 2> J2;
        posterior_jacobians(S.d_x + 3, S.cur + 16, S.d_x[15], S.d_x[16], J, J2);
        for (int i = 0; i < 9; ++i) S.J2so3[i] = J.a[i];
        for (int i = 0; i < 4; ++i) S.J2s2[i] = J2.a[i];
    }
    if (lane == 0) S.stamp[4 + warp] = clock64();
    __syncthreads();
}

// ---- posterior covariance (:272-307) with the reference's in-place ordering; result in S.Pn
__device__ __noinline__ void iekf_posterior(IekfShared& S) {
    const int tid = threadIdx.x;
    copy_doubles(S.Pn, S.P, N * N, tid);                                                   // P_new = P (:274)
    __syncthreads();
    if (tid < N) rows_project(S.Pn, S.P, S.J2so3, S.J2s2, tid);                            // :281-285 (reads P)
    __syncthreads();
    if (tid < N) {
        cols_project(S.Pn, S.P, S.J2so3, S.J2s2, tid);                                     // :287-297: P_new columns from the OLD P ...
        cols_project(S.P, S.P, S.J2so3, S.J2s2, tid);                                      // ... then P's own columns in place
    } else if (tid >= 32 && tid < 38) {
        const int c = tid - 32;                                                            // K_x rows (:299-303), column c
        const double c0 = S.Kx[3 * 6 + c], c1 = S.Kx[4 * 6 + c], c2 = S.Kx[5 * 6 + c];
        const double e0 = S.Kx[15 * 6 + c], e1 = S.Kx[16 * 6 + c];
#pragma unroll
        for (int r = 0; r < 3; ++r) S.Kx[(3 + r) * 6 + c] = S.J2so3[r * 3] * c0 + (S.J2so3[r * 3 + 1] * c1 + S.J2so3[r * 3 + 2] * c2);
        S.Kx[15 * 6 + c] = S.J2s2[0] * e0 + S.J2s2[1] * e1;
        S.Kx[16 * 6 + c] = S.J2s2[2] * e0 + S.J2s2[3] * e1;
    }
    __syncthreads();
    for (int e = tid; e < N * N; e += kIekfThreads) {                                      // :305-307
        const int r = e / N, c = e % N;
        double s = 0.0;
#pragma unroll
        for (int a = 0; a < 6; ++a) s += S.Kx[r * 6 + a] * S.P[a * N + c];
        S.Pn[e] = S.Pn[e] - s;
    }
    __syncthreads();
}

__device__ __forceinline__ void publish_loop_result(const IekfLoopArgs& A, const IekfDev* D, const double* sums, int tid) {
    if (!A.host_out) return;
    IekfHostOut* O = A.host_out;
    copy_doubles(reinterpret_cast<double*>(&O->eskf), reinterpret_cast<const double*>(&D->cur), (int)(sizeof(srl_eskf_state) / 8), tid);
    const int rows = D->passes_run < 32 ? D->passes_run : 32;
    copy_doubles(&O->trace[0][0], &D->trace[0][0], rows * 24, tid);
    if (tid < 4) O->frame_q[tid] = D->frame_q[tid];
    if (tid < 3) O->frame_t[tid] = D->frame_t[tid];
    if (tid < 32) O->sums[tid] = sums[tid];
    if (tid < kLoopMaxPasses) O->step_cycles[tid] = D->step_cycles[tid];
    if (tid < 8) O->stage_cycles[tid] = D->stage_cycles[tid];
    if (tid == 0) { O->status = D->status; O->passes_run = D->passes_run; O->num_residuals_used = D->num_residuals_used; O->converged = D->converged; }
    __syncthreads();
    if (tid == 0) st_release_sys(&O->seq, A.host_seq);
}

// the loop has ended: release every pass kernel still enqueued, hand the result to the host
__device__ __forceinline__ void end_loop(const IekfLoopArgs& A, IekfDev* D, IekfShared& S, int status, int tid) {
    if (tid == 0) {
        D->status = status; D->done = 1;
        st_release_gpu(&D->pose_seq, A.base + 63ull);
    }
    __syncthreads();
    publish_loop_result(A, D, S.sums, tid);
}

__global__ void __launch_bounds__(kIekfThreads, 1) k_iekf_loop(const __grid_constant__ IekfLoopArgs A) {
    __shared__ IekfShared S;
    IekfDev* D = A.dev;
    const IekfInit& init = A.init;
    const int tid = threadIdx.x;

    // ---- srl_iekf_begin (src/optimize.cpp:135-147): install the loop state
    if (tid == 0) {
        *reinterpret_cast<volatile unsigned long long*>(&D->alive_seq) = A.base;
        D->done = 0; D->abort = 0; D->status = SRL_OK; D->pass_index = -1; D->max_iter = init.max_iter;
        D->passes_run = 0; D->converged = 0; D->num_residuals_used = 0; D->frame_id = init.frame_id;
        D->min_neighbors = init.min_neighbors;
        D->laser_cov = init.laser_cov; D->thr_t = init.thr_t; D->thr_r = init.thr_r;
        D->pc = init.pc0;
        for (int i = 0; i < 4; ++i) D->frame_q[i] = init.frame_q[i];
        for (int i = 0; i < 3; ++i) D->frame_t[i] = init.frame_t[i];
    }
    {
        const double* src = reinterpret_cast<const double*>(&init.eskf);
        for (int i = tid; i < (int)(sizeof(srl_eskf_state) / 8); i += kIekfThreads) {
            const double v = src[i];
            reinterpret_cast<double*>(&D->cur)[i] = v;
            reinterpret_cast<double*>(&D->predict)[i] = v;
            if (i < 19) { S.cur[i] = v; S.pred[i] = v; }
            else S.P0[i - 19] = v;
        }
        if (tid < kLoopMaxPasses) D->step_cycles[tid] = 0;
    }
    __syncthreads();
    const double laser_cov = init.laser_cov;
    const int max_iter = init.max_iter;
    int i_pass = -1, passes_run = 0;

    iekf_pre(S, laser_cov);

    for (int it = -1;; ++it) {
        const bool dry = it < 0;
        long long t0 = 0;
        if (dry) {   // warm-up: identity-like sums, typical d_x (overwritten inside iekf_post)
            // ... unless pass 0 is already done (small shards: the pass is shorter than the cold warm-up): then every stage of
            // the warm-up would sit on the critical path, and a cold first step is the cheaper evil
            if (tid == 0) S.go = *reinterpret_cast<const volatile unsigned long long*>(&D->sums_seq) >= A.base + 1ull ? 0 : 1;
            __syncthreads();
            if (!S.go) continue;
            if (tid < 32) S.sums[tid] = (tid == 28) ? 1e9 : ((tid == 0 || tid == 6 || tid == 11 || tid == 15 || tid == 18 || tid == 20) ? 1.0 : 0.0);
            __syncthreads();
        } else {
            if (tid == 0) {
                const unsigned long long* ss = &D->sums_seq;
                const unsigned long long want = A.base + (unsigned long long)it + 1ull;
                long long spins = 0;
                bool ok = true;
                while (ld_relaxed_gpu(ss) < want) {   // the pass never finished (or the host gave up enqueueing): end the loop, do not hang
                    if (++spins > (1ll << 27) || ((spins & 63) == 0 && *reinterpret_cast<const volatile int*>(&D->abort))) { ok = false; break; }
                }
                if (ok) (void)ld_acquire_gpu(ss);
                S.go = ok ? 1 : 0;
            }
            __syncthreads();
            t0 = clock64();
            if (tid == 0) S.stamp[0] = t0;
            if (!S.go) { end_loop(A, D, S, SRL_CUDA_ERROR, tid); return; }
            if (tid < 32) S.sums[tid] = __ldcg(&D->sums[tid]);
            __syncthreads();
            // what srl_update_iekf checks before the step: exchange failure, NaN planarity (:348), too few residuals (:110-123,:155)
            const double nres = S.sums[28];
            int fail = SRL_OK;
            // a failed exchange makes all 32 sums NaN; [31] is a count, which a NaN Jacobian (NaN planarity) never turns into NaN
            if (S.sums[31] != S.sums[31] && A.world > 1) fail = SRL_COMM_ERROR;
            else if (S.sums[31] > 0.0) fail = SRL_NAN_PLANARITY;
            else if ((long long)llrint(nres) < (long long)init.min_neighbors) fail = SRL_TOO_FEW_RESIDUALS;
            passes_run += 1;
            if (tid == 0) { D->passes_run = passes_run; D->num_residuals_used = (int)llrint(nres); }
            if (fail != SRL_OK) { end_loop(A, D, S, fail, tid); return; }
        }

        iekf_post(S, dry);

        if (dry) {
            __syncthreads();
            if (tid == 0) S.go = *reinterpret_cast<const volatile unsigned long long*>(&D->sums_seq) >= A.base + 1ull ? 0 : 1;
            __syncthreads();
            if (S.go) {
                iekf_posterior(S);     // warms the final pass's code too; its inputs are rebuilt by the next iekf_pre ...
                iekf_pre(S, laser_cov);   // ... which also restores P and A6 (dx_new etc. are pure functions of cur / pred)
            }
            continue;
        }
        if (S.singular) { end_loop(A, D, S, SRL_SINGULAR, tid); return; }

        const bool diverged = S.n_dp > 100.0 || S.ang > 100.0;                             // :248-251 `continue`
        const bool converged = !diverged && init.frame_id > 1 && S.n_dp < init.thr_t && S.ang < init.thr_r;   // :265-270
        const bool final_pass = !diverged && (converged || i_pass == max_iter - 1);        // :272
        const bool done = final_pass || (i_pass + 1 >= max_iter);

        // ---- publish the next pass's pose first: that is what the pass kernels are waiting for
        if (!diverged) {
            if (tid < 3) D->pc.t[tid] = S.cur[tid] + S.d_x[tid];
            else if (tid >= 32 && tid < 41) D->pc.Rn[tid - 32] = S.Rn[tid - 32];
            else if (tid >= 64 && tid < 73) D->pc.Rq[tid - 64] = S.Rq[tid - 64];
        }
        if (tid == 0 && done) D->done = 1;
        __syncthreads();
        if (tid == 0) {
            st_release_gpu(&D->pose_seq, done ? A.base + 63ull : A.base + (unsigned long long)it + 1ull);
            if (it < kLoopMaxPasses) D->step_cycles[it] = clock64() - t0;
            for (int i = 1; i < 8; ++i) D->stage_cycles[i] = S.stamp[i] - S.stamp[0];
        }

        // ---- trace row (d_x, frame_t, frame_q as the host loop records them after the step), then the state
        const int row = passes_run - 1;
        if (row < 32) {
            double* trw = D->trace[row];
            if (tid < N) trw[tid] = S.d_x[tid];
            else if (tid >= 32 && tid < 35) trw[17 + tid - 32] = diverged ? D->frame_t[tid - 32] : S.cur[tid - 32] + S.d_x[tid - 32];
            else if (tid >= 64 && tid < 68) trw[20 + tid - 64] = diverged ? D->frame_q[tid - 64] : S.q_new[tid - 64];
        }
        __syncthreads();
        if (!diverged) {
            double nv = 0.0;
            if (tid < 3) nv = S.cur[tid] + S.d_x[tid];
            else if (tid < 7) nv = S.q_new[tid - 3];
            else if (tid < 16) nv = S.cur[tid] + S.d_x[tid - 1];
            else if (tid < 19) nv = S.g_new[tid - 16];
            __syncthreads();
            if (tid < 19) {
                S.cur[tid] = nv;
                reinterpret_cast<double*>(&D->cur)[tid] = nv;            // p3 q4 v3 ba3 bg3 g3 are the first 19 doubles
                if (tid < 3) D->frame_t[tid] = nv;
                else if (tid < 7) D->frame_q[tid - 3] = nv;
            }
        }
        i_pass += 1;
        if (tid == 0) { D->pass_index = i_pass; if (done) D->converged = (final_pass && converged) ? 1 : 0; }
        if (final_pass) {
            iekf_posterior(S);
            copy_doubles(D->cur.cov, S.Pn, N * N, tid);
        }
        if (done) {
            __syncthreads();
            publish_loop_result(A, D, S.sums, tid);
            return;
        }
        __syncthreads();
        iekf_pre(S, laser_cov);   // for the next pass, in the shadow of its kernels
    }
}

// ---- replay (srl_iekf_replay): one warp stands in for a pass.  It waits for the pass's pose exactly like a pass kernel
//      (or leaves when the loop has ended), optionally spins a bounded number of clock ticks, then hands block `p` of the
//      given sums to the loop the way a pass's last block does.  The pass constants it loads are never read.
__global__ void __launch_bounds__(32) k_iekf_feed(const __grid_constant__ IekfFeedArgs A) {
    __shared__ PassConst s_c;
    if (!load_pass_const(A.link, A.c, s_c)) return;
    if (A.delay_cycles > 0) {
        const long long t0 = clock64();
        while (clock64() - t0 < A.delay_cycles) {}
    }
    __syncwarp();
    publish_sums_to_loop(A.link, A.sums[threadIdx.x], threadIdx.x);
}
cudaError_t preload_iekf_feed() {
    cudaFuncAttributes at;
    return cudaFuncGetAttributes(&at, k_iekf_feed);
}
cudaError_t launch_iekf_feed(const IekfFeedArgs& a, cudaStream_t stream) {
    k_iekf_feed<<<1, 32, 0, stream>>>(a);
    return cudaGetLastError();
}

__global__ void k_iekf_abort(IekfDev* D) { *reinterpret_cast<volatile int*>(&D->abort) = 1; }
cudaError_t launch_iekf_abort(IekfDev* dev, cudaStream_t stream) {
    k_iekf_abort<<<1, 1, 0, stream>>>(dev);
    return cudaGetLastError();
}

// ---- can two kernels of this process run at the same time?  Under kernel-serialising tools (ncu, some sanitizer modes,
//      CUDA_LAUNCH_BLOCKING=1) they cannot, and a persistent block that waits for other kernels would only time out.
//      One probe per ctx: a one-thread kernel on the side stream waits (bounded) for a word that a kernel on the main
//      stream sets.
__global__ void k_probe_wait(volatile int* flag, int* result, long long max_cycles) {
    const long long t0 = clock64();
    int seen = 0;
    while (!(seen = *flag)) { if (clock64() - t0 > max_cycles) break; }
    *result = seen ? 1 : 0;
}
__global__ void k_probe_set(volatile int* flag) { *flag = 1; }

cudaError_t probe_concurrent_kernels(cudaStream_t side, cudaStream_t main_stream, int* d_two_ints, bool* concurrent) {
    cudaFuncAttributes at;   // load all three kernels now: a lazy load during the probe would wait for the waiting kernel
    cudaError_t e = cudaFuncGetAttributes(&at, k_probe_wait);
    if (e == cudaSuccess) e = cudaFuncGetAttributes(&at, k_probe_set);
    if (e == cudaSuccess) e = cudaFuncGetAttributes(&at, k_iekf_abort);
    if (e == cudaSuccess) e = cudaFuncGetAttributes(&at, k_iekf_loop);
    if (e == cudaSuccess) e = cudaMemsetAsync(d_two_ints, 0, 2 * sizeof(int), main_stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(main_stream);
    if (e != cudaSuccess) return e;
    k_probe_wait<<<1, 1, 0, side>>>(d_two_ints, d_two_ints + 1, 100ll * 1000 * 1000);   // ~50 ms at 2 GHz
    k_probe_set<<<1, 1, 0, main_stream>>>(d_two_ints);
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(side);
    if (e == cudaSuccess) e = cudaStreamSynchronize(main_stream);
    int h[2] = {0, 0};
    if (e == cudaSuccess) e = cudaMemcpy(h, d_two_ints, sizeof(h), cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) *concurrent = h[1] != 0;
    return e;
}

cudaError_t launch_iekf_loop(const IekfLoopArgs& a, cudaStream_t stream) {
    k_iekf_loop<<<1, kIekfThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

}  // namespace srl
