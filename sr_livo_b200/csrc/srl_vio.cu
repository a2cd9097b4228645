// srl_vio.cu — the two camera updates of imageProcessing::process on the device (row N8): vioEsikf
// (src/imageProcessing.cpp:220-380) and vioPhotometric (:402-552), each one launch of one block with both iterations inside.
//
// Per iteration the block projects the tracked points chunk by chunk: every thread writes its point's Huber-scaled Jacobian
// rows and residuals (and, photometric, the rows' 1 / cov_rgb weights) to shared memory, then a fixed set of threads sums each
// entry of S = HᵀR⁻¹H and g = HᵀR⁻¹r over the chunk in row order (a fixed number of contiguous segments per entry, added in
// segment order), so the result is the same bits on every run.  R_mat_inv is diagonal, which is what turns the reference's
// dense 2n x 11 / 3n x 6 products into these per-point sums.  Warp 0 then runs the D x D algebra (D = 11 or 6):
//   Pw = (J P Jᵀ) w,  A = S + Pw⁻¹,  K r = A⁻¹ g,  K H = A⁻¹ S,  with A⁻¹ = (I + Pw S)⁻¹ Pw (Woodbury: Pw is never inverted)
// by one Gauss-Jordan elimination with partial pivoting (a column per lane); thread 0 applies updateCameraParameters.  The
// file is built with --fmad=false: products and sums are rounded one by one, as the reference's scalar Eigen code does.
#include <cmath>

#include "srl_internal.h"
#include "srl_eskf_math.cuh"

using namespace srl;
using srl::ekf::M3;
using srl::ekf::Q;
using srl::ekf::V3;

namespace {

constexpr int kVioThreads = 256;
constexpr int kVioChunk = 128;           // points projected per round
constexpr int kMinPoints = 10;           // minimum_iteration_points (:218)
constexpr int kIterations = 2;           // num_iterations (:15)

// MODE 0: vioEsikf, state (td, so3, t, fx, fy, cx, cy), two rows per point, row = H (11), r
// MODE 1: vioPhotometric, state (so3, t), three rows per point, row = H (6), r, 1 / cov_rgb
template <int MODE> struct Dims {
    static constexpr int D = MODE == 0 ? 11 : 6;
    static constexpr int RPP = MODE == 0 ? 2 : 3;
    static constexpr int W = MODE == 0 ? D + 1 : D + 2;
    static constexpr int NS = D * (D + 1) / 2;      // upper triangle of S
    static constexpr int E = NS + D + 2;            // + g + acc_residual + points used
    static constexpr int P = kVioThreads / E;       // segments per entry
    static constexpr int SO3 = MODE == 0 ? 1 : 0;   // offset of the rotation in the state vector
};

struct VioArgs {
    ColorMapView cm;
    const unsigned* ids;
    const float* uv;                  // MODE 0
    const double* vel;
    long long n;
    const unsigned char* img;         // MODE 1: BGR8, rows `pitch` bytes apart
    size_t pitch;
    int cols, rows;
    double weight;                    // cam_measurement_weight
    srl_vio_state st;
    double cov[121];
    VioOut* out;
};

// getHuberLoss(residual, 1) (:202-216)
__device__ __forceinline__ double huber(double r) { return r < 1.0 ? 1.0 : (2.0 * sqrt(r) / 1.0 - 1.0) / r; }

// cloudFrame::getRgb with derivatives (src/lioOptimization.cpp:100-140): the centre tap, and the Vec3f sums of eight more
// taps at u -+ 1..4 (dx) and v -+ 1..4 (dy) divided by the float 2 + 4 + 6 + 8 = 20 in double
__device__ __forceinline__ void get_rgb(const VioArgs& a, double u, double v, double c[3], double dx[3], double dy[3]) {
    unsigned char t[3];
    sub_pixel_bgr(a.img, a.pitch, a.cols, a.rows, v, u, t);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) c[ch] = (double)t[ch];
    float l[3] = {0.f, 0.f, 0.f}, r[3] = {0.f, 0.f, 0.f}, pd = 0.f;
#pragma unroll
    for (int b = 1; b < 5; ++b) {
        unsigned char tl[3], tr[3];
        sub_pixel_bgr(a.img, a.pitch, a.cols, a.rows, v, u - b, tl);
        sub_pixel_bgr(a.img, a.pitch, a.cols, a.rows, v, u + b, tr);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) { l[ch] = l[ch] + (float)tl[ch]; r[ch] = r[ch] + (float)tr[ch]; }
        pd = pd + (float)(2 * b);
    }
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) dx[ch] = (double)(r[ch] - l[ch]) / (double)pd;
    float dn[3] = {0.f, 0.f, 0.f}, up[3] = {0.f, 0.f, 0.f};
    pd = 0.f;
#pragma unroll
    for (int b = 1; b < 5; ++b) {
        unsigned char td[3], tu[3];
        sub_pixel_bgr(a.img, a.pitch, a.cols, a.rows, v - b, u, td);
        sub_pixel_bgr(a.img, a.pitch, a.cols, a.rows, v + b, u, tu);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) { dn[ch] = dn[ch] + (float)td[ch]; up[ch] = up[ch] + (float)tu[ch]; }
        pd = pd + (float)(2 * b);
    }
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) dy[ch] = (double)(up[ch] - dn[ch]) / (double)pd;
}

struct Cam {                          // the pose and intrinsics iteration k projects with
    double Rcw[9], tcw[3], RicT[9];   // q_camera_world.toRotationMatrix(), t_camera_world, R_imu_cameraᵀ
    double fx, fy, cx, cy, td;
};

// one point's rows (Huber-scaled, as :324-347 / :476-517); returns false for a photometric point with N_rgb < 3
template <int MODE>
__device__ __forceinline__ bool point_rows(const VioArgs& a, const Cam& c, long long i, double* rows, double& acc) {
    using Dm = Dims<MODE>;
    const unsigned id = a.ids[i];
    const ColorPoint cp = a.cm.cpts[id];
    if (MODE == 1 && cp.n_rgb < 3) return false;
    const float* bp = a.cm.blocks + (size_t)(id / (unsigned)a.cm.block_pts) * (4 * a.cm.block_pts) + 4 * (id % (unsigned)a.cm.block_pts);
    const double pw0 = (double)bp[0], pw1 = (double)bp[1], pw2 = (double)bp[2];
    double x, y, z;
    matvec3_exact(c.Rcw, pw0, pw1, pw2, x, y, z);
    x = x + c.tcw[0]; y = y + c.tcw[1]; z = z + c.tcw[2];
    const double v0 = a.vel[2 * i], v1 = a.vel[2 * i + 1];
    const double pu = (c.fx * x / z + c.cx) + c.td * v0, pv = (c.fy * y / z + c.cy) + c.td * v1;
    // J_u_pc (:330-331), J_u_pc * skew(pc) and -J_u_pc * R_imu_cameraᵀ
    const double J[6] = {c.fx / z, 0.0, -(c.fx * x) / (z * z), 0.0, c.fy / z, -(c.fy * y) / (z * z)};
    const double S[9] = {0.0, -z, y, z, 0.0, -x, -y, x, 0.0};
    if (MODE == 0) {
        const double ex = pu - (double)a.uv[2 * i], ey = pv - (double)a.uv[2 * i + 1];
        const double res = sqrt(ex * ex + ey * ey);
        const double h = huber(res);
        acc = res;
        const double JK[8] = {x / z, 0.0, 1.0, 0.0, 0.0, y / z, 0.0, 1.0};
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            double* row = rows + k * Dm::W;
            row[0] = (k == 0 ? v0 : v1) * h;
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                row[1 + j] = dot3_exact(J[3 * k], J[3 * k + 1], J[3 * k + 2], S[j], S[3 + j], S[6 + j]) * h;
                row[4 + j] = dot3_exact(-J[3 * k], -J[3 * k + 1], -J[3 * k + 2], c.RicT[j], c.RicT[3 + j], c.RicT[6 + j]) * h;
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) row[7 + j] = JK[4 * k + j] * h;
            row[11] = (k == 0 ? ex : ey) * h;
        }
    } else {
        double col[3], dx[3], dy[3];
        get_rgb(a, pu, pv, col, dx, dy);
        double e[3], info[3];
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) { e[ch] = col[ch] - (double)cp.rgb[ch]; info[ch] = 1.0 / (double)cp.cov[ch]; }
        const double h = huber(sqrt(e[0] * e[0] + (e[1] * e[1] + e[2] * e[2])));
        double rs[3];
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) rs[ch] = e[ch] * h;
        acc = (rs[0] * info[0]) * rs[0] + ((rs[1] * info[1]) * rs[1] + (rs[2] * info[2]) * rs[2]);   // :497
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            // J_color_pc row k = (dx_k, dy_k) * J_u_pc
            const double jc[3] = {dx[k] * J[0] + dy[k] * J[3], dx[k] * J[1] + dy[k] * J[4], dx[k] * J[2] + dy[k] * J[5]};
            double* row = rows + k * Dm::W;
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                row[j] = dot3_exact(jc[0], jc[1], jc[2], S[j], S[3 + j], S[6 + j]) * h;
                row[3 + j] = dot3_exact(-jc[0], -jc[1], -jc[2], c.RicT[j], c.RicT[3 + j], c.RicT[6 + j]) * h;
            }
            row[6] = rs[k];
            row[7] = info[k];
        }
    }
    return true;
}

// C = A * B (transB: A * Bᵀ), D x D row-major in shared memory, a column per lane of the calling warp
template <int D>
__device__ __forceinline__ void warp_mm(const double* A, const double* B, double* C, bool transB, int lane) {
    if (lane < D)
        for (int i = 0; i < D; ++i) {
            double s = 0.0;
            for (int k = 0; k < D; ++k) s = s + A[i * D + k] * (transB ? B[lane * D + k] : B[k * D + lane]);
            C[i * D + lane] = s;
        }
    __syncwarp();
}

// Gauss-Jordan elimination of aug = [M | B] (D x 2D) with partial pivoting: aug becomes [I | M⁻¹B].  A column per lane; every
// lane finds the same pivot.  false for a zero or NaN pivot.
template <int D>
__device__ __forceinline__ bool warp_gauss_jordan(double* aug, double* fac, int lane) {
    constexpr int W2 = 2 * D;
    for (int k = 0; k < D; ++k) {
        int p = k;
        double best = fabs(aug[k * W2 + k]);
        for (int i = k + 1; i < D; ++i) {
            const double m = fabs(aug[i * W2 + k]);
            if (m > best) { best = m; p = i; }
        }
        const double piv = aug[p * W2 + k];
        if (!(piv != 0.0) || isnan(piv)) return false;
        __syncwarp();
        if (lane < W2 && p != k) {
            const double t = aug[k * W2 + lane];
            aug[k * W2 + lane] = aug[p * W2 + lane];
            aug[p * W2 + lane] = t;
        }
        __syncwarp();
        if (lane < D) fac[lane] = aug[lane * W2 + k];
        __syncwarp();
        if (lane < W2) {
            const double rk = aug[k * W2 + lane] / piv;
            aug[k * W2 + lane] = rk;
            for (int i = 0; i < D; ++i)
                if (i != k) aug[i * W2 + lane] = aug[i * W2 + lane] - fac[i] * rk;
        }
        __syncwarp();
    }
    return true;
}

struct HostState {                    // p_state, as thread 0 updates it
    Q rotation, q_wc, q_cw;
    M3 Ric;
    double translation[3], tic[3], t_wc[3], t_cw[3];
    double fx, fy, cx, cy, td;
};

__device__ __forceinline__ void load_state(const srl_vio_state& s, HostState& h) {
    h.rotation = ekf::mkq(s.rotation); h.q_wc = ekf::mkq(s.q_world_camera); h.q_cw = ekf::mkq(s.q_camera_world);
    for (int k = 0; k < 9; ++k) h.Ric.a[k] = s.R_imu_camera[k];
#pragma unroll
    for (int k = 0; k < 3; ++k) { h.translation[k] = s.translation[k]; h.tic[k] = s.t_imu_camera[k]; h.t_wc[k] = s.t_world_camera[k]; h.t_cw[k] = s.t_camera_world[k]; }
    h.fx = s.fx; h.fy = s.fy; h.cx = s.cx; h.cy = s.cy; h.td = s.time_td;
}
__device__ __forceinline__ void store_state(const HostState& h, srl_vio_state& s) {
    s.rotation[0] = h.rotation.x; s.rotation[1] = h.rotation.y; s.rotation[2] = h.rotation.z; s.rotation[3] = h.rotation.w;
    s.q_world_camera[0] = h.q_wc.x; s.q_world_camera[1] = h.q_wc.y; s.q_world_camera[2] = h.q_wc.z; s.q_world_camera[3] = h.q_wc.w;
    s.q_camera_world[0] = h.q_cw.x; s.q_camera_world[1] = h.q_cw.y; s.q_camera_world[2] = h.q_cw.z; s.q_camera_world[3] = h.q_cw.w;
    for (int k = 0; k < 9; ++k) s.R_imu_camera[k] = h.Ric.a[k];
#pragma unroll
    for (int k = 0; k < 3; ++k) { s.translation[k] = h.translation[k]; s.t_imu_camera[k] = h.tic[k]; s.t_world_camera[k] = h.t_wc[k]; s.t_camera_world[k] = h.t_cw[k]; }
    s.fx = h.fx; s.fy = h.fy; s.cx = h.cx; s.cy = h.cy; s.time_td = h.td;
}

// updateCameraParameters (both overloads, :382-400 and :554-566) with cloudFrame::refreshPoseForProjection
// (src/lioOptimization.cpp:201-205)
template <int MODE>
__device__ __forceinline__ void update_camera(HostState& h, const double* d) {
    constexpr int o = Dims<MODE>::SO3;
    if (MODE == 0) h.td = h.td + d[0];
    V3 w; w.a[0] = d[o]; w.a[1] = d[o + 1]; w.a[2] = d[o + 2];
    const Q q = ekf::qunit(ekf::qmul(ekf::rot2q(h.Ric), ekf::exp_quat(w)));
    h.Ric = ekf::qrot(q);
#pragma unroll
    for (int k = 0; k < 3; ++k) h.tic[k] = h.tic[k] + d[o + 3 + k];
    if (MODE == 0) { h.fx = h.fx + d[7]; h.fy = h.fy + d[8]; h.cx = h.cx + d[9]; h.cy = h.cy + d[10]; }
    const M3 Rw = ekf::qrot(h.rotation);
    h.q_wc = ekf::rot2q(Rw * h.Ric);
    double r0, r1, r2;
    matvec3_exact(Rw.a, h.tic[0], h.tic[1], h.tic[2], r0, r1, r2);
    h.t_wc[0] = r0 + h.translation[0]; h.t_wc[1] = r1 + h.translation[1]; h.t_wc[2] = r2 + h.translation[2];
    h.q_cw = ekf::qinv(h.q_wc);
    const M3 Rcw = ekf::qrot(h.q_cw);
    double n[9];
    for (int k = 0; k < 9; ++k) n[k] = -Rcw.a[k];
    matvec3_exact(n, h.t_wc[0], h.t_wc[1], h.t_wc[2], h.t_cw[0], h.t_cw[1], h.t_cw[2]);
}

template <int MODE>
__global__ void __launch_bounds__(kVioThreads, 1) k_vio_update(const __grid_constant__ VioArgs a) {
    using Dm = Dims<MODE>;
    constexpr int D = Dm::D, RPP = Dm::RPP, W = Dm::W, E = Dm::E, P = Dm::P, NS = Dm::NS;
    __shared__ double s_rows[kVioChunk * RPP * W];
    __shared__ double s_acc[kVioChunk];
    __shared__ unsigned char s_used[kVioChunk];
    __shared__ double s_part[kVioThreads];
    __shared__ double s_tot[E];
    __shared__ double s_P[D * D], s_J[D * D], s_T[D * D], s_Pw[D * D], s_S[D * D], s_KH[D * D], s_X[D * D];
    __shared__ double s_aug[D * 2 * D];
    __shared__ double s_fac[D], s_g[D], s_dx[D], s_sol[D];
    __shared__ Cam s_cam;
    __shared__ HostState s_h, s_pred;
    __shared__ int s_flag;   // per iteration: 0 go on, 1 break, 2 singular
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    // ids are validated before anything is read through them (srl_color_map_gather_points' rule)
    bool bad = false;
    for (long long i = tid; i < a.n; i += kVioThreads) {
        const unsigned id = a.ids[i];
        const unsigned blk = id / (unsigned)a.cm.block_pts;
        bad |= (long long)blk >= a.cm.n_voxels ||
               id - blk * (unsigned)a.cm.block_pts >= reinterpret_cast<const unsigned*>(a.cm.blocks + (size_t)blk * (4 * a.cm.block_pts))[kMetaCount];
    }
    if (__syncthreads_or(bad)) {
        if (tid == 0) { a.out->status = SRL_BAD_ARG; a.out->result = 0; a.out->iterations = 0; a.out->points_used = 0; }
        return;
    }
    // the working covariance: the whole 11 x 11 (vioEsikf) or its block (1..6, 1..6) (vioPhotometric)
    for (int k = tid; k < D * D; k += kVioThreads) {
        const int r = k / D, c = k % D;
        s_P[k] = MODE == 0 ? a.cov[k] : a.cov[(r + 1) * 11 + c + 1];
    }
    if (tid == 0) {
        load_state(a.st, s_h);
        s_pred = s_h;   // the prediction the steps d_x are taken from (:259-265, :427-428)
    }
    __syncthreads();
    double last_acc = 3e8, acc_out = 0.0;
    int iterations = 0, used_out = 0, status = SRL_OK;
    bool have_k = false;

    for (int iter = 0; iter < kIterations; ++iter) {
        if (tid == 0) {
            // d_x, the state's step from the prediction (:289-304, :454-459)
            const Q dq = ekf::qmul(ekf::qinv(ekf::rot2q(s_pred.Ric)), ekf::rot2q(s_h.Ric));
            const V3 dso3 = ekf::log_so3(ekf::qrot(dq));
            constexpr int o = Dm::SO3;
            if (MODE == 0) s_dx[0] = s_h.td - s_pred.td;
#pragma unroll
            for (int k = 0; k < 3; ++k) { s_dx[o + k] = dso3.a[k]; s_dx[o + 3 + k] = s_h.tic[k] - s_pred.tic[k]; }
            if (MODE == 0) { s_dx[7] = s_h.fx - s_pred.fx; s_dx[8] = s_h.fy - s_pred.fy; s_dx[9] = s_h.cx - s_pred.cx; s_dx[10] = s_h.cy - s_pred.cy; }
            const M3 Rcw = ekf::qrot(s_h.q_cw);
            for (int k = 0; k < 9; ++k) { s_cam.Rcw[k] = Rcw.a[k]; s_cam.RicT[k] = s_h.Ric.a[(k % 3) * 3 + k / 3]; }
#pragma unroll
            for (int k = 0; k < 3; ++k) s_cam.tcw[k] = s_h.t_cw[k];
            s_cam.fx = s_h.fx; s_cam.fy = s_h.fy; s_cam.cx = s_h.cx; s_cam.cy = s_h.cy; s_cam.td = s_h.td;
        }
        __syncthreads();
        // the sums: entry e of thread tid < E is its running total over the chunks; segment (tid / E) of entry (tid % E)
        double total = 0.0;
        const int e = tid % E, seg = tid / E;
        for (long long base = 0; base < a.n; base += kVioChunk) {
            const int cnt = (int)min((long long)kVioChunk, a.n - base);
            if (tid < cnt) {
                double acc = 0.0;
                const bool u = point_rows<MODE>(a, s_cam, base + tid, s_rows + tid * RPP * W, acc);
                if (!u)
                    for (int k = 0; k < RPP * W; ++k) s_rows[tid * RPP * W + k] = 0.0;
                s_acc[tid] = u ? acc : 0.0;
                s_used[tid] = u ? 1 : 0;
            }
            __syncthreads();
            if (seg < P) {
                double s = 0.0;
                if (e < NS + D) {
                    // entry (ea, eb) of S, or ea of g (eb = the residual column)
                    int ea, eb;
                    if (e < NS) {
                        int k = e;
                        ea = 0;
                        while (k >= D - ea) { k -= D - ea; ++ea; }
                        eb = ea + k;
                    } else {
                        ea = e - NS;
                        eb = D;
                    }
                    const int nr = cnt * RPP, len = (nr + P - 1) / P, lo = seg * len, hi = min(nr, lo + len);
                    for (int r = lo; r < hi; ++r) {
                        const double* row = s_rows + r * W;
                        const double ha = MODE == 0 ? row[ea] : row[ea] * row[D + 1];
                        s = s + ha * row[eb];
                    }
                } else {
                    const int len = (cnt + P - 1) / P, lo = seg * len, hi = min(cnt, lo + len);
                    for (int r = lo; r < hi; ++r) s = s + (e == NS + D ? s_acc[r] : (double)s_used[r]);
                }
                s_part[tid] = s;
            }
            __syncthreads();
            if (tid < E) {
                double c = s_part[tid];
                for (int p = 1; p < P; ++p) c = c + s_part[p * E + tid];
                total = total + c;
            }
            __syncthreads();
        }
        if (tid < E) s_tot[tid] = total;
        __syncthreads();
        double acc = s_tot[NS + D];
        const int used = (int)s_tot[NS + D + 1];
        if (MODE == 0) acc = acc / (double)a.n;   // acc_residual /= total_point_size (:351)
        used_out = used;
        if (used < kMinPoints) break;             // :353, :520
        if (warp == 0) {
            // S, g
            for (int k = lane; k < NS; k += 32) {
                int r = k, ea = 0;
                while (r >= D - ea) { r -= D - ea; ++ea; }
                const int eb = ea + r;
                s_S[ea * D + eb] = s_tot[k];
                s_S[eb * D + ea] = s_tot[k];
            }
            if (lane < D) s_g[lane] = s_tot[NS + lane];
            // J_zero (:358-359, :525-526)
            for (int k = lane; k < D * D; k += 32) s_J[k] = (k / D == k % D) ? 1.0 : 0.0;
            __syncwarp();
            if (lane == 0) {
                constexpr int o = Dm::SO3;
                const double* w = s_dx + o;
                const double hw[9] = {0.0, -w[2], w[1], w[2], 0.0, -w[0], -w[1], w[0], 0.0};
                for (int r = 0; r < 3; ++r)
                    for (int c = 0; c < 3; ++c) s_J[(o + r) * D + o + c] = (r == c ? 1.0 : 0.0) - 0.5 * hw[r * 3 + c];
            }
            __syncwarp();
            // Pw = J P Jᵀ w
            warp_mm<D>(s_J, s_P, s_T, false, lane);
            warp_mm<D>(s_T, s_J, s_Pw, true, lane);
            for (int k = lane; k < D * D; k += 32) s_Pw[k] = s_Pw[k] * a.weight;
            __syncwarp();
            // [I + Pw S | Pw]
            warp_mm<D>(s_Pw, s_S, s_T, false, lane);
            for (int k = lane; k < D * D; k += 32) {
                const int r = k / D, c = k % D;
                s_aug[r * 2 * D + c] = (r == c ? 1.0 : 0.0) + s_T[k];
                s_aug[r * 2 * D + D + c] = s_Pw[k];
            }
            __syncwarp();
            const bool ok = warp_gauss_jordan<D>(s_aug, s_fac, lane);
            if (ok) {
                for (int k = lane; k < D * D; k += 32) s_X[k] = s_aug[(k / D) * 2 * D + D + k % D];
                __syncwarp();
                warp_mm<D>(s_X, s_S, s_KH, false, lane);   // K H = A⁻¹ S
                // solution = -K r - (I - K H) J d_x (:362, :529)
                if (lane < D) {
                    double jd = 0.0;
                    for (int k = 0; k < D; ++k) jd = jd + s_J[lane * D + k] * s_dx[k];
                    s_fac[lane] = jd;
                }
                __syncwarp();
                if (lane < D) {
                    double kr = 0.0, t = 0.0;
                    for (int k = 0; k < D; ++k) {
                        kr = kr + s_X[lane * D + k] * s_g[k];
                        t = t + ((lane == k ? 1.0 : 0.0) - s_KH[lane * D + k]) * s_fac[k];
                    }
                    s_sol[lane] = -kr - t;
                }
                __syncwarp();
                if (lane == 0) update_camera<MODE>(s_h, s_sol);
            }
            if (lane == 0) {
                int f = ok ? 0 : 2;
                if (ok) {
                    if (MODE == 1 && acc / (double)a.n < 10) f = 1;   // :533
                    else if (fabs(acc - last_acc) < 0.01) f = 1;      // :366, :538
                }
                s_flag = f;
            }
        }
        __syncthreads();
        const int f = s_flag;
        if (f == 2) { status = SRL_SINGULAR; break; }
        have_k = true;
        ++iterations;
        acc_out = acc;
        last_acc = acc;
        if (f == 1) break;
    }
    // the posterior covariance from the last iteration's K, H and solution (:374-377, :546-549)
    if (status == SRL_OK && have_k && warp == 0) {
        for (int k = lane; k < D * D; k += 32) s_J[k] = (k / D == k % D) ? 1.0 : 0.0;
        __syncwarp();
        if (lane == 0) {
            constexpr int o = Dm::SO3;
            const double* w = s_sol + o;
            const double hw[9] = {0.0, -w[2], w[1], w[2], 0.0, -w[0], -w[1], w[0], 0.0};
            for (int r = 0; r < 3; ++r)
                for (int c = 0; c < 3; ++c) s_J[(o + r) * D + o + c] = (r == c ? 1.0 : 0.0) - 0.5 * hw[r * 3 + c];
        }
        for (int k = lane; k < D * D; k += 32) s_KH[k] = (k / D == k % D ? 1.0 : 0.0) - s_KH[k];
        __syncwarp();
        warp_mm<D>(s_J, s_KH, s_T, false, lane);
        warp_mm<D>(s_T, s_P, s_X, false, lane);
        warp_mm<D>(s_X, s_J, s_P, true, lane);
    }
    __syncthreads();
    VioOut* out = a.out;
    if (tid == 0) {
        out->status = status;
        out->result = 1;   // both return true past the n < 10 test, which the host makes
        out->iterations = iterations;
        out->points_used = used_out;
        out->acc_residual = acc_out;
        store_state(s_h, out->state);
    }
    for (int k = tid; k < 121; k += kVioThreads) {
        const int r = k / 11, c = k % 11;
        double v = a.cov[k];
        if (MODE == 0) v = s_P[k];
        else if (r >= 1 && r <= 6 && c >= 1 && c <= 6) v = s_P[(r - 1) * D + c - 1];
        out->cov[k] = v;
    }
}

int vio_fail(srl_ctx* ctx, int code, const char* fn, const char* msg) { return set_err(ctx, code, std::string(fn) + ": " + msg); }

// everything the two entry points share: argument checks, staging, one launch, one copy back, the state and covariance applied
int vio_run(int mode, srl_image* im, srl_color_map* cm, srl_vio_state* state, const uint32_t* ids, const float* uv, const double* velocity,
            size_t n, int32_t n_new_visited, const uint8_t* bgr, int cols, int rows, size_t pitch, int32_t* result) {
    const char* fn = mode == 0 ? "srl_image_vio_esikf" : "srl_image_vio_photometric";
    if (!im) return SRL_BAD_ARG;
    srl_ctx* ctx = im->ctx;
    if (!cm || !state || !result) return vio_fail(ctx, SRL_BAD_ARG, fn, "cm, state and result are required");
    if (color_map_ctx(cm)->device != ctx->device) return vio_fail(ctx, SRL_BAD_ARG, fn, "the colour map lives on another device");
    if (n > 0x7fffffffULL) return vio_fail(ctx, SRL_BAD_ARG, fn, "n must fit in int32");
    if (n && (!ids || !velocity || (mode == 0 && !uv))) return vio_fail(ctx, SRL_BAD_ARG, fn, "ids, uv (vioEsikf) and velocity are required");
    if (mode == 1) {
        if (!bgr) return vio_fail(ctx, SRL_BAD_ARG, fn, "bgr is required");
        if (cols != im->cols || rows != im->rows) return vio_fail(ctx, SRL_BAD_ARG, fn, "the image must have the handle's output size");
        if (pitch < (size_t)cols * 3) return vio_fail(ctx, SRL_BAD_ARG, fn, "pitch must be at least cols * 3 bytes");
    }
    // total_point_size < minimum_iteration_points (:249, :415): false, nothing changes
    if (n < (size_t)kMinPoints) {
        *result = 0;
        im->vio_ran[mode] = true;
        im->vio_iterations[mode] = 0;
        im->vio_points[mode] = 0;
        im->vio_acc[mode] = 0.0;
        return SRL_OK;
    }
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    Staged<const unsigned> s_ids(ids);
    Staged<const float> s_uv(mode == 0 ? uv : nullptr);
    Staged<const double> s_vel(velocity);
    const bool img_dev = mode == 1 && mem_kind(bgr) == MemKind::Device;
    uint8_t* d_img = nullptr;
    int rc = carve_scratch(ctx, [&](Carve& c) {
        s_ids.place(c, n);
        s_uv.place(c, n * 2);
        s_vel.place(c, n * 2);
        d_img = (mode == 1 && !img_dev) ? c.take<uint8_t>((size_t)cols * rows * 3) : nullptr;
    });
    if (rc != SRL_OK || (rc = s_ids.upload(ctx, n)) != SRL_OK || (rc = s_uv.upload(ctx, n * 2)) != SRL_OK ||
        (rc = s_vel.upload(ctx, n * 2)) != SRL_OK)
        return rc;
    VioArgs a = {};
    a.cm = color_map_view(cm);
    a.ids = s_ids.d;
    a.uv = s_uv.d;
    a.vel = s_vel.d;
    a.n = (long long)n;
    if (mode == 1) {
        if (!img_dev) SRL_CUDA(ctx, cudaMemcpy2DAsync(d_img, (size_t)cols * 3, bgr, pitch, (size_t)cols * 3, rows, cudaMemcpyHostToDevice, st));
        a.img = img_dev ? bgr : d_img;
        a.pitch = img_dev ? pitch : (size_t)cols * 3;
        a.cols = cols;
        a.rows = rows;
    }
    a.weight = std::max(0.001, std::min(5.0 / n_new_visited, 0.01));   // :272, :435 (an int count: 0 gives 0.01)
    a.st = *state;
    for (int k = 0; k < 121; ++k) a.cov[k] = im->cov[k];
    a.out = im->d_vio_out;
    SRL_CUDA(ctx, cudaEventRecord(im->vio_ev[2 * mode], st));
    if (mode == 0) k_vio_update<0><<<1, kVioThreads, 0, st>>>(a);
    else k_vio_update<1><<<1, kVioThreads, 0, st>>>(a);
    SRL_CUDA(ctx, cudaGetLastError());
    SRL_CUDA(ctx, cudaEventRecord(im->vio_ev[2 * mode + 1], st));
    ctx->launches += 1;
    VioOut o;
    SRL_CUDA(ctx, cudaMemcpyAsync(&o, im->d_vio_out, sizeof(VioOut), cudaMemcpyDeviceToHost, st));
    SRL_CUDA(ctx, cudaStreamSynchronize(st));
    im->vio_timed[mode] = true;
    if (o.status == SRL_BAD_ARG) return vio_fail(ctx, SRL_BAD_ARG, fn, "a point id names no stored point");
    if (o.status == SRL_SINGULAR) return vio_fail(ctx, SRL_SINGULAR, fn, "zero or NaN pivot in the update's normal equations");
    *state = o.state;
    for (int k = 0; k < 121; ++k) im->cov[k] = o.cov[k];
    *result = o.result;
    im->vio_ran[mode] = true;
    im->vio_iterations[mode] = o.iterations;
    im->vio_points[mode] = o.points_used;
    im->vio_acc[mode] = o.acc_residual;
    return SRL_OK;
}

}  // namespace

void srl::vio_initial_covariance(double cov[121]) {
    for (int k = 0; k < 121; ++k) cov[k] = 0.0;
    cov[0] = 0.00001;
    for (int i = 1; i < 7; ++i) cov[i * 11 + i] = 1e-3;    // extrinsic between camera and IMU
    for (int i = 7; i < 11; ++i) cov[i * 11 + i] = 1e-3;   // camera intrinsic
}

extern "C" {

int srl_image_vio_esikf(srl_image* img, srl_color_map* cm, srl_vio_state* state, const uint32_t* ids, const float* uv,
                        const double* velocity, size_t n, int32_t n_new_visited, int32_t* result) {
    return vio_run(0, img, cm, state, ids, uv, velocity, n, n_new_visited, nullptr, 0, 0, 0, result);
}

int srl_image_vio_photometric(srl_image* img, srl_color_map* cm, srl_vio_state* state, const uint32_t* ids, const double* velocity,
                              size_t n, int32_t n_new_visited, const uint8_t* bgr, int cols, int rows, size_t pitch, int32_t* result) {
    return vio_run(1, img, cm, state, ids, nullptr, velocity, n, n_new_visited, bgr, cols, rows, pitch, result);
}

int srl_image_covariance(srl_image* img, const double* set, double* get) {
    if (!img) return SRL_BAD_ARG;
    if (set)
        for (int k = 0; k < 121; ++k) img->cov[k] = set[k];
    if (get)
        for (int k = 0; k < 121; ++k) get[k] = img->cov[k];
    return SRL_OK;
}

int srl_image_vio_last_summary(srl_image* img, int32_t which, int32_t* iterations, int32_t* points_used, double* acc_residual) {
    if (!img) return SRL_BAD_ARG;
    if (which != 0 && which != 1) return set_err(img->ctx, SRL_BAD_ARG, "srl_image_vio_last_summary: which is 0 or 1");
    if (!img->vio_ran[which]) return set_err(img->ctx, SRL_BAD_ARG, "srl_image_vio_last_summary: that update has not run yet");
    if (iterations) *iterations = img->vio_iterations[which];
    if (points_used) *points_used = img->vio_points[which];
    if (acc_residual) *acc_residual = img->vio_acc[which];
    return SRL_OK;
}

int srl_image_vio_last_times(srl_image* img, double* esikf_ms, double* photometric_ms) {
    if (!img) return SRL_BAD_ARG;
    srl_ctx* ctx = img->ctx;
    double* outs[2] = {esikf_ms, photometric_ms};
    for (int m = 0; m < 2; ++m) {
        float t = 0.f;
        if (img->vio_timed[m]) {
            SRL_CUDA(ctx, cudaEventSynchronize(img->vio_ev[2 * m + 1]));
            SRL_CUDA(ctx, cudaEventElapsedTime(&t, img->vio_ev[2 * m], img->vio_ev[2 * m + 1]));
        }
        if (outs[m]) *outs[m] = t;
    }
    return SRL_OK;
}

}  // extern "C"
