// srl_points.cu — row N3 of SURVEY.md §8(f): the per-sweep point transforms that sit either side of the scan-matching
// path, one thread per point (reference: src/utility.cpp:203-332).
//
//   srl_distort_frame_by_constant  <- distortFrameByConstant (:203-236): pose slerp/lerp between the first and the last
//                                     IMU state of the sweep, imu_point = R(q_a) (R_il raw + t_il) + t_a
//   srl_distort_frame_by_imu       <- distortFrameByImu (:238-312, "distortion method 1"): constant-acceleration /
//                                     constant-rate propagation inside the IMU interval that holds the point
//   srl_transform_all_imu_point    <- transformAllImuPoint (:320-332): imu_point -> LiDAR frame at the END of the sweep
//   (transformPoint, :314-318, is k_transform / srl_sweep_transform_device in srl_assoc.cu / srl_api.cu)
//
// distortFrameByImu is written as ONE iterator over the points inside a loop over the IMU intervals: a point outside
// the current interval ends the interval and the same point is offered to the next one.  With interval index n_i used
// for point i that is  n_i = min{ n >= n_(i-1) : point i lies in interval n },  and the first point that fits no
// remaining interval stops everything (the rest keep their old imu_point).  IMU timestamps are non-decreasing, so the
// intervals holding a point are a contiguous range [f_i, l_i] and  n_i = max(f_0..f_i)  as long as that is <= l_i:
// an inclusive max-scan plus a min-reduction of the first violating index — exact, and parallel.
//
// Buffers may be host or device pointers (detected per pointer); host buffers are staged through the ctx scratch.
// The quaternion / rotation helpers restate Eigen 3.3.7 (slerp, toRotationMatrix, normalize, product) like the oracle.
#include <cmath>
#include <cstring>
#include <limits>

#include <cub/cub.cuh>

#include "srl_internal.h"

namespace srl {

struct ImuDev {   // the imuState fields the three functions read (include/utility.h)
    double ts;
    double q[4];   // x, y, z, w
    double t[3], v[3], acc[3], gyr[3];
};
static_assert(sizeof(ImuDev) == sizeof(srl_imu_state), "srl_imu_state layout");

struct Q4 { double x, y, z, w; };

__device__ __forceinline__ Q4 q_slerp(const Q4& a, double t, const Q4& b) {   // Eigen QuaternionBase::slerp
    const double one = 1.0 - 2.220446049250313e-16;
    const double d = (a.x * b.x + a.z * b.z) + (a.y * b.y + a.w * b.w);
    const double absD = fabs(d);
    double s0, s1;
    if (absD >= one) { s0 = 1.0 - t; s1 = t; }
    else {
        const double theta = acos(absD);
        const double sinTheta = sin(theta);
        s0 = sin((1.0 - t) * theta) / sinTheta;
        s1 = sin(t * theta) / sinTheta;
    }
    if (d < 0) s1 = -s1;
    return {s0 * a.x + s1 * b.x, s0 * a.y + s1 * b.y, s0 * a.z + s1 * b.z, s0 * a.w + s1 * b.w};
}
__device__ __forceinline__ Q4 q_normalized(const Q4& q) {
    const double n2 = (q.x * q.x + q.z * q.z) + (q.y * q.y + q.w * q.w);
    if (n2 > 0) { const double n = sqrt(n2); return {q.x / n, q.y / n, q.z / n, q.w / n}; }
    return q;
}
__device__ __forceinline__ Q4 q_mul(const Q4& a, const Q4& b) {
    return {a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y, a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z,
            a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x, a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z};
}
__device__ __forceinline__ Q4 q_from_so3(double wx, double wy, double wz) {   // numType::so3ToQuat (include/utility.h:301-324)
    const double n2 = wx * wx + (wy * wy + wz * wz);
    const double theta = sqrt(n2);
    if (theta < 1e-4) return q_normalized({wx / 2.0, wy / 2.0, wz / 2.0, 1.0});
    const double ux = wx / theta, uy = wy / theta, uz = wz / theta;   // Vector3d::normalized()
    const double s = sin(0.5 * theta), c = cos(0.5 * theta);
    return q_normalized({ux * s, uy * s, uz * s, c});
}
__device__ __forceinline__ void mv3(const double* M, double x, double y, double z, double& ox, double& oy, double& oz) {
    ox = M[0] * x + (M[1] * y + M[2] * z);
    oy = M[3] * x + (M[4] * y + M[5] * z);
    oz = M[6] * x + (M[7] * y + M[8] * z);
}
// imu_point = R(q) (R_il raw + t_il) + trans
__device__ __forceinline__ void pose_point(const Q4& q, double tx, double ty, double tz, const double* R_il, const double* t_il,
                                           const double* raw, double* out) {
    const double qq[4] = {q.x, q.y, q.z, q.w};
    double R[9];
    quat_to_rot(qq, R);
    double bx, by, bz, px, py, pz;
    mv3(R_il, raw[0], raw[1], raw[2], bx, by, bz);
    bx += t_il[0]; by += t_il[1]; bz += t_il[2];
    mv3(R, bx, by, bz, px, py, pz);
    out[0] = px + tx; out[1] = py + ty; out[2] = pz + tz;
}

struct PointsConst {
    double R_il[9], t_il[3];
    double time_frame_begin;
    int n_states;
};

__global__ void k_distort_constant(const double* __restrict__ raw, const double* __restrict__ rel, long long n, const ImuDev* __restrict__ st,
                                   const PointsConst c, double* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const ImuDev a = st[0], b = st[c.n_states - 1];
    const double time_frame_end = b.ts;
    double tp = c.time_frame_begin + rel[i] / 1000.0;
    if (fabs(tp - c.time_frame_begin) < 1e-6) tp = c.time_frame_begin + 1e-6;
    if (fabs(tp - time_frame_end) < 1e-6) tp = time_frame_end - 1e-6;
    double alpha = (tp - c.time_frame_begin) / (time_frame_end - c.time_frame_begin);
    if (alpha > 1) alpha = 1;
    if (alpha < 0) alpha = 0;
    const Q4 q = q_slerp({a.q[0], a.q[1], a.q[2], a.q[3]}, alpha, {b.q[0], b.q[1], b.q[2], b.q[3]});
    const double w0 = 1.0 - alpha;
    pose_point(q, w0 * a.t[0] + alpha * b.t[0], w0 * a.t[1] + alpha * b.t[1], w0 * a.t[2] + alpha * b.t[2], c.R_il, c.t_il,
               raw + 3 * i, out + 3 * i);
}

// first / last IMU interval holding each point (the reference's comparisons, literally); f = n_states when none
__global__ void k_imu_intervals(const double* __restrict__ rel, long long n, const ImuDev* __restrict__ st, const PointsConst c,
                                int* __restrict__ f, int* __restrict__ l, int* __restrict__ bad) {
    extern __shared__ double s_ts[];
    for (int k = threadIdx.x; k < c.n_states; k += blockDim.x) s_ts[k] = st[k].ts;
    __syncthreads();
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double tp = c.time_frame_begin + rel[i] / 1000.0;
    int first = c.n_states, last = -1, cnt = 0;
    for (int k = 0; k + 1 < c.n_states; ++k) {
        if (tp > s_ts[k] - 1e-6 && tp < s_ts[k + 1] + 1e-6) { if (first == c.n_states) first = k; last = k; ++cnt; }
    }
    if (cnt > 0 && cnt != last - first + 1) *bad = 1;   // cannot happen with non-decreasing timestamps
    f[i] = first; l[i] = last;
}
struct MaxOp { __device__ __forceinline__ int operator()(int a, int b) const { return a > b ? a : b; } };
__global__ void k_imu_first_violation(const int* __restrict__ m, const int* __restrict__ l, long long n, int n_states, long long* __restrict__ v) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (m[i] >= n_states || m[i] > l[i]) atomicMin(reinterpret_cast<unsigned long long*>(v), (unsigned long long)i);
}
__global__ void k_distort_imu(const double* __restrict__ raw, const double* __restrict__ rel, long long n, const ImuDev* __restrict__ st,
                              const PointsConst c, const int* __restrict__ m, const long long* __restrict__ v, double* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || i >= *v) return;
    const int k = m[i];
    const ImuDev a = st[k], b = st[k + 1];
    double tp = c.time_frame_begin + rel[i] / 1000.0;
    if (fabs(tp - a.ts) < 1e-6) tp = a.ts + 1e-6;
    if (fabs(tp - b.ts) < 1e-6) tp = b.ts - 1e-6;
    const double dt = tp - a.ts;
    const Q4 q = q_normalized(q_mul({a.q[0], a.q[1], a.q[2], a.q[3]}, q_from_so3(b.gyr[0] * dt, b.gyr[1] * dt, b.gyr[2] * dt)));
    const double tx = (a.t[0] + a.v[0] * dt) + ((0.5 * b.acc[0]) * dt) * dt;
    const double ty = (a.t[1] + a.v[1] * dt) + ((0.5 * b.acc[1]) * dt) * dt;
    const double tz = (a.t[2] + a.v[2] * dt) + ((0.5 * b.acc[2]) * dt) * dt;
    pose_point(q, tx, ty, tz, c.R_il, c.t_il, raw + 3 * i, out + 3 * i);
}

struct EndConst { double Rinv[9], tinv[3], Rt[9], off[3]; };
__global__ void k_imu_to_lidar_end(const double* __restrict__ imu, long long n, const EndConst c, double* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double ax, ay, az, bx, by, bz;
    mv3(c.Rinv, imu[3 * i], imu[3 * i + 1], imu[3 * i + 2], ax, ay, az);
    ax += c.tinv[0]; ay += c.tinv[1]; az += c.tinv[2];
    mv3(c.Rt, ax, ay, az, bx, by, bz);
    out[3 * i] = bx - c.off[0]; out[3 * i + 1] = by - c.off[1]; out[3 * i + 2] = bz - c.off[2];
}

}  // namespace srl

using namespace srl;

static int check_common(srl_ctx* ctx, const void* a, const void* b, const srl_imu_state* st, size_t n_states, const double* R_il,
                        const double* t_il, const void* out) {
    if (!ctx) return SRL_BAD_ARG;
    if (!a || !b || !st || !R_il || !t_il || !out) return set_err(ctx, SRL_BAD_ARG, "null pointer");
    if (n_states < 1) return set_err(ctx, SRL_BAD_ARG, "at least one IMU state is needed");
    return SRL_OK;
}

extern "C" {

int srl_distort_frame_by_constant(srl_ctx* ctx, const double* raw_xyz, const double* relative_time_ms, size_t n,
                                  const srl_imu_state* states, size_t n_states, double time_frame_begin, const double R_il[9],
                                  const double t_il[3], double* imu_xyz) {
    int rc = check_common(ctx, raw_xyz, relative_time_ms, states, n_states, R_il, t_il, imu_xyz);
    if (rc != SRL_OK) return rc;
    if (n == 0) return SRL_OK;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    Staged<const double> raw(raw_xyz), rel(relative_time_ms);
    Staged<double> out(imu_xyz);
    ImuDev* st = nullptr;
    rc = carve_scratch(ctx, [&](Carve& c) { st = c.take<ImuDev>(n_states); raw.place(c, n * 3); rel.place(c, n); out.place(c, n * 3); });
    if (rc != SRL_OK) return rc;
    SRL_CUDA(ctx, cudaMemcpyAsync(st, states, n_states * sizeof(ImuDev), cudaMemcpyHostToDevice, ctx->stream));
    if ((rc = raw.upload(ctx, n * 3)) != SRL_OK || (rc = rel.upload(ctx, n)) != SRL_OK) return rc;
    PointsConst c;
    std::memcpy(c.R_il, R_il, sizeof(c.R_il)); std::memcpy(c.t_il, t_il, sizeof(c.t_il));
    c.time_frame_begin = time_frame_begin; c.n_states = (int)n_states;
    const int T = 256;
    k_distort_constant<<<(unsigned)((n + T - 1) / T), T, 0, ctx->stream>>>(raw.d, rel.d, (long long)n, st, c, out.d);
    SRL_CUDA(ctx, cudaGetLastError());
    ctx->launches += 1;
    if ((rc = out.hand_back(ctx, n * 3)) != SRL_OK) return rc;
    SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return SRL_OK;
}

int srl_distort_frame_by_imu(srl_ctx* ctx, const double* raw_xyz, const double* relative_time_ms, size_t n,
                             const srl_imu_state* states, size_t n_states, double time_frame_begin, const double R_il[9],
                             const double t_il[3], double* imu_xyz, int64_t* n_written) {
    int rc = check_common(ctx, raw_xyz, relative_time_ms, states, n_states, R_il, t_il, imu_xyz);
    if (rc != SRL_OK) return rc;
    if (n_written) *n_written = 0;
    if (n == 0 || n_states < 2) return SRL_OK;   // no interval: the reference's outer loop does not run
    for (size_t k = 0; k + 1 < n_states; ++k)
        if (!(states[k].timestamp <= states[k + 1].timestamp)) return set_err(ctx, SRL_BAD_ARG, "IMU timestamps must be non-decreasing");
    if (n_states > 4096) return set_err(ctx, SRL_BAD_ARG, "at most 4096 IMU states per sweep");
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    size_t tmp = 0;
    cub::DeviceScan::InclusiveScan(nullptr, tmp, (int*)nullptr, (int*)nullptr, MaxOp(), (int)n, ctx->stream);
    Staged<const double> raw(raw_xyz), rel(relative_time_ms);
    Staged<double> out(imu_xyz);   // in/out: points the iterator never reaches keep what the caller had
    ImuDev* st = nullptr;
    int *f = nullptr, *l = nullptr, *m = nullptr;
    long long* v = nullptr;   // [0] first violating point, [1] contiguity check
    void* cub_tmp = nullptr;
    rc = carve_scratch(ctx, [&](Carve& c) {
        st = c.take<ImuDev>(n_states);
        raw.place(c, n * 3); rel.place(c, n); out.place(c, n * 3);
        f = c.take<int>(n); l = c.take<int>(n); m = c.take<int>(n);
        v = c.take<long long>(2);
        cub_tmp = c.take<char>(tmp);
    });
    if (rc != SRL_OK) return rc;
    SRL_CUDA(ctx, cudaMemcpyAsync(st, states, n_states * sizeof(ImuDev), cudaMemcpyHostToDevice, ctx->stream));
    if ((rc = raw.upload(ctx, n * 3)) != SRL_OK || (rc = rel.upload(ctx, n)) != SRL_OK || (rc = out.upload(ctx, n * 3)) != SRL_OK) return rc;
    PointsConst c;
    std::memcpy(c.R_il, R_il, sizeof(c.R_il)); std::memcpy(c.t_il, t_il, sizeof(c.t_il));
    c.time_frame_begin = time_frame_begin; c.n_states = (int)n_states;
    const long long init[2] = {(long long)n, 0};
    SRL_CUDA(ctx, cudaMemcpyAsync(v, init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream));
    const int T = 256;
    const unsigned G = (unsigned)((n + T - 1) / T);
    k_imu_intervals<<<G, T, n_states * sizeof(double), ctx->stream>>>(rel.d, (long long)n, st, c, f, l, reinterpret_cast<int*>(v + 1));
    SRL_CUDA(ctx, cudaGetLastError());
    SRL_CUDA(ctx, cub::DeviceScan::InclusiveScan(cub_tmp, tmp, f, m, MaxOp(), (int)n, ctx->stream));
    k_imu_first_violation<<<G, T, 0, ctx->stream>>>(m, l, (long long)n, (int)n_states, v);
    k_distort_imu<<<G, T, 0, ctx->stream>>>(raw.d, rel.d, (long long)n, st, c, m, v, out.d);
    SRL_CUDA(ctx, cudaGetLastError());
    ctx->launches += 4;
    long long hv[2] = {0, 0};
    SRL_CUDA(ctx, cudaMemcpyAsync(hv, v, sizeof(hv), cudaMemcpyDeviceToHost, ctx->stream));
    if ((rc = out.hand_back(ctx, n * 3)) != SRL_OK) return rc;
    SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if ((int)hv[1] != 0) return set_err(ctx, SRL_BAD_ARG, "IMU intervals holding a point are not contiguous");
    if (n_written) *n_written = hv[0];
    return SRL_OK;
}

int srl_transform_all_imu_point(srl_ctx* ctx, const double* imu_xyz, size_t n, const srl_imu_state* last, const double R_il[9],
                                const double t_il[3], double* raw_out) {
    if (!ctx) return SRL_BAD_ARG;
    if (!imu_xyz || !last || !R_il || !t_il || !raw_out) return set_err(ctx, SRL_BAD_ARG, "null pointer");
    if (n == 0) return SRL_OK;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    // the four per-sweep constants of :322-323,329 on the host, same operation order as the oracle
    EndConst c;
    const double* q = last->quat;
    const double n2 = (q[0] * q[0] + q[2] * q[2]) + (q[1] * q[1] + q[3] * q[3]);
    double qi[4] = {0, 0, 0, 0};
    if (n2 > 0) { qi[0] = -q[0] / n2; qi[1] = -q[1] / n2; qi[2] = -q[2] / n2; qi[3] = q[3] / n2; }   // Quaternion::inverse()
    quat_to_rot(qi, c.Rinv);
    for (int r = 0; r < 3; ++r)
        c.tinv[r] = -(c.Rinv[3 * r] * last->trans[0] + (c.Rinv[3 * r + 1] * last->trans[1] + c.Rinv[3 * r + 2] * last->trans[2]));
    for (int r = 0; r < 3; ++r) for (int k = 0; k < 3; ++k) c.Rt[3 * r + k] = R_il[3 * k + r];
    for (int r = 0; r < 3; ++r) c.off[r] = c.Rt[3 * r] * t_il[0] + (c.Rt[3 * r + 1] * t_il[1] + c.Rt[3 * r + 2] * t_il[2]);
    Staged<const double> in(imu_xyz);
    Staged<double> out(raw_out);
    int rc = carve_scratch(ctx, [&](Carve& s) { in.place(s, n * 3); out.place(s, n * 3); });
    if (rc != SRL_OK || (rc = in.upload(ctx, n * 3)) != SRL_OK) return rc;
    const int T = 256;
    k_imu_to_lidar_end<<<(unsigned)((n + T - 1) / T), T, 0, ctx->stream>>>(in.d, (long long)n, c, out.d);
    SRL_CUDA(ctx, cudaGetLastError());
    ctx->launches += 1;
    if ((rc = out.hand_back(ctx, n * 3)) != SRL_OK) return rc;
    SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return SRL_OK;
}

}  // extern "C"
