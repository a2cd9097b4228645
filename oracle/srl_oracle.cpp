/*
 * srl_oracle.cpp — CPU ORACLE for SR-LIVO's LIO scan-matching hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Imported/linked solely by tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs.  The product (sr_livo_b200/)
 * never includes, links or calls anything in this directory.
 *
 * PARITY (see srl_oracle.h): the reference has no tests/golden vectors for this path; this
 * file restates the algorithm line by line and is pinned against the reference's own sources
 * compiled where they lie (oracle/_ref/libsrl_reference.so, tests/test_reference_pin.py) and by
 * self-checks.  PARITY UNPINNED only for the arithmetic inside Eigen / OpenCV calls.
 *
 * What is restated, with the reference location each piece follows
 * (paths relative to /root/reference):
 *   voxel / hash / voxelBlock / rgbPoint      include/cloudMap.h:51-86,124-184, src/cloudMap.cpp:5-29
 *   addPointToMap / addPointsToMap            src/lioOptimization.cpp:400-446,520-554
 *   searchNeighbors (+heap types)             src/optimize.cpp:355-426
 *   computeNeighborhoodDistribution           src/optimize.cpp:316-353
 *   buildPlaneResiduals                       src/optimize.cpp:18-131
 *   updateIEKF                                src/optimize.cpp:133-314
 *   eskfEstimator::observe                    src/eskfEstimator.cpp:219-230
 *   numType::{skewSymmetric,derivativeS2,normalizeR,rotationToSo3,so3ToRotation,
 *             so3ToQuat,quatToSo3}            include/utility.h:194-330
 *   AngularDistance(so3)                      src/utility.cpp:146-153
 *
 * Third-party arithmetic that is NOT under /root/reference and is restated from the
 * library's published algorithm: Eigen 3.3.7 (README.md:48,64 "tested 3.3.7";
 * CMakeLists.txt:49 find_package(Eigen3), not pinned):
 *   Quaternion::toRotationMatrix / normalized / operator* / inverse / ctor-from-matrix
 *   fixed-size 3-term reductions  -> a0 + (a1 + a2)   (redux_novec_unroller halves)
 *   4-term squaredNorm (SSE2 packets of 2) -> (a0 + a2) + (a1 + a3)
 *   SelfAdjointEigenSolver<Matrix3d>::compute: scale by max|coef|, closed-form 3x3
 *     Householder tridiagonalisation, implicit symmetric QR with Wilkinson shift,
 *     ascending selection sort
 *   Matrix<double,17,17>::inverse() -> PartialPivLU
 * libstdc++ std::priority_queue and libm exp/pow/sqrt/acos are used directly.
 *
 * Hash container: the reference's vendored tessil robin-map 0.6.3
 * (thirdLibrary/tessil-src/include/tsl/robin_map.h) when built with -DSRL_ORACLE_TSL
 * and -I<that include dir> (recipe: oracle/Makefile -> oracle/_ref/), otherwise
 * std::unordered_map with the same std::hash<voxel> (only iteration order differs).
 */
#include "srl_oracle.h"

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <limits>
#include <queue>
#include <thread>
#include <tuple>
#include <vector>

#include <tr1/unordered_map>

#ifdef SRL_ORACLE_TSL
#include <tsl/robin_map.h>
#else
#include <unordered_map>
#endif
#include <array>
#include <unordered_map>

namespace {

// ----------------------------------------------------------------------------------
// tiny fixed-size algebra with Eigen 3.3 evaluation orders
// ----------------------------------------------------------------------------------
struct Vec3 {
    double v[3];
    double& operator[](int i) { return v[i]; }
    double operator[](int i) const { return v[i]; }
};
struct Mat3 { double m[9]; /* row-major */
    double& operator()(int r, int c) { return m[r * 3 + c]; }
    double operator()(int r, int c) const { return m[r * 3 + c]; }
};
struct Quat { double x, y, z, w; };

inline Vec3 vsub(const Vec3& a, const Vec3& b) { return {{a[0] - b[0], a[1] - b[1], a[2] - b[2]}}; }
inline Vec3 vadd(const Vec3& a, const Vec3& b) { return {{a[0] + b[0], a[1] + b[1], a[2] + b[2]}}; }
inline Vec3 vscale(const Vec3& a, double s) { return {{a[0] * s, a[1] * s, a[2] * s}}; }
inline Vec3 vdiv(const Vec3& a, double s) { return {{a[0] / s, a[1] / s, a[2] / s}}; }
// Eigen redux for 3 coefficients: c0 + (c1 + c2)
inline double dot3(const Vec3& a, const Vec3& b) { return a[0] * b[0] + (a[1] * b[1] + a[2] * b[2]); }
inline double sqnorm3(const Vec3& a) { return dot3(a, a); }
inline double norm3(const Vec3& a) { return std::sqrt(sqnorm3(a)); }
inline Vec3 normalized3(const Vec3& a) {   // MatrixBase::normalized(): n = squaredNorm; n>0 ? a/sqrt(n) : a
    double n2 = sqnorm3(a);
    if (n2 > 0.0) return vdiv(a, std::sqrt(n2));
    return a;
}
inline Vec3 cross3(const Vec3& a, const Vec3& b) {
    return {{a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]}};
}
inline Vec3 matvec(const Mat3& M, const Vec3& x) {
    Vec3 r;
    for (int i = 0; i < 3; ++i) r[i] = M(i, 0) * x[0] + (M(i, 1) * x[1] + M(i, 2) * x[2]);
    return r;
}
inline Mat3 matmul(const Mat3& A, const Mat3& B) {
    Mat3 C;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) C(i, j) = A(i, 0) * B(0, j) + (A(i, 1) * B(1, j) + A(i, 2) * B(2, j));
    return C;
}
inline Mat3 transpose(const Mat3& A) {
    Mat3 T;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) T(i, j) = A(j, i);
    return T;
}
inline Mat3 identity3() { return {{1, 0, 0, 0, 1, 0, 0, 0, 1}}; }
// numType::skewSymmetric (include/utility.h:205-213)
inline Mat3 skew(const Vec3& a) { return {{0.0, -a[2], a[1], a[2], 0.0, -a[0], -a[1], a[0], 0.0}}; }

// Eigen Quaternion::toRotationMatrix (Geometry/Quaternion.h)
inline Mat3 quat_to_rot(const Quat& q) {
    const double tx = 2.0 * q.x, ty = 2.0 * q.y, tz = 2.0 * q.z;
    const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
    const double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
    const double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
    Mat3 R;
    R(0, 0) = 1.0 - (tyy + tzz); R(0, 1) = txy - twz;          R(0, 2) = txz + twy;
    R(1, 0) = txy + twz;          R(1, 1) = 1.0 - (txx + tzz); R(1, 2) = tyz - twx;
    R(2, 0) = txz - twy;          R(2, 1) = tyz + twx;          R(2, 2) = 1.0 - (txx + tyy);
    return R;
}
// coeffs() = (x,y,z,w); SSE2 packet reduction order (x^2+z^2)+(y^2+w^2)
inline double quat_sqnorm(const Quat& q) { return (q.x * q.x + q.z * q.z) + (q.y * q.y + q.w * q.w); }
inline Quat quat_normalized(const Quat& q) {
    double n2 = quat_sqnorm(q);
    if (n2 > 0.0) { double n = std::sqrt(n2); return {q.x / n, q.y / n, q.z / n, q.w / n}; }
    return q;
}
inline Quat quat_mul(const Quat& a, const Quat& b) {
    return {a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
            a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z,
            a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x,
            a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z};
}
inline Quat quat_inverse(const Quat& q) {   // conjugate / squaredNorm
    double n2 = quat_sqnorm(q);
    if (n2 > 0.0) return {-q.x / n2, -q.y / n2, -q.z / n2, q.w / n2};
    return {0, 0, 0, 0};
}
// Eigen quaternionbase_assign_impl<Matrix3>: Ken Shoemake's method
inline Quat quat_from_rot(const Mat3& m) {
    double q[4];  // x,y,z,w
    double t = m(0, 0) + m(1, 1) + m(2, 2);
    if (t > 0.0) {
        t = std::sqrt(t + 1.0);
        q[3] = 0.5 * t;
        t = 0.5 / t;
        q[0] = (m(2, 1) - m(1, 2)) * t;
        q[1] = (m(0, 2) - m(2, 0)) * t;
        q[2] = (m(1, 0) - m(0, 1)) * t;
    } else {
        int i = 0;
        if (m(1, 1) > m(0, 0)) i = 1;
        if (m(2, 2) > m(i, i)) i = 2;
        int j = (i + 1) % 3, k = (j + 1) % 3;
        t = std::sqrt(m(i, i) - m(j, j) - m(k, k) + 1.0);
        q[i] = 0.5 * t;
        t = 0.5 / t;
        q[3] = (m(k, j) - m(j, k)) * t;
        q[j] = (m(j, i) + m(i, j)) * t;
        q[k] = (m(k, i) + m(i, k)) * t;
    }
    return {q[0], q[1], q[2], q[3]};
}

const double kThetaThreshold = 0.0001;  // include/utility.h:27

// numType::normalizeR (include/utility.h:194-203)
inline Mat3 normalizeR(const Mat3& R) { return quat_to_rot(quat_normalized(quat_from_rot(R))); }
// numType::rotationToSo3 (include/utility.h:267-280) — acos NOT clamped, as in the reference
inline Vec3 rotationToSo3(const Mat3& R_in) {
    Mat3 R = normalizeR(R_in);
    double theta = std::acos((R(0, 0) + R(1, 1) + R(2, 2) - 1.0) / 2.0);
    Vec3 a = {{R(2, 1) - R(1, 2), R(0, 2) - R(2, 0), R(1, 0) - R(0, 1)}};
    if (theta < kThetaThreshold) return vdiv(a, 2.0);
    return vdiv(vscale(a, theta), 2.0 * std::sin(theta));
}
// numType::so3ToRotation (include/utility.h:282-299)
inline Mat3 so3ToRotation(const Vec3& so3) {
    double theta = norm3(so3);
    Mat3 I = identity3(), R;
    if (theta < kThetaThreshold) {
        Mat3 U = skew(so3), UU = matmul(U, U);
        for (int i = 0; i < 9; ++i) R.m[i] = I.m[i] + U.m[i] + 0.5 * UU.m[i];
    } else {
        Mat3 U = skew(normalized3(so3)), UU = matmul(U, U);
        double s = std::sin(theta), c1 = 1.0 - std::cos(theta);
        for (int i = 0; i < 9; ++i) R.m[i] = I.m[i] + s * U.m[i] + c1 * UU.m[i];
    }
    return R;
}
// numType::so3ToQuat (include/utility.h:301-324)
inline Quat so3ToQuat(const Vec3& so3) {
    double theta = norm3(so3);
    if (theta < kThetaThreshold) {
        Vec3 h = vdiv(so3, 2.0);
        return quat_normalized({h[0], h[1], h[2], 1.0});
    }
    Vec3 u = normalized3(so3);
    double s = std::sin(0.5 * theta), c = std::cos(0.5 * theta);
    return quat_normalized({u[0] * s, u[1] * s, u[2] * s, c});
}
// numType::quatToSo3 (include/utility.h:326-330)
inline Vec3 quatToSo3(const Quat& q) { return rotationToSo3(quat_to_rot(q)); }
// numType::derivativeS2 (include/utility.h:215-235): 3x2, row-major [r*2+c]
inline void derivativeS2(const Vec3& g_in, double B[6]) {
    Vec3 g = normalized3(g_in);   // g.normalize(): same n>0 guard
    B[0] = 1.0 - g[0] * g[0] / (1.0 + g[2]);
    B[1] = -g[0] * g[1] / (1.0 + g[2]);
    B[2] = B[1];
    B[3] = 1.0 - g[1] * g[1] / (1.0 + g[2]);
    B[4] = -g[0];
    B[5] = -g[1];
}
// AngularDistance(const Vector3d&) (src/utility.cpp:146-153)
inline double AngularDistance(const Vec3& d_so3) {
    Mat3 R = so3ToRotation(d_so3);
    double n = (R(0, 0) + R(1, 1) + R(2, 2) - 1.0) / 2.0;
    return std::acos(n) * 180.0 / M_PI;
}

// ----------------------------------------------------------------------------------
// Eigen::SelfAdjointEigenSolver<Matrix3d>::compute  (Eigen 3.3.7, iterative path)
// ----------------------------------------------------------------------------------
struct Givens { double c, s; };
inline Givens makeGivens(double p, double q) {   // Jacobi/Jacobi.h, real case
    Givens g;
    if (q == 0.0) { g.c = p < 0.0 ? -1.0 : 1.0; g.s = 0.0; }
    else if (p == 0.0) { g.c = 0.0; g.s = q < 0.0 ? 1.0 : -1.0; }
    else if (std::abs(p) > std::abs(q)) {
        double t = q / p, u = std::sqrt(1.0 + t * t);
        if (p < 0.0) u = -u;
        g.c = 1.0 / u; g.s = -t * g.c;
    } else {
        double t = p / q, u = std::sqrt(1.0 + t * t);
        if (q < 0.0) u = -u;
        g.s = -1.0 / u; g.c = -t * g.s;
    }
    return g;
}

// evals ascending, evecs column k = eigenvector k, stored row-major evecs[r*3+k]
void eig3_sym(const double S[9], double evals[3], double evecs[9]) {
    const int n = 3;
    // lower triangle of the input, scaled to [-1,1]
    double mat[3][3];
    double scale = 0.0;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c <= r; ++c) scale = std::max(scale, std::abs(S[r * 3 + c]));
    if (scale == 0.0) scale = 1.0;
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) mat[r][c] = (c <= r) ? S[r * 3 + c] / scale : 0.0;

    // tridiagonalization_inplace_selector<MatrixType,3,false>::run
    double diag[3], subdiag[2], Q[3][3];
    const double tol = std::numeric_limits<double>::min();
    diag[0] = mat[0][0];
    double v1norm2 = mat[2][0] * mat[2][0];
    if (v1norm2 <= tol) {
        diag[1] = mat[1][1]; diag[2] = mat[2][2];
        subdiag[0] = mat[1][0]; subdiag[1] = mat[2][1];
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) Q[r][c] = (r == c) ? 1.0 : 0.0;
    } else {
        double beta = std::sqrt(mat[1][0] * mat[1][0] + v1norm2);
        double invBeta = 1.0 / beta;
        double m01 = mat[1][0] * invBeta;
        double m02 = mat[2][0] * invBeta;
        double q = 2.0 * m01 * mat[2][1] + m02 * (mat[2][2] - mat[1][1]);
        diag[1] = mat[1][1] + m02 * q;
        diag[2] = mat[2][2] - m02 * q;
        subdiag[0] = beta;
        subdiag[1] = mat[2][1] - m01 * q;
        Q[0][0] = 1; Q[0][1] = 0;   Q[0][2] = 0;
        Q[1][0] = 0; Q[1][1] = m01; Q[1][2] = m02;
        Q[2][0] = 0; Q[2][1] = m02; Q[2][2] = -m01;
    }

    // computeFromTridiagonal_impl
    const double considerAsZero = std::numeric_limits<double>::min();
    const double precision = 2.0 * std::numeric_limits<double>::epsilon();
    const int maxIterations = 30;
    int end = n - 1, start = 0, iter = 0;
    while (end > 0) {
        for (int i = start; i < end; ++i)
            if (std::abs(subdiag[i]) <= (std::abs(diag[i]) + std::abs(diag[i + 1])) * precision ||
                std::abs(subdiag[i]) <= considerAsZero)
                subdiag[i] = 0.0;
        while (end > 0 && subdiag[end - 1] == 0.0) end--;
        if (end <= 0) break;
        iter++;
        if (iter > maxIterations * n) break;
        start = end - 1;
        while (start > 0 && subdiag[start - 1] != 0.0) start--;

        // tridiagonal_qr_step
        double td = (diag[end - 1] - diag[end]) * 0.5;
        double e = subdiag[end - 1];
        double mu = diag[end];
        if (td == 0.0) {
            mu -= std::abs(e);
        } else if (e != 0.0) {
            const double e2 = e * e;
            const double h = std::hypot(td, e);
            if (e2 == 0.0) mu -= e / ((td + (td > 0.0 ? h : -h)) / e);
            else mu -= e2 / (td + (td > 0.0 ? h : -h));
        }
        double x = diag[start] - mu;
        double z = subdiag[start];
        for (int k = start; k < end && z != 0.0; ++k) {
            Givens rot = makeGivens(x, z);
            double sdk = rot.s * diag[k] + rot.c * subdiag[k];
            double dkp1 = rot.s * subdiag[k] + rot.c * diag[k + 1];
            diag[k] = rot.c * (rot.c * diag[k] - rot.s * subdiag[k]) -
                      rot.s * (rot.c * subdiag[k] - rot.s * diag[k + 1]);
            diag[k + 1] = rot.s * sdk + rot.c * dkp1;
            subdiag[k] = rot.c * sdk - rot.s * dkp1;
            if (k > start) subdiag[k - 1] = rot.c * subdiag[k - 1] - rot.s * z;
            x = subdiag[k];
            if (k < end - 1) {
                z = -rot.s * subdiag[k + 1];
                subdiag[k + 1] = rot.c * subdiag[k + 1];
            }
            // Q = Q * G : applyOnTheRight(k, k+1, rot) -> x' = c x - s y ; y' = s x + c y
            for (int r = 0; r < 3; ++r) {
                double xi = Q[r][k], yi = Q[r][k + 1];
                Q[r][k] = rot.c * xi - rot.s * yi;
                Q[r][k + 1] = rot.s * xi + rot.c * yi;
            }
        }
    }
    // ascending selection sort with column swaps
    for (int i = 0; i < n - 1; ++i) {
        int k = 0;
        double mn = diag[i];
        for (int j = 1; j < n - i; ++j)
            if (diag[i + j] < mn) { mn = diag[i + j]; k = j; }
        if (k > 0) {
            std::swap(diag[i], diag[k + i]);
            for (int r = 0; r < 3; ++r) std::swap(Q[r][i], Q[r][k + i]);
        }
    }
    for (int i = 0; i < 3; ++i) evals[i] = diag[i] * scale;
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) evecs[r * 3 + c] = Q[r][c];
}

// ----------------------------------------------------------------------------------
// small dense helpers for the 17-dim ESIKF algebra (row-major)
// ----------------------------------------------------------------------------------
const int NS = 17;

// Eigen Matrix<double,17,17>::inverse(): PartialPivLU then solve for identity.
bool mat_inverse(const double* A, double* Ainv, int n) {
    std::vector<double> lu(A, A + n * n);
    std::vector<int> perm(n);
    for (int i = 0; i < n; ++i) perm[i] = i;
    for (int k = 0; k < n; ++k) {
        int piv = k;
        double best = std::abs(lu[k * n + k]);
        for (int r = k + 1; r < n; ++r)
            if (std::abs(lu[r * n + k]) > best) { best = std::abs(lu[r * n + k]); piv = r; }
        if (best == 0.0) return false;
        if (piv != k) {
            for (int c = 0; c < n; ++c) std::swap(lu[k * n + c], lu[piv * n + c]);
            std::swap(perm[k], perm[piv]);
        }
        for (int r = k + 1; r < n; ++r) {
            lu[r * n + k] /= lu[k * n + k];
            double f = lu[r * n + k];
            for (int c = k + 1; c < n; ++c) lu[r * n + c] -= f * lu[k * n + c];
        }
    }
    for (int col = 0; col < n; ++col) {
        std::vector<double> y(n);
        for (int r = 0; r < n; ++r) {
            double s = (perm[r] == col) ? 1.0 : 0.0;
            for (int c = 0; c < r; ++c) s -= lu[r * n + c] * y[c];
            y[r] = s;
        }
        for (int r = n - 1; r >= 0; --r) {
            double s = y[r];
            for (int c = r + 1; c < n; ++c) s -= lu[r * n + c] * Ainv[c * n + col];
            Ainv[r * n + col] = s / lu[r * n + r];
        }
    }
    return true;
}

// ----------------------------------------------------------------------------------
// map types (include/cloudMap.h)
// ----------------------------------------------------------------------------------
struct voxel {   // include/cloudMap.h:124-145
    voxel() = default;
    voxel(short x_, short y_, short z_) : x(x_), y(y_), z(z_) {}
    bool operator==(const voxel& o) const { return x == o.x && y == o.y && z == o.z; }
    short x, y, z;
};

struct voxel_hash {   // include/cloudMap.h:173-184 (std::hash<voxel>), additive primes in size_t
    std::size_t operator()(const voxel& vox) const {
        const std::size_t kP1 = 73856093, kP2 = 19349669, kP3 = 83492791;
        return vox.x * kP1 + vox.y * kP2 + vox.z * kP3;
    }
};

// rgbPoint: same 80-byte record as the reference (include/cloudMap.h:51-86) so the CPU
// timing sees the same cache footprint; only `position` is on the hot path.
struct rgbPoint {
    float position[3];
    short rgb[3];
    float cov_rgb[3];
    double observe_distance;
    double last_observe_time;
    int point_index;
    short N_rgb;
    short is_out_lier_count;
    alignas(16) double image_velocity[2];

    explicit rgbPoint(const Vec3& p) {   // src/cloudMap.cpp:5-19: position_.cast<float>(), reset()
        position[0] = (float)p[0]; position[1] = (float)p[1]; position[2] = (float)p[2];
        for (int i = 0; i < 3; ++i) { rgb[i] = 0; cov_rgb[i] = 0.f; }
        N_rgb = 0; is_out_lier_count = 0; observe_distance = 0; last_observe_time = 0;
        point_index = 0; image_velocity[0] = image_velocity[1] = 0;
    }
    Vec3 getPosition() const {            // src/cloudMap.cpp:26-29: position.cast<double>()
        return {{(double)position[0], (double)position[1], (double)position[2]}};
    }
};
static_assert(sizeof(rgbPoint) == 80, "rgbPoint must match the reference's 80-byte record");

struct voxelBlock {   // include/cloudMap.h:147-169
    explicit voxelBlock(int num_points_ = 20) : num_points(num_points_) { points.reserve(num_points_); }
    std::vector<rgbPoint> points;
    double last_visited_time = 0.0;
    bool is_recent = false;
    bool IsFull() const { return num_points == (int)points.size(); }
    void AddPoint(const rgbPoint& p) { points.push_back(p); }
    int NumPoints() const { return (int)points.size(); }
    int num_points;
};

#ifdef SRL_ORACLE_TSL
typedef tsl::robin_map<voxel, voxelBlock, voxel_hash> voxelHashMap;   // include/cloudMap.h:171
#define MAP_VALUE(it) ((it).value())
static const char* kBackend = "tsl::robin_map 0.6.3 (reference vendored header)";
#else
typedef std::unordered_map<voxel, voxelBlock, voxel_hash> voxelHashMap;
#define MAP_VALUE(it) ((it)->second)
static const char* kBackend = "std::unordered_map (fallback, same std::hash<voxel>)";
#endif

// lioOptimization::addPointToMap (src/lioOptimization.cpp:400-446); returns 1 if the point was stored
inline int addPointToMap(voxelHashMap& map, rgbPoint& point, double voxel_size, int max_num_points_in_voxel,
                         double min_distance_points, int min_num_points) {
    short kx = static_cast<short>(point.getPosition()[0] / voxel_size);
    short ky = static_cast<short>(point.getPosition()[1] / voxel_size);
    short kz = static_cast<short>(point.getPosition()[2] / voxel_size);

    auto search = map.find(voxel(kx, ky, kz));
    if (search != map.end()) {
        voxelBlock& voxel_block = MAP_VALUE(search);
        if (!voxel_block.IsFull()) {
            double sq_dist_min_to_points = 10 * voxel_size * voxel_size;
            for (int i = 0; i < voxel_block.NumPoints(); ++i) {
                auto& _point = voxel_block.points[i];
                double sq_dist = sqnorm3(vsub(_point.getPosition(), point.getPosition()));
                if (sq_dist < sq_dist_min_to_points) sq_dist_min_to_points = sq_dist;
            }
            if (sq_dist_min_to_points > (min_distance_points * min_distance_points)) {
                if (min_num_points <= 0 || voxel_block.NumPoints() >= min_num_points) {
                    voxel_block.AddPoint(point);
                    return 1;
                }
            }
        }
    } else {
        if (min_num_points <= 0) {
            voxelBlock voxel_block(max_num_points_in_voxel);
            voxel_block.AddPoint(point);
            map[voxel(kx, ky, kz)] = std::move(voxel_block);
            return 1;
        }
    }
    return 0;
}

// ----------------------------------------------------------------------------------
// searchNeighbors (src/optimize.cpp:355-426)
// ----------------------------------------------------------------------------------
// pair_distance_t = tuple<double, Vector3d, voxel> (40 B); the int16 slot that is padding in the
// reference's voxel carries the index-in-block here, so the element stays 40 B.
struct pair_distance_t {
    double distance;
    Vec3 point;
    short vx, vy, vz, idx;
};
static_assert(sizeof(pair_distance_t) == 40, "heap element must stay 40 bytes");
struct comparator {
    bool operator()(const pair_distance_t& l, const pair_distance_t& r) const { return l.distance < r.distance; }
};
typedef std::priority_queue<pair_distance_t, std::vector<pair_distance_t>, comparator> priority_queue_t;

struct SearchDiag {
    int64_t candidates = 0;
    int64_t probes_hit = 0;
    double d_next = std::numeric_limits<double>::infinity();   // (K+1)-th smallest distance
};

template <bool DIAG>
std::vector<pair_distance_t> searchNeighbors(const voxelHashMap& map, const Vec3& point, int nb_voxels_visited,
                                             double size_voxel_map, int max_num_neighbors,
                                             int threshold_voxel_capacity, SearchDiag& diag) {
    short kx = static_cast<short>(point[0] / size_voxel_map);
    short ky = static_cast<short>(point[1] / size_voxel_map);
    short kz = static_cast<short>(point[2] / size_voxel_map);

    priority_queue_t priority_queue;
    voxel voxel_temp(kx, ky, kz);
    for (short kxx = kx - nb_voxels_visited; kxx < kx + nb_voxels_visited + 1; ++kxx) {
        for (short kyy = ky - nb_voxels_visited; kyy < ky + nb_voxels_visited + 1; ++kyy) {
            for (short kzz = kz - nb_voxels_visited; kzz < kz + nb_voxels_visited + 1; ++kzz) {
                voxel_temp.x = kxx; voxel_temp.y = kyy; voxel_temp.z = kzz;
                auto search = map.find(voxel_temp);
                if (search != map.end()) {
                    const voxelBlock& voxel_block = MAP_VALUE(search);
                    diag.probes_hit++;
                    if (voxel_block.NumPoints() < threshold_voxel_capacity) continue;
                    diag.candidates += voxel_block.NumPoints();
                    for (int i = 0; i < voxel_block.NumPoints(); ++i) {
                        const rgbPoint& neighbor = voxel_block.points[i];
                        Vec3 neighbor_point = neighbor.getPosition();
                        double distance = norm3(vsub(neighbor_point, point));
                        if ((int)priority_queue.size() == max_num_neighbors) {
                            if (distance < priority_queue.top().distance) {
                                if (DIAG) diag.d_next = std::min(diag.d_next, priority_queue.top().distance);
                                priority_queue.pop();
                                priority_queue.push({distance, neighbor_point, kxx, kyy, kzz, (short)i});
                            } else if (DIAG) {
                                diag.d_next = std::min(diag.d_next, distance);
                            }
                        } else {
                            priority_queue.push({distance, neighbor_point, kxx, kyy, kzz, (short)i});
                        }
                    }
                }
            }
        }
    }
    auto size = priority_queue.size();
    std::vector<pair_distance_t> closest_neighbors(size);
    for (size_t i = 0; i < size; ++i) {
        closest_neighbors[size - 1 - i] = priority_queue.top();
        priority_queue.pop();
    }
    return closest_neighbors;
}

// ----------------------------------------------------------------------------------
// computeNeighborhoodDistribution (src/optimize.cpp:316-353)
// ----------------------------------------------------------------------------------
struct Neighborhood {
    Vec3 center, normal;
    double covariance[9];
    double a2D;
    bool nan_planarity;
};

Neighborhood computeNeighborhoodDistribution(const std::vector<Vec3>& points) {
    Neighborhood nh;
    Vec3 barycenter = {{0, 0, 0}};
    for (auto& p : points) barycenter = vadd(barycenter, p);
    barycenter = vdiv(barycenter, (double)points.size());
    nh.center = barycenter;

    double C[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (auto& p : points)
        for (int k = 0; k < 3; ++k)
            for (int l = k; l < 3; ++l) C[k * 3 + l] += (p[k] - barycenter[k]) * (p[l] - barycenter[l]);
    C[3] = C[1]; C[6] = C[2]; C[7] = C[5];
    std::memcpy(nh.covariance, C, sizeof(C));

    double evals[3], evecs[9];
    eig3_sym(C, evals, evecs);
    Vec3 normal = normalized3({{evecs[0], evecs[3], evecs[6]}});   // col(0).normalized()
    nh.normal = normal;
    double sigma_1 = std::sqrt(std::abs(evals[2]));
    double sigma_2 = std::sqrt(std::abs(evals[1]));
    double sigma_3 = std::sqrt(std::abs(evals[0]));
    nh.a2D = (sigma_2 - sigma_3) / sigma_1;
    nh.nan_planarity = (nh.a2D != nh.a2D);   // reference throws std::runtime_error("error")
    return nh;
}

// ----------------------------------------------------------------------------------
// buildPlaneResiduals (src/optimize.cpp:18-131) over a keypoint range
// ----------------------------------------------------------------------------------
struct planeParam {   // include/cloudMap.h:97-108
    Vec3 raw_point, norm_vector;
    double jacobians[6];
    double norm_offset, distance, weight;
};

struct PassCtx {
    const voxelHashMap* map;
    const double* raw_xyz;
    Quat end_quat;
    Vec3 end_t, last_t, t_il;
    Mat3 R_il;
    const orc_icp_params* prm;
    orc_debug_out* dbg;
};

struct RangeResult {
    std::vector<planeParam> plane_residuals;
    double loss_sum = 0.0;
    int64_t num_residuals = 0, num_full = 0, sum_candidates = 0, sum_probes = 0, num_visited = 0, num_fragile = 0;
    bool nan_planarity = false;
};

template <bool DIAG>
void buildPlaneResidualsRange(const PassCtx& c, int64_t k_begin, int64_t k_end, RangeResult& res) {
    const orc_icp_params& o = *c.prm;
    const short nb_voxels_visited = o.frame_id < o.init_num_frames ? 2 : (short)o.voxel_neighborhood;   // :21
    const int kMinNumNeighbors = o.min_number_neighbors;                                                 // :22
    const int kThresholdCapacity = o.frame_id < o.init_num_frames ? 1 : o.threshold_voxel_occupancy;     // :23

    double lambda_weight = std::abs(o.weight_alpha);                // :55-61
    double lambda_neighborhood = std::abs(o.weight_neighborhood);
    const double kMaxPointToPlane = o.max_dist_to_plane_icp;
    const double sum = lambda_weight + lambda_neighborhood;
    lambda_weight /= sum;
    lambda_neighborhood /= sum;

    const int K = o.max_number_neighbors;
    std::vector<Vec3> keypoints_world((size_t)(k_end - k_begin));
    // transformKeypoints (:30-40): R recomputed per keypoint, as written
    for (int64_t k = k_begin; k < k_end; ++k) {
        Mat3 R = quat_to_rot(quat_normalized(c.end_quat));
        Vec3 raw = {{c.raw_xyz[3 * k], c.raw_xyz[3 * k + 1], c.raw_xyz[3 * k + 2]}};
        Vec3 p = vadd(matvec(R, vadd(matvec(c.R_il, raw), c.t_il)), c.end_t);
        keypoints_world[(size_t)(k - k_begin)] = p;
        if (DIAG && c.dbg && c.dbg->world_xyz) std::memcpy(c.dbg->world_xyz + 3 * k, p.v, sizeof(p.v));
    }

    for (int64_t k = k_begin; k < k_end; ++k) {   // :68
        const Vec3& kp_point = keypoints_world[(size_t)(k - k_begin)];
        Vec3 raw_point = {{c.raw_xyz[3 * k], c.raw_xyz[3 * k + 1], c.raw_xyz[3 * k + 2]}};
        res.num_visited++;

        SearchDiag sd;
        auto nbrs = searchNeighbors<DIAG>(*c.map, kp_point, nb_voxels_visited, o.size_voxel_map,
                                          o.max_number_neighbors, kThresholdCapacity, sd);   // :73
        res.sum_candidates += sd.candidates;
        res.sum_probes += sd.probes_hit;
        if (DIAG && c.dbg) {
            if (c.dbg->num_candidates) c.dbg->num_candidates[k] = (int32_t)sd.candidates;
            if (c.dbg->nbr || c.dbg->nbr_dist)
                for (int j = 0; j < K; ++j) {
                    bool have = j < (int)nbrs.size();
                    if (c.dbg->nbr) {
                        int16_t* d = c.dbg->nbr + (k * K + j) * 4;
                        d[0] = have ? nbrs[j].vx : -1; d[1] = have ? nbrs[j].vy : -1;
                        d[2] = have ? nbrs[j].vz : -1; d[3] = have ? nbrs[j].idx : -1;
                    }
                    if (c.dbg->nbr_dist) c.dbg->nbr_dist[k * K + j] = have ? nbrs[j].distance : 0.0;
                }
        }
        if (DIAG) {
            // selection robustness: (K+1)-th vs K-th distance, ties inside the list, key near a cell boundary
            bool fragile = false;
            if ((int)nbrs.size() == K) {
                double dK = nbrs[K - 1].distance;
                if (sd.d_next - dK <= 1e-12 * dK) fragile = true;
                for (int j = 1; j < K; ++j)
                    if (nbrs[j].distance == nbrs[j - 1].distance) fragile = true;
            }
            for (int a = 0; a < 3; ++a) {
                double q = kp_point[a] / o.size_voxel_map;
                if (std::abs(q - std::nearbyint(q)) < 1e-9) fragile = true;
            }
            if (fragile) res.num_fragile++;
        }

        if ((int)nbrs.size() < kMinNumNeighbors) {   // :78
            if (DIAG && c.dbg && c.dbg->status) c.dbg->status[k] = 0;
            continue;
        }
        res.num_full++;

        std::vector<Vec3> vector_neighbors(nbrs.size());
        for (size_t j = 0; j < nbrs.size(); ++j) vector_neighbors[j] = nbrs[j].point;

        double weight;
        Vec3 location = vadd(matvec(c.R_il, raw_point), c.t_il);   // :83

        // estimatePointNeighborhood (:42-53)
        Neighborhood neighborhood = computeNeighborhoodDistribution(vector_neighbors);
        if (neighborhood.nan_planarity) res.nan_planarity = true;
        weight = std::pow(neighborhood.a2D, o.power_planarity);
        if (dot3(neighborhood.normal, vsub(c.last_t, location)) < 0)
            neighborhood.normal = vscale(neighborhood.normal, -1.0);

        weight = lambda_weight * weight +
                 lambda_neighborhood * std::exp(-norm3(vsub(vector_neighbors[0], kp_point)) /
                                                (kMaxPointToPlane * kMinNumNeighbors));   // :87-88

        planeParam plane_temp;
        plane_temp.raw_point = location;
        plane_temp.norm_vector = normalized3(neighborhood.normal);                         // :92-93
        plane_temp.norm_offset = -dot3(plane_temp.norm_vector, vector_neighbors[0]);       // :94
        Mat3 Rq = quat_to_rot(c.end_quat);                                                 // un-normalised quaternion (:95)
        plane_temp.distance = dot3(plane_temp.norm_vector, vadd(matvec(Rq, plane_temp.raw_point), c.end_t)) +
                              plane_temp.norm_offset;
        plane_temp.weight = weight;
        for (int j = 0; j < 6; ++j) plane_temp.jacobians[j] = 0.0;

        bool accepted = false;
        if (plane_temp.distance < o.max_dist_to_plane_icp) {   // :98 signed gate
            accepted = true;
            res.num_residuals++;
            for (int j = 0; j < 3; ++j) plane_temp.jacobians[j] = plane_temp.norm_vector[j] * weight;   // :100
            // :101  -(n^T * R') * skew(raw) * w , evaluated left to right
            Vec3 nR;
            for (int j = 0; j < 3; ++j)
                nR[j] = (-plane_temp.norm_vector[0]) * Rq(0, j) +
                        ((-plane_temp.norm_vector[1]) * Rq(1, j) + (-plane_temp.norm_vector[2]) * Rq(2, j));
            Mat3 Sk = skew(plane_temp.raw_point);
            for (int j = 0; j < 3; ++j)
                plane_temp.jacobians[3 + j] = (nR[0] * Sk(0, j) + (nR[1] * Sk(1, j) + nR[2] * Sk(2, j))) * weight;
            res.plane_residuals.push_back(plane_temp);
            res.loss_sum += plane_temp.distance * plane_temp.distance;   // :104
        }
        if (DIAG && c.dbg) {
            if (c.dbg->status) c.dbg->status[k] = accepted ? 2 : 1;
            if (c.dbg->plane) {
                double* d = c.dbg->plane + 16 * k;
                for (int j = 0; j < 3; ++j) { d[j] = plane_temp.raw_point[j]; d[3 + j] = plane_temp.norm_vector[j]; }
                for (int j = 0; j < 6; ++j) d[6 + j] = plane_temp.jacobians[j];
                d[12] = plane_temp.norm_offset; d[13] = plane_temp.distance; d[14] = plane_temp.weight;
                d[15] = neighborhood.a2D;
            }
        }
        if (res.num_residuals >= o.max_num_residuals) break;   // :107
    }
}

// rows -> H_x, h -> HTH, HTh (src/optimize.cpp:160-170,235,239), fixed row order
void accumulateNormalEq(const std::vector<planeParam>& rows, double HTH[36], double HTh[6]) {
    for (const auto& r : rows) {
        double h = r.distance * r.weight;
        for (int a = 0; a < 6; ++a) {
            for (int b = 0; b < 6; ++b) HTH[a * 6 + b] += r.jacobians[a] * r.jacobians[b];
            HTh[a] += r.jacobians[a] * h;
        }
    }
}

int32_t buildPlaneResidualsAll(const PassCtx& c, int64_t n, int nthreads, orc_normal_eq* out,
                               std::vector<planeParam>* rows_out) {
    std::memset(out, 0, sizeof(*out));
    const bool diag = c.dbg != nullptr;
    if (diag && c.dbg->status) for (int64_t k = 0; k < n; ++k) c.dbg->status[k] = -1;

    std::vector<RangeResult> parts;
    if (nthreads <= 1) {
        parts.resize(1);
        if (diag) buildPlaneResidualsRange<true>(c, 0, n, parts[0]);
        else buildPlaneResidualsRange<false>(c, 0, n, parts[0]);
    } else {
        if (c.prm->max_num_residuals < n) return -2;   // the :107 break is sequential; refuse
        parts.resize((size_t)nthreads);
        std::vector<std::thread> th;
        for (int t = 0; t < nthreads; ++t) {
            int64_t b = n * t / nthreads, e = n * (t + 1) / nthreads;
            th.emplace_back([&, t, b, e]() {
                if (diag) buildPlaneResidualsRange<true>(c, b, e, parts[(size_t)t]);
                else buildPlaneResidualsRange<false>(c, b, e, parts[(size_t)t]);
            });
        }
        for (auto& t : th) t.join();
    }
    for (auto& p : parts) {   // fixed-order combine
        double HTH[36] = {0}, HTh[6] = {0};
        accumulateNormalEq(p.plane_residuals, HTH, HTh);
        for (int i = 0; i < 36; ++i) out->HTH[i] += HTH[i];
        for (int i = 0; i < 6; ++i) out->HTh[i] += HTh[i];
        out->loss_sum += p.loss_sum;
        out->num_residuals += p.num_residuals;
        out->num_full_neighborhoods += p.num_full;
        out->sum_candidates += p.sum_candidates;
        out->sum_probes_hit += p.sum_probes;
        out->num_visited += p.num_visited;
        out->num_fragile += p.num_fragile;
        if (p.nan_planarity) out->nan_planarity = 1;
        if (rows_out) rows_out->insert(rows_out->end(), p.plane_residuals.begin(), p.plane_residuals.end());
    }
    out->success = out->num_residuals >= c.prm->min_number_neighbors ? 1 : 0;   // :110
    return 0;
}

PassCtx makeCtx(void* map, const double* raw_xyz, const double q_cur[4], const double t_cur[3], const double t_last[3],
                const double R_il[9], const double t_il[3], const orc_icp_params* prm, orc_debug_out* dbg) {
    PassCtx c;
    c.map = static_cast<const voxelHashMap*>(map);
    c.raw_xyz = raw_xyz;
    c.end_quat = {q_cur[0], q_cur[1], q_cur[2], q_cur[3]};
    c.end_t = {{t_cur[0], t_cur[1], t_cur[2]}};
    c.last_t = {{t_last[0], t_last[1], t_last[2]}};
    c.t_il = {{t_il[0], t_il[1], t_il[2]}};
    std::memcpy(c.R_il.m, R_il, sizeof(double) * 9);
    c.prm = prm;
    c.dbg = dbg;
    return c;
}

// eskfEstimator::observe (src/eskfEstimator.cpp:219-230)
void eskf_observe(orc_eskf_state* s, const double d_x[17]) {
    for (int i = 0; i < 3; ++i) s->p[i] = s->p[i] + d_x[i];
    Quat q = {s->q[0], s->q[1], s->q[2], s->q[3]};
    q = quat_normalized(quat_mul(q, so3ToQuat({{d_x[3], d_x[4], d_x[5]}})));
    s->q[0] = q.x; s->q[1] = q.y; s->q[2] = q.z; s->q[3] = q.w;
    for (int i = 0; i < 3; ++i) {
        s->v[i] = s->v[i] + d_x[6 + i];
        s->ba[i] = s->ba[i] + d_x[9 + i];
        s->bg[i] = s->bg[i] + d_x[12 + i];
    }
    Vec3 g = {{s->g[0], s->g[1], s->g[2]}};
    double B[6];
    derivativeS2(g, B);
    Vec3 so3_dg = {{B[0] * d_x[15] + B[1] * d_x[16], B[2] * d_x[15] + B[3] * d_x[16], B[4] * d_x[15] + B[5] * d_x[16]}};
    Vec3 gn = matvec(so3ToRotation(so3_dg), g);
    s->g[0] = gn[0]; s->g[1] = gn[1]; s->g[2] = gn[2];
}

}  // namespace

// ======================================================================================
// C interface
// ======================================================================================
extern "C" {

void* orc_map_create(void) { return new voxelHashMap(); }
void orc_map_destroy(void* map) { delete static_cast<voxelHashMap*>(map); }
const char* orc_map_backend(void) { return kBackend; }
int64_t orc_map_num_voxels(void* map) { return (int64_t) static_cast<voxelHashMap*>(map)->size(); }
int64_t orc_map_num_points(void* map) {   // lioOptimization::mapSize (src/lioOptimization.cpp:574-581)
    int64_t s = 0;
    for (auto& it : *static_cast<voxelHashMap*>(map)) s += it.second.NumPoints();
    return s;
}

int64_t orc_map_add_points(void* map, const double* xyz, int64_t n, double voxel_size,
                           int32_t max_num_points_in_voxel, double min_distance_points, int32_t min_num_points) {
    voxelHashMap& m = *static_cast<voxelHashMap*>(map);
    int64_t added = 0;
    for (int64_t i = 0; i < n; ++i) {   // src/lioOptimization.cpp:533-537
        rgbPoint rgb_point({{xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]}});
        added += addPointToMap(m, rgb_point, voxel_size, max_num_points_in_voxel, min_distance_points, min_num_points);
    }
    return added;
}

// lioOptimization::removePointsFarFromLocation (src/lioOptimization.cpp:556-572)
int64_t orc_map_remove_far(void* map_, const double location[3], double distance) {
    voxelHashMap& map = *static_cast<voxelHashMap*>(map_);
    std::vector<voxel> voxels_to_erase;
    const Vec3 loc = {{location[0], location[1], location[2]}};
    for (auto& pair : map) {
        const rgbPoint& rgb_point = pair.second.points[0];
        const Vec3 pt = {{(double)rgb_point.position[0], (double)rgb_point.position[1], (double)rgb_point.position[2]}};
        if (sqnorm3(vsub(pt, loc)) > (distance * distance)) voxels_to_erase.push_back(pair.first);
    }
    for (auto& vox : voxels_to_erase) map.erase(vox);
    return (int64_t)voxels_to_erase.size();
}

int64_t orc_map_snapshot(void* map, int32_t cap, int16_t* keys, int32_t* counts, float* xyz) {
    voxelHashMap& m = *static_cast<voxelHashMap*>(map);
    int64_t v = 0;
    for (auto& it : m) {
        keys[3 * v] = it.first.x; keys[3 * v + 1] = it.first.y; keys[3 * v + 2] = it.first.z;
        int c = std::min<int>(it.second.NumPoints(), cap);
        counts[v] = c;
        for (int i = 0; i < cap; ++i)
            for (int a = 0; a < 3; ++a)
                xyz[(v * cap + i) * 3 + a] = i < c ? it.second.points[(size_t)i].position[a] : 0.f;
        ++v;
    }
    return v;
}

void orc_map_load(void* map, const int16_t* keys, const int32_t* counts, const float* xyz, int64_t n_voxels,
                  int32_t cap) {
    voxelHashMap& m = *static_cast<voxelHashMap*>(map);
    for (int64_t v = 0; v < n_voxels; ++v) {
        voxelBlock blk(cap);
        for (int i = 0; i < counts[v]; ++i) {
            rgbPoint p({{0, 0, 0}});
            for (int a = 0; a < 3; ++a) p.position[a] = xyz[(v * cap + i) * 3 + a];
            blk.AddPoint(p);
        }
        m[voxel(keys[3 * v], keys[3 * v + 1], keys[3 * v + 2])] = std::move(blk);
    }
}

int32_t orc_build_plane_residuals(void* map, const double* raw_xyz, int64_t n, const double q_cur[4],
                                  const double t_cur[3], const double t_last[3], const double R_il[9],
                                  const double t_il[3], const orc_icp_params* prm, int32_t nthreads,
                                  orc_normal_eq* out, orc_debug_out* dbg) {
    PassCtx c = makeCtx(map, raw_xyz, q_cur, t_cur, t_last, R_il, t_il, prm, dbg);
    return buildPlaneResidualsAll(c, n, nthreads, out, nullptr);
}

// lioOptimization::updateIEKF (src/optimize.cpp:133-314)
int32_t orc_update_iekf(void* map, const double* raw_xyz, int64_t n, orc_eskf_state* eskf, double frame_q[4],
                        double frame_t[3], const double t_last[3], const double R_il[9], const double t_il[3],
                        const orc_icp_params* prm, int32_t nthreads, int32_t* passes_run,
                        int32_t* num_residuals_used, double* trace, int32_t max_trace_rows) {
    const orc_icp_params& o = *prm;
    int max_num_iter = o.frame_id < o.init_num_frames ? std::max(15, o.num_iters_icp) : o.num_iters_icp;   // :135

    Vec3 p_predict = {{eskf->p[0], eskf->p[1], eskf->p[2]}};                 // :138-143
    Quat q_predict = {eskf->q[0], eskf->q[1], eskf->q[2], eskf->q[3]};
    Vec3 v_predict = {{eskf->v[0], eskf->v[1], eskf->v[2]}};
    Vec3 ba_predict = {{eskf->ba[0], eskf->ba[1], eskf->ba[2]}};
    Vec3 bg_predict = {{eskf->bg[0], eskf->bg[1], eskf->bg[2]}};
    Vec3 g_predict = {{eskf->g[0], eskf->g[1], eskf->g[2]}};

    int passes = 0;
    int32_t success = 1;
    if (num_residuals_used) *num_residuals_used = 0;

    for (int i = -1; i < max_num_iter; i++) {   // :147
        std::vector<planeParam> plane_residuals;
        orc_normal_eq ne;
        PassCtx c = makeCtx(map, raw_xyz, frame_q, frame_t, t_last, R_il, t_il, prm, nullptr);
        int rc = buildPlaneResidualsAll(c, n, nthreads, &ne, &plane_residuals);   // :153
        if (rc != 0) return rc;
        passes++;
        if (num_residuals_used) *num_residuals_used = (int32_t)ne.num_residuals;
        if (!ne.success) { success = 0; break; }   // :155

        const int N = (int)plane_residuals.size();
        Vec3 eskf_p = {{eskf->p[0], eskf->p[1], eskf->p[2]}};
        Quat eskf_q = {eskf->q[0], eskf->q[1], eskf->q[2], eskf->q[3]};
        Vec3 d_p = vsub(eskf_p, p_predict);                                   // :172
        Quat d_q = quat_mul(quat_inverse(q_predict), eskf_q);                 // :173
        Vec3 d_so3 = quatToSo3(d_q);                                          // :174
        Vec3 d_v = vsub({{eskf->v[0], eskf->v[1], eskf->v[2]}}, v_predict);
        Vec3 d_ba = vsub({{eskf->ba[0], eskf->ba[1], eskf->ba[2]}}, ba_predict);
        Vec3 d_bg = vsub({{eskf->bg[0], eskf->bg[1], eskf->bg[2]}}, bg_predict);

        Vec3 g = {{eskf->g[0], eskf->g[1], eskf->g[2]}};
        Vec3 g_predict_normalize = normalized3(g_predict);
        Vec3 g_normalize = normalized3(g);
        Vec3 cross = cross3(g_predict_normalize, g_normalize);               // :187
        double dot = dot3(g_predict_normalize, g_normalize);
        Mat3 R_dg;
        if (std::fabs(1.0 - dot) < 1e-6) R_dg = identity3();
        else {
            Mat3 sk = skew(cross), sk2 = matmul(sk, sk);
            double f = (1.0 - dot);
            double den = cross[0] * cross[0] + cross[1] * cross[1] + cross[2] * cross[2];
            Mat3 I = identity3();
            for (int e = 0; e < 9; ++e) R_dg.m[e] = I.m[e] + sk.m[e] + sk2.m[e] * f / den;   // :197-198
        }
        Vec3 so3_dg = rotationToSo3(R_dg);                                    // :201
        double Bp[6];
        derivativeS2(g_predict, Bp);                                          // :202
        double d_g[2] = {Bp[0] * so3_dg[0] + (Bp[2] * so3_dg[1] + Bp[4] * so3_dg[2]),
                         Bp[1] * so3_dg[0] + (Bp[3] * so3_dg[1] + Bp[5] * so3_dg[2])};   // B^T * so3

        double d_x[NS];
        for (int e = 0; e < 3; ++e) { d_x[e] = d_p[e]; d_x[3 + e] = d_so3[e]; d_x[6 + e] = d_v[e]; d_x[9 + e] = d_ba[e]; d_x[12 + e] = d_bg[e]; }
        d_x[15] = d_g[0]; d_x[16] = d_g[1];

        Mat3 J_k_so3, skd = skew(d_so3);                                      // :213
        { Mat3 I = identity3(); for (int e = 0; e < 9; ++e) J_k_so3.m[e] = I.m[e] - 0.5 * skd.m[e]; }
        // J_k_s2 = I2 + 0.5 * B^T * skew(so3_dg) * B                         // :214
        double J_k_s2[4];
        {
            Mat3 S = skew(so3_dg);
            double SB[6];   // 3x2
            for (int r = 0; r < 3; ++r)
                for (int cc = 0; cc < 2; ++cc) SB[r * 2 + cc] = S(r, 0) * Bp[0 + cc] + (S(r, 1) * Bp[2 + cc] + S(r, 2) * Bp[4 + cc]);
            for (int r = 0; r < 2; ++r)
                for (int cc = 0; cc < 2; ++cc)
                    J_k_s2[r * 2 + cc] = (r == cc ? 1.0 : 0.0) +
                                         0.5 * (Bp[0 + r] * SB[0 + cc] + (Bp[2 + r] * SB[2 + cc] + Bp[4 + r] * SB[4 + cc]));
        }
        double d_x_new[NS];
        std::memcpy(d_x_new, d_x, sizeof(d_x));
        { Vec3 t = matvec(J_k_so3, d_so3); for (int e = 0; e < 3; ++e) d_x_new[3 + e] = t[e]; }             // :217
        d_x_new[15] = J_k_s2[0] * d_g[0] + J_k_s2[1] * d_g[1];                                             // :218
        d_x_new[16] = J_k_s2[2] * d_g[0] + J_k_s2[3] * d_g[1];

        double cov[NS * NS];
        std::memcpy(cov, eskf->cov, sizeof(cov));                             // :220
        auto rows3 = [&](double* M, const Mat3& J) {        // M.block<3,1>(3,j) = J * M.block<3,1>(3,j)
            for (int j = 0; j < NS; ++j) {
                Vec3 col = {{M[3 * NS + j], M[4 * NS + j], M[5 * NS + j]}};
                Vec3 r = matvec(J, col);
                M[3 * NS + j] = r[0]; M[4 * NS + j] = r[1]; M[5 * NS + j] = r[2];
            }
        };
        auto rows2 = [&](double* M, const double* J) {
            for (int j = 0; j < NS; ++j) {
                double a = M[15 * NS + j], b = M[16 * NS + j];
                M[15 * NS + j] = J[0] * a + J[1] * b;
                M[16 * NS + j] = J[2] * a + J[3] * b;
            }
        };
        auto cols3 = [&](double* M, const double* Msrc, const Mat3& J) {   // M(j,3:6) = Msrc(j,3:6) * J^T
            for (int j = 0; j < NS; ++j) {
                Vec3 row = {{Msrc[j * NS + 3], Msrc[j * NS + 4], Msrc[j * NS + 5]}};
                Vec3 r = matvec(J, row);
                M[j * NS + 3] = r[0]; M[j * NS + 4] = r[1]; M[j * NS + 5] = r[2];
            }
        };
        auto cols2 = [&](double* M, const double* Msrc, const double* J) {
            for (int j = 0; j < NS; ++j) {
                double a = Msrc[j * NS + 15], b = Msrc[j * NS + 16];
                M[j * NS + 15] = J[0] * a + J[1] * b;
                M[j * NS + 16] = J[2] * a + J[3] * b;
            }
        };
        rows3(cov, J_k_so3);         // :222-223
        rows2(cov, J_k_s2);          // :225-226
        cols3(cov, cov, J_k_so3);    // :228-229
        cols2(cov, cov, J_k_s2);     // :231-232

        double temp[NS * NS], temp_inv[NS * NS], scaled[NS * NS];
        for (int e = 0; e < NS * NS; ++e) scaled[e] = cov[e] / o.laser_point_cov;   // :234
        if (!mat_inverse(scaled, temp, NS)) return -3;
        double HTH[36];
        std::memcpy(HTH, ne.HTH, sizeof(HTH));                                // :235
        for (int r = 0; r < 6; ++r) for (int cc = 0; cc < 6; ++cc) temp[r * NS + cc] += HTH[r * 6 + cc];   // :236
        if (!mat_inverse(temp, temp_inv, NS)) return -3;                      // :237

        double K_h[NS];
        if (nthreads <= 1) {
            // :239 evaluated as (temp_inv[:, :6] * H_x^T) * h, like Eigen's left-to-right product
            std::vector<double> TH((size_t)NS * (size_t)std::max(N, 1));
            for (int r = 0; r < NS; ++r)
                for (int k = 0; k < N; ++k) {
                    double s = 0.0;
                    for (int a = 0; a < 6; ++a) s += temp_inv[r * NS + a] * plane_residuals[(size_t)k].jacobians[a];
                    TH[(size_t)r * N + k] = s;
                }
            for (int r = 0; r < NS; ++r) {
                double s = 0.0;
                for (int k = 0; k < N; ++k)
                    s += TH[(size_t)r * N + k] * (plane_residuals[(size_t)k].distance * plane_residuals[(size_t)k].weight);
                K_h[r] = s;
            }
        } else {
            for (int r = 0; r < NS; ++r) {
                double s = 0.0;
                for (int a = 0; a < 6; ++a) s += temp_inv[r * NS + a] * ne.HTh[a];
                K_h[r] = s;
            }
        }
        double K_x[NS * NS];
        std::memset(K_x, 0, sizeof(K_x));                                      // :241
        for (int r = 0; r < NS; ++r)
            for (int cc = 0; cc < 6; ++cc) {
                double s = 0.0;
                for (int a = 0; a < 6; ++a) s += temp_inv[r * NS + a] * HTH[a * 6 + cc];
                K_x[r * NS + cc] = s;                                          // :242
            }
        for (int r = 0; r < NS; ++r) {                                         // :244
            double s = 0.0;
            for (int cc = 0; cc < NS; ++cc) s += (K_x[r * NS + cc] - (r == cc ? 1.0 : 0.0)) * d_x_new[cc];
            d_x[r] = -K_h[r] + s;
        }

        Vec3 g_before = {{eskf->g[0], eskf->g[1], eskf->g[2]}};              // :246
        Vec3 dxp = {{d_x[0], d_x[1], d_x[2]}}, dxr = {{d_x[3], d_x[4], d_x[5]}};
        if (norm3(dxp) > 100.0 || AngularDistance(dxr) > 100.0) {            // :248-251
            if (trace && passes <= max_trace_rows) {
                double* tr = trace + (size_t)(passes - 1) * 24;
                std::memcpy(tr, d_x, sizeof(d_x));
                std::memcpy(tr + 17, frame_t, 3 * sizeof(double));
                std::memcpy(tr + 20, frame_q, 4 * sizeof(double));
            }
            continue;
        }

        eskf_observe(eskf, d_x);                                              // :253
        std::memcpy(frame_t, eskf->p, 3 * sizeof(double));                    // :255-256
        std::memcpy(frame_q, eskf->q, 4 * sizeof(double));
        if (trace && passes <= max_trace_rows) {
            double* tr = trace + (size_t)(passes - 1) * 24;
            std::memcpy(tr, d_x, sizeof(d_x));
            std::memcpy(tr + 17, frame_t, 3 * sizeof(double));
            std::memcpy(tr + 20, frame_q, 4 * sizeof(double));
        }

        bool converage = false;
        if (o.frame_id > 1 && norm3(dxp) < o.threshold_translation_norm &&
            AngularDistance(dxr) < o.threshold_orientation_norm)              // :265-270
            converage = true;

        if (converage || i == max_num_iter - 1) {                            // :272-310
            double cov_new[NS * NS];
            std::memcpy(cov_new, cov, sizeof(cov));
            double Bb[6];
            derivativeS2(g_before, Bb);
            { Mat3 I = identity3(), s3 = skew(dxr); for (int e = 0; e < 9; ++e) J_k_so3.m[e] = I.m[e] - 0.5 * s3.m[e]; }
            {
                Vec3 bd = {{Bb[0] * d_x[15] + Bb[1] * d_x[16], Bb[2] * d_x[15] + Bb[3] * d_x[16], Bb[4] * d_x[15] + Bb[5] * d_x[16]}};
                Mat3 S = skew(bd);
                double SB[6];
                for (int r = 0; r < 3; ++r)
                    for (int cc = 0; cc < 2; ++cc) SB[r * 2 + cc] = S(r, 0) * Bb[0 + cc] + (S(r, 1) * Bb[2 + cc] + S(r, 2) * Bb[4 + cc]);
                for (int r = 0; r < 2; ++r)
                    for (int cc = 0; cc < 2; ++cc)
                        J_k_s2[r * 2 + cc] = (r == cc ? 1.0 : 0.0) +
                                             0.5 * (Bb[0 + r] * SB[0 + cc] + (Bb[2 + r] * SB[2 + cc] + Bb[4 + r] * SB[4 + cc]));
            }
            // :281-285 rows of covariance_new from covariance
            for (int j = 0; j < NS; ++j) {
                Vec3 col = {{cov[3 * NS + j], cov[4 * NS + j], cov[5 * NS + j]}};
                Vec3 r = matvec(J_k_so3, col);
                cov_new[3 * NS + j] = r[0]; cov_new[4 * NS + j] = r[1]; cov_new[5 * NS + j] = r[2];
            }
            for (int j = 0; j < NS; ++j) {
                double a = cov[15 * NS + j], b = cov[16 * NS + j];
                cov_new[15 * NS + j] = J_k_s2[0] * a + J_k_s2[1] * b;
                cov_new[16 * NS + j] = J_k_s2[2] * a + J_k_s2[3] * b;
            }
            // :287-297 columns: covariance_new from covariance (overwriting), covariance in place
            cols3(cov_new, cov, J_k_so3);
            cols3(cov, cov, J_k_so3);
            cols2(cov_new, cov, J_k_s2);
            cols2(cov, cov, J_k_s2);
            // :299-303 K_x rows, first 6 columns only
            for (int j = 0; j < 6; ++j) {
                Vec3 col = {{K_x[3 * NS + j], K_x[4 * NS + j], K_x[5 * NS + j]}};
                Vec3 r = matvec(J_k_so3, col);
                K_x[3 * NS + j] = r[0]; K_x[4 * NS + j] = r[1]; K_x[5 * NS + j] = r[2];
            }
            for (int j = 0; j < 6; ++j) {
                double a = K_x[15 * NS + j], b = K_x[16 * NS + j];
                K_x[15 * NS + j] = J_k_s2[0] * a + J_k_s2[1] * b;
                K_x[16 * NS + j] = J_k_s2[2] * a + J_k_s2[3] * b;
            }
            // :305 covariance = covariance_new - K_x[:, :6] * covariance[:6, :]
            for (int r = 0; r < NS; ++r)
                for (int cc = 0; cc < NS; ++cc) {
                    double s = 0.0;
                    for (int a = 0; a < 6; ++a) s += K_x[r * NS + a] * cov[a * NS + cc];
                    eskf->cov[r * NS + cc] = cov_new[r * NS + cc] - s;       // :307 setCovariance
                }
            break;
        }
    }
    if (passes_run) *passes_run = passes;
    return success;
}

// subSampleFrame (src/utility.cpp:167-186) as called by gridSampling (:188-201); vectors hold frame indices instead of
// point3D copies, everything else (container type, hash, key expression, push_back, "n.second[0]") as written
int64_t orc_grid_sampling(const double* xyz, int64_t n, double size_voxel, int32_t* out) {
    std::tr1::unordered_map<voxel, std::vector<int32_t>, voxel_hash> grid;
    for (int i = 0; i < (int)n; i++) {
        auto kx = static_cast<short>(xyz[3 * i] / size_voxel);
        auto ky = static_cast<short>(xyz[3 * i + 1] / size_voxel);
        auto kz = static_cast<short>(xyz[3 * i + 2] / size_voxel);
        grid[voxel(kx, ky, kz)].push_back(i);
    }
    int64_t m = 0;
    for (const auto& g : grid)
        if (g.second.size() > 0) out[m++] = g.second[0];
    return m;
}

// ---- row N3: per-sweep point transforms / undistortion (src/utility.cpp:203-332) --------------------------------
namespace {
// Eigen 3.3.7 QuaternionBase::slerp (Eigen/src/Geometry/Quaternion.h): the dependency is not vendored in the reference;
// this restates its published algorithm.  The 4-coefficient dot reduces as (x+z)+(y+w) like squaredNorm.
inline Quat quat_slerp(const Quat& a, double t, const Quat& b) {
    const double one = 1.0 - std::numeric_limits<double>::epsilon();
    const double d = (a.x * b.x + a.z * b.z) + (a.y * b.y + a.w * b.w);
    const double absD = std::fabs(d);
    double scale0, scale1;
    if (absD >= one) { scale0 = 1.0 - t; scale1 = t; }
    else {
        const double theta = std::acos(absD);
        const double sinTheta = std::sin(theta);
        scale0 = std::sin((1.0 - t) * theta) / sinTheta;
        scale1 = std::sin(t * theta) / sinTheta;
    }
    if (d < 0) scale1 = -scale1;
    return {scale0 * a.x + scale1 * b.x, scale0 * a.y + scale1 * b.y, scale0 * a.z + scale1 * b.z, scale0 * a.w + scale1 * b.w};
}
inline Vec3 v3p(const double* p) { return {{p[0], p[1], p[2]}}; }
inline Mat3 m3p(const double* p) { Mat3 M; std::memcpy(M.m, p, sizeof(M.m)); return M; }
}  // namespace

// distortFrameByConstant (src/utility.cpp:203-236): pose interpolated between the first and last IMU state of the sweep
void orc_distort_frame_by_constant(const double* raw_xyz, const double* relative_time, int64_t n, const orc_imu_state* st,
                                   int64_t n_states, double time_frame_begin, const double R_il[9], const double t_il[3],
                                   double* imu_xyz) {
    if (n_states < 1) return;
    const double time_frame_end = st[n_states - 1].timestamp;
    const Quat quat_begin = {st[0].quat[0], st[0].quat[1], st[0].quat[2], st[0].quat[3]};
    const Quat quat_end = {st[n_states - 1].quat[0], st[n_states - 1].quat[1], st[n_states - 1].quat[2], st[n_states - 1].quat[3]};
    const Vec3 trans_begin = v3p(st[0].trans), trans_end = v3p(st[n_states - 1].trans);
    const Mat3 R = m3p(R_il);
    const Vec3 t = v3p(t_il);
    for (int64_t i = 0; i < n; ++i) {
        double time_point = time_frame_begin + relative_time[i] / 1000.0;
        if (std::fabs(time_point - time_frame_begin) < 1e-6) time_point = time_frame_begin + 1e-6;
        if (std::fabs(time_point - time_frame_end) < 1e-6) time_point = time_frame_end - 1e-6;
        double alpha_time = (time_point - time_frame_begin) / (time_frame_end - time_frame_begin);
        if (alpha_time > 1) alpha_time = 1;
        if (alpha_time < 0) alpha_time = 0;
        const Quat quat_alpha = quat_slerp(quat_begin, alpha_time, quat_end);
        const Vec3 trans_alpha = vadd(vscale(trans_begin, 1.0 - alpha_time), vscale(trans_end, alpha_time));
        const Vec3 p = vadd(matvec(quat_to_rot(quat_alpha), vadd(matvec(R, v3p(raw_xyz + 3 * i)), t)), trans_alpha);
        imu_xyz[3 * i] = p[0]; imu_xyz[3 * i + 1] = p[1]; imu_xyz[3 * i + 2] = p[2];
    }
}

// distortFrameByImu (src/utility.cpp:238-312, "distortion method 1"): one iterator walks the points while the outer loop
// walks the IMU intervals; a point outside the current interval ends that interval, so points are consumed in order
// and whatever is left when the intervals run out keeps its old imu_point.  Returns the number of points written.
int64_t orc_distort_frame_by_imu(const double* raw_xyz, const double* relative_time, int64_t n, const orc_imu_state* st,
                                 int64_t n_states, double time_frame_begin, const double R_il[9], const double t_il[3],
                                 double* imu_xyz) {
    const Mat3 R = m3p(R_il);
    const Vec3 t = v3p(t_il);
    int64_t iter = 0;
    for (int64_t k = 0; k + 1 < n_states; k++) {
        const double time_imu_begin = st[k].timestamp;
        const Quat quat_imu = {st[k].quat[0], st[k].quat[1], st[k].quat[2], st[k].quat[3]};
        const Vec3 trans_imu = v3p(st[k].trans), vel_imu = v3p(st[k].vel);
        const double time_imu_end = st[k + 1].timestamp;
        const Vec3 un_acc = v3p(st[k + 1].un_acc), un_gyr = v3p(st[k + 1].un_gyr);
        while (iter != n) {
            double time_point = time_frame_begin + relative_time[iter] / 1000.0;
            if (time_point > time_imu_begin - 1e-6 && time_point < time_imu_end + 1e-6) {
                if (std::fabs(time_point - time_imu_begin) < 1e-6) time_point = time_imu_begin + 1e-6;
                if (std::fabs(time_point - time_imu_end) < 1e-6) time_point = time_imu_end - 1e-6;
                const double dt = time_point - time_imu_begin;
                const Quat quat_point = quat_normalized(quat_mul(quat_imu, so3ToQuat(vscale(un_gyr, dt))));
                const Vec3 trans_point = vadd(vadd(trans_imu, vscale(vel_imu, dt)), vscale(vscale(vscale(un_acc, 0.5), dt), dt));
                const Vec3 p = vadd(matvec(quat_to_rot(quat_point), vadd(matvec(R, v3p(raw_xyz + 3 * iter)), t)), trans_point);
                imu_xyz[3 * iter] = p[0]; imu_xyz[3 * iter + 1] = p[1]; imu_xyz[3 * iter + 2] = p[2];
                iter++;
            } else {
                break;
            }
        }
    }
    return iter;
}

// transformAllImuPoint (src/utility.cpp:320-332): every imu_point into the LiDAR frame at the END of the sweep
void orc_transform_all_imu_point(const double* imu_xyz, int64_t n, const orc_imu_state* last, const double R_il[9],
                                 const double t_il[3], double* raw_out) {
    const Quat quat_end_inv = quat_inverse({last->quat[0], last->quat[1], last->quat[2], last->quat[3]});
    const Mat3 Rinv = quat_to_rot(quat_end_inv);
    const Vec3 trans_end_inv = vscale(matvec(Rinv, v3p(last->trans)), -1.0);
    const Mat3 Rt = transpose(m3p(R_il));
    const Vec3 off = matvec(Rt, v3p(t_il));
    for (int64_t i = 0; i < n; ++i) {
        const Vec3 p = vsub(matvec(Rt, vadd(matvec(Rinv, v3p(imu_xyz + 3 * i)), trans_end_inv)), off);
        raw_out[3 * i] = p[0]; raw_out[3 * i + 1] = p[1]; raw_out[3 * i + 2] = p[2];
    }
}

void orc_quat_slerp(const double a[4], double t, const double b[4], double out[4]) {
    const Quat q = quat_slerp({a[0], a[1], a[2], a[3]}, t, {b[0], b[1], b[2], b[3]});
    out[0] = q.x; out[1] = q.y; out[2] = q.z; out[3] = q.w;
}

void orc_quat_to_rot(const double q[4], double R[9]) {
    Mat3 M = quat_to_rot({q[0], q[1], q[2], q[3]});
    std::memcpy(R, M.m, sizeof(M.m));
}
void orc_eig3_sym(const double S[9], double evals[3], double evecs[9]) { eig3_sym(S, evals, evecs); }
void orc_eskf_observe(orc_eskf_state* s, const double dx[17]) { eskf_observe(s, dx); }
int32_t orc_mat17_inverse(const double* A, double* Ainv) { return mat_inverse(A, Ainv, NS) ? 1 : 0; }
// ======================================================================================
// Row N4: the colour map (vision side of the map update).  Restates
//   lioOptimization::addPointToColorMap           src/lioOptimization.cpp:448-518
//   its driver loop in addPointsToMap             src/lioOptimization.cpp:520-551 (colour branch only)
//   rgbMapTracker::renderPointsInRecentVoxel /
//   threadRenderPointsInVoxel                     src/rgbMapTracker.cpp:181-237 (sequential: the reference's
//                                                 cv::parallel_for_ + mutex leaves the per-point result unchanged
//                                                 as long as a voxel appears once in the list; duplicates are
//                                                 applied here in list order)
//   cloudFrame::project3dTo2d / if2dPointsAvailable / getRgb / getSubPixel   src/lioOptimization.cpp:49-190
//   rgbPoint::updateRgb                           src/cloudMap.cpp:59-101
// Third-party arithmetic absent from /root/reference: OpenCV's cv::Vec3b operators (double * Vec3b and
// Vec3b + Vec3b saturate every element to uchar with cvRound = round-half-to-even) — restated from
// OpenCV 4's matx.hpp / saturate.hpp; PARITY UNPINNED for that arithmetic (the stand-in cv::Vec3b of oracle/shim restates it the same way).
// ======================================================================================
struct voxelId { int kx, ky, kz; };   // include/cloudMap.h:88-95
struct ColorMap {
    voxelHashMap map;                                                                    // color_voxel_map
    std::unordered_map<long, std::unordered_map<long, std::unordered_map<long, int>>> hash3d;   // hashmap_3d_points (value: index into rgb_points)
    std::vector<std::array<short, 4>> rgb_points;                                        // rgb_points_vec as (voxel key, index in block)
    std::vector<voxelId> recent_temp;                                                    // voxels_recent_visited_temp
    std::vector<voxelId> recent;                                                         // map_tracker->voxels_recent_visited
    long number_of_new_visited_voxel = 0;
};

static int hash3d_exist(ColorMap& cm, long x, long y, long z) {      // Hash_map_3d::if_exist (include/utility.h:105-119)
    auto a = cm.hash3d.find(x);
    if (a == cm.hash3d.end()) return 0;
    auto b = a->second.find(y);
    if (b == a->second.end()) return 0;
    return b->second.find(z) == b->second.end() ? 0 : 1;
}

// lioOptimization::addPointToColorMap (src/lioOptimization.cpp:448-518); returns 1 if the point was stored in a voxel
static int addPointToColorMap(ColorMap& cm, rgbPoint& point, double voxel_size, int max_num_points_in_voxel,
                              double min_distance_points, int min_num_points, double time_sweep_end, double time_last_process) {
    bool add_point = true;
    int stored = 0;
    int point_map_kx = static_cast<short>(point.getPosition()[0] / min_distance_points);
    int point_map_ky = static_cast<short>(point.getPosition()[1] / min_distance_points);
    int point_map_kz = static_cast<short>(point.getPosition()[2] / min_distance_points);
    int kx = static_cast<short>(point.getPosition()[0] / voxel_size);
    int ky = static_cast<short>(point.getPosition()[1] / voxel_size);
    int kz = static_cast<short>(point.getPosition()[2] / voxel_size);
    if (hash3d_exist(cm, point_map_kx, point_map_ky, point_map_kz)) add_point = false;
    auto search = cm.map.find(voxel(kx, ky, kz));
    if (search != cm.map.end()) {
        voxelBlock& voxel_block = MAP_VALUE(search);
        if (!voxel_block.IsFull()) {
            if (min_num_points <= 0 || voxel_block.NumPoints() >= min_num_points) {
                voxel_block.AddPoint(point);
                stored = 1;
                if (add_point) {
                    point.point_index = (int)cm.rgb_points.size();
                    cm.rgb_points.push_back({{(short)kx, (short)ky, (short)kz, (short)(voxel_block.NumPoints() - 1)}});
                    cm.hash3d[point_map_kx][point_map_ky][point_map_kz] = point.point_index;
                }
            }
        }
        if (std::fabs(time_sweep_end - time_last_process) > 1e-5 && std::fabs(voxel_block.last_visited_time - time_sweep_end) > 1e-5) {
            voxel_block.last_visited_time = time_sweep_end;
            cm.recent_temp.push_back({kx, ky, kz});
        }
    } else {
        if (min_num_points <= 0) {
            voxelBlock voxel_block(max_num_points_in_voxel);
            voxel_block.AddPoint(point);
            cm.map[voxel(kx, ky, kz)] = std::move(voxel_block);
            stored = 1;
            if (add_point) {
                point.point_index = (int)cm.rgb_points.size();
                cm.rgb_points.push_back({{(short)kx, (short)ky, (short)kz, 0}});
                cm.hash3d[point_map_kx][point_map_ky][point_map_kz] = point.point_index;
            }
            voxelBlock& vb = cm.map[voxel(kx, ky, kz)];
            if (std::fabs(time_sweep_end - time_last_process) > 1e-5 && std::fabs(vb.last_visited_time - time_sweep_end) > 1e-5) {
                vb.last_visited_time = time_sweep_end;
                cm.recent_temp.push_back({kx, ky, kz});
            }
        }
    }
    return stored;
}

static inline unsigned char sat_u8(double v) {       // cv::saturate_cast<uchar>(double): cvRound (lrint, half to even) then clamp
    long r = std::lrint(v);
    return (unsigned char)(r < 0 ? 0 : (r > 255 ? 255 : r));
}
static inline unsigned char sat_add_u8(unsigned char a, unsigned char b) { int r = (int)a + (int)b; return (unsigned char)(r > 255 ? 255 : r); }

// rgbPoint::updateRgb (src/cloudMap.cpp:59-101)
static int updateRgb(rgbPoint& p, const double rgb_[3], double observe_distance_, const double observe_sigma_[3], double observe_time_) {
    const double process_noise_sigma = 0.1;
    if (p.observe_distance != 0 && (observe_distance_ > p.observe_distance * 1.2)) return 0;
    if (p.N_rgb == 0) {
        p.last_observe_time = observe_time_;
        p.observe_distance = observe_distance_;
        for (int i = 0; i < 3; i++) {
            p.rgb[0] = (short)std::round(rgb_[0]);
            p.rgb[1] = (short)std::round(rgb_[1]);
            p.rgb[2] = (short)std::round(rgb_[2]);
            for (int a = 0; a < 3; ++a) p.cov_rgb[a] = (float)observe_sigma_[a];
        }
        p.N_rgb = 1;
        return 0;
    }
    for (int i = 0; i < 3; i++) {
        p.cov_rgb[i] = (float)(p.cov_rgb[i] + process_noise_sigma * (observe_time_ - p.last_observe_time));   // float(float + double)
        double old_sigma = p.cov_rgb[i];
        p.cov_rgb[i] = (float)std::sqrt(1.0 / (1.0 / (p.cov_rgb[i] * p.cov_rgb[i]) + 1.0 / (observe_sigma_[i] * observe_sigma_[i])));
        p.rgb[i] = (short)(p.cov_rgb[i] * p.cov_rgb[i] * (p.rgb[i] / (old_sigma * old_sigma) + rgb_[i] / (observe_sigma_[i] * observe_sigma_[i])));
    }
    if (observe_distance_ < p.observe_distance) p.observe_distance = observe_distance_;
    p.last_observe_time = observe_time_;
    p.N_rgb++;
    return 1;
}

uint64_t orc_voxel_hash(int16_t x, int16_t y, int16_t z) { return (uint64_t)voxel_hash()(voxel(x, y, z)); }


// ---- colour map C API ---------------------------------------------------------------------------------
void* orc_color_create(void) { return new ColorMap(); }
void orc_color_destroy(void* cm) { delete static_cast<ColorMap*>(cm); }

// the colour branch of lioOptimization::addPointsToMap (src/lioOptimization.cpp:520-551)
int64_t orc_color_add_points(void* cm_, const double* xyz, int64_t n, double voxel_size, int32_t max_num_points_in_voxel,
                             double min_distance_points, int32_t add_point_step, double time_sweep_end, double time_last_process,
                             int32_t to_rendering) {
    ColorMap& cm = *static_cast<ColorMap*>(cm_);
    if (to_rendering) { cm.recent_temp.clear(); std::vector<voxelId>().swap(cm.recent_temp); }
    int number_of_voxels_before_add = (int)cm.recent_temp.size();
    int64_t stored = 0;
    int point_idx = 0;
    for (int64_t i = 0; i < n; ++i) {
        rgbPoint rgb_point({{xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]}});
        if (point_idx % add_point_step == 0)
            stored += addPointToColorMap(cm, rgb_point, voxel_size, max_num_points_in_voxel, min_distance_points, 0, time_sweep_end, time_last_process);
        point_idx++;
    }
    if (to_rendering) {
        cm.recent = cm.recent_temp;
        cm.number_of_new_visited_voxel = (long)cm.recent.size() - number_of_voxels_before_add;
    }
    return stored;
}

// rgbMapTracker::renderPointsInRecentVoxel (src/rgbMapTracker.cpp:181-237) over map_tracker->voxels_recent_visited.
// cam: q_camera_world (x,y,z,w), t_camera_world, t_world_camera, fx, fy, cx, cy, fov_margin  (17 doubles); image BGR u8.
int64_t orc_color_render(void* cm_, const double* cam, const uint8_t* image, int32_t rows, int32_t cols, double obs_time) {
    ColorMap& cm = *static_cast<ColorMap*>(cm_);
    const Mat3 R = quat_to_rot({cam[0], cam[1], cam[2], cam[3]});
    const Vec3 t_cw = {{cam[4], cam[5], cam[6]}}, t_wc = {{cam[7], cam[8], cam[9]}};
    const double fx = cam[10], fy = cam[11], cx = cam[12], cy = cam[13], fov_margin = cam[14];
    const double image_obs_cov = 15;
    const double sigma[3] = {image_obs_cov, image_obs_cov, image_obs_cov};
    int64_t render_point_count = 0;
    auto pix = [&](int r, int c, int ch) -> unsigned char { return image[((size_t)r * cols + c) * 3 + ch]; };
    for (const voxelId& id : cm.recent) {
        voxelBlock& voxel_block = cm.map[voxel((short)id.kx, (short)id.ky, (short)id.kz)];
        for (int point_index = 0; point_index < voxel_block.NumPoints(); point_index++) {
            rgbPoint& point = voxel_block.points[(size_t)point_index];
            const Vec3 point_world = point.getPosition();
            // project3dTo2d (src/lioOptimization.cpp:132-152), scale 1
            const Vec3 pc = vadd(matvec(R, point_world), t_cw);
            if (pc[2] < 0.001) continue;
            double u = (pc[0] * fx / pc[2] + cx) * 1.0;
            double v = (pc[1] * fy / pc[2] + cy) * 1.0;
            // if2dPointsAvailable (:49-60)
            if (!((u / 1.0 >= (fov_margin * cols + 1)) && (std::ceil(u / 1.0) < ((1 - fov_margin) * cols)) &&
                  (v / 1.0 >= (fov_margin * rows + 1)) && (std::ceil(v / 1.0) < ((1 - fov_margin) * rows)))) continue;
            const double point_camera_norm = norm3(vsub(point_world, t_wc));
            // getSubPixel<cv::Vec3b>(rgb_image, v, u, 0) (:71-98): four saturated products, three saturated sums
            const int floor_row = (int)std::floor(v), floor_col = (int)std::floor(u);
            const double frac_row = v - floor_row, frac_col = u - floor_col;
            const int ceil_row = floor_row + 1, ceil_col = floor_col + 1;
            double color[3];
            for (int ch = 0; ch < 3; ++ch) {
                const unsigned char a = sat_u8(pix(floor_row, floor_col, ch) * ((1.0 - frac_row) * (1.0 - frac_col)));
                const unsigned char b = sat_u8(pix(ceil_row, floor_col, ch) * (frac_row * (1.0 - frac_col)));
                const unsigned char c = sat_u8(pix(floor_row, ceil_col, ch) * ((1.0 - frac_row) * frac_col));
                const unsigned char d = sat_u8(pix(ceil_row, ceil_col, ch) * (frac_row * frac_col));
                color[ch] = (double)sat_add_u8(sat_add_u8(sat_add_u8(a, b), c), d);
            }
            if (updateRgb(point, color, point_camera_norm, sigma, obs_time)) render_point_count++;
        }
    }
    return render_point_count;
}

int64_t orc_color_num_voxels(void* cm) { return (int64_t) static_cast<ColorMap*>(cm)->map.size(); }
int64_t orc_color_num_rgb_points(void* cm) { return (int64_t) static_cast<ColorMap*>(cm)->rgb_points.size(); }
int64_t orc_color_num_recent(void* cm) { return (int64_t) static_cast<ColorMap*>(cm)->recent.size(); }
int64_t orc_color_num_new_recent(void* cm) { return (int64_t) static_cast<ColorMap*>(cm)->number_of_new_visited_voxel; }
// voxel contents in container order: keys nv*3, counts nv, xyz nv*cap*3, rgb nv*cap*3, n_rgb nv*cap, cov nv*cap*3,
// obs_dist nv*cap, last_obs nv*cap, last_visited nv
int64_t orc_color_snapshot(void* cm_, int32_t cap, int16_t* keys, int32_t* counts, float* xyz, int16_t* rgb, int16_t* n_rgb,
                           float* cov, double* obs_dist, double* last_obs, double* last_visited) {
    ColorMap& cm = *static_cast<ColorMap*>(cm_);
    int64_t v = 0;
    for (auto& it : cm.map) {
        keys[3 * v] = it.first.x; keys[3 * v + 1] = it.first.y; keys[3 * v + 2] = it.first.z;
        const int c = std::min<int>(it.second.NumPoints(), cap);
        counts[v] = c;
        last_visited[v] = it.second.last_visited_time;
        for (int i = 0; i < cap; ++i) {
            const size_t e = (size_t)v * cap + i;
            const rgbPoint* p = i < c ? &it.second.points[(size_t)i] : nullptr;
            for (int a = 0; a < 3; ++a) {
                xyz[e * 3 + a] = p ? p->position[a] : 0.f;
                rgb[e * 3 + a] = p ? p->rgb[a] : (short)0;
                cov[e * 3 + a] = (p && p->N_rgb != 0) ? p->cov_rgb[a] : 0.f;   // cov_rgb is uninitialised before the first view; a wrapped (negative) N_rgb has one
            }
            n_rgb[e] = p ? p->N_rgb : (short)0;
            obs_dist[e] = p ? p->observe_distance : 0.0;
            last_obs[e] = p ? p->last_observe_time : 0.0;
        }
        ++v;
    }
    return v;
}
void orc_color_lists(void* cm_, int16_t* rgb_points /* n*4 */, int32_t* recent /* m*3 */) {
    ColorMap& cm = *static_cast<ColorMap*>(cm_);
    for (size_t i = 0; i < cm.rgb_points.size(); ++i) for (int a = 0; a < 4; ++a) rgb_points[4 * i + a] = cm.rgb_points[i][(size_t)a];
    for (size_t i = 0; i < cm.recent.size(); ++i) { recent[3 * i] = cm.recent[i].kx; recent[3 * i + 1] = cm.recent[i].ky; recent[3 * i + 2] = cm.recent[i].kz; }
}

}  // extern "C"
