// srl_math.cuh — per-keypoint FP64 math of the scan-matching kernel, host+device.
//
// Everything here is the GPU implementation of what the reference does per keypoint after the
// neighbour search: computeNeighborhoodDistribution (src/optimize.cpp:316-353), the normal flip and
// weight (src/optimize.cpp:42-61,87-88), the signed point-to-plane distance and the 1x6 Jacobian
// (src/optimize.cpp:90-101).  It is compiled for the device (phase 2 of k1_assoc, one thread per
// keypoint) and for the host (srl_host_plane_fit unit hook + the CPU tests of this math).
#pragma once

#include <cmath>
#include <cstdint>

#if defined(__CUDACC__)
#define SRL_HD __host__ __device__ __forceinline__
#else
#define SRL_HD inline
#endif

namespace srl {

// Association-critical arithmetic must not be FMA-contracted: the reference is built without
// -march/-mfma (CMakeLists.txt:4), so its x86 code rounds every product and sum separately.
#if defined(__CUDA_ARCH__)
#define SRL_MUL(a, b) __dmul_rn((a), (b))
#define SRL_ADD(a, b) __dadd_rn((a), (b))
#define SRL_SUB(a, b) __dsub_rn((a), (b))
#define SRL_DIV(a, b) __ddiv_rn((a), (b))
#else
// host build: compiled with -ffp-contract=off (see __graft_entry__.build)
#define SRL_MUL(a, b) ((a) * (b))
#define SRL_ADD(a, b) ((a) + (b))
#define SRL_SUB(a, b) ((a) - (b))
#define SRL_DIV(a, b) ((a) / (b))
#endif

// Eigen's fixed-size 3-term reduction order: c0 + (c1 + c2)
SRL_HD double dot3_exact(double a0, double a1, double a2, double b0, double b1, double b2) {
    return SRL_ADD(SRL_MUL(a0, b0), SRL_ADD(SRL_MUL(a1, b1), SRL_MUL(a2, b2)));
}
// y = M x (row-major 3x3), rows reduced as c0 + (c1 + c2)
SRL_HD void matvec3_exact(const double* M, double x0, double x1, double x2, double& y0, double& y1, double& y2) {
    y0 = dot3_exact(M[0], M[1], M[2], x0, x1, x2);
    y1 = dot3_exact(M[3], M[4], M[5], x0, x1, x2);
    y2 = dot3_exact(M[6], M[7], M[8], x0, x1, x2);
}

// Eigen::Quaterniond::toRotationMatrix, q = (x, y, z, w)
SRL_HD void quat_to_rot(const double* q, double* R) {
    const double tx = 2.0 * q[0], ty = 2.0 * q[1], tz = 2.0 * q[2];
    const double twx = tx * q[3], twy = ty * q[3], twz = tz * q[3];
    const double txx = tx * q[0], txy = ty * q[0], txz = tz * q[0];
    const double tyy = ty * q[1], tyz = tz * q[1], tzz = tz * q[2];
    R[0] = 1.0 - (tyy + tzz); R[1] = txy - twz;         R[2] = txz + twy;
    R[3] = txy + twz;         R[4] = 1.0 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy;         R[7] = tyz + twx;         R[8] = 1.0 - (txx + tyy);
}

// ---------------------------------------------------------------------------------------------
// Symmetric 3x3 eigen-decomposition: scale, Householder tridiagonalisation, implicit QR with
// Wilkinson shift (the algorithm behind Eigen::SelfAdjointEigenSolver<Matrix3d>::compute, which
// the reference calls at src/optimize.cpp:339), written with scalars only so it lives in registers.
// Input: lower triangle s00 s10 s11 s20 s21 s22.  Output: eigenvalues ascending ev[3] and the unit
// eigenvector of the smallest one (n0,n1,n2) (sign arbitrary, fixed later by the flip test).
// ---------------------------------------------------------------------------------------------
// A FP64 division or square root is a ~35-instruction subroutine on the GPU and the per-keypoint fit is one dependent chain
// per thread (k1_fit: a single wave of ~21 warps per SM, bound by that chain): on the device reciprocals and reciprocal
// square roots (MUFU seed + Newton steps, ~1 ulp) followed by multiplies replace them wherever only the 1e-5 relative
// parity of the plane / residual is at stake.  Association-critical arithmetic (keys, distances that order neighbours)
// never goes through these.  The host build keeps the textbook operations.
#if defined(__CUDA_ARCH__)
SRL_HD double fast_rcp(double x) { return __drcp_rn(x); }
SRL_HD double fast_rsqrt(double x) { return rsqrt(x); }
#else
SRL_HD double fast_rcp(double x) { return 1.0 / x; }
SRL_HD double fast_rsqrt(double x) { return 1.0 / sqrt(x); }
#endif

struct Givens { double c, s; };
SRL_HD Givens make_givens(double p, double q) {
    Givens g;
    if (q == 0.0) { g.c = p < 0.0 ? -1.0 : 1.0; g.s = 0.0; }
    else if (p == 0.0) { g.c = 0.0; g.s = q < 0.0 ? 1.0 : -1.0; }
#if defined(__CUDA_ARCH__)
    else {   // both branches below reduce to c = p / r, s = -q / r with r = sqrt(p^2 + q^2); operands are scaled to <= 1
        const double rinv = fast_rsqrt(p * p + q * q);
        g.c = p * rinv; g.s = -q * rinv;
    }
#else
    else if (fabs(p) > fabs(q)) {
        double t = q / p, u = sqrt(1.0 + t * t);
        if (p < 0.0) u = -u;
        g.c = 1.0 / u; g.s = -t * g.c;
    } else {
        double t = p / q, u = sqrt(1.0 + t * t);
        if (q < 0.0) u = -u;
        g.s = -1.0 / u; g.c = -t * g.s;
    }
#endif
    return g;
}

SRL_HD void eig3_sym(double s00, double s10, double s11, double s20, double s21, double s22,
                     double ev[3], double& n0, double& n1, double& n2) {
    double scale = fmax(fmax(fabs(s00), fabs(s10)), fmax(fmax(fabs(s11), fabs(s20)), fmax(fabs(s21), fabs(s22))));
    if (scale == 0.0) scale = 1.0;
#if defined(__CUDA_ARCH__)
    { const double is = fast_rcp(scale); s00 *= is; s10 *= is; s11 *= is; s20 *= is; s21 *= is; s22 *= is; }
#else
    s00 /= scale; s10 /= scale; s11 /= scale; s20 /= scale; s21 /= scale; s22 /= scale;
#endif

    double d0, d1, d2, e0, e1;
    // Q columns: q?0 q?1 q?2
    double q00 = 1, q01 = 0, q02 = 0, q10 = 0, q11, q12, q20 = 0, q21, q22;
    d0 = s00;
    const double tiny = 2.2250738585072014e-308;
    double v1norm2 = s20 * s20;
    if (v1norm2 <= tiny) {
        d1 = s11; d2 = s22; e0 = s10; e1 = s21;
        q11 = 1; q12 = 0; q21 = 0; q22 = 1;
    } else {
#if defined(__CUDA_ARCH__)
        const double b2 = s10 * s10 + v1norm2;
        double invBeta = fast_rsqrt(b2);
        double beta = b2 * invBeta;
#else
        double beta = sqrt(s10 * s10 + v1norm2);
        double invBeta = 1.0 / beta;
#endif
        double m01 = s10 * invBeta, m02 = s20 * invBeta;
        double qq = 2.0 * m01 * s21 + m02 * (s22 - s11);
        d1 = s11 + m02 * qq;
        d2 = s22 - m02 * qq;
        e0 = beta;
        e1 = s21 - m01 * qq;
        q11 = m01; q12 = m02; q21 = m02; q22 = -m01;
    }

    const double precision = 2.0 * 2.220446049250313e-16;
    for (int iter = 0; iter < 90; ++iter) {
        if (fabs(e0) <= (fabs(d0) + fabs(d1)) * precision || fabs(e0) <= tiny) e0 = 0.0;
        if (fabs(e1) <= (fabs(d1) + fabs(d2)) * precision || fabs(e1) <= tiny) e1 = 0.0;
        // largest unreduced block [start, end]
        int end = (e1 != 0.0) ? 2 : ((e0 != 0.0) ? 1 : 0);
        if (end == 0) break;
        int start = (end == 2 && e0 != 0.0) ? 0 : end - 1;

        // Wilkinson shift from the trailing 2x2 of the block
        double da = (end == 2) ? d1 : d0, db = (end == 2) ? d2 : d1, eb = (end == 2) ? e1 : e0;
        double td = (da - db) * 0.5;
        double mu = db;
        if (td == 0.0) {
            mu -= fabs(eb);
        } else if (eb != 0.0) {
            double e2 = eb * eb;
#if defined(__CUDA_ARCH__)
            double h = sqrt(td * td + e2);                 // scaled operands: no overflow to guard against
            double den = td + (td > 0.0 ? h : -h);
            if (e2 == 0.0) mu -= eb / (den / eb);
            else mu -= e2 * fast_rcp(den);
#else
            double h = hypot(td, eb);
            double den = td + (td > 0.0 ? h : -h);
            if (e2 == 0.0) mu -= eb / (den / eb);
            else mu -= e2 / den;
#endif
        }
        double x = ((start == 0) ? d0 : d1) - mu;
        double z = (start == 0) ? e0 : e1;
        // k = 0 rotation (rows/cols 0,1)
        if (start == 0 && z != 0.0) {
            Givens r = make_givens(x, z);
            double sdk = r.s * d0 + r.c * e0;
            double dkp1 = r.s * e0 + r.c * d1;
            d0 = r.c * (r.c * d0 - r.s * e0) - r.s * (r.c * e0 - r.s * d1);
            d1 = r.s * sdk + r.c * dkp1;
            e0 = r.c * sdk - r.s * dkp1;
            x = e0;
            if (end == 2) { z = -r.s * e1; e1 = r.c * e1; }
            double a, b;
            a = q00; b = q01; q00 = r.c * a - r.s * b; q01 = r.s * a + r.c * b;
            a = q10; b = q11; q10 = r.c * a - r.s * b; q11 = r.s * a + r.c * b;
            a = q20; b = q21; q20 = r.c * a - r.s * b; q21 = r.s * a + r.c * b;
        }
        // k = 1 rotation (rows/cols 1,2)
        if (end == 2 && z != 0.0) {
            Givens r = make_givens(x, z);
            double sdk = r.s * d1 + r.c * e1;
            double dkp1 = r.s * e1 + r.c * d2;
            d1 = r.c * (r.c * d1 - r.s * e1) - r.s * (r.c * e1 - r.s * d2);
            d2 = r.s * sdk + r.c * dkp1;
            e1 = r.c * sdk - r.s * dkp1;
            if (start == 0) e0 = r.c * e0 - r.s * z;
            double a, b;
            a = q01; b = q02; q01 = r.c * a - r.s * b; q02 = r.s * a + r.c * b;
            a = q11; b = q12; q11 = r.c * a - r.s * b; q12 = r.s * a + r.c * b;
            a = q21; b = q22; q21 = r.c * a - r.s * b; q22 = r.s * a + r.c * b;
        }
    }
    // ascending order; carry the eigenvector of the smallest eigenvalue
    int imin = 0;
    double lo = d0;
    if (d1 < lo) { lo = d1; imin = 1; }
    if (d2 < lo) { lo = d2; imin = 2; }
    double r0 = (imin == 0) ? d1 : d0, r1 = (imin == 2) ? d1 : d2;   // the two that remain
    double mid = fmin(r0, r1), hi = fmax(r0, r1);
    double vx = (imin == 0) ? q00 : ((imin == 1) ? q01 : q02);
    double vy = (imin == 0) ? q10 : ((imin == 1) ? q11 : q12);
    double vz = (imin == 0) ? q20 : ((imin == 1) ? q21 : q22);
    ev[0] = lo * scale; ev[1] = mid * scale; ev[2] = hi * scale;
    double nn = vx * vx + (vy * vy + vz * vz);
#if defined(__CUDA_ARCH__)
    if (nn > 0.0) { const double rs = fast_rsqrt(nn); vx *= rs; vy *= rs; vz *= rs; }
#else
    if (nn > 0.0) { double inv = sqrt(nn); vx /= inv; vy /= inv; vz /= inv; }
#endif
    n0 = vx; n1 = vy; n2 = vz;
}

// ---------------------------------------------------------------------------------------------
// Closed-form variant for the device (k1_fit is one dependent chain per thread, and the QR iteration above runs for the
// slowest lane of the warp: 6-8 rounds of Givens rotations, each with reciprocal square roots, where the lanes need 3-5):
// eigenvalues by the trigonometric solution of the characteristic cubic, the eigenvector of the smallest one as the
// largest cross product of two rows of A - lambda_min I.  No data-dependent loop, no divergence.  The smallest eigenvalue
// carries an absolute error of ~eps * lambda_max (it enters the planarity only through sqrt(|lambda_min|) / sqrt(lambda_max),
// far inside the 1e-5 budget), the eigenvector an error of ~eps * lambda_max / (lambda_mid - lambda_min).  Returns false —
// the caller then runs the QR iteration, i.e. the reference's algorithm — when the matrix is (numerically) a multiple
// of the identity or the two smallest eigenvalues are closer than 1e-3 of the spread, where that bound degrades (host test
// over the ones of 200k random planar / edge-like scatter matrices that pass this test: normal within 5e-11, planarity within 3e-8 of the QR result).
// ---------------------------------------------------------------------------------------------
SRL_HD bool eig3_sym_closed(double s00, double s10, double s11, double s20, double s21, double s22, double ev[3], double& n0,
                            double& n1, double& n2) {
    const double scale = fmax(fmax(fabs(s00), fabs(s10)), fmax(fmax(fabs(s11), fabs(s20)), fmax(fabs(s21), fabs(s22))));
    if (!(scale > 0.0)) return false;
    const double is = fast_rcp(scale);
    const double a00 = s00 * is, a01 = s10 * is, a11 = s11 * is, a02 = s20 * is, a12 = s21 * is, a22 = s22 * is;
    const double q = (a00 + a11 + a22) * (1.0 / 3.0);
    const double b00 = a00 - q, b11 = a11 - q, b22 = a22 - q;
    const double p1 = a01 * a01 + a02 * a02 + a12 * a12;
    const double p2 = b00 * b00 + b11 * b11 + b22 * b22 + 2.0 * p1;
    if (!(p2 > 1e-24)) return false;
    const double ip = fast_rsqrt(p2 * (1.0 / 6.0));            // 1 / p
    const double p = p2 * (1.0 / 6.0) * ip;
    // r = det((A - qI) / p) / 2, clamped: |r| may exceed 1 by rounding
    const double c00 = b00 * ip, c11 = b11 * ip, c22 = b22 * ip, c01 = a01 * ip, c02 = a02 * ip, c12 = a12 * ip;
    double r = 0.5 * (c00 * (c11 * c22 - c12 * c12) - c01 * (c01 * c22 - c12 * c02) + c02 * (c01 * c12 - c11 * c02));
    r = fmin(1.0, fmax(-1.0, r));
    const double phi = acos(r) * (1.0 / 3.0);
    double sn, cs;
#if defined(__CUDA_ARCH__)
    sincos(phi, &sn, &cs);
#else
    sn = sin(phi); cs = cos(phi);
#endif
    // cos(phi + 2 pi / 3) = -cos(phi) / 2 - sqrt(3) / 2 * sin(phi)
    const double lmax = q + 2.0 * p * cs;
    const double lmin = q + 2.0 * p * (-0.5 * cs - 0.86602540378443864676 * sn);
    const double lmid = 3.0 * q - lmax - lmin;
    // the two smallest eigenvalues close together (edges, poles: r -> 1) is where acos loses up to half the digits of lmin
    // and the null vector of A - lmin I is poorly determined: leave those to the QR iteration
    if (!((lmid - lmin) > 1e-3 * (lmax - lmin))) return false;
    // eigenvector of lmin: rows of A - lmin I, the largest of the three cross products
    const double m00 = a00 - lmin, m11 = a11 - lmin, m22 = a22 - lmin;
    const double x0 = a01 * a12 - a02 * m11, y0 = a02 * a01 - m00 * a12, z0 = m00 * m11 - a01 * a01;      // r0 x r1
    const double x1 = a01 * m22 - a02 * a12, y1 = a02 * a02 - m00 * m22, z1 = m00 * a12 - a01 * a02;      // r0 x r2
    const double x2 = m11 * m22 - a12 * a12, y2 = a12 * a02 - a01 * m22, z2 = a01 * a12 - m11 * a02;      // r1 x r2
    const double w0 = x0 * x0 + (y0 * y0 + z0 * z0), w1 = x1 * x1 + (y1 * y1 + z1 * z1), w2 = x2 * x2 + (y2 * y2 + z2 * z2);
    double vx = x0, vy = y0, vz = z0, w = w0;
    if (w1 > w) { vx = x1; vy = y1; vz = z1; w = w1; }
    if (w2 > w) { vx = x2; vy = y2; vz = z2; w = w2; }
    if (!(w > 1e-20)) return false;
    const double rs = fast_rsqrt(w);
    n0 = vx * rs; n1 = vy * rs; n2 = vz * rs;
    ev[0] = lmin * scale; ev[1] = lmid * scale; ev[2] = lmax * scale;
    return true;
}

// ---------------------------------------------------------------------------------------------
// constants of one ESIKF pass (host-computed once, passed by value to the kernel)
// ---------------------------------------------------------------------------------------------
struct PassConst {
    double Rn[9];     // end_quat.normalized().toRotationMatrix()  (src/optimize.cpp:35)
    double Rq[9];     // end_quat.toRotationMatrix()               (src/optimize.cpp:95,101)
    double t[3];      // end_t
    double t_last[3]; // last_state->translation
    double R_il[9];
    double t_il[3];
    double size;          // size_voxel_map
    double lambda_w;      // normalised weights (src/optimize.cpp:55-61)
    double lambda_n;
    double power;         // power_planarity
    double dmax;          // max_dist_to_plane_icp
    double exp_den;       // kMaxPointToPlane * kMinNumNeighbors
    int K;                // max_number_neighbors
    int Kmin;             // min_number_neighbors
    int nb;               // voxels visited per side
    int thr_occ;          // threshold_voxel_occupancy (effective)
    double inv_size;      // 1 / size when size is a power of two (then x * inv_size == x / size bit for bit), else 0
    double pad_;
};
// the voxel coordinate of src/optimize.cpp:372-374 before truncation: a correctly rounded division (a ~35-instruction
// subroutine on the GPU), or one multiply when the voxel size is a power of two — the quotient is exact either way then
SRL_HD double voxel_quotient(double x, const PassConst& c) { return c.inv_size != 0.0 ? SRL_MUL(x, c.inv_size) : SRL_DIV(x, c.size); }

struct PlaneRow {
    double nx, ny, nz;   // norm_vector
    double J[6];
    double offset, distance, weight, a2D;
    int accepted;        // distance < dmax
    int nan_planarity;
};

// Neighbour accessor NB: nbv.get(j, x, y, z) yields the j-th stored neighbour (FP32 map coordinates) and
// nbv.use(j) says whether slot j is one of the K neighbours (= vector_neighbors, src/optimize.cpp:73); KS > 0 is the
// compile-time number of SLOTS (>= K).  (n0x,n0y,n0z) is the NEAREST neighbour (vector_neighbors[0]).
// p = keypoint in world frame, b = R_il*raw + t_il.  KS > 0 makes the neighbour loops compile-time (registers).
template <int KS, class NB>
SRL_HD void plane_residual(const NB& nbv, int K, double n0x, double n0y, double n0z, const PassConst& c, double px, double py,
                           double pz, double bx, double by, double bz, PlaneRow& out) {
    // barycenter: sequential sum then divide (src/optimize.cpp:320-326)
    double mx = 0.0, my = 0.0, mz = 0.0;
#pragma unroll
    for (int j = 0; j < (KS > 0 ? KS : K); ++j) {
        if (!nbv.use(j)) continue;
        float x, y, z;
        nbv.get(j, x, y, z);
        mx += (double)x; my += (double)y; mz += (double)z;
    }
#if defined(__CUDA_ARCH__)
    { const double invK = fast_rcp((double)K); mx *= invK; my *= invK; mz *= invK; }
#else
    mx /= (double)K; my /= (double)K; mz /= (double)K;
#endif
    // un-normalised scatter, upper triangle (src/optimize.cpp:328-338)
    double c00 = 0, c01 = 0, c02 = 0, c11 = 0, c12 = 0, c22 = 0;
#pragma unroll
    for (int j = 0; j < (KS > 0 ? KS : K); ++j) {
        if (!nbv.use(j)) continue;
        float x, y, z;
        nbv.get(j, x, y, z);
        double dx = (double)x - mx, dy = (double)y - my, dz = (double)z - mz;
        c00 += dx * dx; c01 += dx * dy; c02 += dx * dz; c11 += dy * dy; c12 += dy * dz; c22 += dz * dz;
    }
    // K copies of one point: the reference's scatter is exactly 0, its a2D 0 / 0, and it throws (:348).  The device's
    // arithmetic (a rounded 1 / K, contracted products) can leave a scatter of a few FP64 ulp^2 instead -- k1_fast's fit
    // returned a2D ~ -2e-9 for such a neighbourhood.  That residue stays below 2^-90 |nearest|^2 (a mean off by 2 ulp at
    // most), so only a scatter that small has its points compared with the nearest one.
    bool collapsed = false;
    if (!(c00 + c11 + c22 > 8.0779356694631609e-28 * (n0x * n0x + n0y * n0y + n0z * n0z))) {
        collapsed = true;
#pragma unroll
        for (int j = 0; j < (KS > 0 ? KS : K); ++j) {
            if (!nbv.use(j)) continue;
            float x, y, z;
            nbv.get(j, x, y, z);
            collapsed = collapsed && (double)x == n0x && (double)y == n0y && (double)z == n0z;
        }
    }
    double ev[3], nx, ny, nz;
#if defined(__CUDA_ARCH__)
    if (!eig3_sym_closed(c00, c01, c11, c02, c12, c22, ev, nx, ny, nz))
#endif
    eig3_sym(c00, c01, c11, c02, c12, c22, ev, nx, ny, nz);
#if defined(__CUDA_ARCH__)
    double sigma_2 = sqrt(fabs(ev[1])), sigma_3 = sqrt(fabs(ev[0]));
    double a2D = (sigma_2 - sigma_3) * fast_rsqrt(fabs(ev[2]));   // (0 - 0) * inf = NaN like the reference's 0 / 0
#else
    double sigma_1 = sqrt(fabs(ev[2])), sigma_2 = sqrt(fabs(ev[1])), sigma_3 = sqrt(fabs(ev[0]));
    double a2D = (sigma_2 - sigma_3) / sigma_1;           // src/optimize.cpp:343-346
#endif
    if (collapsed) a2D = nan("");
    out.a2D = a2D;
    out.nan_planarity = (a2D != a2D) ? 1 : 0;
    double planarity_weight = (c.power == 2.0) ? a2D * a2D : pow(a2D, c.power);   // :47
    // normal flip: world-frame normal against body-frame location, as in the reference (:49-51)
    if (nx * (c.t_last[0] - bx) + (ny * (c.t_last[1] - by) + nz * (c.t_last[2] - bz)) < 0.0) { nx = -nx; ny = -ny; nz = -nz; }
    // weight (:87-88)
    double ex = n0x - px, ey = n0y - py, ez = n0z - pz;
    double dist0 = sqrt(ex * ex + (ey * ey + ez * ez));
#if defined(__CUDA_ARCH__)
    double weight = c.lambda_w * planarity_weight + c.lambda_n * exp(-dist0 * fast_rcp(c.exp_den));
#else
    double weight = c.lambda_w * planarity_weight + c.lambda_n * exp(-dist0 / c.exp_den);
#endif
    // plane (:92-96)
    double nn = nx * nx + (ny * ny + nz * nz);
#if defined(__CUDA_ARCH__)
    if (nn > 0.0) { const double rs = fast_rsqrt(nn); nx *= rs; ny *= rs; nz *= rs; }
#else
    if (nn > 0.0) { double s = sqrt(nn); nx /= s; ny /= s; nz /= s; }
#endif
    double offset = -(nx * n0x + (ny * n0y + nz * n0z));
    double wx = c.Rq[0] * bx + (c.Rq[1] * by + c.Rq[2] * bz) + c.t[0];
    double wy = c.Rq[3] * bx + (c.Rq[4] * by + c.Rq[5] * bz) + c.t[1];
    double wz = c.Rq[6] * bx + (c.Rq[7] * by + c.Rq[8] * bz) + c.t[2];
    double distance = nx * wx + (ny * wy + nz * wz) + offset;
    out.nx = nx; out.ny = ny; out.nz = nz;
    out.offset = offset; out.distance = distance; out.weight = weight;
    out.accepted = (distance < c.dmax) ? 1 : 0;            // signed gate (:98)
    // Jacobian (:100-101):  [ w n^T ,  -w n^T R' [b]x ]
    double rx = -(nx * c.Rq[0] + (ny * c.Rq[3] + nz * c.Rq[6]));
    double ry = -(nx * c.Rq[1] + (ny * c.Rq[4] + nz * c.Rq[7]));
    double rz = -(nx * c.Rq[2] + (ny * c.Rq[5] + nz * c.Rq[8]));
    out.J[0] = nx * weight; out.J[1] = ny * weight; out.J[2] = nz * weight;
    // row * skew(b): [ ry*bz - rz*by , rz*bx - rx*bz , rx*by - ry*bx ]
    out.J[3] = (ry * bz - rz * by) * weight;
    out.J[4] = (rz * bx - rx * bz) * weight;
    out.J[5] = (rx * by - ry * bx) * weight;
}

}  // namespace srl
