// srl_lk.cu — the optical-flow tracker's pyramidal Lucas-Kanade on the device: LKOpticalFlowKernel::trackImage
// (src/lkpyramid.cpp:755-795), bit for bit.
//
// Each image is built once into one of two buffer sets (the reference's curr_img_pyr / curr_img_deriv_I_buff) and serves as
// the previous image of the next call; the sets swap by pointer, as swapImageBuffer does.  Per set and level:
//   img  (rows + 2 win_h) x (cols + 2 win_w) bytes: the level with a REFLECT_101 border of the window's size (:541-588)
//   der  the same count of (Ix, Iy) shorts: calcSharrDeriv of the level (:57-154) inside, zero in the border (:646-668)
// The level's own pixels sit at (win_h, win_w).  Level 0 is the image, level l the pyrDown of level l-1.  pyrDown and the
// Scharr filter both read the padded level instead of applying their own REFLECT_101 index rule: the padding is REFLECT_101 and
// at least 3 wide, and both reach at most 2 (pyrDown) or 1 (Scharr) pixels past an edge, so they read the same pixels.
//
// k_lk_track: one warp per point, every level from max_level down to 0 (calculateLKOpticalFlow, :174-496, err == nullptr).
// The integer work (14-bit bilinear weights, the window patch, the temporal differences) is spread over the lanes; the float
// sums run as serial chains in the reference's SSE2 lane order, one chain per lane:
//   A11/A12/A22 (:257-330): lanes 0-11 are the four SSE lanes of each (x = 4c + lane % 4 over rows, then chunks), lanes 12-14
//     the scalar tails (x >= 4 * (w / 4)); then A = tail + (((l0 + l1) + l2) + l3)
//   b1/b2 (:382-435): lanes 0-7 are the lanes of qb0 and qb1 (each the float of one _mm_madd_epi16 pair per 8-pixel chunk), lanes
//     8-9 the scalar tails (x >= 8 * (w / 8)); then bbuf = qb0 + qb1, ib1 = tail1 + (bbuf0 + bbuf2), ib2 = tail2 + (bbuf1 + bbuf3)
// The integer products are exact; the partial sums exceed 2^24, so their order decides the bits.  Every float operation that
// matters is an explicit _rn intrinsic (no contraction; the file is also built with --fmad=false), sqrt and division are IEEE.
// Magnitudes (tests/test_lk_edges_pin.py pins them on 0/255 scenes): |Scharr| <= 4080, |diff| <= 8160, so every weighted sum
// fits 32 bits and packs/subs never saturate, while a madd pair reaches 2 * 8160 * 4080 > 2^24 and a tail product 8160 * 4080:
// their int -> float conversions round, as _mm_cvtepi32_ps / cvtsi2ss round them, to nearest even (__int2float_rn).
// Non-finite and huge coordinates: cvFloor gives INT_MIN outside the int range and for NaN, so such a point is outside at
// every level and only scaled; a NaN comes back as the input NaN with its quiet bit set, as the reference's x86 code returns it.
#include <algorithm>
#include <cfloat>
#include <climits>
#include <cstring>

#include "srl_internal.h"

using namespace srl;

namespace {

constexpr int kLkMaxLevels = 9;        // max_level 0..8
constexpr int kLkWarps = 4;            // points per block of k_lk_track
constexpr int kLkBlock = kLkWarps * 32;

struct LkTrackArgs {
    const float2* prev_pts;
    float2* next_pts;
    uint8_t* status;
    int n;
    int win_w, win_h, max_level, max_count;
    double epsilon;
    float min_eig;
    const uint8_t* I[kLkMaxLevels];    // previous image, padded
    const short2* dI[kLkMaxLevels];    // its derivatives, padded
    const uint8_t* J[kLkMaxLevels];    // this image, padded
    int cols[kLkMaxLevels], rows[kLkMaxLevels];
    unsigned long long* n_tracked;     // += status of every point
};

// cv::borderInterpolate for BORDER_REFLECT_101 (len >= 2)
__device__ __forceinline__ int reflect101(int p, int len) {
    while ((unsigned)p >= (unsigned)len) p = p < 0 ? -p : 2 * len - p - 2;
    return p;
}

// cvFloor as the reference's x86-64 build has it: (int)v (cvttss2si: INT_MIN outside the int range and for NaN) - (i > v)
__device__ __forceinline__ int cv_floor(float v) {
    const int i = (v >= -2147483648.f && v < 2147483648.f) ? __float2int_rz(v) : INT_MIN;
    return i - ((float)i > v ? 1 : 0);
}

// level 0: the image with a REFLECT_101 border of (win_h, win_w)
__global__ void k_lk_level0(const uint8_t* __restrict__ src, size_t src_pitch, int cols, int rows, int ww, int wh, uint8_t* __restrict__ dst) {
    const int pw = cols + 2 * ww, ph = rows + 2 * wh;
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= pw || y >= ph) return;
    dst[(size_t)y * pw + x] = src[(size_t)reflect101(y - wh, rows) * src_pitch + reflect101(x - ww, cols)];
}

// level l from padded level l-1 (cols_s x rows_s inside): pyrDown's [1 4 6 4 1]^2 taps at (2x, 2y), (s + 128) >> 8, written with a
// REFLECT_101 border (the border pixel is the pyrDown value of the pixel it reflects)
__global__ void k_lk_pyrdown(const uint8_t* __restrict__ src, int cols_s, int cols, int rows, int ww, int wh, uint8_t* __restrict__ dst) {
    const int pw = cols + 2 * ww, ph = rows + 2 * wh, spw = cols_s + 2 * ww;
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= pw || y >= ph) return;
    const int ix = reflect101(x - ww, cols), iy = reflect101(y - wh, rows);
    const uint8_t* s = src + (size_t)(2 * iy - 2 + wh) * spw + (2 * ix - 2 + ww);
    int r[5];
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        const uint8_t* q = s + (size_t)k * spw;
        r[k] = q[2] * 6 + (q[1] + q[3]) * 4 + q[0] + q[4];
    }
    dst[(size_t)y * pw + x] = (uint8_t)((r[2] * 6 + (r[1] + r[3]) * 4 + r[0] + r[4] + 128) >> 8);
}

struct LkScharrArgs {
    const uint8_t* img[kLkMaxLevels];
    short2* der[kLkMaxLevels];
    int cols[kLkMaxLevels], rows[kLkMaxLevels];
    int ww, wh;
};
// calcSharrDeriv of every level (blockIdx.z = level): Ix = d/dx of (3, 10, 3) down the column, Iy = d/dy of (3, 10, 3) along the
// row, zero in the border of the derivative buffer
__global__ void k_lk_scharr(const __grid_constant__ LkScharrArgs a) {
    const int l = blockIdx.z;
    const int cols = a.cols[l], rows = a.rows[l];
    const int pw = cols + 2 * a.ww, ph = rows + 2 * a.wh;
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= pw || y >= ph) return;
    short2 d = make_short2(0, 0);
    if (x >= a.ww && x < a.ww + cols && y >= a.wh && y < a.wh + rows) {
        const uint8_t* c = a.img[l] + (size_t)y * pw + x;
        const uint8_t* u = c - pw;
        const uint8_t* b = c + pw;
        const int t0m = (u[-1] + b[-1]) * 3 + c[-1] * 10, t0p = (u[1] + b[1]) * 3 + c[1] * 10;
        const int t1m = b[-1] - u[-1], t1 = b[0] - u[0], t1p = b[1] - u[1];
        d = make_short2((short)(t0p - t0m), (short)((t1p + t1m) * 3 + t1 * 10));
    }
    a.der[l][(size_t)y * pw + x] = d;
}

__device__ __forceinline__ void lk_weights(float a, float b, int& w00, int& w01, int& w10, int& w11) {
    const float ia = __fsub_rn(1.f, a), ib = __fsub_rn(1.f, b);
    w00 = __float2int_rn(__fmul_rn(__fmul_rn(ia, ib), 16384.f));
    w01 = __float2int_rn(__fmul_rn(__fmul_rn(a, ib), 16384.f));
    w10 = __float2int_rn(__fmul_rn(__fmul_rn(ia, b), 16384.f));
    w11 = 16384 - w00 - w01 - w10;
}

__global__ void __launch_bounds__(kLkBlock) k_lk_track(const __grid_constant__ LkTrackArgs A) {
    extern __shared__ __align__(16) unsigned char lk_smem[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int pt = blockIdx.x * kLkWarps + wid;
    if (pt >= A.n) return;   // the whole warp
    const int W = A.win_w, H = A.win_h, area = W * H;
    const size_t stride = ((size_t)area * 8 + 15) & ~(size_t)15;
    short2* dIw = reinterpret_cast<short2*>(lk_smem + stride * wid);   // interpolated (Ix, Iy) of the patch
    short* Iw = reinterpret_cast<short*>(dIw + area);                  // interpolated previous image, << 5
    short* Dw = Iw + area;                                             // this image minus Iw, per iteration
    const float hwx = (W - 1) * 0.5f, hwy = (H - 1) * 0.5f;
    const float FLT_SCALE = 1.f / (1 << 20);
    const float2 p0 = A.prev_pts[pt];
    float2 cur = p0;           // nextPts[ptidx]
    unsigned char st = 1;
    const int nc4 = W / 4, nc8 = W / 8;
    for (int level = A.max_level; level >= 0; --level) {
        const float sc = (float)(1. / (1 << level));
        float px = __fmul_rn(p0.x, sc), py = __fmul_rn(p0.y, sc);
        float nx, ny;
        if (level == A.max_level) { nx = px; ny = py; }   // with OPTFLOW_USE_INITIAL_FLOW nextPts == prevPts here: the same
        else { nx = __fmul_rn(cur.x, 2.f); ny = __fmul_rn(cur.y, 2.f); }
        cur = make_float2(nx, ny);
        px = __fsub_rn(px, hwx);
        py = __fsub_rn(py, hwy);
        const int ipx = cv_floor(px), ipy = cv_floor(py);
        const int cols = A.cols[level], rows = A.rows[level];
        if (ipx < -W || ipx >= cols || ipy < -H || ipy >= rows) {
            if (level == 0) st = 0;
            continue;
        }
        const int pitch = cols + 2 * W;
        int w00, w01, w10, w11;
        lk_weights(__fsub_rn(px, (float)ipx), __fsub_rn(py, (float)ipy), w00, w01, w10, w11);
        {
            const size_t o = (size_t)(ipy + H) * pitch + (ipx + W);
            const uint8_t* __restrict__ Ib = A.I[level] + o;
            const short2* __restrict__ dIb = A.dI[level] + o;
            for (int p = lane; p < area; p += 32) {
                const int y = p / W, x = p - y * W;
                const int q = y * pitch + x;
                const int ival = (__ldg(Ib + q) * w00 + __ldg(Ib + q + 1) * w01 + __ldg(Ib + q + pitch) * w10 + __ldg(Ib + q + pitch + 1) * w11 + (1 << 8)) >> 9;
                const short2 d00 = dIb[q], d01 = dIb[q + 1], d10 = dIb[q + pitch], d11 = dIb[q + pitch + 1];
                const int ix = (d00.x * w00 + d01.x * w01 + d10.x * w10 + d11.x * w11 + (1 << 13)) >> 14;
                const int iy = (d00.y * w00 + d01.y * w01 + d10.y * w10 + d11.y * w11 + (1 << 13)) >> 14;
                Iw[p] = (short)ival;
                dIw[p] = make_short2((short)ix, (short)iy);
            }
        }
        __syncwarp();
        float acc = 0.f;
        if (lane < 12) {            // SSE lane (lane & 3) of A11 (lanes 0-3), A12 (4-7), A22 (8-11)
            const int m = lane >> 2, k = lane & 3;
            for (int y = 0; y < H; ++y)
                for (int c = 0; c < nc4; ++c) {
                    const short2 g = dIw[y * W + 4 * c + k];
                    const float fx = (float)g.x, fy = (float)g.y;
                    acc = __fadd_rn(acc, m == 0 ? __fmul_rn(fx, fx) : m == 1 ? __fmul_rn(fx, fy) : __fmul_rn(fy, fy));
                }
        } else if (lane < 15) {     // scalar tail of A11, A12, A22
            const int m = lane - 12;
            for (int y = 0; y < H; ++y)
                for (int x = 4 * nc4; x < W; ++x) {
                    const short2 g = dIw[y * W + x];
                    acc = __fadd_rn(acc, __int2float_rn(m == 0 ? g.x * g.x : m == 1 ? g.x * g.y : g.y * g.y));
                }
        }
        float Am[3];
#pragma unroll
        for (int m = 0; m < 3; ++m) {
            const float l0 = __shfl_sync(0xffffffffu, acc, 4 * m), l1 = __shfl_sync(0xffffffffu, acc, 4 * m + 1);
            const float l2 = __shfl_sync(0xffffffffu, acc, 4 * m + 2), l3 = __shfl_sync(0xffffffffu, acc, 4 * m + 3);
            const float t = __shfl_sync(0xffffffffu, acc, 12 + m);
            Am[m] = __fmul_rn(__fadd_rn(t, __fadd_rn(__fadd_rn(__fadd_rn(l0, l1), l2), l3)), FLT_SCALE);
        }
        const float A11 = Am[0], A12 = Am[1], A22 = Am[2];
        float D = __fsub_rn(__fmul_rn(A11, A22), __fmul_rn(A12, A12));
        const float dd = __fsub_rn(A11, A22);
        const float disc = __fadd_rn(__fmul_rn(dd, dd), __fmul_rn(__fmul_rn(4.f, A12), A12));
        const float minEig = __fdiv_rn(__fsub_rn(__fadd_rn(A22, A11), __fsqrt_rn(disc)), (float)(2 * W * H));
        if (minEig < A.min_eig || D < FLT_EPSILON) {
            if (level == 0) st = 0;
            continue;
        }
        D = __fdiv_rn(1.f, D);
        nx = __fsub_rn(nx, hwx);
        ny = __fsub_rn(ny, hwy);
        float pdx = 0.f, pdy = 0.f;
        for (int j = 0; j < A.max_count; ++j) {
            const int inx = cv_floor(nx), iny = cv_floor(ny);
            if (inx < -W || inx >= cols || iny < -H || iny >= rows) {
                if (level == 0) st = 0;
                break;
            }
            lk_weights(__fsub_rn(nx, (float)inx), __fsub_rn(ny, (float)iny), w00, w01, w10, w11);
            const uint8_t* __restrict__ Jb = A.J[level] + (size_t)(iny + H) * pitch + (inx + W);
            __syncwarp();   // the previous iteration's chains are done with Dw
            for (int p = lane; p < area; p += 32) {
                const int y = p / W, x = p - y * W;
                const int q = y * pitch + x;
                const int v = (__ldg(Jb + q) * w00 + __ldg(Jb + q + 1) * w01 + __ldg(Jb + q + pitch) * w10 + __ldg(Jb + q + pitch + 1) * w11 + (1 << 8)) >> 9;
                Dw[p] = (short)(v - Iw[p]);
            }
            __syncwarp();
            float bacc = 0.f;
            if (lane < 8) {         // lane k of qb0 (lanes 0-3) and qb1 (4-7): pixel j and j + 4 of each 8-pixel chunk, Ix or Iy
                const int jj = 2 * (lane >> 2) + ((lane & 3) >> 1), comp = lane & 1;
                for (int y = 0; y < H; ++y)
                    for (int c = 0; c < nc8; ++c) {
                        const int b0 = y * W + 8 * c + jj;
                        const short2 g0 = dIw[b0], g4 = dIw[b0 + 4];
                        const int v = comp ? Dw[b0] * g0.y + Dw[b0 + 4] * g4.y : Dw[b0] * g0.x + Dw[b0 + 4] * g4.x;
                        bacc = __fadd_rn(bacc, __int2float_rn(v));
                    }
            } else if (lane < 10) { // scalar tails of ib1 (lane 8) and ib2 (lane 9)
                const int comp = lane - 8;
                for (int y = 0; y < H; ++y)
                    for (int x = 8 * nc8; x < W; ++x) {
                        const int b0 = y * W + x;
                        const short2 g = dIw[b0];
                        bacc = __fadd_rn(bacc, __int2float_rn(Dw[b0] * (comp ? g.y : g.x)));
                    }
            }
            float bb[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) bb[k] = __fadd_rn(__shfl_sync(0xffffffffu, bacc, k), __shfl_sync(0xffffffffu, bacc, 4 + k));
            const float ib1 = __fadd_rn(__shfl_sync(0xffffffffu, bacc, 8), __fadd_rn(bb[0], bb[2]));
            const float ib2 = __fadd_rn(__shfl_sync(0xffffffffu, bacc, 9), __fadd_rn(bb[1], bb[3]));
            const float b1 = __fmul_rn(ib1, FLT_SCALE), b2 = __fmul_rn(ib2, FLT_SCALE);
            const float dx = __fmul_rn(__fsub_rn(__fmul_rn(A12, b2), __fmul_rn(A22, b1)), D);
            const float dy = __fmul_rn(__fsub_rn(__fmul_rn(A12, b1), __fmul_rn(A11, b2)), D);
            nx = __fadd_rn(nx, dx);
            ny = __fadd_rn(ny, dy);
            cur = make_float2(__fadd_rn(nx, hwx), __fadd_rn(ny, hwy));
            if (__dadd_rn(__dmul_rn((double)dx, (double)dx), __dmul_rn((double)dy, (double)dy)) <= A.epsilon) break;
            if (j > 0 && (double)fabsf(__fadd_rn(dx, pdx)) < 0.01 && (double)fabsf(__fadd_rn(dy, pdy)) < 0.01) {
                cur.x = __fsub_rn(cur.x, __fmul_rn(dx, 0.5f));
                cur.y = __fsub_rn(cur.y, __fmul_rn(dy, 0.5f));
                break;
            }
            pdx = dx;
            pdy = dy;
        }
        __syncwarp();   // the chains are done with Iw / dIw before the next level rewrites them
    }
    if (lane == 0) {
        // A NaN coordinate is outside at every level, so its output is only ever scaled.  The reference's x86 products return
        // that NaN with its quiet bit set; PTX arithmetic returns the canonical NaN, so the input's bits are restored here.
        if (isnan(p0.x)) cur.x = __int_as_float(__float_as_int(p0.x) | 0x00400000);
        if (isnan(p0.y)) cur.y = __int_as_float(__float_as_int(p0.y) | 0x00400000);
        A.next_pts[pt] = cur;
        A.status[pt] = st;
        if (st) atomicAdd(A.n_tracked, 1ull);
    }
}

__global__ void k_lk_copy_pts(const float2* __restrict__ src, float2* __restrict__ dst, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = src[i];
}

}  // namespace

struct srl_lk {
    srl_ctx* ctx = nullptr;
    int device = 0;
    int win_w = 21, win_h = 21;
    int max_level = 3;              // LKOpticalFlowKernel::maxLevel: the first image's pyramid build overwrites it (:609-619)
    int max_count = 30;
    double epsilon = 0.01;
    int flags = 0;
    float min_eig = 1e-4f;
    int cols = 0, rows = 0;         // the first image's size; 0 before it
    int lcols[kLkMaxLevels] = {0}, lrows[kLkMaxLevels] = {0};
    uint8_t* img[2][kLkMaxLevels] = {{nullptr}};
    short2* der[2][kLkMaxLevels] = {{nullptr}};
    int prev = 0;                   // the set holding the previous image
    bool have_prev = false;
    unsigned long long* d_count = nullptr;
    cudaEvent_t ev[3] = {nullptr, nullptr, nullptr};   // call start, pyramid built, points tracked
    bool timed = false;
};
srl_ctx* srl::lk_ctx(const srl_lk* lk) { return lk->ctx; }

namespace {

void lk_free(srl_lk* lk) {
    for (int s = 0; s < 2; ++s)
        for (int l = 0; l < kLkMaxLevels; ++l) {
            if (lk->img[s][l]) cudaFree(lk->img[s][l]);
            if (lk->der[s][l]) cudaFree(lk->der[s][l]);
            lk->img[s][l] = nullptr;
            lk->der[s][l] = nullptr;
        }
}

// The first image: the level count of opencvBuildOpticalFlowPyramid (:561-624) and both buffer sets
int lk_allocate(srl_lk* lk, int cols, int rows) {
    srl_ctx* ctx = lk->ctx;
    int w = cols, h = rows, top = lk->max_level;
    for (int level = 0; level <= lk->max_level; ++level) {
        lk->lcols[level] = w;
        lk->lrows[level] = h;
        w = (w + 1) / 2;
        h = (h + 1) / 2;
        if (w <= lk->win_w || h <= lk->win_h) { top = level; break; }
    }
    lk->max_level = top;
    for (int s = 0; s < 2; ++s)
        for (int l = 0; l <= top; ++l) {
            const size_t px = (size_t)(lk->lcols[l] + 2 * lk->win_w) * (lk->lrows[l] + 2 * lk->win_h);
            SRL_CUDA(ctx, cudaMalloc(&lk->img[s][l], px));
            SRL_CUDA(ctx, cudaMalloc(&lk->der[s][l], px * sizeof(short2)));
        }
    lk->cols = cols;
    lk->rows = rows;
    return SRL_OK;
}

// pyramid and derivatives of one image into set s
int lk_build(srl_lk* lk, int s, const uint8_t* d_img, size_t pitch) {
    srl_ctx* ctx = lk->ctx;
    cudaStream_t st = ctx->stream;
    const int ww = lk->win_w, wh = lk->win_h, T = 256;
    for (int l = 0; l <= lk->max_level; ++l) {
        const int pw = lk->lcols[l] + 2 * ww, ph = lk->lrows[l] + 2 * wh;
        const dim3 grid((pw + T - 1) / T, ph);
        if (l == 0) k_lk_level0<<<grid, T, 0, st>>>(d_img, pitch, lk->cols, lk->rows, ww, wh, lk->img[s][0]);
        else k_lk_pyrdown<<<grid, T, 0, st>>>(lk->img[s][l - 1], lk->lcols[l - 1], lk->lcols[l], lk->lrows[l], ww, wh, lk->img[s][l]);
        SRL_CUDA(ctx, cudaGetLastError());
    }
    LkScharrArgs a = {};
    for (int l = 0; l <= lk->max_level; ++l) {
        a.img[l] = lk->img[s][l];
        a.der[l] = lk->der[s][l];
        a.cols[l] = lk->lcols[l];
        a.rows[l] = lk->lrows[l];
    }
    a.ww = ww;
    a.wh = wh;
    const int pw = lk->cols + 2 * ww, ph = lk->rows + 2 * wh;
    k_lk_scharr<<<dim3((pw + T - 1) / T, ph, lk->max_level + 1), T, 0, st>>>(a);
    SRL_CUDA(ctx, cudaGetLastError());
    ctx->launches += lk->max_level + 2;
    return SRL_OK;
}

}  // namespace

extern "C" {

int srl_lk_create(srl_ctx* ctx, const srl_lk_params* p, srl_lk** out) {
    if (!ctx || !p || !out) return SRL_BAD_ARG;
    *out = nullptr;
    if (p->win_w < 3 || p->win_w > 31 || p->win_h < 3 || p->win_h > 31)
        return set_err(ctx, SRL_BAD_ARG, "srl_lk_create: the window must be 3..31 pixels in each dimension");
    if (p->max_level < 0 || p->max_level > kLkMaxLevels - 1) return set_err(ctx, SRL_BAD_ARG, "srl_lk_create: max_level must be 0..8");
    auto* lk = new srl_lk;
    lk->ctx = ctx;
    lk->device = ctx->device;
    lk->win_w = p->win_w;
    lk->win_h = p->win_h;
    lk->max_level = p->max_level;
    // setTerminationCriteria (:670-682)
    lk->max_count = (p->criteria_type & SRL_LK_COUNT) == 0 ? 30 : std::min(std::max(p->max_count, 0), 100);
    lk->epsilon = (p->criteria_type & SRL_LK_EPS) == 0 ? 0.01 : std::min(std::max(p->epsilon, 0.), 10.);
    lk->flags = p->flags;
    lk->min_eig = (float)p->min_eig_threshold;
    cudaError_t e = cudaSetDevice(ctx->device);
    if (e == cudaSuccess) e = cudaMalloc(&lk->d_count, sizeof(unsigned long long));
    for (int i = 0; i < 3 && e == cudaSuccess; ++i) e = cudaEventCreate(&lk->ev[i]);
    if (e != cudaSuccess) {
        srl_lk_destroy(lk);
        return cuda_fail(ctx, e, "srl_lk_create");
    }
    *out = lk;
    return SRL_OK;
}

void srl_lk_destroy(srl_lk* lk) {
    if (!lk) return;
    cudaSetDevice(lk->device);   // not through lk->ctx: a handle may outlive its ctx (cudaFree waits for the device itself)
    lk_free(lk);
    if (lk->d_count) cudaFree(lk->d_count);
    for (auto& e : lk->ev)
        if (e) cudaEventDestroy(e);
    delete lk;
}

int srl_lk_track_image(srl_lk* lk, const uint8_t* gray, int cols, int rows, size_t pitch, const float* last_pts, size_t n, float* curr_pts,
                       uint8_t* status, int64_t* n_tracked) {
    if (!lk || !n_tracked) return SRL_BAD_ARG;
    *n_tracked = 0;
    srl_ctx* ctx = lk->ctx;
    if (!gray || cols <= 0 || rows <= 0 || pitch < (size_t)cols) return set_err(ctx, SRL_BAD_ARG, "srl_lk_track_image: an image with pitch >= cols is required");
    if (n && (!last_pts || !curr_pts || !status)) return set_err(ctx, SRL_BAD_ARG, "srl_lk_track_image: last_pts, curr_pts and status are required");
    if (n > 0x7fffffff) return set_err(ctx, SRL_BAD_ARG, "srl_lk_track_image: at most 2^31 - 1 points");
    if (cols < lk->win_w + 1 || rows < lk->win_h + 1) return set_err(ctx, SRL_BAD_ARG, "srl_lk_track_image: the image must be larger than the window");
    if (lk->cols && (cols != lk->cols || rows != lk->rows))
        return set_err(ctx, SRL_BAD_ARG, "srl_lk_track_image: every image must have the size of the first one");
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    if (!lk->cols) {
        int rc = lk_allocate(lk, cols, rows);
        if (rc != SRL_OK) { lk_free(lk); lk->cols = lk->rows = 0; return rc; }
    }
    const bool img_dev = mem_kind(gray) == MemKind::Device;
    Staged<const float> in_pts(last_pts);
    Staged<float> out_pts(curr_pts);
    Staged<uint8_t> out_st(status);
    uint8_t* d_img = nullptr;
    int rc = carve_scratch(ctx, [&](Carve& c) {
        d_img = img_dev ? nullptr : c.take<uint8_t>((size_t)cols * rows);
        in_pts.place(c, n * 2);
        out_pts.place(c, n * 2);
        out_st.place(c, n);
    });
    if (rc != SRL_OK || (rc = in_pts.upload(ctx, n * 2)) != SRL_OK) return rc;
    SRL_CUDA(ctx, cudaEventRecord(lk->ev[0], st));
    const uint8_t* src = gray;
    size_t src_pitch = pitch;
    if (!img_dev) {
        SRL_CUDA(ctx, cudaMemcpy2DAsync(d_img, cols, gray, pitch, cols, rows, cudaMemcpyHostToDevice, st));
        src = d_img;
        src_pitch = cols;
    }
    const int cur = lk->have_prev ? 1 - lk->prev : lk->prev;
    if ((rc = lk_build(lk, cur, src, src_pitch)) != SRL_OK) return rc;
    SRL_CUDA(ctx, cudaEventRecord(lk->ev[1], st));
    if (!lk->have_prev) {   // the first image (:762-773): curr_tracked_pts = last_tracked_pts, status untouched, 0 returned
        if (n) {
            k_lk_copy_pts<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(reinterpret_cast<const float2*>(in_pts.d), reinterpret_cast<float2*>(out_pts.d), (int)n);
            SRL_CUDA(ctx, cudaGetLastError());
            ctx->launches += 1;
        }
        SRL_CUDA(ctx, cudaEventRecord(lk->ev[2], st));
        lk->have_prev = true;
        lk->prev = cur;
        lk->timed = true;
        if ((rc = out_pts.hand_back(ctx, n * 2)) != SRL_OK) return rc;
        SRL_CUDA(ctx, cudaStreamSynchronize(st));
        return SRL_OK;
    }
    SRL_CUDA(ctx, cudaMemsetAsync(lk->d_count, 0, sizeof(unsigned long long), st));
    if (n) {
        LkTrackArgs a = {};
        a.prev_pts = reinterpret_cast<const float2*>(in_pts.d);
        a.next_pts = reinterpret_cast<float2*>(out_pts.d);
        a.status = out_st.d;
        a.n = (int)n;
        a.win_w = lk->win_w;
        a.win_h = lk->win_h;
        a.max_level = lk->max_level;
        a.max_count = lk->max_count;
        a.epsilon = lk->epsilon;
        a.min_eig = lk->min_eig;
        for (int l = 0; l <= lk->max_level; ++l) {
            a.I[l] = lk->img[lk->prev][l];
            a.dI[l] = lk->der[lk->prev][l];
            a.J[l] = lk->img[cur][l];
            a.cols[l] = lk->lcols[l];
            a.rows[l] = lk->lrows[l];
        }
        a.n_tracked = lk->d_count;
        const size_t smem = (((size_t)lk->win_w * lk->win_h * 8 + 15) & ~(size_t)15) * kLkWarps;
        k_lk_track<<<(unsigned)((n + kLkWarps - 1) / kLkWarps), kLkBlock, smem, st>>>(a);
        SRL_CUDA(ctx, cudaGetLastError());
        ctx->launches += 1;
    }
    SRL_CUDA(ctx, cudaEventRecord(lk->ev[2], st));
    lk->prev = cur;   // swapImageBuffer (:792)
    lk->timed = true;
    unsigned long long cnt = 0;
    SRL_CUDA(ctx, cudaMemcpyAsync(&cnt, lk->d_count, sizeof(cnt), cudaMemcpyDeviceToHost, st));
    if ((rc = out_pts.hand_back(ctx, n * 2)) != SRL_OK || (rc = out_st.hand_back(ctx, n)) != SRL_OK) return rc;
    SRL_CUDA(ctx, cudaStreamSynchronize(st));
    *n_tracked = (int64_t)cnt;
    return SRL_OK;
}

int srl_lk_info(srl_lk* lk, int32_t* max_level, int32_t* cols, int32_t* rows) {
    if (!lk) return SRL_BAD_ARG;
    if (max_level) *max_level = lk->max_level;
    if (cols) *cols = lk->cols;
    if (rows) *rows = lk->rows;
    return SRL_OK;
}

int srl_lk_download_level(srl_lk* lk, int which, int level, uint8_t* img, int16_t* deriv) {
    if (!lk) return SRL_BAD_ARG;
    srl_ctx* ctx = lk->ctx;
    if (!lk->have_prev || level < 0 || level > lk->max_level || (which != 0 && which != 1))
        return set_err(ctx, SRL_BAD_ARG, "srl_lk_download_level: no such level (which is 0 or 1, level <= max_level, after the first image)");
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    const int s = which == 0 ? lk->prev : 1 - lk->prev;
    const size_t px = (size_t)(lk->lcols[level] + 2 * lk->win_w) * (lk->lrows[level] + 2 * lk->win_h);
    SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (img) SRL_CUDA(ctx, cudaMemcpy(img, lk->img[s][level], px, cudaMemcpyDefault));
    if (deriv) SRL_CUDA(ctx, cudaMemcpy(deriv, lk->der[s][level], px * sizeof(short2), cudaMemcpyDefault));
    return SRL_OK;
}

int srl_lk_last_times(srl_lk* lk, double* pyramid_ms, double* track_ms) {
    if (!lk) return SRL_BAD_ARG;
    srl_ctx* ctx = lk->ctx;
    if (!lk->timed) return set_err(ctx, SRL_BAD_ARG, "srl_lk_last_times: no image has been tracked yet");
    float a = 0.f, b = 0.f;
    SRL_CUDA(ctx, cudaEventSynchronize(lk->ev[2]));
    SRL_CUDA(ctx, cudaEventElapsedTime(&a, lk->ev[0], lk->ev[1]));
    SRL_CUDA(ctx, cudaEventElapsedTime(&b, lk->ev[1], lk->ev[2]));
    if (pyramid_ms) *pyramid_ms = a;
    if (track_ms) *track_ms = b;
    return SRL_OK;
}

}  // extern "C"
