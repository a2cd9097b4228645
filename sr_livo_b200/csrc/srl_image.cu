// srl_image.cu — the camera image preparation of imageProcessing::process (src/imageProcessing.cpp:91-125,166-200) on the device,
// bit for bit OpenCV's:
//   once per object (the first-image step, :93-104): the undistortion map of initUndistortRectifyMap(K, dist, I, K, size,
//     CV_16SC2), kept in that format: map1 = (iu >> 5, iv >> 5) saturated to int16 pairs, map2 = (iv & 31) * 32 + (iu & 31),
//     iu = cvRound(32 u)
//   per image (:120-125), three kernels after the upload:
//     k_img_remap        remap INTER_LINEAR (BORDER_CONSTANT 0, per tap) of the BGR8 image, then from each undistorted pixel the
//                        COLOR_RGB2GRAY grey (channel 0, B, weighted as R) and the COLOR_BGR2YCrCb planes; the undistorted image
//                        itself is never stored
//     k_img_clahe_lut    CLAHE's per-tile LUTs of both planes: grey at clip 3, Y at clip 1, one (t, t) grid from the output's cols
//     k_img_clahe_apply  the LUT blend of both planes: the equalised grey (gray_image), and YCrCb2BGR of (Y', Cr, Cb) (rgb_image)
// The map is FP64 in OpenCV's scalar order (per row, _x/_y/_w stepped by += ir[0], ...), the blend float32 in
// CLAHE_Interpolation_Body's expression: the file is built with --fmad=false so that every product is rounded on its own.
// Everything else is integer arithmetic.
#include <cmath>
#include <climits>

#include "srl_internal.h"

using namespace srl;

namespace {

constexpr int kImgPlanes = 4;          // grey, Y, Cr, Cb of the undistorted image
constexpr int kMinOut = 16;            // the smallest output accepted: CLAHE's 4 x 4 grid of tiles of at least 4 x 4
constexpr int kMaxSide = 32767;        // map1 holds int16 source coordinates

// cv::borderInterpolate for BORDER_REFLECT_101 (len >= 2)
__device__ __forceinline__ int reflect101(int p, int len) {
    while ((unsigned)p >= (unsigned)len) p = p < 0 ? -p : 2 * len - p - 2;
    return p;
}

// saturate_cast<int>(double) as x86-64 cvRound has it (cvtsd2si): nearest even, INT_MIN outside the int range and for NaN
__device__ __forceinline__ int cv_round(double v) {
    const double r = rint(v);
    return (r >= -2147483648.0 && r <= 2147483647.0) ? (int)r : INT_MIN;
}

// saturate_cast<short>(int)
__device__ __forceinline__ short sat_short(int v) { return (short)min(max(v, -32768), 32767); }

struct MapArgs {
    double ir[9];                      // inv(K), row-major
    double fx, fy, u0, v0, k1, k2, p1, p2, k3;
    int cols, rows;
    short2* map1;
    uint16_t* map2;
};

// initUndistortRectifyMap: one thread per output row, the row's columns in order (the accumulation along the row is sequential)
__global__ void k_img_map(const __grid_constant__ MapArgs a) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.rows) return;
    const double* ir = a.ir;
    double _x = i * ir[1] + ir[2], _y = i * ir[4] + ir[5], _w = i * ir[7] + ir[8];
    short2* m1 = a.map1 + (size_t)i * a.cols;
    uint16_t* m2 = a.map2 + (size_t)i * a.cols;
    for (int j = 0; j < a.cols; ++j, _x += ir[0], _y += ir[3], _w += ir[6]) {
        const double w = 1. / _w, x = _x * w, y = _y * w;
        const double x2 = x * x, y2 = y * y;
        const double r2 = x2 + y2, _2xy = 2 * x * y;
        // k4..k6 and s1..s4 are zero and there is no tilt: the denominator is 1 and the thin-prism terms add +0
        const double kr = 1 + ((a.k3 * r2 + a.k2) * r2 + a.k1) * r2;
        const double xd = x * kr + a.p1 * _2xy + a.p2 * (r2 + 2 * x2);
        const double yd = y * kr + a.p1 * (r2 + 2 * y2) + a.p2 * _2xy;
        const int iu = cv_round((a.fx * xd + a.u0) * 32), iv = cv_round((a.fy * yd + a.v0) * 32);
        // saturate_cast<short> as OpenCV's vectorised pack: INT_MIN gives -32768, not the wrapped 0 that would sample a real
        // pixel, and a coordinate past +-32767 px stays outside the image
        m1[j] = make_short2(sat_short(iu >> 5), sat_short(iv >> 5));
        m2[j] = (uint16_t)((iv & 31) * 32 + (iu & 31));
    }
}

struct RemapArgs {
    const uint8_t* src;                // BGR8, in_cols x in_rows, rows src_pitch bytes apart
    size_t src_pitch;
    int in_cols, in_rows, cols, rows;
    const short2* map1;
    const uint16_t* map2;
    uint8_t* planes;                   // kImgPlanes planes of cols * rows: grey, Y, Cr, Cb
};

__global__ void k_img_remap(const __grid_constant__ RemapArgs a) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= a.cols) return;
    const size_t p = (size_t)y * a.cols + x;
    const short2 s = a.map1[p];
    const int f = a.map2[p], fx = f & 31, fy = f >> 5;
    // the 15-bit bilinear weights of remap's fixed-point table, in tap order (0, 0), (1, 0), (0, 1), (1, 1)
    const int w[4] = {(32 - fx) * (32 - fy) * 32, fx * (32 - fy) * 32, (32 - fx) * fy * 32, fx * fy * 32};
    int acc[3] = {0, 0, 0};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int X = s.x + (k & 1), Y = s.y + (k >> 1);
        if (X >= 0 && X < a.in_cols && Y >= 0 && Y < a.in_rows) {   // a tap outside reads the border value 0
            const uint8_t* q = a.src + (size_t)Y * a.src_pitch + (size_t)X * 3;
#pragma unroll
            for (int c = 0; c < 3; ++c) acc[c] += q[c] * w[k];
        }
    }
    const int b = (acc[0] + (1 << 14)) >> 15, g = (acc[1] + (1 << 14)) >> 15, r = (acc[2] + (1 << 14)) >> 15;
    const size_t n = (size_t)a.cols * a.rows;
    // COLOR_RGB2GRAY: 15-bit weights, channel 0 as R
    a.planes[p] = (uint8_t)((b * 9798 + g * 19235 + r * 3735 + (1 << 14)) >> 15);
    // COLOR_BGR2YCrCb: 14-bit weights; Y <= 255 and Cr, Cb are clamped as saturate_cast<uchar> does
    const int Y = (b * 1868 + g * 9617 + r * 4899 + (1 << 13)) >> 14;
    const int cr = ((r - Y) * 11682 + (128 << 14) + (1 << 13)) >> 14;
    const int cb = ((b - Y) * 9241 + (128 << 14) + (1 << 13)) >> 14;
    a.planes[n + p] = (uint8_t)Y;
    a.planes[2 * n + p] = (uint8_t)min(max(cr, 0), 255);
    a.planes[3 * n + p] = (uint8_t)min(max(cb, 0), 255);
}

struct ClaheArgs {
    const uint8_t* planes;
    uint8_t* lut;                      // [plane 0..1][ty][tx][256]
    int cols, rows, tiles, tw, th;     // tw x th: the tile of the (possibly padded) grid
    int clip_limit[2];                 // grey, Y
    float lut_scale;                   // 255.f / (tw * th)
    float inv_tw, inv_th;              // 1.f / tw, 1.f / th
    uint8_t* gray_out;
    uint8_t* bgr_out;
};

// one block of 256 threads per (tile, plane): the tile's histogram read through REFLECT_101 where the grid pads the plane, then
// clipping, redistribution and the integer prefix sum of CLAHE_CalcLut_Body; thread i owns bin i
__global__ void __launch_bounds__(256) k_img_clahe_lut(const __grid_constant__ ClaheArgs a) {
    __shared__ int hist[256];
    __shared__ int warp_sum[8];
    const int bin = threadIdx.x, lane = bin & 31, wid = bin >> 5;
    const int tile = blockIdx.x, plane = blockIdx.y;
    const int ty = tile / a.tiles, tx = tile - ty * a.tiles;
    const uint8_t* src = a.planes + (size_t)plane * a.cols * a.rows;   // plane 0 grey, plane 1 Y
    hist[bin] = 0;
    __syncthreads();
    const int area = a.tw * a.th;
    for (int k = bin; k < area; k += 256) {
        const int r = k / a.tw, c = k - r * a.tw;
        const int y = reflect101(ty * a.th + r, a.rows), x = reflect101(tx * a.tw + c, a.cols);
        atomicAdd(&hist[src[(size_t)y * a.cols + x]], 1);
    }
    __syncthreads();
    const int limit = a.clip_limit[plane];
    int h = hist[bin];
    int excess = max(h - limit, 0);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) excess += __shfl_xor_sync(0xffffffffu, excess, o);
    if (lane == 0) warp_sum[wid] = excess;
    __syncthreads();
    int clipped = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) clipped += warp_sum[k];
    __syncthreads();   // warp_sum is reused by the scan
    // the residual loop gives one more to bins 0, step, 2 step, ... while residual lasts: bin i gets it iff i % step == 0 and
    // i / step < residual (step * residual <= 256 leaves enough such bins)
    const int residual = clipped & 255, step = residual ? max(256 / residual, 1) : 1;
    h = min(h, limit) + (clipped >> 8) + ((residual && bin % step == 0 && bin / step < residual) ? 1 : 0);
    int sum = h;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, sum, o);
        if (lane >= o) sum += v;
    }
    if (lane == 31) warp_sum[wid] = sum;
    __syncthreads();
    for (int k = 0; k < wid; ++k) sum += warp_sum[k];
    // saturate_cast<uchar>((float)sum * lutScale): cvRound of a float rounds half to even
    const int v = __float2int_rn(__fmul_rn(__int2float_rn(sum), a.lut_scale));
    a.lut[((size_t)plane * a.tiles * a.tiles + tile) * 256 + bin] = (uint8_t)min(max(v, 0), 255);
}

// CLAHE_Interpolation_Body's tile coordinate along one axis: (first tile, second tile, weight of the second, of the first)
__device__ __forceinline__ void clahe_axis(int v, float inv, int tiles, int& t1, int& t2, float& a, float& a1) {
    const float tf = __fsub_rn(__fmul_rn(__int2float_rn(v), inv), 0.5f);
    const int f = __float2int_rd(tf);
    a = __fsub_rn(tf, __int2float_rn(f));
    a1 = __fsub_rn(1.f, a);
    t1 = max(f, 0);
    t2 = min(f + 1, tiles - 1);
}

__device__ __forceinline__ int clahe_blend(const uint8_t* lut, int tiles, int ty1, int ty2, int tx1, int tx2, int v, float xa, float xa1,
                                           float ya, float ya1) {
    const float l1a = lut[(ty1 * tiles + tx1) * 256 + v], l1b = lut[(ty1 * tiles + tx2) * 256 + v];
    const float l2a = lut[(ty2 * tiles + tx1) * 256 + v], l2b = lut[(ty2 * tiles + tx2) * 256 + v];
    const float res = __fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(l1a, xa1), __fmul_rn(l1b, xa)), ya1),
                                __fmul_rn(__fadd_rn(__fmul_rn(l2a, xa1), __fmul_rn(l2b, xa)), ya));
    return min(max(__float2int_rn(res), 0), 255);
}

// one thread per pixel: the equalised grey, and the equalised Y with the pixel's Cr, Cb back to BGR8 (COLOR_YCrCb2BGR, 14 bits)
__global__ void k_img_clahe_apply(const __grid_constant__ ClaheArgs a) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= a.cols) return;
    int tx1, tx2, ty1, ty2;
    float xa, xa1, ya, ya1;
    clahe_axis(x, a.inv_tw, a.tiles, tx1, tx2, xa, xa1);
    clahe_axis(y, a.inv_th, a.tiles, ty1, ty2, ya, ya1);
    const size_t n = (size_t)a.cols * a.rows, p = (size_t)y * a.cols + x;
    const size_t lut_plane = (size_t)a.tiles * a.tiles * 256;
    a.gray_out[p] = (uint8_t)clahe_blend(a.lut, a.tiles, ty1, ty2, tx1, tx2, a.planes[p], xa, xa1, ya, ya1);
    const int Y = clahe_blend(a.lut + lut_plane, a.tiles, ty1, ty2, tx1, tx2, a.planes[n + p], xa, xa1, ya, ya1);
    const int cr = a.planes[2 * n + p] - 128, cb = a.planes[3 * n + p] - 128;
    const int b = Y + ((cb * 29049 + (1 << 13)) >> 14);
    const int g = Y + ((cb * -5636 + cr * -11698 + (1 << 13)) >> 14);
    const int r = Y + ((cr * 22987 + (1 << 13)) >> 14);
    uint8_t* o = a.bgr_out + p * 3;
    o[0] = (uint8_t)min(max(b, 0), 255);
    o[1] = (uint8_t)min(max(g, 0), 255);
    o[2] = (uint8_t)min(max(r, 0), 255);
}

// Mat::inv(DECOMP_LU) of a 3x3 double matrix: the cofactors times 1 / det3, each product rounded (the host code is built with
// -ffp-contract=off).  false for a zero or non-finite determinant.
bool inv3(const double* m, double* o) {
    auto a = [m](int r, int c) { return m[r * 3 + c]; };
    double d = a(0, 0) * (a(1, 1) * a(2, 2) - a(1, 2) * a(2, 1)) - a(0, 1) * (a(1, 0) * a(2, 2) - a(1, 2) * a(2, 0)) +
               a(0, 2) * (a(1, 0) * a(2, 1) - a(1, 1) * a(2, 0));
    if (d == 0. || !std::isfinite(d)) return false;
    d = 1. / d;
    o[0] = (a(1, 1) * a(2, 2) - a(1, 2) * a(2, 1)) * d;
    o[1] = (a(0, 2) * a(2, 1) - a(0, 1) * a(2, 2)) * d;
    o[2] = (a(0, 1) * a(1, 2) - a(0, 2) * a(1, 1)) * d;
    o[3] = (a(1, 2) * a(2, 0) - a(1, 0) * a(2, 2)) * d;
    o[4] = (a(0, 0) * a(2, 2) - a(0, 2) * a(2, 0)) * d;
    o[5] = (a(0, 2) * a(1, 0) - a(0, 0) * a(1, 2)) * d;
    o[6] = (a(1, 0) * a(2, 1) - a(1, 1) * a(2, 0)) * d;
    o[7] = (a(0, 1) * a(2, 0) - a(0, 0) * a(2, 1)) * d;
    o[8] = (a(0, 0) * a(1, 1) - a(0, 1) * a(1, 0)) * d;
    for (int k = 0; k < 9; ++k)
        if (!std::isfinite(o[k])) return false;
    return true;
}

}  // namespace

extern "C" {

int srl_image_create(srl_ctx* ctx, const srl_image_params* p, int cols, int rows, srl_image** out) {
    if (!ctx || !p || !out) return SRL_BAD_ARG;
    *out = nullptr;
    if (cols <= 0 || rows <= 0 || cols > kMaxSide || rows > kMaxSide || p->image_width <= 0 || p->image_height <= 0)
        return set_err(ctx, SRL_BAD_ARG, "srl_image_create: the input size and image_width / image_height must be positive (at most 32767)");
    for (double v : p->camera_intrinsic)
        if (!std::isfinite(v)) return set_err(ctx, SRL_BAD_ARG, "srl_image_create: camera_intrinsic must be finite");
    for (double v : p->camera_dist_coeffs)
        if (!std::isfinite(v)) return set_err(ctx, SRL_BAD_ARG, "srl_image_create: camera_dist_coeffs must be finite");
    // the first-image step (:93-104): the scale factor, the scaled intrinsics and the truncated cv::Size of the output
    const double s = p->image_width * 1.0 / cols;
    double K[9];
    for (int k = 0; k < 9; ++k) K[k] = p->camera_intrinsic[k];
    K[0] = K[0] / s;
    K[2] = K[2] / s;
    K[4] = K[4] / s;
    K[5] = K[5] / s;
    const double oc = p->image_width / s, orow = p->image_height / s;
    if (!(oc >= kMinOut && orow >= kMinOut && oc <= kMaxSide && orow <= kMaxSide))
        return set_err(ctx, SRL_BAD_ARG, "srl_image_create: the output (image_width, image_height) / scale factor must be 16..32767 pixels each way");
    double ir[9];
    if (!inv3(K, ir)) return set_err(ctx, SRL_BAD_ARG, "srl_image_create: the scaled camera_intrinsic has no finite inverse");
    std::unique_ptr<srl_image> im(new srl_image);
    im->ctx = ctx;
    im->device = ctx->device;
    vio_initial_covariance(im->cov);
    im->in_cols = cols;
    im->in_rows = rows;
    im->cols = (int)oc;
    im->rows = (int)orow;
    im->scale = s;
    for (int k = 0; k < 9; ++k) im->K[k] = K[k];
    // imageEqualize's grid (:169): both dimensions from cols.  CLAHE pads a plane that the grid does not divide in either
    // dimension by tiles - size % tiles in both (a full tile where it divides).
    const int t = (int)std::max(im->cols * 32.0 / 640, 4.0);
    im->tiles = t;
    const bool pad = im->cols % t != 0 || im->rows % t != 0;
    im->tw = (im->cols + (pad ? t - im->cols % t : 0)) / t;
    im->th = (im->rows + (pad ? t - im->rows % t : 0)) / t;
    const size_t n = (size_t)im->cols * im->rows;
    cudaError_t e = cudaSetDevice(ctx->device);
    if (e == cudaSuccess) e = im->map1.alloc(n);
    if (e == cudaSuccess) e = im->map2.alloc(n);
    if (e == cudaSuccess) e = im->planes.alloc(n * kImgPlanes);
    if (e == cudaSuccess) e = im->lut.alloc((size_t)2 * t * t * 256);
    for (int i = 0; i < 4 && e == cudaSuccess; ++i) e = im->ev[i].create();
    for (int i = 0; i < 4 && e == cudaSuccess; ++i) e = im->vio_ev[i].create();
    if (e == cudaSuccess) e = im->d_vio_out.alloc(1);
    if (e == cudaSuccess) {
        MapArgs a = {};
        for (int k = 0; k < 9; ++k) a.ir[k] = ir[k];
        a.fx = K[0];
        a.fy = K[4];
        a.u0 = K[2];
        a.v0 = K[5];
        a.k1 = p->camera_dist_coeffs[0];
        a.k2 = p->camera_dist_coeffs[1];
        a.p1 = p->camera_dist_coeffs[2];
        a.p2 = p->camera_dist_coeffs[3];
        a.k3 = p->camera_dist_coeffs[4];
        a.cols = im->cols;
        a.rows = im->rows;
        a.map1 = im->map1;
        a.map2 = im->map2;
        k_img_map<<<(im->rows + 63) / 64, 64, 0, ctx->stream>>>(a);
        e = cudaGetLastError();
        ctx->launches += 1;
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) return cuda_fail(ctx, e, "srl_image_create");
    *out = im.release();
    return SRL_OK;
}

void srl_image_destroy(srl_image* im) {
    if (!im) return;
    cudaSetDevice(im->device);
    delete im;
}

int srl_image_process(srl_image* im, const uint8_t* bgr, int cols, int rows, size_t pitch, uint8_t* rgb_out, uint8_t* gray_out) {
    if (!im) return SRL_BAD_ARG;
    srl_ctx* ctx = im->ctx;
    if (!bgr || !rgb_out || !gray_out) return set_err(ctx, SRL_BAD_ARG, "srl_image_process: bgr, rgb_out and gray_out are required");
    if (cols != im->in_cols || rows != im->in_rows)
        return set_err(ctx, SRL_BAD_ARG, "srl_image_process: the image must have the size given at creation");
    if (pitch < (size_t)cols * 3) return set_err(ctx, SRL_BAD_ARG, "srl_image_process: pitch must be at least cols * 3 bytes");
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    const size_t n = (size_t)im->cols * im->rows;
    const bool in_dev = mem_kind(bgr) == MemKind::Device;
    Staged<uint8_t> rgb(rgb_out), gray(gray_out);
    uint8_t* d_in = nullptr;
    int rc = carve_scratch(ctx, [&](Carve& c) {
        d_in = in_dev ? nullptr : c.take<uint8_t>((size_t)cols * rows * 3);
        rgb.place(c, n * 3);
        gray.place(c, n);
    });
    if (rc != SRL_OK) return rc;
    SRL_CUDA(ctx, cudaEventRecord(im->ev[0], st));
    const uint8_t* src = bgr;
    size_t src_pitch = pitch;
    if (!in_dev) {
        SRL_CUDA(ctx, cudaMemcpy2DAsync(d_in, (size_t)cols * 3, bgr, pitch, (size_t)cols * 3, rows, cudaMemcpyHostToDevice, st));
        src = d_in;
        src_pitch = (size_t)cols * 3;
    }
    SRL_CUDA(ctx, cudaEventRecord(im->ev[1], st));
    const int T = 128;
    const dim3 grid((im->cols + T - 1) / T, im->rows);
    RemapArgs ra = {src, src_pitch, cols, rows, im->cols, im->rows, im->map1, im->map2, im->planes};
    k_img_remap<<<grid, T, 0, st>>>(ra);
    SRL_CUDA(ctx, cudaGetLastError());
    SRL_CUDA(ctx, cudaEventRecord(im->ev[2], st));
    ClaheArgs ca = {};
    ca.planes = im->planes;
    ca.lut = im->lut;
    ca.cols = im->cols;
    ca.rows = im->rows;
    ca.tiles = im->tiles;
    ca.tw = im->tw;
    ca.th = im->th;
    const int area = im->tw * im->th;
    // createCLAHE(3) on the grey plane (:124, imageEqualize amp 3) and createCLAHE(1) on Y (:195): max((int)(clip * area / 256), 1)
    ca.clip_limit[0] = std::max((int)(3.0 * area / 256), 1);
    ca.clip_limit[1] = std::max((int)(1.0 * area / 256), 1);
    ca.lut_scale = 255.f / (float)area;
    ca.inv_tw = 1.f / (float)im->tw;
    ca.inv_th = 1.f / (float)im->th;
    ca.gray_out = gray.d;
    ca.bgr_out = rgb.d;
    k_img_clahe_lut<<<dim3(im->tiles * im->tiles, 2), 256, 0, st>>>(ca);
    SRL_CUDA(ctx, cudaGetLastError());
    k_img_clahe_apply<<<grid, T, 0, st>>>(ca);
    SRL_CUDA(ctx, cudaGetLastError());
    SRL_CUDA(ctx, cudaEventRecord(im->ev[3], st));
    ctx->launches += 3;
    im->timed = true;
    if ((rc = rgb.hand_back(ctx, n * 3)) != SRL_OK || (rc = gray.hand_back(ctx, n)) != SRL_OK) return rc;
    SRL_CUDA(ctx, cudaStreamSynchronize(st));
    return SRL_OK;
}

int srl_image_info(srl_image* im, int32_t* out_cols, int32_t* out_rows, int32_t* tiles, double* scale_factor, double intrinsic[9]) {
    if (!im) return SRL_BAD_ARG;
    if (out_cols) *out_cols = im->cols;
    if (out_rows) *out_rows = im->rows;
    if (tiles) *tiles = im->tiles;
    if (scale_factor) *scale_factor = im->scale;
    if (intrinsic)
        for (int k = 0; k < 9; ++k) intrinsic[k] = im->K[k];
    return SRL_OK;
}

int srl_image_download_maps(srl_image* im, int16_t* map1, uint16_t* map2) {
    if (!im) return SRL_BAD_ARG;
    srl_ctx* ctx = im->ctx;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    const size_t n = (size_t)im->cols * im->rows;
    SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (map1) SRL_CUDA(ctx, cudaMemcpy(map1, im->map1, n * sizeof(short2), cudaMemcpyDefault));
    if (map2) SRL_CUDA(ctx, cudaMemcpy(map2, im->map2, n * sizeof(uint16_t), cudaMemcpyDefault));
    return SRL_OK;
}

int srl_image_last_times(srl_image* im, double* upload_ms, double* remap_ms, double* clahe_ms) {
    if (!im) return SRL_BAD_ARG;
    srl_ctx* ctx = im->ctx;
    if (!im->timed) return set_err(ctx, SRL_BAD_ARG, "srl_image_last_times: no image has been processed yet");
    float t[3] = {0.f, 0.f, 0.f};
    SRL_CUDA(ctx, cudaEventSynchronize(im->ev[3]));
    for (int k = 0; k < 3; ++k) SRL_CUDA(ctx, cudaEventElapsedTime(&t[k], im->ev[k], im->ev[k + 1]));
    if (upload_ms) *upload_ms = t[0];
    if (remap_ms) *remap_ms = t[1];
    if (clahe_ms) *clahe_ms = t[2];
    return SRL_OK;
}

}  // extern "C"
