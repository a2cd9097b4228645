// srl_frame.cu — lioOptimization::buildFrame (src/lioOptimization.cpp:786-893) on the device: makePointTimestamp, the
// undistortion of row N3, the two std::shuffle calls around subSampleFrame, transformAllImuPoint and transformPoint.
//
// The shuffles are the reference's std::shuffle(frame, boost::mt19937_64) with a default-seeded engine shared by both calls.
// libstdc++ (bits/stl_algo.h, shuffle) draws swap targets for two positions at a time: with n even one draw in [0, 2) swaps
// position 1 first, then positions i, i+1 take one draw x in [0, (i+1)(i+2)) and swap with x / (i+2) and x % (i+2).  A draw
// (bits/uniform_int_dist.h) is Lemire's multiply-shift with rejection (rule 0, libstdc++ with __int128) or the division
// downscale (rule 1, libstdc++ without __int128 and libstdc++ <= 10).  The swap targets depend only on n and the engine, so:
//   1. k_mt64 generates the engine's output words (one block, 312-word twists);
//   2. k_draws turns word d into draw d assuming no rejection and flags the first draw whose rejection test fires; the host
//      redoes the draws from there sequentially (probability < 1e-5 per 100k-point shuffle);
//   3. the steps (j_k, k), "swap(a[k], a[j_k])" with j_k <= k, are sorted, and k_resolve gives every final position its
//      source: the largest k > p with j_k = p if there is one (a[k] lands there last), else what position j_p held just
//      before step p, resolved the same way one level down (positions strictly decrease, expected depth ~ ln n).
#include <algorithm>
#include <chrono>
#include <cstring>
#include <random>
#include <vector>

#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include "srl_internal.h"

namespace srl {
namespace {

constexpr int kMtN = 312, kMtM = 156;
constexpr unsigned long long kMtUpper = 0xFFFFFFFF80000000ULL, kMtLower = 0x7FFFFFFFULL, kMtA = 0xB5026F5AA96619E9ULL;

// std::mt19937_64 at its default seed (5489): outputs [0, count)
__global__ void k_mt64(unsigned long long* __restrict__ out, long long count) {
    __shared__ unsigned long long mt[kMtN];
    const int t = threadIdx.x;
    if (t == 0) {
        mt[0] = 5489ULL;
        for (int i = 1; i < kMtN; ++i) mt[i] = 6364136223846793005ULL * (mt[i - 1] ^ (mt[i - 1] >> 62)) + (unsigned long long)i;
    }
    __syncthreads();
    for (long long base = 0; base < count; base += kMtN) {
        unsigned long long v = 0;
        if (t < kMtN - kMtM) {   // mt[i + m] not yet rewritten
            const unsigned long long x = (mt[t] & kMtUpper) | (mt[t + 1] & kMtLower);
            v = mt[t + kMtM] ^ (x >> 1) ^ ((x & 1ULL) ? kMtA : 0ULL);
        }
        __syncthreads();
        if (t < kMtN - kMtM) mt[t] = v;
        __syncthreads();
        if (t >= kMtN - kMtM && t < kMtN) {   // mt[i + m - n] already rewritten; mt[0] too for the last word
            const unsigned long long x = (mt[t] & kMtUpper) | (mt[(t + 1) % kMtN] & kMtLower);
            v = mt[t - (kMtN - kMtM)] ^ (x >> 1) ^ ((x & 1ULL) ? kMtA : 0ULL);
        }
        __syncthreads();
        if (t >= kMtN - kMtM && t < kMtN) mt[t] = v;
        __syncthreads();
        if (t < kMtN && base + t < count) {
            unsigned long long y = mt[t];
            y ^= (y >> 29) & 0x5555555555555555ULL;
            y ^= (y << 17) & 0x71D67FFFEDA60000ULL;
            y ^= (y << 37) & 0xFFF7EEE000000000ULL;
            y ^= y >> 43;
            out[base + t] = y;
        }
    }
}

// draw d of a shuffle over n: the position it serves and the range of its uniform_int_distribution
__host__ __device__ __forceinline__ void draw_step(long long d, long long n, long long& i, unsigned long long& range) {
    if ((n & 1) == 0) {
        if (d == 0) { i = 1; range = 2; return; }
        i = 2 * d;
    } else {
        i = 2 * d + 1;
    }
    range = (unsigned long long)(i + 1) * (unsigned long long)(i + 2);
}
__host__ __device__ __forceinline__ long long num_draws(long long n) { return n <= 1 ? 0 : ((n & 1) == 0 ? 1 : 0) + (n - 1) / 2; }

// one attempt of uniform_int_distribution<uint64>{0, range - 1} on word w; false when the rule rejects w
__host__ __device__ __forceinline__ bool draw_try(unsigned long long w, unsigned long long range, int rule, unsigned long long& x) {
    if (rule == 0) {
#ifdef __CUDA_ARCH__
        const unsigned long long lo = w * range, hi = __umul64hi(w, range);
#else
        const unsigned __int128 p = (unsigned __int128)w * range;
        const unsigned long long lo = (unsigned long long)p, hi = (unsigned long long)(p >> 64);
#endif
        x = hi;
        return !(lo < range && lo < (0ULL - range) % range);
    }
    const unsigned long long scaling = ~0ULL / range, past = range * scaling;
    x = w / scaling;
    return w < past;
}

// the k-th step is "swap(a[k], a[j_k])"; keys (j_k << 32 | k) for the sort, first rejected draw into *first_rej
__global__ void k_draws(const unsigned long long* __restrict__ words, long long n, int rule, unsigned int* __restrict__ j,
                        unsigned long long* __restrict__ keys, unsigned long long* __restrict__ first_rej) {
    const long long d = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= num_draws(n)) return;
    long long i; unsigned long long range, x;
    draw_step(d, n, i, range);
    if (!draw_try(words[d], range, rule, x)) atomicMin(first_rej, (unsigned long long)d);
    if (range == 2) {
        j[1] = (unsigned)x; keys[0] = (x << 32) | 1ULL;
    } else {
        const unsigned long long b1 = (unsigned long long)(i + 2), j0 = x / b1, j1 = x % b1;
        j[i] = (unsigned)j0; keys[i - 1] = (j0 << 32) | (unsigned long long)i;
        j[i + 1] = (unsigned)j1; keys[i] = (j1 << 32) | (unsigned long long)(i + 1);
    }
}

// out[p] = in[source of final position p] (in == nullptr: the identity), keys sorted ascending, n - 1 of them
__global__ void k_resolve(const unsigned long long* __restrict__ keys, const unsigned int* __restrict__ j, long long n,
                          const unsigned int* __restrict__ in, unsigned int* __restrict__ out) {
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const long long nk = n - 1;
    unsigned long long q = (unsigned long long)p, t = (unsigned long long)n;
    unsigned long long src;
    for (;;) {
        // last key below (q, t): the latest step k < t that swapped into position q
        const unsigned long long bound = (q << 32) | t;
        long long lo = 0, hi = nk;
        while (lo < hi) { const long long mid = (lo + hi) >> 1; if (keys[mid] < bound) lo = mid + 1; else hi = mid; }
        if (lo > 0) {
            const unsigned long long kk = keys[lo - 1];
            if ((kk >> 32) == q && (kk & 0xFFFFFFFFULL) > q) { src = kk & 0xFFFFFFFFULL; break; }
        }
        if (q == 0 || j[q] == q) { src = q; break; }
        t = q; q = j[q];
    }
    out[p] = in ? in[src] : (unsigned)src;
}

__global__ void k_gather_u32(const unsigned int* __restrict__ in, const unsigned int* __restrict__ idx, long long n, unsigned int* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = in[idx[i]];
}
__global__ void k_gather_xyz(const double* __restrict__ in, const unsigned int* __restrict__ idx, long long n, double* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned s = idx[i];
    out[3 * i] = in[3 * s]; out[3 * i + 1] = in[3 * s + 1]; out[3 * i + 2] = in[3 * s + 2];
}

// makePointTimestamp's erase (branch without point time): the points that stay, flagged
__global__ void k_ts_keep(const double* __restrict__ ts, long long n, double begin, double end, unsigned char* __restrict__ keep) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) keep[i] = !(ts[i] > end) && !(ts[i] < begin);
}
// makePointTimestamp over the kept points (sel == nullptr: all of them), in their order
__global__ void k_ts_gather(const double* __restrict__ raw, const double* __restrict__ ts, const unsigned int* __restrict__ sel, long long n,
                            double begin, double delta_t, int clamp, double* __restrict__ raw1, double* __restrict__ ts1,
                            double* __restrict__ rel1, double* __restrict__ alpha1, unsigned int* __restrict__ src1) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const unsigned i = sel ? sel[k] : (unsigned)k;
    const double stamp = ts[i];
    double rel = stamp - begin;
    double alpha = rel / delta_t;
    rel = rel * 1000.0;
    if (clamp && alpha > 1.0) alpha = 1.0 - 1e-5;
    raw1[3 * k] = raw[3 * i]; raw1[3 * k + 1] = raw[3 * i + 1]; raw1[3 * k + 2] = raw[3 * i + 2];
    ts1[k] = stamp; rel1[k] = rel; alpha1[k] = alpha; src1[k] = i;
}
// the frame in its final order: per-point fields of the kept point c[p]
__global__ void k_frame_gather(const unsigned int* __restrict__ c, long long m, const double* __restrict__ imu1, const double* __restrict__ ts1,
                               const double* __restrict__ rel1, const double* __restrict__ alpha1, const unsigned int* __restrict__ src1,
                               int alpha_one, double* __restrict__ imu, double* __restrict__ ts, double* __restrict__ rel,
                               double* __restrict__ alpha, int* __restrict__ src) {
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= m) return;
    const unsigned i = c[p];
    imu[3 * p] = imu1[3 * i]; imu[3 * p + 1] = imu1[3 * i + 1]; imu[3 * p + 2] = imu1[3 * i + 2];
    ts[p] = ts1[i]; rel[p] = rel1[i]; alpha[p] = alpha_one ? 1.0 : alpha1[i]; src[p] = (int)src1[i];
}

inline unsigned grid_of(long long n, int T = 256) { return (unsigned)((n + T - 1) / T); }

}  // namespace

// The engine's output words: the device-generated mt19937_64 stream, or a caller's stream (test replay).
struct WordStream {
    srl_ctx* ctx = nullptr;
    const unsigned long long* replay = nullptr;   // host, n_replay words; nullptr: mt19937_64 at its default seed
    size_t n_replay = 0;
    DevArray<unsigned long long> d_words;         // device copy of words [0, n_words)
    size_t n_words = 0;
    size_t pos = 0;                               // next unused word
    bool host = false;                            // option "shuffle_on_host": draw on the host from a host engine
    std::mt19937_64 host_engine;

    // words [0, need) on the device
    int ensure(size_t need) {
        if (need <= n_words) return SRL_OK;
        if (replay && need > n_replay) return set_err(ctx, SRL_BAD_ARG, "replayed engine stream exhausted");
        const size_t count = replay ? n_replay : std::max(need + 4096, 2 * n_words);
        SRL_CUDA(ctx, d_words.alloc(std::max<size_t>(count, 1)));
        if (replay) {
            SRL_CUDA(ctx, cudaMemcpyAsync(d_words, replay, count * sizeof(unsigned long long), cudaMemcpyHostToDevice, ctx->stream));
        } else {
            k_mt64<<<1, kMtN, 0, ctx->stream>>>(d_words, (long long)count);
            SRL_CUDA(ctx, cudaGetLastError());
            ctx->launches += 1;
        }
        n_words = count;
        return SRL_OK;
    }
    // word k on the host (the sequential redo after a rejection)
    int word(size_t k, std::vector<unsigned long long>& cache, size_t& cache_base, unsigned long long& w) {
        if (k < cache_base || k >= cache_base + cache.size()) {
            int rc = ensure(std::max(k + 1, std::min(k + 4096, replay ? n_replay : k + 4096)));
            if (rc != SRL_OK) return rc;
            cache_base = k;
            cache.resize(std::min<size_t>(4096, n_words - k));
            SRL_CUDA(ctx, cudaMemcpyAsync(cache.data(), d_words + k, cache.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
            SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        }
        w = cache[k - cache_base];
        return SRL_OK;
    }
};

// Work buffers of one shuffle over up to `cap` elements
struct ShuffleWork {
    unsigned int* j = nullptr;
    unsigned long long* keys = nullptr;
    unsigned long long* keys_sorted = nullptr;
    unsigned long long* first_rej = nullptr;
    void* cub_tmp = nullptr;
    size_t cub_bytes = 0;
};

// out[p] = in[perm[p]] for std::shuffle's permutation perm of n elements (in == nullptr: out = perm).  Consumes the words.
static int shuffle_indices(srl_ctx* ctx, WordStream& ws, ShuffleWork& w, const unsigned int* in, unsigned int* out, long long n,
                           int rule, int64_t* rejections) {
    cudaStream_t st = ctx->stream;
    const int T = 256;
    if (n == 0) return SRL_OK;
    const long long D = num_draws(n);
    if (ws.host) {   // sequential Fisher-Yates on the host, then one upload
        std::vector<unsigned int> a((size_t)n);
        if (in) { SRL_CUDA(ctx, cudaMemcpyAsync(a.data(), in, (size_t)n * 4, cudaMemcpyDeviceToHost, st)); SRL_CUDA(ctx, cudaStreamSynchronize(st)); }
        else for (long long i = 0; i < n; ++i) a[(size_t)i] = (unsigned)i;
        for (long long d = 0; d < D; ++d) {
            long long i; unsigned long long range, x;
            draw_step(d, n, i, range);
            for (;;) {
                if (ws.replay && ws.pos >= ws.n_replay) return set_err(ctx, SRL_BAD_ARG, "replayed engine stream exhausted");
                const unsigned long long wd = ws.replay ? ws.replay[ws.pos] : ws.host_engine();
                ++ws.pos;
                if (draw_try(wd, range, rule, x)) break;
                ++*rejections;
            }
            if (range == 2) std::swap(a[1], a[(size_t)x]);
            else { std::swap(a[(size_t)i], a[(size_t)(x / (i + 2))]); std::swap(a[(size_t)i + 1], a[(size_t)(x % (i + 2))]); }
        }
        SRL_CUDA(ctx, cudaMemcpyAsync(out, a.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
        SRL_CUDA(ctx, cudaStreamSynchronize(st));
        return SRL_OK;
    }
    if (D == 0) {   // n == 1
        if (in) SRL_CUDA(ctx, cudaMemcpyAsync(out, in, 4, cudaMemcpyDeviceToDevice, st));
        else SRL_CUDA(ctx, cudaMemsetAsync(out, 0, 4, st));
        return SRL_OK;
    }
    int rc = ws.ensure(ws.pos + (size_t)D);
    if (rc != SRL_OK) return rc;
    const unsigned long long none = ~0ULL;
    SRL_CUDA(ctx, cudaMemcpyAsync(w.first_rej, &none, 8, cudaMemcpyHostToDevice, st));
    SRL_CUDA(ctx, cudaMemsetAsync(w.j, 0, 4, st));   // j[0] is never read; keep it defined
    k_draws<<<grid_of(D), T, 0, st>>>(ws.d_words + ws.pos, n, rule, w.j, w.keys, w.first_rej);
    SRL_CUDA(ctx, cudaGetLastError());
    ctx->launches += 1;
    unsigned long long first = none;
    SRL_CUDA(ctx, cudaMemcpyAsync(&first, w.first_rej, 8, cudaMemcpyDeviceToHost, st));
    SRL_CUDA(ctx, cudaStreamSynchronize(st));
    if (first == none) {
        ws.pos += (size_t)D;
    } else {   // a rejection: draws [first, D) again on the host, each consuming words until one is accepted
        std::vector<unsigned long long> cache, keys;
        std::vector<unsigned int> jv;
        size_t cache_base = 0, k = ws.pos + (size_t)first;
        long long i0 = 0; unsigned long long r0;
        draw_step((long long)first, n, i0, r0);
        for (long long d = (long long)first; d < D; ++d) {
            long long i; unsigned long long range, x;
            draw_step(d, n, i, range);
            for (;;) {
                unsigned long long wd;
                if ((rc = ws.word(k++, cache, cache_base, wd)) != SRL_OK) return rc;
                if (draw_try(wd, range, rule, x)) break;
                ++*rejections;
            }
            if (range == 2) { jv.push_back((unsigned)x); keys.push_back((x << 32) | 1ULL); }
            else {
                const unsigned long long b1 = (unsigned long long)(i + 2);
                jv.push_back((unsigned)(x / b1)); keys.push_back(((x / b1) << 32) | (unsigned long long)i);
                jv.push_back((unsigned)(x % b1)); keys.push_back(((x % b1) << 32) | (unsigned long long)(i + 1));
            }
        }
        ws.pos = k;
        // the redone steps are positions i0 .. n-1 (keys i0-1 .. n-2), contiguous
        SRL_CUDA(ctx, cudaMemcpyAsync(w.j + i0, jv.data(), jv.size() * 4, cudaMemcpyHostToDevice, st));
        SRL_CUDA(ctx, cudaMemcpyAsync(w.keys + (i0 - 1), keys.data(), keys.size() * 8, cudaMemcpyHostToDevice, st));
    }
    int end_bit = 32;
    while (end_bit < 64 && ((unsigned long long)n >> (end_bit - 32)) != 0) ++end_bit;
    size_t tb = w.cub_bytes;
    SRL_CUDA(ctx, cub::DeviceRadixSort::SortKeys(w.cub_tmp, tb, w.keys, w.keys_sorted, (int)(n - 1), 0, end_bit, st));
    k_resolve<<<grid_of(n), T, 0, st>>>(w.keys_sorted, w.j, n, in, out);
    SRL_CUDA(ctx, cudaGetLastError());
    SRL_CUDA(ctx, cudaStreamSynchronize(st));
    ctx->launches += 2;
    return SRL_OK;
}

// the work buffers of one shuffle over up to `cap` elements (w.cub_bytes set by the caller)
static void shuffle_work_layout(ShuffleWork& w, Carve& c, size_t cap) {
    w.j = c.take<unsigned int>(cap + 1);
    w.keys = c.take<unsigned long long>(cap + 1);
    w.keys_sorted = c.take<unsigned long long>(cap + 1);
    w.first_rej = c.take<unsigned long long>(1);
    w.cub_tmp = c.take<char>(w.cub_bytes);
}

}  // namespace srl

using namespace srl;

struct srl_cloud_frame {
    srl_ctx* ctx = nullptr;
    int device = 0;
    size_t capacity = 0;
    size_t n = 0;
    DevArray<char> mem;
    // the frame, final order
    double *raw = nullptr, *point = nullptr, *imu = nullptr, *rel = nullptr, *alpha = nullptr, *ts = nullptr;
    int* src = nullptr;
    // after makePointTimestamp, sweep order
    double *raw1 = nullptr, *ts1 = nullptr, *rel1 = nullptr, *alpha1 = nullptr, *imu1 = nullptr;
    unsigned int* src1 = nullptr;
    // staging, selections and index compositions
    double *in_raw = nullptr, *in_ts = nullptr, *pt = nullptr;
    unsigned char* keep = nullptr;
    unsigned int *ca = nullptr, *cb = nullptr, *sel = nullptr;
    int* d_count = nullptr;
    void* sel_tmp = nullptr;
    size_t sel_bytes = 0;
    ShuffleWork sw;
};

// the frame's arrays, its selection's and its shuffles' work buffers for up to `cap` points (sel_bytes and sw.cub_bytes set)
static void frame_layout(srl_cloud_frame& f, Carve& c, size_t cap) {
    f.raw = c.take<double>(cap * 3); f.point = c.take<double>(cap * 3); f.imu = c.take<double>(cap * 3);
    f.rel = c.take<double>(cap); f.alpha = c.take<double>(cap); f.ts = c.take<double>(cap);
    f.src = c.take<int>(cap);
    f.raw1 = c.take<double>(cap * 3); f.imu1 = c.take<double>(cap * 3);
    f.ts1 = c.take<double>(cap); f.rel1 = c.take<double>(cap); f.alpha1 = c.take<double>(cap);
    f.src1 = c.take<unsigned int>(cap);
    f.in_raw = c.take<double>(cap * 3); f.pt = c.take<double>(cap * 3);
    f.in_ts = c.take<double>(cap);
    f.keep = c.take<unsigned char>(cap);
    f.ca = c.take<unsigned int>(cap); f.cb = c.take<unsigned int>(cap); f.sel = c.take<unsigned int>(cap);
    f.d_count = c.take<int>(1);
    f.sel_tmp = c.take<char>(f.sel_bytes);
    shuffle_work_layout(f.sw, c, cap);
}

static int frame_reserve(srl_cloud_frame* f, size_t cap) {
    srl_ctx* ctx = f->ctx;
    if (cap <= f->capacity && f->mem) return SRL_OK;
    cap = std::max(cap, f->capacity * 2);
    cap = std::max<size_t>(cap, 1024);
    srl_cloud_frame g;   // the grown frame, laid out first to measure it
    g.ctx = ctx;
    g.device = f->device;
    g.capacity = cap;
    cub::DeviceSelect::Flagged(nullptr, g.sel_bytes, (unsigned int*)nullptr, (unsigned char*)nullptr, (unsigned int*)nullptr, (int*)nullptr, (int)cap);
    cub::DeviceRadixSort::SortKeys(nullptr, g.sw.cub_bytes, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)cap, 0, 64);
    Carve probe;
    frame_layout(g, probe, cap);
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    SRL_CUDA(ctx, g.mem.alloc(probe.used));
    Carve c{g.mem, 0};
    frame_layout(g, c, cap);
    if (f->mem && f->n) {   // the frame moves with its block: a build refused after growing still leaves it as it was
        const size_t n = f->n;
        const cudaMemcpyKind dd = cudaMemcpyDeviceToDevice;
        cudaStream_t st = ctx->stream;
        SRL_CUDA(ctx, cudaMemcpyAsync(g.raw, f->raw, n * 24, dd, st)); SRL_CUDA(ctx, cudaMemcpyAsync(g.point, f->point, n * 24, dd, st));
        SRL_CUDA(ctx, cudaMemcpyAsync(g.imu, f->imu, n * 24, dd, st)); SRL_CUDA(ctx, cudaMemcpyAsync(g.rel, f->rel, n * 8, dd, st));
        SRL_CUDA(ctx, cudaMemcpyAsync(g.alpha, f->alpha, n * 8, dd, st)); SRL_CUDA(ctx, cudaMemcpyAsync(g.ts, f->ts, n * 8, dd, st));
        SRL_CUDA(ctx, cudaMemcpyAsync(g.src, f->src, n * 4, dd, st));
        SRL_CUDA(ctx, cudaStreamSynchronize(st));
        g.n = n;
    }
    *f = std::move(g);
    return SRL_OK;
}

static double ms_since(std::chrono::steady_clock::time_point& t0) {
    const auto t1 = std::chrono::steady_clock::now();
    const double ms = std::chrono::duration<double, std::milli>(t1 - t0).count();
    t0 = t1;
    return ms;
}

extern "C" {

int srl_cloud_frame_create(srl_ctx* ctx, size_t capacity, srl_cloud_frame** out) {
    if (!ctx || !out) return SRL_BAD_ARG;
    *out = nullptr;
    if (capacity > 0x7fffffffULL) return set_err(ctx, SRL_BAD_ARG, "srl_cloud_frame_create: capacity must fit in int32");
    std::unique_ptr<srl_cloud_frame> f(new srl_cloud_frame());
    f->ctx = ctx;
    f->device = ctx->device;
    const int rc = frame_reserve(f.get(), capacity);
    if (rc != SRL_OK) return rc;
    *out = f.release();
    return SRL_OK;
}
void srl_cloud_frame_destroy(srl_cloud_frame* f) {
    if (!f) return;
    cudaSetDevice(f->device);
    cudaDeviceSynchronize();   // the last build's kernels and copies have finished
    delete f;
}
size_t srl_cloud_frame_size(const srl_cloud_frame* f) { return f ? f->n : 0; }
int srl_cloud_frame_device(srl_cloud_frame* f, srl_cloud_frame_ptrs* p) {
    if (!f || !p) return SRL_BAD_ARG;
    p->raw_point = f->raw; p->point = f->point; p->imu_point = f->imu;
    p->relative_time = f->rel; p->alpha_time = f->alpha; p->timestamp = f->ts; p->source_index = f->src;
    return SRL_OK;
}
int srl_cloud_frame_download(srl_cloud_frame* f, double* raw_point, double* point, double* imu_point, double* relative_time,
                             double* alpha_time, double* timestamp, int32_t* source_index) {
    if (!f) return SRL_BAD_ARG;
    srl_ctx* ctx = f->ctx;
    const size_t n = f->n;
    if (n == 0) return SRL_OK;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    if (raw_point) SRL_CUDA(ctx, cudaMemcpyAsync(raw_point, f->raw, n * 24, cudaMemcpyDeviceToHost, st));
    if (point) SRL_CUDA(ctx, cudaMemcpyAsync(point, f->point, n * 24, cudaMemcpyDeviceToHost, st));
    if (imu_point) SRL_CUDA(ctx, cudaMemcpyAsync(imu_point, f->imu, n * 24, cudaMemcpyDeviceToHost, st));
    if (relative_time) SRL_CUDA(ctx, cudaMemcpyAsync(relative_time, f->rel, n * 8, cudaMemcpyDeviceToHost, st));
    if (alpha_time) SRL_CUDA(ctx, cudaMemcpyAsync(alpha_time, f->alpha, n * 8, cudaMemcpyDeviceToHost, st));
    if (timestamp) SRL_CUDA(ctx, cudaMemcpyAsync(timestamp, f->ts, n * 8, cudaMemcpyDeviceToHost, st));
    if (source_index) SRL_CUDA(ctx, cudaMemcpyAsync(source_index, f->src, n * 4, cudaMemcpyDeviceToHost, st));
    SRL_CUDA(ctx, cudaStreamSynchronize(st));
    return SRL_OK;
}

int srl_build_frame(srl_ctx* ctx, const double* raw_xyz, const double* timestamp, size_t n, const srl_imu_state* states,
                    size_t n_states, const srl_build_frame_params* prm, srl_cloud_frame* f, srl_build_frame_info* info) {
    if (!ctx) return SRL_BAD_ARG;
    if (!prm || !f || f->ctx != ctx || !states || (n && (!raw_xyz || !timestamp))) return set_err(ctx, SRL_BAD_ARG, "srl_build_frame: null argument");
    if (prm->motion_compensation != 0 && prm->motion_compensation != 1)
        return set_err(ctx, SRL_BAD_ARG, "srl_build_frame: motion_compensation must be 0 (IMU) or 1 (CONSTANT_VELOCITY)");
    if (n_states < 1) return set_err(ctx, SRL_BAD_ARG, "srl_build_frame: at least one IMU state is needed");
    if (n > 0x7fffffffULL) return set_err(ctx, SRL_BAD_ARG, "srl_build_frame: n must fit in int32");
    const double sample_size = prm->index_frame < prm->init_num_frames ? prm->init_voxel_size : prm->voxel_size;
    if (prm->voxel_size > 0 && !(sample_size > 0)) return set_err(ctx, SRL_BAD_ARG, "srl_build_frame: the subsample cell size must be > 0");
    int rc = frame_reserve(f, n);
    if (rc != SRL_OK) return rc;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    const int T = 256;
    srl_build_frame_info inf;
    std::memset(&inf, 0, sizeof(inf));
    auto t0 = std::chrono::steady_clock::now();

    // bookkeeping (src/lioOptimization.cpp:823-829,855-858,880-889)
    const double time_frame_begin = prm->timestamp_begin, time_end = prm->timestamp_begin + prm->timestamp_offset;
    inf.time_sweep_begin = prm->timestamp_begin;
    inf.time_sweep_end = time_end;
    inf.time_frame_begin = time_frame_begin;
    inf.time_frame_end = time_end;
    inf.offset_begin = 0;
    inf.offset_end = prm->timestamp_offset;
    double dt_offset = 0;
    if (prm->index_frame > 1) dt_offset -= time_frame_begin - prm->prev_time_sweep_end;
    inf.dt_offset = dt_offset;
    inf.frame_id = prm->index_frame;
    inf.sample_size = sample_size;
    inf.n_input = (int64_t)n;

    // 1. makePointTimestamp (:786-819)
    const double* raw = raw_xyz; const double* ts = timestamp;
    if (n && mem_kind(raw_xyz) != MemKind::Device) { SRL_CUDA(ctx, cudaMemcpyAsync(f->in_raw, raw_xyz, n * 24, cudaMemcpyHostToDevice, st)); raw = f->in_raw; }
    if (n && mem_kind(timestamp) != MemKind::Device) { SRL_CUDA(ctx, cudaMemcpyAsync(f->in_ts, timestamp, n * 8, cudaMemcpyHostToDevice, st)); ts = f->in_ts; }
    const double delta_t = time_end - time_frame_begin;
    long long n1 = (long long)n;
    if (n && prm->point_time_enable) {
        k_ts_gather<<<grid_of(n1), T, 0, st>>>(raw, ts, nullptr, n1, time_frame_begin, delta_t, 1, f->raw1, f->ts1, f->rel1, f->alpha1, f->src1);
        SRL_CUDA(ctx, cudaGetLastError());
        ctx->launches += 1;
    } else if (n) {
        k_ts_keep<<<grid_of(n1), T, 0, st>>>(ts, n1, time_frame_begin, time_end, f->keep);
        size_t tb = f->sel_bytes;
        SRL_CUDA(ctx, cub::DeviceSelect::Flagged(f->sel_tmp, tb, thrust::counting_iterator<unsigned int>(0), f->keep, f->ca, f->d_count, (int)n, st));
        int kept = 0;
        SRL_CUDA(ctx, cudaMemcpyAsync(&kept, f->d_count, 4, cudaMemcpyDeviceToHost, st));
        SRL_CUDA(ctx, cudaStreamSynchronize(st));
        n1 = kept;
        if (n1) k_ts_gather<<<grid_of(n1), T, 0, st>>>(raw, ts, f->ca, n1, time_frame_begin, delta_t, 0, f->raw1, f->ts1, f->rel1, f->alpha1, f->src1);
        SRL_CUDA(ctx, cudaGetLastError());
        ctx->launches += 3;
    }
    inf.n_timestamped = n1;
    SRL_CUDA(ctx, cudaStreamSynchronize(st));
    inf.stage_ms[0] = ms_since(t0);

    // 2. undistortion (:831-834).  imu_point starts at 0: points the IMU walk never reaches keep it (the reference leaves
    //    them whatever the cut sweep held)
    if (n1) SRL_CUDA(ctx, cudaMemsetAsync(f->imu1, 0, (size_t)n1 * 24, st));
    inf.n_imu_written = n1;
    if (prm->motion_compensation == 1) {
        rc = srl_distort_frame_by_constant(ctx, f->raw1, f->rel1, (size_t)n1, states, n_states, time_frame_begin, prm->R_il, prm->t_il, f->imu1);
    } else {
        int64_t written = 0;
        rc = srl_distort_frame_by_imu(ctx, f->raw1, f->rel1, (size_t)n1, states, n_states, time_frame_begin, prm->R_il, prm->t_il, f->imu1, &written);
        inf.n_imu_written = written;
    }
    if (rc != SRL_OK) return rc;
    inf.stage_ms[1] = ms_since(t0);

    // 3. shuffle 1 (:838-841); the engine is default-seeded per call and shared with shuffle 2
    WordStream ws;
    ws.ctx = ctx;
    ws.host = ctx->shuffle_on_host;
    int64_t rej = 0;
    if ((rc = shuffle_indices(ctx, ws, f->sw, nullptr, f->ca, n1, ctx->shuffle_rule, &rej)) != SRL_OK) return rc;
    inf.stage_ms[2] = ms_since(t0);

    // 4. subSampleFrame (:843-845): cells of point, which is still the raw LiDAR coordinate here (src/cloudProcessing.cpp:143)
    long long m = n1;
    const unsigned int* c = f->ca;
    if (prm->voxel_size > 0) {
        if (n1) {
            k_gather_xyz<<<grid_of(n1), T, 0, st>>>(f->raw1, f->ca, n1, f->pt);
            SRL_CUDA(ctx, cudaGetLastError());
            ctx->launches += 1;
            std::vector<uint32_t> keep((size_t)n1);
            size_t mk = 0;
            if ((rc = srl_grid_sampling(ctx, f->pt, (size_t)n1, sample_size, keep.data(), &mk)) != SRL_OK) return rc;
            m = (long long)mk;
            if (m) {
                SRL_CUDA(ctx, cudaMemcpyAsync(f->sel, keep.data(), (size_t)m * 4, cudaMemcpyHostToDevice, st));
                k_gather_u32<<<grid_of(m), T, 0, st>>>(f->ca, f->sel, m, f->cb);
                SRL_CUDA(ctx, cudaGetLastError());
                ctx->launches += 1;
            }
        }
        inf.stage_ms[3] = ms_since(t0);
        // 5. shuffle 2 (:847), the same engine
        if ((rc = shuffle_indices(ctx, ws, f->sw, f->cb, f->ca, m, ctx->shuffle_rule, &rej)) != SRL_OK) return rc;
        inf.stage_ms[4] = ms_since(t0);
    }
    inf.engine_words = (int64_t)ws.pos;
    inf.shuffle_rejections = rej;
    inf.n_points = m;

    // 6-7. the frame in its final order, transformAllImuPoint (:850), alpha_time and transformPoint (:860-878)
    f->n = (size_t)m;
    if (m) {
        k_frame_gather<<<grid_of(m), T, 0, st>>>(c, m, f->imu1, f->ts1, f->rel1, f->alpha1, f->src1, prm->index_frame <= 2 ? 1 : 0,
                                                 f->imu, f->ts, f->rel, f->alpha, f->src);
        SRL_CUDA(ctx, cudaGetLastError());
        ctx->launches += 1;
        if ((rc = srl_transform_all_imu_point(ctx, f->imu, (size_t)m, &states[n_states - 1], prm->R_il, prm->t_il, f->raw)) != SRL_OK) return rc;
        PassConst pc;
        std::memset(&pc, 0, sizeof(pc));
        const double q_id[4] = {0, 0, 0, 1};
        quat_to_rot(prm->index_frame > 2 ? prm->q_pred : q_id, pc.Rq);
        for (int i = 0; i < 3; ++i) { pc.t[i] = prm->index_frame > 2 ? prm->t_pred[i] : 0.0; pc.t_il[i] = prm->t_il[i]; }
        for (int i = 0; i < 9; ++i) pc.R_il[i] = prm->R_il[i];
        SRL_CUDA(ctx, launch_transform(f->raw, m, pc, f->point, st));
        ctx->launches += 1;
    }
    SRL_CUDA(ctx, cudaStreamSynchronize(st));
    inf.stage_ms[5] = ms_since(t0);
    if (info) *info = inf;
    return SRL_OK;
}

int srl_shuffle_replay(srl_ctx* ctx, const uint64_t* words, size_t n_words, size_t n, int32_t rule, uint32_t* perm_out,
                       size_t* words_used, uint64_t* next_word) {
    if (!ctx || (n && !perm_out) || (words && n_words == 0)) return SRL_BAD_ARG;
    if (rule != 0 && rule != 1) return set_err(ctx, SRL_BAD_ARG, "shuffle rule must be 0 (Lemire) or 1 (division)");
    if (n > 0x7fffffffULL) return set_err(ctx, SRL_BAD_ARG, "srl_shuffle_replay: n must fit in int32");
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    srl_cloud_frame f;
    f.ctx = ctx;
    f.device = ctx->device;
    int rc = frame_reserve(&f, n);
    if (rc != SRL_OK) return rc;
    WordStream ws;
    ws.ctx = ctx;
    ws.replay = reinterpret_cast<const unsigned long long*>(words);
    ws.n_replay = n_words;
    ws.host = ctx->shuffle_on_host;
    int64_t rej = 0;
    rc = shuffle_indices(ctx, ws, f.sw, nullptr, f.ca, (long long)n, rule, &rej);
    if (rc == SRL_OK && n) rc = cudaMemcpy(perm_out, f.ca, n * 4, cudaMemcpyDeviceToHost) == cudaSuccess ? SRL_OK : set_err(ctx, SRL_CUDA_ERROR, "copy");
    if (rc == SRL_OK && words_used) *words_used = ws.pos;
    if (rc == SRL_OK && next_word) {
        if (ws.host && !ws.replay) *next_word = ws.host_engine();
        else if (ws.replay) *next_word = ws.pos < n_words ? words[ws.pos] : 0;
        else {
            std::vector<unsigned long long> cache; size_t base = 0; unsigned long long w = 0;
            rc = ws.word(ws.pos, cache, base, w);
            *next_word = w;
        }
    }
    cudaStreamSynchronize(ctx->stream);
    return rc;
}

}  // extern "C"
