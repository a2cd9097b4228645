// srl_lidar.cu — cloudProcessing on the device (DESIGN.md row N10): the four handlers of src/cloudProcessing.cpp decode a message
// as it comes off the wire, order its points exactly as libstdc++'s std::sort does, filter them as written, and append them to
// a device-resident point_buffer that srl_lidar_cut pops as getMeasurements does (src/lioOptimization.cpp:719-723, 759-763).
//
// std::sort (libstdc++'s introsort) runs level by level: every segment of a level is one block, which partitions it in the
// two-scan form of __unguarded_partition (A = positions >= pivot left to right, B = positions <= pivot right to left; the
// sequential loop swaps A[k] <-> B[k] for the k below the first crossing and returns min(A[K], B[K-1])).  A segment whose depth
// limit is spent is heapsorted by one thread exactly as __partial_sort does; the segments of 16 or fewer end with a stable
// insertion sort each, which is what __final_insertion_sort does to them.  tests/cloud_processing_ref.py restates both forms.
//
// Compiled with --fmad=false: the keys, the blind test and the timestamps round every product and sum as the reference does.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <limits>

#include "srl_internal.h"

using namespace srl;

struct srl_lidar {
    srl_ctx* ctx = nullptr;
    int device = 0;
    srl_lidar_params p{};
    double scale = 1.0;                 // time_unit_scale: a double holding the float literal
    double last_end_time = -1.0;
    int given_offset_time = 0;
    int sweep_id = 0;
    // the queue: points [head, tail) of three device arrays of cap points
    DevArray<double> d_xyz, d_rel, d_ts;
    size_t cap = 0, head = 0, tail = 0;
    double front_ts = NAN, back_ts = NAN;
    DevArray<void> d_out;               // LidarOut
    PinnedArray<void> h_out;
};

namespace {

constexpr int kSortThreads = 1024;
constexpr int kThreshold = 16;          // _S_threshold
using SortScan = cub::BlockScan<int, kSortThreads>;

struct Seg {
    int first, last, depth;
};
struct LidarOut {
    long long appended;     // points appended to the queue
    long long count;        // points sorted
    double dt_last;         // dt_last_point
    double front_ts, back_ts;
    int given;              // given_offset_time of this message
    int bad;                // 1: ring >= N_SCANS on the yaw path, 2: NaN sort key
    long long cut_count;    // srl_lidar_cut: points popped
    int heapsorts;
    int pad_;
};
// the sort's scratch, carved per call
struct SortBufs {
    double* key;
    int* val;
    int* A;
    int* B;
    Seg* seg[2];
    int2* leaves;
    int* counters;          // [0, levels]: segments of each level; [levels + 1]: leaves; [levels + 2]: heapsorts
};

__host__ __device__ inline int lg(long long n) { int r = 0; while (n > 1) { n >>= 1; ++r; } return r; }

template <class T> __device__ __forceinline__ T ld(const unsigned char* p) {
    T v;
    unsigned char* d = reinterpret_cast<unsigned char*>(&v);
#pragma unroll
    for (int i = 0; i < (int)sizeof(T); ++i) d[i] = p[i];
    return v;
}

__device__ __forceinline__ void swap_kv(double* key, int* val, int i, int j) {
    const double k = key[i]; key[i] = key[j]; key[j] = k;
    const int v = val[i]; val[i] = val[j]; val[j] = v;
}

// __push_heap / __adjust_heap / __make_heap + __sort_heap over [first, first + len): __partial_sort(first, last, last)
__device__ void push_heap(double* key, int* val, int first, int hole, int top, double vk, int vv) {
    int parent = (hole - 1) / 2;
    while (hole > top && key[first + parent] < vk) {
        key[first + hole] = key[first + parent];
        val[first + hole] = val[first + parent];
        hole = parent;
        parent = (hole - 1) / 2;
    }
    key[first + hole] = vk;
    val[first + hole] = vv;
}
__device__ void adjust_heap(double* key, int* val, int first, int hole, int len, double vk, int vv) {
    const int top = hole;
    int second = hole;
    while (second < (len - 1) / 2) {
        second = 2 * (second + 1);
        if (key[first + second] < key[first + second - 1]) second--;
        key[first + hole] = key[first + second];
        val[first + hole] = val[first + second];
        hole = second;
    }
    if ((len & 1) == 0 && second == (len - 2) / 2) {
        second = 2 * (second + 1);
        key[first + hole] = key[first + second - 1];
        val[first + hole] = val[first + second - 1];
        hole = second - 1;
    }
    push_heap(key, val, first, hole, top, vk, vv);
}
__device__ void heapsort(double* key, int* val, int first, int last) {
    const int len = last - first;
    if (len >= 2) {
        for (int parent = (len - 2) / 2;; --parent) {
            adjust_heap(key, val, first, parent, len, key[first + parent], val[first + parent]);
            if (parent == 0) break;
        }
    }
    while (last - first > 1) {
        --last;
        const double vk = key[last];
        const int vv = val[last];
        key[last] = key[first];
        val[last] = val[first];
        adjust_heap(key, val, first, 0, last - first, vk, vv);
    }
}
// __move_median_to_first(result, a, b, c)
__device__ void move_median_to_first(double* key, int* val, int r, int a, int b, int c) {
    const double ka = key[a], kb = key[b], kc = key[c];
    int m;
    if (ka < kb) m = kb < kc ? b : (ka < kc ? c : a);
    else m = ka < kc ? a : (kb < kc ? c : b);
    swap_kv(key, val, r, m);
}

__device__ __forceinline__ void push_child(const SortBufs& s, int level, int first, int last, int depth) {
    const int n = last - first;
    if (n > kThreshold) {
        const int slot = atomicAdd(&s.counters[level + 1], 1);
        s.seg[(level + 1) & 1][slot] = Seg{first, last, depth};
    } else if (n > 1) {
        const int slot = atomicAdd(&s.counters[s.counters[-1] + 1], 1);
        s.leaves[slot] = make_int2(first, last);
    }
}

// the root segment: [0, count) with depth limit 2 * floor(log2 count); nothing when the keys were refused
__global__ void k_sort_root(SortBufs s, const long long* d_count, const int* d_bad) {
    const int n = (d_bad && *d_bad) ? 0 : (int)*d_count;
    if (n > kThreshold) {
        s.seg[0][0] = Seg{0, n, 2 * lg(n)};
        s.counters[0] = 1;
    } else if (n > 1) {
        s.leaves[0] = make_int2(0, n);
        s.counters[s.counters[-1] + 1] = 1;
    }
}

// one level of __introsort_loop: block b takes segments b, b + grid, ...
__global__ void __launch_bounds__(kSortThreads) k_sort_level(SortBufs s, int level) {
    __shared__ typename SortScan::TempStorage tmp;
    __shared__ int sh_K;
    const int nseg = s.counters[level];
    for (int si = blockIdx.x; si < nseg; si += gridDim.x) {
        const Seg g = s.seg[level & 1][si];
        if (g.depth == 0) {
            if (threadIdx.x == 0) {
                heapsort(s.key, s.val, g.first, g.last);
                atomicAdd(&s.counters[s.counters[-1] + 2], 1);
            }
            continue;
        }
        if (threadIdx.x == 0) move_median_to_first(s.key, s.val, g.first, g.first + 1, g.first + (g.last - g.first) / 2, g.last - 1);
        __syncthreads();
        const double p = s.key[g.first];
        const int lo = g.first + 1, hi = g.last;
        // A: positions in [lo, hi) whose key is not below the pivot, left to right
        int nA = 0;
        for (int t0 = lo; t0 < hi; t0 += kSortThreads) {
            const int i = t0 + (int)threadIdx.x;
            const int f = (i < hi && !(s.key[i] < p)) ? 1 : 0;
            int r, tot;
            SortScan(tmp).ExclusiveSum(f, r, tot);
            if (f) s.A[g.first + nA + r] = i;
            nA += tot;
            __syncthreads();
        }
        // B: positions whose key is not above the pivot, right to left
        int nB = 0;
        for (int t0 = hi - 1; t0 >= lo; t0 -= kSortThreads) {
            const int i = t0 - (int)threadIdx.x;
            const int f = (i >= lo && !(p < s.key[i])) ? 1 : 0;
            int r, tot;
            SortScan(tmp).ExclusiveSum(f, r, tot);
            if (f) s.B[g.first + nB + r] = i;
            nB += tot;
            __syncthreads();
        }
        // K: the first k where A[k] >= B[k]
        const int m = min(nA, nB);
        if (threadIdx.x == 0) sh_K = m;
        __syncthreads();
        for (int k = threadIdx.x; k < m; k += kSortThreads)
            if (s.A[g.first + k] >= s.B[g.first + k]) atomicMin(&sh_K, k);
        __syncthreads();
        const int K = sh_K;
        for (int k = threadIdx.x; k < K; k += kSortThreads) swap_kv(s.key, s.val, s.A[g.first + k], s.B[g.first + k]);
        if (threadIdx.x == 0) {
            const int ca = K < nA ? s.A[g.first + K] : hi;
            const int cb = K > 0 ? s.B[g.first + K - 1] : hi;
            const int cut = min(ca, cb);
            push_child(s, level, cut, g.last, g.depth - 1);
            push_child(s, level, g.first, cut, g.depth - 1);
        }
        __syncthreads();
    }
}

// __final_insertion_sort on each leaf: a stable insertion sort
__global__ void k_sort_leaves(SortBufs s) {
    const int nl = s.counters[s.counters[-1] + 1];
    for (int li = blockIdx.x * blockDim.x + threadIdx.x; li < nl; li += gridDim.x * blockDim.x) {
        const int2 r = s.leaves[li];
        for (int i = r.x + 1; i < r.y; ++i) {
            const double vk = s.key[i];
            const int vv = s.val[i];
            int j = i;
            while (j > r.x && vk < s.key[j - 1]) {
                s.key[j] = s.key[j - 1];
                s.val[j] = s.val[j - 1];
                --j;
            }
            s.key[j] = vk;
            s.val[j] = vv;
        }
    }
}

// scratch of the sort over at most n keys
struct SortLayout {
    int levels;
    size_t nseg;
    void take(Carve& c, SortBufs& s, size_t n) {
        levels = 2 * lg((long long)std::max<size_t>(n, 1));
        nseg = n / (kThreshold + 1) + 2;
        s.key = c.take<double>(n);
        s.val = c.take<int>(n);
        s.A = c.take<int>(n);
        s.B = c.take<int>(n);
        s.seg[0] = c.take<Seg>(nseg);
        s.seg[1] = c.take<Seg>(nseg);
        s.leaves = c.take<int2>(n + 1);
        s.counters = c.take<int>(levels + 5);
    }
};

// counters[0] holds the level count so that counters + 1 is the array the kernels index (counters[-1] = levels)
int run_sort(srl_ctx* ctx, SortBufs s, const SortLayout& L, size_t n_max, const long long* d_count, const int* d_bad) {
    cudaStream_t st = ctx->stream;
    int* base = s.counters;
    SRL_CUDA(ctx, cudaMemsetAsync(base, 0, (L.levels + 5) * sizeof(int), st));
    SRL_CUDA(ctx, cudaMemcpyAsync(base, &L.levels, sizeof(int), cudaMemcpyHostToDevice, st));
    s.counters = base + 1;
    k_sort_root<<<1, 1, 0, st>>>(s, d_count, d_bad);
    int launches = 1;
    for (int level = 0; level <= L.levels; ++level) {
        const long long bound = std::min<long long>({1LL << std::min(level, 40), (long long)L.nseg, (long long)ctx->sm_count});
        k_sort_level<<<(unsigned)std::max<long long>(bound, 1), kSortThreads, 0, st>>>(s, level);
        ++launches;
    }
    const unsigned lg_grid = (unsigned)std::min<size_t>((n_max / 2 + 255) / 256 + 1, 4096);
    k_sort_leaves<<<lg_grid, 256, 0, st>>>(s);
    ctx->launches += launches + 1;
    SRL_CUDA(ctx, cudaGetLastError());
    return SRL_OK;
}

// ---- decoding
struct CloudArgs {
    const unsigned char* data;
    int n, step, ox, oy, oz, ot, oring, type;   // type: 2 VELO, 3 OUST, 4 ROBO
    int width;
    long long row_step;
    int n_scans;
    double scale, omega, stamp, last_end_time, blind2;
    int filter;
};
// point i of row i / width
__device__ __forceinline__ const unsigned char* cloud_point(const CloudArgs& a, int i) {
    return a.data + (size_t)(i / a.width) * (size_t)a.row_step + (size_t)(i % a.width) * (size_t)a.step;
}
__device__ __forceinline__ double cloud_time(const CloudArgs& a, int i) {
    const unsigned char* p = cloud_point(a, i) + a.ot;
    if (a.type == 2) return (double)ld<float>(p);
    if (a.type == 3) return (double)ld<unsigned>(p);
    return ld<double>(p);
}
__device__ __forceinline__ int cloud_ring(const CloudArgs& a, int i) {
    if (a.oring < 0) return 0;
    const unsigned char* p = cloud_point(a, i) + a.oring;
    return a.type == 3 ? (int)p[0] : (int)ld<unsigned short>(p);
}
__device__ __forceinline__ void cloud_xyz(const CloudArgs& a, int i, double& x, double& y, double& z) {
    const unsigned char* p = cloud_point(a, i);
    x = (double)ld<float>(p + a.ox);
    y = (double)ld<float>(p + a.oy);
    z = (double)ld<float>(p + a.oz);
}
__device__ __forceinline__ double yaw_deg(double x, double y) { return __dmul_rn(atan2(y, x), 57.2957); }

__global__ void k_ring_first_init(int* first, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) first[i] = INT_MAX;
}
// the given flag (the last point's time > 0, in input order) and the first point of each ring
__global__ void k_cloud_rings(CloudArgs a, int* ring_first, int* d_bad) {
    const bool given = cloud_time(a, a.n - 1) > 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
        if (given) return;
        const int r = cloud_ring(a, i);
        if (r >= a.n_scans) atomicMax(d_bad, 1);
        else atomicMin(&ring_first[r], i);
    }
}
// sort keys: the time field (given) or the yaw-derived relative_time
__global__ void k_cloud_keys(CloudArgs a, const int* ring_first, double* key, int* val, int* d_bad) {
    const bool given = cloud_time(a, a.n - 1) > 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
        double k;
        if (given) {
            k = cloud_time(a, i);
        } else {
            const int r = cloud_ring(a, i);
            if (r >= a.n_scans) { k = 0.0; }
            else if (ring_first[r] == i) { k = 0.0; }
            else {
                double x, y, z, x0, y0, z0;
                cloud_xyz(a, i, x, y, z);
                cloud_xyz(a, ring_first[r], x0, y0, z0);
                const double yaw = yaw_deg(x, y), yf = yaw_deg(x0, y0);
                k = yaw <= yf ? __ddiv_rn(__dsub_rn(yf, yaw), a.omega) : __ddiv_rn(__dadd_rn(__dsub_rn(yf, yaw), 360.0), a.omega);
            }
        }
        if (k != k) atomicMax(d_bad, 2);
        key[i] = k;
        val[i] = i;
    }
}
// ---- Livox CustomPoint records
struct LivoxArgs {
    const unsigned char* rec;
    int n, stride, n_scans;
    double scale, stamp, blind2;
    int filter;
};
__device__ __forceinline__ float lv_f(const LivoxArgs& a, int i, int off) { return ld<float>(a.rec + (size_t)i * a.stride + off); }
// the r3live gate of livoxHandler (:136-153) on record i >= 1
__global__ void k_livox_flags(LivoxArgs a, int* flags) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
        int keep = 0;
        if (i >= 1) {
            const unsigned char* r = a.rec + (size_t)i * a.stride;
            const float x = ld<float>(r + 4), y = ld<float>(r + 8), z = ld<float>(r + 12);
            const unsigned tag = r[17], line = r[18];
            // IS_VALID's unqualified abs is the float overload; the float compares with the double 1e8
            if ((int)line < a.n_scans && !((double)fabsf(x) > 1e8) && !((double)fabsf(y) > 1e8) && !((double)fabsf(z) > 1e8) &&
                (double)x > 0.7) {
                if (!((double)x > 2.0 && ((tag & 0x03u) != 0 || (tag & 0x0Cu) != 0))) {
                    const float xp = lv_f(a, i - 1, 4), yp = lv_f(a, i - 1, 8), zp = lv_f(a, i - 1, 12);
                    keep = ((double)fabsf(__fsub_rn(x, xp)) > 1e-7 || (double)fabsf(__fsub_rn(y, yp)) > 1e-7 ||
                            (double)fabsf(__fsub_rn(z, zp)) > 1e-7) ? 1 : 0;
                }
            }
        }
        flags[i] = keep;
    }
}
__global__ void k_livox_keys(LivoxArgs a, const int* cand, const long long* d_count, double* key, int* val) {
    const int n = (int)*d_count;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int j = cand[i];
        key[i] = __dmul_rn((double)ld<unsigned>(a.rec + (size_t)j * a.stride), a.scale);
        val[i] = j;
    }
}

// the emission of both paths: flag pass (out == nullptr) and scatter pass
struct Queue {
    double* xyz;
    double* rel;
    double* ts;
    long long tail;
};
template <bool kLivox>
__device__ __forceinline__ bool emit_point(const LivoxArgs& la, const CloudArgs& ca, const double* key, const int* val,
                                           const int* ring_first, int i, bool given, double* xyz, double& rel, double& ts) {
    if (kLivox) {
        if (((unsigned)i + 1u) % (unsigned)la.filter != 0u) return false;
        const unsigned char* r = la.rec + (size_t)val[i] * la.stride;
        xyz[0] = (double)ld<float>(r + 4); xyz[1] = (double)ld<float>(r + 8); xyz[2] = (double)ld<float>(r + 12);
        if (!(__dadd_rn(__dadd_rn(__dmul_rn(xyz[0], xyz[0]), __dmul_rn(xyz[1], xyz[1])), __dmul_rn(xyz[2], xyz[2])) > la.blind2)) return false;
        rel = key[i];
        ts = __dadd_rn(__ddiv_rn(rel, 1000.0), la.stamp);
        return true;
    }
    if (i % ca.filter != 0) return false;
    const int j = val[i];
    cloud_xyz(ca, j, xyz[0], xyz[1], xyz[2]);
    if (given) {
        if (!(__dadd_rn(__dadd_rn(__dmul_rn(xyz[0], xyz[0]), __dmul_rn(xyz[1], xyz[1])), __dmul_rn(xyz[2], xyz[2])) > ca.blind2)) return false;
        rel = ca.type == 4 ? __dmul_rn(__dsub_rn(key[i], key[0]), ca.scale) : __dmul_rn(key[i], ca.scale);
        ts = __dadd_rn(__ddiv_rn(rel, 1000.0), ca.stamp);
    } else {
        // no blind test; the first point of its ring keeps relative_time 0 and point3D's default timestamp 0
        rel = key[i];
        ts = ring_first[cloud_ring(ca, j)] == j ? 0.0 : __dadd_rn(__ddiv_rn(rel, 1000.0), ca.stamp);
    }
    return ts > ca.last_end_time;
}

template <bool kLivox>
__global__ void k_emit(LivoxArgs la, CloudArgs ca, const double* key, const int* val, const long long* d_count, const int* d_bad,
                       const int* ring_first, int* flags, const int* pos, Queue q) {
    const int n = (d_bad && *d_bad) ? 0 : (int)*d_count;
    const int n_all = kLivox ? la.n : ca.n;
    const bool given = kLivox ? true : cloud_time(ca, ca.n - 1) > 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_all; i += gridDim.x * blockDim.x) {
        double xyz[3], rel = 0.0, ts = 0.0;
        bool keep = false;
        if (i < n) keep = emit_point<kLivox>(la, ca, key, val, ring_first, i, given, xyz, rel, ts);
        if (!pos) {
            flags[i] = keep ? 1 : 0;
        } else if (keep) {
            const long long o = q.tail + pos[i];
            q.xyz[3 * o] = xyz[0]; q.xyz[3 * o + 1] = xyz[1]; q.xyz[3 * o + 2] = xyz[2];
            q.rel[o] = rel;
            q.ts[o] = ts;
        }
    }
}

// what the host keeps: appended count, dt_last_point, the given flag, the queue's front and back timestamps
template <bool kLivox>
__global__ void k_finish(LivoxArgs la, CloudArgs ca, const double* key, const long long* d_count, const int* d_bad, const int* flags,
                         const int* pos, int n_all, Queue q, long long head, LidarOut* out, const int* heapsorts) {
    const long long n = *d_count;
    out->count = n;
    out->bad = d_bad ? *d_bad : 0;
    out->given = kLivox ? 0 : (cloud_time(ca, ca.n - 1) > 0 ? 1 : 0);
    const long long app = (n_all > 0 && !out->bad) ? (long long)pos[n_all - 1] + flags[n_all - 1] : 0;
    out->appended = app;
    out->dt_last = n > 0 ? ((kLivox || !out->given) ? key[n - 1] : __dmul_rn(key[n - 1], ca.scale)) : 0.0;
    const long long tail = q.tail + app;
    out->front_ts = tail > head ? q.ts[head] : NAN;
    out->back_ts = tail > head ? q.ts[tail - 1] : NAN;
    out->heapsorts = heapsorts ? *heapsorts : 0;
}

// the first queued point whose timestamp is not below t
__global__ void k_cut(const double* ts, long long head, long long tail, double t, unsigned long long* first) {
    for (long long i = head + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < tail; i += (long long)gridDim.x * blockDim.x)
        if (!(ts[i] < t)) { atomicMin(first, (unsigned long long)i); return; }
}
__global__ void k_cut_finish(const double* ts, long long head, long long tail, const unsigned long long* first, LidarOut* out) {
    const unsigned long long fu = *first;   // all ones when no queued point stops the pops
    const long long f = fu < (unsigned long long)tail ? (long long)fu : tail;
    out->cut_count = f - head;
    out->front_ts = f < tail ? ts[f] : NAN;
}

__global__ void k_replay_keys(const double* in, int n, double* key, int* val, int* d_bad) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const double k = in[i];
        if (k != k) atomicMax(d_bad, 2);
        key[i] = k;
        val[i] = i;
    }
}

unsigned grid_for(size_t n, int threads = 256) { return (unsigned)std::max<size_t>(1, std::min<size_t>((n + threads - 1) / threads, 8192)); }

// room for `extra` more points behind the queue: a full queue moves to buffers of at least twice its size
int reserve(srl_lidar* l, size_t extra) {
    srl_ctx* ctx = l->ctx;
    const size_t size = l->tail - l->head;
    if (l->tail + extra <= l->cap) return SRL_OK;
    size_t cap = l->cap;
    if (size + extra > cap || l->head == 0) cap = std::max(2 * cap, size + extra);
    DevArray<double> xyz, rel, ts;
    SRL_CUDA(ctx, xyz.alloc(cap * 3));
    SRL_CUDA(ctx, rel.alloc(cap));
    SRL_CUDA(ctx, ts.alloc(cap));
    if (size) {
        SRL_CUDA(ctx, cudaMemcpyAsync(xyz, l->d_xyz + 3 * l->head, size * 3 * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
        SRL_CUDA(ctx, cudaMemcpyAsync(rel, l->d_rel + l->head, size * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
        SRL_CUDA(ctx, cudaMemcpyAsync(ts, l->d_ts + l->head, size * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
    }
    SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    l->d_xyz = std::move(xyz); l->d_rel = std::move(rel); l->d_ts = std::move(ts);
    l->cap = cap;
    l->tail = size;
    l->head = 0;
    return SRL_OK;
}

// the common tail of both handlers: emission flags, their scan, the scatter, the summary and its read-back
template <bool kLivox>
int emit_and_finish(srl_lidar* l, const LivoxArgs& la, const CloudArgs& ca, const SortBufs& s, const long long* d_count, const int* d_bad,
                    const int* ring_first, int* flags, int* pos, void* cub_tmp, size_t cub_bytes, int n_all, LidarOut* h) {
    srl_ctx* ctx = l->ctx;
    cudaStream_t st = ctx->stream;
    Queue q{l->d_xyz, l->d_rel, l->d_ts, (long long)l->tail};
    const unsigned grid = grid_for(n_all);
    k_emit<kLivox><<<grid, 256, 0, st>>>(la, ca, s.key, s.val, d_count, d_bad, ring_first, flags, nullptr, q);
    SRL_CUDA(ctx, cub::DeviceScan::ExclusiveSum(cub_tmp, cub_bytes, flags, pos, n_all, st));
    k_emit<kLivox><<<grid, 256, 0, st>>>(la, ca, s.key, s.val, d_count, d_bad, ring_first, flags, pos, q);
    k_finish<kLivox><<<1, 1, 0, st>>>(la, ca, s.key, d_count, d_bad, flags, pos, n_all, q, (long long)l->head,
                                      static_cast<LidarOut*>(l->d_out.get()), nullptr);
    ctx->launches += 4;
    SRL_CUDA(ctx, cudaGetLastError());
    SRL_CUDA(ctx, cudaMemcpyAsync(h, l->d_out, sizeof(LidarOut), cudaMemcpyDeviceToHost, st));
    SRL_CUDA(ctx, cudaStreamSynchronize(st));
    return SRL_OK;
}

void apply_out(srl_lidar* l, const LidarOut& o) {
    l->tail += (size_t)o.appended;
    l->front_ts = o.front_ts;
    l->back_ts = o.back_ts;
}

}  // namespace

extern "C" {

int srl_lidar_create(srl_ctx* ctx, const srl_lidar_params* params, size_t initial_capacity, srl_lidar** out) {
    if (!ctx || !params || !out) return SRL_BAD_ARG;
    *out = nullptr;
    const srl_lidar_params& p = *params;
    if (p.lidar_type < 1 || p.lidar_type > 4) return set_err(ctx, SRL_BAD_ARG, "srl_lidar_create: lidar_type must be 1..4");
    if (p.n_scans < 1 || p.scan_rate < 1 || p.point_filter_num < 1)
        return set_err(ctx, SRL_BAD_ARG, "srl_lidar_create: n_scans, scan_rate and point_filter_num must be >= 1");
    if (initial_capacity > 0x7fffffffULL) return set_err(ctx, SRL_BAD_ARG, "srl_lidar_create: capacity must fit in int32");
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    std::unique_ptr<srl_lidar> l(new srl_lidar());
    l->ctx = ctx;
    l->device = ctx->device;
    l->p = p;
    // setTimeUnit: float literals held in a double
    l->scale = p.time_unit == 0 ? (double)1.e3f : p.time_unit == 2 ? (double)1.e-3f : p.time_unit == 3 ? (double)1.e-6f : (double)1.f;
    cudaError_t e = l->d_out.alloc(sizeof(LidarOut));
    if (e == cudaSuccess) e = l->h_out.alloc(sizeof(LidarOut));
    if (e != cudaSuccess) return cuda_fail(ctx, e, "srl_lidar_create");
    const int rc = reserve(l.get(), std::max<size_t>(initial_capacity, 1));
    if (rc != SRL_OK) return rc;
    *out = l.release();
    return SRL_OK;
}

void srl_lidar_destroy(srl_lidar* l) {
    if (!l) return;
    cudaSetDevice(l->device);
    cudaDeviceSynchronize();   // the last message's copy into the pinned summary has landed
    delete l;
}

int srl_lidar_livox(srl_lidar* l, const uint8_t* records, size_t n, size_t stride, double stamp, int64_t* appended) {
    if (!l) return SRL_BAD_ARG;
    srl_ctx* ctx = l->ctx;
    if (appended) *appended = 0;
    if (n > 0 && !records) return set_err(ctx, SRL_BAD_ARG, "srl_lidar_livox: null records");
    if (stride < 19) return set_err(ctx, SRL_BAD_ARG, "srl_lidar_livox: stride must be >= 19");
    if (n > 0x7fffffffULL || n * stride > (size_t)1 << 40) return set_err(ctx, SRL_BAD_ARG, "srl_lidar_livox: message too large");
    if (n < 2) return SRL_OK;   // record 0 is never taken: nothing to append, last_end_time kept
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    int rc = reserve(l, n);
    if (rc != SRL_OK) return rc;
    cudaStream_t st = ctx->stream;
    Staged<const uint8_t> in(records);
    SortBufs s{};
    SortLayout L{};
    int *flags = nullptr, *pos = nullptr, *cand = nullptr;
    long long* d_count = nullptr;
    void* cub_tmp = nullptr;
    size_t b1 = 0, b2 = 0;
    cub::DeviceSelect::Flagged(nullptr, b1, thrust::counting_iterator<int>(0), (int*)nullptr, (int*)nullptr, (long long*)nullptr, (int)n, st);
    cub::DeviceScan::ExclusiveSum(nullptr, b2, (int*)nullptr, (int*)nullptr, (int)n, st);
    size_t cub_bytes = std::max(b1, b2);
    rc = carve_scratch(ctx, [&](Carve& c) {
        in.place(c, n * stride);
        L.take(c, s, n);
        flags = c.take<int>(n);
        pos = c.take<int>(n);
        cand = c.take<int>(n);
        d_count = c.take<long long>(1);
        cub_tmp = c.take<char>(cub_bytes);
    });
    if (rc != SRL_OK) return rc;
    rc = in.upload(ctx, n * stride);
    if (rc != SRL_OK) return rc;
    LivoxArgs la{in.d, (int)n, (int)stride, l->p.n_scans, l->scale, stamp, l->p.blind * l->p.blind, l->p.point_filter_num};
    CloudArgs ca{};
    k_livox_flags<<<grid_for(n), 256, 0, st>>>(la, flags);
    SRL_CUDA(ctx, cub::DeviceSelect::Flagged(cub_tmp, cub_bytes, thrust::counting_iterator<int>(0), flags, cand, d_count, (int)n, st));
    k_livox_keys<<<grid_for(n), 256, 0, st>>>(la, cand, d_count, s.key, s.val);
    ctx->launches += 2;
    rc = run_sort(ctx, s, L, n, d_count, nullptr);
    if (rc != SRL_OK) return rc;
    s.counters += 1;
    LidarOut& h = *static_cast<LidarOut*>(l->h_out.get());
    rc = emit_and_finish<true>(l, la, ca, s, d_count, nullptr, nullptr, flags, pos, cub_tmp, cub_bytes, (int)n, &h);
    if (rc != SRL_OK) return rc;
    apply_out(l, h);
    if (h.count > 0) l->last_end_time = stamp + h.dt_last / 1000.0;
    if (appended) *appended = h.appended;
    return SRL_OK;
}

int srl_lidar_process(srl_lidar* l, const uint8_t* data, size_t n, const srl_cloud2_layout* layout, double stamp, int64_t* appended) {
    if (!l) return SRL_BAD_ARG;
    srl_ctx* ctx = l->ctx;
    if (appended) *appended = 0;
    const int type = l->p.lidar_type;
    if (type == 1) return set_err(ctx, SRL_BAD_ARG, "srl_lidar_process: a Livox lidar takes srl_lidar_livox");
    if (!layout || (n > 0 && !data)) return set_err(ctx, SRL_BAD_ARG, "srl_lidar_process: null layout or data");
    const srl_cloud2_layout& y = *layout;
    const int tsz = type == 4 ? 8 : 4, rsz = type == 3 ? 1 : 2;
    const long long step = y.point_step;
    auto fits = [&](int off, int sz) { return off >= 0 && off + sz <= step; };
    if (!fits(y.off_x, 4) || !fits(y.off_y, 4) || !fits(y.off_z, 4) || !fits(y.off_time, tsz) || (y.off_ring >= 0 && !fits(y.off_ring, rsz)))
        return set_err(ctx, SRL_BAD_ARG, "srl_lidar_process: a field lies outside point_step");
    if (n > 0x7fffffffULL || n * (size_t)step > (size_t)1 << 40) return set_err(ctx, SRL_BAD_ARG, "srl_lidar_process: message too large");
    const size_t width = y.width ? y.width : std::max<size_t>(n, 1);
    const size_t row_step = y.row_step ? y.row_step : width * (size_t)step;
    if (row_step < width * (size_t)step || n % width != 0 || row_step > ((size_t)1 << 40) / std::max<size_t>(n / width, 1))
        return set_err(ctx, SRL_BAD_ARG, "srl_lidar_process: row_step below width * point_step, or n not a multiple of width");
    if (n == 0) { l->sweep_id++; return SRL_OK; }
    const size_t bytes = (n / width) * row_step;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    int rc = reserve(l, n);
    if (rc != SRL_OK) return rc;
    cudaStream_t st = ctx->stream;
    Staged<const uint8_t> in(data);
    SortBufs s{};
    SortLayout L{};
    int *flags = nullptr, *pos = nullptr, *ring_first = nullptr, *d_bad = nullptr;
    long long* d_count = nullptr;
    void* cub_tmp = nullptr;
    size_t cub_bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, cub_bytes, (int*)nullptr, (int*)nullptr, (int)n, st);
    rc = carve_scratch(ctx, [&](Carve& c) {
        in.place(c, bytes);
        L.take(c, s, n);
        flags = c.take<int>(n);
        pos = c.take<int>(n);
        ring_first = c.take<int>(l->p.n_scans);
        d_bad = c.take<int>(1);
        d_count = c.take<long long>(1);
        cub_tmp = c.take<char>(cub_bytes);
    });
    if (rc != SRL_OK) return rc;
    rc = in.upload(ctx, bytes);
    if (rc != SRL_OK) return rc;
    CloudArgs ca{in.d, (int)n, (int)step, y.off_x, y.off_y, y.off_z, y.off_time, y.off_ring, type, (int)width, (long long)row_step,
                 l->p.n_scans, l->scale,
                 0.361 * l->p.scan_rate, stamp, l->last_end_time, l->p.blind * l->p.blind, l->p.point_filter_num};
    LivoxArgs la{};
    const long long nn = (long long)n;
    SRL_CUDA(ctx, cudaMemsetAsync(d_bad, 0, sizeof(int), st));
    SRL_CUDA(ctx, cudaMemcpyAsync(d_count, &nn, sizeof(nn), cudaMemcpyHostToDevice, st));
    k_ring_first_init<<<(l->p.n_scans + 255) / 256, 256, 0, st>>>(ring_first, l->p.n_scans);
    k_cloud_rings<<<grid_for(n), 256, 0, st>>>(ca, ring_first, d_bad);
    k_cloud_keys<<<grid_for(n), 256, 0, st>>>(ca, ring_first, s.key, s.val, d_bad);
    ctx->launches += 3;
    rc = run_sort(ctx, s, L, n, d_count, d_bad);
    if (rc != SRL_OK) return rc;
    s.counters += 1;
    LidarOut& h = *static_cast<LidarOut*>(l->h_out.get());
    rc = emit_and_finish<false>(l, la, ca, s, d_count, d_bad, ring_first, flags, pos, cub_tmp, cub_bytes, (int)n, &h);
    if (rc != SRL_OK) return rc;
    if (h.bad) return set_err(ctx, SRL_BAD_ARG, h.bad == 1 ? "srl_lidar_process: ring >= n_scans" : "srl_lidar_process: NaN sort key");
    apply_out(l, h);
    l->given_offset_time = h.given;
    l->last_end_time = stamp + h.dt_last / 1000.0;
    l->sweep_id++;
    if (appended) *appended = h.appended;
    return SRL_OK;
}

int srl_lidar_cut(srl_lidar* l, double t, int64_t* count, const double** raw_xyz, const double** timestamp) {
    if (!l) return SRL_BAD_ARG;
    srl_ctx* ctx = l->ctx;
    const size_t head = l->head;
    if (count) *count = 0;
    if (raw_xyz) *raw_xyz = l->d_xyz + 3 * head;
    if (timestamp) *timestamp = l->d_ts + head;
    if (l->tail == head) return SRL_OK;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    unsigned long long* first = nullptr;
    int rc = carve_scratch(ctx, [&](Carve& c) { first = c.take<unsigned long long>(1); });
    if (rc != SRL_OK) return rc;
    SRL_CUDA(ctx, cudaMemsetAsync(first, 0xff, sizeof(unsigned long long), st));
    k_cut<<<grid_for(l->tail - head), 256, 0, st>>>(l->d_ts, (long long)head, (long long)l->tail, t, first);
    k_cut_finish<<<1, 1, 0, st>>>(l->d_ts, (long long)head, (long long)l->tail, first, static_cast<LidarOut*>(l->d_out.get()));
    ctx->launches += 2;
    SRL_CUDA(ctx, cudaGetLastError());
    LidarOut& h = *static_cast<LidarOut*>(l->h_out.get());
    SRL_CUDA(ctx, cudaMemcpyAsync(&h, l->d_out, sizeof(LidarOut), cudaMemcpyDeviceToHost, st));
    SRL_CUDA(ctx, cudaStreamSynchronize(st));
    l->head += (size_t)h.cut_count;
    l->front_ts = h.front_ts;
    if (l->head == l->tail) l->back_ts = NAN;
    if (count) *count = h.cut_count;
    return SRL_OK;
}

int srl_lidar_info_get(srl_lidar* l, srl_lidar_info* info) {
    if (!l || !info) return SRL_BAD_ARG;
    info->last_end_time = l->last_end_time;
    info->given_offset_time = l->given_offset_time;
    info->sweep_id = l->sweep_id;
    info->sweep_interval = 1 / double(l->p.scan_rate);
    info->size = (int64_t)(l->tail - l->head);
    info->front_timestamp = l->front_ts;
    info->back_timestamp = l->back_ts;
    info->capacity = (int64_t)l->cap;
    return SRL_OK;
}

int srl_lidar_download(srl_lidar* l, double* raw_xyz, double* relative_time, double* timestamp) {
    if (!l) return SRL_BAD_ARG;
    srl_ctx* ctx = l->ctx;
    const size_t n = l->tail - l->head;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    int rc = SRL_OK;
    if (raw_xyz && rc == SRL_OK) rc = copy_to_host(ctx, raw_xyz, l->d_xyz + 3 * l->head, n * 3 * sizeof(double));
    if (relative_time && rc == SRL_OK) rc = copy_to_host(ctx, relative_time, l->d_rel + l->head, n * sizeof(double));
    if (timestamp && rc == SRL_OK) rc = copy_to_host(ctx, timestamp, l->d_ts + l->head, n * sizeof(double));
    return rc;
}

int srl_lidar_sort_replay(srl_ctx* ctx, const double* keys, size_t n, int32_t* perm_out, int32_t* heapsorts) {
    if (!ctx || (n > 0 && (!keys || !perm_out))) return SRL_BAD_ARG;
    if (n > 0x7fffffffULL) return set_err(ctx, SRL_BAD_ARG, "srl_lidar_sort_replay: n must fit in int32");
    if (heapsorts) *heapsorts = 0;
    if (n == 0) return SRL_OK;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    Staged<const double> in(keys);
    SortBufs s{};
    SortLayout L{};
    long long* d_count = nullptr;
    int* d_bad = nullptr;
    int rc = carve_scratch(ctx, [&](Carve& c) {
        in.place(c, n);
        L.take(c, s, n);
        d_count = c.take<long long>(1);
        d_bad = c.take<int>(1);
    });
    if (rc != SRL_OK) return rc;
    rc = in.upload(ctx, n);
    if (rc != SRL_OK) return rc;
    const long long nn = (long long)n;
    SRL_CUDA(ctx, cudaMemsetAsync(d_bad, 0, sizeof(int), st));
    SRL_CUDA(ctx, cudaMemcpyAsync(d_count, &nn, sizeof(nn), cudaMemcpyHostToDevice, st));
    k_replay_keys<<<grid_for(n), 256, 0, st>>>(in.d, (int)n, s.key, s.val, d_bad);
    ctx->launches += 1;
    rc = run_sort(ctx, s, L, n, d_count, d_bad);
    if (rc != SRL_OK) return rc;
    int tail[2] = {0, 0};
    SRL_CUDA(ctx, cudaMemcpyAsync(&tail[0], d_bad, sizeof(int), cudaMemcpyDeviceToHost, st));
    SRL_CUDA(ctx, cudaMemcpyAsync(&tail[1], s.counters + L.levels + 3, sizeof(int), cudaMemcpyDeviceToHost, st));
    SRL_CUDA(ctx, cudaStreamSynchronize(st));
    if (tail[0]) return set_err(ctx, SRL_BAD_ARG, "srl_lidar_sort_replay: NaN key");
    if (heapsorts) *heapsorts = tail[1];
    return copy_to_host(ctx, perm_out, s.val, n * sizeof(int32_t));
}

}  // extern "C"
