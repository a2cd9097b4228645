// srl_flow_tracker.cu — the optical-flow tracker's bookkeeping around its Lucas-Kanade (DESIGN.md row N9): opticalFlowTracker's
// init / trackImage (src/opticalFlowTracker.cpp:111-211), removeOutlierUsingRansacPnp (:267-323) with the caller's inliers, and
// updateAndAppendTrackPoints (:13-102).  The reference keeps map_rgb_points_in_last_image_pose / _cur_image_pose as
// std::map<rgbPoint*, cv::Point2f>; here both sets live on the device as arrays sorted by colour-map point id, the device's
// fixed stand-in for the pointer order (DESIGN.md section 5).  Sets hold a few hundred points, so the per-set passes run in
// one block of kSetThreads threads that walks the set in tiles with a carried block scan; only the refresh candidates (up to
// about 10^4) get grid-wide kernels and a device sort.  Every entry point ends with at most one read-back of counts.
//
// Compiled with --fmad=false: the velocities, the reprojection errors and the projections round every product and sum on its
// own, as the reference's scalar code does.
#include <cub/cub.cuh>

#include <algorithm>
#include <cmath>
#include <limits>

#include "srl_internal.h"

using namespace srl;

namespace {

constexpr int kSetThreads = 1024;
constexpr unsigned kNoId = 0xffffffffu;
using SetScan = cub::BlockScan<int, kSetThreads>;

struct MaxI { __device__ __forceinline__ int operator()(int a, int b) const { return b > a ? b : a; } };

__device__ __forceinline__ const float* point_xyz(const ColorMapView& m, unsigned id) {
    const unsigned blk = id / (unsigned)m.block_pts;
    return m.blocks + (size_t)blk * (4 * m.block_pts) + 4 * (size_t)(id - blk * (unsigned)m.block_pts);
}
__device__ __forceinline__ unsigned long long cell_key(double u, double v, double min_dis, int u0, int v0, int bits_v) {
    const int cu = projection_cell(u, min_dis), cv = projection_cell(v, min_dis);
    return ((unsigned long long)(unsigned)(cu - u0) << bits_v) | (unsigned long long)(unsigned)(cv - v0);
}
// the first index in sorted[0, n) whose value is not below x
__device__ __forceinline__ int lower_bound_u32(const unsigned* sorted, int n, unsigned x) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (sorted[mid] < x) lo = mid + 1; else hi = mid;
    }
    return lo;
}
// if2dPointsAvailable(x, y, 1.0, 0.05) (src/lioOptimization.cpp:48-60): the margin is given, so the frame's own is not read
__device__ __forceinline__ bool in_margin(double x, double y, int cols, int rows) {
    const double m = 0.05;
    return x >= __dadd_rn(__dmul_rn(m, (double)cols), 1.0) && ceil(x) < __dmul_rn(__dsub_rn(1.0, m), (double)cols) &&
           y >= __dadd_rn(__dmul_rn(m, (double)rows), 1.0) && ceil(y) < __dmul_rn(__dsub_rn(1.0, m), (double)rows);
}
// (cur - last) / dt with cv::Point_<float> arithmetic: a float difference, saturate_cast<float>(x / dt), widened to double;
// Point2f(1e-3, 1e-3) when dt < 1e-5 (:164-169)
__device__ __forceinline__ double velocity(float cur, float last, double dt) {
    if (dt < 1e-5) return (double)1e-3f;
    return (double)__double2float_rn(__ddiv_rn((double)__fsub_rn(cur, last), dt));
}

// trackImage after the Lucas-Kanade call (:136-171): the matches (status set) in `last` order with their margin flag and
// velocity, and `cur` = the matches inside the 0.05 margin whose mask byte is set (mask null: all).  With lk_uv == nullptr
// the match list is kept and only `cur` is rebuilt from it (rejectMatches).  counts[0] = matches, counts[1] = cur.
__global__ void __launch_bounds__(kSetThreads) k_ft_track(int n, const unsigned* __restrict__ last_ids, const float2* __restrict__ last_uv,
                                                          const float2* __restrict__ lk_uv, const unsigned char* __restrict__ status,
                                                          double dt, int cols, int rows, unsigned* m_ids, float2* m_last, float2* m_uv,
                                                          double2* m_vel, unsigned char* m_in, const unsigned char* __restrict__ mask,
                                                          unsigned* c_ids, float2* c_uv, double2* c_vel, long long* counts) {
    __shared__ typename SetScan::TempStorage tmp;
    int base_m = 0, base_c = 0;
    for (int t0 = 0; t0 < n; t0 += kSetThreads) {
        const int i = t0 + (int)threadIdx.x;
        bool match = false, in = false;
        if (i < n) {
            if (lk_uv) {
                match = status[i] != 0;
                if (match) in = in_margin((double)lk_uv[i].x, (double)lk_uv[i].y, cols, rows);
            } else {
                match = true;
                in = m_in[i] != 0;
            }
            in = in && (!mask || mask[i] != 0);
        }
        // matches in the low 16 bits, cur entries in the high 16 bits: a tile holds at most kSetThreads of each
        int pre, tot;
        SetScan(tmp).ExclusiveSum((match ? 1 : 0) | (in ? 1 << 16 : 0), pre, tot);
        __syncthreads();
        if (i < n && match) {
            const int jm = lk_uv ? base_m + (pre & 0xffff) : i;
            double2 vel;
            if (lk_uv) {
                const float2 a = lk_uv[i], b = last_uv[i];
                vel = make_double2(velocity(a.x, b.x, dt), velocity(a.y, b.y, dt));
                m_ids[jm] = last_ids[i]; m_last[jm] = b; m_uv[jm] = a; m_vel[jm] = vel;
                m_in[jm] = in ? 1 : 0;                             // no mask while tracking
            } else {
                vel = m_vel[i];
            }
            if (in) {
                const int jc = base_c + (pre >> 16);
                c_ids[jc] = m_ids[jm]; c_uv[jc] = m_uv[jm]; c_vel[jc] = vel;
            }
        }
        base_m += tot & 0xffff;
        base_c += tot >> 16;
    }
    if (threadIdx.x == 0) { counts[0] = lk_uv ? base_m : n; counts[1] = base_c; }
}

// A list of (id, payload index) pairs sorted by id kept once per id: the last pair of each run (keep_last, init's map
// assignment) or the first (the PnP inliers: equal ids carry equal uv there).  Out of range payload indices (>= n_src or
// negative) count in counts[1] and write nothing useful.  counts[0] = the unique ids.
__global__ void __launch_bounds__(kSetThreads) k_ft_unique(int n, const unsigned* __restrict__ ids_sorted, const int* __restrict__ src_sorted,
                                                           bool keep_last, const float2* __restrict__ uv, const double2* __restrict__ vel,
                                                           int n_src, unsigned* o_ids, float2* o_uv, double2* o_vel, long long* counts) {
    __shared__ typename SetScan::TempStorage tmp;
    int base = 0, bad = 0;
    for (int t0 = 0; t0 < n; t0 += kSetThreads) {
        const int k = t0 + (int)threadIdx.x;
        bool take = false;
        if (k < n) {
            const int s = src_sorted[k];
            if (s < 0 || s >= n_src) ++bad;
            take = keep_last ? (k == n - 1 || ids_sorted[k + 1] != ids_sorted[k]) : (k == 0 || ids_sorted[k - 1] != ids_sorted[k]);
        }
        int pre, tot;
        SetScan(tmp).ExclusiveSum(take ? 1 : 0, pre, tot);
        __syncthreads();
        if (take) {
            const int s = src_sorted[k];
            if (s >= 0 && s < n_src) {
                o_ids[base + pre] = ids_sorted[k];
                o_uv[base + pre] = uv[s];
                if (o_vel) o_vel[base + pre] = vel[s];
            }
        }
        base += tot;
    }
    const int bad_all = __syncthreads_count(bad);
    if (threadIdx.x == 0) { counts[0] = base; counts[1] = bad_all; }
}
__global__ void k_ft_pairs(const unsigned* __restrict__ ids, const int* __restrict__ idx, int n, const unsigned* __restrict__ cur_ids,
                           int n_cur, unsigned* keys, int* vals) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    if (ids) { keys[k] = ids[k]; vals[k] = k; return; }
    const int s = idx[k];                                          // an inlier index into cur
    keys[k] = (s >= 0 && s < n_cur) ? cur_ids[s] : kNoId;
    vals[k] = s;
}

// updateAndAppendTrackPoints, loop 1 (:22-61) over `last` in id order.  The reference's u_d, v_d keep the last values
// project3dTo2d wrote, so an entry whose camera z < 0.001 measures its error against the latest earlier entry that got that
// far (erased ones included): an inclusive max-scan of those entries' indices.  Before any such entry the reference reads
// uninitialised doubles; here the error is NaN there, so the entry is kept with its count reset (DESIGN.md section 5).
// Writes the outlier counts, the survivors (ids, uv), and the sort entries of the kept points whose projection succeeded
// (cell key, rank = index); every other entry gets `none`.  counts[0] = survivors.
__global__ void __launch_bounds__(kSetThreads) k_ft_loop1(int n, const unsigned* __restrict__ ids, const float2* __restrict__ uv, ColorMapView m,
                                                          ColorPoint* cpts, CamConst c, double min_dis, int u0, int v0, int bits_v,
                                                          unsigned long long none, double thr, double2* proj, unsigned* s_ids,
                                                          float2* s_uv, unsigned long long* keys, int* ranks, long long* counts) {
    __shared__ typename SetScan::TempStorage tmp;
    __shared__ int carry;
    if (threadIdx.x == 0) carry = -1;
    int base = 0;
    for (int t0 = 0; t0 < n; t0 += kSetThreads) {
        const int i = t0 + (int)threadIdx.x;
        bool z_ok = false, res = false;
        if (i < n) {
            const float* p = point_xyz(m, ids[i]);
            double u = 0.0, v = 0.0;
            res = project_in_image(c, (double)p[0], (double)p[1], (double)p[2], u, v, &z_ok);
            proj[i] = make_double2(u, v);
        }
        __syncthreads();                                           // proj of the tile (and carry) visible to the block
        int src, tile_max;
        SetScan(tmp).InclusiveScan(z_ok ? i : -1, src, MaxI(), tile_max);
        src = max(src, carry);
        bool keep = false;
        unsigned long long key = none;
        if (i < n) {
            const unsigned id = ids[i];
            double err = CUDART_NAN;
            double ud = 0.0, vd = 0.0;
            if (src >= 0) {
                const double2 q = proj[src];
                ud = q.x; vd = q.y;
                const double a = __dsub_rn(ud, (double)uv[i].x), b = __dsub_rn(vd, (double)uv[i].y);
                err = __dsqrt_rn(__dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b)));   // Eigen::Vector2d::norm
            }
            short cnt = cpts[id].outlier_count;
            keep = true;
            if (err > thr) {
                cnt = (short)(cnt + 1);
                if (cnt > 1 || err > __dmul_rn(thr, 2.0)) { cnt = 0; keep = false; }
            } else {
                cnt = 0;
            }
            cpts[id].outlier_count = cnt;
            if (keep && res) key = cell_key(ud, vd, min_dis, u0, v0, bits_v);
            keys[i] = key;
            ranks[i] = i;
        }
        int pre, tot;
        __syncthreads();
        SetScan(tmp).ExclusiveSum(keep ? 1 : 0, pre, tot);
        if (keep) { s_ids[base + pre] = ids[i]; s_uv[base + pre] = uv[i]; }
        base += tot;
        __syncthreads();
        if (threadIdx.x == 0) carry = max(carry, tile_max);
    }
    if (threadIdx.x == 0) counts[0] = base;
}
// loop 2's candidates (:63-99), j in selection order: a candidate still in `last` is skipped; the others whose projection
// succeeds enter the sort with their cell and rank n_last + j
__global__ void k_ft_candidates(int mcand, const unsigned* __restrict__ cand, ColorMapView m, CamConst c, double min_dis, int u0, int v0,
                                int bits_v, unsigned long long none, const unsigned* __restrict__ s_ids, const long long* counts, int n_last,
                                unsigned char* nonmember, float2* c_uv, unsigned long long* keys, int* ranks) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= mcand) return;
    const unsigned id = cand[j];
    const int ns = (int)counts[0];
    const int pos = lower_bound_u32(s_ids, ns, id);
    const bool member = pos < ns && s_ids[pos] == id;
    unsigned long long key = none;
    if (!member) {
        const float* p = point_xyz(m, id);
        double u, v;
        if (project_in_image(c, (double)p[0], (double)p[1], (double)p[2], u, v)) {
            key = cell_key(u, v, min_dis, u0, v0, bits_v);
            c_uv[j] = make_float2(__double2float_rn(u), __double2float_rn(v));   // cv::Point2f(u_d, v_d)
        }
    }
    nonmember[j] = member ? 0 : 1;
    keys[n_last + j] = key;
    ranks[n_last + j] = n_last + j;
}
// a cell belongs to the first entry of its run in (cell, rank) order: a candidate wins when it heads its run
__global__ void k_ft_winners(int total, const unsigned long long* __restrict__ keys, const int* __restrict__ ranks, int n_last,
                             unsigned long long none, unsigned char* win) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= total) return;
    const unsigned long long key = keys[k];
    if (key == none || (k > 0 && keys[k - 1] == key) || ranks[k] < n_last) return;
    win[ranks[k] - n_last] = 1;
}
// the candidates that enter `last` (:94-97): the first max - size0 winners when size0 < max; otherwise only the first
// non-member, if it wins.  Written in selection order, padded with kNoId up to n_pad; counts[1] = how many.
__global__ void __launch_bounds__(kSetThreads) k_ft_select(int mcand, const unsigned* __restrict__ cand, const unsigned char* __restrict__ win,
                                                           const unsigned char* __restrict__ nonmember, const float2* __restrict__ c_uv,
                                                           int max_points, int n_pad, long long* counts, unsigned* i_ids,
                                                           unsigned long long* i_uv) {
    __shared__ typename SetScan::TempStorage tmp;
    __shared__ int first_nm;
    const int size0 = (int)counts[0];
    if (threadIdx.x == 0) first_nm = INT_MAX;
    __syncthreads();
    int taken = 0;
    if (size0 < max_points) {
        const int quota = max_points - size0;
        for (int t0 = 0; t0 < mcand && taken < quota; t0 += kSetThreads) {
            const int j = t0 + (int)threadIdx.x;
            const bool w = j < mcand && win[j];
            int pre, tot;
            SetScan(tmp).ExclusiveSum(w ? 1 : 0, pre, tot);
            if (w && taken + pre < quota) {
                i_ids[taken + pre] = cand[j];
                i_uv[taken + pre] = reinterpret_cast<const unsigned long long*>(c_uv)[j];
            }
            taken = min(quota, taken + tot);
            __syncthreads();
        }
    } else {
        for (int j = threadIdx.x; j < mcand; j += kSetThreads)
            if (nonmember[j]) atomicMin(&first_nm, j);
        __syncthreads();
        if (first_nm < mcand && win[first_nm]) {
            if (threadIdx.x == 0) { i_ids[0] = cand[first_nm]; i_uv[0] = reinterpret_cast<const unsigned long long*>(c_uv)[first_nm]; }
            taken = 1;
        }
    }
    __syncthreads();
    for (int k = taken + (int)threadIdx.x; k < n_pad; k += kSetThreads) i_ids[k] = kNoId;
    if (threadIdx.x == 0) counts[1] = taken;
}
// new last = survivors and inserted points merged by id (the two are disjoint)
__global__ void k_ft_merge(const unsigned* __restrict__ s_ids, const float2* __restrict__ s_uv, const unsigned* __restrict__ i_ids,
                           const unsigned long long* __restrict__ i_uv, const long long* counts, int n_bound, unsigned* l_ids, float2* l_uv) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    const int ns = (int)counts[0], ni = (int)counts[1];
    if (t < ns) {
        const int p = t + lower_bound_u32(i_ids, ni, s_ids[t]);
        l_ids[p] = s_ids[t]; l_uv[p] = s_uv[t];
    } else if (t - ns < ni && t < n_bound) {
        const int k = t - ns;
        const int p = k + lower_bound_u32(s_ids, ns, i_ids[k]);
        l_ids[p] = i_ids[k]; l_uv[p] = reinterpret_cast<const float2*>(i_uv)[k];
    }
}
__global__ void k_ft_counts(const unsigned* __restrict__ ids, int n, const ColorPoint* __restrict__ cpts, short* out) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n) out[k] = cpts[ids[k]].outlier_count;
}

// room for n elements in a device array that grows by reallocation, keeping its first `keep` elements
template <class T> int grow(srl_ctx* ctx, DevArray<T>& b, size_t n, size_t keep) {
    if (n <= b.size()) return SRL_OK;
    size_t cap = std::max<size_t>(b.size() * 2, 256);
    while (cap < n) cap *= 2;
    DevArray<T> p;
    SRL_CUDA(ctx, p.alloc(cap));
    if (keep) SRL_CUDA(ctx, cudaMemcpyAsync(p, b, keep * sizeof(T), cudaMemcpyDeviceToDevice, ctx->stream));
    b = std::move(p);                                      // cudaFree of the old array waits for the copy
    return SRL_OK;
}

}  // namespace

struct srl_flow_tracker {
    srl_ctx* ctx = nullptr;
    int device = 0;
    srl_color_map* cm = nullptr;
    srl_lk* lk = nullptr;
    int max_points = 300;
    double last_time = 0.0;
    bool have_time = false;
    int64_t n_last = 0, n_match = 0, n_cur = 0;
    DevArray<unsigned> last_ids, m_ids, c_ids, new_ids;
    DevArray<float2> last_uv, m_last, m_uv, c_uv, lk_uv, new_uv;   // new_*: init's set until its Lucas-Kanade call succeeded
    DevArray<double2> m_vel, c_vel;
    DevArray<unsigned char> m_in, lk_status;
    DevArray<long long> d_counts;           // [0, 4)
    PinnedArray<long long> h_counts;        // [0, 4)
};

namespace {
int ft_fail(srl_flow_tracker* t, const char* fn, const char* what) { return set_err(t->ctx, SRL_BAD_ARG, std::string(fn) + ": " + what); }
int read_counts(srl_flow_tracker* t, int k) {
    SRL_CUDA(t->ctx, cudaMemcpyAsync(t->h_counts, t->d_counts, k * sizeof(long long), cudaMemcpyDeviceToHost, t->ctx->stream));
    SRL_CUDA(t->ctx, cudaStreamSynchronize(t->ctx->stream));
    return SRL_OK;
}
// the points of `ids` must be stored points of the colour map (srl_color_map_gather_points checks them and writes nothing)
int check_ids(srl_flow_tracker* t, const uint32_t* ids, size_t n) {
    if (n == 0) return SRL_OK;
    return srl_color_map_gather_points(t->cm, ids, n, nullptr, nullptr, nullptr, nullptr, nullptr);
}
// the match list, cur and the Lucas-Kanade outputs for sets of n points; the match list and cur keep what they hold
int ensure_match_sets(srl_flow_tracker* t, size_t n) {
    int rc;
    const size_t nm = (size_t)t->n_match, nc = (size_t)t->n_cur;
    if ((rc = grow(t->ctx, t->m_ids, n, nm)) != SRL_OK || (rc = grow(t->ctx, t->m_last, n, nm)) != SRL_OK ||
        (rc = grow(t->ctx, t->m_uv, n, nm)) != SRL_OK || (rc = grow(t->ctx, t->m_vel, n, nm)) != SRL_OK ||
        (rc = grow(t->ctx, t->m_in, n, nm)) != SRL_OK || (rc = grow(t->ctx, t->c_ids, n, nc)) != SRL_OK ||
        (rc = grow(t->ctx, t->c_uv, n, nc)) != SRL_OK || (rc = grow(t->ctx, t->c_vel, n, nc)) != SRL_OK ||
        (rc = grow(t->ctx, t->lk_uv, n, 0)) != SRL_OK || (rc = grow(t->ctx, t->lk_status, n, 0)) != SRL_OK)
        return rc;
    return SRL_OK;
}
int ensure_last(srl_flow_tracker* t, size_t n) {
    int rc;
    if ((rc = grow(t->ctx, t->last_ids, n, (size_t)t->n_last)) != SRL_OK || (rc = grow(t->ctx, t->last_uv, n, (size_t)t->n_last)) != SRL_OK)
        return rc;
    return ensure_match_sets(t, n);
}
// Lucas-Kanade over n points' uv into lk_uv / lk_status
int run_lk(srl_flow_tracker* t, const uint8_t* gray, int cols, int rows, size_t pitch, const float2* uv, int64_t n, int64_t* n_tracked) {
    return srl_lk_track_image(t->lk, gray, cols, rows, pitch, reinterpret_cast<const float*>(uv), (size_t)n,
                              reinterpret_cast<float*>(t->lk_uv.get()), t->lk_status, n_tracked);
}
}  // namespace

extern "C" {

int srl_flow_tracker_create(srl_ctx* ctx, srl_color_map* cm, srl_lk* lk, int32_t maximum_tracked_points, srl_flow_tracker** out) {
    if (!ctx || !out) return SRL_BAD_ARG;
    *out = nullptr;
    if (!cm || !lk) return set_err(ctx, SRL_BAD_ARG, "srl_flow_tracker_create: a colour map and a Lucas-Kanade tracker are required");
    if (color_map_ctx(cm) != ctx || lk_ctx(lk) != ctx)
        return set_err(ctx, SRL_BAD_ARG, "srl_flow_tracker_create: the colour map and the Lucas-Kanade tracker must use this ctx");
    if (maximum_tracked_points < 1) return set_err(ctx, SRL_BAD_ARG, "srl_flow_tracker_create: maximum_tracked_points must be >= 1");
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    std::unique_ptr<srl_flow_tracker> t(new srl_flow_tracker());
    t->ctx = ctx; t->device = ctx->device; t->cm = cm; t->lk = lk; t->max_points = maximum_tracked_points;
    cudaError_t e = t->d_counts.alloc(4);
    if (e == cudaSuccess) e = t->h_counts.alloc(4);
    if (e != cudaSuccess) return cuda_fail(ctx, e, "srl_flow_tracker_create");
    *out = t.release();
    return SRL_OK;
}

void srl_flow_tracker_destroy(srl_flow_tracker* t) {
    if (!t) return;
    cudaSetDevice(t->device);
    delete t;
}

int srl_flow_tracker_init(srl_flow_tracker* t, const uint8_t* gray, int cols, int rows, size_t pitch, double image_time,
                          const uint32_t* ids, const float* uv, size_t n) {
    static const char* fn = "srl_flow_tracker_init";
    if (!t) return SRL_BAD_ARG;
    srl_ctx* ctx = t->ctx;
    if (n && (!ids || !uv)) return ft_fail(t, fn, "ids and uv are required");
    if (n > 0x7fffffff) return ft_fail(t, fn, "at most 2^31 - 1 points");
    if (!gray) return ft_fail(t, fn, "the image is required");
    int rc = check_ids(t, ids, n);
    if (rc != SRL_OK) return rc;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    // the new set is built aside and replaces last only once the Lucas-Kanade call has accepted the image
    if ((rc = grow(ctx, t->new_ids, n, 0)) != SRL_OK || (rc = grow(ctx, t->new_uv, n, 0)) != SRL_OK || (rc = ensure_match_sets(t, n)) != SRL_OK)
        return rc;
    int64_t n_new = 0;
    if (n) {
        const int nn = (int)n;
        size_t tmp_sort = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, tmp_sort, (unsigned*)nullptr, (unsigned*)nullptr, (int*)nullptr, (int*)nullptr, nn, 0, 32, st);
        Staged<const unsigned> s_ids(ids);
        Staged<const float> s_uv(uv);
        unsigned *keys_a = nullptr, *keys_b = nullptr;
        int *vals_a = nullptr, *vals_b = nullptr;
        void* d_tmp = nullptr;
        rc = carve_scratch(ctx, [&](Carve& c) {
            s_ids.place(c, n); s_uv.place(c, 2 * n);
            keys_a = c.take<unsigned>(n); keys_b = c.take<unsigned>(n); vals_a = c.take<int>(n); vals_b = c.take<int>(n);
            d_tmp = c.take<char>(tmp_sort);
        });
        if (rc != SRL_OK || (rc = s_ids.upload(ctx, n)) != SRL_OK || (rc = s_uv.upload(ctx, 2 * n)) != SRL_OK) return rc;
        const unsigned gb = (unsigned)((n + 255) / 256);
        k_ft_pairs<<<gb, 256, 0, st>>>(s_ids.d, nullptr, nn, nullptr, 0, keys_a, vals_a);
        SRL_CUDA(ctx, cudaGetLastError());
        SRL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(d_tmp, tmp_sort, keys_a, keys_b, vals_a, vals_b, nn, 0, 32, st));   // stable
        // setTrackPoints (:205-208): map[id] = uv in input order, so a later duplicate overwrites an earlier one
        k_ft_unique<<<1, kSetThreads, 0, st>>>(nn, keys_b, vals_b, true, reinterpret_cast<const float2*>(s_uv.d), nullptr, nn,
                                               t->new_ids, t->new_uv, nullptr, t->d_counts);
        SRL_CUDA(ctx, cudaGetLastError());
        ctx->launches += 3;
        if ((rc = read_counts(t, 1)) != SRL_OK) return rc;
        n_new = t->h_counts[0];
    }
    int64_t k = 0;
    if ((rc = run_lk(t, gray, cols, rows, pitch, t->new_uv, n_new, &k)) != SRL_OK) return rc;   // :196: on the first image, the pyramid only
    std::swap(t->last_ids, t->new_ids);
    std::swap(t->last_uv, t->new_uv);
    t->n_last = n_new;
    t->last_time = image_time;                                     // init (:192-193)
    t->have_time = true;
    return SRL_OK;
}

int srl_flow_tracker_track_image(srl_flow_tracker* t, const uint8_t* gray, int cols, int rows, size_t pitch, double image_time,
                                 int32_t* lk_called) {
    static const char* fn = "srl_flow_tracker_track_image";
    if (!t) return SRL_BAD_ARG;
    srl_ctx* ctx = t->ctx;
    if (lk_called) *lk_called = 0;
    if (!gray) return ft_fail(t, fn, "the image is required");
    if (!t->have_time) return ft_fail(t, fn, "init has not been called");
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    t->n_cur = 0;                                                  // :115
    t->n_match = 0;
    const double dt = image_time - t->last_time;                   // :153, against the time before this call
    if (t->n_last < 30) {                                          // :128-132: no Lucas-Kanade, the pyramid is not consumed
        t->last_time = image_time;
        return SRL_OK;
    }
    int64_t tracked = 0;
    int rc = run_lk(t, gray, cols, rows, pitch, t->last_uv, t->n_last, &tracked);
    if (rc != SRL_OK) return rc;
    if (lk_called) *lk_called = 1;
    k_ft_track<<<1, kSetThreads, 0, ctx->stream>>>((int)t->n_last, t->last_ids, t->last_uv, t->lk_uv, t->lk_status, dt, cols, rows,
                                                   t->m_ids, t->m_last, t->m_uv, t->m_vel, t->m_in, nullptr, t->c_ids, t->c_uv,
                                                   t->c_vel, t->d_counts);
    SRL_CUDA(ctx, cudaGetLastError());
    ctx->launches += 1;
    if ((rc = read_counts(t, 2)) != SRL_OK) return rc;
    t->n_match = t->h_counts[0];
    t->n_cur = t->h_counts[1];
    t->last_time = image_time;                                     // :185; `last` itself is not changed (:179-182)
    return SRL_OK;
}

int srl_flow_tracker_reject_matches(srl_flow_tracker* t, const uint8_t* mask, size_t n) {
    static const char* fn = "srl_flow_tracker_reject_matches";
    if (!t) return SRL_BAD_ARG;
    srl_ctx* ctx = t->ctx;
    if (mask && n != (size_t)t->n_match) return ft_fail(t, fn, "the mask must have one byte per match");
    if (t->n_match == 0) return SRL_OK;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    Staged<const unsigned char> s_mask(mask);
    int rc = carve_scratch(ctx, [&](Carve& c) { s_mask.place(c, n); });
    if (rc != SRL_OK || (rc = s_mask.upload(ctx, mask ? n : 0)) != SRL_OK) return rc;
    k_ft_track<<<1, kSetThreads, 0, ctx->stream>>>((int)t->n_match, nullptr, nullptr, nullptr, nullptr, 0.0, 0, 0, t->m_ids, t->m_last,
                                                   t->m_uv, t->m_vel, t->m_in, s_mask.d, t->c_ids, t->c_uv, t->c_vel,
                                                   t->d_counts);
    SRL_CUDA(ctx, cudaGetLastError());
    ctx->launches += 1;
    if ((rc = read_counts(t, 2)) != SRL_OK) return rc;
    t->n_cur = t->h_counts[1];
    return SRL_OK;
}

int srl_flow_tracker_remove_outliers(srl_flow_tracker* t, const int32_t* inliers, size_t n, int32_t* result) {
    static const char* fn = "srl_flow_tracker_remove_outliers";
    if (!t || !result) return SRL_BAD_ARG;
    srl_ctx* ctx = t->ctx;
    *result = 0;
    if (n > 0x7fffffff) return ft_fail(t, fn, "at most 2^31 - 1 inliers");
    if (t->n_cur < 10) return SRL_OK;                              // :286-289
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    const size_t nc = (size_t)t->n_cur;
    if (!inliers) {                                                // every entry of cur is an inlier: last = cur
        int rc = ensure_last(t, nc);
        if (rc != SRL_OK) return rc;
        SRL_CUDA(ctx, cudaMemcpyAsync(t->last_ids, t->c_ids, nc * sizeof(unsigned), cudaMemcpyDeviceToDevice, st));
        SRL_CUDA(ctx, cudaMemcpyAsync(t->last_uv, t->c_uv, nc * sizeof(float2), cudaMemcpyDeviceToDevice, st));
        SRL_CUDA(ctx, cudaStreamSynchronize(st));
        t->n_last = t->n_cur;
        *result = 1;
        return SRL_OK;
    }
    const int nn = (int)n;
    size_t tmp_sort = 0;
    if (n) cub::DeviceRadixSort::SortPairs(nullptr, tmp_sort, (unsigned*)nullptr, (unsigned*)nullptr, (int*)nullptr, (int*)nullptr, nn, 0, 32, st);
    Staged<const int> s_in(inliers);
    unsigned *keys_a = nullptr, *keys_b = nullptr, *o_ids = nullptr;
    int *vals_a = nullptr, *vals_b = nullptr;
    float2* o_uv = nullptr;
    double2* o_vel = nullptr;
    void* d_tmp = nullptr;
    int rc = carve_scratch(ctx, [&](Carve& c) {
        s_in.place(c, n);
        keys_a = c.take<unsigned>(n); keys_b = c.take<unsigned>(n); vals_a = c.take<int>(n); vals_b = c.take<int>(n);
        o_ids = c.take<unsigned>(n); o_uv = c.take<float2>(n); o_vel = c.take<double2>(n);
        d_tmp = c.take<char>(tmp_sort);
    });
    if (rc != SRL_OK || (rc = s_in.upload(ctx, n)) != SRL_OK) return rc;
    long long uniq = 0;
    if (n) {
        k_ft_pairs<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(nullptr, reinterpret_cast<const int*>(s_in.d), nn, t->c_ids, (int)nc, keys_a, vals_a);
        SRL_CUDA(ctx, cudaGetLastError());
        SRL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(d_tmp, tmp_sort, keys_a, keys_b, vals_a, vals_b, nn, 0, 32, st));
        // :310-317: both maps take the inliers with their current uv; std::map sorts them and drops repeats
        k_ft_unique<<<1, kSetThreads, 0, st>>>(nn, keys_b, vals_b, false, t->c_uv, t->c_vel, (int)nc, o_ids, o_uv, o_vel, t->d_counts);
        SRL_CUDA(ctx, cudaGetLastError());
        ctx->launches += 3;
        if ((rc = read_counts(t, 2)) != SRL_OK) return rc;
        if (t->h_counts[1]) return ft_fail(t, fn, "an inlier index lies outside [0, number of current points)");
        uniq = t->h_counts[0];
    }
    if ((rc = ensure_last(t, (size_t)uniq)) != SRL_OK) return rc;
    if (uniq) {
        const size_t u = (size_t)uniq;
        SRL_CUDA(ctx, cudaMemcpyAsync(t->last_ids, o_ids, u * sizeof(unsigned), cudaMemcpyDeviceToDevice, st));
        SRL_CUDA(ctx, cudaMemcpyAsync(t->last_uv, o_uv, u * sizeof(float2), cudaMemcpyDeviceToDevice, st));
        SRL_CUDA(ctx, cudaMemcpyAsync(t->c_ids, o_ids, u * sizeof(unsigned), cudaMemcpyDeviceToDevice, st));
        SRL_CUDA(ctx, cudaMemcpyAsync(t->c_uv, o_uv, u * sizeof(float2), cudaMemcpyDeviceToDevice, st));
        SRL_CUDA(ctx, cudaMemcpyAsync(t->c_vel, o_vel, u * sizeof(double2), cudaMemcpyDeviceToDevice, st));
        SRL_CUDA(ctx, cudaStreamSynchronize(st));
    }
    t->n_last = t->n_cur = uniq;
    *result = 1;
    return SRL_OK;
}

int srl_flow_tracker_update_and_append(srl_flow_tracker* t, const srl_camera* cam, double mini_distance, const uint32_t* candidates,
                                       size_t n_candidates) {
    static const char* fn = "srl_flow_tracker_update_and_append";
    if (!t) return SRL_BAD_ARG;
    srl_ctx* ctx = t->ctx;
    if (!cam) return ft_fail(t, fn, "the camera is required");
    if (n_candidates && !candidates) return ft_fail(t, fn, "candidates is NULL");
    if (n_candidates > 0x3fffffff) return ft_fail(t, fn, "at most 2^30 - 1 candidates");
    if (cam->cols < 2 || cam->rows < 2) return ft_fail(t, fn, "the image needs cols >= 2 and rows >= 2");
    if (!(std::isfinite(mini_distance) && mini_distance > 0)) return ft_fail(t, fn, "mini_distance must be finite and > 0");
    int u0 = 0, v0 = 0, bits_u = 0, bits_v = 0;
    if (!std::isfinite(cam->fov_margin) || !cell_axis(cam->fov_margin, cam->cols, mini_distance, u0, bits_u) ||
        !cell_axis(cam->fov_margin, cam->rows, mini_distance, v0, bits_v))
        return ft_fail(t, fn, "the cell coordinates of the FoV window do not fit an int");
    int rc = check_ids(t, candidates, n_candidates);
    if (rc != SRL_OK) return rc;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    const int end_bit = bits_u + bits_v;
    const unsigned long long none = end_bit >= 64 ? ~0ull : (1ull << end_bit) - 1ull;
    const int nl = (int)t->n_last, mc = (int)n_candidates;
    const int total = nl + mc;
    // at most max(max - size0, 1) <= max candidates enter, so the new set holds at most max(n_last + 1, max) points
    const int n_ins = std::min(mc, t->max_points);
    if ((rc = ensure_last(t, std::max<size_t>((size_t)nl + 1, (size_t)t->max_points))) != SRL_OK) return rc;
    size_t tmp_a = 0, tmp_b = 0;
    if (total) cub::DeviceRadixSort::SortPairs(nullptr, tmp_a, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int*)nullptr,
                                               (int*)nullptr, total, 0, std::max(end_bit, 1), st);
    if (n_ins) cub::DeviceRadixSort::SortPairs(nullptr, tmp_b, (unsigned*)nullptr, (unsigned*)nullptr, (unsigned long long*)nullptr,
                                               (unsigned long long*)nullptr, n_ins, 0, 32, st);
    Staged<const unsigned> s_cand(candidates);
    double2* proj = nullptr;
    unsigned *s_ids = nullptr, *i_ids = nullptr, *i_ids_b = nullptr;
    float2 *s_uv = nullptr, *c_uv = nullptr;
    unsigned long long *keys_a = nullptr, *keys_b = nullptr, *i_uv = nullptr, *i_uv_b = nullptr;
    int *ranks_a = nullptr, *ranks_b = nullptr;
    unsigned char *nonmember = nullptr, *win = nullptr;
    void* d_tmp = nullptr;
    const size_t L = (size_t)nl, M = (size_t)mc, T = (size_t)total, I = (size_t)n_ins;
    rc = carve_scratch(ctx, [&](Carve& c) {
        s_cand.place(c, M);
        proj = c.take<double2>(L); s_ids = c.take<unsigned>(L); s_uv = c.take<float2>(L);
        keys_a = c.take<unsigned long long>(T); keys_b = c.take<unsigned long long>(T); ranks_a = c.take<int>(T); ranks_b = c.take<int>(T);
        nonmember = c.take<unsigned char>(M); win = c.take<unsigned char>(M); c_uv = c.take<float2>(M);
        i_ids = c.take<unsigned>(I); i_ids_b = c.take<unsigned>(I); i_uv = c.take<unsigned long long>(I); i_uv_b = c.take<unsigned long long>(I);
        d_tmp = c.take<char>(std::max(tmp_a, tmp_b));
    });
    if (rc != SRL_OK || (rc = s_cand.upload(ctx, M)) != SRL_OK) return rc;
    const CamConst cc = camera_constants(cam);
    const ColorMapView mv = color_map_view(t->cm);
    const double thr = 2.0 * (double)cam->cols / 320.0;            // :18
    SRL_CUDA(ctx, cudaMemsetAsync(t->d_counts, 0, 2 * sizeof(long long), st));
    k_ft_loop1<<<1, kSetThreads, 0, st>>>(nl, t->last_ids, t->last_uv, mv, color_map_states(t->cm), cc, mini_distance, u0, v0, bits_v,
                                          none, thr, proj, s_ids, s_uv, keys_a, ranks_a, t->d_counts);
    SRL_CUDA(ctx, cudaGetLastError());
    int launches = 1;
    if (mc) {
        SRL_CUDA(ctx, cudaMemsetAsync(win, 0, M, st));
        const unsigned gm = (unsigned)((mc + 255) / 256), gt = (unsigned)((total + 255) / 256);
        k_ft_candidates<<<gm, 256, 0, st>>>(mc, s_cand.d, mv, cc, mini_distance, u0, v0, bits_v, none, s_ids, t->d_counts, nl, nonmember, c_uv,
                                            keys_a, ranks_a);
        SRL_CUDA(ctx, cudaGetLastError());
        size_t tb = tmp_a;
        SRL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(d_tmp, tb, keys_a, keys_b, ranks_a, ranks_b, total, 0, std::max(end_bit, 1), st));   // stable
        k_ft_winners<<<gt, 256, 0, st>>>(total, keys_b, ranks_b, nl, none, win);
        SRL_CUDA(ctx, cudaGetLastError());
        k_ft_select<<<1, kSetThreads, 0, st>>>(mc, s_cand.d, win, nonmember, c_uv, t->max_points, n_ins, t->d_counts, i_ids, i_uv);
        SRL_CUDA(ctx, cudaGetLastError());
        tb = tmp_b;
        SRL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(d_tmp, tb, i_ids, i_ids_b, i_uv, i_uv_b, n_ins, 0, 32, st));   // padding sorts last
        launches += 5;
    }
    const int bound = nl + n_ins;
    if (bound) {
        k_ft_merge<<<(unsigned)((bound + 255) / 256), 256, 0, st>>>(s_ids, s_uv, mc ? i_ids_b : nullptr, mc ? i_uv_b : nullptr, t->d_counts,
                                                                    bound, t->last_ids, t->last_uv);
        SRL_CUDA(ctx, cudaGetLastError());
        ++launches;
    }
    ctx->launches += launches;
    if ((rc = read_counts(t, 2)) != SRL_OK) return rc;
    t->n_last = t->h_counts[0] + t->h_counts[1];
    return SRL_OK;
}

int srl_flow_tracker_sets(srl_flow_tracker* t, srl_flow_tracker_sets_out* out) {
    if (!t || !out) return SRL_BAD_ARG;
    out->n_match = t->n_match; out->n_cur = t->n_cur; out->n_last = t->n_last;
    out->match_ids = t->m_ids;
    out->match_last_uv = reinterpret_cast<const float*>(t->m_last.get());
    out->match_uv = reinterpret_cast<const float*>(t->m_uv.get());
    out->cur_ids = t->c_ids;
    out->cur_uv = reinterpret_cast<const float*>(t->c_uv.get());
    out->cur_velocity = reinterpret_cast<const double*>(t->c_vel.get());
    out->last_ids = t->last_ids;
    out->last_uv = reinterpret_cast<const float*>(t->last_uv.get());
    out->last_image_time = t->last_time;
    return SRL_OK;
}

int srl_flow_tracker_outlier_counts(srl_flow_tracker* t, const uint32_t* ids, size_t n, int16_t* counts) {
    static const char* fn = "srl_flow_tracker_outlier_counts";
    if (!t) return SRL_BAD_ARG;
    srl_ctx* ctx = t->ctx;
    if (n && (!ids || !counts)) return ft_fail(t, fn, "ids and counts are required");
    if (n > 0x7fffffff) return ft_fail(t, fn, "at most 2^31 - 1 ids");
    if (n == 0) return SRL_OK;
    int rc = check_ids(t, ids, n);
    if (rc != SRL_OK) return rc;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    Staged<const unsigned> s_ids(ids);
    Staged<short> s_out(counts);
    rc = carve_scratch(ctx, [&](Carve& c) { s_ids.place(c, n); s_out.place(c, n); });
    if (rc != SRL_OK || (rc = s_ids.upload(ctx, n)) != SRL_OK) return rc;
    k_ft_counts<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(s_ids.d, (int)n, color_map_states(t->cm), s_out.d);
    SRL_CUDA(ctx, cudaGetLastError());
    ctx->launches += 1;
    if ((rc = s_out.hand_back(ctx, n)) != SRL_OK) return rc;
    SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return SRL_OK;
}

}  // extern "C"
