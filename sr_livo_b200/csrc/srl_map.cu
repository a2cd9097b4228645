// srl_map.cu — HBM-resident voxel map: bulk mirror (K4) and order-preserving insertion (K3).
//
// K3 replaces lioOptimization::addPointsToMap / addPointToMap (src/lioOptimization.cpp:400-446,520-554):
// the reference inserts the registered frame point by point, and a point's acceptance depends on the points
// already accepted into its voxel (including earlier points of the same sweep).  Voxels are independent of each
// other, so the GPU version is: float-round + key per point -> stable radix sort by key (keeps sweep order inside
// a voxel) -> one warp per touched voxel replays the reference's sequential rule over that voxel's points.
// Resulting block contents (points and their order) are identical to the reference's voxelBlock::points.
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <limits>
#include <mutex>
#include <tr1/unordered_map>

#include "srl_internal.h"

namespace srl {

constexpr unsigned long long kInvalidKey = 1ull << 49;

__device__ __forceinline__ int slot_find_rw(const Slot* slots, unsigned int mask, unsigned long long key, int x, int y, int z) {
    unsigned int idx = hash_key(x, y, z) & mask;
    for (;;) {
        const unsigned long long k = slots[idx].key;
        if (k == key) return (int)idx;
        if (k == 0ull) return -1;
        idx = (idx + 1) & mask;
    }
}

__device__ __forceinline__ int slot_claim(Slot* slots, unsigned int mask, unsigned long long key, int x, int y, int z,
                                          unsigned int block, unsigned int count) {
    unsigned int idx = hash_key(x, y, z) & mask;
    for (;;) {
        const unsigned long long old = atomicCAS(&slots[idx].key, 0ull, key);
        if (old == 0ull) { slots[idx].block = block; slots[idx].count = count; return (int)idx; }
        if (old == key) return -1;   // duplicate key (caller guarantees uniqueness)
        idx = (idx + 1) & mask;
    }
}

// a slot table (voxel map or fine-cell set) moved into a larger one: one thread per old slot, key / block / count unchanged
__global__ void k_rehash(const Slot* __restrict__ old_slots, long long n_old, Slot* slots, unsigned int mask) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_old) return;
    const Slot s = old_slots[i];
    if (s.key == 0ull) return;
    short x, y, z;
    unpack_key(s.key, x, y, z);
    slot_claim(slots, mask, s.key, x, y, z, s.block, s.count);
}

// ---- K4: bulk mirror of a host voxelHashMap ---------------------------------------------------------------
__global__ void k_upload_slots(Slot* slots, unsigned int mask, float* blocks, const short* keys, const int* counts,
                               long long n_voxels, int* dup_flag) {
    const long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= n_voxels) return;
    const int x = keys[3 * v], y = keys[3 * v + 1], z = keys[3 * v + 2];
    const unsigned long long key = pack_key(x, y, z);
    if (slot_claim(slots, mask, key, x, y, z, (unsigned)v, (unsigned)counts[v]) < 0) *dup_flag = 1;
    unsigned int* meta = reinterpret_cast<unsigned int*>(blocks + (size_t)v * kBlockFloats);
    meta[kMetaKeyLo] = (unsigned int)(key & 0xffffffffu); meta[kMetaKeyHi] = (unsigned int)(key >> 32); meta[kMetaCount] = (unsigned)counts[v];
}
__global__ void k_upload_points(float* blocks, const float* xyz, long long n_voxels, int cap) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_voxels * cap) return;
    const long long v = e / cap;
    const int i = (int)(e % cap);
    float* b = blocks + (size_t)v * kBlockFloats + 4 * i;
    b[0] = xyz[3 * e]; b[1] = xyz[3 * e + 1]; b[2] = xyz[3 * e + 2];
}
__global__ void k_download(const float* blocks, int block_pts, long long n_voxels, int cap, short* keys, int* counts, float* xyz) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_voxels * cap) return;
    const long long v = e / cap;
    const int i = (int)(e % cap);
    const float* b = blocks + (size_t)v * (4 * block_pts);
    const unsigned int* meta = reinterpret_cast<const unsigned int*>(b);
    const int cnt = (int)meta[kMetaCount];
    if (i == 0) {
        short x, y, z;
        unpack_key((unsigned long long)meta[kMetaKeyLo] | ((unsigned long long)meta[kMetaKeyHi] << 32), x, y, z);
        keys[3 * v] = x; keys[3 * v + 1] = y; keys[3 * v + 2] = z;
        counts[v] = cnt;
    }
    xyz[3 * e] = i < cnt ? b[4 * i] : 0.f;
    xyz[3 * e + 1] = i < cnt ? b[4 * i + 1] : 0.f;
    xyz[3 * e + 2] = i < cnt ? b[4 * i + 2] : 0.f;
}

// ---- K3: insertion ------------------------------------------------------------------------------------------
// rgbPoint ctor: position = position_.cast<float>() (src/cloudMap.cpp:5-9); key from the float-rounded position
// (src/lioOptimization.cpp:403-405).  The key is static_cast<short>(q) as the reference is compiled for x86-64, the colour
// map's rule (k_color_keys): truncation to int32, then the low 16 bits, so voxels 65536 apart share a key.  NaN, +-inf
// and |q| >= 2^31 drop the point.
__global__ void k_insert_keys(const double* __restrict__ xyz, long long n, double size, unsigned long long* keys,
                              unsigned int* idx, float* fxyz) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float fx = __double2float_rn(xyz[3 * i]), fy = __double2float_rn(xyz[3 * i + 1]), fz = __double2float_rn(xyz[3 * i + 2]);
    fxyz[3 * i] = fx; fxyz[3 * i + 1] = fy; fxyz[3 * i + 2] = fz;
    const double qx = __ddiv_rn((double)fx, size), qy = __ddiv_rn((double)fy, size), qz = __ddiv_rn((double)fz, size);
    constexpr double kI32 = 2147483648.0;
    unsigned long long key = kInvalidKey;
    if (fabs(qx) < kI32 && fabs(qy) < kI32 && fabs(qz) < kI32) key = pack_key((int)qx, (int)qy, (int)qz);
    keys[i] = key;
    idx[i] = (unsigned int)i;
}

__global__ void k_seg_flags(const unsigned long long* __restrict__ keys, long long n, unsigned char* flags) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const unsigned long long k = keys[j];
    flags[j] = (k != kInvalidKey && (j == 0 || keys[j - 1] != k)) ? 1 : 0;
}

__global__ void k_seg_lookup(const Slot* slots, unsigned int mask, const unsigned long long* __restrict__ keys,
                             const unsigned int* __restrict__ seg_start, const int* n_seg_p, int allow_new,
                             int* seg_slot, unsigned int* is_new) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= *n_seg_p) return;
    const unsigned long long key = keys[seg_start[s]];
    short x, y, z;
    unpack_key(key, x, y, z);
    const int slot = slot_find_rw(slots, mask, key, x, y, z);
    seg_slot[s] = slot;
    is_new[s] = (slot < 0 && allow_new) ? 1u : 0u;
}

// a new voxel of segment s takes the next free block: slot claimed, key and count 0 written into the block's metadata
__device__ __forceinline__ void seg_claim(Slot* slots, unsigned int mask, float* blocks, size_t block_floats, const unsigned long long* __restrict__ keys,
                                          const unsigned int* __restrict__ seg_start, const int* n_seg_p,
                                          const unsigned int* __restrict__ is_new, const unsigned int* __restrict__ new_rank,
                                          long long block_base, int* seg_slot) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= *n_seg_p || !is_new[s]) return;
    const unsigned long long key = keys[seg_start[s]];
    short x, y, z;
    unpack_key(key, x, y, z);
    const unsigned int blk = (unsigned int)(block_base + new_rank[s]);
    seg_slot[s] = slot_claim(slots, mask, key, x, y, z, blk, 0u);
    unsigned int* meta = reinterpret_cast<unsigned int*>(blocks + (size_t)blk * block_floats);
    meta[kMetaKeyLo] = (unsigned int)(key & 0xffffffffu); meta[kMetaKeyHi] = (unsigned int)(key >> 32); meta[kMetaCount] = 0;
}
__global__ void k_seg_claim(Slot* slots, unsigned int mask, float* blocks, const unsigned long long* __restrict__ keys,
                            const unsigned int* __restrict__ seg_start, const int* n_seg_p,
                            const unsigned int* __restrict__ is_new, const unsigned int* __restrict__ new_rank,
                            long long block_base, int* seg_slot) {
    seg_claim(slots, mask, blocks, kBlockFloats, keys, seg_start, n_seg_p, is_new, new_rank, block_base, seg_slot);
}

// one warp per touched voxel: the reference's per-point rule, replayed in sweep order.
// pub (nullable, one byte per sweep point, zeroed by the caller): set for a point appended to a voxel that map.find found,
// i.e. one that was in the slot table before this call or was created by an earlier point of the sweep; those are the points
// addPointToPcl puts into the published cloud (:432).  A point that creates its voxel (:437-444) is stored but not published.
__global__ void __launch_bounds__(256) k_seg_process(Slot* slots, float* blocks, const unsigned long long* __restrict__ keys,
                                                      const unsigned int* __restrict__ idx, const float* __restrict__ fxyz,
                                                      const unsigned int* __restrict__ seg_start, const int* n_seg_p,
                                                      const int* __restrict__ seg_slot, long long n, double size, int cap,
                                                      double min_dist, int min_num_points, long long* n_points,
                                                      const unsigned int* __restrict__ is_new, unsigned char* pub) {
    const int lane = threadIdx.x & 31;
    const int s = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    if (s >= *n_seg_p) return;
    const int slot = seg_slot[s];
    if (slot < 0) return;   // voxel absent and min_num_points > 0: nothing is ever created (:437)
    bool found = pub ? !is_new[s] : false;
    const unsigned int blk = slots[slot].block;
    int count = (int)slots[slot].count;
    float* bp = blocks + (size_t)blk * kBlockFloats;
    float ex = 0.f, ey = 0.f, ez = 0.f;
    if (lane < count) { ex = bp[4 * lane]; ey = bp[4 * lane + 1]; ez = bp[4 * lane + 2]; }
    const long long start = seg_start[s];
    const unsigned long long key = keys[start];
    const double sq_init = 10 * size * size;            // :413
    const double min_sq = min_dist * min_dist;          // :427
    int added = 0;
    for (long long j = start; j < n; ++j) {
        if (keys[j] != key) break;
        if (count >= cap) break;                        // IsFull(): nothing more is ever added (:411)
        const unsigned int i = idx[j];
        const float fx = fxyz[3 * (size_t)i], fy = fxyz[3 * (size_t)i + 1], fz = fxyz[3 * (size_t)i + 2];
        bool add;
        if (is_new[s] && count == 0) {
            add = (min_num_points <= 0);                // absent voxel: created with the point (:437-445)
        } else {                                        // found voxel, an uploaded empty one included: no lane holds a point
                                                        // then, so sq_min = 10 size^2 (:413-427)
            double sq = CUDART_INF;
            if (lane < count) {
                const double dx = __dsub_rn((double)ex, (double)fx), dy = __dsub_rn((double)ey, (double)fy), dz = __dsub_rn((double)ez, (double)fz);
                sq = __dadd_rn(__dmul_rn(dx, dx), __dadd_rn(__dmul_rn(dy, dy), __dmul_rn(dz, dz)));
            }
#pragma unroll
            for (int o = 16; o >= 1; o >>= 1) sq = fmin(sq, __shfl_xor_sync(0xffffffffu, sq, o));
            const double sq_min = fmin(sq_init, sq);
            add = (sq_min > min_sq) && (min_num_points <= 0 || count >= min_num_points);   // :427-433
        }
        if (add) {
            if (lane == count) { ex = fx; ey = fy; ez = fz; bp[4 * count] = fx; bp[4 * count + 1] = fy; bp[4 * count + 2] = fz; }
            if (pub) {
                if (found && lane == 0) pub[i] = 1;
                found = true;
            }
            ++count; ++added;
        }
    }
    if (lane == 0 && added) {
        slots[slot].count = (unsigned int)count;
        reinterpret_cast<unsigned int*>(bp)[kMetaCount] = (unsigned int)count;
        atomicAdd(reinterpret_cast<unsigned long long*>(n_points), (unsigned long long)added);
    }
}

// ---- N2: gridSampling / subSampleFrame (src/utility.cpp:167-201) ----------------------------------------------------
// cell key from the DOUBLE coordinate (src/utility.cpp:171-173: static_cast<short>(frame[i].point[k] / size_voxel))
__global__ void k_cell_keys(const double* __restrict__ xyz, long long n, double size, unsigned long long* keys, unsigned int* idx) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double qx = __ddiv_rn(xyz[3 * i], size), qy = __ddiv_rn(xyz[3 * i + 1], size), qz = __ddiv_rn(xyz[3 * i + 2], size);
    unsigned long long key = kInvalidKey;
    if (fabs(qx) < 32765.0 && fabs(qy) < 32765.0 && fabs(qz) < 32765.0) key = pack_key((int)qx, (int)qy, (int)qz);
    keys[i] = key;
    idx[i] = (unsigned int)i;
}
// after the stable sort by cell: the head of each run is the cell's first point in frame order; flag it at its own index
__global__ void k_first_in_cell(const unsigned long long* __restrict__ keys_sorted, const unsigned int* __restrict__ idx_sorted,
                                long long n, unsigned char* is_first) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const unsigned long long k = keys_sorted[j];
    is_first[idx_sorted[j]] = (k != kInvalidKey && (j == 0 || keys_sorted[j - 1] != k)) ? 1 : 0;
}

// ---- N4: colour map (src/lioOptimization.cpp:448-551 colour branch; src/rgbMapTracker.cpp:181-237; src/cloudMap.cpp:59-101) ----
// The colour map is a second voxel map (same slot table / block pool) whose points carry a colour estimate, plus
//   * a fine occupancy set (cells of min_distance_points, the reference's Hash_map_3d hashmap_3d_points) that decides
//     which stored points also enter rgb_points_vec, and
//   * the list of voxels the last rendering sweep visited first (voxels_recent_visited), which the renderer walks.
// addPointToColorMap is sequential in the reference; the same (sort by voxel, replay per voxel in sweep order) scheme as K3
// reproduces it: a voxel accepts the first (cap - count) offered points, a fine cell is claimed by the first ACCEPTED
// point of the sweep that falls into it, and both lists are emitted in sweep order.
constexpr unsigned kNoIndex = 0xffffffffu;
constexpr int kColorMaxCap = 128;   // largest max_num_points_in_voxel of a colour map (the shipped configs use 20, 50 and 100)

// selected points (every step-th of the frame): voxel key + fine key from the float-rounded position (getPosition()).
// Both keys are static_cast<short>(q) as the reference is compiled for x86-64: truncation to int32 (cvttsd2si), then the low
// 16 bits, so a key wraps past |q| = 32767 (0.01 m fine cells: |x| >= 327.68 m) and cells 655.36 m apart share a key.
// pack_key keeps those 16 bits, so a wrapped key is an ordinary key: valid bit 48 set, never 0 (empty slot) or kInvalidKey.
// NaN, +-inf and |q| >= 2^31 (where the int32 conversion itself is undefined) drop the point.
__global__ void k_color_keys(const double* __restrict__ xyz, long long m, int step, double size, double fine, unsigned long long* vkeys,
                             unsigned long long* fkeys, unsigned int* idx, float* fxyz) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const long long i = j * step;
    const float fx = __double2float_rn(xyz[3 * i]), fy = __double2float_rn(xyz[3 * i + 1]), fz = __double2float_rn(xyz[3 * i + 2]);
    fxyz[3 * j] = fx; fxyz[3 * j + 1] = fy; fxyz[3 * j + 2] = fz;
    const double qx = __ddiv_rn((double)fx, size), qy = __ddiv_rn((double)fy, size), qz = __ddiv_rn((double)fz, size);
    const double gx = __ddiv_rn((double)fx, fine), gy = __ddiv_rn((double)fy, fine), gz = __ddiv_rn((double)fz, fine);
    constexpr double kI32 = 2147483648.0;
    const bool ok = fabs(qx) < kI32 && fabs(qy) < kI32 && fabs(qz) < kI32 && fabs(gx) < kI32 && fabs(gy) < kI32 && fabs(gz) < kI32;
    vkeys[j] = ok ? pack_key((int)qx, (int)qy, (int)qz) : kInvalidKey;
    fkeys[j] = ok ? pack_key((int)gx, (int)gy, (int)gz) : kInvalidKey;
    idx[j] = (unsigned int)j;
}

// k_seg_claim with the colour map's block stride
__global__ void k_color_seg_claim(Slot* slots, unsigned int mask, float* blocks, int block_pts, const unsigned long long* __restrict__ keys,
                                  const unsigned int* __restrict__ seg_start, const int* n_seg_p,
                                  const unsigned int* __restrict__ is_new, const unsigned int* __restrict__ new_rank,
                                  long long block_base, int* seg_slot) {
    seg_claim(slots, mask, blocks, (size_t)(4 * block_pts), keys, seg_start, n_seg_p, is_new, new_rank, block_base, seg_slot);
}

// one thread per touched voxel: append the first (cap - count) offered points in sweep order, note the visit
__global__ void k_color_seg_process(Slot* slots, float* blocks, ColorPoint* cpts, double* last_visited,
                                    const unsigned long long* __restrict__ keys, const unsigned int* __restrict__ idx,
                                    const float* __restrict__ fxyz, const unsigned int* __restrict__ seg_start, const int* n_seg_p,
                                    const int* __restrict__ seg_slot, const unsigned int* __restrict__ is_new, long long m, int cap,
                                    int block_pts, double t_end, double t_last_process, unsigned int* accept_id, unsigned int* seg_first,
                                    long long* n_points) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= *n_seg_p) return;
    seg_first[s] = kNoIndex;
    const int slot = seg_slot[s];
    if (slot < 0) return;
    const unsigned int blk = slots[slot].block;
    int count = (int)slots[slot].count;
    float* bp = blocks + (size_t)blk * (4 * block_pts);
    const long long start = seg_start[s];
    const unsigned long long key = keys[start];
    if (is_new[s]) last_visited[blk] = 0.0;                       // voxelBlock::last_visited_time = 0.0 (include/cloudMap.h:153)
    int added = 0;
    for (long long j = start; j < m && keys[j] == key && count < cap; ++j) {
        const unsigned int i = idx[j];
        bp[4 * count] = fxyz[3 * (size_t)i]; bp[4 * count + 1] = fxyz[3 * (size_t)i + 1]; bp[4 * count + 2] = fxyz[3 * (size_t)i + 2];
        ColorPoint cp;                                            // rgbPoint::reset() (src/cloudMap.cpp:12-19)
        cp.rgb[0] = cp.rgb[1] = cp.rgb[2] = 0; cp.n_rgb = 0; cp.cov[0] = cp.cov[1] = cp.cov[2] = 0.f; cp.outlier_count = 0; cp.pad = 0; cp.obs_dist = 0.0; cp.last_obs = 0.0;
        cpts[(size_t)blk * block_pts + count] = cp;
        accept_id[i] = blk * (unsigned)block_pts + (unsigned)count;
        ++count; ++added;
    }
    if (added) {
        slots[slot].count = (unsigned int)count;
        reinterpret_cast<unsigned int*>(bp)[kMetaCount] = (unsigned int)count;
        atomicAdd(reinterpret_cast<unsigned long long*>(n_points), (unsigned long long)added);
    }
    // :486-490 / :509-513: once per voxel and sweep end time, whether or not a point was stored
    if (fabs(t_end - t_last_process) > 1e-5 && fabs(last_visited[blk] - t_end) > 1e-5) {
        last_visited[blk] = t_end;
        seg_first[s] = idx[start];                                // the sweep position of the voxel's first offered point
    }
}
__global__ void k_color_seg_keys(const unsigned long long* __restrict__ keys, const unsigned int* __restrict__ seg_start, const int* n_seg_p,
                                 unsigned long long* seg_key) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < *n_seg_p) seg_key[s] = keys[seg_start[s]];
}
// after sorting the visited voxels by the sweep position of their first point: write them as the (emptied) recent list
__global__ void k_color_append_recent(const unsigned int* __restrict__ first_sorted, const unsigned long long* __restrict__ key_sorted,
                                      int n_seg, unsigned long long* recent, long long* counters) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_seg || first_sorted[t] == kNoIndex) return;
    recent[t] = key_sorted[t];
    if (t + 1 == n_seg || first_sorted[t + 1] == kNoIndex) counters[3] = t + 1;   // how many were listed (read by the host)
}
// accepted points only keep their fine key
__global__ void k_color_mask_fine(unsigned long long* fkeys, const unsigned int* __restrict__ accept_id, long long m) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j < m && accept_id[j] == kNoIndex) fkeys[j] = kInvalidKey;
}
// heads of the fine-cell runs (= the first accepted point of the sweep in that cell) whose cell is still free win
__global__ void k_color_fine_winners(const Slot* fine, unsigned int fmask, const unsigned long long* __restrict__ fk_sorted,
                                     const unsigned int* __restrict__ idx_sorted, long long m, unsigned int* winner) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const unsigned long long k = fk_sorted[j];
    if (k == kInvalidKey || (j > 0 && fk_sorted[j - 1] == k)) return;
    short x, y, z;
    unpack_key(k, x, y, z);
    if (slot_find_rw(fine, fmask, k, x, y, z) < 0) winner[idx_sorted[j]] = 1u;
}
__global__ void k_color_emit_rgb(Slot* fine, unsigned int fmask, const unsigned long long* __restrict__ fkeys_by_idx,
                                 const unsigned int* __restrict__ winner, const unsigned int* __restrict__ rank,
                                 const unsigned int* __restrict__ accept_id, long long m, unsigned int* rgb_points, long long* counters,
                                 long long capacity) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m || !winner[j]) return;
    const long long pos = counters[0] + rank[j];
    if (pos < capacity) rgb_points[pos] = accept_id[j];            // point.point_index = rgb_points_vec.size() (:478, :503)
    const unsigned long long k = fkeys_by_idx[j];
    short x, y, z;
    unpack_key(k, x, y, z);
    slot_claim(fine, fmask, k, x, y, z, (unsigned)pos, 1u);       // hashmap_3d_points.insert (:481, :506)
}

// (point_world - t_world_camera).norm(), the 3-term sum as c0 + (c1 + c2) (DESIGN.md section 2)
__device__ __forceinline__ double camera_distance(const CamConst& c, double px, double py, double pz) {
    const double dx = __dsub_rn(px, c.t_wc[0]), dy = __dsub_rn(py, c.t_wc[1]), dz = __dsub_rn(pz, c.t_wc[2]);
    return __dsqrt_rn(__dadd_rn(__dmul_rn(dx, dx), __dadd_rn(__dmul_rn(dy, dy), __dmul_rn(dz, dz))));
}
// one stored point: project, sample the image, fuse `reps` times in a row (the voxel's repetitions in the recent list);
// returns how many of those fusions updateRgb counted
__device__ __forceinline__ unsigned render_point(const float* __restrict__ bp, ColorPoint* cpt, const CamConst& c,
                                                 const unsigned char* __restrict__ img, double obs_time, int reps) {
    const double px = (double)bp[0], py = (double)bp[1], pz = (double)bp[2];
    double u, v;
    if (!project_in_image(c, px, py, pz, u, v)) return 0;
    const double dist = camera_distance(c, px, py, pz);
    // getSubPixel<cv::Vec3b> (:71-98).  The +1 taps are clamped to the last row / column, which changes no value for
    // fov_margin >= 0 (negative margins are refused by srl_color_map_render_recent): fr + 1 == rows needs ceil(v) <= rows - 1,
    // because the window's upper bound fl(1 - fov) * rows is at most rows; so v == rows - 1 exactly, frac_r == 0 and
    // w10 == w11 == 0.  The same holds for columns.  The lower bound v >= fl(fov * rows) + 1 >= 1 keeps fr >= 0.  The
    // reference reads row `rows` there with weight 0.
    unsigned char bgr[3];
    sub_pixel_bgr(img, (size_t)c.cols * 3, c.cols, c.rows, v, u, bgr);
    double color[3];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) color[ch] = (double)bgr[ch];
    // rgbPoint::updateRgb (src/cloudMap.cpp:59-101), mixed float / double arithmetic as written there
    ColorPoint cp = *cpt;
    const double sigma = 15.0, process_noise_sigma = 0.1;
    unsigned rendered = 0;
    for (int rep = 0; rep < reps; ++rep) {
        if (cp.obs_dist != 0 && (dist > __dmul_rn(cp.obs_dist, 1.2))) continue;
        if (cp.n_rgb == 0) {
            cp.last_obs = obs_time; cp.obs_dist = dist;
#pragma unroll
            for (int i = 0; i < 3; ++i) { cp.rgb[i] = (short)round(color[i]); cp.cov[i] = (float)sigma; }
            cp.n_rgb = 1;
            continue;
        }
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            cp.cov[i] = __double2float_rn(__dadd_rn((double)cp.cov[i], __dmul_rn(process_noise_sigma, __dsub_rn(obs_time, cp.last_obs))));
            const double old_sigma = (double)cp.cov[i];
            const double c2 = (double)__fmul_rn(cp.cov[i], cp.cov[i]);
            cp.cov[i] = __double2float_rn(__dsqrt_rn(__ddiv_rn(1.0, __dadd_rn(__ddiv_rn(1.0, c2), __ddiv_rn(1.0, __dmul_rn(sigma, sigma))))));
            const double n2 = (double)__fmul_rn(cp.cov[i], cp.cov[i]);
            const double mix = __dadd_rn(__ddiv_rn((double)cp.rgb[i], __dmul_rn(old_sigma, old_sigma)), __ddiv_rn(color[i], __dmul_rn(sigma, sigma)));
            cp.rgb[i] = (short)(int)__dmul_rn(n2, mix);           // double -> short truncates
        }
        if (dist < cp.obs_dist) cp.obs_dist = dist;
        cp.last_obs = obs_time;
        cp.n_rgb = (short)(cp.n_rgb + 1);
        ++rendered;
    }
    *cpt = cp;
    return rendered;
}
// one warp per distinct recent voxel; its lanes walk the block in strides of 32 (point lane, lane + 32, ...), so a block of up
// to kColorMaxCap points takes up to 4 rounds.  Points are independent; a voxel listed `mult` times is fused `mult` times in a
// row, which is the list order for each of its points.
__global__ void __launch_bounds__(256) k_color_render(const Slot* slots, unsigned int mask, const float* __restrict__ blocks, int block_pts,
                                                       ColorPoint* cpts, const unsigned long long* __restrict__ uniq_keys,
                                                       const int* __restrict__ mult, const int* n_uniq_p, CamConst c,
                                                       const unsigned char* __restrict__ img, double obs_time, unsigned long long* n_rendered) {
    const int lane = threadIdx.x & 31;
    const int u_i = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    if (u_i >= *n_uniq_p) return;
    const unsigned long long key = uniq_keys[u_i];
    short kx, ky, kz;
    unpack_key(key, kx, ky, kz);
    const int slot = slot_find_rw(slots, mask, key, kx, ky, kz);
    if (slot < 0) return;
    const unsigned blk = slots[slot].block;
    const int count = (int)slots[slot].count;
    const int reps = mult[u_i];
    const float* bp = blocks + (size_t)blk * (4 * block_pts);
    ColorPoint* cb = cpts + (size_t)blk * block_pts;
    unsigned rendered = 0;
    for (int i = lane; i < count; i += 32) rendered += render_point(bp + 4 * i, cb + i, c, img, obs_time, reps);
    if (rendered) atomicAdd(n_rendered, (unsigned long long)rendered);
}
// colour state + last visited time in the block order of srl_map_download
__global__ void k_color_download(const ColorPoint* __restrict__ cpts, const float* __restrict__ blocks, const double* __restrict__ last_visited,
                                 int block_pts, long long n_voxels, int cap, short* rgb, short* n_rgb, float* cov, double* obs_dist,
                                 double* last_obs, double* visited) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_voxels * cap) return;
    const long long v = e / cap;
    const int i = (int)(e % cap);
    const int cnt = (int)reinterpret_cast<const unsigned int*>(blocks + (size_t)v * (4 * block_pts))[kMetaCount];
    const bool on = i < cnt;
    const ColorPoint cp = cpts[(size_t)v * block_pts + i];
    for (int a = 0; a < 3; ++a) { rgb[3 * e + a] = on ? cp.rgb[a] : (short)0; cov[3 * e + a] = (on && cp.n_rgb != 0) ? cp.cov[a] : 0.f; }
    n_rgb[e] = on ? cp.n_rgb : (short)0;
    obs_dist[e] = on ? cp.obs_dist : 0.0;
    last_obs[e] = on ? cp.last_obs : 0.0;
    if (i == 0) visited[v] = last_visited[v];
}
// rgb_points_vec entries (point ids block * block_pts + i) as (voxel key, index in block)
__global__ void k_color_rgb_ids(const unsigned int* __restrict__ rgb_points, long long n, const float* __restrict__ blocks, int block_pts, short* out) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const unsigned id = rgb_points[t];
    const unsigned blk = id / (unsigned)block_pts;
    const unsigned int* meta = reinterpret_cast<const unsigned int*>(blocks + (size_t)blk * (4 * block_pts));
    short x, y, z;
    unpack_key((unsigned long long)meta[kMetaKeyLo] | ((unsigned long long)meta[kMetaKeyHi] << 32), x, y, z);
    out[4 * t] = x; out[4 * t + 1] = y; out[4 * t + 2] = z; out[4 * t + 3] = (short)(id - blk * (unsigned)block_pts);
}

// ---- rgbMapTracker::selectPointsForProjection (src/rgbMapTracker.cpp:45-152) -----------------------------------------------
// The reference walks the candidates in point_index order and keeps, per pixel cell, a winner and its depth stored as a
// float; a later candidate takes the cell when (float)stored > depth.  That stored float is the running minimum of the
// candidates' float depths (DESIGN.md section 4), so a cell's winner is its last candidate whose depth is below the minimum of
// the float depths before it, or its first candidate.  Here: cell keys per candidate, a stable sort by cell, a segmented
// exclusive min-scan of the float depths, a segmented "last flagged" reduction, and an order-preserving compaction.
//
// Candidate j is point_index p = j * skip of the candidate list: the last point of the voxel d_recent[p] (recent mode) or
// rgb_points_vec[p].  One that passes the depth bounds and the projection gets the key of its cell (u, v), each offset by the
// window's lower bound and packed as (u - u0) << bits_v | (v - v0); the others get `none`, which no cell produces.
__global__ void k_proj_candidates(const Slot* slots, unsigned int mask, const float* __restrict__ blocks, int block_pts,
                                  const unsigned long long* __restrict__ recent, const unsigned int* __restrict__ rgb_points, long long m,
                                  int skip, CamConst c, double min_dis, double min_depth, double max_depth, int u0, int v0, int bits_v,
                                  unsigned long long none, unsigned long long* key, unsigned int* ord, unsigned int* cand_id, double* depth,
                                  float2* uv) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const long long p = j * skip;
    unsigned id = kNoIndex;
    if (recent) {                                                    // map[voxel].points.back() (:76-82)
        const unsigned long long vk = recent[p];
        short kx, ky, kz;
        unpack_key(vk, kx, ky, kz);
        const int slot = slot_find_rw(slots, mask, vk, kx, ky, kz);
        if (slot >= 0 && slots[slot].count > 0) id = slots[slot].block * (unsigned)block_pts + slots[slot].count - 1u;
    } else {
        id = rgb_points[p];
    }
    unsigned long long k = none;
    double d = 0.0;
    if (id != kNoIndex) {
        const unsigned blk = id / (unsigned)block_pts;
        const float* bp = blocks + (size_t)blk * (4 * block_pts) + 4 * (size_t)(id - blk * (unsigned)block_pts);
        const double px = (double)bp[0], py = (double)bp[1], pz = (double)bp[2];
        d = camera_distance(c, px, py, pz);                         // :97
        double u, v;
        if (!(d > max_depth) && !(d < min_depth) && project_in_image(c, px, py, pz, u, v)) {   // :99-114
            const int cu = projection_cell(u, min_dis), cv = projection_cell(v, min_dis);   // :116-117
            k = ((unsigned long long)(unsigned)(cu - u0) << bits_v) | (unsigned long long)(unsigned)(cv - v0);
            uv[j] = make_float2(__double2float_rn(u), __double2float_rn(v));   // cv::Point2f(u_f, v_f)
        }
    }
    key[j] = k;
    ord[j] = (unsigned)j;
    cand_id[j] = id;
    depth[j] = d;
}
// the float depths in cell order: mask_depth holds (float)depth (:134)
__global__ void k_proj_float_depths(const unsigned int* __restrict__ ord_sorted, const double* __restrict__ depth, long long m, float* fd) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k < m) fd[k] = __double2float_rn(depth[ord_sorted[k]]);
}
// sorted position k takes its cell when its depth is below the minimum of the float depths before it in the cell (the float
// widened, as `mask_depth[u][v] > depth` compares at :119); the first of a cell sees +inf.  Value: k if it takes the cell, else -1.
__global__ void k_proj_takers(const unsigned long long* __restrict__ key_sorted, const unsigned int* __restrict__ ord_sorted,
                              const double* __restrict__ depth, const float* __restrict__ prefix_min, long long m, unsigned long long none,
                              int* taker) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= m) return;
    taker[k] = (key_sorted[k] != none && depth[ord_sorted[k]] < (double)prefix_min[k]) ? (int)k : -1;
}
// the last taker of each cell is its winner: flag it in candidate order
__global__ void k_proj_mark_winners(const int* __restrict__ last_taker, const int* n_cells_p, const unsigned int* __restrict__ ord_sorted,
                                    unsigned char* win) {
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= *n_cells_p) return;
    const int k = last_taker[r];
    if (k >= 0) win[ord_sorted[k]] = 1;
}
// the winners in point_index order (std::map order, :141-151): point id, the stored position, the float uv
__global__ void k_proj_gather(const unsigned int* __restrict__ sel, long long n, const unsigned int* __restrict__ cand_id,
                              const float2* __restrict__ cand_uv, const float* __restrict__ blocks, int block_pts, unsigned int* ids,
                              float* xyz, float* uv) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const unsigned j = sel[k];
    const unsigned id = cand_id[j];
    if (ids) ids[k] = id;
    if (xyz) {
        const unsigned blk = id / (unsigned)block_pts;
        const float* bp = blocks + (size_t)blk * (4 * block_pts) + 4 * (size_t)(id - blk * (unsigned)block_pts);
        xyz[3 * k] = bp[0]; xyz[3 * k + 1] = bp[1]; xyz[3 * k + 2] = bp[2];
    }
    if (uv) { const float2 w = cand_uv[j]; uv[2 * k] = w.x; uv[2 * k + 1] = w.y; }
}
struct ProjMinF { __device__ __forceinline__ float operator()(float a, float b) const { return b < a ? b : a; } };
struct ProjMaxI { __device__ __forceinline__ int operator()(int a, int b) const { return b > a ? b : a; } };
struct ProjKeyEq { __device__ __forceinline__ bool operator()(unsigned long long a, unsigned long long b) const { return a == b; } };

// ---- the tracker's per-point reads: gather by point id -------------------------------------------------------------------
// an id is known when its block is one of the map's voxels and its index is below that voxel's count
__global__ void k_color_check_ids(const unsigned int* __restrict__ ids, long long n, const float* __restrict__ blocks, int block_pts,
                                  long long n_voxels, unsigned long long* n_bad) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    bool bad = false;
    if (t < n) {
        const unsigned id = ids[t];
        const unsigned blk = id / (unsigned)block_pts;
        bad = (long long)blk >= n_voxels ||
              id - blk * (unsigned)block_pts >= reinterpret_cast<const unsigned int*>(blocks + (size_t)blk * (4 * block_pts))[kMetaCount];
    }
    const unsigned b = __ballot_sync(0xffffffffu, bad);
    if ((threadIdx.x & 31) == 0 && b) atomicAdd(n_bad, (unsigned long long)__popc(b));
}
// position, BGR state, N_rgb and covariance of each id (cov 0 while N_rgb == 0, like srl_color_map_download_state: a
// wrapped, negative N_rgb has a covariance)
__global__ void k_color_gather(const unsigned int* __restrict__ ids, long long n, const float* __restrict__ blocks, int block_pts,
                               const ColorPoint* __restrict__ cpts, float* xyz, short* rgb, short* n_rgb, float* cov) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const unsigned id = ids[t];
    const unsigned blk = id / (unsigned)block_pts;
    if (xyz) {
        const float* bp = blocks + (size_t)blk * (4 * block_pts) + 4 * (size_t)(id - blk * (unsigned)block_pts);
        xyz[3 * t] = bp[0]; xyz[3 * t + 1] = bp[1]; xyz[3 * t + 2] = bp[2];
    }
    const ColorPoint cp = cpts[id];
    if (rgb) { rgb[3 * t] = cp.rgb[0]; rgb[3 * t + 1] = cp.rgb[1]; rgb[3 * t + 2] = cp.rgb[2]; }
    if (n_rgb) n_rgb[t] = cp.n_rgb;
    if (cov) for (int a = 0; a < 3; ++a) cov[3 * t + a] = cp.n_rgb != 0 ? cp.cov[a] : 0.f;
}

__global__ void k_gather_points(const double* __restrict__ xyz, const unsigned int* __restrict__ sel, int m, double* out) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const size_t i = sel[j];
    out[3 * j] = xyz[3 * i]; out[3 * j + 1] = xyz[3 * i + 1]; out[3 * j + 2] = xyz[3 * i + 2];
}

// ---- the published maps ----------------------------------------------------------------------------------------------
// addPointToPcl (src/lioOptimization.cpp:1346-1355) over the published points in sweep order: x, y, z the stored floats,
// intensity = 50 * (z - translation.z()) in FP64 (float z widened), rounded once to float
__global__ void k_publish_gather(const float* __restrict__ fxyz, const unsigned int* __restrict__ sel, const int* n_sel_p, double tz,
                                 float* out) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= *n_sel_p) return;
    const size_t i = sel[j];
    const float z = fxyz[3 * i + 2];
    out[4 * j] = fxyz[3 * i]; out[4 * j + 1] = fxyz[3 * i + 1]; out[4 * j + 2] = z;
    out[4 * j + 3] = __double2float_rn(__dmul_rn(50.0, __dsub_rn((double)z, tz)));
}
// position p of the export (publish order: rgb_points_vec index p; save order: index n - 1 - p, so index 0 is never reached)
// -> flag N_rgb >= min_views (short against int, :1221, :1404); the flagged count is added to *count
__global__ void k_color_export_flags(const unsigned int* __restrict__ rgb_points, const ColorPoint* __restrict__ cpts, long long m,
                                     long long n, int order, int min_views, unsigned char* flags, unsigned long long* count) {
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    bool f = false;
    if (p < m) {
        const unsigned id = rgb_points[order ? n - 1 - p : p];
        f = (int)cpts[id].n_rgb >= min_views;
        flags[p] = f ? 1 : 0;
    }
    const unsigned b = __ballot_sync(0xffffffffu, f);
    if ((threadIdx.x & 31) == 0 && b) atomicAdd(count, (unsigned long long)__popc(b));
}
// the flagged positions of one chunk (sel relative to base) -> getPosition() as stored, r = rgb[2], g = rgb[1], b = rgb[0]: the BGR
// state swapped, short -> double -> uint8_t as g++ compiles it on x86-64 (int32 truncation, low 8 bits)
__global__ void k_color_export_gather(const unsigned int* __restrict__ rgb_points, const float* __restrict__ blocks, int block_pts,
                                      const ColorPoint* __restrict__ cpts, const unsigned int* __restrict__ sel, const int* n_sel_p,
                                      long long base, long long n, int order, float* xyz, unsigned char* rgb) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= *n_sel_p) return;
    const long long p = base + sel[k];
    const unsigned id = rgb_points[order ? n - 1 - p : p];
    const unsigned blk = id / (unsigned)block_pts;
    const float* b = blocks + (size_t)blk * (4 * block_pts) + 4 * (size_t)(id - blk * (unsigned)block_pts);
    xyz[3 * k] = b[0]; xyz[3 * k + 1] = b[1]; xyz[3 * k + 2] = b[2];
    const ColorPoint& cp = cpts[id];
    rgb[3 * k] = (unsigned char)(cp.rgb[2] & 0xff); rgb[3 * k + 1] = (unsigned char)(cp.rgb[1] & 0xff); rgb[3 * k + 2] = (unsigned char)(cp.rgb[0] & 0xff);
}

// ---- growth: arrays on CUDA VMM, slot tables rebuilt -----------------------------------------------------------------
// The driver's VMM calls come through the runtime's entry-point query, so the library does not link libcuda.
struct VmmApi {
    PFN_cuMemGetAllocationGranularity_v10020 granularity = nullptr;
    PFN_cuMemAddressReserve_v10020 reserve = nullptr;
    PFN_cuMemAddressFree_v10020 free_va = nullptr;
    PFN_cuMemCreate_v10020 create = nullptr;
    PFN_cuMemRelease_v10020 release = nullptr;
    PFN_cuMemMap_v10020 map = nullptr;
    PFN_cuMemUnmap_v10020 unmap = nullptr;
    PFN_cuMemSetAccess_v10020 set_access = nullptr;
    bool ok = false;
};
static const VmmApi& vmm() {
    static VmmApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        auto get = [](const char* name, void** fn) {
            cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
            return cudaGetDriverEntryPointByVersion(name, fn, 12000, cudaEnableDefault, &q) == cudaSuccess &&
                   q == cudaDriverEntryPointSuccess && *fn != nullptr;
        };
        api.ok = get("cuMemGetAllocationGranularity", reinterpret_cast<void**>(&api.granularity)) &&
                 get("cuMemAddressReserve", reinterpret_cast<void**>(&api.reserve)) &&
                 get("cuMemAddressFree", reinterpret_cast<void**>(&api.free_va)) &&
                 get("cuMemCreate", reinterpret_cast<void**>(&api.create)) &&
                 get("cuMemRelease", reinterpret_cast<void**>(&api.release)) &&
                 get("cuMemMap", reinterpret_cast<void**>(&api.map)) &&
                 get("cuMemUnmap", reinterpret_cast<void**>(&api.unmap)) &&
                 get("cuMemSetAccess", reinterpret_cast<void**>(&api.set_access));
    });
    return api;
}
static CUmemAllocationProp vm_prop(int device) {
    CUmemAllocationProp p = {};
    p.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    p.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    p.location.id = device;
    return p;
}
static int vm_fail(srl_ctx* ctx, CUresult r, const char* where) {
    return set_err(ctx, SRL_CUDA_ERROR, std::string(where) + " failed (CUresult " + std::to_string((int)r) + ")");
}
// address space for limit_bytes, in multiples of the recommended granularity; nothing mapped yet
static int vm_reserve(srl_ctx* ctx, VmArray& a, size_t limit_bytes) {
    const VmmApi& api = vmm();
    if (!api.ok) return set_err(ctx, SRL_CUDA_ERROR, "the driver does not provide the CUDA virtual memory management calls");
    const CUmemAllocationProp prop = vm_prop(ctx->device);
    size_t g = 0;
    CUresult r = api.granularity(&g, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED);
    if (r != CUDA_SUCCESS) return vm_fail(ctx, r, "cuMemGetAllocationGranularity");
    const size_t bytes = align_up(std::max<size_t>(limit_bytes, 1), g);
    CUdeviceptr p = 0;
    if ((r = api.reserve(&p, bytes, g, 0, 0)) != CUDA_SUCCESS) return vm_fail(ctx, r, "cuMemAddressReserve");
    a.base = p; a.granularity = g; a.reserved = bytes; a.mapped = 0;
    return SRL_OK;
}
// map memory behind the array up to at least `bytes` (zero-filled on the ctx stream); on failure the array is as it was
static int vm_grow(srl_ctx* ctx, VmArray& a, size_t bytes) {
    const size_t target = std::min(a.reserved, align_up(bytes, a.granularity));
    if (target <= a.mapped) return SRL_OK;
    const VmmApi& api = vmm();
    const size_t size = target - a.mapped;
    const CUdeviceptr at = a.base + a.mapped;
    const CUmemAllocationProp prop = vm_prop(ctx->device);
    CUmemGenericAllocationHandle h = 0;
    CUresult r = api.create(&h, size, &prop, 0);
    if (r != CUDA_SUCCESS) return vm_fail(ctx, r, "cuMemCreate");
    if ((r = api.map(at, size, 0, h, 0)) != CUDA_SUCCESS) { api.release(h); return vm_fail(ctx, r, "cuMemMap"); }
    CUmemAccessDesc acc = {};
    acc.location = prop.location;
    acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    if ((r = api.set_access(at, size, &acc, 1)) != CUDA_SUCCESS) { api.unmap(at, size); api.release(h); return vm_fail(ctx, r, "cuMemSetAccess"); }
    a.chunks.emplace_back(h, size);
    a.mapped = target;
    SRL_CUDA(ctx, cudaMemsetAsync(reinterpret_cast<void*>(at), 0, size, ctx->stream));
    return SRL_OK;
}
VmArray::~VmArray() {
    if (!base) return;
    cudaDeviceSynchronize();
    const VmmApi& api = vmm();
    size_t off = 0;
    for (const auto& c : chunks) { api.unmap(base + off, c.second); api.release(c.first); off += c.second; }
    api.free_va(base, reserved);
}
// the sizing rule of the slot tables: the smallest power of two >= 1024 that keeps n entries at load <= 0.5 (at most 2^32
// slots, where the 32-bit probe mask is still exact)
static size_t table_slots(size_t n) {
    size_t c = 1024;
    while (c < 2 * n && c < (size_t(1) << 32)) c <<= 1;
    return c;
}
// make room for n entries: a larger table, rehashed on the device from the old one (k_rehash); unchanged on failure
static int table_grow(srl_ctx* ctx, DevArray<Slot>& slots, size_t& capacity, size_t n) {
    const size_t cap = table_slots(n);
    if (cap <= capacity) return SRL_OK;
    DevArray<Slot> fresh;
    cudaError_t e = fresh.alloc(cap);
    if (e != cudaSuccess) return cuda_fail(ctx, e, "slot table growth/cudaMalloc");
    e = cudaMemsetAsync(fresh, 0, cap * sizeof(Slot), ctx->stream);
    if (e == cudaSuccess && capacity) {
        const int T = 256;
        k_rehash<<<(unsigned)((capacity + T - 1) / T), T, 0, ctx->stream>>>(slots, (long long)capacity, fresh, (unsigned)(cap - 1));
        ctx->launches += 1;
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) return cuda_fail(ctx, e, "slot table growth");
    slots = std::move(fresh); capacity = cap;
    return SRL_OK;
}

}  // namespace srl

using namespace srl;

int srl::check_lio_map(srl_ctx* ctx, const srl_map* m) {
    if (m->block_pts == kBlockCap) return SRL_OK;
    return set_err(ctx, SRL_BAD_ARG, "map has " + std::to_string(m->block_pts) + " points per block; the LIO path needs " + std::to_string(kBlockCap));
}

// ---- N4: colour map host side ---------------------------------------------------------------------------------------
// the projection constants of a camera (renderer, selection, optical-flow tracker)
CamConst srl::camera_constants(const srl_camera* cam) {
    CamConst c;
    quat_to_rot(cam->q_camera_world, c.R);
    for (int i = 0; i < 3; ++i) { c.t_cw[i] = cam->t_camera_world[i]; c.t_wc[i] = cam->t_world_camera[i]; }
    c.fx = cam->fx; c.fy = cam->fy; c.cx = cam->cx; c.cy = cam->cy; c.fov = cam->fov_margin; c.cols = cam->cols; c.rows = cam->rows;
    return c;
}
struct srl_color_map {
    srl_ctx* ctx = nullptr;
    int device = 0;
    std::unique_ptr<srl_map> vox;           // color_voxel_map (include/lioOptimization.h:275)
    double min_dist = 0.15;
    // per voxel (committed with vox->committed_voxels)
    srl::VmArray cpts_mem, last_visited_mem;
    srl::ColorPoint* d_cpts = nullptr;      // committed_voxels * block_pts
    double* d_last_visited = nullptr;       // committed_voxels
    // per rgb point (committed_rgb_points of at most max_rgb_points)
    srl::DevArray<srl::Slot> d_fine;        // hashmap_3d_points as an occupancy set: key = fine cell, block = index into rgb_points
    size_t fine_capacity = 0;
    srl::VmArray rgb_mem;
    unsigned int* d_rgb_points = nullptr;   // rgb_points_vec: point ids (block * block_pts + index)
    size_t max_rgb_points = 0, committed_rgb_points = 0;
    // per recent voxel (committed_recent of at most recent_capacity = max_voxels: a call lists each voxel at most once)
    srl::VmArray recent_temp_mem, recent_mem;
    unsigned long long* d_recent_temp = nullptr;   // voxels_recent_visited_temp of the current rendering call (packed keys)
    unsigned long long* d_recent = nullptr;        // map_tracker->voxels_recent_visited
    size_t recent_capacity = 0, committed_recent = 0;
    srl::DevArray<long long> d_counters;    // [0] rgb points, [3] recent voxels listed by the call
    int64_t n_rgb_points = 0, n_recent = 0, n_new_recent = 0;
};

ColorMapView srl::color_map_view(const srl_color_map* cm) {
    return ColorMapView{cm->vox->d_blocks, cm->d_cpts, cm->vox->block_pts, (long long)cm->vox->n_voxels};
}
srl_ctx* srl::color_map_ctx(const srl_color_map* cm) { return cm->ctx; }
ColorPoint* srl::color_map_states(srl_color_map* cm) { return cm->d_cpts; }

// the colour state of committed_voxels voxels (called by map_grow before the blocks grow)
static int color_map_grow_voxels(srl_color_map* cm, size_t committed_voxels) {
    const size_t pts = committed_voxels * (size_t)cm->vox->block_pts;
    int rc = vm_grow(cm->ctx, cm->cpts_mem, pts * sizeof(ColorPoint));
    if (rc != SRL_OK) return rc;
    return vm_grow(cm->ctx, cm->last_visited_mem, committed_voxels * sizeof(double));
}
// the rgb list and the fine set for at least `need` rgb points (same doubling rule as the voxels)
static int color_map_grow_rgb(srl_color_map* cm, size_t need) {
    need = std::min(need, cm->max_rgb_points);
    if (need <= cm->committed_rgb_points) return SRL_OK;
    const size_t n = std::min(cm->max_rgb_points, std::max(2 * cm->committed_rgb_points, need));
    int rc = vm_grow(cm->ctx, cm->rgb_mem, n * sizeof(unsigned int));
    if (rc != SRL_OK) return rc;
    if ((rc = table_grow(cm->ctx, cm->d_fine, cm->fine_capacity, n)) != SRL_OK) return rc;
    cm->committed_rgb_points = n;
    return SRL_OK;
}
// both recent-voxel lists (the rendering copies one into the other) for at least `need` entries
static int color_map_grow_recent(srl_color_map* cm, size_t need) {
    need = std::min(need, cm->recent_capacity);
    if (need <= cm->committed_recent) return SRL_OK;
    const size_t n = std::min(cm->recent_capacity, std::max(2 * cm->committed_recent, need));
    int rc = vm_grow(cm->ctx, cm->recent_temp_mem, n * sizeof(unsigned long long));
    if (rc != SRL_OK) return rc;
    if ((rc = vm_grow(cm->ctx, cm->recent_mem, n * sizeof(unsigned long long))) != SRL_OK) return rc;
    cm->committed_recent = n;
    return SRL_OK;
}

// commit blocks for at least `need` voxels, capped at max_voxels: the committed count doubles, or jumps to `need` when that
// is more.  Blocks, the slot table and an owning colour map's per-voxel arrays grow together.  On failure the map keeps
// its contents and committed count (arrays grown before the failing one keep their extra memory unused).
static int map_grow(srl_map* m, size_t need) {
    need = std::min(need, m->max_voxels);
    if (need <= m->committed_voxels) return SRL_OK;
    const size_t nv = std::min(m->max_voxels, std::max(2 * m->committed_voxels, need));
    int rc;
    if (m->owner && (rc = color_map_grow_voxels(m->owner, nv)) != SRL_OK) return rc;
    if ((rc = vm_grow(m->ctx, m->blocks_mem, nv * 4 * (size_t)m->block_pts * sizeof(float))) != SRL_OK) return rc;
    if ((rc = table_grow(m->ctx, m->d_slots, m->capacity, nv)) != SRL_OK) return rc;
    m->committed_voxels = nv;
    return SRL_OK;
}

// the total of an exclusive scan over n > 0 flags: its last rank plus the last flag
static int scan_total(srl_ctx* ctx, const unsigned* flags, const unsigned* rank, long long n, long long* total) {
    unsigned last_rank = 0, last_flag = 0;
    SRL_CUDA(ctx, cudaMemcpyAsync(&last_rank, rank + (n - 1), sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream));
    SRL_CUDA(ctx, cudaMemcpyAsync(&last_flag, flags + (n - 1), sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream));
    SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *total = (long long)last_rank + last_flag;
    return SRL_OK;
}

// The voxel segments of a batch of points: their keys sorted stably (sweep order inside a voxel) with the points' indices,
// the start of every run of one valid key, and per run its slot and whether its voxel is new, with the rank of the new ones.
struct Segments {
    unsigned long long *keys, *keys_sorted;
    unsigned *idx, *idx_sorted;
    unsigned char* flags;
    unsigned *start, *is_new, *new_rank;
    int* slot;
    int* d_count;
    void* tmp;          // CUB temporary storage of segment_tmp_bytes (or more)
    size_t tmp_bytes;
    void place(Carve& c, size_t n, size_t tmp_size) {
        keys = c.take<unsigned long long>(n); keys_sorted = c.take<unsigned long long>(n);
        idx = c.take<unsigned>(n); idx_sorted = c.take<unsigned>(n);
        flags = c.take<unsigned char>(n);
        start = c.take<unsigned>(n); slot = c.take<int>(n); is_new = c.take<unsigned>(n); new_rank = c.take<unsigned>(n);
        d_count = c.take<int>(1);
        tmp = c.take<char>(tmp_size); tmp_bytes = tmp_size;
    }
};
// CUB temporary storage for the sort, the selection and the scan of n keys (also every other selection or scan over n)
static size_t segment_tmp_bytes(int n, cudaStream_t st) {
    size_t tmp_sort = 0, tmp_sel = 0, tmp_scan = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tmp_sort, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (unsigned*)nullptr,
                                    (unsigned*)nullptr, n, 0, 50, st);
    cub::DeviceSelect::Flagged(nullptr, tmp_sel, thrust::counting_iterator<unsigned int>(0), (unsigned char*)nullptr, (unsigned*)nullptr,
                               (int*)nullptr, n, st);
    cub::DeviceScan::ExclusiveSum(nullptr, tmp_scan, (unsigned*)nullptr, (unsigned*)nullptr, n, st);
    return std::max(tmp_sort, std::max(tmp_sel, tmp_scan));
}
// sort the n keys in s.keys (with s.idx) and find the starts of their runs; *n_seg = the number of runs
static int segment_keys(srl_ctx* ctx, const Segments& s, int n, int* n_seg) {
    cudaStream_t st = ctx->stream;
    const int T = 256;
    size_t tb = s.tmp_bytes;
    cub::DeviceRadixSort::SortPairs(s.tmp, tb, s.keys, s.keys_sorted, s.idx, s.idx_sorted, n, 0, 50, st);
    k_seg_flags<<<(unsigned)((n + T - 1) / T), T, 0, st>>>(s.keys_sorted, (long long)n, s.flags);
    tb = s.tmp_bytes;
    cub::DeviceSelect::Flagged(s.tmp, tb, thrust::counting_iterator<unsigned int>(0), s.flags, s.start, s.d_count, n, st);
    *n_seg = 0;
    SRL_CUDA(ctx, cudaMemcpyAsync(n_seg, s.d_count, sizeof(int), cudaMemcpyDeviceToHost, st));
    SRL_CUDA(ctx, cudaStreamSynchronize(st));
    ctx->launches += 3;
    return SRL_OK;
}
// the voxels of n_seg > 0 runs: the map grows for up to n_seg new ones (before the lookup, which stores slot indices), each
// run finds its slot (allow_new: an absent voxel is new), the new ones are ranked and counted.  SRL_MAP_FULL past max_voxels.
static int count_new_voxels(srl_map* m, const Segments& s, int n_seg, bool allow_new, const char* who, long long* total_new) {
    srl_ctx* ctx = m->ctx;
    int rc = map_grow(m, (size_t)m->n_voxels + (size_t)n_seg);
    if (rc != SRL_OK) return rc;
    const int T = 256;
    k_seg_lookup<<<(unsigned)((n_seg + T - 1) / T), T, 0, ctx->stream>>>(m->d_slots, (unsigned)(m->capacity - 1), s.keys_sorted, s.start,
                                                                       s.d_count, allow_new ? 1 : 0, s.slot, s.is_new);
    size_t tb = s.tmp_bytes;
    cub::DeviceScan::ExclusiveSum(s.tmp, tb, s.is_new, s.new_rank, n_seg, ctx->stream);
    if ((rc = scan_total(ctx, s.is_new, s.new_rank, n_seg, total_new)) != SRL_OK) return rc;
    ctx->launches += 2;
    if ((size_t)(m->n_voxels + *total_new) > m->max_voxels)
        return set_err(ctx, SRL_MAP_FULL, std::string(who) + ": voxel pool exhausted (raise max_voxels)");
    return SRL_OK;
}

// the pool reserves address space for max_voxels blocks of block_pts float4 and commits initial_voxels of them
// (arguments already checked)
static int map_create(srl_ctx* ctx, double voxel_size, int32_t max_num_points_in_voxel, int block_pts, size_t initial_voxels,
                      size_t max_voxels, srl_map** out) {
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    std::unique_ptr<srl_map> m(new srl_map());
    m->ctx = ctx; m->device = ctx->device; m->voxel_size = voxel_size; m->cap = max_num_points_in_voxel; m->block_pts = block_pts; m->max_voxels = max_voxels;
    const size_t block_bytes = 4 * (size_t)block_pts * sizeof(float);
    int rc;
    if ((rc = vm_reserve(ctx, m->blocks_mem, max_voxels * block_bytes)) != SRL_OK ||
        (rc = vm_grow(ctx, m->blocks_mem, initial_voxels * block_bytes)) != SRL_OK ||
        (rc = table_grow(ctx, m->d_slots, m->capacity, initial_voxels)) != SRL_OK)
        return rc;
    m->d_blocks = reinterpret_cast<float*>(m->blocks_mem.base);
    m->committed_voxels = initial_voxels;
    SRL_CUDA(ctx, m->d_counters.alloc(4));
    if ((rc = srl_map_clear(m.get())) != SRL_OK) return rc;
    *out = m.release();
    return SRL_OK;
}

extern "C" {

int srl_map_create_growable(srl_ctx* ctx, double voxel_size, int32_t max_num_points_in_voxel, size_t initial_voxels, size_t max_voxels,
                            srl_map** out) {
    if (!ctx || !out) return SRL_BAD_ARG;
    if (!(voxel_size > 0) || max_num_points_in_voxel < 1 || max_num_points_in_voxel > kBlockCap || max_voxels == 0)
        return set_err(ctx, SRL_BAD_ARG, "srl_map_create: voxel_size>0, 1<=max_num_points_in_voxel<=20, max_voxels>0 required");
    // the pass kernels address points as 32-bit float indices into the block pool (block * 80 + 4 * i)
    if (max_voxels > (size_t(1) << 25)) return set_err(ctx, SRL_BAD_ARG, "srl_map_create: max_voxels is limited to 2^25 (33.5 M voxels, 10.7 GB of blocks)");
    if (initial_voxels < 1 || initial_voxels > max_voxels) return set_err(ctx, SRL_BAD_ARG, "srl_map_create_growable: 1 <= initial_voxels <= max_voxels required");
    return map_create(ctx, voxel_size, max_num_points_in_voxel, kBlockCap, initial_voxels, max_voxels, out);
}

int srl_map_create(srl_ctx* ctx, double voxel_size, int32_t max_num_points_in_voxel, size_t max_voxels, srl_map** out) {
    return srl_map_create_growable(ctx, voxel_size, max_num_points_in_voxel, max_voxels, max_voxels, out);
}

void srl_map_destroy(srl_map* m) {
    if (!m) return;
    cudaSetDevice(m->device);
    delete m;
}

int srl_map_capacity(srl_map* m, size_t* committed_voxels, size_t* slot_capacity, size_t* committed_bytes) {
    if (!m) return SRL_BAD_ARG;
    if (committed_voxels) *committed_voxels = m->committed_voxels;
    if (slot_capacity) *slot_capacity = m->capacity;
    if (committed_bytes) *committed_bytes = m->blocks_mem.mapped + m->capacity * sizeof(Slot);
    return SRL_OK;
}

int srl_map_clear(srl_map* m) {
    if (!m) return SRL_BAD_ARG;
    srl_ctx* ctx = m->ctx;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    SRL_CUDA(ctx, cudaMemsetAsync(m->d_slots, 0, m->capacity * sizeof(Slot), ctx->stream));
    SRL_CUDA(ctx, cudaMemsetAsync(m->d_counters, 0, 4 * sizeof(long long), ctx->stream));
    SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    m->n_voxels = 0;
    return SRL_OK;
}

// ---- removePointsFarFromLocation (src/lioOptimization.cpp:556-572; row N4): a voxel goes when its FIRST point is farther
// than `distance` from `location`.  Open addressing has no cheap erase, and the block pool must stay dense (block index
// = slot payload), so eviction is mark -> compact the pool (stable: surviving blocks keep their relative order) ->
// rebuild the slot table from the keys kept in the blocks.
__global__ void k_far_flags(const float* __restrict__ blocks, long long n_voxels, double lx, double ly, double lz, double dist2,
                            unsigned* __restrict__ keep) {
    const long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= n_voxels) return;
    const float* b = blocks + (size_t)v * kBlockFloats;
    const unsigned cnt = reinterpret_cast<const unsigned*>(b)[kMetaCount];
    // rgbPoint::getPosition() widens the stored floats; (pt - location).squaredNorm() reduces as x^2 + (y^2 + z^2)
    const double dx = __dsub_rn((double)b[0], lx), dy = __dsub_rn((double)b[1], ly), dz = __dsub_rn((double)b[2], lz);
    const double d2 = __dadd_rn(__dmul_rn(dx, dx), __dadd_rn(__dmul_rn(dy, dy), __dmul_rn(dz, dz)));
    keep[v] = (cnt > 0 && !(d2 > dist2)) ? 1u : 0u;
}
__global__ void k_compact_blocks(const float* __restrict__ blocks, long long n_voxels, const unsigned* __restrict__ keep,
                                 const unsigned* __restrict__ new_index, float* __restrict__ out) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // one float4 per thread
    const long long v = e / (kBlockFloats / 4);
    if (v >= n_voxels || !keep[v]) return;
    const int q = (int)(e % (kBlockFloats / 4));
    reinterpret_cast<float4*>(out + (size_t)new_index[v] * kBlockFloats)[q] = reinterpret_cast<const float4*>(blocks + (size_t)v * kBlockFloats)[q];
}
__global__ void k_rebuild_slots(Slot* slots, unsigned int mask, const float* __restrict__ blocks, long long n_voxels, long long* n_points) {
    const long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= n_voxels) return;
    const unsigned int* meta = reinterpret_cast<const unsigned int*>(blocks + (size_t)v * kBlockFloats);
    const unsigned long long key = (unsigned long long)meta[kMetaKeyLo] | ((unsigned long long)meta[kMetaKeyHi] << 32);
    short x, y, z;
    unpack_key(key, x, y, z);
    slot_claim(slots, mask, key, x, y, z, (unsigned)v, meta[kMetaCount]);
    atomicAdd(reinterpret_cast<unsigned long long*>(n_points), (unsigned long long)meta[kMetaCount]);
}

int srl_map_remove_far(srl_map* m, const double location[3], double distance, int64_t* n_removed) {
    if (!m || !location) return SRL_BAD_ARG;
    srl_ctx* ctx = m->ctx;
    if (int rc = check_lio_map(ctx, m)) return rc;
    // the compaction moves blocks, which a colour map's per-point state, rgb list and point ids are indexed by
    if (m->owner) return set_err(ctx, SRL_BAD_ARG, "srl_map_remove_far: the map is a colour map's voxel map (eviction would move its point ids)");
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    if (n_removed) *n_removed = 0;
    const long long nv = (long long)m->n_voxels;
    if (nv == 0) return SRL_OK;
    size_t tmp = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, tmp, (unsigned*)nullptr, (unsigned*)nullptr, (int)nv, ctx->stream);
    unsigned *keep = nullptr, *nidx = nullptr;
    void* cub_tmp = nullptr;
    float* pool = nullptr;   // worst case every block survives: the compacted copy needs a pool-sized scratch
    int rc = carve_scratch(ctx, [&](Carve& c) {
        keep = c.take<unsigned>(nv); nidx = c.take<unsigned>(nv);
        cub_tmp = c.take<char>(tmp);
        pool = c.take<float>((size_t)nv * kBlockFloats);
    });
    if (rc != SRL_OK) return rc;
    const int T = 256;
    k_far_flags<<<(unsigned)((nv + T - 1) / T), T, 0, ctx->stream>>>(m->d_blocks, nv, location[0], location[1], location[2], distance * distance, keep);
    SRL_CUDA(ctx, cudaGetLastError());
    SRL_CUDA(ctx, cub::DeviceScan::ExclusiveSum(cub_tmp, tmp, keep, nidx, (int)nv, ctx->stream));
    long long n_keep = 0;
    if ((rc = scan_total(ctx, keep, nidx, nv, &n_keep)) != SRL_OK) return rc;
    ctx->launches += 2;
    if (n_keep == nv) return SRL_OK;   // nothing to evict
    const long long n_quads = nv * (kBlockFloats / 4);
    k_compact_blocks<<<(unsigned)((n_quads + T - 1) / T), T, 0, ctx->stream>>>(m->d_blocks, nv, keep, nidx, pool);
    SRL_CUDA(ctx, cudaGetLastError());
    if (n_keep > 0) SRL_CUDA(ctx, cudaMemcpyAsync(m->d_blocks, pool, (size_t)n_keep * kBlockFloats * sizeof(float), cudaMemcpyDeviceToDevice, ctx->stream));
    SRL_CUDA(ctx, cudaMemsetAsync(m->d_slots, 0, m->capacity * sizeof(Slot), ctx->stream));
    SRL_CUDA(ctx, cudaMemsetAsync(m->d_counters, 0, sizeof(long long), ctx->stream));
    if (n_keep > 0) {
        k_rebuild_slots<<<(unsigned)((n_keep + T - 1) / T), T, 0, ctx->stream>>>(m->d_slots, (unsigned)(m->capacity - 1), m->d_blocks, n_keep, m->d_counters);
        SRL_CUDA(ctx, cudaGetLastError());
    }
    SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->launches += 2;
    m->n_voxels = n_keep;
    if (n_removed) *n_removed = nv - n_keep;
    return SRL_OK;
}

int srl_map_stats(srl_map* m, int64_t* n_voxels, int64_t* n_points) {
    if (!m) return SRL_BAD_ARG;
    srl_ctx* ctx = m->ctx;
    long long np = 0;
    SRL_CUDA(ctx, cudaMemcpyAsync(&np, m->d_counters, sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream));
    SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (n_voxels) *n_voxels = m->n_voxels;
    if (n_points) *n_points = np;
    return SRL_OK;
}

int srl_map_upload(srl_map* m, const int16_t* keys, const int32_t* counts, const float* xyz, size_t n_voxels) {
    if (!m || (n_voxels && (!keys || !counts || !xyz))) return SRL_BAD_ARG;
    srl_ctx* ctx = m->ctx;
    if (int rc = check_lio_map(ctx, m)) return rc;
    if (n_voxels > m->max_voxels) return set_err(ctx, SRL_MAP_FULL, "srl_map_upload: more voxels than max_voxels");
    int rc = map_grow(m, n_voxels);
    if (rc != SRL_OK) return rc;
    rc = srl_map_clear(m);
    if (rc != SRL_OK || n_voxels == 0) return rc;
    const int cap = m->cap;
    long long total_pts = 0;
    for (size_t v = 0; v < n_voxels; ++v) {
        if (counts[v] < 0 || counts[v] > cap) return set_err(ctx, SRL_BAD_ARG, "srl_map_upload: count outside [0, cap]");
        total_pts += counts[v];
    }
    short* d_keys = nullptr;
    int *d_cnt = nullptr, *d_dup = nullptr;
    float* d_xyz = nullptr;
    rc = carve_scratch(ctx, [&](Carve& c) {
        d_keys = c.take<short>(n_voxels * 3); d_cnt = c.take<int>(n_voxels); d_xyz = c.take<float>(n_voxels * cap * 3); d_dup = c.take<int>(1);
    });
    if (rc != SRL_OK) return rc;
    SRL_CUDA(ctx, cudaMemcpyAsync(d_keys, keys, n_voxels * 3 * sizeof(short), cudaMemcpyHostToDevice, ctx->stream));
    SRL_CUDA(ctx, cudaMemcpyAsync(d_cnt, counts, n_voxels * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    SRL_CUDA(ctx, cudaMemcpyAsync(d_xyz, xyz, n_voxels * cap * 3 * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    SRL_CUDA(ctx, cudaMemsetAsync(d_dup, 0, sizeof(int), ctx->stream));
    const int T = 256;
    k_upload_slots<<<(unsigned)((n_voxels + T - 1) / T), T, 0, ctx->stream>>>(m->d_slots, (unsigned)(m->capacity - 1), m->d_blocks,
                                                                             d_keys, d_cnt, (long long)n_voxels, d_dup);
    k_upload_points<<<(unsigned)((n_voxels * cap + T - 1) / T), T, 0, ctx->stream>>>(m->d_blocks, d_xyz, (long long)n_voxels, cap);
    ctx->launches += 2;
    SRL_CUDA(ctx, cudaGetLastError());
    int dup = 0;
    SRL_CUDA(ctx, cudaMemcpyAsync(&dup, d_dup, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    SRL_CUDA(ctx, cudaMemcpyAsync(m->d_counters, &total_pts, sizeof(long long), cudaMemcpyHostToDevice, ctx->stream));
    SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (dup) return set_err(ctx, SRL_BAD_ARG, "srl_map_upload: duplicate voxel keys");
    m->n_voxels = (int64_t)n_voxels;
    return SRL_OK;
}

int srl_map_download(srl_map* m, int16_t* keys, int32_t* counts, float* xyz, size_t max_voxels, int64_t* n_voxels) {
    if (!m) return SRL_BAD_ARG;
    srl_ctx* ctx = m->ctx;
    const size_t nv = (size_t)m->n_voxels;
    if (n_voxels) *n_voxels = (int64_t)nv;
    if (nv == 0) return SRL_OK;
    if (nv > max_voxels || !keys || !counts || !xyz) return set_err(ctx, SRL_BAD_ARG, "srl_map_download: output too small");
    const int cap = m->cap;
    short* d_keys = nullptr;
    int* d_cnt = nullptr;
    float* d_xyz = nullptr;
    int rc = carve_scratch(ctx, [&](Carve& c) { d_keys = c.take<short>(nv * 3); d_cnt = c.take<int>(nv); d_xyz = c.take<float>(nv * cap * 3); });
    if (rc != SRL_OK) return rc;
    const int T = 256;
    k_download<<<(unsigned)((nv * cap + T - 1) / T), T, 0, ctx->stream>>>(m->d_blocks, m->block_pts, (long long)nv, cap, d_keys, d_cnt, d_xyz);
    ctx->launches += 1;
    SRL_CUDA(ctx, cudaGetLastError());
    SRL_CUDA(ctx, cudaMemcpyAsync(keys, d_keys, nv * 3 * sizeof(short), cudaMemcpyDeviceToHost, ctx->stream));
    SRL_CUDA(ctx, cudaMemcpyAsync(counts, d_cnt, nv * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    SRL_CUDA(ctx, cudaMemcpyAsync(xyz, d_xyz, nv * cap * 3 * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return SRL_OK;
}

// where an insert's points come from: n world points in a caller's buffer (host or device, detected per pointer), or the
// resident sweep under the pose (q, t) when sweep is set
struct InsertSource {
    const double* xyz;
    size_t n;
    srl_sweep* sweep;
    const double *q, *t, *R_il, *t_il;
};
// the registered cloud of an insert (addPointToPcl, src/lioOptimization.cpp:432,1346-1355)
struct PublishArgs {
    double translation_z;   // p_frame->p_state->translation.z()
    float* xyzi_out;        // host or device, max_out * 4 floats
    size_t max_out;
    int64_t* n_published;
};

// addPointsToMap (and with pa its published cloud) for every srl_map_insert* entry point; nothing is touched before the
// argument checks pass
static int insert_entry(srl_map* m, const InsertSource& src, double min_distance_points, int32_t min_num_points, int64_t* n_added,
                        const PublishArgs* pa) {
    srl_ctx* ctx = m->ctx;
    const size_t n = src.n;
    if (n_added) *n_added = 0;
    if (pa && pa->n_published) *pa->n_published = 0;
    if (int rc = check_lio_map(ctx, m)) return rc;
    if (pa && n && !pa->xyzi_out) return set_err(ctx, SRL_BAD_ARG, "srl_map_insert_published: xyzi_out is NULL");
    if (pa && pa->max_out < n) return set_err(ctx, SRL_BAD_ARG, "srl_map_insert_published: max_out < n (up to n points can be published)");
    if (n > 0x7fffffffULL) return set_err(ctx, SRL_BAD_ARG, "srl_map_insert: n must fit in int32");
    if (src.sweep && src.sweep->ctx != ctx) return set_err(ctx, SRL_BAD_ARG, "map and sweep belong to different contexts");
    if (n == 0) return SRL_OK;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    const int N = (int)n;
    const size_t tmp_bytes = segment_tmp_bytes(N, st);
    Staged<const double> in(src.sweep ? nullptr : src.xyz);
    Staged<float> cloud(pa ? pa->xyzi_out : nullptr);
    double* d_registered = nullptr;   // the sweep's points under the pose
    Segments s;
    float* fxyz = nullptr;
    unsigned char* pub = nullptr;     // publication: per-point flags, the selected sweep indices and their count
    unsigned int* pub_sel = nullptr;
    int* d_npub = nullptr;
    int rc = carve_scratch(ctx, [&](Carve& c) {
        if (src.sweep) d_registered = c.take<double>(n * 3);
        in.place(c, n * 3);
        s.place(c, n, tmp_bytes);
        fxyz = c.take<float>(n * 3);
        if (pa) { pub = c.take<unsigned char>(n); pub_sel = c.take<unsigned int>(n); d_npub = c.take<int>(1); cloud.place(c, n * 4); }
    });
    if (rc != SRL_OK) return rc;
    if (src.sweep) rc = srl_sweep_transform_device(ctx, src.sweep, src.q, src.t, src.R_il, src.t_il, d_registered);
    else rc = in.upload(ctx, n * 3);
    if (rc != SRL_OK) return rc;
    if (pa) SRL_CUDA(ctx, cudaMemsetAsync(pub, 0, n, st));

    const int T = 256;
    const unsigned gb = (unsigned)((n + T - 1) / T);
    k_insert_keys<<<gb, T, 0, st>>>(src.sweep ? d_registered : in.d, (long long)n, m->voxel_size, s.keys, s.idx, fxyz);
    ctx->launches += 1;
    int n_seg = 0;
    if ((rc = segment_keys(ctx, s, N, &n_seg)) != SRL_OK) return rc;
    if (n_seg == 0) return SRL_OK;
    long long total_new = 0;
    if ((rc = count_new_voxels(m, s, n_seg, min_num_points <= 0, "srl_map_insert", &total_new)) != SRL_OK) return rc;
    long long before = 0, after = 0;
    SRL_CUDA(ctx, cudaMemcpyAsync(&before, m->d_counters, sizeof(long long), cudaMemcpyDeviceToHost, st));
    if (total_new > 0) {
        k_seg_claim<<<(unsigned)((n_seg + T - 1) / T), T, 0, st>>>(m->d_slots, (unsigned)(m->capacity - 1), m->d_blocks, s.keys_sorted, s.start,
                                                                   s.d_count, s.is_new, s.new_rank, (long long)m->n_voxels, s.slot);
        ctx->launches += 1;
    }
    const unsigned gw = (unsigned)(((long long)n_seg * 32 + T - 1) / T);
    k_seg_process<<<gw, T, 0, st>>>(m->d_slots, m->d_blocks, s.keys_sorted, s.idx_sorted, fxyz, s.start, s.d_count, s.slot, (long long)n,
                                    m->voxel_size, m->cap, min_distance_points, min_num_points, m->d_counters, s.is_new, pub);
    ctx->launches += 1;
    SRL_CUDA(ctx, cudaGetLastError());
    int n_pub = 0;
    if (pa) {   // order-preserving compaction of the flagged points, then their (x, y, z, intensity)
        size_t tb = tmp_bytes;
        SRL_CUDA(ctx, cub::DeviceSelect::Flagged(s.tmp, tb, thrust::counting_iterator<unsigned int>(0), pub, pub_sel, d_npub, N, st));
        k_publish_gather<<<gb, T, 0, st>>>(fxyz, pub_sel, d_npub, pa->translation_z, cloud.d);
        SRL_CUDA(ctx, cudaGetLastError());
        SRL_CUDA(ctx, cudaMemcpyAsync(&n_pub, d_npub, sizeof(int), cudaMemcpyDeviceToHost, st));
        ctx->launches += 2;
    }
    SRL_CUDA(ctx, cudaMemcpyAsync(&after, m->d_counters, sizeof(long long), cudaMemcpyDeviceToHost, st));
    SRL_CUDA(ctx, cudaStreamSynchronize(st));
    m->n_voxels += total_new;
    if (n_added) *n_added = after - before;
    if (!pa) return SRL_OK;
    if ((rc = cloud.hand_back(ctx, (size_t)n_pub * 4)) != SRL_OK) return rc;
    if (pa->n_published) *pa->n_published = n_pub;
    return SRL_OK;
}

namespace {
struct CellKey { short x, y, z; bool operator==(const CellKey& o) const { return x == o.x && y == o.y && z == o.z; } };
struct CellHash {   // std::hash<voxel> of the reference (include/cloudMap.h:173-184)
    std::size_t operator()(const CellKey& v) const {
        const std::size_t kP1 = 73856093, kP2 = 19349669, kP3 = 83492791;
        return v.x * kP1 + v.y * kP2 + v.z * kP3;
    }
};
}  // namespace

int srl_grid_sampling(srl_ctx* ctx, const double* xyz_world, size_t n, double size, uint32_t* out, size_t* n_out) {
    if (!ctx || (n && (!xyz_world || !out)) || !n_out || !(size > 0)) return SRL_BAD_ARG;
    *n_out = 0;
    if (n == 0) return SRL_OK;
    if (n > 0x7fffffffULL) return set_err(ctx, SRL_BAD_ARG, "srl_grid_sampling: n must fit in int32");
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    size_t tmp_sort = 0, tmp_sel = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tmp_sort, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (unsigned int*)nullptr,
                                    (unsigned int*)nullptr, (int)n, 0, 50, st);
    cub::DeviceSelect::Flagged(nullptr, tmp_sel, thrust::counting_iterator<unsigned int>(0), (unsigned char*)nullptr,
                               (unsigned int*)nullptr, (int*)nullptr, (int)n, st);
    const size_t tmp_bytes = std::max(tmp_sort, tmp_sel);
    // the frame may already be in HBM (e.g. the output of srl_distort_frame_* / srl_sweep_transform_device): no H2D then, and
    // the coordinates of the kept points are gathered for the replay below
    Staged<const double> in(xyz_world);
    double* first_dev = nullptr;
    unsigned long long *ka = nullptr, *kb = nullptr;
    unsigned int *ia = nullptr, *ib = nullptr, *sel = nullptr;
    unsigned char* is_first = nullptr;
    int* d_count = nullptr;
    void* d_tmp = nullptr;
    int rc = carve_scratch(ctx, [&](Carve& c) {
        in.place(c, n * 3);
        if (in.dev) first_dev = c.take<double>(n * 3);
        ka = c.take<unsigned long long>(n); kb = c.take<unsigned long long>(n);
        ia = c.take<unsigned int>(n); ib = c.take<unsigned int>(n); sel = c.take<unsigned int>(n);
        is_first = c.take<unsigned char>(n);
        d_count = c.take<int>(1);
        d_tmp = c.take<char>(tmp_bytes);
    });
    if (rc != SRL_OK || (rc = in.upload(ctx, n * 3)) != SRL_OK) return rc;
    const double* d_xyz = in.d;
    const int T = 256;
    const unsigned gb = (unsigned)((n + T - 1) / T);
    k_cell_keys<<<gb, T, 0, st>>>(d_xyz, (long long)n, size, ka, ia);
    size_t tb = tmp_bytes;
    cub::DeviceRadixSort::SortPairs(d_tmp, tb, ka, kb, ia, ib, (int)n, 0, 50, st);
    k_first_in_cell<<<gb, T, 0, st>>>(kb, ib, (long long)n, is_first);
    tb = tmp_bytes;
    cub::DeviceSelect::Flagged(d_tmp, tb, thrust::counting_iterator<unsigned int>(0), is_first, sel, d_count, (int)n, st);
    ctx->launches += 2;
    SRL_CUDA(ctx, cudaGetLastError());
    int m = 0;
    SRL_CUDA(ctx, cudaMemcpyAsync(&m, d_count, sizeof(int), cudaMemcpyDeviceToHost, st));
    SRL_CUDA(ctx, cudaStreamSynchronize(st));
    std::vector<unsigned int> first((size_t)m);
    if (m) SRL_CUDA(ctx, cudaMemcpy(first.data(), sel, (size_t)m * sizeof(unsigned int), cudaMemcpyDeviceToHost));
    std::vector<double> first_xyz;                       // device input: the coordinates of those points come back, not the frame
    if (in.dev && m) {
        k_gather_points<<<(unsigned)((m + T - 1) / T), T, 0, st>>>(d_xyz, sel, m, first_dev);
        SRL_CUDA(ctx, cudaGetLastError());
        first_xyz.resize((size_t)m * 3);
        SRL_CUDA(ctx, cudaMemcpyAsync(first_xyz.data(), first_dev, (size_t)m * 24, cudaMemcpyDeviceToHost, st));
        SRL_CUDA(ctx, cudaStreamSynchronize(st));
    }
    // `first` = the frame indices that open a new cell, in frame order: exactly the sequence of node insertions the
    // reference's grid sees (later points of a cell only push_back into an existing node).  Replaying it through the same
    // libstdc++ container gives the reference's iteration order (src/utility.cpp:180-187).
    std::tr1::unordered_map<CellKey, unsigned int, CellHash> grid;
    for (int j = 0; j < m; ++j) {
        const unsigned int i = first[(size_t)j];
        const double* pt = in.dev ? &first_xyz[3 * (size_t)j] : &xyz_world[3 * (size_t)i];
        CellKey k;
        k.x = static_cast<short>(pt[0] / size);
        k.y = static_cast<short>(pt[1] / size);
        k.z = static_cast<short>(pt[2] / size);
        grid[k] = i;
    }
    size_t w = 0;
    for (std::tr1::unordered_map<CellKey, unsigned int, CellHash>::const_iterator it = grid.begin(); it != grid.end(); ++it) out[w++] = it->second;
    *n_out = w;
    return SRL_OK;
}


int srl_color_map_create_growable(srl_ctx* ctx, double voxel_size, int32_t max_num_points_in_voxel, size_t initial_voxels, size_t max_voxels,
                                  double min_distance_points, srl_color_map** out) {
    if (!ctx || !out || !(min_distance_points > 0)) return SRL_BAD_ARG;
    *out = nullptr;
    if (!(voxel_size > 0) || max_num_points_in_voxel < 1 || max_num_points_in_voxel > kColorMaxCap || max_voxels == 0)
        return set_err(ctx, SRL_BAD_ARG, "srl_color_map_create: voxel_size>0, 1<=max_num_points_in_voxel<=128, max_voxels>0 required");
    // up to kBlockCap points the pool keeps the LIO layout (the map also works with the LIO entry points), beyond it a block
    // holds exactly cap points
    const int block_pts = std::max(max_num_points_in_voxel, kBlockCap);
    // point ids block * block_pts + i are 32-bit and kNoIndex stays free
    if (max_voxels >= ((size_t(1) << 32) + block_pts - 1) / block_pts)
        return set_err(ctx, SRL_BAD_ARG, "srl_color_map_create: max_voxels * points per block must stay below 2^32 (32-bit point ids)");
    if (initial_voxels < 1 || initial_voxels > max_voxels)
        return set_err(ctx, SRL_BAD_ARG, "srl_color_map_create_growable: 1 <= initial_voxels <= max_voxels required");
    std::unique_ptr<srl_color_map> cm(new srl_color_map());
    cm->ctx = ctx; cm->device = ctx->device; cm->min_dist = min_distance_points;
    srl_map* vox = nullptr;
    int rc = block_pts == kBlockCap ? srl_map_create_growable(ctx, voxel_size, max_num_points_in_voxel, initial_voxels, max_voxels, &vox)
                                    : map_create(ctx, voxel_size, max_num_points_in_voxel, block_pts, initial_voxels, max_voxels, &vox);
    if (rc != SRL_OK) return rc;
    cm->vox.reset(vox);
    cm->max_rgb_points = max_voxels * (size_t)block_pts;
    cm->recent_capacity = max_voxels;
    if ((rc = vm_reserve(ctx, cm->cpts_mem, cm->max_rgb_points * sizeof(ColorPoint))) != SRL_OK ||
        (rc = vm_reserve(ctx, cm->last_visited_mem, max_voxels * sizeof(double))) != SRL_OK ||
        (rc = vm_reserve(ctx, cm->rgb_mem, cm->max_rgb_points * sizeof(unsigned int))) != SRL_OK ||
        (rc = vm_reserve(ctx, cm->recent_temp_mem, cm->recent_capacity * sizeof(unsigned long long))) != SRL_OK ||
        (rc = vm_reserve(ctx, cm->recent_mem, cm->recent_capacity * sizeof(unsigned long long))) != SRL_OK ||
        (rc = color_map_grow_voxels(cm.get(), initial_voxels)) != SRL_OK ||
        (rc = color_map_grow_rgb(cm.get(), initial_voxels * (size_t)block_pts)) != SRL_OK ||
        (rc = color_map_grow_recent(cm.get(), initial_voxels)) != SRL_OK)
        return rc;
    cm->d_cpts = reinterpret_cast<ColorPoint*>(cm->cpts_mem.base);
    cm->d_last_visited = reinterpret_cast<double*>(cm->last_visited_mem.base);
    cm->d_rgb_points = reinterpret_cast<unsigned int*>(cm->rgb_mem.base);
    cm->d_recent_temp = reinterpret_cast<unsigned long long*>(cm->recent_temp_mem.base);
    cm->d_recent = reinterpret_cast<unsigned long long*>(cm->recent_mem.base);
    cudaError_t e;
    if ((e = cm->d_counters.alloc(8)) != cudaSuccess ||
        (e = cudaMemsetAsync(cm->d_counters, 0, 8 * sizeof(long long), ctx->stream)) != cudaSuccess ||
        (e = cudaStreamSynchronize(ctx->stream)) != cudaSuccess)
        return cuda_fail(ctx, e, "srl_color_map_create");
    cm->vox->owner = cm.get();
    *out = cm.release();
    return SRL_OK;
}

int srl_color_map_create(srl_ctx* ctx, double voxel_size, int32_t max_num_points_in_voxel, size_t max_voxels, double min_distance_points,
                         srl_color_map** out) {
    return srl_color_map_create_growable(ctx, voxel_size, max_num_points_in_voxel, max_voxels, max_voxels, min_distance_points, out);
}

void srl_color_map_destroy(srl_color_map* cm) {
    if (!cm) return;
    cudaSetDevice(cm->device);
    delete cm;
}

srl_map* srl_color_map_voxels(srl_color_map* cm) { return cm ? cm->vox.get() : nullptr; }

int srl_color_map_capacity(srl_color_map* cm, size_t* committed_voxels, size_t* fine_capacity, size_t* committed_rgb_points,
                           size_t* committed_bytes) {
    if (!cm) return SRL_BAD_ARG;
    size_t vox_bytes = 0;
    srl_map_capacity(cm->vox.get(), committed_voxels, nullptr, &vox_bytes);
    if (fine_capacity) *fine_capacity = cm->fine_capacity;
    if (committed_rgb_points) *committed_rgb_points = cm->committed_rgb_points;
    if (committed_bytes)
        *committed_bytes = vox_bytes + cm->cpts_mem.mapped + cm->last_visited_mem.mapped + cm->fine_capacity * sizeof(Slot) +
                           cm->rgb_mem.mapped + cm->recent_temp_mem.mapped + cm->recent_mem.mapped;
    return SRL_OK;
}

int srl_color_map_stats(srl_color_map* cm, int64_t* n_voxels, int64_t* n_points, int64_t* n_rgb_points, int64_t* n_recent, int64_t* n_new_recent) {
    if (!cm) return SRL_BAD_ARG;
    int rc = srl_map_stats(cm->vox.get(), n_voxels, n_points);
    if (n_rgb_points) *n_rgb_points = cm->n_rgb_points;
    if (n_recent) *n_recent = cm->n_recent;
    if (n_new_recent) *n_new_recent = cm->n_new_recent;
    return rc;
}

int srl_color_map_add_points(srl_color_map* cm, const double* xyz_world, size_t n, int32_t add_point_step, double time_sweep_end,
                             double time_last_process, int32_t to_rendering, int64_t* n_stored) {
    if (!cm || (n && !xyz_world) || add_point_step < 1) return SRL_BAD_ARG;
    srl_ctx* ctx = cm->ctx;
    srl_map* m = cm->vox.get();
    cudaStream_t st = ctx->stream;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    if (n_stored) *n_stored = 0;
    // The reference appends to voxels_recent_visited_temp in every call, but only a rendering call publishes the list, and it
    // clears it first (:523-527, :544-550): what a call without rendering appends is never read.  Such a call lists nothing;
    // only its last_visited updates matter.  A rendering call lists each voxel at most once, so the list never outgrows
    // max_voxels, and number_of_new_visited_voxel is its whole length.
    int64_t n_listed = 0;
    const size_t msel = (n + (size_t)add_point_step - 1) / (size_t)add_point_step;   // points with idx % step == 0
    if (msel > 0x7fffffffULL) return set_err(ctx, SRL_BAD_ARG, "srl_color_map_add_points: too many points");
    if (msel) {
        const int M = (int)msel;
        size_t tmp_sort32 = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, tmp_sort32, (unsigned int*)nullptr, (unsigned int*)nullptr, (unsigned long long*)nullptr,
                                        (unsigned long long*)nullptr, M, 0, 32, st);
        const size_t tmp_bytes = std::max(segment_tmp_bytes(M, st), tmp_sort32);
        Staged<const double> in(xyz_world);
        Segments s;
        unsigned long long *fk_a = nullptr, *fk_b = nullptr, *seg_key = nullptr;
        unsigned int *idx_c = nullptr, *accept_id = nullptr, *seg_first = nullptr, *seg_first_sorted = nullptr, *winner = nullptr, *wrank = nullptr;
        float* fxyz = nullptr;
        int rc = carve_scratch(ctx, [&](Carve& c) {
            in.place(c, n * 3);
            s.place(c, msel, tmp_bytes);
            fk_a = c.take<unsigned long long>(msel); fk_b = c.take<unsigned long long>(msel); seg_key = c.take<unsigned long long>(msel);
            idx_c = c.take<unsigned int>(msel); accept_id = c.take<unsigned int>(msel);
            seg_first = c.take<unsigned int>(msel); seg_first_sorted = c.take<unsigned int>(msel);
            winner = c.take<unsigned int>(msel); wrank = c.take<unsigned int>(msel);
            fxyz = c.take<float>(msel * 3);
        });
        if (rc != SRL_OK || (rc = in.upload(ctx, n * 3)) != SRL_OK) return rc;
        const int T = 256;
        const unsigned gb = (unsigned)((msel + T - 1) / T);
        k_color_keys<<<gb, T, 0, st>>>(in.d, (long long)msel, add_point_step, m->voxel_size, cm->min_dist, s.keys, fk_a, s.idx, fxyz);
        SRL_CUDA(ctx, cudaMemsetAsync(accept_id, 0xff, msel * 4, st));
        SRL_CUDA(ctx, cudaMemsetAsync(winner, 0, msel * 4, st));
        ctx->launches += 1;
        int n_seg = 0;
        if ((rc = segment_keys(ctx, s, M, &n_seg)) != SRL_OK) return rc;
        if (n_seg > 0) {
            long long total_new = 0;   // min_num_points = 0 (:539): an absent voxel is new
            if ((rc = count_new_voxels(m, s, n_seg, true, "srl_color_map_add_points", &total_new)) != SRL_OK) return rc;
            const unsigned vmask = (unsigned)(m->capacity - 1);
            const unsigned gs = (unsigned)((n_seg + T - 1) / T);
            long long before = 0, after = 0;
            SRL_CUDA(ctx, cudaMemcpyAsync(&before, m->d_counters, sizeof(long long), cudaMemcpyDeviceToHost, st));
            if (total_new > 0)
                k_color_seg_claim<<<gs, T, 0, st>>>(m->d_slots, vmask, m->d_blocks, m->block_pts, s.keys_sorted, s.start, s.d_count, s.is_new,
                                                    s.new_rank, (long long)m->n_voxels, s.slot);
            k_color_seg_process<<<gs, T, 0, st>>>(m->d_slots, m->d_blocks, cm->d_cpts, cm->d_last_visited, s.keys_sorted, s.idx_sorted, fxyz,
                                                  s.start, s.d_count, s.slot, s.is_new, (long long)msel, m->cap, m->block_pts, time_sweep_end,
                                                  time_last_process, accept_id, seg_first, m->d_counters);
            m->n_voxels += total_new;
            const long long host_cnt[4] = {cm->n_rgb_points, 0, 0, 0};
            SRL_CUDA(ctx, cudaMemcpyAsync(cm->d_counters, host_cnt, sizeof(host_cnt), cudaMemcpyHostToDevice, st));
            size_t tb = tmp_bytes;
            if (to_rendering) {
                // ---- recent list: the voxels this sweep visited for the first time, in the order of their first point.
                // n_seg <= n_voxels <= max_voxels entries at most.
                k_color_seg_keys<<<gs, T, 0, st>>>(s.keys_sorted, s.start, s.d_count, seg_key);
                cub::DeviceRadixSort::SortPairs(s.tmp, tb, seg_first, seg_first_sorted, seg_key, fk_b /* reused as sorted keys */, n_seg, 0, 32, st);
                if ((rc = color_map_grow_recent(cm, (size_t)n_seg)) != SRL_OK) return rc;
                k_color_append_recent<<<gs, T, 0, st>>>(seg_first_sorted, fk_b, n_seg, cm->d_recent_temp, cm->d_counters);
                SRL_CUDA(ctx, cudaMemcpyAsync(&n_listed, cm->d_counters + 3, sizeof(long long), cudaMemcpyDeviceToHost, st));
            }
            SRL_CUDA(ctx, cudaMemcpyAsync(&after, m->d_counters, sizeof(long long), cudaMemcpyDeviceToHost, st));
            SRL_CUDA(ctx, cudaStreamSynchronize(st));
            if (n_stored) *n_stored = after - before;
            // ---- rgb_points_vec: the first accepted point of the sweep in every still-free fine cell, in sweep order.
            // Every winner is a stored point, so the list and the fine set grow for the points just stored, before any claim.
            if ((rc = color_map_grow_rgb(cm, (size_t)cm->n_rgb_points + (size_t)(after - before))) != SRL_OK) return rc;
            const unsigned fmask = (unsigned)(cm->fine_capacity - 1);
            k_color_mask_fine<<<gb, T, 0, st>>>(fk_a, accept_id, (long long)msel);
            tb = tmp_bytes;
            cub::DeviceRadixSort::SortPairs(s.tmp, tb, fk_a, fk_b, s.idx, idx_c, M, 0, 50, st);
            k_color_fine_winners<<<gb, T, 0, st>>>(cm->d_fine, fmask, fk_b, idx_c, (long long)msel, winner);
            tb = tmp_bytes;
            cub::DeviceScan::ExclusiveSum(s.tmp, tb, winner, wrank, M, st);
            long long n_win = 0;
            if ((rc = scan_total(ctx, winner, wrank, M, &n_win)) != SRL_OK) return rc;
            if ((size_t)(cm->n_rgb_points + n_win) > cm->max_rgb_points)
                return set_err(ctx, SRL_MAP_FULL, "srl_color_map_add_points: rgb point list exhausted");
            if (n_win > 0)
                k_color_emit_rgb<<<gb, T, 0, st>>>(cm->d_fine, fmask, fk_a, winner, wrank, accept_id, (long long)msel, cm->d_rgb_points, cm->d_counters,
                                                   (long long)cm->committed_rgb_points);
            SRL_CUDA(ctx, cudaGetLastError());
            cm->n_rgb_points += n_win;
            ctx->launches += 10;
        }
    }
    if (to_rendering) {                                                         // :544-550
        if (n_listed) SRL_CUDA(ctx, cudaMemcpyAsync(cm->d_recent, cm->d_recent_temp, (size_t)n_listed * 8, cudaMemcpyDeviceToDevice, st));
        cm->n_recent = cm->n_new_recent = n_listed;
    }
    SRL_CUDA(ctx, cudaStreamSynchronize(st));
    return SRL_OK;
}

int srl_color_map_render_recent(srl_color_map* cm, const srl_camera* cam, const uint8_t* image_bgr, double obs_time, int64_t* n_rendered) {
    if (!cm || !cam || !image_bgr || cam->cols < 2 || cam->rows < 2) return SRL_BAD_ARG;
    srl_ctx* ctx = cm->ctx;
    // a negative margin widens the window past the image with non-zero weights: reads outside the image (the reference's
    // behaviour is undefined there, and it only renders with margin 0.005).  !(>= 0) also refuses NaN.
    if (!(cam->fov_margin >= 0.0)) return set_err(ctx, SRL_BAD_ARG, "srl_color_map_render_recent: fov_margin must be >= 0");
    srl_map* m = cm->vox.get();
    cudaStream_t st = ctx->stream;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    if (n_rendered) *n_rendered = 0;
    const size_t nr = (size_t)cm->n_recent;
    if (nr == 0) return SRL_OK;
    const size_t img_bytes = (size_t)cam->rows * cam->cols * 3;
    size_t tmp_sort = 0, tmp_rle = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, tmp_sort, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)nr, 0, 50, st);
    cub::DeviceRunLengthEncode::Encode(nullptr, tmp_rle, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int*)nullptr, (int*)nullptr, (int)nr, st);
    const size_t tmp_bytes = std::max(tmp_sort, tmp_rle);
    Staged<const uint8_t> img(image_bgr);
    unsigned long long *sorted = nullptr, *uniq = nullptr, *d_count = nullptr;
    int *mult = nullptr, *d_nuniq = nullptr;
    void* d_tmp = nullptr;
    int rc = carve_scratch(ctx, [&](Carve& c) {
        img.place(c, img_bytes);
        sorted = c.take<unsigned long long>(nr); uniq = c.take<unsigned long long>(nr);
        mult = c.take<int>(nr); d_nuniq = c.take<int>(1); d_count = c.take<unsigned long long>(1);
        d_tmp = c.take<char>(tmp_bytes);
    });
    if (rc != SRL_OK || (rc = img.upload(ctx, img_bytes)) != SRL_OK) return rc;
    SRL_CUDA(ctx, cudaMemsetAsync(d_count, 0, 8, st));
    size_t tb = tmp_bytes;
    cub::DeviceRadixSort::SortKeys(d_tmp, tb, cm->d_recent, sorted, (int)nr, 0, 50, st);
    tb = tmp_bytes;
    cub::DeviceRunLengthEncode::Encode(d_tmp, tb, sorted, uniq, mult, d_nuniq, (int)nr, st);
    const int T = 256;
    k_color_render<<<(unsigned)((nr * 32 + T - 1) / T), T, 0, st>>>(m->d_slots, (unsigned)(m->capacity - 1), m->d_blocks, m->block_pts, cm->d_cpts, uniq, mult,
                                                               d_nuniq, camera_constants(cam), img.d, obs_time, d_count);
    SRL_CUDA(ctx, cudaGetLastError());
    unsigned long long cnt = 0;
    SRL_CUDA(ctx, cudaMemcpyAsync(&cnt, d_count, 8, cudaMemcpyDeviceToHost, st));
    SRL_CUDA(ctx, cudaStreamSynchronize(st));
    ctx->launches += 3;
    if (n_rendered) *n_rendered = (int64_t)cnt;
    return SRL_OK;
}

int srl_color_map_download_state(srl_color_map* cm, size_t max_voxels, int16_t* rgb, int16_t* n_rgb, float* cov, double* obs_dist, double* last_obs,
                                 double* last_visited) {
    if (!cm) return SRL_BAD_ARG;
    srl_ctx* ctx = cm->ctx;
    srl_map* m = cm->vox.get();
    const size_t nv = (size_t)m->n_voxels;
    if (nv == 0) return SRL_OK;
    if (nv > max_voxels || !rgb || !n_rgb || !cov || !obs_dist || !last_obs || !last_visited) return set_err(ctx, SRL_BAD_ARG, "srl_color_map_download_state: output too small");
    const int cap = m->cap;
    const size_t e = nv * (size_t)cap;
    short *d_rgb = nullptr, *d_n = nullptr;
    float* d_cov = nullptr;
    double *d_od = nullptr, *d_lo = nullptr, *d_lv = nullptr;
    int rc = carve_scratch(ctx, [&](Carve& c) {
        d_rgb = c.take<short>(e * 3); d_n = c.take<short>(e); d_cov = c.take<float>(e * 3);
        d_od = c.take<double>(e); d_lo = c.take<double>(e); d_lv = c.take<double>(nv);
    });
    if (rc != SRL_OK) return rc;
    const int T = 256;
    k_color_download<<<(unsigned)((e + T - 1) / T), T, 0, ctx->stream>>>(cm->d_cpts, m->d_blocks, cm->d_last_visited, m->block_pts, (long long)nv, cap, d_rgb, d_n, d_cov,
                                                                         d_od, d_lo, d_lv);
    SRL_CUDA(ctx, cudaGetLastError());
    SRL_CUDA(ctx, cudaMemcpyAsync(rgb, d_rgb, e * 6, cudaMemcpyDeviceToHost, ctx->stream));
    SRL_CUDA(ctx, cudaMemcpyAsync(n_rgb, d_n, e * 2, cudaMemcpyDeviceToHost, ctx->stream));
    SRL_CUDA(ctx, cudaMemcpyAsync(cov, d_cov, e * 12, cudaMemcpyDeviceToHost, ctx->stream));
    SRL_CUDA(ctx, cudaMemcpyAsync(obs_dist, d_od, e * 8, cudaMemcpyDeviceToHost, ctx->stream));
    SRL_CUDA(ctx, cudaMemcpyAsync(last_obs, d_lo, e * 8, cudaMemcpyDeviceToHost, ctx->stream));
    SRL_CUDA(ctx, cudaMemcpyAsync(last_visited, d_lv, nv * 8, cudaMemcpyDeviceToHost, ctx->stream));
    SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return SRL_OK;
}

int srl_color_map_download_lists(srl_color_map* cm, int16_t* rgb_points /* n_rgb_points * 4 */, int16_t* recent /* n_recent * 3 */) {
    if (!cm) return SRL_BAD_ARG;
    srl_ctx* ctx = cm->ctx;
    srl_map* m = cm->vox.get();
    std::vector<unsigned long long> keys(recent ? (size_t)cm->n_recent : 0);
    if (cm->n_rgb_points && rgb_points) {
        const size_t n = (size_t)cm->n_rgb_points;
        short* d_out = nullptr;
        int rc = carve_scratch(ctx, [&](Carve& c) { d_out = c.take<short>(n * 4); });
        if (rc != SRL_OK) return rc;
        const int T = 256;
        k_color_rgb_ids<<<(unsigned)((n + T - 1) / T), T, 0, ctx->stream>>>(cm->d_rgb_points, (long long)n, m->d_blocks, m->block_pts, d_out);
        SRL_CUDA(ctx, cudaGetLastError());
        SRL_CUDA(ctx, cudaMemcpyAsync(rgb_points, d_out, n * 8, cudaMemcpyDeviceToHost, ctx->stream));
    }
    if (!keys.empty()) SRL_CUDA(ctx, cudaMemcpyAsync(keys.data(), cm->d_recent, keys.size() * 8, cudaMemcpyDeviceToHost, ctx->stream));
    SRL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (size_t i = 0; i < keys.size(); ++i) { short x, y, z; unpack_key(keys[i], x, y, z); recent[3 * i] = x; recent[3 * i + 1] = y; recent[3 * i + 2] = z; }
    return SRL_OK;
}

int srl_map_insert(srl_map* m, const double* xyz_world, size_t n, double min_distance_points, int32_t min_num_points,
                   int64_t* n_added) {
    if (!m || (n && !xyz_world)) return SRL_BAD_ARG;
    return insert_entry(m, InsertSource{xyz_world, n, nullptr}, min_distance_points, min_num_points, n_added, nullptr);
}

int srl_map_insert_device(srl_map* m, const double* d_xyz_world, size_t n, double min_distance_points, int32_t min_num_points,
                          int64_t* n_added) {
    return srl_map_insert(m, d_xyz_world, n, min_distance_points, min_num_points, n_added);
}

int srl_map_insert_sweep(srl_map* m, srl_sweep* sw, const double q[4], const double t[3], const double R_il[9], const double t_il[3],
                         double min_distance_points, int32_t min_num_points, int64_t* n_added) {
    if (!m || !sw || !q || !t || !R_il || !t_il) return SRL_BAD_ARG;
    return insert_entry(m, InsertSource{nullptr, sw->n, sw, q, t, R_il, t_il}, min_distance_points, min_num_points, n_added, nullptr);
}

int srl_map_insert_published(srl_map* m, const double* xyz_world, size_t n, double min_distance_points, int32_t min_num_points,
                             double translation_z, float* xyzi_out, size_t max_out, int64_t* n_added, int64_t* n_published) {
    if (!m || (n && !xyz_world)) return SRL_BAD_ARG;
    const PublishArgs pa{translation_z, xyzi_out, max_out, n_published};
    return insert_entry(m, InsertSource{xyz_world, n, nullptr}, min_distance_points, min_num_points, n_added, &pa);
}

int srl_map_insert_sweep_published(srl_map* m, srl_sweep* sw, const double q[4], const double t[3], const double R_il[9],
                                   const double t_il[3], double min_distance_points, int32_t min_num_points, float* xyzi_out,
                                   size_t max_out, int64_t* n_added, int64_t* n_published) {
    if (!m || !sw || !q || !t || !R_il || !t_il) return SRL_BAD_ARG;
    const PublishArgs pa{t[2], xyzi_out, max_out, n_published};
    return insert_entry(m, InsertSource{nullptr, sw->n, sw, q, t, R_il, t_il}, min_distance_points, min_num_points, n_added, &pa);
}

int srl_color_map_export(srl_color_map* cm, int32_t min_views, int32_t order, float* xyz, uint8_t* rgb, size_t max_points, int64_t* n_out) {
    if (!cm || !n_out) return SRL_BAD_ARG;
    *n_out = 0;
    srl_ctx* ctx = cm->ctx;
    if (order != 0 && order != 1) return set_err(ctx, SRL_BAD_ARG, "srl_color_map_export: order is 0 (publish) or 1 (save)");
    if ((xyz == nullptr) != (rgb == nullptr)) return set_err(ctx, SRL_BAD_ARG, "srl_color_map_export: xyz and rgb are both NULL (count) or both set");
    const long long n = cm->n_rgb_points;
    const long long m = order ? std::max(n - 1, 0LL) : n;   // saveColorPoints stops before index 0 (:1398)
    if (m == 0) return SRL_OK;
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    srl_map* vm = cm->vox.get();
    const long long chunk = std::min<long long>(m, 1ll << 22);
    size_t tmp_sel = 0;
    cub::DeviceSelect::Flagged(nullptr, tmp_sel, thrust::counting_iterator<unsigned int>(0), (unsigned char*)nullptr, (unsigned int*)nullptr,
                               (int*)nullptr, (int)chunk, st);
    Staged<float> out_xyz(xyz);
    Staged<uint8_t> out_rgb(rgb);
    unsigned char* flags = nullptr;
    unsigned long long* d_count = nullptr;
    int* d_nsel = nullptr;
    unsigned int* sel = nullptr;
    void* d_tmp = nullptr;
    int rc = carve_scratch(ctx, [&](Carve& c) {
        flags = c.take<unsigned char>((size_t)m);
        d_count = c.take<unsigned long long>(1); d_nsel = c.take<int>(1);
        sel = c.take<unsigned int>((size_t)chunk);
        d_tmp = c.take<char>(tmp_sel);
        out_xyz.place(c, (size_t)chunk * 3); out_rgb.place(c, (size_t)chunk * 3);   // one chunk of a host output at a time
    });
    if (rc != SRL_OK) return rc;
    const int T = 256;
    SRL_CUDA(ctx, cudaMemsetAsync(d_count, 0, 8, st));
    k_color_export_flags<<<(unsigned)((m + T - 1) / T), T, 0, st>>>(cm->d_rgb_points, cm->d_cpts, m, n, order, min_views, flags, d_count);
    SRL_CUDA(ctx, cudaGetLastError());
    unsigned long long total = 0;
    SRL_CUDA(ctx, cudaMemcpyAsync(&total, d_count, 8, cudaMemcpyDeviceToHost, st));
    SRL_CUDA(ctx, cudaStreamSynchronize(st));
    ctx->launches += 1;
    *n_out = (int64_t)total;
    if (!xyz || total == 0) return SRL_OK;
    if (total > max_points) return set_err(ctx, SRL_BAD_ARG, "srl_color_map_export: max_points is smaller than the number of points (count with NULL outputs first)");
    // one chunk of positions at a time: compact its flags (sweep of the list in output order), gather, hand over
    size_t off = 0;
    for (long long base = 0; base < m; base += chunk) {
        const long long len = std::min(chunk, m - base);
        size_t tb = tmp_sel;
        SRL_CUDA(ctx, cub::DeviceSelect::Flagged(d_tmp, tb, thrust::counting_iterator<unsigned int>(0), flags + base, sel, d_nsel, (int)len, st));
        float* dx = out_xyz.dev ? xyz + 3 * off : out_xyz.d;
        unsigned char* dr = out_rgb.dev ? rgb + 3 * off : out_rgb.d;
        k_color_export_gather<<<(unsigned)((len + T - 1) / T), T, 0, st>>>(cm->d_rgb_points, vm->d_blocks, vm->block_pts, cm->d_cpts, sel, d_nsel,
                                                                          base, n, order, dx, dr);
        SRL_CUDA(ctx, cudaGetLastError());
        int k = 0;
        SRL_CUDA(ctx, cudaMemcpyAsync(&k, d_nsel, sizeof(int), cudaMemcpyDeviceToHost, st));
        SRL_CUDA(ctx, cudaStreamSynchronize(st));
        ctx->launches += 2;
        if ((rc = out_xyz.hand_back(ctx, (size_t)k * 3, 3 * off)) != SRL_OK || (rc = out_rgb.hand_back(ctx, (size_t)k * 3, 3 * off)) != SRL_OK)
            return rc;
        off += (size_t)k;
    }
    return SRL_OK;
}

}  // extern "C"

// ---- selectPointsForProjection / the tracker's gather ------------------------------------------------------------------
// The cell coordinates of one image axis: if2dPointsAvailable accepts fov * size + 1 <= x and ceil(x) < (1 - fov) * size, so
// |x| <= a = max(|lo|, |hi|), and the cell std::round(x / d) * d lies within 2a + 1 of zero (it is 0, or |x / d| >= 1/2 and
// |round(x / d)| <= 2 |x / d|).  The axis is offset by -b (b = ceil(2a) + 2) and takes `bits` bits, with 2^bits > 2b + 1 so that
// an all-ones field never comes from a cell.  False when b does not fit an int or x / d can overflow.
bool srl::cell_axis(double fov, int size, double min_dis, int& offset, int& bits) {
    const double lo = fov * (double)size + 1.0, hi = (1.0 - fov) * (double)size;
    const double a = std::max(std::fabs(lo), std::fabs(hi));
    if (!(a < 1e9) || !(a / min_dis < 1e300)) return false;
    const double b = std::ceil(2.0 * a) + 2.0;
    if (!(b <= 2147483647.0)) return false;
    offset = -(int)b;
    const unsigned long long span = 2ull * (unsigned long long)b + 2ull;
    bits = 0;
    while ((1ull << bits) < span) ++bits;
    return true;
}

extern "C" {

int srl_color_map_select_for_projection(srl_color_map* cm, const srl_camera* cam, const srl_projection_params* prm, uint32_t* point_ids,
                                        float* xyz, float* uv, size_t max_points, int64_t* n_out) {
    if (!cm || !n_out) return SRL_BAD_ARG;
    *n_out = 0;
    srl_ctx* ctx = cm->ctx;
    if (!cam || !prm) return set_err(ctx, SRL_BAD_ARG, "srl_color_map_select_for_projection: camera and parameters are required");
    if (cam->cols < 2 || cam->rows < 2) return set_err(ctx, SRL_BAD_ARG, "srl_color_map_select_for_projection: the image needs cols >= 2 and rows >= 2");
    if (!(std::isfinite(prm->minimum_dis) && prm->minimum_dis > 0))
        return set_err(ctx, SRL_BAD_ARG, "srl_color_map_select_for_projection: minimum_dis must be finite and > 0");
    if (prm->skip_step < 1) return set_err(ctx, SRL_BAD_ARG, "srl_color_map_select_for_projection: skip_step must be >= 1");
    int u0 = 0, v0 = 0, bits_u = 0, bits_v = 0;
    if (!std::isfinite(cam->fov_margin) || !cell_axis(cam->fov_margin, cam->cols, prm->minimum_dis, u0, bits_u) ||
        !cell_axis(cam->fov_margin, cam->rows, prm->minimum_dis, v0, bits_v))
        return set_err(ctx, SRL_BAD_ARG, "srl_color_map_select_for_projection: the cell coordinates of the FoV window do not fit an int");
    const int end_bit = bits_u + bits_v;
    const unsigned long long none = end_bit >= 64 ? ~0ull : (1ull << end_bit) - 1ull;
    // :74-89: the last point of every recent voxel, or rgb_points_vec when use_all_points is set or the recent list is empty
    const bool recent = !prm->use_all_points && cm->n_recent > 0;
    const long long total = recent ? cm->n_recent : cm->n_rgb_points;
    const long long m = (total + prm->skip_step - 1) / prm->skip_step;
    if (m == 0) return SRL_OK;
    if (m > 0x7fffffffLL) return set_err(ctx, SRL_BAD_ARG, "srl_color_map_select_for_projection: more than 2^31 - 1 candidates");
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    srl_map* vm = cm->vox.get();
    const int n = (int)m;
    size_t tmp_sort = 0, tmp_scan = 0, tmp_red = 0, tmp_sel = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tmp_sort, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (unsigned int*)nullptr,
                                    (unsigned int*)nullptr, n, 0, std::max(end_bit, 1), st);
    cub::DeviceScan::ExclusiveScanByKey(nullptr, tmp_scan, (unsigned long long*)nullptr, (float*)nullptr, (float*)nullptr, ProjMinF(),
                                        std::numeric_limits<float>::infinity(), n, ProjKeyEq(), st);
    cub::DeviceReduce::ReduceByKey(nullptr, tmp_red, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int*)nullptr, (int*)nullptr,
                                   (int*)nullptr, ProjMaxI(), n, st);
    cub::DeviceSelect::Flagged(nullptr, tmp_sel, thrust::counting_iterator<unsigned int>(0), (unsigned char*)nullptr, (unsigned int*)nullptr,
                               (int*)nullptr, n, st);
    const size_t tmp_bytes = std::max(std::max(tmp_sort, tmp_scan), std::max(tmp_red, tmp_sel));
    const size_t M = (size_t)m;
    Staged<unsigned int> o_ids(point_ids);
    Staged<float> o_xyz(xyz), o_uv(uv);
    unsigned long long *key_a = nullptr, *key_b = nullptr, *cells = nullptr;
    unsigned int *ord_a = nullptr, *ord_b = nullptr, *cand_id = nullptr, *sel = nullptr;
    double* depth = nullptr;
    float2* cand_uv = nullptr;
    float *fd = nullptr, *pre = nullptr;
    int *taker = nullptr, *last_taker = nullptr, *d_ncells = nullptr, *d_nsel = nullptr;
    unsigned char* win = nullptr;
    void* d_tmp = nullptr;
    int rc = carve_scratch(ctx, [&](Carve& c) {
        key_a = c.take<unsigned long long>(M); key_b = c.take<unsigned long long>(M); cells = c.take<unsigned long long>(M);
        ord_a = c.take<unsigned int>(M); ord_b = c.take<unsigned int>(M);
        depth = c.take<double>(M); cand_id = c.take<unsigned int>(M); cand_uv = c.take<float2>(M);
        fd = c.take<float>(M); pre = c.take<float>(M);
        taker = c.take<int>(M); last_taker = c.take<int>(M);
        win = c.take<unsigned char>(M); sel = c.take<unsigned int>(M);
        d_ncells = c.take<int>(1); d_nsel = c.take<int>(1);
        d_tmp = c.take<char>(tmp_bytes);
        o_ids.place(c, M); o_xyz.place(c, M * 3); o_uv.place(c, M * 2);
    });
    if (rc != SRL_OK) return rc;
    const int T = 256;
    const unsigned gb = (unsigned)((m + T - 1) / T);
    SRL_CUDA(ctx, cudaMemsetAsync(win, 0, M, st));
    k_proj_candidates<<<gb, T, 0, st>>>(vm->d_slots, (unsigned)(vm->capacity - 1), vm->d_blocks, vm->block_pts, recent ? cm->d_recent : nullptr,
                                        cm->d_rgb_points, m, prm->skip_step, camera_constants(cam), prm->minimum_dis, prm->minimum_depth,
                                        prm->maximum_depth, u0, v0, bits_v, none, key_a, ord_a, cand_id, depth, cand_uv);
    SRL_CUDA(ctx, cudaGetLastError());
    size_t tb = tmp_bytes;
    SRL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(d_tmp, tb, key_a, key_b, ord_a, ord_b, n, 0, std::max(end_bit, 1), st));   // stable
    k_proj_float_depths<<<gb, T, 0, st>>>(ord_b, depth, m, fd);
    SRL_CUDA(ctx, cudaGetLastError());
    tb = tmp_bytes;
    SRL_CUDA(ctx, cub::DeviceScan::ExclusiveScanByKey(d_tmp, tb, key_b, fd, pre, ProjMinF(), std::numeric_limits<float>::infinity(), n, ProjKeyEq(), st));
    k_proj_takers<<<gb, T, 0, st>>>(key_b, ord_b, depth, pre, m, none, taker);
    SRL_CUDA(ctx, cudaGetLastError());
    tb = tmp_bytes;
    SRL_CUDA(ctx, cub::DeviceReduce::ReduceByKey(d_tmp, tb, key_b, cells, taker, last_taker, d_ncells, ProjMaxI(), n, st));
    k_proj_mark_winners<<<gb, T, 0, st>>>(last_taker, d_ncells, ord_b, win);
    SRL_CUDA(ctx, cudaGetLastError());
    tb = tmp_bytes;
    SRL_CUDA(ctx, cub::DeviceSelect::Flagged(d_tmp, tb, thrust::counting_iterator<unsigned int>(0), win, sel, d_nsel, n, st));
    int k = 0;
    SRL_CUDA(ctx, cudaMemcpyAsync(&k, d_nsel, sizeof(int), cudaMemcpyDeviceToHost, st));
    SRL_CUDA(ctx, cudaStreamSynchronize(st));
    ctx->launches += 8;
    *n_out = k;
    if ((!point_ids && !xyz && !uv) || k == 0) return SRL_OK;
    if ((size_t)k > max_points) return set_err(ctx, SRL_BAD_ARG, "srl_color_map_select_for_projection: max_points is smaller than the number of points (count with NULL outputs first)");
    k_proj_gather<<<(unsigned)((k + T - 1) / T), T, 0, st>>>(sel, k, cand_id, cand_uv, vm->d_blocks, vm->block_pts, o_ids.d, o_xyz.d, o_uv.d);
    SRL_CUDA(ctx, cudaGetLastError());
    ctx->launches += 1;
    if ((rc = o_ids.hand_back(ctx, (size_t)k)) != SRL_OK || (rc = o_xyz.hand_back(ctx, (size_t)k * 3)) != SRL_OK ||
        (rc = o_uv.hand_back(ctx, (size_t)k * 2)) != SRL_OK)
        return rc;
    SRL_CUDA(ctx, cudaStreamSynchronize(st));
    return SRL_OK;
}

int srl_color_map_gather_points(srl_color_map* cm, const uint32_t* point_ids, size_t n, float* xyz, int16_t* rgb, int16_t* n_rgb, float* cov,
                                int16_t* key_index) {
    if (!cm) return SRL_BAD_ARG;
    srl_ctx* ctx = cm->ctx;
    if (n && !point_ids) return set_err(ctx, SRL_BAD_ARG, "srl_color_map_gather_points: point_ids is NULL");
    if (n == 0) return SRL_OK;
    if (n > 0x7fffffffULL) return set_err(ctx, SRL_BAD_ARG, "srl_color_map_gather_points: n must fit in int32");
    SRL_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    srl_map* vm = cm->vox.get();
    Staged<const unsigned int> ids(point_ids);
    Staged<float> o_xyz(xyz), o_cov(cov);
    Staged<short> o_rgb(rgb), o_nr(n_rgb), o_ki(key_index);
    unsigned long long* d_bad = nullptr;
    int rc = carve_scratch(ctx, [&](Carve& c) {
        ids.place(c, n);
        d_bad = c.take<unsigned long long>(1);
        o_xyz.place(c, n * 3); o_rgb.place(c, n * 3); o_nr.place(c, n); o_cov.place(c, n * 3); o_ki.place(c, n * 4);
    });
    if (rc != SRL_OK || (rc = ids.upload(ctx, n)) != SRL_OK) return rc;
    const int T = 256;
    const unsigned gb = (unsigned)((n + T - 1) / T);
    SRL_CUDA(ctx, cudaMemsetAsync(d_bad, 0, 8, st));
    k_color_check_ids<<<gb, T, 0, st>>>(ids.d, (long long)n, vm->d_blocks, vm->block_pts, (long long)vm->n_voxels, d_bad);
    SRL_CUDA(ctx, cudaGetLastError());
    unsigned long long bad = 0;
    SRL_CUDA(ctx, cudaMemcpyAsync(&bad, d_bad, 8, cudaMemcpyDeviceToHost, st));
    SRL_CUDA(ctx, cudaStreamSynchronize(st));
    ctx->launches += 1;
    if (bad) return set_err(ctx, SRL_BAD_ARG, "srl_color_map_gather_points: " + std::to_string(bad) + " point id(s) name no stored point");
    if (xyz || rgb || n_rgb || cov) {
        k_color_gather<<<gb, T, 0, st>>>(ids.d, (long long)n, vm->d_blocks, vm->block_pts, cm->d_cpts, o_xyz.d, o_rgb.d, o_nr.d, o_cov.d);
        SRL_CUDA(ctx, cudaGetLastError());
        ctx->launches += 1;
    }
    if (key_index) {
        k_color_rgb_ids<<<gb, T, 0, st>>>(ids.d, (long long)n, vm->d_blocks, vm->block_pts, o_ki.d);
        SRL_CUDA(ctx, cudaGetLastError());
        ctx->launches += 1;
    }
    if ((rc = o_xyz.hand_back(ctx, n * 3)) != SRL_OK || (rc = o_rgb.hand_back(ctx, n * 3)) != SRL_OK || (rc = o_nr.hand_back(ctx, n)) != SRL_OK ||
        (rc = o_cov.hand_back(ctx, n * 3)) != SRL_OK || (rc = o_ki.hand_back(ctx, n * 4)) != SRL_OK)
        return rc;
    SRL_CUDA(ctx, cudaStreamSynchronize(st));
    return SRL_OK;
}

}  // extern "C"
