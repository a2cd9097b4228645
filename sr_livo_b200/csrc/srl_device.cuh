// srl_device.cuh — HBM layout of the voxel map and shared device helpers.
//
// Layout (GPU-first, not a translation of tsl::robin_map<voxel, voxelBlock>, include/cloudMap.h:171):
//   slot table : open addressing, power-of-two capacity >= 2 x committed voxels (load <= 0.5), 16-byte slots
//                { u64 key (x,y,z as u16 | valid bit 48), u32 block, u32 count } -> one LDG.128 per probe.
//   block pool : one 320-byte block per voxel = 20 x float4 (x, y, z, w): a point is ONE 16-byte load for a
//                thread that scans candidates (k1_fast), and 20 lanes x 16 B = 320 contiguous bytes for a warp
//                (k1_assoc).  The unused w lanes carry the block's metadata: pt[0].w / pt[1].w = key bits,
//                pt[2].w = count.  Points keep the reference's insertion order, so index i in the block == index
//                in voxelBlock::points.
// Only key -> block *content* has to match the reference; probe order / hash are our own.
#pragma once

#include <cuda_runtime.h>
#include <cstdint>

namespace srl {

constexpr int kBlockFloats = 80;   // 320 B
constexpr int kBlockCap = 20;      // max_num_points_in_voxel supported by the block layout (all reference configs use 20)
constexpr int kMetaKeyLo = 0 * 4 + 3, kMetaKeyHi = 1 * 4 + 3, kMetaCount = 2 * 4 + 3;   // float index of the w lanes used

struct ColorPoint {            // colour state of one stored point of a colour map (rgbPoint minus position), index = block * block_pts + i
    short rgb[3]; short n_rgb;
    float cov[3]; float pad;
    double obs_dist, last_obs;
};

struct __align__(16) Slot {
    unsigned long long key;   // 0 = empty
    unsigned int block;
    unsigned int count;
};

struct MapView {               // the map as the pass kernels address it
    Slot* slots;
    unsigned int mask;        // capacity - 1
    float* blocks;            // n_blocks * kBlockFloats floats
};

__host__ __device__ __forceinline__ unsigned long long pack_key(int x, int y, int z) {
    return (unsigned long long)(unsigned short)x | ((unsigned long long)(unsigned short)y << 16) |
           ((unsigned long long)(unsigned short)z << 32) | (1ull << 48);
}
__host__ __device__ __forceinline__ void unpack_key(unsigned long long k, short& x, short& y, short& z) {
    x = (short)(k & 0xffff); y = (short)((k >> 16) & 0xffff); z = (short)((k >> 32) & 0xffff);
}
__host__ __device__ __forceinline__ unsigned int hash_key(int x, int y, int z) {
    unsigned int h = (unsigned int)x * 73856093u ^ (unsigned int)y * 19349669u ^ (unsigned int)z * 83492791u;
    h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13;
    return h;
}

// The order in which the pass kernels visit the voxels around a keypoint's voxel: first the 27 offsets with |.|inf <= 1,
// then the other 98 of the 5x5x5 cube, each part by squared norm, then x, y, z ascending.  N = 125 is k1_assoc's table
// (c_off), N = 27 the nb <= 1 table of k1_fast / k1_scan / k1_fit (c_off_fast).  Entry i is (x, y, z, 0) at [4i, 4i + 4).
template <int N>
struct VoxelOffsets {
    signed char v[4 * N];
    __host__ __device__ constexpr signed char operator[](int i) const { return v[i]; }
};
template <int N>
constexpr VoxelOffsets<N> voxel_offsets() {
    VoxelOffsets<N> t{};
    int n = 0;
    for (int outer = 0; outer <= 1; ++outer)
        for (int d2 = 0; d2 <= 12; ++d2)
            for (int x = -2; x <= 2; ++x)
                for (int y = -2; y <= 2; ++y)
                    for (int z = -2; z <= 2; ++z) {
                        const bool inner = x >= -1 && x <= 1 && y >= -1 && y <= 1 && z >= -1 && z <= 1;
                        if (inner == (outer == 1) || x * x + y * y + z * z != d2 || n == N) continue;
                        t.v[4 * n] = (signed char)x; t.v[4 * n + 1] = (signed char)y; t.v[4 * n + 2] = (signed char)z;
                        ++n;
                    }
    return t;
}

#if defined(__CUDACC__)
// read-only probe (query kernels): linear probing, one 16-byte load per step
__device__ __forceinline__ bool map_find(const Slot* __restrict__ slots, unsigned int mask, int x, int y, int z,
                                         unsigned int& block, unsigned int& count) {
    const unsigned long long key = pack_key(x, y, z);
    unsigned int idx = hash_key(x, y, z) & mask;
    for (;;) {
        const uint4 s = __ldg(reinterpret_cast<const uint4*>(slots + idx));
        const unsigned long long k = (unsigned long long)s.x | ((unsigned long long)s.y << 32);
        if (k == key) { block = s.z; count = s.w; return true; }
        if (k == 0ull) return false;
        idx = (idx + 1) & mask;
    }
}
#endif

}  // namespace srl
