// fls_ivox.cuh — device-side incremental-voxel map (iVox) and its bounded 5-NN lookup.
//
// Replaces IVoxMap (include/ivox_map/ivox_map.h:16-74, src/ivox_map/ivox_map.cpp upstream):
// the unordered_map + std::list LRU + per-voxel std::vector becomes
//   * one voxel-contiguous SoA float4 point array (points of a voxel adjacent, voxels in Morton order,
//     insertion order preserved inside a voxel) + an open-addressing table of 16-byte slots
//     {packed key, start, count}, load factor <= 0.5  (the "occupied" table), and
//   * per-centre STENCIL LISTS: for every voxel whose stencil touches an occupied voxel, the candidate
//     sequence GetClosestPoint would visit (stencil order, then insertion order) stored contiguously, with a
//     second table {centre key -> list start, list length}.  One probe + one streaming scan per query.
#pragma once
#include "fls_common.cuh"

namespace fls {

struct IvoxView {
    const float4* __restrict__ pts;    // voxel-contiguous points
    const HashSlot* __restrict__ tab;  // occupied-voxel table
    unsigned mask;
    float inv_res;
    float max_range2;
    int n_stencil;
    const float4* __restrict__ lists;   // stencil lists (may be null)
    const HashSlot* __restrict__ ctab;  // centre table
    unsigned cmask;
    unsigned fast_knn;  // 1: every stencil candidate is provably within max_range (range test and exact rounding not needed up front)
};

// stencil offsets in the reference's order (src/ivox_map/ivox_map.cpp:43-66 upstream)
static __device__ __constant__ signed char c_stencil[27][4] = {
    {0, 0, 0, 0},  {-1, 0, 0, 0}, {1, 0, 0, 0},  {0, 1, 0, 0},   {0, -1, 0, 0}, {0, 0, -1, 0},  {0, 0, 1, 0},  {1, 1, 0, 0},  {-1, 1, 0, 0},
    {1, -1, 0, 0}, {-1, -1, 0, 0}, {1, 0, 1, 0}, {-1, 0, 1, 0},  {1, 0, -1, 0}, {-1, 0, -1, 0}, {0, 1, 1, 0},  {0, -1, 1, 0}, {0, 1, -1, 0},
    {0, -1, -1, 0}, {1, 1, 1, 0}, {-1, 1, 1, 0}, {1, -1, 1, 0},  {1, 1, -1, 0}, {-1, -1, 1, 0}, {-1, 1, -1, 0}, {1, -1, -1, 0}, {-1, -1, -1, 0}};

// IVoxMap::Pos2Grid (ivox_map.cpp:145-147 upstream): round(p * inv_res), fp32 product, half away from zero
__device__ __forceinline__ int ivox_coord(float v, float inv_res) { return (int)roundf(__fmul_rn(v, inv_res)); }
// uniform search grid (bounded exact NN): floor(p * inv_cell)
__device__ __forceinline__ int floor_coord(float v, float inv_res) { return (int)floorf(__fmul_rn(v, inv_res)); }

__host__ __device__ __forceinline__ unsigned compact21(unsigned long long x) {  // inverse of spread21
    x &= 0x1249249249249249ULL;
    x = (x | x >> 2) & 0x10c30c30c30c30c3ULL;
    x = (x | x >> 4) & 0x100f00f00f00f00fULL;
    x = (x | x >> 8) & 0x1f0000ff0000ffULL;
    x = (x | x >> 16) & 0x1f00000000ffffULL;
    x = (x | x >> 32) & 0x1fffffULL;
    return (unsigned)x;
}
__host__ __device__ __forceinline__ void morton_decode(unsigned long long m, int& x, int& y, int& z) {
    x = (int)compact21(m) - (1 << 20);
    y = (int)compact21(m >> 1) - (1 << 20);
    z = (int)compact21(m >> 2) - (1 << 20);
}

}  // namespace fls
