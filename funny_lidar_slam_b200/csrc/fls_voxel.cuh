// fls_voxel.cuh — the arithmetic of pcl::VoxelGrid<PointXYZI>::filter (PCL 1.10, as wrapped by VoxelGridCloud,
// include/common/pointcloud_utility.h:216-224,263-271 upstream; SURVEY.md §8c), shared by the single-cloud filter
// (fls_voxelgrid.cu) and the segmented keyframe pass (fls_keyframes.cu) so both round exactly alike:
//   bounding box -> dx*dy*dz > INT_MAX: input unchanged -> cell = floor(x*inv) - min_b (fp32) -> linear id
//   -> one centroid per occupied cell: fp32 running sums in input order, divided by float(n).
#pragma once
#include <cuda_runtime.h>
#include <math.h>

#include <cstring>

namespace fls {

// order-preserving float <-> uint encoding so a bounding box can be reduced with integer atomicMin / atomicMax
__device__ __forceinline__ unsigned f2ord(float f) {
    const unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float ord2f(unsigned o) {
    const unsigned u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float f;
    memcpy(&f, &u, 4);
    return f;
#endif
}

// bounding box in the f2ord encoding; {0xffffffff, 0} is the empty box
struct MinMaxOrd {
    unsigned mn[3], mx[3];
};

__host__ __device__ __forceinline__ float vg_mul(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}

// Grid parameters of one cloud from its bounding box and inv = 1.0f / leaf.  `overflow`: PCL's "Leaf size is too small"
// (dx*dy*dz > INT_MAX) — the filter returns its input unchanged.
struct VgParams {
    int minb[3];
    int divb[3];
    int mul1, mul2;
    bool overflow;
};
__host__ __device__ __forceinline__ VgParams vg_params(const float mn[3], const float mx[3], float inv) {
    VgParams p;
    long long d[3];
    for (int a = 0; a < 3; ++a) {
        d[a] = (long long)vg_mul(mx[a] - mn[a], inv) + 1;
        p.minb[a] = (int)floorf(vg_mul(mn[a], inv));
        p.divb[a] = (int)floorf(vg_mul(mx[a], inv)) - p.minb[a] + 1;
    }
    p.overflow = d[0] * d[1] * d[2] > 2147483647LL;
    p.mul1 = p.divb[0];
    p.mul2 = p.overflow ? 0 : p.divb[0] * p.divb[1];
    return p;
}
__host__ __device__ __forceinline__ VgParams vg_params(const MinMaxOrd& o, float inv) {
    float mn[3], mx[3];
    for (int a = 0; a < 3; ++a) {
        mn[a] = ord2f(o.mn[a]);
        mx[a] = ord2f(o.mx[a]);
    }
    return vg_params(mn, mx, inv);
}

// linear cell id i + j*dx + k*dx*dy with i = floor(x*inv) - min_b[0] in fp32 (and so on)
__device__ __forceinline__ unsigned vg_cell_id(const float4& p, float inv, const VgParams& g) {
    const int i0 = (int)(floorf(__fmul_rn(p.x, inv)) - (float)g.minb[0]);
    const int i1 = (int)(floorf(__fmul_rn(p.y, inv)) - (float)g.minb[1]);
    const int i2 = (int)(floorf(__fmul_rn(p.z, inv)) - (float)g.minb[2]);
    return (unsigned)(i0 + i1 * g.mul1 + i2 * g.mul2);
}

// CentroidPoint accumulators of PCL: sequential fp32 sums of xyz and intensity, divided by float(n)
struct VgCentroid {
    float sx = 0.f, sy = 0.f, sz = 0.f, si = 0.f;
    __device__ __forceinline__ void add(const float4& p) {
        sx = __fadd_rn(sx, p.x);
        sy = __fadd_rn(sy, p.y);
        sz = __fadd_rn(sz, p.z);
        si = __fadd_rn(si, p.w);
    }
    __device__ __forceinline__ float4 mean(unsigned c) const {
        const float n = (float)c;
        return make_float4(__fdiv_rn(sx, n), __fdiv_rn(sy, n), __fdiv_rn(sz, n), __fdiv_rn(si, n));
    }
};

}  // namespace fls
