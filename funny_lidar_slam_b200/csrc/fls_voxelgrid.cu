// fls_voxelgrid.cu — K7: pcl::VoxelGrid<PointXYZI>::filter as wrapped by VoxelGridCloud
// (include/common/pointcloud_utility.h:216-224,263-271 upstream; PCL 1.10 semantics, SURVEY.md §8c):
//   bounding box -> cell = floor(x*inv_leaf) - min_b (fp32) -> linear id -> sort by id -> one fp32 centroid
//   (xyz AND intensity) per occupied cell, cells in ascending id; dx*dy*dz > INT_MAX returns the input unchanged.
// The radix sort is stable, so every centroid is summed in input order — the order the oracle pins.  The key and centroid
// arithmetic lives in fls_voxel.cuh, shared with the keyframe store's segmented pass (fls_keyframes.cu).
#include "fls_maps.h"
#include "fls_voxel.cuh"

namespace fls {
namespace {

__global__ void minmax_kernel(const float4* __restrict__ pts, size_t n, MinMaxOrd* __restrict__ out) {
    __shared__ float s[6][256];
    float mn0 = INFINITY, mn1 = INFINITY, mn2 = INFINITY, mx0 = -INFINITY, mx1 = -INFINITY, mx2 = -INFINITY;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float4 p = pts[i];
        mn0 = fminf(mn0, p.x); mx0 = fmaxf(mx0, p.x);
        mn1 = fminf(mn1, p.y); mx1 = fmaxf(mx1, p.y);
        mn2 = fminf(mn2, p.z); mx2 = fmaxf(mx2, p.z);
    }
    s[0][threadIdx.x] = mn0; s[1][threadIdx.x] = mn1; s[2][threadIdx.x] = mn2;
    s[3][threadIdx.x] = mx0; s[4][threadIdx.x] = mx1; s[5][threadIdx.x] = mx2;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) {
            for (int k = 0; k < 3; ++k) s[k][threadIdx.x] = fminf(s[k][threadIdx.x], s[k][threadIdx.x + o]);
            for (int k = 3; k < 6; ++k) s[k][threadIdx.x] = fmaxf(s[k][threadIdx.x], s[k][threadIdx.x + o]);
        }
        __syncthreads();
    }
    if (threadIdx.x < 3) atomicMin(&out->mn[threadIdx.x], f2ord(s[threadIdx.x][0]));
    else if (threadIdx.x < 6) atomicMax(&out->mx[threadIdx.x - 3], f2ord(s[threadIdx.x][0]));
}

__global__ void minmax_init_kernel(MinMaxOrd* o) {
    for (int k = 0; k < 3; ++k) {
        o->mn[k] = 0xffffffffu;
        o->mx[k] = 0u;
    }
}

__global__ void vg_keys_kernel(const float4* __restrict__ pts, size_t n, float inv, VgParams g, unsigned* __restrict__ keys, unsigned* __restrict__ idx) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    keys[i] = vg_cell_id(pts[i], inv, g);
    idx[i] = (unsigned)i;
}

// one thread per occupied cell: sequential fp32 sums in input order (CentroidPoint accumulators of PCL)
__global__ void vg_centroid_kernel(const float4* __restrict__ pts, const unsigned* __restrict__ idx_sorted, const unsigned* __restrict__ starts,
                                   const unsigned* __restrict__ counts, int runs, float4* __restrict__ out) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= runs) return;
    const unsigned s = starts[r], c = counts[r];
    VgCentroid acc;
    for (unsigned k = 0; k < c; ++k) acc.add(__ldg(pts + idx_sorted[s + k]));
    out[r] = acc.mean(c);
}

}  // namespace

// Returns the number of output points; d_out must hold n records.  Waits twice (bounding box, run count) — both values size the
// following launches.
size_t voxel_grid_device(const float4* d_pts, size_t n, float leaf, float4* d_out, BuildScratch& sc, Call& c) {
    if (n == 0) return 0;
    const cudaStream_t st = c.stream;
    const float inv = 1.0f / leaf;
    sc.minmax.reserve(16);
    MinMaxOrd* d_mm = reinterpret_cast<MinMaxOrd*>(sc.minmax.p);
    minmax_init_kernel<<<1, 1, 0, st>>>(d_mm);
    const unsigned nb = grid_for(n, 256) < 592 ? grid_for(n, 256) : 592;
    minmax_kernel<<<nb, 256, 0, st>>>(d_pts, n, d_mm);
    MinMaxOrd ho;
    FLS_CUDA(cudaMemcpyAsync(&ho, d_mm, sizeof(ho), cudaMemcpyDeviceToHost, st));
    c.sync();
    c.launches += 2;
    const VgParams g = vg_params(ho, inv);
    if (g.overflow) {  // PCL: "Leaf size is too small" -> output = input
        FLS_CUDA(cudaMemcpyAsync(d_out, d_pts, n * sizeof(float4), cudaMemcpyDeviceToDevice, st));
        return n;
    }
    sc.reserve_runs<unsigned>(n);
    vg_keys_kernel<<<grid_for(n, 256), 256, 0, st>>>(d_pts, n, inv, g, sc.k32a.p, sc.idx.p);
    int end_bit = 1;
    {
        const long long maxid = (long long)g.divb[0] * g.divb[1] * g.divb[2];
        while ((1LL << end_bit) < maxid && end_bit < 32) ++end_bit;
    }
    sc.sort_pairs<unsigned>(n, end_bit, c);
    const int runs = sc.encode_runs<unsigned>(n, c);
    sc.run_starts(runs, c);
    vg_centroid_kernel<<<grid_for(runs, 128), 128, 0, st>>>(d_pts, sc.idx_sorted.p, sc.starts.p, sc.counts.p, runs, d_out);
    FLS_CUDA(cudaGetLastError());
    c.launches += 6;
    return (size_t)runs;
}

}  // namespace fls
