// fls_info.cuh — FLS_FLAG_INFORMATION: the information matrix of a Match at the pose it returns (DESIGN.md §3.13).
//
// After the Gauss-Newton loop and before the Match's read-back (and before mapping mode inserts the scan), one evaluation pass runs
// the plug-in's per-point term from a fresh correspondence search at the final pose, which it reads from the scan's GnState on the
// device.  A single Match is a batch of one.  Two launches per Match call, whatever the number of scans:
//   info_points_kernel<Args> — scan s owns CTAs [cta0[s], cta0[s + 1]); each CTA sums its points' terms in a fixed order (per-thread
//                              sums, warp shuffles, warp rows in order) and writes one row of kNumAcc partials;
//   info_fold_kernel (fls_info.cu) — adds each scan's rows in CTA order (no atomics: the same bits on every call), maps H and g
//                              from the plug-in's dx to the fusion parameterization and writes the scan's fls_information record.
// The pass never reads or writes the loop's scratch (persistent per-point records and flags, LL rows, GnState): what follows it
// sees exactly what it would see without the flag.
//
// A plug-in opts in with a specialization of InfoTerm for its loop arguments:
//   kBlock, kLanes        block size and lanes per point (a lane group shares one neighbour search, as in the plug-in's loop);
//   count(a)              points of the scan;
//   point(a, i, pose, posef, sub, mask, acc)   adds point i's term at `pose` (row-major R, t; posef: the same in float) to acc in
//                         the plug-in's dx order: H upper triangle [0, 21), -sum J^T W r [21, 27), terms at kAccValid, residual at kAccRes.
#pragma once
#include <cstring>

#include "fls_gn.cuh"
#include "fls_handle.h"

namespace fls {

template <class Args>
struct InfoTerm;

// the scans of one evaluation, passed by value (no copy of their own)
template <class Args>
struct InfoBatch {
    Args a[kMaxBatch];
    const GnState* state[kMaxBatch];  // the final pose of each scan
    int cta0[kMaxBatch + 1];
    int B;
};

#ifdef __CUDACC__
// the term of a point with Jacobian J (6) and residual r, W = 1 (LOAM point-to-plane and corner terms)
__device__ __forceinline__ void info_add_J(const double (&J)[6], double r, double (&acc)[kNumAcc]) {
#pragma unroll
    for (int p = 0; p < 6; ++p)
#pragma unroll
        for (int q = p; q < 6; ++q) acc[tri6(p, q)] += J[p] * J[q];
#pragma unroll
    for (int p = 0; p < 6; ++p) acc[21 + p] -= J[p] * r;
    acc[kAccValid] += 1.0;
    acc[kAccRes] += r;
}

template <class Args>
__global__ void __launch_bounds__(InfoTerm<Args>::kBlock) info_points_kernel(const __grid_constant__ InfoBatch<Args> b, double* __restrict__ part) {
    using T = InfoTerm<Args>;
    constexpr int BLOCK = T::kBlock, L = T::kLanes, PER = BLOCK / L;
    __shared__ double s_pose[12];
    __shared__ float s_posef[12];
    __shared__ double s_red[BLOCK / 32][kAccStride];
    __shared__ int s_w;
    if (threadIdx.x == 0) {
        int w = 0;
        while (w + 1 < b.B && (int)blockIdx.x >= b.cta0[w + 1]) ++w;
        s_w = w;
    }
    __syncthreads();
    const int w = s_w;
    if (threadIdx.x < 12) {
        const GnState* st = b.state[w];
        const double v = threadIdx.x < 9 ? __ldcg(&st->R[threadIdx.x]) : __ldcg(&st->t[threadIdx.x - 9]);
        s_pose[threadIdx.x] = v;
        s_posef[threadIdx.x] = (float)v;
    }
    __syncthreads();
    const Args& a = b.a[w];
    const int cta = (int)blockIdx.x - b.cta0[w], ncta = b.cta0[w + 1] - b.cta0[w];
    const int sub = threadIdx.x & (L - 1);
    const unsigned mask = L >= 32 ? 0xffffffffu : ((1u << L) - 1u) << ((threadIdx.x & 31) & ~(L - 1));
    double acc[kNumAcc];
#pragma unroll
    for (int k = 0; k < kNumAcc; ++k) acc[k] = 0.0;
    const int n = T::count(a);
    for (int i = cta * PER + (int)threadIdx.x / L; i < n; i += ncta * PER) T::point(a, i, s_pose, s_posef, sub, mask, acc);
    gn_warp_rows<BLOCK>(acc, s_red);
    __syncthreads();
    if (threadIdx.x < 32) {
        double v = 0.0;
#pragma unroll
        for (int k = 0; k < BLOCK / 32; ++k) v += s_red[k][threadIdx.x];
        part[(size_t)blockIdx.x * kAccStride + threadIdx.x] = v;
    }
}
#endif

// the fold of an evaluation: every scan's CTA rows, its final pose and the plug-in whose dx the sums are in (fls_info.cu)
struct InfoFold {
    const GnState* state[kMaxBatch];
    int cta0[kMaxBatch + 1];
    int method;
};
void launch_info_fold(const InfoFold& f, int B, const double* part, fls_information* out, cudaStream_t st);

// Enqueues the evaluation of the B scans a[0..B) of the Match in progress (scan s's final pose: h.state.p + s) on the call's stream
// and marks the Match as evaluated, so that read_back copies the records.  Scan s gets one CTA per point group of a block, all scaled
// down together when the kernel's co-resident CTAs cannot hold them (the sizing of match_subgrids).
template <class Args>
void enqueue_information(Handle& h, const Args* a, int B) {
    using T = InfoTerm<Args>;
    constexpr int per_cta = T::kBlock / T::kLanes;
    const int cap = coresident_ctas((const void*)info_points_kernel<Args>, T::kBlock, 0, h.cfg.device);
    static_assert(sizeof(InfoBatch<Args>) <= 32000, "the batch travels as a kernel argument");
    InfoBatch<Args> b;
    std::memset(&b, 0, sizeof(b));
    InfoFold f;
    std::memset(&f, 0, sizeof(f));
    int need[kMaxBatch], tot_need = 0;
    for (int s = 0; s < B; ++s) {
        need[s] = (T::count(a[s]) + per_cta - 1) / per_cta;
        if (need[s] < 1) need[s] = 1;
        tot_need += need[s];
    }
    int grid = 0;
    for (int s = 0; s < B; ++s) {
        int n = tot_need <= cap ? need[s] : (int)((long long)need[s] * (cap - B) / tot_need) + 1;
        if (n < 1) n = 1;
        b.a[s] = a[s];
        b.state[s] = f.state[s] = h.state.p + s;
        b.cta0[s] = f.cta0[s] = grid;
        grid += n;
    }
    b.cta0[B] = f.cta0[B] = grid;
    b.B = B;
    f.method = h.cfg.method;
    double* part = h.info_part.reserve((size_t)grid * kAccStride);
    info_points_kernel<Args><<<grid, T::kBlock, 0, h.call.stream>>>(b, part);
    FLS_CUDA(cudaGetLastError());
    launch_info_fold(f, B, part, h.info.p, h.call.stream);
    h.call.launches += kInfoLaunches;
    h.info_enqueued = true;
}

}  // namespace fls
