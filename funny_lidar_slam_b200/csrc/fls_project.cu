// fls_project.cu — PointcloudProjector::Project (src/loam/pointcloud_projector.cpp:32-133 upstream) on the device:
// range gate, column from the 7th-order FastAtan2 polynomial (include/common/math_function.h:159-186), "first hit wins"
// per (ring, column) cell, then the row-major compaction that produces ordered_cloud_ / point_depth_vec_ /
// point_col_index_vec_ / row_start_index_vec_ / row_end_index_vec_ — the arrays the feature extractor (K4) consumes.
//
// The sequential "first point to reach a cell keeps it" (:90-91) becomes an atomicMin on the point's position in the
// raw cloud: the smallest index is by definition the first one the sequential loop would have seen.  The per-point
// de-skew (ProcessPoint, :100-103) runs on the winner of every cell when the caller passes the IMU orientation buffer
// (fls_project_imu; fls_deskew.cuh); without one the points pass through unchanged.
#include <cub/cub.cuh>

#include "fls_atan.cuh"
#include "fls_deskew.cuh"
#include "fls_frontend.h"

namespace fls {
namespace {

__device__ __forceinline__ float depth_ref(float x, float y, float z) {
    return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
}

__global__ void proj_clear_kernel(unsigned* __restrict__ winner, size_t cells) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i < cells) winner[i] = 0xffffffffu;
}

__global__ void proj_claim_kernel(const float4* __restrict__ raw, const int* __restrict__ ring, const float* __restrict__ time, DeskewView dv, int n,
                                  int V, int H, float h_res, float min_d, float max_d, unsigned* __restrict__ winner) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const float4 p = raw[k];
    const float depth = depth_ref(p.x, p.y, p.z);
    if (depth < min_d || depth > max_d) return;  // :59-61
    const int row = ring[k];
    int col = (int)roundf(__fdiv_rn(fast_atan2_ref(p.y, p.x), h_res)) + H / 2;  // :64-65
    if (col >= H) col -= H;
    if (row >= V || row < 0 || col < 0 || col >= H) return;  // :81-82
    if (dv.m > 0) {  // ProcessPoint fails for a time outside the IMU buffer: the point returns without claiming its cell (:100-103)
        const unsigned long long t = (unsigned long long)((long long)dv.ref_time + trunc_i64(__dmul_rn((double)time[k], 1.0e6)));
        if (dv.m < 2 || dv.t[0] > t || dv.t[dv.m - 1] < t) return;
    }
    atomicMin(&winner[(size_t)row * H + col], (unsigned)k);  // :86-87 first hit wins
}

__global__ void proj_flags_kernel(const unsigned* __restrict__ winner, size_t cells, unsigned* __restrict__ flag) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i < cells) flag[i] = winner[i] != 0xffffffffu ? 1u : 0u;
}

__global__ void proj_emit_kernel(const float4* __restrict__ raw, const float* __restrict__ time, DeskewView dv, const unsigned* __restrict__ winner,
                                 const unsigned* __restrict__ excl, int V, int H,
                                 float4* __restrict__ ordered, float* __restrict__ depth, int* __restrict__ col, int* __restrict__ row_start,
                                 int* __restrict__ row_end, unsigned* __restrict__ total) {
    const size_t cells = (size_t)V * H;
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= cells) return;
    const unsigned w = winner[i];
    const unsigned pos = excl[i];
    if (w != 0xffffffffu) {
        const float4 p = raw[w];
        float4 q = p;
        if (dv.m > 0) deskew_point(dv, p.x, p.y, p.z, time[w], q.x, q.y, q.z);  // :100-103; the range stays the raw point's (:57, :105)
        ordered[pos] = q;
        depth[pos] = depth_ref(p.x, p.y, p.z);
        col[pos] = (int)(i % (size_t)H);
    }
    const int c = (int)(i % (size_t)H), r = (int)(i / (size_t)H);
    if (c == 0) row_start[r] = (int)pos + 5;  // :115
    if (c == H - 1) {
        const unsigned end = pos + (w != 0xffffffffu ? 1u : 0u);
        row_end[r] = (int)end - 6;  // :131
        if (r == V - 1) *total = end;
    }
}

struct ProjWorkspace : Workspace {
    ProjStage s;
};

}  // namespace

int make_deskew_view(const fls_imu_buffer* imu, DevBuf<unsigned long long>& d_t, DevBuf<double>& d_q, cudaStream_t st, DeskewView& v,
                     bool& ref_outside);

int enqueue_project(ProjStage& w, const void* raw, const int* ring, const float* time, const fls_imu_buffer* imu, size_t n, size_t stride, int V, int H,
                    float h_res, float min_d, float max_d, cudaStream_t st, long long* h2d, int* launches, bool src_on_device) {
    const size_t cells = (size_t)V * H;
    DeskewView dv;
    const bool use_imu = imu && imu->n_imu && time;
    bool ref_outside;
    const int rc = make_deskew_view(use_imu ? imu : nullptr, w.imu_t, w.imu_q, st, dv, ref_outside);
    if (rc != FLS_OK) return rc;
    if (dv.m > 0) *h2d += (long long)(imu->n_imu * (sizeof(unsigned long long) + 4 * sizeof(double)));
    if (ref_outside) n = 0;  // SetRefTime failed: no point is accepted
    w.raw.reserve(n + 1);
    w.ring.reserve(n + 1);
    w.time.reserve(n + 1);
    // the records the kernels read: the caller's device arrays, or the stage buffers the host records are uploaded to
    const float4* d_raw = src_on_device ? reinterpret_cast<const float4*>(raw) : w.raw.p;
    const int* d_ring = src_on_device ? ring : w.ring.p;
    const float* d_time = src_on_device && use_imu ? time : w.time.p;
    if (n && use_imu && !src_on_device) {
        FLS_CUDA(cudaMemcpyAsync(w.time.p, time, n * sizeof(float), cudaMemcpyHostToDevice, st));
        *h2d += (long long)(n * sizeof(float));
    }
    w.winner.reserve(cells);
    w.flag.reserve(cells);
    w.excl.reserve(cells);
    w.total.reserve(1);
    w.ordered.reserve(cells);
    w.depth.reserve(cells);
    w.col.reserve(cells);
    w.rows.reserve((size_t)V * 2);
    if (n && !src_on_device) {
        upload_records(raw, n, stride, w.raw.p, w.staging, st, h2d, launches);
        FLS_CUDA(cudaMemcpyAsync(w.ring.p, ring, n * sizeof(int), cudaMemcpyHostToDevice, st));
        *h2d += (long long)(n * sizeof(int));
    }
    const unsigned gc = (unsigned)((cells + 255) / 256);
    proj_clear_kernel<<<gc, 256, 0, st>>>(w.winner.p, cells);
    if (n) proj_claim_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_raw, d_ring, d_time, dv, (int)n, V, H, h_res, min_d, max_d, w.winner.p);
    proj_flags_kernel<<<gc, 256, 0, st>>>(w.winner.p, cells, w.flag.p);
    cub_pass(w.cub_tmp, [&](void* tmp, size_t& bytes) { return cub::DeviceScan::ExclusiveSum(tmp, bytes, w.flag.p, w.excl.p, (int)cells, st); });
    // upstream leaves the tails of depth / col as they were (resize to V*H, col zero-filled): zero both
    FLS_CUDA(cudaMemsetAsync(w.depth.p, 0, cells * sizeof(float), st));
    FLS_CUDA(cudaMemsetAsync(w.col.p, 0, cells * sizeof(int), st));
    proj_emit_kernel<<<gc, 256, 0, st>>>(d_raw, d_time, dv, w.winner.p, w.excl.p, V, H, w.ordered.p, w.depth.p, w.col.p, w.rows.p, w.rows.p + V, w.total.p);
    FLS_CUDA(cudaGetLastError());
    *launches += n ? 5 : 4;
    return FLS_OK;
}

// Host driver: raw cloud (host, `stride` bytes per record) + ring per point -> projector arrays (host).  depth_out / col_out hold V*H
// entries (the first *n_out are meaningful, as upstream), ordered_out V*H packed float4 records.
int project_device(int device, const void* raw, const int* ring, const float* time, const fls_imu_buffer* imu, size_t n, size_t stride, int V, int H,
                   float h_res, float min_d, float max_d, float* ordered_out, float* depth_out, int* col_out, int* row_start, int* row_end, size_t* n_out) {
    *n_out = 0;
    if (V <= 0 || H <= 0 || !(h_res > 0.f) || n > 0x7fffffffull) return FLS_ERR_INVALID_ARG;
    const size_t cells = (size_t)V * H;
    if (cells > 0x7fffffffull) return FLS_ERR_INVALID_ARG;
    return with_workspace<ProjWorkspace>(device, [&](ProjWorkspace& ws) -> int {
        cudaStream_t st = ws.st;
        ProjStage& w = ws.s;
        long long h2d = 0;
        int launches = 0;
        const int rc = enqueue_project(w, raw, ring, time, imu, n, stride, V, H, h_res, min_d, max_d, st, &h2d, &launches, false);
        if (rc != FLS_OK) return rc;
        unsigned total = 0;
        FLS_CUDA(cudaMemcpyAsync(&total, w.total.p, sizeof(total), cudaMemcpyDeviceToHost, st));
        FLS_CUDA(cudaMemcpyAsync(depth_out, w.depth.p, cells * sizeof(float), cudaMemcpyDeviceToHost, st));
        FLS_CUDA(cudaMemcpyAsync(col_out, w.col.p, cells * sizeof(int), cudaMemcpyDeviceToHost, st));
        FLS_CUDA(cudaMemcpyAsync(row_start, w.rows.p, (size_t)V * sizeof(int), cudaMemcpyDeviceToHost, st));
        FLS_CUDA(cudaMemcpyAsync(row_end, w.rows.p + V, (size_t)V * sizeof(int), cudaMemcpyDeviceToHost, st));
        FLS_CUDA(cudaStreamSynchronize(st));
        if (total) FLS_CUDA(cudaMemcpy(ordered_out, w.ordered.p, (size_t)total * sizeof(float4), cudaMemcpyDeviceToHost));
        *n_out = total;
        return FLS_OK;
    });
}

}  // namespace fls
