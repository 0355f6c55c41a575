// fls_preprocess.cu — the point pipeline in front of the registration plug-ins (SURVEY.md §8f-2), on the device:
// PreProcessing::Run's branch for PointToPlane_IVOX / PointToPlane_KdTree / IcpOptimized / IncrementalNDT
// (src/slam/preprocessing.cpp:181-225 upstream): range gate -> IMU de-skew of every point (fls_deskew.cuh) -> ordered_cloud_
// (every kept point) and planar_cloud_ (every lidar_point_jump_span-th RAW index among the kept ones, then pcl::VoxelGrid).
// fls_preprocess reads host records {x, y, z, intensity, time}; fls_preprocess_device reads float4 xyzi + float time already in device
// memory (fls_convert_cloud's outputs).  Both run run_preprocess below: the same kernels on the same values.
#include <cub/cub.cuh>

#include <cmath>

#include "fls_deskew.cuh"
#include "fls_frontend.h"
#include "fls_maps.h"

namespace fls {

bool deskew_ref_inverse(const unsigned long long* t, const double* q, size_t m, unsigned long long ref, double* qri) {
    if (m < 2 || t[0] > ref || t[m - 1] < ref) return false;
    size_t l;
    if (t[0] == ref) l = 0;
    else if (t[m - 1] == ref) l = m - 2;
    else {
        l = m - 1;
        while (ref < t[l]) --l;
    }
    const size_t r = l + 1;
    const double s = double(ref - t[l]) / double(t[r] - t[l]);
    const double u = 1.0 - s;
    volatile double qx = q[4 * l] * u + q[4 * r] * s, qy = q[4 * l + 1] * u + q[4 * r + 1] * s, qz = q[4 * l + 2] * u + q[4 * r + 2] * s,
                    qw = q[4 * l + 3] * u + q[4 * r + 3] * s;
    // Eigen 3.3.7's guards: normalized() leaves a quaternion whose squared norm is not > 0 as it is, inverse() of one returns zero
    const double sq = ((qx * qx + qy * qy) + qz * qz) + qw * qw;
    double nx = qx, ny = qy, nz = qz, nw = qw;
    if (sq > 0.0) {
        const double n = std::sqrt(sq);
        nx = qx / n, ny = qy / n, nz = qz / n, nw = qw / n;
    }
    const double n2 = ((nx * nx + ny * ny) + nz * nz) + nw * nw;
    if (n2 > 0.0) {
        qri[0] = -nx / n2;
        qri[1] = -ny / n2;
        qri[2] = -nz / n2;
        qri[3] = nw / n2;
    } else {
        qri[0] = qri[1] = qri[2] = qri[3] = 0.0;
    }
    return true;
}

namespace {

__device__ __forceinline__ float depth_ref_pp(float x, float y, float z) {
    return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
}

// one thread per raw point: gate + de-skew; flags: bit 0 kept (ordered cloud), bit 1 kept and i % jump == 0 (planar candidates).
// Point i is xyzi[xs*i .. xs*i+3] with its time at t[ts*i] (host records: xs = ts = 5; device arrays: xs = 4, ts = 1).
__global__ void pp_point_kernel(const float* __restrict__ xyzi, int xs, const float* __restrict__ t, int ts, int n, DeskewView dv, float min_d,
                                float max_d, int jump, float4* __restrict__ corrected, unsigned* __restrict__ f_ord, unsigned* __restrict__ f_pl) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* p = xyzi + (size_t)xs * i;
    float x = p[0], y = p[1], z = p[2];
    bool keep = true;
    const float depth = depth_ref_pp(x, y, z);
    if (depth < min_d || depth > max_d) keep = false;  // preprocessing.cpp:199-203
    if (keep && dv.m > 0) keep = deskew_point(dv, x, y, z, t[(size_t)ts * i], x, y, z);  // :205-211
    corrected[i] = make_float4(x, y, z, p[3]);
    f_ord[i] = keep ? 1u : 0u;
    f_pl[i] = (keep && (i % jump) == 0) ? 1u : 0u;  // :219-222
}
__global__ void pp_scatter_kernel(const float4* __restrict__ corrected, int n, const unsigned* __restrict__ f, const unsigned* __restrict__ excl,
                                  float4* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && f[i]) out[excl[i]] = corrected[i];
}

struct PpWorkspace : Workspace {
    DevBuf<float> raw;
    DevBuf<float4> corrected, ordered, planar, filtered;
    DevBuf<unsigned> f_ord, f_pl, e_ord, e_pl;
    DevBuf<unsigned long long> imu_t;
    DevBuf<double> imu_q;
    DevBuf<unsigned char> cub_tmp;
    BuildScratch scratch;
};

}  // namespace

// uploads the IMU samples and fills the view.  ref_outside: ref_time is outside the buffer (SetRefTime fails; the view stays the
// identity).  Returns FLS_ERR_INVALID_ARG for a null array, more than 2^31 - 1 samples, or a stamp followed by a smaller one:
// deskew_point finds the interval by bisection, upstream by a downward scan (data_searcher.h:100-134), and the two pick the same
// pair only on ascending stamps (equal ones allowed).
int make_deskew_view(const fls_imu_buffer* imu, DevBuf<unsigned long long>& d_t, DevBuf<double>& d_q, cudaStream_t st, DeskewView& v,
                     bool& ref_outside) {
    std::memset(&v, 0, sizeof(v));
    ref_outside = false;
    if (!imu || imu->n_imu == 0) return FLS_OK;  // identity
    if (!imu->imu_time_us || !imu->imu_quat_xyzw || imu->n_imu > 0x7fffffffull) return FLS_ERR_INVALID_ARG;
    for (size_t k = 1; k < imu->n_imu; ++k)
        if (imu->imu_time_us[k] < imu->imu_time_us[k - 1]) return FLS_ERR_INVALID_ARG;
    if (!deskew_ref_inverse(reinterpret_cast<const unsigned long long*>(imu->imu_time_us), imu->imu_quat_xyzw, imu->n_imu, imu->ref_time_us, v.qri)) {
        ref_outside = true;
        return FLS_OK;
    }
    d_t.reserve(imu->n_imu);
    d_q.reserve(imu->n_imu * 4);
    FLS_CUDA(cudaMemcpyAsync(d_t.p, imu->imu_time_us, imu->n_imu * sizeof(unsigned long long), cudaMemcpyHostToDevice, st));
    FLS_CUDA(cudaMemcpyAsync(d_q.p, imu->imu_quat_xyzw, imu->n_imu * 4 * sizeof(double), cudaMemcpyHostToDevice, st));
    v.t = d_t.p;
    v.q = d_q.p;
    v.m = (int)imu->n_imu;
    v.ref_time = imu->ref_time_us;
    for (int k = 0; k < 16; ++k) v.T[k] = imu->T_lidar_to_imu[k];
    return FLS_OK;
}

namespace {

// The points are host records {x, y, z, intensity, time} (src_on_device false: uploaded first) or device arrays (float4 xyzi, float time).
// ordered_cloud_ goes to ordered_out (host) and / or d_ordered, planar_cloud_ to planar_out and / or d_planar (NULL: not written).
int run_preprocess(int device, const float* xyzi, const float* time, bool src_on_device, size_t n, const fls_imu_buffer* imu, float min_d, float max_d,
                   int jump_span, float leaf, float* ordered_out, float* d_ordered, size_t* n_ordered, float* planar_out, float* d_planar,
                   size_t* n_planar) {
    *n_ordered = *n_planar = 0;
    if (n > 0x7fffffffull || jump_span < 1 || !(leaf > 0.f)) return FLS_ERR_INVALID_ARG;
    if (n == 0) return FLS_OK;
    return with_workspace<PpWorkspace>(device, [&](PpWorkspace& w) -> int {
        cudaStream_t st = w.st;
        DeskewView dv;
        bool ref_outside;
        const int rc = make_deskew_view(imu, w.imu_t, w.imu_q, st, dv, ref_outside);
        if (rc != FLS_OK) return rc;
        if (ref_outside) return FLS_OK;  // SetRefTime failed: upstream drops the scan (:178-183) -> empty clouds
        w.corrected.reserve(n);
        float4* ord = d_ordered ? reinterpret_cast<float4*>(d_ordered) : w.ordered.reserve(n);
        w.planar.reserve(n);
        float4* filtered = d_planar ? reinterpret_cast<float4*>(d_planar) : w.filtered.reserve(n);
        w.f_ord.reserve(n);
        w.f_pl.reserve(n);
        w.e_ord.reserve(n);
        w.e_pl.reserve(n);
        const float *px = xyzi, *pt = time;
        int xs = 4, ts = 1;
        if (!src_on_device) {
            w.raw.reserve(n * 5);
            FLS_CUDA(cudaMemcpyAsync(w.raw.p, xyzi, n * 5 * sizeof(float), cudaMemcpyHostToDevice, st));
            px = w.raw.p;
            pt = w.raw.p + 4;
            xs = ts = 5;
        }
        const unsigned g = (unsigned)((n + 255) / 256);
        pp_point_kernel<<<g, 256, 0, st>>>(px, xs, pt, ts, (int)n, dv, min_d, max_d, jump_span, w.corrected.p, w.f_ord.p, w.f_pl.p);
        auto scan_ord = [&](void* tmp, size_t& bytes) { return cub::DeviceScan::ExclusiveSum(tmp, bytes, w.f_ord.p, w.e_ord.p, (int)n, st); };
        auto scan_pl = [&](void* tmp, size_t& bytes) { return cub::DeviceScan::ExclusiveSum(tmp, bytes, w.f_pl.p, w.e_pl.p, (int)n, st); };
        cub_reserve(w.cub_tmp, scan_ord, scan_pl);
        cub_run(w.cub_tmp, scan_ord);
        cub_run(w.cub_tmp, scan_pl);
        pp_scatter_kernel<<<g, 256, 0, st>>>(w.corrected.p, (int)n, w.f_ord.p, w.e_ord.p, ord);
        pp_scatter_kernel<<<g, 256, 0, st>>>(w.corrected.p, (int)n, w.f_pl.p, w.e_pl.p, w.planar.p);
        unsigned last[4] = {0, 0, 0, 0};
        FLS_CUDA(cudaMemcpyAsync(&last[0], w.e_ord.p + (n - 1), sizeof(unsigned), cudaMemcpyDeviceToHost, st));
        FLS_CUDA(cudaMemcpyAsync(&last[1], w.f_ord.p + (n - 1), sizeof(unsigned), cudaMemcpyDeviceToHost, st));
        FLS_CUDA(cudaMemcpyAsync(&last[2], w.e_pl.p + (n - 1), sizeof(unsigned), cudaMemcpyDeviceToHost, st));
        FLS_CUDA(cudaMemcpyAsync(&last[3], w.f_pl.p + (n - 1), sizeof(unsigned), cudaMemcpyDeviceToHost, st));
        FLS_CUDA(cudaStreamSynchronize(st));
        const size_t no = (size_t)last[0] + last[1], npl = (size_t)last[2] + last[3];
        int l = 0;
        const size_t nf = npl ? voxel_grid_device(w.planar.p, npl, leaf, filtered, w.scratch, st, &l) : 0;  // :224-225
        if (no && ordered_out) FLS_CUDA(cudaMemcpyAsync(ordered_out, ord, no * sizeof(float4), cudaMemcpyDeviceToHost, st));
        if (nf && planar_out) FLS_CUDA(cudaMemcpyAsync(planar_out, filtered, nf * sizeof(float4), cudaMemcpyDeviceToHost, st));
        FLS_CUDA(cudaStreamSynchronize(st));
        *n_ordered = no;
        *n_planar = nf;
        return FLS_OK;
    });
}

}  // namespace

int preprocess_device(int device, const float* raw_xyzit, size_t n, const fls_imu_buffer* imu, float min_d, float max_d, int jump_span, float leaf,
                      float* ordered_out, size_t* n_ordered, float* planar_out, size_t* n_planar) {
    return run_preprocess(device, raw_xyzit, nullptr, false, n, imu, min_d, max_d, jump_span, leaf, ordered_out, nullptr, n_ordered, planar_out, nullptr,
                          n_planar);
}

int preprocess_device_input(int device, const float* d_xyzi, const float* d_time, size_t n, const fls_imu_buffer* imu, float min_d, float max_d,
                            int jump_span, float leaf, float* ordered_out, float* d_ordered, size_t* n_ordered, float* planar_out, float* d_planar,
                            size_t* n_planar) {
    return run_preprocess(device, d_xyzi, d_time, true, n, imu, min_d, max_d, jump_span, leaf, ordered_out, d_ordered, n_ordered, planar_out, d_planar,
                          n_planar);
}

}  // namespace fls
