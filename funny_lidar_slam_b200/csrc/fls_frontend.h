// fls_frontend.h — the LOAM front-end stages as enqueue functions on device buffers and a caller stream: the projector
// (fls_project.cu) and the feature extractor (fls_features.cu); the voxel filter is voxel_grid_device (fls_voxelgrid.cu).
// The per-stage entries (fls_project_imu, fls_extract_features, fls_voxel_grid) and the fused LoamFull front end
// (fls_preprocess_loam, fls_frontend.cu) run the same stage code.
#pragma once
#include "fls_maps.h"

namespace fls {

// projector scratch and outputs on the device
struct ProjStage {
    DevBuf<float4> raw, ordered;
    DevBuf<unsigned char> staging;
    DevBuf<int> ring, col, rows;  // rows: [row_start V][row_end V]
    DevBuf<unsigned> winner, flag, excl, total;
    DevBuf<float> depth, time;
    DevBuf<unsigned long long> imu_t;
    DevBuf<double> imu_q;
    DevBuf<unsigned char> cub_tmp;
};

// Uploads the raw records (+ ring, and time and the IMU samples when de-skewing) and enqueues PointcloudProjector::Project on
// c.stream: s.ordered / s.depth / s.col (V*H entries, the first *s.total meaningful), s.rows, s.total.  A reference time outside the
// IMU buffer accepts no point.  `vel` (NULL: rotation only) is the body velocity of the *_motion entries.  Counts the bytes it copies
// and the kernels it launches; nothing waits.
// src_on_device: raw (packed float4, stride 16), ring and time are device arrays on the stream's device and only the IMU samples
// are uploaded; the kernels are the same.
int enqueue_project(ProjStage& s, const void* raw, const int* ring, const float* time, const fls_imu_buffer* imu, const double* vel, size_t n,
                    size_t stride, int V, int H, float h_res, float min_d, float max_d, Call& c, bool src_on_device);

// launch shape of the feature kernels, from the host copy of the row bounds
struct FeatPlan {
    bool active;  // false: fewer than 12 ordered points or no rows, no features (the kernels are not launched)
    int n, n_rows, max_len, max_ring, lpad, lcap;
    size_t planar_cap, smem_sort, smem_ring;
};
// FLS_ERR_INVALID_ARG for row bounds outside [0, n), FLS_ERR_UNSUPPORTED when a block or ring exceeds the shared-memory working set
int plan_features(const int* row_start, const int* row_end, int n_rows, size_t n, FeatPlan& p);

struct FeatStage {
    DevBuf<float> rough;
    DevBuf<unsigned char> meta;
    DevBuf<unsigned long long> sorted;
    DevBuf<int> out;  // per-ring picks, segment counts and offsets, the two totals
};

// Enqueues FeatureExtractor::ExtractFeatures on the projector's device arrays (d_rows = [row_start V][row_end V]) and compacts the
// per-ring results in upstream's emission order: the indices into d_idx (corners first, then the planar points; NULL: skipped)
// and / or the gathered records of d_ordered into d_corner / d_planar (NULL: skipped).  Six kernels.  Returns the device address
// of {n_corner, n_planar}.
const int* enqueue_features(FeatStage& s, const FeatPlan& p, int device, const float* d_depth, const int* d_col, const int* d_rows, float corner_thr,
                            float planar_thr, const float4* d_ordered, int* d_idx, float4* d_corner, float4* d_planar, cudaStream_t st);
constexpr int kFeatLaunches = 6;

// algorithmic bytes of each stage: its inputs read once and its outputs written once (the feature stage also writes and reads its
// roughness, meta bytes and sort keys)
inline long long project_algo_bytes(size_t n_raw, bool with_time, size_t n_ordered) {
    return (long long)(n_raw * (16 + 4 + (with_time ? 4 : 0)) + n_ordered * (16 + 4 + 4));
}
inline long long feature_algo_bytes(size_t n, size_t n_corner, size_t n_planar) {
    return (long long)(n * (4 + 4 + 2 * 4 + 2 * 1 + 2 * 8) + (n_corner + n_planar) * 4);
}
inline long long voxel_algo_bytes(size_t n_in, size_t n_out) { return (long long)((n_in + n_out) * 16); }

// fls_preprocess_loam (src_on_device false) and fls_preprocess_loam_device (true: raw / ring / time are device arrays, stride 16)
// after their argument checks (fls_frontend.cu)
int preprocess_loam_device(const fls_loam_frontend_cfg& c, const void* raw, const int* ring, const float* time, size_t n, size_t stride,
                           const fls_imu_buffer* imu, const double* vel, float* corner, float* planar, float* d_corner, float* d_planar, size_t* n_corner,
                           size_t* n_planar, fls_match_stats* stats, bool src_on_device);

// fls_convert_cloud after its argument checks (fls_convert.cu)
int convert_cloud_device(const fls_convert_cfg& c, const fls_pointcloud2& m, float* xyzi, int* ring, float* time, float* d_xyzi, int* d_ring,
                         float* d_time, size_t* n, fls_convert_result* res, fls_match_stats* stats);

// fls_preprocess_device (device float4 xyzi + float time) after its argument checks (fls_preprocess.cu; the host entry's driver is
// preprocess_device, fls_maps.h)
int preprocess_device_input(int device, const float* d_xyzi, const float* d_time, size_t n, const fls_imu_buffer* imu, const double* vel, float min_d,
                            float max_d, int jump_span, float leaf, float* ordered_out, float* d_ordered, size_t* n_ordered, float* planar_out,
                            float* d_planar, size_t* n_planar);

}  // namespace fls
