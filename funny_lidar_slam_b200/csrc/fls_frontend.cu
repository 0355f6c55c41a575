// fls_frontend.cu — PreProcessing::Run, the LoamFull branch (src/slam/preprocessing.cpp:226-237 upstream), in one call:
// PointcloudProjector::Project with the per-point de-skew -> FeatureExtractor::ExtractFeatures -> corner_voxel_filter_ and
// planer_voxel_filter_.  The stages are the ones behind fls_project_imu, fls_extract_features and fls_voxel_grid (fls_frontend.h);
// point data stays on the device between them.  The host reads back only the sizes that shape a later launch (DESIGN.md §3.8).
#include "fls_frontend.h"

namespace fls {
namespace {

// Stage buffers of its own: the call takes its workspace's lock only (never the projector's or the extractor's), so it cannot
// deadlock against them.
struct LoamWorkspace : Workspace {
    ProjStage proj;
    FeatStage feat;
    BuildScratch vg;
    DevBuf<float4> corner, planar, corner_f, planar_f;  // gathered features, filtered clouds (when the caller gives no device output)
    PinnedBuf<int> h_small;                              // [n_ordered][row_start V][row_end V] or [n_corner, n_planar]
};

}  // namespace

int preprocess_loam_device(const fls_loam_frontend_cfg& c, const void* raw, const int* ring, const float* time, size_t n, size_t stride,
                           const fls_imu_buffer* imu, const double* vel, float* corner, float* planar, float* d_corner, float* d_planar, size_t* n_corner,
                           size_t* n_planar, fls_match_stats* stats, bool src_on_device) {
    *n_corner = *n_planar = 0;
    const int V = c.n_rows, H = c.n_cols;
    return with_workspace<LoamWorkspace>(c.device, [&](LoamWorkspace& w) -> int {
        Call& call = w.call;
        const cudaStream_t st = call.stream;
        int* const h_small = w.h_small.reserve((size_t)2 * V + 1);
        call.begin();
        // ---- projector (+ de-skew) ----
        int rc = enqueue_project(w.proj, raw, ring, time, imu, vel, n, stride, V, H, c.horizontal_resolution, c.min_distance, c.max_distance, call, src_on_device);
        if (rc != FLS_OK) return rc;
        // sync 1: n_ordered and the row bounds size the feature kernels (shared memory, planar capacity)
        FLS_CUDA(cudaMemcpyAsync(h_small, w.proj.total.p, sizeof(int), cudaMemcpyDeviceToHost, st));
        FLS_CUDA(cudaMemcpyAsync(h_small + 1, w.proj.rows.p, (size_t)2 * V * sizeof(int), cudaMemcpyDeviceToHost, st));
        call.sync();
        call.d2h += (long long)((2 * (size_t)V + 1) * sizeof(int));
        const size_t n_ord = (size_t)(unsigned)h_small[0];
        FeatPlan p;
        rc = plan_features(h_small + 1, h_small + 1 + V, V, n_ord, p);
        if (rc != FLS_OK) return rc;  // a ring or block beyond the shared-memory working set: FLS_ERR_UNSUPPORTED, nothing written
        // ---- features, gathered into two contiguous clouds ----
        size_t nc = 0, np = 0;
        if (p.active) {
            w.corner.reserve((size_t)V * 120);
            w.planar.reserve(p.planar_cap + 1);
            const int* d_tot = enqueue_features(w.feat, p, c.device, w.proj.depth.p, w.proj.col.p, w.proj.rows.p, c.corner_threshold, c.planar_threshold,
                                                w.proj.ordered.p, nullptr, w.corner.p, w.planar.p, st);
            call.launches += kFeatLaunches;
            // sync 2: the feature counts size the voxel filters
            FLS_CUDA(cudaMemcpyAsync(h_small, d_tot, 2 * sizeof(int), cudaMemcpyDeviceToHost, st));
            call.sync();
            call.d2h += 2 * sizeof(int);
            nc = (size_t)h_small[0];
            np = (size_t)h_small[1];
        }
        // ---- voxel filters (syncs 3-6: bounding box and run count of each), straight into the caller's device buffers ----
        float4* oc = d_corner ? reinterpret_cast<float4*>(d_corner) : w.corner_f.reserve(nc + 1);
        float4* op = d_planar ? reinterpret_cast<float4*>(d_planar) : w.planar_f.reserve(np + 1);
        const size_t mc = voxel_grid_device(w.corner.p, nc, c.corner_leaf, oc, w.vg, call);
        const size_t mp = voxel_grid_device(w.planar.p, np, c.planar_leaf, op, w.vg, call);
        if (corner && mc) FLS_CUDA(cudaMemcpyAsync(corner, oc, mc * sizeof(float4), cudaMemcpyDeviceToHost, st));
        if (planar && mp) FLS_CUDA(cudaMemcpyAsync(planar, op, mp * sizeof(float4), cudaMemcpyDeviceToHost, st));
        call.d2h += (long long)(((corner ? mc : 0) + (planar ? mp : 0)) * sizeof(float4));
        call.end(stats);  // sync 7: the outputs are complete when the call returns
        *n_corner = mc;
        *n_planar = mp;
        if (stats) {
            stats->n_source = (long long)n;
            const bool with_time = imu && imu->n_imu && time;
            stats->algo_bytes = project_algo_bytes(n, with_time, n_ord) + (p.active ? feature_algo_bytes(n_ord, nc, np) : 0) +
                                voxel_algo_bytes(nc, mc) + voxel_algo_bytes(np, mp);
        }
        return FLS_OK;
    });
}

}  // namespace fls
