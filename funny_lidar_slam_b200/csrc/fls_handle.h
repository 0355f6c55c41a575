// fls_handle.h — the object behind `fls_handle*`: configuration, stream, device-resident map and scan state.
#pragma once
#include <deque>
#include <memory>
#include <vector>

#include "fls_common.cuh"
#include "fls_kernels.h"
#include "fls_maps.h"

namespace fls {

struct Handle {
    fls_config cfg;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;

    // per-call accounting (fls_match_stats)
    int launches = 0;
    long long h2d_bytes = 0, d2h_bytes = 0;
    float last_gpu_ms = 0.f;

    // scan-side buffers
    DevBuf<unsigned char> raw;  // strided caller records before repacking
    DevBuf<float4> src;         // uploaded scan (packed float4)
    DevBuf<float4> src_f;       // scan after Match's own VoxelGridCloud (ICP / NDT)
    DevBuf<float4> stage;       // clouds handed to AddCloudToLocalMap
    DevBuf<float4> stage2;      // transformed / filtered intermediates
    DevBuf<float4> rec0, rec1;  // persistent per-point {J, |d|} records (LOAM plug-ins)
    DevBuf<unsigned char> flags;
    DevBuf<unsigned> tickets;   // chunk ticket counters of the LOAM-iVox kernel (dynamic work distribution)
    DevBuf<uint4> ll_rows;      // LL hand-over records of the persistent LOAM-iVox kernel: [grid][32] rows + pose record
    unsigned match_epoch = 0;   // tag prefix of those records
    unsigned char* h_batch = nullptr;  // pinned staging of the per-batch tables (poses, offsets, scan descriptors, CTA map, pointers)
    size_t h_batch_cap = 0;
    DevBuf<unsigned char> d_batch;
    DevBuf<GnState> state;
    GnState* h_state = nullptr;  // pinned
    DevBuf<fls_iter_log> log;
    std::vector<fls_iter_log> h_log;  // FLS_FLAG_ITER_LOG: log_cap entries per scan of the last Match
    int log_cap = 0;
    std::vector<int> log_n = {0};     // entries of each scan's log (one element per scan of the last Match)
    double T_final[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    cudaEvent_t prof_ev[2] = {nullptr, nullptr};  // FLS_FLAG_PROFILE: around the fused Gauss-Newton launch of a Match
    bool profile = false;
    long long per_point_iter_bytes = 0;  // fixed part of the algorithmic bytes per point-iteration (set by match_*)
    long long per_cand_bytes = 0;        // bytes per scanned map record
    BuildScratch scratch;                // voxel-grid passes of Match

    // optional caller-owned device buffer that receives {pose, converged, iterations} per scan (fls_set_result_buffer_device)
    double* result_buf = nullptr;
    size_t result_cap = 0;

    // source cloud of the last Match (for GetFitnessScore): device pointer + count
    const float4* last_src = nullptr;
    size_t last_src_n = 0;

    // maps
    IvoxMap ivox;      // LoamPointToPlaneIVOX
    NdtMap ndt;        // IncrementalNDT
    bool ndt_first_scan = true;  // flag_first_scan_ (incremental_ndt.h:394)
    bool have_last = false;  // `static last_T` of IsNeedAddCloud (icp_optimized.h:219, kd-tree plug-ins)  [quirk 7]
    double last_T[16];

    // IcpOptimized and the kd-tree LOAM plug-ins (LoamPointToPlaneKdtree, LoamFull): sliding window of clouds -> VoxelGrid ->
    // exact search grid
    struct Cloud {
        DevBuf<float4> buf;
        size_t n = 0;
    };
    struct WindowMap {
        std::deque<std::unique_ptr<Cloud>> deque;  // cloud_deque_ / planar_cloud_deque_ / corner_cloud_deque_
        DevBuf<float4> merged;                     // concatenation of the window
        DevBuf<float4> cloud;                      // what upstream builds the kd-tree on
        size_t n = 0;
        IvoxMap grid;                              // floor-keyed uniform grid over `cloud`
    };
    WindowMap icp_map;  // cloud_deque_ / local_map_ptr_ (icp_optimized.h:173-187, 246)
    WindowMap kd_planar, kd_corner;
    DevBuf<double> rec_d;       // persistent {J[6], residual} records of the kd-tree plug-ins
    DevBuf<float4> src2;        // uploaded corner features (LoamFull)

    // GetFitnessScore support: cloud the upstream kd-tree is built on (fit_pts: fit_cloud, or the ICP window's filtered map)
    // + a search grid sized for max_range
    DevBuf<float4> fit_cloud;
    const float4* fit_pts = nullptr;
    size_t fit_cloud_n = 0;
    unsigned long long fit_cloud_version = 0, fit_grid_version = ~0ull;
    float fit_grid_range = -1.f;
    IvoxMap fit_grid;
    DevBuf<double> fit_out;

    explicit Handle(const fls_config& c);
    ~Handle();
    void init();     // body of the constructor
    void release();  // streams, events, pinned memory
    Handle(const Handle&) = delete;
    Handle& operator=(const Handle&) = delete;

    void begin_call();
    void end_call(fls_match_stats* st);
    const float4* upload(const void* pts, size_t n, size_t stride, DevBuf<float4>& dst);
    void upload_into(const void* pts, size_t n, size_t stride, float4* dst);  // dst: room for n records
    IvoxView ivox_view() const;
    IvoxView grid_view(const IvoxMap& g) const;
    void set_fit_cloud(const float4* d, size_t n);  // copies
    void set_fit_view(const float4* d, size_t n);   // refers to d until the next call

    // ---- the host half of a Match, shared by the plug-ins ----
    GnParams gn_params(int method, int min_effective) const;
    unsigned next_ll_epoch(size_t n_records);  // LL records for the next launch; returns its tag base
    fls_iter_log* scan_log(int s) { return log_cap ? log.p + (size_t)s * log_cap : nullptr; }
    double* scan_result(int s) { return (result_buf && (size_t)s < result_cap) ? result_buf + (size_t)s * kResultLen : nullptr; }
    unsigned char* batch_table(size_t bytes);  // pinned staging of a per-batch table ...
    void send_batch_table(size_t bytes);       // ... and its copy to d_batch
    // the fused Gauss-Newton launch: roofline byte rates, profile events around `launch`, the launch counter and the source
    // cloud GetFitnessScore reads afterwards
    template <class F>
    void gn_launch(long long point_iter_bytes, long long cand_bytes, const float4* src, size_t src_n, F&& launch) {
        per_point_iter_bytes = point_iter_bytes;
        per_cand_bytes = cand_bytes;
        if (profile) FLS_CUDA(cudaEventRecord(prof_ev[0], stream));
        launch();
        if (profile) FLS_CUDA(cudaEventRecord(prof_ev[1], stream));
        launches++;
        last_src = src;
        last_src_n = src_n;
    }
    void read_back(int n_scans);  // enqueues the copy of the states and of every scan's iteration log
    // after end_call: T / converged / stats and log_n of every scan (call-level figures on stats[0]), T_final from scan 0
    void unpack(int n_scans, const size_t* n_source, double* T, int* converged, fls_match_stats* st);

    int add_cloud_ivox(const void* pts, size_t n, size_t stride);
    int match_p2plane_ivox(const float4* d_src, size_t n, double* T, int* converged, fls_match_stats* st);
    // n_scans independent scans against the (static) map in ONE persistent launch; d_scans: host array of device pointers
    int match_ivox_batch(int n_scans, const float4* const* d_scans, const size_t* n, double* T, int* converged, fls_match_stats* st);
    // the same in two halves (fls_match_batch_begin / _end): enqueue without waiting, then wait + unpack
    int enqueue_ivox_batch(int n_scans, const float4* const* d_scans, const size_t* n, const double* T);
    int finish_ivox_batch(double* T, int* converged, fls_match_stats* st);
    std::vector<size_t> pend_n;  // scans of the batch in flight (empty: none)
    bool pend_v9 = false;
    unsigned* h_abort = nullptr;  // watchdog word of the last v9 launch (pinned, behind h_state; read back with the states)

    int add_cloud_ndt(const float4* d_cloud, size_t n);
    int match_ndt(const float4* d_src, size_t n, double* T, int* converged, fls_match_stats* st);
    int match_ndt_batch(int n_scans, const float4* const* d_scans, const size_t* n, double* T, int* converged, fls_match_stats* st);

    int add_cloud_icp(const float4* d_cloud, size_t n);
    int match_icp(const float4* d_src, size_t n, double* T, int* converged, fls_match_stats* st);

    // filter_mode 0: always VoxelGrid(leaf); 1: only once the window holds more than 5 clouds (loam_full_kdtree.h:91-99)
    int window_add(WindowMap& w, const float4* d_cloud, size_t n, size_t window, float leaf, int filter_mode, bool replace);
    int add_cloud_kd(const float4* d_planar, size_t n_planar, const float4* d_corner, size_t n_corner);
    int match_kd(const float4* d_planar, size_t n_planar, const float4* d_corner, size_t n_corner, double* T, int* converged, fls_match_stats* st);
    bool need_add_cloud(const double* T);

    int fitness(float max_range, float* score);

    // localization-mode map path (fls_localmap.cu): resident global map, +-100 m crop around the pose when needed
    DevBuf<float4> global_map;
    size_t global_n = 0;
    DevBuf<unsigned char> crop_keep;
    double local_edge[6] = {0, 0, 0, 0, 0, 0};
    bool have_edge = false;
    int set_global_map(const void* pts, size_t n, size_t stride);
    int update_local_map(const double* T_colmajor, int* updated, size_t* n_local);
};

}  // namespace fls
