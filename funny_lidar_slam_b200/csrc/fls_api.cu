// fls_api.cu — the C ABI of include/fls_b200.h: handle lifetime, host<->device staging, GetFitnessScore and the host half of a
// Match that every plug-in shares.  Each plug-in's own Match / AddCloudToLocalMap sits next to its kernels (Plugin, fls_handle.h).
// The Gauss-Newton loop itself runs on the device (one persistent kernel per Match or per batch: residuals, 6x6 reduction, solve,
// pose update and stop rule); the host reads the 744-byte state block of every scan back once.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>

#include "fls_frontend.h"
#include "fls_gn.cuh"
#include "fls_handle.h"

namespace fls {

static thread_local std::string g_last_error;
void set_last_error(const std::string& s) { g_last_error = s; }
const char* last_error_cstr() { return g_last_error.c_str(); }

int check_device(int device) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || device < 0 || device >= n || device >= kMaxDevices) return FLS_ERR_NO_DEVICE;
    return FLS_OK;
}

Handle::Handle(const fls_config& c) : cfg(c) {
    try {
        init();
    } catch (...) {  // a throwing constructor does not run the destructor: give back what was acquired so far
        release();
        throw;
    }
}

void Handle::release() {
    for (auto& e : prof_ev) {
        if (e) cudaEventDestroy(e);
        e = nullptr;
    }
    if (call.e0) cudaEventDestroy(call.e0);
    if (call.e1) cudaEventDestroy(call.e1);
    call.e0 = call.e1 = nullptr;
    if (call.stream) cudaStreamDestroy(call.stream);
    call.stream = nullptr;
}

void Handle::init() {
    FLS_CUDA(cudaSetDevice(cfg.device));
    FLS_CUDA(cudaStreamCreateWithFlags(&call.stream, cudaStreamNonBlocking));
    FLS_CUDA(cudaEventCreate(&call.e0));
    FLS_CUDA(cudaEventCreate(&call.e1));
    h_state.reserve(kMaxBatch);
    state.reserve(kMaxBatch);
    switch (cfg.method) {
        case FLS_P2PLANE_IVOX: plugin = make_ivox_plugin(*this); break;
        case FLS_NDT: plugin = make_ndt_plugin(*this); break;
        case FLS_ICP_P2P: plugin = make_icp_plugin(*this); break;
        default: plugin = make_kd_plugin(*this); break;  // FLS_P2PLANE_KNN, FLS_LOAM_FULL
    }
    profile = (cfg.flags & FLS_FLAG_PROFILE) != 0;
    if (profile)
        for (auto& e : prof_ev) FLS_CUDA(cudaEventCreate(&e));
    if (cfg.flags & FLS_FLAG_ITER_LOG) {
        log_cap = cfg.max_iterations > 0 ? cfg.max_iterations : 1;
        log.reserve((size_t)log_cap * kMaxBatch);
        h_log.resize((size_t)log_cap * kMaxBatch);
    }
    if (cfg.flags & FLS_FLAG_INFORMATION) {
        info_on = true;
        info.reserve(kMaxBatch);
        h_info.reserve(kMaxBatch);
    }
}

Handle::~Handle() {
    cudaSetDevice(cfg.device);
    if (call.stream) cudaStreamSynchronize(call.stream);
    release();
}

// Copy a caller cloud (host memory, `stride` bytes per record) into packed float4 device memory.
void Handle::upload_into(const void* pts, size_t n, size_t stride, float4* dst) {
    upload_records(pts, n, stride, dst, raw, call);
}

const float4* Handle::upload(const void* pts, size_t n, size_t stride, DevBuf<float4>& dst) {
    dst.reserve(n);
    upload_into(pts, n, stride, dst.p);
    return dst.p;
}

int Handle::begin_batch(int B, const void* const* scans, const size_t* n, size_t host_stride, const float4** ptrs, fls_match_stats* st) {
    if (st) std::memset(st, 0, sizeof(*st) * (size_t)B);
    begin_call();
    size_t total = 0, n_max = 0;
    for (int s = 0; s < B; ++s) {
        if (!scans[s] && n[s]) return FLS_ERR_INVALID_ARG;
        total += n[s];
        n_max = std::max(n_max, n[s]);
    }
    if (!host_stride) {
        for (int s = 0; s < B; ++s) ptrs[s] = static_cast<const float4*>(scans[s]);
        return FLS_OK;
    }
    src.reserve(total + 1);
    if (host_stride != FLS_LAYOUT_PACKED) raw.reserve(n_max * host_stride);
    size_t off = 0;
    for (int s = 0; s < B; ++s) {
        ptrs[s] = src.p + off;
        upload_into(scans[s], n[s], host_stride, src.p + off);
        off += n[s];
    }
    return FLS_OK;
}

void Handle::begin_call() {
    FLS_CUDA(cudaSetDevice(cfg.device));
    call.begin();
}

void Handle::set_fit_cloud(const float4* d, size_t n) {
    fit_cloud.reserve(n);
    if (n) FLS_CUDA(cudaMemcpyAsync(fit_cloud.p, d, n * sizeof(float4), cudaMemcpyDeviceToDevice, call.stream));
    set_fit_view(fit_cloud.p, n);
}

void Handle::set_fit_view(const float4* d, size_t n) {
    fit_pts = d;
    fit_cloud_n = n;
    fit_cloud_version++;
}

// ---- the host half of a Match ----------------------------------------------------------------------------------------
GnParams Handle::gn_params(int method, int min_effective) const {
    GnParams p;
    p.method = method;
    p.max_iterations = cfg.max_iterations;
    p.min_effective = min_effective;
    p.rot_thres = cfg.rotation_converge_thres;
    p.pos_thres = cfg.position_converge_thres;
    return p;
}

// LL hand-over records (fls_gn.cuh): never cleared, since tags are unique per Match and iteration; zeroed only when
// (re)allocated, so that uninitialised memory cannot alias a tag
unsigned Handle::next_ll_epoch(size_t n_records) {
    const size_t cap0 = ll_rows.cap;
    ll_rows.reserve(n_records);
    if (ll_rows.cap != cap0) FLS_CUDA(cudaMemsetAsync(ll_rows.p, 0, ll_rows.cap * sizeof(uint4), call.stream));
    match_epoch = (match_epoch + 1) & 0xffffffu;
    if (match_epoch == 0) match_epoch = 1;
    return match_epoch << 8;
}

void Handle::read_back(int B) {
    // h_log is about to hold this call's logs: until unpack records their sizes, no scan has one (a Match that fails after
    // its launch, e.g. through the v9 watchdog, leaves no log rather than a mix of two calls)
    log_n.assign(1, 0);
    FLS_CUDA(cudaMemcpyAsync(h_state.p, state.p, sizeof(GnState) * (size_t)B, cudaMemcpyDeviceToHost, call.stream));
    call.d2h += (long long)(sizeof(GnState) * (size_t)B);
    if (log_cap) {
        const size_t bytes = sizeof(fls_iter_log) * (size_t)log_cap * (size_t)B;
        FLS_CUDA(cudaMemcpyAsync(h_log.data(), log.p, bytes, cudaMemcpyDeviceToHost, call.stream));
        call.d2h += (long long)bytes;
    }
    info_n = 0;
    if (info_enqueued) {
        const size_t bytes = sizeof(fls_information) * (size_t)B;
        FLS_CUDA(cudaMemcpyAsync(h_info.p, info.p, bytes, cudaMemcpyDeviceToHost, call.stream));
        call.d2h += (long long)bytes;
    }
}

void Handle::unpack(int B, const size_t* n, double* T, int* converged, fls_match_stats* st) {
    float kernel_ms = 0.f;
    if (profile) FLS_CUDA(cudaEventElapsedTime(&kernel_ms, prof_ev[0], prof_ev[1]));
    for (int s = 0; s < B; ++s) {
        const GnState& gs = h_state.p[s];
        gn_pose_T(gs.R, gs.t, T + 16 * s);
        if (converged) converged[s] = gs.converged;
        if (st) {
            fls_match_stats& o = st[s];
            if (s > 0) std::memset(&o, 0, sizeof(o));  // call-level figures (times, launches, copies) are reported on scan 0
            o.iterations = gs.iter;
            o.converged = gs.converged;
            o.n_source = (long long)n[s];
            o.n_valid = gs.n_valid;
            o.sum_residual = gs.sum_res;
            if (profile) {
                // algorithmic bytes are per scan; the launch and its time are shared by the batch and reported on scan 0
                o.algo_bytes = (long long)gs.iter * (long long)n[s] * per_point_iter_bytes + (long long)(gs.cand_total + 0.5) * per_cand_bytes;
                o.kernel_ms = s == 0 ? kernel_ms : 0.f;
                o.kernel_launches = s == 0 ? 1 : 0;
            }
        }
    }
    std::memcpy(T_final, T, sizeof(T_final));
    log_n.resize(B);
    for (int s = 0; s < B; ++s) log_n[s] = h_state.p[s].iter < log_cap ? h_state.p[s].iter : log_cap;
    info_n = info_enqueued ? B : 0;
    info_enqueued = false;
}

int Handle::filter_batch(int B, const float4* const* d, const size_t* n, float leaf, DevBuf<float4>& dst, size_t* off, size_t* ns) {
    // room for every distinct source: a scan that repeats an earlier (pointer, count) is filtered once (relocalization refines many
    // poses of one scan)
    auto first_of = [&](int s) {
        int first = 0;
        while (first < s && !(d[first] == d[s] && n[first] == n[s])) ++first;
        return first;
    };
    size_t total_in = 0;
    for (int s = 0; s < B; ++s)
        if (first_of(s) == s) total_in += n[s];
    dst.reserve(total_in + 1);
    size_t end = 0;
    for (int s = 0; s < B; ++s) {
        const int first = first_of(s);
        if (first < s) {
            off[s] = off[first];
            ns[s] = ns[first];
            continue;
        }
        const size_t nf = voxel_grid_device(d[s], n[s], leaf, dst.p + end, scratch, call);
        if (nf > 0x3fffffffull) return FLS_ERR_INVALID_ARG;
        off[s] = end;
        ns[s] = nf;
        end += nf;
    }
    return FLS_OK;
}

int Handle::inserted(int rc, fls_match_stats* st) {
    call.sync();
    if (st) st->gpu_launches = call.launches;
    return rc;
}

// IsNeedAddCloud of the ICP and kd-tree LOAM plug-ins
bool KeyFrameGate::need(const double* T, double dist_thre, double rot_thre) {
    if (!have_last) {
        std::memcpy(last_T, T, 16 * sizeof(double));
        have_last = true;
    }
    const GnPose last = gn_pose(last_T), cur = gn_pose(T);
    const double* Rl = last.R;
    double Rli[9], Rd[9];
    {  // 3x3 inverse by cofactors
        const double c00 = Rl[4] * Rl[8] - Rl[5] * Rl[7], c01 = Rl[5] * Rl[6] - Rl[3] * Rl[8], c02 = Rl[3] * Rl[7] - Rl[4] * Rl[6];
        const double id = 1.0 / (Rl[0] * c00 + Rl[1] * c01 + Rl[2] * c02);
        Rli[0] = c00 * id; Rli[1] = (Rl[2] * Rl[7] - Rl[1] * Rl[8]) * id; Rli[2] = (Rl[1] * Rl[5] - Rl[2] * Rl[4]) * id;
        Rli[3] = c01 * id; Rli[4] = (Rl[0] * Rl[8] - Rl[2] * Rl[6]) * id; Rli[5] = (Rl[2] * Rl[3] - Rl[0] * Rl[5]) * id;
        Rli[6] = c02 * id; Rli[7] = (Rl[1] * Rl[6] - Rl[0] * Rl[7]) * id; Rli[8] = (Rl[0] * Rl[4] - Rl[1] * Rl[3]) * id;
    }
    mat3_mul(Rli, cur.R, Rd);
    const double roll = std::atan2(Rd[7], Rd[8]), pitch = std::asin(-Rd[6]), yaw = std::atan2(Rd[3], Rd[0]);
    const double dt[3] = {T[12] - last_T[12], T[13] - last_T[13], T[14] - last_T[14]};
    if (norm3(dt) > dist_thre || std::fabs(roll) > rot_thre || std::fabs(pitch) > rot_thre || std::fabs(yaw) > rot_thre) {
        std::memcpy(last_T, T, 16 * sizeof(double));
        return true;
    }
    return false;
}

}  // namespace fls

// =====================================================================================================================
using fls::check_device;
using fls::Handle;
using fls::Plugin;
using fls::stride_ok;

// the configuration check fls_preprocess_loam and fls_preprocess_loam_device share
static bool loam_frontend_cfg_ok(const fls_loam_frontend_cfg& c) {
    return c.n_rows > 0 && c.n_cols > 0 && (long long)c.n_rows * c.n_cols <= 0x7fffffffll && c.horizontal_resolution > 0.f && c.corner_leaf > 0.f &&
           c.planar_leaf > 0.f &&
           // the reference CHECK_NE()s both feature thresholds against FloatNaN (feature_extractor.cpp:19-20)
           c.corner_threshold < 3.0e38f && c.planar_threshold < 3.0e38f;
}

// The body velocity of the *_motion entries: NULL (rotation only), or three finite components.  Checked before anything is written.
static bool velocity_ok(const double* v) { return !v || (std::isfinite(v[0]) && std::isfinite(v[1]) && std::isfinite(v[2])); }

// Every Match entry runs through this: the call starts without an information record and leaves one only when it returns FLS_OK
// (an argument check, a refusal or an error caught by FLS_CATCH all leave none).
template <class F>
static int info_scoped(fls_handle* hh, F&& call) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    if (h) h->info_reset();
    const int rc = call();
    if (h && rc != FLS_OK) h->info_reset();
    return rc;
}

// stage buffers of fls_voxel_grid
struct VoxelWorkspace : fls::Workspace {
    fls::DevBuf<unsigned char> raw;
    fls::DevBuf<float4> in, out;
    fls::BuildScratch sc;
};

extern "C" {

int fls_abi_version(void) { return FLS_ABI_VERSION; }

int fls_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

const char* fls_last_error(void) { return fls::last_error_cstr(); }

int fls_project(int device, const void* raw, const int32_t* ring, size_t n, size_t stride, int32_t n_rows, int32_t n_cols, float horizontal_resolution,
                float min_distance, float max_distance, float* ordered, float* depth, int32_t* col, int32_t* row_start, int32_t* row_end,
                size_t* n_ordered) {
    if ((!raw && n) || (!ring && n) || !ordered || !depth || !col || !row_start || !row_end || !n_ordered || !stride_ok(stride))
        return FLS_ERR_INVALID_ARG;
    if (check_device(device) != FLS_OK) return FLS_ERR_NO_DEVICE;
    FLS_TRY
    return fls::project_device(device, raw, ring, nullptr, nullptr, nullptr, n, stride, n_rows, n_cols, horizontal_resolution, min_distance, max_distance, ordered,
                               depth, col, row_start, row_end, n_ordered);
    FLS_CATCH
}

// fls_project_imu and fls_project_imu_motion (vel NULL: rotation only)
static int project_imu_entry(int device, const void* raw, const int32_t* ring, const float* time, size_t n, size_t stride, const fls_imu_buffer* imu,
                             const double* vel, int32_t n_rows, int32_t n_cols, float horizontal_resolution, float min_distance, float max_distance,
                             float* ordered, float* depth, int32_t* col, int32_t* row_start, int32_t* row_end, size_t* n_ordered) {
    if ((!raw && n) || (!ring && n) || !ordered || !depth || !col || !row_start || !row_end || !n_ordered || !stride_ok(stride))
        return FLS_ERR_INVALID_ARG;
    if (imu && imu->n_imu && !time && n) return FLS_ERR_INVALID_ARG;
    if (check_device(device) != FLS_OK) return FLS_ERR_NO_DEVICE;
    FLS_TRY
    return fls::project_device(device, raw, ring, time, imu, vel, n, stride, n_rows, n_cols, horizontal_resolution, min_distance, max_distance, ordered,
                               depth, col, row_start, row_end, n_ordered);
    FLS_CATCH
}

int fls_project_imu(int device, const void* raw, const int32_t* ring, const float* time, size_t n, size_t stride, const fls_imu_buffer* imu,
                    int32_t n_rows, int32_t n_cols, float horizontal_resolution, float min_distance, float max_distance, float* ordered, float* depth,
                    int32_t* col, int32_t* row_start, int32_t* row_end, size_t* n_ordered) {
    return project_imu_entry(device, raw, ring, time, n, stride, imu, nullptr, n_rows, n_cols, horizontal_resolution, min_distance, max_distance, ordered,
                             depth, col, row_start, row_end, n_ordered);
}

int fls_project_imu_motion(int device, const void* raw, const int32_t* ring, const float* time, size_t n, size_t stride, const fls_imu_buffer* imu,
                           int32_t n_rows, int32_t n_cols, float horizontal_resolution, float min_distance, float max_distance, float* ordered,
                           float* depth, int32_t* col, int32_t* row_start, int32_t* row_end, size_t* n_ordered, const double velocity_imu[3]) {
    if (!velocity_ok(velocity_imu)) return FLS_ERR_INVALID_ARG;
    return project_imu_entry(device, raw, ring, time, n, stride, imu, velocity_imu, n_rows, n_cols, horizontal_resolution, min_distance, max_distance,
                             ordered, depth, col, row_start, row_end, n_ordered);
}

// fls_preprocess and fls_preprocess_motion
static int preprocess_entry(int device, const float* raw_xyzit, size_t n, const fls_imu_buffer* imu, const double* vel, float min_distance,
                            float max_distance, int32_t jump_span, float planar_leaf, float* ordered, size_t* n_ordered, float* planar, size_t* n_planar) {
    if ((!raw_xyzit && n) || !ordered || !planar || !n_ordered || !n_planar || jump_span < 1 || !(planar_leaf > 0.f)) return FLS_ERR_INVALID_ARG;
    if (check_device(device) != FLS_OK) return FLS_ERR_NO_DEVICE;
    FLS_TRY
    return fls::preprocess_device(device, raw_xyzit, n, imu, vel, min_distance, max_distance, jump_span, planar_leaf, ordered, n_ordered, planar, n_planar);
    FLS_CATCH
}

int fls_preprocess(int device, const float* raw_xyzit, size_t n, const fls_imu_buffer* imu, float min_distance, float max_distance, int32_t jump_span,
                   float planar_leaf, float* ordered, size_t* n_ordered, float* planar, size_t* n_planar) {
    return preprocess_entry(device, raw_xyzit, n, imu, nullptr, min_distance, max_distance, jump_span, planar_leaf, ordered, n_ordered, planar, n_planar);
}

int fls_preprocess_motion(int device, const float* raw_xyzit, size_t n, const fls_imu_buffer* imu, float min_distance, float max_distance,
                          int32_t jump_span, float planar_leaf, float* ordered, size_t* n_ordered, float* planar, size_t* n_planar,
                          const double velocity_imu[3]) {
    if (!velocity_ok(velocity_imu)) return FLS_ERR_INVALID_ARG;
    return preprocess_entry(device, raw_xyzit, n, imu, velocity_imu, min_distance, max_distance, jump_span, planar_leaf, ordered, n_ordered, planar,
                            n_planar);
}

const char* fls_strerror(int status) {
    switch (status) {
        case FLS_OK: return "ok";
        case FLS_ERR_INVALID_ARG: return "invalid argument";
        case FLS_ERR_CUDA: return "CUDA runtime error (see fls_last_error)";
        case FLS_ERR_NO_DEVICE: return "no sm_90 CUDA device (this library has no CPU fallback)";
        case FLS_ERR_UNSUPPORTED: return "method or mode not supported by this build";
        case FLS_ERR_NO_MAP: return "Match called before AddCloudToLocalMap";
        case FLS_ERR_CAPACITY: return "voxel capacity reached (LRU eviction is not emulated on the device)";
        case FLS_ERR_TOO_FEW_POINTS: return "too few points";
        default: return "unknown status";
    }
}

int fls_config_default(fls_config* c, int method) {
    if (!c || method < 0 || method > FLS_LOAM_FULL) return FLS_ERR_INVALID_ARG;
    std::memset(c, 0, sizeof(*c));
    c->method = method;
    c->device = 0;
    c->localization_mode = 1;
    c->max_iterations = 10;               // config/localization/config_turing.yaml:49
    c->position_converge_thres = 0.01;    // :51
    c->rotation_converge_thres = 0.01;    // :52
    c->point_to_planar_thres = 0.1;       // :50
    c->ivox_resolution = 0.5f;            // loam_point_to_plane_ivox.h:55
    c->ivox_nearby = FLS_NEARBY18;        // :56
    c->ivox_capacity = 1000000;           // ivox_map.h:35
    c->ivox_max_range = 5.0f;             // ivox_map.h:58
    c->ivox_k = 5;                        // ivox_map.h:57
    c->ndt_voxel_size = 1.0;              // config/mapping/config_nclt_ndt.yaml:42-51
    c->ndt_outlier_thres = 5.0;
    c->ndt_min_points_in_voxel = 5;
    c->ndt_max_points_in_voxel = 50;
    c->ndt_min_effective_pts = 50;
    c->ndt_capacity = 100000;
    c->icp_max_correspond_distance = 1.0;  // config/localization/config_nclt_icp.yaml:42-48
    c->rot_thre_add_cloud = 0.2;
    c->dist_thre_add_cloud = 1.0;
    c->local_map_size = 50;
    c->source_cloud_filter_size = 0.2f;
    c->map_cloud_filter_size = 0.4f;
    c->point_search_thres = 1.0;
    c->line_ratio_thres = 3.0;
    c->corner_map_filter_size = 0.2f;
    c->corner_local_map_size = 50;
    if (method == FLS_NDT) {
        c->max_iterations = 30;
        c->position_converge_thres = 0.005;
        c->rotation_converge_thres = 0.005;
    } else if (method == FLS_ICP_P2P) {
        c->max_iterations = 30;
        c->position_converge_thres = 0.005;
        c->rotation_converge_thres = 0.005;
        c->source_cloud_filter_size = 0.4f;
    } else if (method == FLS_P2PLANE_KNN) {
        c->max_iterations = 8;  // config/localization/config_nclt.yaml:45
        c->position_converge_thres = 0.005;
        c->rotation_converge_thres = 0.005;
        c->map_cloud_filter_size = 0.5f;
    } else if (method == FLS_LOAM_FULL) {
        c->max_iterations = 30;  // config/mapping/config_nclt_loam_full.yaml:40-58
        c->rotation_converge_thres = 0.05;
        c->point_to_planar_thres = 0.2;
    }
    return FLS_OK;
}

static int validate(const fls_config* c) {
    if (!c) return FLS_ERR_INVALID_ARG;
    if (c->method < 0 || c->method > FLS_LOAM_FULL) return FLS_ERR_INVALID_ARG;
    // the reference CHECK_NE()s every threshold against its "NaN" sentinel = numeric_limits::max (constant_variable.h:10-15)
    if (c->max_iterations <= 0 || c->max_iterations == 2147483647) return FLS_ERR_INVALID_ARG;
    if (c->max_iterations > 254) return FLS_ERR_UNSUPPORTED;  // 8-bit iteration field of the hand-over tags (fls_gn.cuh); upstream configs use 8-30
    if (!(c->position_converge_thres < 1e300) || !(c->rotation_converge_thres < 1e300)) return FLS_ERR_INVALID_ARG;
    if (c->ivox_nearby < 0 || c->ivox_nearby > 3) return FLS_ERR_INVALID_ARG;
    if (c->method == FLS_P2PLANE_IVOX) {
        if (!(c->point_to_planar_thres < 1e300) || !(c->ivox_resolution > 0.f)) return FLS_ERR_INVALID_ARG;
        if (c->ivox_k != 5) return FLS_ERR_UNSUPPORTED;  // upstream always asks for 5 (loam_point_to_plane_ivox.h:269)
    } else if (c->method == FLS_NDT) {
        if (!(c->ndt_voxel_size > 0) || !(c->ndt_voxel_size < 1e300) || !(c->ndt_outlier_thres < 1e300) || !(c->source_cloud_filter_size > 0.f) ||
            c->ndt_capacity <= 0 || c->ndt_capacity == 2147483647 || c->ndt_min_points_in_voxel < 0 || c->ndt_min_points_in_voxel > 64)
            return FLS_ERR_INVALID_ARG;
    } else if (c->method == FLS_ICP_P2P) {
        if (!(c->icp_max_correspond_distance > 0) || !(c->icp_max_correspond_distance < 1e300) || !(c->source_cloud_filter_size > 0.f) ||
            !(c->map_cloud_filter_size > 0.f) || c->local_map_size <= 0)
            return FLS_ERR_INVALID_ARG;
    } else if (c->method == FLS_P2PLANE_KNN) {
        if (!(c->point_to_planar_thres < 1e300) || !(c->rot_thre_add_cloud < 1e300) || !(c->dist_thre_add_cloud < 1e300) ||
            !(c->map_cloud_filter_size > 0.f) || c->local_map_size <= 0)
            return FLS_ERR_INVALID_ARG;  // loam_point_to_plane_kdtree.h:43-50
    } else {
        if (!(c->point_to_planar_thres < 1e300) || !(c->point_search_thres < 1e300) || !(c->point_search_thres > 0) ||
            !(c->line_ratio_thres < 1e300) || !(c->rot_thre_add_cloud < 1e300) || !(c->dist_thre_add_cloud < 1e300) ||
            !(c->map_cloud_filter_size > 0.f) || !(c->corner_map_filter_size > 0.f) || c->local_map_size <= 0 || c->corner_local_map_size <= 0)
            return FLS_ERR_INVALID_ARG;  // loam_full_kdtree.h:41-53
    }
    return FLS_OK;
}

int fls_create(const fls_config* cfg, fls_handle** out) {
    if (!out) return FLS_ERR_INVALID_ARG;
    *out = nullptr;
    const int v = validate(cfg);
    if (v != FLS_OK) return v;
    if (check_device(cfg->device) != FLS_OK) {
        fls::set_last_error("no usable CUDA device");
        return FLS_ERR_NO_DEVICE;
    }
    FLS_TRY
    FLS_CUDA(cudaSetDevice(cfg->device));  // the handle's members allocate on the device they serve
    Handle* h = new Handle(*cfg);
    *out = reinterpret_cast<fls_handle*>(h);
    return FLS_OK;
    FLS_CATCH
}

void fls_destroy(fls_handle* h) { delete reinterpret_cast<Handle*>(h); }

int fls_add_cloud(fls_handle* hh, int n_clouds, const void* const* pts, const size_t* n, size_t stride) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    if (!h || !pts || !n || n_clouds < 1 || !stride_ok(stride)) return FLS_ERR_INVALID_ARG;
    // CHECK_EQ(cloud_list.size(), 1) everywhere except LoamFull, which takes {planar, corner} (loam_full_kdtree.h:66-68)
    const bool two = h->plugin->reads == Plugin::kPlanarCorner;
    if (n_clouds != (two ? 2 : 1)) return FLS_ERR_INVALID_ARG;
    for (int k = 0; k < n_clouds; ++k)
        if (!pts[k] && n[k]) return FLS_ERR_INVALID_ARG;
    FLS_TRY
    h->begin_call();
    int rc = h->plugin->add_check();
    if (rc == FLS_OK) {
        const float4* d = h->upload(pts[0], n[0], stride, h->up_cloud);
        const float4* dc = two ? h->upload(pts[1], n[1], stride, h->up_corner) : nullptr;
        rc = h->plugin->add_cloud(d, n[0], dc, two ? n[1] : 0);
    }
    h->call.end(nullptr);
    return rc;
    FLS_CATCH
}

// A single-scan Match on the clouds the plug-in reads: the ordered scan (NDT, ICP), the planar features (LOAM-iVox, kd-tree
// point-to-plane) or the planar and corner features (LoamFull).  FLS_ERR_INVALID_ARG when one of them is NULL but not empty.
// The clouds are host records of `host_stride` bytes, uploaded here, or (host_stride 0) packed float4 already on the device.
static int match_clouds(Handle* h, const void* ordered, size_t n_ordered, const void* planar, size_t n_planar, const void* corner, size_t n_corner,
                        size_t host_stride, double* T, int* converged, fls_match_stats* st) {
    if (!h || !T) return FLS_ERR_INVALID_ARG;
    const Plugin::Clouds reads = h->plugin->reads;
    const void* p = reads == Plugin::kOrdered ? ordered : planar;
    const size_t n = reads == Plugin::kOrdered ? n_ordered : n_planar;
    const bool two = reads == Plugin::kPlanarCorner;
    if (!p && n) return FLS_ERR_INVALID_ARG;
    if (two && !corner && n_corner) return FLS_ERR_INVALID_ARG;
    FLS_TRY
    if (st) std::memset(st, 0, sizeof(*st));
    h->begin_call();
    auto dev = [&](const void* q, size_t m, fls::DevBuf<float4>& buf) {
        return host_stride ? h->upload(q, m, host_stride, buf) : static_cast<const float4*>(q);
    };
    const float4* d = dev(p, n, h->src);
    const float4* dc = two ? dev(corner, n_corner, h->src2) : nullptr;
    return h->plugin->match(d, n, dc, two ? n_corner : 0, T, converged, st);
    FLS_CATCH
}

int fls_match(fls_handle* hh, const void* ordered, size_t n_ordered, const void* planar, size_t n_planar, const void* corner, size_t n_corner,
              size_t stride, double T[16], int* converged, fls_match_stats* st) {
    return info_scoped(hh, [&] {
        if (!stride_ok(stride)) return (int)FLS_ERR_INVALID_ARG;
        return match_clouds(reinterpret_cast<Handle*>(hh), ordered, n_ordered, planar, n_planar, corner, n_corner, stride, T, converged, st);
    });
}

int fls_match_device(fls_handle* hh, const void* d_points, size_t n, double T[16], int* converged, fls_match_stats* st) {
    return info_scoped(hh, [&] {
        Handle* h = reinterpret_cast<Handle*>(hh);
        // LoamFull reads two feature clouds: fls_match_cluster_device
        if (h && T && h->plugin->reads == Plugin::kPlanarCorner) return (int)(!d_points && n ? FLS_ERR_INVALID_ARG : FLS_ERR_UNSUPPORTED);
        // the one cloud is the ordered scan or the planar features, whichever the plug-in reads
        return match_clouds(h, d_points, n, d_points, n, nullptr, 0, 0, T, converged, st);
    });
}

int fls_match_cluster_device(fls_handle* hh, const void* d_ordered, size_t n_ordered, const void* d_planar, size_t n_planar, const void* d_corner,
                             size_t n_corner, double T[16], int* converged, fls_match_stats* st) {
    return info_scoped(hh, [&] {
        return match_clouds(reinterpret_cast<Handle*>(hh), d_ordered, n_ordered, d_planar, n_planar, d_corner, n_corner, 0, T, converged, st);
    });
}

// A batch Match of host scans of `host_stride` bytes or (0) device scans.  Scans of one batch are matched against the same map state:
// only meaningful when Match does not modify the map.
static int match_batch(fls_handle* hh, int n_scans, const void* const* scans, const size_t* n, size_t host_stride, double* T, int* converged,
                       fls_match_stats* st) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    if (!h || !scans || !n || !T || n_scans < 1 || n_scans > fls::kMaxBatch) return FLS_ERR_INVALID_ARG;
    if (n_scans > 1 && !h->cfg.localization_mode) return FLS_ERR_UNSUPPORTED;
    FLS_TRY
    return h->plugin->match_batch(n_scans, scans, n, host_stride, T, converged, st);
    FLS_CATCH
}

// The first half of a batch Match (fls_match_batch_begin*): the batch must find the same map when it ends, whatever its size.
static int batch_begin(fls_handle* hh, int n_scans, const void* const* scans, const size_t* n, size_t host_stride, const double* T) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    if (!h || !scans || !n || !T || n_scans < 1 || n_scans > fls::kMaxBatch) return FLS_ERR_INVALID_ARG;
    if (!h->cfg.localization_mode) return FLS_ERR_UNSUPPORTED;
    if (h->plugin->batch_pending()) return FLS_ERR_INVALID_ARG;  // one batch in flight per handle
    FLS_TRY
    return h->plugin->batch_begin(n_scans, scans, n, host_stride, T);
    FLS_CATCH
}

int fls_match_batch(fls_handle* hh, int n_scans, const void* const* planar, const size_t* n, size_t stride, double* T, int* converged,
                    fls_match_stats* st) {
    return info_scoped(hh, [&] { return stride_ok(stride) ? match_batch(hh, n_scans, planar, n, stride, T, converged, st) : (int)FLS_ERR_INVALID_ARG; });
}

int fls_match_batch_device(fls_handle* hh, int n_scans, const void* const* d_planar, const size_t* n, double* T, int* converged,
                           fls_match_stats* st) {
    return info_scoped(hh, [&] { return match_batch(hh, n_scans, d_planar, n, 0, T, converged, st); });
}

int fls_match_batch_begin(fls_handle* hh, int n_scans, const void* const* planar, const size_t* n, size_t stride, const double* T) {
    return info_scoped(hh, [&] { return stride_ok(stride) ? batch_begin(hh, n_scans, planar, n, stride, T) : (int)FLS_ERR_INVALID_ARG; });
}

int fls_match_batch_begin_device(fls_handle* hh, int n_scans, const void* const* d_planar, const size_t* n, const double* T) {
    return info_scoped(hh, [&] { return batch_begin(hh, n_scans, d_planar, n, 0, T); });
}

static int batch_end(Handle* h, double* T, int* converged, fls_match_stats* st) {
    if (!h || !T) return FLS_ERR_INVALID_ARG;
    const int B = h->plugin->batch_pending();
    if (!B) return FLS_ERR_INVALID_ARG;
    FLS_TRY
    if (st) std::memset(st, 0, sizeof(*st) * (size_t)B);
    return h->plugin->batch_end(T, converged, st);
    FLS_CATCH
}

int fls_match_batch_end(fls_handle* hh, double* T, int* converged, fls_match_stats* st) {
    // the records of the batch were enqueued by _begin (which left none readable): only an error clears them
    Handle* h = reinterpret_cast<Handle*>(hh);
    const int rc = batch_end(h, T, converged, st);
    if (h && rc != FLS_OK) h->info_reset();
    return rc;
}

int fls_fitness(fls_handle* hh, float max_range, float* score) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    if (!h || !score) return FLS_ERR_INVALID_ARG;
    FLS_TRY
    return h->fitness(max_range, score);
    FLS_CATCH
}

// fls_relocalize (wide: fls_relocalize_wide) of a host scan of `host_stride` bytes per record or (0) a device scan, or with guesses
// (G of them, checked by guesses_ok) fls_relocalize_multi: the checks that need no device first, then the plug-ins and modes without a batch Match in
// localization mode, which answer with no side effect
static int relocalize(fls_handle* hh, bool wide, const void* scan, size_t n, size_t host_stride, const fls_reloc_cfg* cfg, const double* guesses,
                      int G, double* T, fls_reloc_result* out, double* refined_T, int32_t* refined_converged, float* refined_fitness,
                      int64_t* refined_index, double* coarse_scores, size_t coarse_cap, int64_t* evaluations) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    if (h) h->info_reset();  // no record after any relocalization call
    if (!h || !cfg || !T || !out || (!scan && n) || (coarse_cap && !coarse_scores) || n > 0x3fffffffull) return FLS_ERR_INVALID_ARG;
    fls::RelocGrid g;
    const int v = fls::reloc_grid(*cfg, &g, wide);
    if (v != FLS_OK) return v;
    if (g.P > fls::kRelocWideMaxHypotheses / G) return FLS_ERR_INVALID_ARG;  // G * P > 2^31
    if (!h->cfg.localization_mode || (h->cfg.method != FLS_P2PLANE_IVOX && h->cfg.method != FLS_NDT)) return FLS_ERR_UNSUPPORTED;
    if (h->plugin->batch_pending()) return FLS_ERR_INVALID_ARG;  // one batch in flight per handle (fls_match_batch_begin)
    if (h->fit_cloud_n == 0) return FLS_ERR_NO_MAP;
    // the internal Matches of a relocalization do not evaluate their information
    struct Suspend {
        Handle* h;
        bool on;
        ~Suspend() {
            h->info_on = on;
            h->info_reset();
        }
    } suspend{h, h->info_on};
    h->info_on = false;
    FLS_TRY
    h->begin_call();
    const float4* d = host_stride ? h->upload(scan, n, host_stride, h->src) : static_cast<const float4*>(scan);
    return h->relocalize(d, n, *cfg, g, wide, guesses, G, T, out, refined_T, refined_converged, refined_fitness, refined_index, coarse_scores,
                         coarse_cap, evaluations);
    FLS_CATCH
}

int fls_relocalize(fls_handle* hh, const void* scan, size_t n, size_t stride, const fls_reloc_cfg* cfg, double T[16], fls_reloc_result* out,
                   double* refined_T, int32_t* refined_converged, float* refined_fitness, int64_t* refined_index, double* coarse_scores,
                   size_t coarse_cap) {
    if (!stride_ok(stride)) return FLS_ERR_INVALID_ARG;
    return relocalize(hh, false, scan, n, stride, cfg, T, 1, T, out, refined_T, refined_converged, refined_fitness, refined_index, coarse_scores,
                      coarse_cap, nullptr);
}

int fls_relocalize_device(fls_handle* hh, const void* d_scan, size_t n, const fls_reloc_cfg* cfg, double T[16], fls_reloc_result* out,
                          double* refined_T, int32_t* refined_converged, float* refined_fitness, int64_t* refined_index, double* coarse_scores,
                          size_t coarse_cap) {
    return relocalize(hh, false, d_scan, n, 0, cfg, T, 1, T, out, refined_T, refined_converged, refined_fitness, refined_index, coarse_scores,
                      coarse_cap, nullptr);
}

int fls_relocalize_wide(fls_handle* hh, const void* scan, size_t n, size_t stride, const fls_reloc_cfg* cfg, double T[16], fls_reloc_result* out,
                        double* refined_T, int32_t* refined_converged, float* refined_fitness, int64_t* refined_index, int64_t* evaluations) {
    if (!stride_ok(stride)) return FLS_ERR_INVALID_ARG;
    return relocalize(hh, true, scan, n, stride, cfg, T, 1, T, out, refined_T, refined_converged, refined_fitness, refined_index, nullptr, 0,
                      evaluations);
}

int fls_relocalize_wide_device(fls_handle* hh, const void* d_scan, size_t n, const fls_reloc_cfg* cfg, double T[16], fls_reloc_result* out,
                               double* refined_T, int32_t* refined_converged, float* refined_fitness, int64_t* refined_index, int64_t* evaluations) {
    return relocalize(hh, true, d_scan, n, 0, cfg, T, 1, T, out, refined_T, refined_converged, refined_fitness, refined_index, nullptr, 0, evaluations);
}

// fls_relocalize_multi's own checks: 1..64 guesses, every entry finite
static bool guesses_ok(const double* guesses, int G) {
    if (!guesses || G < 1 || G > fls::kRelocMaxGuesses) return false;
    for (int k = 0; k < 16 * G; ++k)
        if (!std::isfinite(guesses[k])) return false;
    return true;
}

int fls_relocalize_multi(fls_handle* hh, const void* scan, size_t n, size_t stride, const fls_reloc_cfg* cfg, const double* guesses, int32_t n_guesses,
                         double T[16], fls_reloc_result* out, double* refined_T, int32_t* refined_converged, float* refined_fitness,
                         int64_t* refined_index, int64_t* evaluations) {
    if (!stride_ok(stride) || !guesses_ok(guesses, n_guesses)) return FLS_ERR_INVALID_ARG;
    return relocalize(hh, true, scan, n, stride, cfg, guesses, n_guesses, T, out, refined_T, refined_converged, refined_fitness, refined_index, nullptr, 0,
                      evaluations);
}

int fls_relocalize_multi_device(fls_handle* hh, const void* d_scan, size_t n, const fls_reloc_cfg* cfg, const double* guesses, int32_t n_guesses,
                                double T[16], fls_reloc_result* out, double* refined_T, int32_t* refined_converged, float* refined_fitness,
                                int64_t* refined_index, int64_t* evaluations) {
    if (!guesses_ok(guesses, n_guesses)) return FLS_ERR_INVALID_ARG;
    return relocalize(hh, true, d_scan, n, 0, cfg, guesses, n_guesses, T, out, refined_T, refined_converged, refined_fitness, refined_index, nullptr, 0,
                      evaluations);
}

int fls_relocalize_wide_levels(const fls_handle* hh, int64_t* nodes, int capacity) {
    const Handle* h = reinterpret_cast<const Handle*>(hh);
    if (!h || capacity < 0 || (capacity && !nodes)) return FLS_ERR_INVALID_ARG;
    return h->relocalize_levels(nodes, capacity);
}

int fls_set_result_buffer_device(fls_handle* hh, double* d_results, size_t capacity_scans) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    if (!h || (d_results && capacity_scans == 0)) return FLS_ERR_INVALID_ARG;
    h->result_buf = d_results;
    h->result_cap = d_results ? capacity_scans : 0;
    return FLS_OK;
}

int fls_get_iter_log_scan(const fls_handle* hh, int scan, fls_iter_log* out, int capacity) {
    const Handle* h = reinterpret_cast<const Handle*>(hh);
    if (!h || !out || capacity < 0 || scan < 0 || (size_t)scan >= h->log_n.size()) return FLS_ERR_INVALID_ARG;
    const int n = h->log_n[scan] < capacity ? h->log_n[scan] : capacity;
    const fls_iter_log* src = h->h_log.data() + (size_t)scan * h->log_cap;
    for (int i = 0; i < n; ++i) out[i] = src[i];
    return n;
}

int fls_get_iter_log(const fls_handle* hh, fls_iter_log* out, int capacity) { return fls_get_iter_log_scan(hh, 0, out, capacity); }

int fls_set_global_map(fls_handle* hh, const void* pts, size_t n, size_t stride) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    if (!h || (!pts && n) || !stride_ok(stride)) return FLS_ERR_INVALID_ARG;
    FLS_TRY
    h->begin_call();
    const int rc = h->set_global_map(pts, n, stride);
    h->call.end(nullptr);
    return rc;
    FLS_CATCH
}

int fls_update_local_map(fls_handle* hh, const double* T, int* updated, size_t* n_local) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    if (!h || !T) return FLS_ERR_INVALID_ARG;
    FLS_TRY
    h->begin_call();
    const int rc = h->update_local_map(T, updated, n_local);
    h->call.end(nullptr);
    return rc;
    FLS_CATCH
}

int fls_pcd_read(const char* path, float* xyzi, size_t capacity, size_t* n) {
    if (!path || !n || (capacity && !xyzi)) return FLS_ERR_INVALID_ARG;
    FLS_TRY
    std::vector<float> v;
    std::string err;
    const int rc = fls::pcd_read(path, v, err);
    if (rc != FLS_OK) {
        fls::set_last_error(err);
        return rc;
    }
    *n = v.size() / 4;
    const size_t m = *n < capacity ? *n : capacity;
    if (m) std::memcpy(xyzi, v.data(), m * 16);
    return FLS_OK;
    FLS_CATCH
}

int fls_pcd_write(const char* path, const float* xyzi, size_t n) {
    if (!path || (!xyzi && n)) return FLS_ERR_INVALID_ARG;
    FLS_TRY
    std::string err;
    const int rc = fls::pcd_write(path, xyzi, n, err);
    if (rc != FLS_OK) fls::set_last_error(err);
    return rc;
    FLS_CATCH
}

int fls_get_voxel_keys(fls_handle* hh, int32_t* keys_xyz, size_t capacity, size_t* n) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    if (!h || !n || (capacity && !keys_xyz)) return FLS_ERR_INVALID_ARG;
    FLS_TRY
    std::vector<unsigned long long> packed;
    size_t n_vox = 0;
    const int rc = h->plugin->voxel_keys(packed, capacity, &n_vox);
    if (rc != FLS_OK) return rc;
    for (size_t i = 0; i < packed.size(); ++i) {
        const unsigned long long k = packed[i];
        const int c[3] = {(int)((k >> 42) & 0x1fffffu), (int)((k >> 21) & 0x1fffffu), (int)(k & 0x1fffffu)};
        for (int a = 0; a < 3; ++a) keys_xyz[3 * i + a] = (c[a] & 0x100000) ? c[a] - 0x200000 : c[a];  // 21-bit two's complement
    }
    *n = n_vox;
    return FLS_OK;
    FLS_CATCH
}

int fls_get_ndt_voxels(fls_handle* hh, fls_ndt_voxel* out, size_t capacity, size_t* n) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    if (!h || !n || (capacity && !out)) return FLS_ERR_INVALID_ARG;
    FLS_TRY
    std::vector<fls_ndt_voxel> v;
    const int rc = h->plugin->ndt_voxels(v);
    if (rc != FLS_OK) return rc;
    std::sort(v.begin(), v.end(), [](const fls_ndt_voxel& a, const fls_ndt_voxel& b) {
        return std::lexicographical_compare(a.key, a.key + 3, b.key, b.key + 3);
    });
    const size_t m = v.size() < capacity ? v.size() : capacity;
    if (m) std::memcpy(out, v.data(), m * sizeof(fls_ndt_voxel));
    *n = v.size();
    return FLS_OK;
    FLS_CATCH
}

int fls_get_map_points(fls_handle* hh, float* xyzi, size_t capacity, size_t* n) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    if (!h || !n || (capacity && !xyzi)) return FLS_ERR_INVALID_ARG;
    FLS_TRY
    return h->plugin->map_points(xyzi, capacity, n);
    FLS_CATCH
}

int fls_get_map_info(const fls_handle* hh, fls_map_info* out) {
    const Handle* h = reinterpret_cast<const Handle*>(hh);
    if (!h || !out) return FLS_ERR_INVALID_ARG;
    std::memset(out, 0, sizeof(*out));
    h->plugin->map_info(out);
    return FLS_OK;
}

int fls_ivox_add_points(fls_handle* hh, const void* pts, size_t n, size_t stride) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    if (!h || (!pts && n) || !stride_ok(stride)) return FLS_ERR_INVALID_ARG;
    FLS_TRY
    return h->plugin->ivox_add_points(pts, n, stride);
    FLS_CATCH
}

int fls_ivox_knn(fls_handle* hh, const void* queries, size_t n, size_t stride, int k, float* out_pts, int32_t* out_count) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    if (!h || !queries || !out_pts || !out_count || k != 5 || !stride_ok(stride)) return FLS_ERR_INVALID_ARG;
    FLS_TRY
    return h->plugin->ivox_knn(queries, n, stride, out_pts, out_count);
    FLS_CATCH
}

int fls_voxel_grid(int device, const void* pts, size_t n, size_t stride, float leaf, float* out, size_t* n_out) {
    if ((!pts && n) || !out || !n_out || !stride_ok(stride) || !(leaf > 0.f)) return FLS_ERR_INVALID_ARG;
    if (check_device(device) != FLS_OK) return FLS_ERR_NO_DEVICE;
    FLS_TRY
    *n_out = 0;
    if (n == 0) return FLS_OK;
    return fls::with_workspace<VoxelWorkspace>(device, [&](VoxelWorkspace& w) -> int {
        fls::Call& c = w.call;
        c.begin();
        w.in.reserve(n);
        w.out.reserve(n);
        fls::upload_records(pts, n, stride, w.in.p, w.raw, c);
        const size_t m = fls::voxel_grid_device(w.in.p, n, leaf, w.out.p, w.sc, c);
        FLS_CUDA(cudaMemcpyAsync(out, w.out.p, m * 16, cudaMemcpyDeviceToHost, c.stream));
        c.sync();
        *n_out = m;
        return FLS_OK;
    });
    FLS_CATCH
}

// fls_preprocess_loam and fls_preprocess_loam_motion
static int preprocess_loam_entry(const fls_loam_frontend_cfg* cfg, const void* raw, const int32_t* ring, const float* time, size_t n, size_t stride,
                                 const fls_imu_buffer* imu, const double* vel, float* corner, float* planar, float* d_corner, float* d_planar,
                                 size_t* n_corner, size_t* n_planar, fls_match_stats* stats) {
    if (!cfg || !n_corner || !n_planar) return FLS_ERR_INVALID_ARG;
    *n_corner = *n_planar = 0;
    if ((!raw && n) || (!ring && n) || !stride_ok(stride) || n > 0x7fffffffull) return FLS_ERR_INVALID_ARG;
    if (!corner && !planar && !d_corner && !d_planar) return FLS_ERR_INVALID_ARG;
    if (!loam_frontend_cfg_ok(*cfg)) return FLS_ERR_INVALID_ARG;
    if (imu && imu->n_imu && !time && n) return FLS_ERR_INVALID_ARG;
    if (check_device(cfg->device) != FLS_OK) return FLS_ERR_NO_DEVICE;
    FLS_TRY
    return fls::preprocess_loam_device(*cfg, raw, ring, time, n, stride, imu, vel, corner, planar, d_corner, d_planar, n_corner, n_planar, stats, false);
    FLS_CATCH
}

int fls_preprocess_loam(const fls_loam_frontend_cfg* cfg, const void* raw, const int32_t* ring, const float* time, size_t n, size_t stride,
                        const fls_imu_buffer* imu, float* corner, float* planar, float* d_corner, float* d_planar, size_t* n_corner, size_t* n_planar,
                        fls_match_stats* stats) {
    return preprocess_loam_entry(cfg, raw, ring, time, n, stride, imu, nullptr, corner, planar, d_corner, d_planar, n_corner, n_planar, stats);
}

int fls_preprocess_loam_motion(const fls_loam_frontend_cfg* cfg, const void* raw, const int32_t* ring, const float* time, size_t n, size_t stride,
                               const fls_imu_buffer* imu, float* corner, float* planar, float* d_corner, float* d_planar, size_t* n_corner,
                               size_t* n_planar, fls_match_stats* stats, const double velocity_imu[3]) {
    if (!velocity_ok(velocity_imu)) return FLS_ERR_INVALID_ARG;
    return preprocess_loam_entry(cfg, raw, ring, time, n, stride, imu, velocity_imu, corner, planar, d_corner, d_planar, n_corner, n_planar, stats);
}

// fls_preprocess_loam_device and fls_preprocess_loam_device_motion
static int preprocess_loam_device_entry(const fls_loam_frontend_cfg* cfg, const float* d_xyzi, const int32_t* d_ring, const float* d_time, size_t n,
                                        const fls_imu_buffer* imu, const double* vel, float* corner, float* planar, float* d_corner, float* d_planar,
                                        size_t* n_corner, size_t* n_planar, fls_match_stats* stats) {
    if (!cfg || !n_corner || !n_planar) return FLS_ERR_INVALID_ARG;
    *n_corner = *n_planar = 0;
    if ((!d_xyzi && n) || (!d_ring && n) || n > 0x7fffffffull) return FLS_ERR_INVALID_ARG;
    if (!corner && !planar && !d_corner && !d_planar) return FLS_ERR_INVALID_ARG;
    if (!loam_frontend_cfg_ok(*cfg)) return FLS_ERR_INVALID_ARG;
    if (imu && imu->n_imu && !d_time && n) return FLS_ERR_INVALID_ARG;
    if (check_device(cfg->device) != FLS_OK) return FLS_ERR_NO_DEVICE;
    FLS_TRY
    return fls::preprocess_loam_device(*cfg, d_xyzi, d_ring, d_time, n, FLS_LAYOUT_PACKED, imu, vel, corner, planar, d_corner, d_planar, n_corner,
                                       n_planar, stats, true);
    FLS_CATCH
}

int fls_preprocess_loam_device(const fls_loam_frontend_cfg* cfg, const float* d_xyzi, const int32_t* d_ring, const float* d_time, size_t n,
                               const fls_imu_buffer* imu, float* corner, float* planar, float* d_corner, float* d_planar, size_t* n_corner,
                               size_t* n_planar, fls_match_stats* stats) {
    return preprocess_loam_device_entry(cfg, d_xyzi, d_ring, d_time, n, imu, nullptr, corner, planar, d_corner, d_planar, n_corner, n_planar, stats);
}

int fls_preprocess_loam_device_motion(const fls_loam_frontend_cfg* cfg, const float* d_xyzi, const int32_t* d_ring, const float* d_time, size_t n,
                                      const fls_imu_buffer* imu, float* corner, float* planar, float* d_corner, float* d_planar, size_t* n_corner,
                                      size_t* n_planar, fls_match_stats* stats, const double velocity_imu[3]) {
    if (!velocity_ok(velocity_imu)) return FLS_ERR_INVALID_ARG;
    return preprocess_loam_device_entry(cfg, d_xyzi, d_ring, d_time, n, imu, velocity_imu, corner, planar, d_corner, d_planar, n_corner, n_planar, stats);
}

// fls_preprocess_device and fls_preprocess_device_motion
static int preprocess_device_entry(int device, const float* d_xyzi, const float* d_time, size_t n, const fls_imu_buffer* imu, const double* vel,
                                   float min_distance, float max_distance, int32_t jump_span, float planar_leaf, float* ordered, float* d_ordered,
                                   size_t* n_ordered, float* planar, float* d_planar, size_t* n_planar) {
    if (!n_ordered || !n_planar) return FLS_ERR_INVALID_ARG;
    *n_ordered = *n_planar = 0;
    if ((!d_xyzi && n) || (!ordered && !d_ordered && !planar && !d_planar) || jump_span < 1 || !(planar_leaf > 0.f)) return FLS_ERR_INVALID_ARG;
    if (imu && imu->n_imu && !d_time && n) return FLS_ERR_INVALID_ARG;
    if (check_device(device) != FLS_OK) return FLS_ERR_NO_DEVICE;
    FLS_TRY
    return fls::preprocess_device_input(device, d_xyzi, d_time, n, imu, vel, min_distance, max_distance, jump_span, planar_leaf, ordered, d_ordered,
                                        n_ordered, planar, d_planar, n_planar);
    FLS_CATCH
}

int fls_preprocess_device(int device, const float* d_xyzi, const float* d_time, size_t n, const fls_imu_buffer* imu, float min_distance,
                          float max_distance, int32_t jump_span, float planar_leaf, float* ordered, float* d_ordered, size_t* n_ordered, float* planar,
                          float* d_planar, size_t* n_planar) {
    return preprocess_device_entry(device, d_xyzi, d_time, n, imu, nullptr, min_distance, max_distance, jump_span, planar_leaf, ordered, d_ordered,
                                   n_ordered, planar, d_planar, n_planar);
}

int fls_preprocess_device_motion(int device, const float* d_xyzi, const float* d_time, size_t n, const fls_imu_buffer* imu, float min_distance,
                                 float max_distance, int32_t jump_span, float planar_leaf, float* ordered, float* d_ordered, size_t* n_ordered,
                                 float* planar, float* d_planar, size_t* n_planar, const double velocity_imu[3]) {
    if (!velocity_ok(velocity_imu)) return FLS_ERR_INVALID_ARG;
    return preprocess_device_entry(device, d_xyzi, d_time, n, imu, velocity_imu, min_distance, max_distance, jump_span, planar_leaf, ordered, d_ordered,
                                   n_ordered, planar, d_planar, n_planar);
}

int fls_convert_cloud(const fls_convert_cfg* cfg, const fls_pointcloud2* msg, float* xyzi, int32_t* ring, float* time, float* d_xyzi, int32_t* d_ring,
                      float* d_time, size_t* n, fls_convert_result* result, fls_match_stats* stats) {
    if (!cfg || !msg || !n || !result) return FLS_ERR_INVALID_ARG;
    *n = 0;
    const size_t cap = (size_t)msg->width * msg->height;
    if (cfg->lidar_type < FLS_LIDAR_VELODYNE || cfg->lidar_type > FLS_LIDAR_NONE || cfg->n_rows <= 0 || !std::isfinite(cfg->time_scale))
        return FLS_ERR_INVALID_ARG;
    // LidarModel's FLT_MAX sentinels of lower_angle_ / v_res_ (include/lidar/lidar_model.h:90-91) must be set for None
    if (cfg->lidar_type == FLS_LIDAR_NONE && (!(cfg->v_res > 0.f) || !(cfg->v_res < 3.0e38f) || !(std::fabs(cfg->lower_angle) < 3.0e38f)))
        return FLS_ERR_INVALID_ARG;
    if (cap > 0x7fffffffull || (cap && !msg->data) || (msg->n_fields && !msg->fields)) return FLS_ERR_INVALID_ARG;
    if ((size_t)msg->row_step < (size_t)msg->width * msg->point_step) return FLS_ERR_INVALID_ARG;
    for (uint32_t j = 0; j < msg->n_fields; ++j) {
        const fls_point_field& f = msg->fields[j];
        static const unsigned kSize[9] = {0, 1, 1, 2, 2, 4, 4, 4, 8};
        if (!f.name) return FLS_ERR_INVALID_ARG;
        if (f.datatype >= 1 && f.datatype <= 8 && (uint64_t)f.offset + (uint64_t)kSize[f.datatype] * (f.count ? f.count : 1) > msg->point_step)
            return FLS_ERR_INVALID_ARG;
    }
    if (msg->is_bigendian) return FLS_ERR_UNSUPPORTED;
    if (!xyzi && !ring && !time && !d_xyzi && !d_ring && !d_time) return FLS_ERR_INVALID_ARG;
    if (check_device(cfg->device) != FLS_OK) return FLS_ERR_NO_DEVICE;
    FLS_TRY
    return fls::convert_cloud_device(*cfg, *msg, xyzi, ring, time, d_xyzi, d_ring, d_time, n, result, stats);
    FLS_CATCH
}

int fls_extract_features(const fls_feature_cfg* cfg, const float* depth, const int32_t* col, size_t n, const int32_t* row_start,
                         const int32_t* row_end, int32_t n_rows, int32_t* corner_idx, size_t* n_corner, int32_t* planar_idx, size_t* n_planar,
                         fls_match_stats* stats) {
    if (!cfg || !depth || !col || !row_start || !row_end || !corner_idx || !n_corner || !planar_idx || !n_planar || n_rows < 0)
        return FLS_ERR_INVALID_ARG;
    // the reference CHECK_NE()s both thresholds against FloatNaN (feature_extractor.cpp:19-20)
    if (!(cfg->corner_threshold < 3.0e38f) || !(cfg->planar_threshold < 3.0e38f)) return FLS_ERR_INVALID_ARG;
    if (check_device(cfg->device) != FLS_OK) return FLS_ERR_NO_DEVICE;
    FLS_TRY
    return fls::extract_features_device(cfg->device, depth, col, n, row_start, row_end, n_rows, cfg->corner_threshold, cfg->planar_threshold,
                                        corner_idx, n_corner, planar_idx, n_planar, stats);
    FLS_CATCH
}

}  // extern "C"
