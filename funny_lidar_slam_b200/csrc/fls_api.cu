// fls_api.cu — the C ABI of include/fls_b200.h: handle lifetime, host<->device staging and the host side of
// each plug-in's Match / AddCloudToLocalMap / GetFitnessScore.  The Gauss-Newton loop itself runs on the
// device (one persistent kernel per Match or per batch: residuals, 6x6 reduction, solve, pose update and stop rule);
// the host reads the 744-byte state block of every scan back once.
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
    if (h_state) cudaFreeHost(h_state);
    h_state = nullptr;
    h_batch.release();
    for (auto& e : prof_ev) {
        if (e) cudaEventDestroy(e);
        e = nullptr;
    }
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    ev0 = ev1 = nullptr;
    if (stream) cudaStreamDestroy(stream);
    stream = nullptr;
}

void Handle::init() {
    FLS_CUDA(cudaSetDevice(cfg.device));
    FLS_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    FLS_CUDA(cudaEventCreate(&ev0));
    FLS_CUDA(cudaEventCreate(&ev1));
    FLS_CUDA(cudaMallocHost(&h_state, sizeof(GnState) * kMaxBatch + 64));
    h_abort = reinterpret_cast<unsigned*>(h_state + kMaxBatch);  // pinned: a copy into pageable memory would make the enqueue wait for the kernel
    *h_abort = 0;
    state.reserve(kMaxBatch);
    fit_out.reserve(2);
    ivox.set_resolution(cfg.ivox_resolution);
    ivox.key_mode = 0;
    ivox.incremental = cfg.method == FLS_P2PLANE_IVOX && !cfg.localization_mode;  // mapping mode: the map grows by small inserts
    {
        static const int counts[4] = {1, 7, 19, 27};
        ivox.n_stencil = counts[cfg.ivox_nearby];
    }
    ndt.configure(cfg.ndt_voxel_size, cfg.ndt_min_points_in_voxel, cfg.ndt_max_points_in_voxel, cfg.ndt_capacity);
    // search grid of the bounded exact 1-NN: cell >= sqrt(max_correspond_distance)  [quirk 4]
    icp_map.grid.key_mode = 1;
    icp_map.grid.set_resolution((float)(std::sqrt(cfg.icp_max_correspond_distance > 0 ? cfg.icp_max_correspond_distance : 1.0) * 1.001));
    fit_grid.key_mode = 1;
    // exact-search grids of the kd-tree plug-ins: LoamFull only needs neighbours inside sqrt(point_search_thres), so a cell
    // of that size settles every query in the 27-cell pass; the ungated point-to-plane variant uses ~2 map leafs
    kd_planar.grid.key_mode = kd_corner.grid.key_mode = 1;
    if (cfg.method == FLS_LOAM_FULL) {
        const float c = (float)(std::sqrt(cfg.point_search_thres > 0 ? cfg.point_search_thres : 1.0) * 1.001);
        kd_planar.grid.set_resolution(c);
        kd_corner.grid.set_resolution(c);
    } else {
        const float c = 2.0f * (cfg.map_cloud_filter_size > 0.f ? cfg.map_cloud_filter_size : 0.5f);
        kd_planar.grid.set_resolution(c < 0.8f ? 0.8f : c);
        kd_corner.grid.set_resolution(1.0f);
    }
    profile = (cfg.flags & FLS_FLAG_PROFILE) != 0;
    if (profile)
        for (auto& e : prof_ev) FLS_CUDA(cudaEventCreate(&e));
    if (cfg.flags & FLS_FLAG_ITER_LOG) {
        log_cap = cfg.max_iterations > 0 ? cfg.max_iterations : 1;
        log.reserve((size_t)log_cap * kMaxBatch);
        h_log.resize((size_t)log_cap * kMaxBatch);
    }
}

Handle::~Handle() {
    cudaSetDevice(cfg.device);
    if (stream) cudaStreamSynchronize(stream);
    release();
}

// Copy a caller cloud (host memory, `stride` bytes per record) into packed float4 device memory.
void Handle::upload_into(const void* pts, size_t n, size_t stride, float4* dst) {
    upload_records(pts, n, stride, dst, raw, stream, &h2d_bytes, &launches);
}

const float4* Handle::upload(const void* pts, size_t n, size_t stride, DevBuf<float4>& dst) {
    dst.reserve(n);
    upload_into(pts, n, stride, dst.p);
    return dst.p;
}

IvoxView Handle::grid_view(const IvoxMap& g) const {
    IvoxView v;
    v.pts = g.pts_sorted.p;
    v.tab = g.table.p;
    v.mask = g.mask;
    v.inv_res = g.inv_res;
    v.max_range2 = cfg.ivox_max_range * cfg.ivox_max_range;
    static const int counts[4] = {1, 7, 19, 27};
    v.n_stencil = counts[cfg.ivox_nearby];
    v.lists = g.lists.p;
    v.ctab = g.ctab.p;
    v.cmask = g.cmask;
    // a query and a candidate of its stencil differ by at most 2*res per axis with a non-zero offset and res otherwise:
    // d^2 <= 12 res^2 for the full 26-neighbourhood
    v.fast_knn = 12.0 * 1.01 * (double)g.res * (double)g.res < (double)v.max_range2 ? 1u : 0u;
    return v;
}
IvoxView Handle::ivox_view() const { return grid_view(ivox); }

void Handle::begin_call() {
    FLS_CUDA(cudaSetDevice(cfg.device));
    launches = 0;
    h2d_bytes = d2h_bytes = 0;
    FLS_CUDA(cudaEventRecord(ev0, stream));
}

void Handle::end_call(fls_match_stats* st) {
    FLS_CUDA(cudaEventRecord(ev1, stream));
    FLS_CUDA(cudaStreamSynchronize(stream));
    fill_call_stats(st, ev0, ev1, launches, h2d_bytes, d2h_bytes);
}

void Handle::set_fit_cloud(const float4* d, size_t n) {
    fit_cloud.reserve(n);
    if (n) FLS_CUDA(cudaMemcpyAsync(fit_cloud.p, d, n * sizeof(float4), cudaMemcpyDeviceToDevice, stream));
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
    if (ll_rows.cap != cap0) FLS_CUDA(cudaMemsetAsync(ll_rows.p, 0, ll_rows.cap * sizeof(uint4), stream));
    match_epoch = (match_epoch + 1) & 0xffffffu;
    if (match_epoch == 0) match_epoch = 1;
    return match_epoch << 8;
}

unsigned char* Handle::batch_table(size_t bytes) {
    d_batch.reserve(bytes);
    return h_batch.reserve(bytes);
}

void Handle::send_batch_table(size_t bytes) {
    FLS_CUDA(cudaMemcpyAsync(d_batch.p, h_batch.p, bytes, cudaMemcpyHostToDevice, stream));
    h2d_bytes += (long long)bytes;
}

void Handle::read_back(int B) {
    // h_log is about to hold this call's logs: until unpack records their sizes, no scan has one (a Match that fails after
    // its launch, e.g. through the v9 watchdog, leaves no log rather than a mix of two calls)
    log_n.assign(1, 0);
    FLS_CUDA(cudaMemcpyAsync(h_state, state.p, sizeof(GnState) * (size_t)B, cudaMemcpyDeviceToHost, stream));
    d2h_bytes += (long long)(sizeof(GnState) * (size_t)B);
    if (log_cap) {
        const size_t bytes = sizeof(fls_iter_log) * (size_t)log_cap * (size_t)B;
        FLS_CUDA(cudaMemcpyAsync(h_log.data(), log.p, bytes, cudaMemcpyDeviceToHost, stream));
        d2h_bytes += (long long)bytes;
    }
}

void Handle::unpack(int B, const size_t* n, double* T, int* converged, fls_match_stats* st) {
    float kernel_ms = 0.f;
    if (profile) FLS_CUDA(cudaEventElapsedTime(&kernel_ms, prof_ev[0], prof_ev[1]));
    for (int s = 0; s < B; ++s) {
        const GnState& gs = h_state[s];
        double* Ts = T + 16 * s;
        for (int r = 0; r < 3; ++r) {
            for (int c = 0; c < 3; ++c) Ts[c * 4 + r] = gs.R[r * 3 + c];
            Ts[12 + r] = gs.t[r];
        }
        Ts[3] = Ts[7] = Ts[11] = 0.0;
        Ts[15] = 1.0;
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
    for (int s = 0; s < B; ++s) log_n[s] = h_state[s].iter < log_cap ? h_state[s].iter : log_cap;
}

// control block of a single-scan persistent GN loop (K2 / K3 / K5): CTA rows + pose record + stop rule
static GnLoopCtl make_ctl(Handle& h, int method, int grid, int min_effective) {
    GnLoopCtl c;
    c.tag_base = h.next_ll_epoch((size_t)grid * 32 + kLlPoseLen);
    c.state = h.state.p;
    c.ll_rows = h.ll_rows.p;
    c.ll_pose = h.ll_rows.p + (size_t)grid * 32;
    c.gp = h.gn_params(method, min_effective);
    c.log = h.scan_log(0);
    c.log_cap = h.log_cap;
    c.result = h.scan_result(0);
    return c;
}

// single-scan Match: wait, then unpack
static void finish_match(Handle& h, double* T, int* converged, fls_match_stats* st, size_t n_source) {
    h.read_back(1);
    h.end_call(st);
    h.unpack(1, &n_source, T, converged, st);
}

// ---- LoamPointToPlaneIVOX ------------------------------------------------------------------------------------
int Handle::add_cloud_ivox(const void* pts, size_t n, size_t stride) {
    if (cfg.localization_mode) ivox.clear();  // loam_point_to_plane_ivox.h:64-69 upstream: map re-created per call
    else if (ivox.n_pts != 0) return FLS_ERR_UNSUPPORTED;  // external non-first insert relies on Match-internal caches upstream
    const float4* d = upload(pts, n, stride, stage);
    const int rc = ivox.append_and_build(d, n, cfg.ivox_capacity, stream);
    launches += ivox.launches;
    ivox.launches = 0;
    if (cfg.localization_mode) set_fit_cloud(d, n);  // :134-138 kd-tree over the raw planar cloud
    return rc;
}

// The whole LoamPointToPlaneIVOX Match of `n_scans` independent scans in one persistent launch (K1, fls_p2plane.cu).
// A single Match is the batch of one.
int Handle::match_ivox_batch(int B, const float4* const* d_scans, const size_t* n, double* T, int* converged, fls_match_stats* st) {
    const int rc = enqueue_ivox_batch(B, d_scans, n, T);
    if (rc != FLS_OK) return rc;
    return finish_ivox_batch(T, converged, st);
}

// everything of a batch up to the asynchronous read-back of the states: nothing here waits for the device
int Handle::enqueue_ivox_batch(int B, const float4* const* d_scans, const size_t* n, const double* T) {
    if (ivox.n_pts == 0) return FLS_ERR_NO_MAP;
    if (B < 1 || B > kMaxBatch) return FLS_ERR_INVALID_ARG;
    int off[kMaxBatch + 1];
    off[0] = 0;
    int grid = 1;
    // K1 generations: the dataflow kernel (v9: TMA-staged runs, work ring, DMMA sums — fls_p2plane_v9.cu) serves batches; a single
    // Match runs on the barrier kernel (v8, fls_p2plane.cu) whose one-chunk-per-warp round has the shorter hand-over (DESIGN.md
    // §3.1 has the H100 numbers)
    const bool use_v9 = B > 1;
    for (int s = 0; s < B; ++s) {
        if (n[s] > 0x3fffffffull || (long long)off[s] + (long long)n[s] > 0x7ffffff0ll) return FLS_ERR_INVALID_ARG;
        off[s + 1] = off[s] + (int)n[s];
        const int g = use_v9 ? p2plane_v9_grid((int)n[s], cfg.device) : p2plane_grid((int)n[s], cfg.device);
        if (g > grid) grid = g;
    }
    const int n_total = off[B];
    const size_t nt = (size_t)n_total;
    rec0.reserve(nt + 1);
    rec1.reserve(nt + 1);
    flags.reserve(nt + 1);
    src_f.reserve(nt + 1);
    // one LL row per CTA + one LL pose record per scan (+ the group rows of v9)
    const unsigned tag_base = next_ll_epoch((size_t)B * grid * 32 + (size_t)B * kLlPoseLen + (size_t)B * 16 * 32);
    // ---- per-batch tables, staged in one pinned block and sent with one copy -------------------------------------------
    const size_t o_pose = 0, o_off = o_pose + sizeof(PoseArg) * kMaxBatch, o_toff = o_off + sizeof(int) * (kMaxBatch + 4),
                 o_desc = o_toff + sizeof(int) * (kMaxBatch + 4), o_ptr = o_desc + sizeof(P2PlaneScan) * kMaxBatch;
    const size_t tbl_bytes = o_ptr + sizeof(void*) * kMaxBatch;
    unsigned char* const tbl = batch_table(tbl_bytes);
    PoseArg* hp = reinterpret_cast<PoseArg*>(tbl + o_pose);
    int* ho = reinterpret_cast<int*>(tbl + o_off);
    int* ht = reinterpret_cast<int*>(tbl + o_toff);
    ht[0] = 0;
    P2PlaneScan* hd = reinterpret_cast<P2PlaneScan*>(tbl + o_desc);
    const float4** hq = reinterpret_cast<const float4**>(tbl + o_ptr);
    uint4* pose_base = ll_rows.p + (size_t)B * grid * 32;
    for (int s = 0; s < B; ++s) {
        const double* Ts = T + 16 * s;
        for (int r = 0; r < 3; ++r) {
            for (int c = 0; c < 3; ++c) hp[s].R[r * 3 + c] = Ts[c * 4 + r];
            hp[s].t[r] = Ts[12 + r];
        }
        ho[s] = off[s];
        ht[s + 1] = ht[s] + order_tiles((int)n[s]);
        hq[s] = d_scans[s];
        P2PlaneScan& d = hd[s];
        d.src = src_f.p + off[s];
        d.n = (int)n[s];
        d.tag_base = tag_base;
        d.state = state.p + s;
        d.rec0 = rec0.p + off[s];
        d.rec1 = rec1.p + off[s];
        d.flags = flags.p + off[s];
        d.rows = ll_rows.p + (size_t)s * grid * 32;
        d.ll_pose = pose_base + (size_t)s * kLlPoseLen;
        d.log = scan_log(s);
        d.result = scan_result(s);
        d.grows = pose_base + (size_t)B * kLlPoseLen + (size_t)s * 16 * 32;
    }
    ho[B] = off[B];
    send_batch_table(tbl_bytes);
    const PoseArg* d_poses = reinterpret_cast<const PoseArg*>(d_batch.p + o_pose);
    const int* d_off = reinterpret_cast<const int*>(d_batch.p + o_off);
    const int* d_toff = reinterpret_cast<const int*>(d_batch.p + o_toff);
    const P2PlaneScan* d_desc = reinterpret_cast<const P2PlaneScan*>(d_batch.p + o_desc);
    const float4* const* d_ptrs = reinterpret_cast<const float4* const*>(d_batch.p + o_ptr);
    // chunk tickets of v9's dynamic work distribution: one counter per (scan, iteration) + the watchdog's abort word, zeroed by
    // the prep kernel
    const int ticket_stride = cfg.max_iterations + 2;
    const int n_tickets = use_v9 ? B * ticket_stride + 4 : 0;
    if (use_v9) tickets.reserve((size_t)n_tickets);
    // ONE prep kernel for the whole batch (state init, flag and ticket reset): every tile of a scan ends up in Morton order of the
    // voxel its points fall into at the initial pose (locality only: the sums are order-free up to fp64 rounding, and the
    // persistent per-point records live in the same order for the whole Match)
    prepare_queries(d_ptrs, d_off, d_toff, ht[B], B, d_poses, state.p, ivox_view(), flags.p, src_f.p, use_v9 ? tickets.p : nullptr, n_tickets,
                    stream, &launches);
    P2PlaneLoopArgs a;
    a.map = ivox_view();
    a.plane_thres = cfg.point_to_planar_thres;
    a.gp = gn_params(FLS_P2PLANE_IVOX, 50);
    a.log_cap = log_cap;
    a.scans = d_desc;
    a.n_scans = B;
    a.tickets = nullptr;
    a.ticket_stride = 0;
    a.abort_word = nullptr;
    // roofline accounting (SURVEY.md §8d, K1 — the REFERENCE algorithm's traffic): 16 B source point + n_stencil x 16 B
    // slot probes + 32 B persistent record per point-iteration, 16 B per map record resident in the stencil voxels.
    gn_launch(16 + 16LL * a.map.n_stencil + 32, 16, d_scans[0], n[0], [&] {
        if (use_v9) {
            a.ticket_stride = ticket_stride;
            a.tickets = tickets.p;
            a.abort_word = tickets.p + (size_t)B * a.ticket_stride;
            launch_p2plane_v9(a, grid, stream);
        } else {
            launch_p2plane_loop(a, grid, stream);
        }
    });
    // ---- read back: every scan's state (+ its iteration log) ----------------------------------------------------------
    read_back(B);
    *h_abort = 0;
    if (use_v9) FLS_CUDA(cudaMemcpyAsync(h_abort, a.abort_word, sizeof(unsigned), cudaMemcpyDeviceToHost, stream));
    pend_n.assign(n, n + B);
    pend_v9 = use_v9;
    return FLS_OK;
}

// waits for the batch enqueued last and unpacks its results
int Handle::finish_ivox_batch(double* T, int* converged, fls_match_stats* st) {
    const int B = (int)pend_n.size();
    if (B < 1) return FLS_ERR_INVALID_ARG;
    end_call(st);
    if (pend_v9 && *h_abort) {
        pend_n.clear();
        set_last_error("p2plane_v9_kernel: watchdog — a wait loop gave up after 4 s (hand-over protocol error)");
        return FLS_ERR_CUDA;
    }
    unpack(B, pend_n.data(), T, converged, st);
    pend_n.clear();
    return FLS_OK;
}

int Handle::match_p2plane_ivox(const float4* d_src, size_t n, double* T, int* converged, fls_match_stats* st) {
    const float4* scans[1] = {d_src};
    const size_t ns[1] = {n};
    int conv = 0;
    const int rc = match_ivox_batch(1, scans, ns, T, &conv, st);
    if (rc != FLS_OK) return rc;
    if (converged) *converged = conv;
    const int ni = (int)n;
    if (h_state->converged && !cfg.localization_mode) {
        // :205-206 — the scan enters the map through the cached-5-NN rule (body-frame points, final pose)  [quirk 8]
        stage.reserve(n + 1);
        stage2.reserve(n + 1);
        const GnState& s = *h_state;
        const size_t n_add = select_ivox_inserts(ivox_view(), d_src, ni, s.Rprev, s.tprev, s.R, s.t, 0.5 /* filter_size_map_min_ (:351) */,
                                                 stage2.p, stage.p, scratch, stream, &launches);
        const int rc2 = ivox.append_and_build(stage.p, n_add, cfg.ivox_capacity, stream);
        launches += ivox.launches;
        ivox.launches = 0;
        FLS_CUDA(cudaStreamSynchronize(stream));
        if (st) st->gpu_launches = launches;
        if (rc2 != FLS_OK) return rc2;
    }
    return FLS_OK;
}

// ---- IncrementalNDT ----------------------------------------------------------------------------------------------
int Handle::add_cloud_ndt(const float4* d_cloud, size_t n) {
    const int rc = ndt.add_cloud(d_cloud, n, cfg.source_cloud_filter_size, ndt_first_scan, stream);
    launches += ndt.launches;
    ndt.launches = 0;
    if (cfg.localization_mode && rc == FLS_OK) {
        // kdtree_flann_.setInputCloud(cloud_world) — the voxel-filtered cloud (incremental_ndt.h:188-190)
        const size_t nf = voxel_grid_device(d_cloud, n, cfg.source_cloud_filter_size, ndt.filtered.p, ndt.scratch, stream, &launches);
        set_fit_cloud(ndt.filtered.p, nf);
    }
    ndt_first_scan = cfg.localization_mode != 0;  // :222-226
    return rc;
}

int Handle::match_ndt(const float4* d_in, size_t n_in, double* T, int* converged, fls_match_stats* st) {
    if (ndt.n_vox == 0) return FLS_ERR_NO_MAP;  // CHECK(!grids_.empty())
    src_f.reserve(n_in);
    const size_t n = voxel_grid_device(d_in, n_in, cfg.source_cloud_filter_size, src_f.p, scratch, stream, &launches);  // :232
    const int ni = (int)n;
    const int grid = ndt_grid(ni, cfg.device);
    GnLoopCtl ctl = make_ctl(*this, FLS_NDT, grid, cfg.ndt_min_effective_pts);
    double T_in[16];
    std::memcpy(T_in, T, sizeof(T_in));
    launch_gn_init(state.p, T, stream);
    launches++;
    NdtArgs a;
    a.src = src_f.p;
    a.n = ni;
    a.map = ndt.view();
    a.outlier_thres = cfg.ndt_outlier_thres;
    a.state = state.p;
    // roofline accounting (SURVEY.md §8d, K2): 16 B source point + 7 x 16 B slot probes per point-iteration,
    // 80 B voxel record per estimated voxel hit; the 6x6 sums are fused (no per-point output).
    gn_launch(16 + 16LL * 7, 80, src_f.p, n, [&] { launch_ndt_loop(a, ctl, grid, stream); });
    finish_match(*this, T, converged, st, n);
    if (!h_state->failed && !cfg.localization_mode) {
        // :326-330 — the scan enters the map transformed by the INPUT guess T, not the optimised pose  [quirk 6]
        stage2.reserve(n);
        launch_transform_f(src_f.p, n, T_in, stage2.p, stream);
        launches++;
        const int rc2 = add_cloud_ndt(stage2.p, n);
        FLS_CUDA(cudaStreamSynchronize(stream));
        if (st) st->gpu_launches = launches;
        if (rc2 != FLS_OK) return rc2;
    }
    return FLS_OK;
}

// n_scans independent IncrementalNDT::Match calls against the same (static) map in ONE cooperative launch (fls_ndt.cu:
// ndt_gn_batch_kernel — one sub-grid and one persistent Gauss-Newton loop per scan).  Localization semantics only: the map is
// not modified (incremental_ndt.h:222-226, flag_first_scan_ stays set).
int Handle::match_ndt_batch(int B, const float4* const* d_scans, const size_t* n_in, double* T, int* converged, fls_match_stats* st) {
    if (ndt.n_vox == 0) return FLS_ERR_NO_MAP;
    if (B < 1 || B > kMaxBatch) return FLS_ERR_INVALID_ARG;
    size_t total_in = 0;
    for (int s = 0; s < B; ++s) total_in += n_in[s];
    src_f.reserve(total_in + 1);
    // VoxelGridCloud of every source (incremental_ndt.h:232), back to back in one buffer
    size_t off[kMaxBatch + 1];
    off[0] = 0;
    for (int s = 0; s < B; ++s) {
        const size_t nf = voxel_grid_device(d_scans[s], n_in[s], cfg.source_cloud_filter_size, src_f.p + off[s], scratch, stream, &launches);
        if (nf > 0x3fffffffull) return FLS_ERR_INVALID_ARG;
        off[s + 1] = off[s] + nf;
    }
    // sub-grids: every scan gets the CTAs its points need, scaled down together when the device cannot hold them all
    const int cap = ndt_max_grid(cfg.device);
    int need[kMaxBatch], tot_need = 0;
    for (int s = 0; s < B; ++s) {
        need[s] = (int)((off[s + 1] - off[s] + kNdtBlock - 1) / kNdtBlock);
        if (need[s] < 1) need[s] = 1;
        tot_need += need[s];
    }
    if (B > cap) return FLS_ERR_INVALID_ARG;
    int ncta[kMaxBatch], grid = 0;
    for (int s = 0; s < B; ++s) {
        ncta[s] = tot_need <= cap ? need[s] : (int)((long long)need[s] * (cap - B) / tot_need) + 1;
        grid += ncta[s];
    }
    const unsigned tag_base = next_ll_epoch((size_t)grid * 32 + (size_t)B * kLlPoseLen);
    const size_t tbl_bytes = sizeof(NdtBatchItem) * (size_t)B;
    NdtBatchItem* items = reinterpret_cast<NdtBatchItem*>(batch_table(tbl_bytes));
    uint4* pose_base = ll_rows.p + (size_t)grid * 32;
    size_t ns[kMaxBatch];
    int cta0 = 0;
    for (int s = 0; s < B; ++s) {
        launch_gn_init(state.p + s, T + 16 * s, stream);
        launches++;
        ns[s] = off[s + 1] - off[s];
        NdtBatchItem& it = items[s];
        std::memset(&it, 0, sizeof(it));
        it.a.src = src_f.p + off[s];
        it.a.n = (int)ns[s];
        it.a.map = ndt.view();
        it.a.outlier_thres = cfg.ndt_outlier_thres;
        it.a.state = state.p + s;
        it.ctl.state = state.p + s;
        it.ctl.ll_rows = ll_rows.p + (size_t)cta0 * 32;
        it.ctl.ll_pose = pose_base + (size_t)s * kLlPoseLen;
        it.ctl.tag_base = tag_base;
        it.ctl.gp = gn_params(FLS_NDT, cfg.ndt_min_effective_pts);
        it.ctl.log = scan_log(s);
        it.ctl.log_cap = log_cap;
        it.ctl.result = scan_result(s);
        it.cta0 = cta0;
        it.ncta = ncta[s];
        cta0 += ncta[s];
    }
    send_batch_table(tbl_bytes);
    gn_launch(16 + 16LL * 7, 80, src_f.p, ns[0],
              [&] { launch_ndt_batch(reinterpret_cast<const NdtBatchItem*>(d_batch.p), B, grid, stream); });
    read_back(B);
    end_call(st);
    unpack(B, ns, T, converged, st);
    return FLS_OK;
}

// ---- IcpOptimized ------------------------------------------------------------------------------------------------
int Handle::add_cloud_icp(const float4* d_cloud, size_t n) {
    // icp_optimized.h:173-187: mapping mode slides a window of the last local_map_size clouds, localization mode replaces
    // the map; both end in local_map_ptr_ = VoxelGridCloud(local_map_ptr_, map_cloud_filter_size_)
    const int rc = window_add(icp_map, d_cloud, n, (size_t)cfg.local_map_size, cfg.map_cloud_filter_size, 0, cfg.localization_mode != 0);
    set_fit_view(icp_map.cloud.p, icp_map.n);  // GetFitnessScore searches the same cloud
    return rc;
}

static void mat3_from_T(const double* T, double* R) {
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) R[r * 3 + c] = T[c * 4 + r];
}

// IsNeedAddCloud (icp_optimized.h:218-236, loam_point_to_plane_kdtree.h:186-202, loam_full_kdtree.h:356-371): key-frame
// gating on translation / RPY deltas against a persistent last_T that starts at the first pose it sees  [quirk 7]
bool Handle::need_add_cloud(const double* T) {
    if (!have_last) {
        std::memcpy(last_T, T, 16 * sizeof(double));
        have_last = true;
    }
    double Rl[9], Rc[9], Rli[9], Rd[9];
    mat3_from_T(last_T, Rl);
    mat3_from_T(T, Rc);
    {  // 3x3 inverse by cofactors
        const double c00 = Rl[4] * Rl[8] - Rl[5] * Rl[7], c01 = Rl[5] * Rl[6] - Rl[3] * Rl[8], c02 = Rl[3] * Rl[7] - Rl[4] * Rl[6];
        const double id = 1.0 / (Rl[0] * c00 + Rl[1] * c01 + Rl[2] * c02);
        Rli[0] = c00 * id; Rli[1] = (Rl[2] * Rl[7] - Rl[1] * Rl[8]) * id; Rli[2] = (Rl[1] * Rl[5] - Rl[2] * Rl[4]) * id;
        Rli[3] = c01 * id; Rli[4] = (Rl[0] * Rl[8] - Rl[2] * Rl[6]) * id; Rli[5] = (Rl[2] * Rl[3] - Rl[0] * Rl[5]) * id;
        Rli[6] = c02 * id; Rli[7] = (Rl[1] * Rl[6] - Rl[0] * Rl[7]) * id; Rli[8] = (Rl[0] * Rl[4] - Rl[1] * Rl[3]) * id;
    }
    mat3_mul(Rli, Rc, Rd);
    const double roll = std::atan2(Rd[7], Rd[8]), pitch = std::asin(-Rd[6]), yaw = std::atan2(Rd[3], Rd[0]);
    const double dt[3] = {T[12] - last_T[12], T[13] - last_T[13], T[14] - last_T[14]};
    if (norm3(dt) > cfg.dist_thre_add_cloud || std::fabs(roll) > cfg.rot_thre_add_cloud || std::fabs(pitch) > cfg.rot_thre_add_cloud ||
        std::fabs(yaw) > cfg.rot_thre_add_cloud) {
        std::memcpy(last_T, T, 16 * sizeof(double));
        return true;
    }
    return false;
}

int Handle::match_icp(const float4* d_in, size_t n_in, double* T, int* converged, fls_match_stats* st) {
    if (n_in <= 10) return FLS_ERR_TOO_FEW_POINTS;  // CHECK_GT(ordered_cloud_.size(), 10u)  (:55)
    if (icp_map.grid.n_pts == 0) return FLS_ERR_NO_MAP;
    src_f.reserve(n_in);
    const size_t n = voxel_grid_device(d_in, n_in, cfg.source_cloud_filter_size, src_f.p, scratch, stream, &launches);  // :57
    const int ni = (int)n;
    const int grid = icp_grid_blocks(ni, cfg.device);
    GnLoopCtl ctl = make_ctl(*this, FLS_ICP_P2P, grid, 0);
    launch_gn_init(state.p, T, stream);
    launches++;
    IcpArgs a;
    a.src = src_f.p;
    a.n = ni;
    a.map = grid_view(icp_map.grid);
    a.max_corr = cfg.icp_max_correspond_distance;
    a.state = state.p;
    // roofline accounting (SURVEY.md §8d, K3): 16 B source point + 27 x 16 B slot probes, 16 B per scanned map record
    gn_launch(16 + 16LL * 27, 16, src_f.p, n, [&] { launch_icp_loop(a, ctl, grid, stream); });
    finish_match(*this, T, converged, st, n);
    if (h_state->converged && !cfg.localization_mode) {
        // IsNeedAddCloud (:218-236): key-frame gating on translation / RPY deltas against a persistent last_T
        if (need_add_cloud(T)) {
            stage.reserve(n);
            launch_transform_f(src_f.p, n, T, stage.p, stream);  // :156 TransformPointCloud(source, final) in float
            launches++;
            const int rc2 = add_cloud_icp(stage.p, n);
            FLS_CUDA(cudaStreamSynchronize(stream));
            if (st) st->gpu_launches = launches;
            if (rc2 != FLS_OK) return rc2;
        }
    }
    return FLS_OK;
}

// ---- LoamPointToPlaneKdtree / LoamFull -------------------------------------------------------------------------------
static LoamGrid loam_grid_of(const Handle::WindowMap& w) {
    LoamGrid g;
    g.pts = w.grid.pts_sorted.p;
    g.tab = w.grid.table.p;
    g.mask = w.grid.mask;
    g.inv_cell = w.grid.inv_res;
    g.cell = w.grid.res;
    g.n_pts = (unsigned)w.grid.n_pts;
    return g;
}

int Handle::window_add(WindowMap& w, const float4* d_cloud, size_t n, size_t window, float leaf, int filter_mode, bool replace) {
    const float4* merged = d_cloud;
    size_t n_merged = n;
    size_t depth = 1;
    if (!replace) {
        std::unique_ptr<Cloud> c(new Cloud());
        c->buf.reserve(n);
        if (n) FLS_CUDA(cudaMemcpyAsync(c->buf.p, d_cloud, n * sizeof(float4), cudaMemcpyDeviceToDevice, stream));
        c->n = n;
        w.deque.push_back(std::move(c));
        if (w.deque.size() > window) {
            FLS_CUDA(cudaStreamSynchronize(stream));  // the evicted buffer may still feed a copy in flight
            w.deque.pop_front();
        }
        n_merged = 0;
        for (auto& q : w.deque) n_merged += q->n;
        w.merged.reserve(n_merged);
        size_t off = 0;
        for (auto& q : w.deque) {
            if (q->n) FLS_CUDA(cudaMemcpyAsync(w.merged.p + off, q->buf.p, q->n * sizeof(float4), cudaMemcpyDeviceToDevice, stream));
            off += q->n;
        }
        merged = w.merged.p;
        depth = w.deque.size();
    }
    w.cloud.reserve(n_merged);
    if (filter_mode == 0 || depth > 5) {
        w.n = voxel_grid_device(merged, n_merged, leaf, w.cloud.p, scratch, stream, &launches);
    } else {
        if (n_merged) FLS_CUDA(cudaMemcpyAsync(w.cloud.p, merged, n_merged * sizeof(float4), cudaMemcpyDeviceToDevice, stream));
        w.n = n_merged;
    }
    w.grid.clear();
    const int rc = w.grid.append_and_build(w.cloud.p, w.n, 0, stream);
    launches += w.grid.launches;
    w.grid.launches = 0;
    return rc;
}

int Handle::add_cloud_kd(const float4* d_planar, size_t n_planar, const float4* d_corner, size_t n_corner) {
    if (cfg.method == FLS_P2PLANE_KNN) {
        // loam_point_to_plane_kdtree.h:56-80: localization mode replaces the map, mapping mode slides a window; both
        // end in VoxelGridCloud(local_map, map_cloud_filter_size) + kd-tree
        const int rc = window_add(kd_planar, d_planar, n_planar, (size_t)cfg.local_map_size, cfg.map_cloud_filter_size, 0,
                                  cfg.localization_mode != 0);
        if (rc == FLS_OK) set_fit_cloud(kd_planar.cloud.p, kd_planar.n);  // GetFitnessScore searches the same tree (:159-183)
        return rc;
    }
    // loam_full_kdtree.h:66-104: {planar, corner}, both windows slide, filters only beyond 5 clouds
    int rc = window_add(kd_planar, d_planar, n_planar, (size_t)cfg.local_map_size, cfg.map_cloud_filter_size, 1, false);
    if (rc != FLS_OK) return rc;
    return window_add(kd_corner, d_corner, n_corner, (size_t)cfg.corner_local_map_size, cfg.corner_map_filter_size, 1, false);
}

int Handle::match_kd(const float4* d_planar, size_t n_planar, const float4* d_corner, size_t n_corner, double* T, int* converged,
                     fls_match_stats* st) {
    const bool full = cfg.method == FLS_LOAM_FULL;
    if (kd_planar.n == 0) return FLS_ERR_NO_MAP;
    if (!full) n_corner = 0;
    const size_t n = n_planar + n_corner;
    const int ni = (int)n;
    const int grid = loam_grid_blocks(ni, cfg.device);
    GnLoopCtl ctl = make_ctl(*this, cfg.method, grid, 50);
    launch_gn_init(state.p, T, stream);
    launches++;
    rec_d.reserve(n * 8 + 8);
    flags.reserve(n + 1);
    LoamArgs a;
    a.corner = d_corner;
    a.n_corner = (int)n_corner;
    a.planar = d_planar;
    a.n_planar = (int)n_planar;
    a.planar_map = loam_grid_of(kd_planar);
    a.corner_map = full ? loam_grid_of(kd_corner) : a.planar_map;
    a.plane_thres = cfg.point_to_planar_thres;
    a.search_thres = full ? cfg.point_search_thres : INFINITY;
    a.line_ratio = cfg.line_ratio_thres;
    a.gate = full ? (float)cfg.point_search_thres * 1.0001f : INFINITY;
    a.state = state.p;
    a.rec = rec_d.p;
    a.flags = flags.p;
    // roofline accounting (K5): 16 B source point + 27 x 16 B slot probes + 56 B persistent record, 16 B per scanned map record
    gn_launch(16 + 16LL * 27 + 56, 16, d_planar, n_planar, [&] {
        launch_loam_loop(a, ctl, grid, stream);
        launches++;  // the flag reset in front of the loop
    });
    finish_match(*this, T, converged, st, n);
    // key-frame insertion: loam_point_to_plane_kdtree.h:146-150 (gate evaluated before the mode test), loam_full_kdtree.h:178-186
    if (h_state->converged && need_add_cloud(T) && (full || !cfg.localization_mode)) {
        int rc2;
        if (full) {
            stage.reserve(n_planar);
            stage2.reserve(n_corner);
            launch_transform_d(d_planar, n_planar, T, stage.p, stream);  // pcl::transformPointCloud(cloud, out, T_) with the double matrix
            launch_transform_d(d_corner, n_corner, T, stage2.p, stream);
            launches += 2;
            rc2 = add_cloud_kd(stage.p, n_planar, stage2.p, n_corner);
        } else {
            stage.reserve(n_planar);
            launch_transform_f(d_planar, n_planar, T, stage.p, stream);  // TransformPointCloud(source, final): fp32 with R, t cast to float
            launches++;
            rc2 = add_cloud_kd(stage.p, n_planar, nullptr, 0);
        }
        FLS_CUDA(cudaStreamSynchronize(stream));
        if (st) st->gpu_launches = launches;
        if (rc2 != FLS_OK) return rc2;
    }
    return FLS_OK;
}

// ---- GetFitnessScore -------------------------------------------------------------------------------------------------
int Handle::fitness(float max_range, float* score) {
    *score = 3.402823466e+38f;  // FloatNaN / "no inliers" upstream
    if (cfg.method == FLS_LOAM_FULL) return FLS_OK;  // loam_full_kdtree.h:206-208 FloatNaN
    // ICP and the kd-tree point-to-plane plug-in always search their tree; NDT / iVox return FloatNaN outside localization mode
    if (cfg.method != FLS_ICP_P2P && cfg.method != FLS_P2PLANE_KNN && !cfg.localization_mode) return FLS_OK;
    if (fit_cloud_n == 0 || last_src == nullptr || last_src_n == 0 || !(max_range > 0.f)) return FLS_OK;
    begin_call();
    if (fit_grid_version != fit_cloud_version || fit_grid_range != max_range) {
        fit_grid.set_resolution(std::sqrt(max_range) * 1.001f);
        fit_grid.clear();
        const int rc = fit_grid.append_and_build(fit_pts, fit_cloud_n, 0, stream);
        launches += fit_grid.launches;
        fit_grid.launches = 0;
        if (rc != FLS_OK) return rc;
        fit_grid_version = fit_cloud_version;
        fit_grid_range = max_range;
    }
    launch_fitness(grid_view(fit_grid), last_src, (int)last_src_n, T_final, max_range, fit_out.p, stream);
    launches++;
    double h[2] = {0, 0};
    FLS_CUDA(cudaMemcpyAsync(h, fit_out.p, sizeof(h), cudaMemcpyDeviceToHost, stream));
    end_call(nullptr);
    if (h[1] > 0) *score = (float)(h[0] / h[1]);
    return FLS_OK;
}

}  // namespace fls

// =====================================================================================================================
using fls::check_device;
using fls::Handle;
using fls::stride_ok;

// the configuration check fls_preprocess_loam and fls_preprocess_loam_device share
static bool loam_frontend_cfg_ok(const fls_loam_frontend_cfg& c) {
    return c.n_rows > 0 && c.n_cols > 0 && (long long)c.n_rows * c.n_cols <= 0x7fffffffll && c.horizontal_resolution > 0.f && c.corner_leaf > 0.f &&
           c.planar_leaf > 0.f &&
           // the reference CHECK_NE()s both feature thresholds against FloatNaN (feature_extractor.cpp:19-20)
           c.corner_threshold < 3.0e38f && c.planar_threshold < 3.0e38f;
}

// The checks the four batch Match entries share.  `begin` (fls_match_batch_begin*): the batch runs on LOAM-iVox only and must find
// the same map when it ends, whatever its size.
static int check_match_batch(const Handle* h, int n_scans, const void* pts, const size_t* n, const void* T, size_t stride, bool begin) {
    if (!h || !pts || !n || !T || n_scans < 1 || n_scans > fls::kMaxBatch || !stride_ok(stride)) return FLS_ERR_INVALID_ARG;
    if (h->cfg.method != FLS_P2PLANE_IVOX && (begin || h->cfg.method != FLS_NDT)) return FLS_ERR_UNSUPPORTED;
    // scans of one batch are matched against the same map state: only meaningful when Match does not modify the map
    if ((begin || n_scans > 1) && !h->cfg.localization_mode) return FLS_ERR_UNSUPPORTED;
    return FLS_OK;
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
    return fls::project_device(device, raw, ring, nullptr, nullptr, n, stride, n_rows, n_cols, horizontal_resolution, min_distance, max_distance, ordered,
                               depth, col, row_start, row_end, n_ordered);
    FLS_CATCH
}

int fls_project_imu(int device, const void* raw, const int32_t* ring, const float* time, size_t n, size_t stride, const fls_imu_buffer* imu,
                    int32_t n_rows, int32_t n_cols, float horizontal_resolution, float min_distance, float max_distance, float* ordered, float* depth,
                    int32_t* col, int32_t* row_start, int32_t* row_end, size_t* n_ordered) {
    if ((!raw && n) || (!ring && n) || !ordered || !depth || !col || !row_start || !row_end || !n_ordered || !stride_ok(stride))
        return FLS_ERR_INVALID_ARG;
    if (imu && imu->n_imu && !time && n) return FLS_ERR_INVALID_ARG;
    if (check_device(device) != FLS_OK) return FLS_ERR_NO_DEVICE;
    FLS_TRY
    return fls::project_device(device, raw, ring, time, imu, n, stride, n_rows, n_cols, horizontal_resolution, min_distance, max_distance, ordered,
                               depth, col, row_start, row_end, n_ordered);
    FLS_CATCH
}

int fls_preprocess(int device, const float* raw_xyzit, size_t n, const fls_imu_buffer* imu, float min_distance, float max_distance, int32_t jump_span,
                   float planar_leaf, float* ordered, size_t* n_ordered, float* planar, size_t* n_planar) {
    if ((!raw_xyzit && n) || !ordered || !planar || !n_ordered || !n_planar || jump_span < 1 || !(planar_leaf > 0.f)) return FLS_ERR_INVALID_ARG;
    if (check_device(device) != FLS_OK) return FLS_ERR_NO_DEVICE;
    FLS_TRY
    return fls::preprocess_device(device, raw_xyzit, n, imu, min_distance, max_distance, jump_span, planar_leaf, ordered, n_ordered, planar, n_planar);
    FLS_CATCH
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
    const int want = h->cfg.method == FLS_LOAM_FULL ? 2 : 1;
    if (n_clouds != want) return FLS_ERR_INVALID_ARG;
    for (int k = 0; k < n_clouds; ++k)
        if (!pts[k] && n[k]) return FLS_ERR_INVALID_ARG;
    FLS_TRY
    h->begin_call();
    int rc = FLS_ERR_UNSUPPORTED;
    switch (h->cfg.method) {
        case FLS_P2PLANE_IVOX: rc = h->add_cloud_ivox(pts[0], n[0], stride); break;
        case FLS_NDT: rc = h->add_cloud_ndt(h->upload(pts[0], n[0], stride, h->stage), n[0]); break;
        case FLS_ICP_P2P: rc = h->add_cloud_icp(h->upload(pts[0], n[0], stride, h->stage), n[0]); break;
        case FLS_P2PLANE_KNN: rc = h->add_cloud_kd(h->upload(pts[0], n[0], stride, h->stage), n[0], nullptr, 0); break;
        case FLS_LOAM_FULL: {
            const float4* dp = h->upload(pts[0], n[0], stride, h->stage);
            const float4* dc = h->upload(pts[1], n[1], stride, h->stage2);
            rc = h->add_cloud_kd(dp, n[0], dc, n[1]);
            break;
        }
        default: break;
    }
    h->end_call(nullptr);
    return rc;
    FLS_CATCH
}

static int match_dispatch(Handle* h, const float4* d_ordered, size_t n_ordered, const float4* d_planar, size_t n_planar, const float4* d_corner,
                          size_t n_corner, double* T, int* converged, fls_match_stats* st) {
    switch (h->cfg.method) {
        case FLS_P2PLANE_IVOX: return h->match_p2plane_ivox(d_planar, n_planar, T, converged, st);
        case FLS_NDT: return h->match_ndt(d_ordered, n_ordered, T, converged, st);
        case FLS_ICP_P2P: return h->match_icp(d_ordered, n_ordered, T, converged, st);
        case FLS_P2PLANE_KNN:
        case FLS_LOAM_FULL: return h->match_kd(d_planar, n_planar, d_corner, n_corner, T, converged, st);
        default: return FLS_ERR_UNSUPPORTED;
    }
}

int fls_match(fls_handle* hh, const void* ordered, size_t n_ordered, const void* planar, size_t n_planar, const void* corner, size_t n_corner,
              size_t stride, double T[16], int* converged, fls_match_stats* st) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    if (!h || !T || !stride_ok(stride)) return FLS_ERR_INVALID_ARG;
    FLS_TRY
    if (st) std::memset(st, 0, sizeof(*st));
    h->begin_call();
    const float4* d_ord = nullptr;
    const float4* d_pla = nullptr;
    const float4* d_cor = nullptr;
    const bool uses_planar = h->cfg.method >= FLS_P2PLANE_IVOX;
    if (uses_planar) {
        if (!planar && n_planar) return FLS_ERR_INVALID_ARG;
        d_pla = h->upload(planar, n_planar, stride, h->src);
        if (h->cfg.method == FLS_LOAM_FULL) {
            if (!corner && n_corner) return FLS_ERR_INVALID_ARG;
            d_cor = h->upload(corner, n_corner, stride, h->src2);
        } else {
            n_corner = 0;
        }
    } else {
        if (!ordered && n_ordered) return FLS_ERR_INVALID_ARG;
        d_ord = h->upload(ordered, n_ordered, stride, h->src);
    }
    return match_dispatch(h, d_ord, n_ordered, d_pla, n_planar, d_cor, n_corner, T, converged, st);
    FLS_CATCH
}

int fls_match_device(fls_handle* hh, const void* d_points, size_t n, double T[16], int* converged, fls_match_stats* st) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    if (!h || !T || (!d_points && n)) return FLS_ERR_INVALID_ARG;
    FLS_TRY
    if (st) std::memset(st, 0, sizeof(*st));
    h->begin_call();
    const float4* d = static_cast<const float4*>(d_points);
    if (h->cfg.method == FLS_LOAM_FULL) return FLS_ERR_UNSUPPORTED;  // two feature clouds: use fls_match
    return match_dispatch(h, d, n, d, n, nullptr, 0, T, converged, st);
    FLS_CATCH
}

int fls_match_cluster_device(fls_handle* hh, const void* d_ordered, size_t n_ordered, const void* d_planar, size_t n_planar, const void* d_corner,
                             size_t n_corner, double T[16], int* converged, fls_match_stats* st) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    if (!h || !T) return FLS_ERR_INVALID_ARG;
    // the clouds each plug-in reads, as in fls_match
    const bool uses_planar = h->cfg.method >= FLS_P2PLANE_IVOX;
    if (uses_planar) {
        if (!d_planar && n_planar) return FLS_ERR_INVALID_ARG;
        if (h->cfg.method == FLS_LOAM_FULL) {
            if (!d_corner && n_corner) return FLS_ERR_INVALID_ARG;
        } else {
            n_corner = 0;
        }
    } else if (!d_ordered && n_ordered) {
        return FLS_ERR_INVALID_ARG;
    }
    FLS_TRY
    if (st) std::memset(st, 0, sizeof(*st));
    h->begin_call();
    return match_dispatch(h, static_cast<const float4*>(d_ordered), n_ordered, static_cast<const float4*>(d_planar), n_planar,
                          static_cast<const float4*>(d_corner), n_corner, T, converged, st);
    FLS_CATCH
}

// Uploads the host scans of a batch back to back into the handle's scan buffer; ptrs[s] receives scan s
static int upload_scans(Handle* h, int B, const void* const* pts, const size_t* n, size_t stride, const float4** ptrs) {
    size_t total = 0, n_max = 0;
    for (int s = 0; s < B; ++s) {
        if (!pts[s] && n[s]) return FLS_ERR_INVALID_ARG;
        total += n[s];
        n_max = std::max(n_max, n[s]);
    }
    h->src.reserve(total + 1);
    if (stride != FLS_LAYOUT_PACKED) h->raw.reserve(n_max * stride);
    size_t off = 0;
    for (int s = 0; s < B; ++s) {
        ptrs[s] = h->src.p + off;
        h->upload_into(pts[s], n[s], stride, h->src.p + off);
        off += n[s];
    }
    return FLS_OK;
}

static int device_scans(int B, const void* const* d_pts, const size_t* n, const float4** ptrs) {
    for (int s = 0; s < B; ++s) {
        if (!d_pts[s] && n[s]) return FLS_ERR_INVALID_ARG;
        ptrs[s] = static_cast<const float4*>(d_pts[s]);
    }
    return FLS_OK;
}

// a batch Match: NDT batch / NDT single / LOAM-iVox single / LOAM-iVox batch
static int match_batch_route(Handle* h, int B, const float4* const* ptrs, const size_t* n, double* T, int* converged, fls_match_stats* st) {
    if (h->cfg.method == FLS_NDT) return B == 1 ? h->match_ndt(ptrs[0], n[0], T, converged, st) : h->match_ndt_batch(B, ptrs, n, T, converged, st);
    if (B == 1) return h->match_p2plane_ivox(ptrs[0], n[0], T, converged, st);
    return h->match_ivox_batch(B, ptrs, n, T, converged, st);
}

int fls_match_batch(fls_handle* hh, int n_scans, const void* const* planar, const size_t* n, size_t stride, double* T, int* converged,
                    fls_match_stats* st) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    const int chk = check_match_batch(h, n_scans, planar, n, T, stride, false);
    if (chk != FLS_OK) return chk;
    FLS_TRY
    if (st) std::memset(st, 0, sizeof(*st) * (size_t)n_scans);
    h->begin_call();
    const float4* ptrs[fls::kMaxBatch];
    const int rc = upload_scans(h, n_scans, planar, n, stride, ptrs);
    if (rc != FLS_OK) return rc;
    return match_batch_route(h, n_scans, ptrs, n, T, converged, st);
    FLS_CATCH
}

int fls_match_batch_begin(fls_handle* hh, int n_scans, const void* const* planar, const size_t* n, size_t stride, const double* T) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    const int chk = check_match_batch(h, n_scans, planar, n, T, stride, true);
    if (chk != FLS_OK) return chk;
    if (!h->pend_n.empty()) return FLS_ERR_INVALID_ARG;  // one batch in flight per handle
    FLS_TRY
    h->begin_call();
    const float4* ptrs[fls::kMaxBatch];
    const int rc = upload_scans(h, n_scans, planar, n, stride, ptrs);
    if (rc != FLS_OK) return rc;
    return h->enqueue_ivox_batch(n_scans, ptrs, n, T);
    FLS_CATCH
}

int fls_match_batch_begin_device(fls_handle* hh, int n_scans, const void* const* d_planar, const size_t* n, const double* T) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    const int chk = check_match_batch(h, n_scans, d_planar, n, T, FLS_LAYOUT_PACKED, true);
    if (chk != FLS_OK) return chk;
    if (!h->pend_n.empty()) return FLS_ERR_INVALID_ARG;
    FLS_TRY
    h->begin_call();
    const float4* ptrs[fls::kMaxBatch];
    const int rc = device_scans(n_scans, d_planar, n, ptrs);
    if (rc != FLS_OK) return rc;
    return h->enqueue_ivox_batch(n_scans, ptrs, n, T);
    FLS_CATCH
}

int fls_match_batch_end(fls_handle* hh, double* T, int* converged, fls_match_stats* st) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    if (!h || !T) return FLS_ERR_INVALID_ARG;
    if (h->pend_n.empty()) return FLS_ERR_INVALID_ARG;
    FLS_TRY
    if (st) std::memset(st, 0, sizeof(*st) * h->pend_n.size());
    return h->finish_ivox_batch(T, converged, st);
    FLS_CATCH
}

int fls_match_batch_device(fls_handle* hh, int n_scans, const void* const* d_planar, const size_t* n, double* T, int* converged,
                           fls_match_stats* st) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    const int chk = check_match_batch(h, n_scans, d_planar, n, T, FLS_LAYOUT_PACKED, false);
    if (chk != FLS_OK) return chk;
    FLS_TRY
    if (st) std::memset(st, 0, sizeof(*st) * (size_t)n_scans);
    h->begin_call();
    const float4* ptrs[fls::kMaxBatch];
    const int rc = device_scans(n_scans, d_planar, n, ptrs);
    if (rc != FLS_OK) return rc;
    return match_batch_route(h, n_scans, ptrs, n, T, converged, st);
    FLS_CATCH
}

int fls_fitness(fls_handle* hh, float max_range, float* score) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    if (!h || !score) return FLS_ERR_INVALID_ARG;
    FLS_TRY
    return h->fitness(max_range, score);
    FLS_CATCH
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
    h->end_call(nullptr);
    return rc;
    FLS_CATCH
}

int fls_update_local_map(fls_handle* hh, const double* T, int* updated, size_t* n_local) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    if (!h || !T) return FLS_ERR_INVALID_ARG;
    FLS_TRY
    h->begin_call();
    const int rc = h->update_local_map(T, updated, n_local);
    h->end_call(nullptr);
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
    if (h->cfg.method != FLS_NDT && h->cfg.method != FLS_P2PLANE_IVOX) return FLS_ERR_UNSUPPORTED;
    FLS_TRY
    FLS_CUDA(cudaSetDevice(h->cfg.device));
    std::vector<unsigned long long> packed(capacity + 1);
    const size_t m = h->cfg.method == FLS_NDT ? h->ndt.dump_keys(packed.data(), capacity, h->stream) : h->ivox.dump_keys(packed.data(), capacity, h->stream);
    for (size_t i = 0; i < m; ++i) {
        const unsigned long long k = packed[i];
        const int c[3] = {(int)((k >> 42) & 0x1fffffu), (int)((k >> 21) & 0x1fffffu), (int)(k & 0x1fffffu)};
        for (int a = 0; a < 3; ++a) keys_xyz[3 * i + a] = (c[a] & 0x100000) ? c[a] - 0x200000 : c[a];  // 21-bit two's complement
    }
    *n = h->cfg.method == FLS_NDT ? h->ndt.n_vox : h->ivox.n_vox;
    return FLS_OK;
    FLS_CATCH
}

int fls_get_ndt_voxels(fls_handle* hh, fls_ndt_voxel* out, size_t capacity, size_t* n) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    if (!h || !n || (capacity && !out)) return FLS_ERR_INVALID_ARG;
    if (h->cfg.method != FLS_NDT) return FLS_ERR_UNSUPPORTED;
    FLS_TRY
    FLS_CUDA(cudaSetDevice(h->cfg.device));
    std::vector<fls_ndt_voxel> v;
    h->ndt.dump_voxels(v, h->stream);
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
    if (h->cfg.method != FLS_P2PLANE_IVOX) return FLS_ERR_UNSUPPORTED;
    FLS_TRY
    FLS_CUDA(cudaSetDevice(h->cfg.device));
    FLS_CUDA(cudaStreamSynchronize(h->stream));
    const size_t m = h->ivox.n_pts < capacity ? h->ivox.n_pts : capacity;
    if (m) FLS_CUDA(cudaMemcpy(xyzi, h->ivox.pts_all.p, m * sizeof(float4), cudaMemcpyDeviceToHost));
    *n = h->ivox.n_pts;
    return FLS_OK;
    FLS_CATCH
}

int fls_get_map_info(const fls_handle* hh, fls_map_info* out) {
    const Handle* h = reinterpret_cast<const Handle*>(hh);
    if (!h || !out) return FLS_ERR_INVALID_ARG;
    std::memset(out, 0, sizeof(*out));
    if (h->cfg.method == FLS_P2PLANE_IVOX) {
        out->n_points = (long long)h->ivox.n_pts;
        out->n_voxels = (long long)h->ivox.n_vox;
        out->table_slots = h->ivox.n_pts ? (long long)h->ivox.mask + 1 : 0;
        out->bytes = (long long)h->ivox.bytes();
        out->incremental_inserts = (long long)h->ivox.n_incremental;
        out->full_builds = (long long)h->ivox.n_full;
    } else if (h->cfg.method == FLS_NDT) {
        out->n_voxels = (long long)h->ndt.n_vox;
        out->table_slots = (long long)h->ndt.slots;
        out->bytes = (long long)h->ndt.bytes();
    } else if (h->cfg.method == FLS_ICP_P2P) {
        out->n_points = (long long)h->icp_map.grid.n_pts;
        out->n_voxels = (long long)h->icp_map.grid.n_vox;
        out->table_slots = h->icp_map.grid.n_pts ? (long long)h->icp_map.grid.mask + 1 : 0;
        out->bytes = (long long)h->icp_map.grid.bytes();
    } else {  // kd-tree plug-ins: planar map (+ corner map for LoamFull)
        const bool full = h->cfg.method == FLS_LOAM_FULL;
        out->n_points = (long long)(h->kd_planar.n + (full ? h->kd_corner.n : 0));
        out->n_voxels = (long long)(h->kd_planar.grid.n_vox + (full ? h->kd_corner.grid.n_vox : 0));
        out->table_slots = (h->kd_planar.n ? (long long)h->kd_planar.grid.mask + 1 : 0) + (full && h->kd_corner.n ? (long long)h->kd_corner.grid.mask + 1 : 0);
        out->bytes = (long long)(h->kd_planar.grid.bytes() + h->kd_planar.cloud.bytes() + (full ? h->kd_corner.grid.bytes() + h->kd_corner.cloud.bytes() : 0));
    }
    return FLS_OK;
}

int fls_ivox_add_points(fls_handle* hh, const void* pts, size_t n, size_t stride) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    if (!h || (!pts && n) || !stride_ok(stride)) return FLS_ERR_INVALID_ARG;
    if (h->cfg.method != FLS_P2PLANE_IVOX) return FLS_ERR_UNSUPPORTED;
    FLS_TRY
    h->begin_call();
    const float4* d = h->upload(pts, n, stride, h->stage);
    const int rc = h->ivox.append_and_build(d, n, h->cfg.ivox_capacity, h->stream);
    h->launches += h->ivox.launches;
    h->ivox.launches = 0;
    h->end_call(nullptr);
    return rc;
    FLS_CATCH
}

int fls_ivox_knn(fls_handle* hh, const void* queries, size_t n, size_t stride, int k, float* out_pts, int32_t* out_count) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    if (!h || !queries || !out_pts || !out_count || k != 5 || !stride_ok(stride)) return FLS_ERR_INVALID_ARG;
    if (h->cfg.method != FLS_P2PLANE_IVOX) return FLS_ERR_UNSUPPORTED;
    if (h->ivox.n_pts == 0) return FLS_ERR_NO_MAP;
    FLS_TRY
    h->begin_call();
    const float4* dq = h->upload(queries, n, stride, h->src);
    fls::DevBuf<float4> d_out;
    fls::DevBuf<int> d_found;
    d_out.reserve(n * 5);
    d_found.reserve(n);
    fls::launch_ivox_knn_test(h->ivox_view(), dq, (int)n, d_out.p, d_found.p, h->stream);
    FLS_CUDA(cudaMemcpyAsync(out_pts, d_out.p, n * 5 * sizeof(float4), cudaMemcpyDeviceToHost, h->stream));
    FLS_CUDA(cudaMemcpyAsync(out_count, d_found.p, n * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    h->end_call(nullptr);
    return FLS_OK;
    FLS_CATCH
}

int fls_voxel_grid(int device, const void* pts, size_t n, size_t stride, float leaf, float* out, size_t* n_out) {
    if ((!pts && n) || !out || !n_out || !stride_ok(stride) || !(leaf > 0.f)) return FLS_ERR_INVALID_ARG;
    if (check_device(device) != FLS_OK) return FLS_ERR_NO_DEVICE;
    FLS_TRY
    *n_out = 0;
    if (n == 0) return FLS_OK;
    return fls::with_workspace<VoxelWorkspace>(device, [&](VoxelWorkspace& w) -> int {
        long long h2d = 0;
        int launches = 0;
        w.in.reserve(n);
        w.out.reserve(n);
        fls::upload_records(pts, n, stride, w.in.p, w.raw, w.st, &h2d, &launches);
        const size_t m = fls::voxel_grid_device(w.in.p, n, leaf, w.out.p, w.sc, w.st, &launches);
        FLS_CUDA(cudaMemcpyAsync(out, w.out.p, m * 16, cudaMemcpyDeviceToHost, w.st));
        FLS_CUDA(cudaStreamSynchronize(w.st));
        *n_out = m;
        return FLS_OK;
    });
    FLS_CATCH
}

int fls_preprocess_loam(const fls_loam_frontend_cfg* cfg, const void* raw, const int32_t* ring, const float* time, size_t n, size_t stride,
                        const fls_imu_buffer* imu, float* corner, float* planar, float* d_corner, float* d_planar, size_t* n_corner, size_t* n_planar,
                        fls_match_stats* stats) {
    if (!cfg || !n_corner || !n_planar) return FLS_ERR_INVALID_ARG;
    *n_corner = *n_planar = 0;
    if ((!raw && n) || (!ring && n) || !stride_ok(stride) || n > 0x7fffffffull) return FLS_ERR_INVALID_ARG;
    if (!corner && !planar && !d_corner && !d_planar) return FLS_ERR_INVALID_ARG;
    if (!loam_frontend_cfg_ok(*cfg)) return FLS_ERR_INVALID_ARG;
    if (imu && imu->n_imu && !time && n) return FLS_ERR_INVALID_ARG;
    if (check_device(cfg->device) != FLS_OK) return FLS_ERR_NO_DEVICE;
    FLS_TRY
    return fls::preprocess_loam_device(*cfg, raw, ring, time, n, stride, imu, corner, planar, d_corner, d_planar, n_corner, n_planar, stats, false);
    FLS_CATCH
}

int fls_preprocess_loam_device(const fls_loam_frontend_cfg* cfg, const float* d_xyzi, const int32_t* d_ring, const float* d_time, size_t n,
                               const fls_imu_buffer* imu, float* corner, float* planar, float* d_corner, float* d_planar, size_t* n_corner,
                               size_t* n_planar, fls_match_stats* stats) {
    if (!cfg || !n_corner || !n_planar) return FLS_ERR_INVALID_ARG;
    *n_corner = *n_planar = 0;
    if ((!d_xyzi && n) || (!d_ring && n) || n > 0x7fffffffull) return FLS_ERR_INVALID_ARG;
    if (!corner && !planar && !d_corner && !d_planar) return FLS_ERR_INVALID_ARG;
    if (!loam_frontend_cfg_ok(*cfg)) return FLS_ERR_INVALID_ARG;
    if (imu && imu->n_imu && !d_time && n) return FLS_ERR_INVALID_ARG;
    if (check_device(cfg->device) != FLS_OK) return FLS_ERR_NO_DEVICE;
    FLS_TRY
    return fls::preprocess_loam_device(*cfg, d_xyzi, d_ring, d_time, n, FLS_LAYOUT_PACKED, imu, corner, planar, d_corner, d_planar, n_corner, n_planar,
                                       stats, true);
    FLS_CATCH
}

int fls_preprocess_device(int device, const float* d_xyzi, const float* d_time, size_t n, const fls_imu_buffer* imu, float min_distance,
                          float max_distance, int32_t jump_span, float planar_leaf, float* ordered, float* d_ordered, size_t* n_ordered, float* planar,
                          float* d_planar, size_t* n_planar) {
    if (!n_ordered || !n_planar) return FLS_ERR_INVALID_ARG;
    *n_ordered = *n_planar = 0;
    if ((!d_xyzi && n) || (!ordered && !d_ordered && !planar && !d_planar) || jump_span < 1 || !(planar_leaf > 0.f)) return FLS_ERR_INVALID_ARG;
    if (imu && imu->n_imu && !d_time && n) return FLS_ERR_INVALID_ARG;
    if (check_device(device) != FLS_OK) return FLS_ERR_NO_DEVICE;
    FLS_TRY
    return fls::preprocess_device_input(device, d_xyzi, d_time, n, imu, min_distance, max_distance, jump_span, planar_leaf, ordered, d_ordered, n_ordered,
                                        planar, d_planar, n_planar);
    FLS_CATCH
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
