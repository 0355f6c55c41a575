// fls_handle.h — the object behind `fls_handle*`: configuration, the Call its entries run on, what every plug-in's Match shares, and the one
// registration plug-in that cfg.method names, which owns its map and the buffers only it uses.
#pragma once
#include <memory>
#include <vector>

#include "fls_common.cuh"
#include "fls_kernels.h"
#include "fls_maps.h"

namespace fls {

struct Handle;

// One registration plug-in (RegistrationInterface upstream: Match, AddCloudToLocalMap, GetFitnessScore).  It owns its map and the
// buffers only it uses, configures them when it is made, and hands GetFitnessScore the cloud it searches (Handle::set_fit_*) when
// AddCloudToLocalMap changes it; a plug-in without that cloud never does.  What a plug-in does not override is FLS_ERR_UNSUPPORTED.
struct Plugin {
    enum Clouds { kOrdered, kPlanar, kPlanarCorner };
    Handle& h;
    const Clouds reads;  // the clouds Match reads; AddCloudToLocalMap takes as many maps (LoamFull: {planar, corner})
    Plugin(Handle& handle, Clouds c) : h(handle), reads(c) {}
    virtual ~Plugin() = default;

    // what AddCloudToLocalMap returns before it reads a cloud (FLS_OK: it goes ahead)
    virtual int add_check() const { return FLS_OK; }
    // AddCloudToLocalMap of device clouds: the map cloud (+ the corner map when reads == kPlanarCorner)
    virtual int add_cloud(const float4* d, size_t n, const float4* d_corner, size_t n_corner) = 0;
    // Match of device clouds: the ordered scan or the planar features (+ the corner features when reads == kPlanarCorner)
    virtual int match(const float4* d, size_t n, const float4* d_corner, size_t n_corner, double* T, int* converged, fls_match_stats* st) = 0;
    virtual void map_info(fls_map_info* out) const = 0;

    // The plug-in-specific entries below do all their work in the override, from selecting the device or beginning the call on, so
    // that a plug-in without the entry answers with no side effect.
    // n_scans independent scans against the (static) map; the scans are host records of `host_stride` bytes or (0) device float4
    virtual int match_batch(int n_scans, const void* const* scans, const size_t* n, size_t host_stride, double* T, int* converged,
                            fls_match_stats* st) {
        return FLS_ERR_UNSUPPORTED;
    }
    // the same in two halves (fls_match_batch_begin / _end): enqueue without waiting, then wait and unpack
    virtual int batch_begin(int n_scans, const void* const* scans, const size_t* n, size_t host_stride, const double* T) {
        return FLS_ERR_UNSUPPORTED;
    }
    virtual int batch_end(double* T, int* converged, fls_match_stats* st) { return FLS_ERR_UNSUPPORTED; }
    virtual int batch_pending() const { return 0; }  // scans of the batch in flight
    // packed keys of the occupied voxels (at most cap of them; n: how many the map holds)
    virtual int voxel_keys(std::vector<unsigned long long>& packed, size_t cap, size_t* n) { return FLS_ERR_UNSUPPORTED; }
    virtual int ndt_voxels(std::vector<fls_ndt_voxel>& out) { return FLS_ERR_UNSUPPORTED; }
    virtual int map_points(float* xyzi, size_t cap, size_t* n) { return FLS_ERR_UNSUPPORTED; }
    virtual int ivox_knn(const void* queries, size_t n, size_t stride, float* out_pts, int32_t* out_count) { return FLS_ERR_UNSUPPORTED; }
    virtual int ivox_add_points(const void* pts, size_t n, size_t stride) { return FLS_ERR_UNSUPPORTED; }
};
std::unique_ptr<Plugin> make_ivox_plugin(Handle& h);  // LoamPointToPlaneIVOX (fls_p2plane.cu)
std::unique_ptr<Plugin> make_ndt_plugin(Handle& h);   // IncrementalNDT (fls_ndt.cu)
std::unique_ptr<Plugin> make_icp_plugin(Handle& h);   // IcpOptimized (fls_icp.cu)
std::unique_ptr<Plugin> make_kd_plugin(Handle& h);    // LoamPointToPlaneKdtree and LoamFull (fls_loam.cu)

// FLS_FLAG_INFORMATION: the evaluation of a Match's scans at their returned poses, enqueued before its read-back (fls_info.cuh), and
// the launches it adds to the call
template <class Args>
void enqueue_information(Handle& h, const Args* a, int B);
static constexpr int kInfoLaunches = 2;

// IsNeedAddCloud (icp_optimized.h:218-236, loam_point_to_plane_kdtree.h:186-202, loam_full_kdtree.h:356-371): key-frame gating on
// translation / RPY deltas against a persistent last_T that starts at the first pose it sees  [quirk 7]
struct KeyFrameGate {
    bool have_last = false;  // `static last_T` upstream
    double last_T[16];
    bool need(const double* T, double dist_thre, double rot_thre);
};

// the hypothesis grid of fls_relocalize (fls_b200.h): offsets -I..I in x and y, yaw offsets k0..K (n_yaw of them), P hypotheses
static constexpr long long kRelocMaxHypotheses = 1LL << 20;
static constexpr long long kRelocWideMaxHypotheses = 1LL << 31;  // and I <= 32767: fls_relocalize_wide, and G * P for fls_relocalize_multi
static constexpr int kRelocMaxGuesses = 64;                       // fls_relocalize_multi
struct RelocGrid {
    int I = 0, K = 0, k0 = 0;
    long long n_yaw = 1, P = 1;  // n_yaw reaches 2^31 on the full circle of the wide cap
};
// checks a relocalization configuration and sizes its grid (FLS_ERR_INVALID_ARG: see fls_relocalize, and fls_relocalize_wide's caps
// when wide)
int reloc_grid(const fls_reloc_cfg& c, RelocGrid* g, bool wide = false);
struct Reloc;  // relocalization's state on a handle (fls_reloc.cu)
struct RelocFree {
    void operator()(Reloc* r) const;
};

struct Handle {
    fls_config cfg;
    Call call;  // the stream of every entry, its timing events and the accounting of the current call

    // upload staging
    DevBuf<unsigned char> raw;  // strided caller records before repacking
    DevBuf<float4> src, src2;   // uploaded scans / queries, and LoamFull's corner features
    DevBuf<float4> up_cloud, up_corner;  // clouds uploaded for AddCloudToLocalMap (LoamFull: {planar, corner}) or as the global map

    // Gauss-Newton state shared by the plug-ins
    DevBuf<uint4> ll_rows;      // LL hand-over records of the persistent kernels: [grid][32] rows + pose records
    unsigned match_epoch = 0;   // tag prefix of those records
    DevBuf<unsigned char> subgrid_items;  // the items of a match_subgrids launch (GnBatchItem<Args>[B])
    DevBuf<GnState> state;
    PinnedBuf<GnState> h_state;  // the states of the last Match, read back (room for kMaxBatch)
    DevBuf<fls_iter_log> log;
    std::vector<fls_iter_log> h_log;  // FLS_FLAG_ITER_LOG: log_cap entries per scan of the last Match
    int log_cap = 0;
    std::vector<int> log_n = {0};     // entries of each scan's log (one element per scan of the last Match)
    double T_final[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    cudaEvent_t prof_ev[2] = {nullptr, nullptr};  // FLS_FLAG_PROFILE: around the fused Gauss-Newton launch of a Match
    bool profile = false;
    long long per_point_iter_bytes = 0;  // fixed part of the algorithmic bytes per point-iteration (set by gn_launch)
    long long per_cand_bytes = 0;        // bytes per scanned map record
    BuildScratch scratch;                // voxel-grid passes of Match and the local-map crop

    // FLS_FLAG_INFORMATION (fls_info.cuh): each Match evaluates its scans' records after its loop (enqueue_information) and read_back
    // copies them with the states; info_n of them belong to the last Match call (0: none)
    bool info_on = false;        // the handle's flag, off while a relocalization runs its internal Matches
    bool info_enqueued = false;  // the Match in progress has enqueued its evaluation
    int info_n = 0;
    DevBuf<fls_information> info;
    PinnedBuf<fls_information> h_info;
    DevBuf<double> info_part;  // per-CTA partial sums of the evaluation
    void info_reset() {  // a Match call begins, or one ended without records
        info_n = 0;
        info_enqueued = false;
    }

    // optional caller-owned device buffer that receives {pose, converged, iterations} per scan (fls_set_result_buffer_device)
    double* result_buf = nullptr;
    size_t result_cap = 0;

    // source cloud of the last Match (for GetFitnessScore): device pointer + count
    const float4* last_src = nullptr;
    size_t last_src_n = 0;

    std::unique_ptr<Plugin> plugin;

    // GetFitnessScore support: cloud the upstream kd-tree is built on (fit_pts: fit_cloud, or a cloud the plug-in keeps) + a search
    // grid sized for max_range; the poses scored, per-tile partials and per-pose {sum, count} of the scoring kernel (fls_reloc.cu)
    DevBuf<float4> fit_cloud;
    const float4* fit_pts = nullptr;
    size_t fit_cloud_n = 0;
    unsigned long long fit_cloud_version = 0, fit_grid_version = ~0ull;
    float fit_grid_range = -1.f;
    SearchGrid fit_grid;
    DevBuf<double> fit_pose, fit_part_sum, fit_out;
    DevBuf<unsigned> fit_part_cnt, fit_cnt;
    // relocalization's buffers, lattice and level record (fls_reloc.cu), made by its first call
    std::unique_ptr<Reloc, RelocFree> reloc;

    explicit Handle(const fls_config& c);
    ~Handle();
    void init();     // body of the constructor
    void release();  // streams, events, pinned memory
    Handle(const Handle&) = delete;
    Handle& operator=(const Handle&) = delete;

    void begin_call();  // makes cfg.device current and begins the call
    const float4* upload(const void* pts, size_t n, size_t stride, DevBuf<float4>& dst);
    void upload_into(const void* pts, size_t n, size_t stride, float4* dst);  // dst: room for n records
    // begin_call of a batch Match (clearing st[n_scans] when given) and its scans as device pointers: host records of `host_stride`
    // bytes go back to back into src, device scans as they are
    int begin_batch(int n_scans, const void* const* scans, const size_t* n, size_t host_stride, const float4** ptrs, fls_match_stats* st);
    void set_fit_cloud(const float4* d, size_t n);  // copies
    void set_fit_view(const float4* d, size_t n);   // refers to d until the next call

    // ---- the host half of a Match, shared by the plug-ins ----
    GnParams gn_params(int method, int min_effective) const;
    unsigned next_ll_epoch(size_t n_records);  // LL records for the next launch; returns its tag base
    fls_iter_log* scan_log(int s) { return log_cap ? log.p + (size_t)s * log_cap : nullptr; }
    double* scan_result(int s) { return (result_buf && (size_t)s < result_cap) ? result_buf + (size_t)s * kResultLen : nullptr; }
    // the control block of scan s's loop in a launch of tag base `tag_base`: its state, LL rows and pose record, the plug-in's
    // parameters, its iteration log and its result record
    GnLoopCtl loop_ctl(int s, int method, int min_effective, unsigned tag_base, uint4* rows, uint4* pose) {
        GnLoopCtl c;
        c.state = state.p + s;
        c.ll_rows = rows;
        c.ll_pose = pose;
        c.tag_base = tag_base;
        c.gp = gn_params(method, min_effective);
        c.log = scan_log(s);
        c.log_cap = log_cap;
        c.result = scan_result(s);
        return c;
    }
    // the fused Gauss-Newton launch: roofline byte rates, profile events around `launch`, the launch counter and the source
    // cloud GetFitnessScore reads afterwards
    template <class F>
    void gn_launch(long long point_iter_bytes, long long cand_bytes, const float4* src, size_t src_n, F&& launch) {
        per_point_iter_bytes = point_iter_bytes;
        per_cand_bytes = cand_bytes;
        if (profile) FLS_CUDA(cudaEventRecord(prof_ev[0], call.stream));
        launch();
        if (profile) FLS_CUDA(cudaEventRecord(prof_ev[1], call.stream));
        call.launches++;
        last_src = src;
        last_src_n = src_n;
    }
    void read_back(int n_scans);  // enqueues the copy of the states and of every scan's iteration log
    // after call.end: T / converged / stats and log_n of every scan (call-level figures on stats[0]), T_final from scan 0
    void unpack(int n_scans, const size_t* n_source, double* T, int* converged, fls_match_stats* st);
    // A single-scan Match on a persistent kernel of `grid` CTAs (NDT, ICP): control block, state from T, the gn_launch of
    // launch(ctl), the information evaluation of the loop arguments `a` when the flag is on, then the wait and T / converged / stats
    // of a scan of n_source points
    template <class Args, class F>
    void match_single(int method, int min_effective, int grid, long long point_iter_bytes, long long cand_bytes, const float4* src, size_t src_n,
                      size_t n_source, double* T, int* converged, fls_match_stats* st, const Args& a, F&& launch) {
        const unsigned tag_base = next_ll_epoch((size_t)grid * 32 + kLlPoseLen);  // may move ll_rows
        const GnLoopCtl ctl = loop_ctl(0, method, min_effective, tag_base, ll_rows.p, ll_rows.p + (size_t)grid * 32);
        launch_gn_init(state.p, T, call.stream);
        call.launches++;
        gn_launch(point_iter_bytes, cand_bytes, src, src_n, [&] { launch(ctl); });
        if (info_on) enqueue_information(*this, &a, 1);
        read_back(1);
        call.end(st);
        unpack(1, &n_source, T, converged, st);
    }
    // ---- a Match of one or more scans on sub-grids of one cooperative launch (NDT, ICP and kd-tree LOAM batches, kd-tree LOAM Match) ----
    // VoxelGridCloud of every distinct source of a batch, back to back in dst: scan s reads [off[s], off[s] + ns[s]), and a scan that
    // repeats an earlier (pointer, count) reads the range of its first occurrence.  FLS_ERR_INVALID_ARG past 2^30 filtered points.
    int filter_batch(int B, const float4* const* d, const size_t* n, float leaf, DevBuf<float4>& dst, size_t* off, size_t* ns);
    // The Gauss-Newton half of such a Match; a single kd-tree LOAM Match is B = 1, whose sub-grid is the whole grid.  Scan s (ns[s]
    // points, also its n_source) gets one CTA per `per_cta` points, all scaled down together when the `cap` co-resident CTAs of the
    // kernel cannot hold them (more scans than CTAs: FLS_ERR_INVALID_ARG).  Then, per scan: its control block and its item, whose arguments
    // fill(s, item.a) sets, and one launch that starts its state from T and writes the item to subgrid_items; the gn_launch of
    // launch(d_items, grid), the information evaluation of every scan's arguments when the flag is on, the wait, and T / converged /
    // stats of every scan.  fit_src / fit_n: the cloud GetFitnessScore reads afterwards.
    template <class Args, class Fill, class Launch>
    int match_subgrids(int method, int min_effective, int B, const size_t* ns, int per_cta, int cap, long long point_iter_bytes, long long cand_bytes,
                       const float4* fit_src, size_t fit_n, double* T, int* converged, fls_match_stats* st, Fill&& fill, Launch&& launch) {
        int need[kMaxBatch], tot_need = 0;
        for (int s = 0; s < B; ++s) {
            need[s] = (int)((ns[s] + per_cta - 1) / per_cta);
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
        GnBatchItem<Args>* d_items = reinterpret_cast<GnBatchItem<Args>*>(subgrid_items.reserve(sizeof(GnBatchItem<Args>) * (size_t)B));
        uint4* pose_base = ll_rows.p + (size_t)grid * 32;
        int cta0 = 0;
        Args args[kMaxBatch];  // what the information evaluation reads
        for (int s = 0; s < B; ++s) {
            GnBatchItem<Args> it;
            std::memset(&it, 0, sizeof(it));
            fill(s, it.a);
            if (info_on) args[s] = it.a;
            it.ctl = loop_ctl(s, method, min_effective, tag_base, ll_rows.p + (size_t)cta0 * 32, pose_base + (size_t)s * kLlPoseLen);
            it.cta0 = cta0;
            it.ncta = ncta[s];
            cta0 += ncta[s];
            launch_gn_start(it, d_items + s, T + 16 * s, call.stream);
            call.launches++;
        }
        gn_launch(point_iter_bytes, cand_bytes, fit_src, fit_n, [&] { launch(d_items, grid); });
        if (info_on) enqueue_information(*this, args, B);
        read_back(B);
        call.end(st);
        unpack(B, ns, T, converged, st);
        return FLS_OK;
    }
    // end of a Match that added its scan to the map with status rc: waits for the insertion and counts its launches too
    int inserted(int rc, fls_match_stats* st);

    int fitness(float max_range, float* score);
    int fit_grid_for(float max_range);  // (re)builds fit_grid for max_range when needed
    void fitness_enqueue(const float4* d_src, size_t n, int P, float max_range);  // P poses of fit_pose -> fit_out / fit_cnt
    // fls_relocalize, or fls_relocalize_wide / fls_relocalize_multi when wide, on a device scan (the call has begun; g from
    // reloc_grid(c, &g, wide)) over the grids of G column-major guesses (G = 1 and guesses == T for the single-guess entries; T
    // receives the chosen pose, or guess 0 after an empty coarse cloud); coarse_scores and coarse_cap are fls_relocalize's,
    // evaluations those of the wide entries
    int relocalize(const float4* d_scan, size_t n, const fls_reloc_cfg& c, const RelocGrid& g, bool wide, const double* guesses, int G, double* T,
                   fls_reloc_result* out, double* refined_T, int32_t* refined_converged, float* refined_fitness, int64_t* refined_index,
                   double* coarse_scores, size_t coarse_cap, int64_t* evaluations);
    int relocalize_levels(int64_t* nodes, int capacity) const;  // fls_relocalize_wide_levels (0 levels before a wide call)

    // localization-mode map path (fls_localmap.cu): resident global map, +-100 m crop around the pose when needed
    DevBuf<float4> global_map;
    size_t global_n = 0;
    DevBuf<unsigned char> crop_keep;
    DevBuf<float4> local_map;  // the last crop, handed to AddCloudToLocalMap
    double local_edge[6] = {0, 0, 0, 0, 0, 0};
    bool have_edge = false;
    int set_global_map(const void* pts, size_t n, size_t stride);
    int update_local_map(const double* T_colmajor, int* updated, size_t* n_local);
};

}  // namespace fls
