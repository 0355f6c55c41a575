// fls_icp.cu — K3: bounded exact 1-NN point-to-point residual + reduction (IcpOptimized).
//
// IcpOptimized::Match (include/registration/icp_optimized.h:54-163 upstream) asks a kd-tree for the exact
// nearest map point and then rejects it when d^2 > max_correspond_distance [quirk 4: squared distance against
// an unsquared threshold].  A correspondence can therefore only survive inside radius sqrt(threshold), so a
// uniform grid with cell >= that radius searched over its 27-cell neighbourhood returns the identical
// correspondence for every accepted point and "nothing" exactly where upstream rejects.  IcpPlugin at the end is the plug-in's host
// half: its sliding-window local map, AddCloudToLocalMap and Match.
#include <cmath>

#include "fls_gn.cuh"
#include "fls_handle.h"
#include "fls_info.cuh"

namespace fls {

static constexpr int kIcpBlock = 512;  // 64 queries x 8 lanes per CTA: few rows for the folder

struct IcpArgs {
    const float4* __restrict__ src;  // voxel-filtered scan, body frame
    int n;
    GridView map;  // search grid over the voxel-filtered local map
    double max_corr;
    GnState* state;
};

namespace {

// Sub-warp version for the Gauss-Newton loop: kIcpLanes lanes share one query, lane `sub` visits stencil cells
// sub, sub+kIcpLanes, ...; the winner is the lexicographic minimum of (d2, stencil position, point index) — the same
// point the sequential scan above keeps (strict '<' in visit order).  All lanes of the group return the result.
static constexpr int kIcpLanes = 8;
__device__ __forceinline__ bool grid_nn1_coop(const GridView& g, int sub, unsigned group_mask, float qx, float qy, float qz, float& best_d,
                                              unsigned& best_j, unsigned& n_cand, unsigned& n_hits) {
    best_d = INFINITY;
    best_j = 0xffffffffu;
    unsigned best_s = 0xffffu;
    n_cand = 0;
    n_hits = 0;
    const float ux = __fmul_rn(qx, g.inv_cell), uy = __fmul_rn(qy, g.inv_cell), uz = __fmul_rn(qz, g.inv_cell);
    const int kx = (int)floorf(ux), ky = (int)floorf(uy), kz = (int)floorf(uz);
#pragma unroll 1
    for (int s = sub; s < 27; s += kIcpLanes) {
        const int cx = kx + c_stencil[s][0], cy = ky + c_stencil[s][1], cz = kz + c_stencil[s][2];
        unsigned start, count;
        if (!table_find(g.tab, g.mask, pack_key(cx, cy, cz), start, count)) continue;
        n_cand += count;
        n_hits += 1;
#pragma unroll 2
        for (unsigned j = start; j < start + count; ++j) {
            const float4 p = __ldg(g.pts + j);
            const float d = dist2_ref(p.x, p.y, p.z, qx, qy, qz);
            if (d < best_d) {
                best_d = d;
                best_j = j;
                best_s = (unsigned)s;
            }
        }
    }
#pragma unroll
    for (int o = kIcpLanes / 2; o > 0; o >>= 1) {
        const float od = __shfl_xor_sync(group_mask, best_d, o);
        const unsigned oj = __shfl_xor_sync(group_mask, best_j, o);
        const unsigned os = __shfl_xor_sync(group_mask, best_s, o);
        const bool take = (od < best_d) || (od == best_d && (os < best_s || (os == best_s && oj < best_j)));
        if (take) {
            best_d = od;
            best_j = oj;
            best_s = os;
        }
    }
    return best_j != 0xffffffffu;
}

// Source point i's term at the pose s_pose (row-major R, t; s_posef: the same cast to float) into the sums `acc`: the bounded
// 1-NN of the point moved by the float pose, the max_correspond_distance gate and J = [I | -R hat(p)] in dx = [dt, dθ] order
// (icp_optimized.h:80-126).  Called by all kIcpLanes lanes of the point's group; lane 0 adds the term.  The Gauss-Newton loop and
// the information evaluation (fls_info.cuh) both call it.
__device__ __forceinline__ void icp_point(const IcpArgs& a, int i, const double* s_pose, const float* s_posef, int sub, unsigned group_mask,
                                          double (&acc)[kNumAcc]) {
    const float4 sp = a.src[i];
    const float qx = xform_row_f(s_posef[0], s_posef[1], s_posef[2], s_posef[9], sp.x, sp.y, sp.z);
    const float qy = xform_row_f(s_posef[3], s_posef[4], s_posef[5], s_posef[10], sp.x, sp.y, sp.z);
    const float qz = xform_row_f(s_posef[6], s_posef[7], s_posef[8], s_posef[11], sp.x, sp.y, sp.z);
    float d2;
    unsigned j, nc, nh;
    const bool found = grid_nn1_coop(a.map, sub, group_mask, qx, qy, qz, d2, j, nc, nh);
    acc[kAccCand] += (double)nc;
    acc[kAccHits] += (double)nh;
    if (sub == 0 && found && !((double)d2 > a.max_corr)) {  // icp_optimized.h:87
        const float4 m = __ldg(a.map.pts + j);
        const double e0 = (double)qx - (double)m.x, e1 = (double)qy - (double)m.y, e2 = (double)qz - (double)m.z;
        const double px = sp.x, py = sp.y, pz = sp.z;
        const double* R = s_pose;
        double A[3][3];  // -R * hat(p)   (:100)
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const double r0 = R[r * 3 + 0], r1 = R[r * 3 + 1], r2 = R[r * 3 + 2];
            A[r][0] = -(r1 * pz - r2 * py);
            A[r][1] = -(r2 * px - r0 * pz);
            A[r][2] = -(r0 * py - r1 * px);
        }
        // dx = [dt(0..2), dθ(3..5)]:  H = [[I, A],[A^T, A^T A]],  b = -[e ; A^T e]
        acc[tri6(0, 0)] += 1.0; acc[tri6(1, 1)] += 1.0; acc[tri6(2, 2)] += 1.0;
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) acc[tri6(r, 3 + c)] += A[r][c];
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = r; c < 3; ++c) acc[tri6(3 + r, 3 + c)] += A[0][r] * A[0][c] + A[1][r] * A[1][c] + A[2][r] * A[2][c];
        acc[21] -= e0; acc[22] -= e1; acc[23] -= e2;
#pragma unroll
        for (int r = 0; r < 3; ++r) acc[24 + r] -= (A[0][r] * e0 + A[1][r] * e1 + A[2][r] * e2);
        acc[kAccValid] += 1.0;
        acc[kAccRes] += sqrt(e0 * e0 + e1 * e1 + e2 * e2);  // total_res += error.norm()  (:126)
    }
}

// One persistent launch runs every Gauss-Newton iteration of a Match (gn_handover, fls_gn.cuh), on the CTAs (cta, ncta) of the
// sub-grid that serves the scan.
template <int BLOCK>
__device__ __forceinline__ void icp_gn_loop(const IcpArgs& a, const GnLoopCtl& ctl, const int cta, const int ncta) {
    __shared__ double s_pose[12];
    __shared__ float s_posef[12];
    const int sub = threadIdx.x & (kIcpLanes - 1);
    const unsigned group_mask = ((1u << kIcpLanes) - 1u) << ((threadIdx.x & 31) & ~(kIcpLanes - 1));
    constexpr int kPerBlock = BLOCK / kIcpLanes;
    if (threadIdx.x < 12) s_pose[threadIdx.x] = threadIdx.x < 9 ? __ldcg(&a.state->R[threadIdx.x]) : __ldcg(&a.state->t[threadIdx.x - 9]);
    __syncthreads();
    for (int it = 0; it < ctl.gp.max_iterations; ++it) {  // the hand-over leaves the next pose in s_pose
        if (threadIdx.x < 12) s_posef[threadIdx.x] = (float)s_pose[threadIdx.x];  // R.cast<float>(), t.cast<float>()  (pointcloud_utility.h:145-146)
        __syncthreads();
        double acc[kNumAcc];
#pragma unroll
        for (int k = 0; k < kNumAcc; ++k) acc[k] = 0.0;

        for (int i = (unsigned)cta * kPerBlock + threadIdx.x / kIcpLanes; i < a.n; i += (unsigned)ncta * kPerBlock) {
            icp_point(a, i, s_pose, s_posef, sub, group_mask, acc);
        }
        if (gn_handover<BLOCK>(acc, ctl, it, s_pose, cta, ncta)) break;
    }
}

template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) icp_gn_kernel(IcpArgs a, GnLoopCtl ctl) {
    icp_gn_loop<BLOCK>(a, ctl, (int)blockIdx.x, (int)gridDim.x);
}

// a batch of scans, one sub-grid each (gn_batch_loop, fls_gn.cuh)
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) icp_gn_batch_kernel(const GnBatchItem<IcpArgs>* __restrict__ items, int n_scans) {
    gn_batch_loop<BLOCK>(items, n_scans, [](const IcpArgs& a, const GnLoopCtl& ctl, int cta, int ncta) { icp_gn_loop<BLOCK>(a, ctl, cta, ncta); });
}

}  // namespace

// FLS_FLAG_INFORMATION: the loop's per-point term (fls_info.cuh), W = I
template <>
struct InfoTerm<IcpArgs> {
    static constexpr int kBlock = kIcpBlock, kLanes = kIcpLanes;
    static __host__ __device__ int count(const IcpArgs& a) { return a.n; }
    static __device__ __forceinline__ void point(const IcpArgs& a, int i, const double* pose, const float* posef, int sub, unsigned mask,
                                                 double (&acc)[kNumAcc]) {
        icp_point(a, i, pose, posef, sub, mask, acc);
    }
};

static int icp_grid_blocks(int n, int device) {
    const int per_block = kIcpBlock / kIcpLanes;
    return clamp_grid((n + per_block - 1) / per_block, coresident_ctas((const void*)icp_gn_kernel<kIcpBlock>, kIcpBlock, 0, device));
}
static void launch_icp_loop(const IcpArgs& a, const GnLoopCtl& ctl, int grid, cudaStream_t st) {
    launch_cooperative(icp_gn_kernel<kIcpBlock>, grid, kIcpBlock, 0, st, a, ctl);
}
static int icp_max_grid(int device) { return coresident_ctas((const void*)icp_gn_batch_kernel<kIcpBlock>, kIcpBlock, 0, device); }
static void launch_icp_batch(const GnBatchItem<IcpArgs>* d_items, int n_scans, int grid, cudaStream_t st) {
    launch_cooperative(icp_gn_batch_kernel<kIcpBlock>, grid, kIcpBlock, 0, st, d_items, n_scans);
}

// ---- IcpOptimized ------------------------------------------------------------------------------------------------

class IcpPlugin final : public Plugin {
    WindowMap window;  // cloud_deque_ / local_map_ptr_ (icp_optimized.h:173-187, 246)
    KeyFrameGate gate;
    DevBuf<float4> scan;  // VoxelGridCloud of the source (:57)
    DevBuf<float4> ins;   // Match-internal insert: the filtered scan at its final pose

  public:
    explicit IcpPlugin(Handle& handle) : Plugin(handle, kOrdered) {
        // search grid of the bounded exact 1-NN: cell >= sqrt(max_correspond_distance)  [quirk 4]
        const double d = h.cfg.icp_max_correspond_distance;
        window.grid.res = (float)(std::sqrt(d > 0 ? d : 1.0) * 1.001);
    }

    int add_cloud(const float4* d_cloud, size_t n, const float4*, size_t) override {
        // icp_optimized.h:173-187: mapping mode slides a window of the last local_map_size clouds, localization mode replaces
        // the map; both end in local_map_ptr_ = VoxelGridCloud(local_map_ptr_, map_cloud_filter_size_)
        const int rc = window_add(window, d_cloud, n, (size_t)h.cfg.local_map_size, h.cfg.map_cloud_filter_size, true, h.cfg.localization_mode != 0,
                                  h.scratch, h.call);
        h.set_fit_view(window.cloud.p, window.n);  // GetFitnessScore searches the same cloud
        return rc;
    }

    int match(const float4* d_in, size_t n_in, const float4*, size_t, double* T, int* converged, fls_match_stats* st) override {
        const fls_config& cfg = h.cfg;
        if (n_in <= 10) return FLS_ERR_TOO_FEW_POINTS;  // CHECK_GT(ordered_cloud_.size(), 10u)  (:55)
        if (window.grid.n_pts == 0) return FLS_ERR_NO_MAP;
        scan.reserve(n_in);
        const size_t n = voxel_grid_device(d_in, n_in, cfg.source_cloud_filter_size, scan.p, h.scratch, h.call);  // :57
        const int ni = (int)n;
        const int grid = icp_grid_blocks(ni, cfg.device);
        IcpArgs a;
        a.src = scan.p;
        a.n = ni;
        a.map = window.grid.view();
        a.max_corr = cfg.icp_max_correspond_distance;
        a.state = h.state.p;
        // roofline accounting (SURVEY.md §8d, K3): 16 B source point + 27 x 16 B slot probes, 16 B per scanned map record
        h.match_single(FLS_ICP_P2P, 0, grid, 16 + 16LL * 27, 16, scan.p, n, n, T, converged, st, a,
                       [&](const GnLoopCtl& ctl) { launch_icp_loop(a, ctl, grid, h.call.stream); });
        // IsNeedAddCloud (:218-236): key-frame gating on translation / RPY deltas against a persistent last_T
        if (h.h_state.p->converged && !cfg.localization_mode && gate.need(T, cfg.dist_thre_add_cloud, cfg.rot_thre_add_cloud)) {
            ins.reserve(n);
            launch_transform_f(scan.p, n, T, ins.p, h.call.stream);  // :156 TransformPointCloud(source, final) in float
            h.call.launches++;
            return h.inserted(add_cloud(ins.p, n, nullptr, 0), st);
        }
        return FLS_OK;
    }

    // n_scans independent IcpOptimized::Match calls against the same (static) map in ONE cooperative launch (icp_gn_batch_kernel —
    // one sub-grid and one persistent Gauss-Newton loop per scan).  The single Match's refusals come first, before anything is
    // uploaded or launched; a batch of one is the single Match.
    int match_batch(int B, const void* const* scans, const size_t* n_in, size_t host_stride, double* T, int* converged,
                    fls_match_stats* st) override {
        for (int s = 0; s < B; ++s)
            if (!scans[s] && n_in[s]) return FLS_ERR_INVALID_ARG;
        for (int s = 0; s < B; ++s)
            if (n_in[s] <= 10) return FLS_ERR_TOO_FEW_POINTS;  // CHECK_GT(ordered_cloud_.size(), 10u)  (:55)
        if (window.grid.n_pts == 0) return FLS_ERR_NO_MAP;
        const float4* d_scans[kMaxBatch];
        const int rc = h.begin_batch(B, scans, n_in, host_stride, d_scans, st);
        if (rc != FLS_OK) return rc;
        if (B == 1) return match(d_scans[0], n_in[0], nullptr, 0, T, converged, st);
        const fls_config& cfg = h.cfg;
        size_t off[kMaxBatch], ns[kMaxBatch];
        const int rf = h.filter_batch(B, d_scans, n_in, cfg.source_cloud_filter_size, scan, off, ns);  // :57
        if (rf != FLS_OK) return rf;
        const GridView view = window.grid.view();
        return h.match_subgrids<IcpArgs>(FLS_ICP_P2P, 0, B, ns, kIcpBlock / kIcpLanes, icp_max_grid(cfg.device), 16 + 16LL * 27, 16, scan.p + off[0],
                                         ns[0], T, converged, st,
                                         [&](int s, IcpArgs& a) {
                                             a.src = scan.p + off[s];
                                             a.n = (int)ns[s];
                                             a.map = view;
                                             a.max_corr = cfg.icp_max_correspond_distance;
                                             a.state = h.state.p + s;
                                         },
                                         [&](const GnBatchItem<IcpArgs>* d_items, int grid) { launch_icp_batch(d_items, B, grid, h.call.stream); });
    }

    void map_info(fls_map_info* out) const override {
        const SearchGrid& g = window.grid;
        out->n_points = (long long)g.n_pts;
        out->n_voxels = (long long)g.n_vox;
        out->table_slots = g.n_pts ? (long long)g.table.slots : 0;
        out->bytes = (long long)g.bytes();
    }
};

std::unique_ptr<Plugin> make_icp_plugin(Handle& h) { return std::make_unique<IcpPlugin>(h); }

}  // namespace fls
