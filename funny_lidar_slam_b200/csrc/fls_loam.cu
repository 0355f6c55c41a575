// fls_loam.cu — K5: the kd-tree LOAM plug-ins as one persistent Gauss-Newton kernel.
//
//   LoamPointToPlaneKdtree::Match  (include/registration/loam_point_to_plane_kdtree.h:82-157,204-288 upstream)
//   LoamFull::Match / CornerMatch / PlanarMatch  (include/registration/loam_full_kdtree.h:106-204,211-273,275-345)
//
// Both ask pcl::KdTreeFLANN for the EXACT 5 nearest map points of every transformed feature point — no radius: the
// LoamFull gate `d2[4] > point_search_thres` is applied after the search (:227,:291) and the kd-tree point-to-plane
// variant has no gate at all.  The GPU index is a uniform grid (floor keys, open-addressing table, cell-contiguous
// points) searched by expanding cubes: after the cube of Chebyshev radius R every unseen point is farther than
// (R + distance of the query to the nearest face of its own cell) cells, so the search stops — exactly — as soon as
// the current 5th distance is inside that bound; a finite gate stops it as soon as the bound passes the gate (the
// caller rejects the point either way), and a query that is still not settled after kMaxShell rings scans the whole
// map (far-away / tiny maps; exact by construction).  Ties in distance are broken by visit order (FLANN's order is
// unspecified too).
//
// The loop structure is the shared persistent one (gn_handover, fls_gn.cuh): one thread per feature point, corner
// points first then planar points (the order upstream sums them, :347-372), every class with its own persistent
// {J, residual} record and flag byte for the "flags reset once per Match" rule [quirk 1].
//
// KdPlugin at the end is the host half both plug-ins share: the sliding-window planar (and LoamFull's corner) local map,
// AddCloudToLocalMap and Match.
#include <cmath>

#include "fls_eig.cuh"
#include "fls_gn.cuh"
#include "fls_handle.h"
#include "fls_info.cuh"
#include "fls_plane.cuh"

namespace fls {

static constexpr int kLoamBlock = 256;

struct LoamArgs {
    const float4* __restrict__ corner;  // body-frame corner features (LoamFull only)
    int n_corner;
    const float4* __restrict__ planar;  // body-frame planar features
    int n_planar;
    GridView corner_map, planar_map;  // exact unbounded 5-NN over these
    double plane_thres;    // point_to_planar_thres
    double search_thres;   // point_search_thres on the 5th squared distance (+inf: none)
    double line_ratio;     // line_ratio_thres
    float gate;            // search_thres as the search's stop bound
    GnState* state;
    double* __restrict__ rec;  // [n_corner + n_planar][8] persistent {J[6], residual, -}
    unsigned char* __restrict__ flags;
};

namespace {

constexpr int kMaxShell = 6;

__device__ __forceinline__ void scan_cell(const GridView& g, int cx, int cy, int cz, float qx, float qy, float qz, Top5& nn, unsigned& n_cand) {
    unsigned start, count;
    if (!table_find(g.tab, g.mask, pack_key(cx, cy, cz), start, count)) return;
    n_cand += count;
#pragma unroll 2
    for (unsigned j = start; j < start + count; ++j) {
        const float4 p = __ldg(g.pts + j);
        nn.push(dist2_ref(p.x, p.y, p.z, qx, qy, qz), j);
    }
}

// kLoamLanes lanes share one query: lane `sub` visits every kLoamLanes-th cell, keeps a PRIVATE top-5 (the private lists
// of a group are disjoint), and the group's answer is their butterfly merge.
static constexpr int kLoamLanes = 8;

__device__ __forceinline__ void merge_group(Top5& m, unsigned group_mask) {
#pragma unroll
    for (int o = kLoamLanes / 2; o > 0; o >>= 1) {
        const float e0 = __shfl_xor_sync(group_mask, m.d0, o), e1 = __shfl_xor_sync(group_mask, m.d1, o), e2 = __shfl_xor_sync(group_mask, m.d2, o),
                    e3 = __shfl_xor_sync(group_mask, m.d3, o), e4 = __shfl_xor_sync(group_mask, m.d4, o);
        const unsigned j0 = __shfl_xor_sync(group_mask, m.k0, o), j1 = __shfl_xor_sync(group_mask, m.k1, o), j2 = __shfl_xor_sync(group_mask, m.k2, o),
                       j3 = __shfl_xor_sync(group_mask, m.k3, o), j4 = __shfl_xor_sync(group_mask, m.k4, o);
        m.push(e0, j0);
        m.push(e1, j1);
        m.push(e2, j2);
        m.push(e3, j3);
        m.push(e4, j4);
    }
}

// exact 5-NN; `gate` = squared distance beyond which the caller rejects the point anyway (INFINITY: none).
// Called by all lanes of a group with the same query; every lane returns the group's merged result in `nn`.
__device__ __noinline__ void grid_knn5(const GridView& g, int sub, unsigned group_mask, float qx, float qy, float qz, float gate, Top5& nn,
                                       unsigned& n_cand) {
    nn.init();
    n_cand = 0;
    if (g.n_pts < 5u) return;  // the tree cannot return 5 neighbours
    const float ux = __fmul_rn(qx, g.inv_cell), uy = __fmul_rn(qy, g.inv_cell), uz = __fmul_rn(qz, g.inv_cell);
    const float fx0 = floorf(ux), fy0 = floorf(uy), fz0 = floorf(uz);
    const int kx = (int)fx0, ky = (int)fy0, kz = (int)fz0;
    // distance (in cells) from the query to the nearest face of its own cell
    const float fx = ux - fx0, fy = uy - fy0, fz = uz - fz0;
    const float face = fminf(fminf(fminf(fx, 1.f - fx), fminf(fy, 1.f - fy)), fminf(fz, 1.f - fz));
    Top5 mine;
    mine.init();
#pragma unroll 1
    for (int s = sub; s < 27; s += kLoamLanes) scan_cell(g, kx + c_stencil[s][0], ky + c_stencil[s][1], kz + c_stencil[s][2], qx, qy, qz, mine, n_cand);
#pragma unroll 1
    for (int R = 1;; ++R) {
        nn = mine;
        merge_group(nn, group_mask);
        const float edge = ((float)R + face) * g.cell * 0.9995f;  // conservative: keys are floor(fl(p * inv_cell))
        const float b2 = edge * edge;
        if (nn.full() && nn.d4 <= b2) return;  // settled
        if (b2 > gate) return;                 // everything unseen lies beyond the gate
        if (R >= kMaxShell) break;
        const int S = R + 1;  // ring of Chebyshev radius S
        int cell = 0;
#pragma unroll 1
        for (int dz = -S; dz <= S; ++dz)
#pragma unroll 1
            for (int dy = -S; dy <= S; ++dy) {
                const bool face_row = (dz == -S || dz == S || dy == -S || dy == S);
#pragma unroll 1
                for (int dx = -S; dx <= S; dx += (face_row ? 1 : 2 * S), ++cell)
                    if ((cell & (kLoamLanes - 1)) == sub) scan_cell(g, kx + dx, ky + dy, kz + dz, qx, qy, qz, mine, n_cand);
            }
    }
    // exhaustive scan (far query or very sparse map)
    mine.init();
#pragma unroll 1
    for (unsigned j = (unsigned)sub; j < g.n_pts; j += kLoamLanes) {
        const float4 p = __ldg(g.pts + j);
        mine.push(dist2_ref(p.x, p.y, p.z, qx, qy, qz), j);
    }
    n_cand += g.n_pts / kLoamLanes;
    nn = mine;
    merge_group(nn, group_mask);
}

// LoamFull::CornerMatch per point (:219-270): line through the 5 neighbours by the principal axis of their covariance
__device__ __forceinline__ bool corner_term(const float4* __restrict__ P, const unsigned (&js)[5], const float4 sp, float qx, float qy, float qz,
                                            const double* __restrict__ pose, double line_ratio, double (&J)[6], double& res) {
    double X[5][3], c[3] = {0, 0, 0};
#pragma unroll
    for (int j = 0; j < 5; ++j) {
        const float4 a = __ldg(P + js[j]);
        X[j][0] = a.x; X[j][1] = a.y; X[j][2] = a.z;
        c[0] += X[j][0]; c[1] += X[j][1]; c[2] += X[j][2];
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) c[a] /= 5.0;  // rowwise().mean()  (:237)
    double S[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
    for (int j = 0; j < 5; ++j)
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int b = 0; b < 3; ++b) S[a * 3 + b] += (X[j][a] - c[a]) * (X[j][b] - c[b]);
#pragma unroll
    for (int k = 0; k < 9; ++k) S[k] /= 5.0;  // :239-242
    double lam[3], V[9];
    sym_eig3_dev(S, lam, V);
    if (lam[0] <= line_ratio * lam[1]) return false;  // :249
    const double nx = V[0], ny = V[3], nz = V[6];    // V.col(0); J does not depend on its sign
    const double vx = (double)qx - c[0], vy = (double)qy - c[1], vz = (double)qz - c[2];
    const double wx = vy * nz - vz * ny, wy = vz * nx - vx * nz, wz = vx * ny - vy * nx;  // (q - c) x n
    const double d = sqrt(wx * wx + wy * wy + wz * wz);                                   // :260
    const double ux = wx / d, uy = wy / d, uz = wz / d;
    // J.tail = (-n^)^T u = n x u ; J.head = (n^ (Rp)^)^T u = (Rp) x (n x u)   (:264-265)
    const double tx = ny * uz - nz * uy, ty = nz * ux - nx * uz, tz = nx * uy - ny * ux;
    const double px = sp.x, py = sp.y, pz = sp.z;
    const double rx = pose[0] * px + pose[1] * py + pose[2] * pz;
    const double ry = pose[3] * px + pose[4] * py + pose[5] * pz;
    const double rz = pose[6] * px + pose[7] * py + pose[8] * pz;
    J[0] = ry * tz - rz * ty;
    J[1] = rz * tx - rx * tz;
    J[2] = rx * ty - ry * tx;
    J[3] = tx;
    J[4] = ty;
    J[5] = tz;
    res = d;
    return true;
}

// Feature point i's fresh term at the pose s_pose (row-major R, t): corner points [0, n_corner) then planar points, the exact 5-NN of
// the point moved by the double pose, the point_search_thres gate and the line or plane fit -> J (6) and residual r in dx = [dθ, dt]
// order; n_cand: the map records it scanned.  Called by all kLoamLanes lanes of the point's group; returns true on lane 0 when the
// point has a term.  The Gauss-Newton loop and the information evaluation (fls_info.cuh) both call it.
__device__ __forceinline__ bool loam_point(const LoamArgs& a, int i, const double* s_pose, int sub, unsigned group_mask, double (&J)[6], double& r,
                                           unsigned& n_cand) {
    const bool is_corner = i < a.n_corner;
    const float4 sp = is_corner ? a.corner[i] : a.planar[i - a.n_corner];
    // pcl::transformPoint with the double transform, stored back as fp32 (:219-220, :284-285, kdtree :211-212)
    const float qx = xform_row_d(s_pose[0], s_pose[1], s_pose[2], s_pose[9], (double)sp.x, (double)sp.y, (double)sp.z);
    const float qy = xform_row_d(s_pose[3], s_pose[4], s_pose[5], s_pose[10], (double)sp.x, (double)sp.y, (double)sp.z);
    const float qz = xform_row_d(s_pose[6], s_pose[7], s_pose[8], s_pose[11], (double)sp.x, (double)sp.y, (double)sp.z);
    const GridView& g = is_corner ? a.corner_map : a.planar_map;
    Top5 nn;
    grid_knn5(g, sub, group_mask, qx, qy, qz, a.gate, nn, n_cand);
    bool use = false;
    if (sub == 0 && nn.full() && !((double)nn.d4 > a.search_thres)) {  // :227 / :291 (search_thres = +inf for the kd-tree point-to-plane plug-in)
        const unsigned js[5] = {nn.k0, nn.k1, nn.k2, nn.k3, nn.k4};
        unsigned fb = 0;
        use = is_corner ? corner_term(g.pts, js, sp, qx, qy, qz, s_pose, a.line_ratio, J, r)
                        : plane_term(g.pts, js, sp, qx, qy, qz, s_pose, a.plane_thres, J, r, fb);
    }
    return use;
}

// One persistent launch runs every Gauss-Newton iteration of a Match, on the CTAs (cta, ncta) of the sub-grid that serves the scan.
template <int BLOCK>
__device__ __forceinline__ void loam_gn_loop(const LoamArgs& a, const GnLoopCtl& ctl, const int cta, const int ncta) {
    __shared__ double s_pose[12];
    const int n_total = a.n_corner + a.n_planar;
    const int sub = threadIdx.x & (kLoamLanes - 1);
    const unsigned group_mask = ((1u << kLoamLanes) - 1u) << ((threadIdx.x & 31) & ~(kLoamLanes - 1));
    constexpr int kPerBlock = BLOCK / kLoamLanes;
    if (threadIdx.x < 12) s_pose[threadIdx.x] = threadIdx.x < 9 ? __ldcg(&a.state->R[threadIdx.x]) : __ldcg(&a.state->t[threadIdx.x - 9]);
    __syncthreads();
    for (int it = 0; it < ctl.gp.max_iterations; ++it) {  // the hand-over leaves the next pose in s_pose
        double acc[kNumAcc];
#pragma unroll
        for (int k = 0; k < kNumAcc; ++k) acc[k] = 0.0;
        for (int i = (unsigned)cta * kPerBlock + threadIdx.x / kLoamLanes; i < n_total; i += (unsigned)ncta * kPerBlock) {
            const bool is_corner = i < a.n_corner;
            double J[6], r = 0.0;
            unsigned n_cand;
            bool use = loam_point(a, i, s_pose, sub, group_mask, J, r, n_cand);
            acc[kAccCand] += (double)n_cand;
            if (sub != 0) continue;  // lane 0 of the group owns the point's record and sums
            double* rec = a.rec + (size_t)i * 8;
            if (use) {
#pragma unroll
                for (int k = 0; k < 6; ++k) rec[k] = J[k];
                rec[6] = r;
                a.flags[i] = 1;
            } else if (a.flags[i]) {  // stale contribution [quirk 1]
#pragma unroll
                for (int k = 0; k < 6; ++k) J[k] = rec[k];
                r = rec[6];
                use = true;
            }
            if (use) {
#pragma unroll
                for (int p = 0; p < 6; ++p)
#pragma unroll
                    for (int q = p; q < 6; ++q) acc[tri6(p, q)] += J[p] * J[q];
#pragma unroll
                for (int p = 0; p < 6; ++p) acc[21 + p] -= J[p] * r;
                acc[kAccRes] += r;
                if (is_corner) acc[kAccHits] += 1.0;  // number_valid_corner_ (reported, never gates)
                else acc[kAccValid] += 1.0;           // number_valid_planar_ (the < 50 failure test)
            }
        }
        if (gn_handover<BLOCK>(acc, ctl, it, s_pose, cta, ncta)) break;
    }
}

// every scan of a Match on its own sub-grid (gn_batch_loop, fls_gn.cuh); each scan's records and flags are its own range of one buffer
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) loam_gn_kernel(const GnBatchItem<LoamArgs>* __restrict__ items, int n_scans) {
    gn_batch_loop<BLOCK>(items, n_scans, [](const LoamArgs& a, const GnLoopCtl& ctl, int cta, int ncta) { loam_gn_loop<BLOCK>(a, ctl, cta, ncta); });
}


__global__ void loam_clear_flags_kernel(unsigned char* flags, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) flags[i] = 0;
}

}  // namespace

// FLS_FLAG_INFORMATION (fls_info.cuh): W = 1; LoamFull counts its corner and planar terms alike
template <>
struct InfoTerm<LoamArgs> {
    static constexpr int kBlock = kLoamBlock, kLanes = kLoamLanes;
    static __host__ __device__ int count(const LoamArgs& a) { return a.n_corner + a.n_planar; }
    static __device__ __forceinline__ void point(const LoamArgs& a, int i, const double* pose, const float*, int sub, unsigned mask,
                                                 double (&acc)[kNumAcc]) {
        double J[6], r = 0.0;
        unsigned n_cand;
        if (loam_point(a, i, pose, sub, mask, J, r, n_cand)) info_add_J(J, r, acc);
    }
};

static int loam_max_grid(int device) { return coresident_ctas((const void*)loam_gn_kernel<kLoamBlock>, kLoamBlock, 0, device); }
// clears the flags of every scan of the Match (n of them in all) in one launch when there are any, then the loop kernel
static void launch_loam(const GnBatchItem<LoamArgs>* d_items, int n_scans, unsigned char* flags, size_t n, int grid, cudaStream_t st) {
    if (n > 0) loam_clear_flags_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(flags, (int)n);
    launch_cooperative(loam_gn_kernel<kLoamBlock>, grid, kLoamBlock, 0, st, d_items, n_scans);
}

// ---- LoamPointToPlaneKdtree / LoamFull -------------------------------------------------------------------------------

static void window_info(const WindowMap& w, fls_map_info* out) {
    out->n_points += (long long)w.n;
    out->n_voxels += (long long)w.grid.n_vox;
    out->table_slots += w.n ? (long long)w.grid.table.slots : 0;
    out->bytes += (long long)(w.grid.bytes() + w.cloud.bytes());
}

class KdPlugin final : public Plugin {
    const bool full;             // LoamFull: {planar, corner} maps and features
    WindowMap planar;            // planar_cloud_deque_ and the search grid over it
    std::unique_ptr<WindowMap> corner;  // corner_cloud_deque_ and its grid: LoamFull only
    KeyFrameGate gate;
    DevBuf<double> rec;          // persistent {J[6], residual} records
    DevBuf<unsigned char> flags;
    DevBuf<float4> ins, ins_corner;  // Match-internal insert: the features at their final pose

    // The Match of B scans, in ONE cooperative launch (loam_gn_kernel — one sub-grid and one persistent Gauss-Newton loop per scan).
    // Scan s is the planar features d_planar[s] (n_planar[s] points) and, when d_corner is given (LoamFull), the corner features
    // d_corner[s] (n_corner[s] points); it owns records and flags [off[s], off[s] + its points) of one buffer, cleared together.
    int match_scans(int B, const float4* const* d_planar, const size_t* n_planar, const float4* const* d_corner, const size_t* n_corner, double* T,
                    int* converged, fls_match_stats* st) {
        const fls_config& cfg = h.cfg;
        if (planar.n == 0) return FLS_ERR_NO_MAP;
        size_t ns[kMaxBatch], off[kMaxBatch], total = 0;
        for (int s = 0; s < B; ++s) {
            ns[s] = n_planar[s] + (d_corner ? n_corner[s] : 0);
            if (ns[s] > 0x3fffffffull) return FLS_ERR_INVALID_ARG;
            off[s] = total;
            total += ns[s];
        }
        if (total > 0x7fffffffull) return FLS_ERR_INVALID_ARG;  // flags and records of a Match are indexed by int
        rec.reserve(total * 8 + 8);
        flags.reserve(total + 1);
        const GridView planar_view = planar.grid.view();
        const GridView corner_view = full ? corner->grid.view() : planar_view;
        // roofline accounting (K5): 16 B source point + 27 x 16 B slot probes + 56 B persistent record, 16 B per scanned map record.
        // GetFitnessScore reads the planar features.
        return h.match_subgrids<LoamArgs>(cfg.method, 50, B, ns, kLoamBlock / kLoamLanes, loam_max_grid(cfg.device), 16 + 16LL * 27 + 56, 16,
                                          d_planar[0], n_planar[0], T, converged, st,
                                          [&](int s, LoamArgs& a) {
                                              a.corner = d_corner ? d_corner[s] : nullptr;
                                              a.n_corner = d_corner ? (int)n_corner[s] : 0;
                                              a.planar = d_planar[s];
                                              a.n_planar = (int)n_planar[s];
                                              a.planar_map = planar_view;
                                              a.corner_map = corner_view;
                                              a.plane_thres = cfg.point_to_planar_thres;
                                              a.search_thres = full ? cfg.point_search_thres : INFINITY;
                                              a.line_ratio = cfg.line_ratio_thres;
                                              a.gate = full ? (float)cfg.point_search_thres * 1.0001f : INFINITY;
                                              a.state = h.state.p + s;
                                              a.rec = rec.p + off[s] * 8;
                                              a.flags = flags.p + off[s];
                                          },
                                          [&](const GnBatchItem<LoamArgs>* d_items, int grid) {
                                              launch_loam(d_items, B, flags.p, total, grid, h.call.stream);
                                              if (total > 0) h.call.launches++;  // the flag reset in front of the loop
                                          });
    }

  public:
    explicit KdPlugin(Handle& handle) : Plugin(handle, handle.cfg.method == FLS_LOAM_FULL ? kPlanarCorner : kPlanar), full(reads == kPlanarCorner) {
        const fls_config& cfg = h.cfg;
        // exact-search grids: LoamFull only needs neighbours inside sqrt(point_search_thres), so a cell of that size settles every
        // query in the 27-cell pass; the ungated point-to-plane variant uses ~2 map leafs
        if (full) {
            const float c = (float)(std::sqrt(cfg.point_search_thres > 0 ? cfg.point_search_thres : 1.0) * 1.001);
            planar.grid.res = c;
            corner = std::make_unique<WindowMap>();
            corner->grid.res = c;
        } else {
            const float c = 2.0f * (cfg.map_cloud_filter_size > 0.f ? cfg.map_cloud_filter_size : 0.5f);
            planar.grid.res = c < 0.8f ? 0.8f : c;
        }
    }

    int add_cloud(const float4* d_planar, size_t n_planar, const float4* d_corner, size_t n_corner) override {
        const fls_config& cfg = h.cfg;
        if (!full) {
            // loam_point_to_plane_kdtree.h:56-80: localization mode replaces the map, mapping mode slides a window; both
            // end in VoxelGridCloud(local_map, map_cloud_filter_size) + kd-tree
            const int rc = window_add(planar, d_planar, n_planar, (size_t)cfg.local_map_size, cfg.map_cloud_filter_size, true, cfg.localization_mode != 0,
                                      h.scratch, h.call);
            if (rc == FLS_OK) h.set_fit_cloud(planar.cloud.p, planar.n);  // GetFitnessScore searches the same tree (:159-183)
            return rc;
        }
        // loam_full_kdtree.h:66-104: {planar, corner}, both windows slide, filters only beyond 5 clouds
        const int rc = window_add(planar, d_planar, n_planar, (size_t)cfg.local_map_size, cfg.map_cloud_filter_size, false, false, h.scratch, h.call);
        if (rc != FLS_OK) return rc;
        return window_add(*corner, d_corner, n_corner, (size_t)cfg.corner_local_map_size, cfg.corner_map_filter_size, false, false, h.scratch, h.call);
    }

    int match(const float4* d_planar, size_t n_planar, const float4* d_corner, size_t n_corner, double* T, int* converged,
              fls_match_stats* st) override {
        const fls_config& cfg = h.cfg;
        const int rc = match_scans(1, &d_planar, &n_planar, &d_corner, &n_corner, T, converged, st);
        if (rc != FLS_OK) return rc;
        // key-frame insertion: loam_point_to_plane_kdtree.h:146-150 (gate evaluated before the mode test), loam_full_kdtree.h:178-186
        if (h.h_state.p->converged && gate.need(T, cfg.dist_thre_add_cloud, cfg.rot_thre_add_cloud) && (full || !cfg.localization_mode)) {
            int rc2;
            if (full) {
                ins.reserve(n_planar);
                ins_corner.reserve(n_corner);
                launch_transform_d(d_planar, n_planar, T, ins.p, h.call.stream);  // pcl::transformPointCloud(cloud, out, T_) with the double matrix
                launch_transform_d(d_corner, n_corner, T, ins_corner.p, h.call.stream);
                h.call.launches += 2;
                rc2 = add_cloud(ins.p, n_planar, ins_corner.p, n_corner);
            } else {
                ins.reserve(n_planar);
                launch_transform_f(d_planar, n_planar, T, ins.p, h.call.stream);  // TransformPointCloud(source, final): fp32 with R, t cast to float
                h.call.launches++;
                rc2 = add_cloud(ins.p, n_planar, nullptr, 0);
            }
            return h.inserted(rc2, st);
        }
        return FLS_OK;
    }

    // n_scans independent LoamPointToPlaneKdtree::Match calls on planar features against the same (static) map in ONE cooperative
    // launch.  The key-frame gate is left alone: in localization mode nothing is inserted, so its last_T cannot be observed.  A
    // batch of one is the single Match; LoamFull reads two clouds per scan and has no batch.
    int match_batch(int B, const void* const* scans, const size_t* n_in, size_t host_stride, double* T, int* converged,
                    fls_match_stats* st) override {
        if (full) return FLS_ERR_UNSUPPORTED;
        const float4* d_scans[kMaxBatch];
        const int rc = h.begin_batch(B, scans, n_in, host_stride, d_scans, st);
        if (rc != FLS_OK) return rc;
        if (B == 1) return match(d_scans[0], n_in[0], nullptr, 0, T, converged, st);
        return match_scans(B, d_scans, n_in, nullptr, nullptr, T, converged, st);
    }

    void map_info(fls_map_info* out) const override {  // planar map (+ corner map for LoamFull)
        window_info(planar, out);
        if (full) window_info(*corner, out);
    }
};

std::unique_ptr<Plugin> make_kd_plugin(Handle& h) { return std::make_unique<KdPlugin>(h); }

}  // namespace fls
