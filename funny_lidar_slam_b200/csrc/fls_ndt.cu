// fls_ndt.cu — K2 (NDT residual + reduction) and K8-NDT (voxel map build / incremental update).
//
// IncrementalNDT (include/registration/incremental_ndt.h upstream) keeps an unordered_map of list nodes holding
// {points_, mu_, sigma_, information_, ndt_estimated_, num_points_}.  Here:
//   * table  : open-addressing slots {packed key (C-truncation of q/voxel, [quirk 5]), voxel index, estimated flag}
//   * hot    : 80-byte records {mu, symmetric information} — the only thing the Match kernel reads
//   * cold   : sigma, counters and a carry buffer of <= min_points_in_voxel pending points per voxel, touched only
//              by AddCloudToLocalMap / UpdateVoxel (:130-227)
// LRU eviction at `capacity` (:203-206) is emulated exactly: stamps per voxel + a host simulation of the sequential insert
// (NdtMap::evict_lru).  The table and the eviction pass are the ones the iVox map uses: VoxelTable and LruEviction in fls_map.cu.
// NdtPlugin at the end is the plug-in's host half: its map, AddCloudToLocalMap and the single and batch Match.
#include <cub/cub.cuh>

#include <cstring>

#include "fls_gn.cuh"
#include "fls_eig.cuh"
#include "fls_handle.h"
#include "fls_info.cuh"
#include "fls_maps.h"

namespace fls {

static constexpr int kNdtBlock = 512;  // few CTA rows for the folder: a dense scan fills the device with ~150-300 CTAs instead of > 1000

struct NdtArgs {
    const float4* __restrict__ src;  // voxel-filtered scan, body frame
    int n;
    NdtView map;
    double outlier_thres;
    GnState* state;
};

namespace {

__device__ __forceinline__ int ndt_coord(double v, double inv) { return (int)__dmul_rn(v, inv); }  // cast<int>() truncates

__global__ void ndt_keys_kernel(const float4* __restrict__ pts, size_t n, double inv, unsigned long long* __restrict__ keys,
                                unsigned* __restrict__ idx) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 p = pts[i];
    keys[i] = pack_key(ndt_coord((double)p.x, inv), ndt_coord((double)p.y, inv), ndt_coord((double)p.z, inv));
    idx[i] = (unsigned)i;
}

__device__ __forceinline__ void inv3_sym_reg(const double* S, double* Ai) {
    // cofactor inverse of a general 3x3 (Eigen's fixed-size inverse, incremental_ndt.h:134,151 upstream)
    const double c00 = S[4] * S[8] - S[5] * S[7], c01 = S[5] * S[6] - S[3] * S[8], c02 = S[3] * S[7] - S[4] * S[6];
    const double det = S[0] * c00 + S[1] * c01 + S[2] * c02;
    const double id = 1.0 / det;
    Ai[0] = c00 * id; Ai[1] = (S[2] * S[7] - S[1] * S[8]) * id; Ai[2] = (S[1] * S[5] - S[2] * S[4]) * id;
    Ai[3] = c01 * id; Ai[4] = (S[0] * S[8] - S[2] * S[6]) * id; Ai[5] = (S[2] * S[3] - S[0] * S[5]) * id;
    Ai[6] = c02 * id; Ai[7] = (S[1] * S[6] - S[0] * S[7]) * id; Ai[8] = (S[0] * S[4] - S[1] * S[3]) * id;
}

struct NdtUpdateArgs {
    const float4* __restrict__ pts;          // filtered cloud, map frame
    const unsigned* __restrict__ idx_sorted;  // point indices grouped by voxel (stable => cloud order inside a voxel)
    const unsigned long long* __restrict__ run_keys;
    const unsigned* __restrict__ starts;
    const unsigned* __restrict__ counts;
    int runs;
    HashSlot* tab;
    unsigned mask;
    NdtHot* hot;
    NdtCold* cold;
    double* carry;
    int* counter;  // NdtMap::counter
    const int* free_list;
    int n_free;
    unsigned long long call_hi;  // call number << 32
    long long capacity;
    int min_pts, max_pts;
    int first_scan;
};

// sequential mean / covariance over the carried points followed by the run's points (incremental_ndt.h:92-110)
__device__ void mean_cov_seq(const double* carry, int nc, const float4* __restrict__ pts, const unsigned* __restrict__ idx, unsigned s, unsigned c,
                             double* mean, double* cov) {
    const int n = nc + (int)c;
    double sm[3] = {0, 0, 0};
    for (int k = 0; k < nc; ++k)
        for (int a = 0; a < 3; ++a) sm[a] += carry[k * 3 + a];
    for (unsigned k = 0; k < c; ++k) {
        const float4 p = __ldg(pts + idx[s + k]);
        sm[0] += (double)p.x;
        sm[1] += (double)p.y;
        sm[2] += (double)p.z;
    }
    for (int a = 0; a < 3; ++a) mean[a] = sm[a] / (double)n;
    double cc[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int k = 0; k < nc; ++k) {
        const double v[3] = {carry[k * 3] - mean[0], carry[k * 3 + 1] - mean[1], carry[k * 3 + 2] - mean[2]};
        for (int a = 0; a < 3; ++a)
            for (int b = 0; b < 3; ++b) cc[a * 3 + b] += v[a] * v[b];
    }
    for (unsigned k = 0; k < c; ++k) {
        const float4 p = __ldg(pts + idx[s + k]);
        const double v[3] = {(double)p.x - mean[0], (double)p.y - mean[1], (double)p.z - mean[2]};
        for (int a = 0; a < 3; ++a)
            for (int b = 0; b < 3; ++b) cc[a * 3 + b] += v[a] * v[b];
    }
    for (int a = 0; a < 9; ++a) cov[a] = cc[a] / (double)(n - 1);
}

__device__ __forceinline__ void store_hot(NdtHot* h, const double* mu, const double* info) {
    h->mu[0] = mu[0]; h->mu[1] = mu[1]; h->mu[2] = mu[2];
    h->info[0] = info[0];
    h->info[1] = 0.5 * (info[1] + info[3]);
    h->info[2] = 0.5 * (info[2] + info[6]);
    h->info[3] = info[4];
    h->info[4] = 0.5 * (info[5] + info[7]);
    h->info[5] = info[8];
    h->pad = 0.0;
}

// one thread per touched voxel: find-or-create, then UpdateVoxel (incremental_ndt.h:130-179 upstream)
__global__ void ndt_update_kernel(NdtUpdateArgs a, int* overflow) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= a.runs) return;
    const unsigned long long key = a.run_keys[r];
    const unsigned s = a.starts[r], c = a.counts[r];
    bool created;
    const unsigned h = table_claim(a.tab, a.mask, key, created);
    unsigned vi;
    if (created) {
        // indices of evicted voxels first (the LRU tail was evicted before this kernel: NdtMap::evict_lru), then fresh ones
        int id;
        const int k = atomicAdd(a.counter + NdtMap::kFreeCursor, 1);
        if (k < a.n_free) id = a.free_list[a.n_free - 1 - k];  // the list is a stack
        else id = atomicAdd(a.counter + NdtMap::kHiWater, 1);
        if ((long long)id >= a.capacity) atomicExch(overflow, 1);  // cannot happen once the eviction ran
        vi = (unsigned)id;
        a.tab[h].start = vi;
    } else {
        vi = a.tab[h].start;
    }
    if ((long long)vi >= a.capacity) return;
    NdtCold& cd = a.cold[vi];
    double* carry = a.carry + (size_t)vi * a.min_pts * 3;
    if (created) {
        cd.num_points = 0;
        cd.carry_count = 0;
        cd.estimated = 0;
        cd.alive = 1;
        cd.key = key;
        for (int k = 0; k < 9; ++k) cd.sigma[k] = 0;
    }
    cd.stamp = a.call_hi | (unsigned long long)a.idx_sorted[s + c - 1];  // moved to the front by its last point of this call (:208-210)
    if (!cd.estimated) cd.num_points += (int)c;  // VoxelData ctor / AddPoint (:66-76): counted only before the first estimate

    double mu[3], info[9];
    if (a.first_scan) {  // :131-143 — every touched voxel is (re-)estimated from the points of this call only
        if (c > 1u) {
            mean_cov_seq(carry, 0, a.pts, a.idx_sorted, s, c, mu, cd.sigma);
            double S[9];
            for (int k = 0; k < 9; ++k) S[k] = cd.sigma[k] + ((k % 4 == 0) ? 1.0e-3 : 0.0);
            inv3_sym_reg(S, info);
        } else {
            const float4 p = a.pts[a.idx_sorted[s]];
            mu[0] = (double)p.x; mu[1] = (double)p.y; mu[2] = (double)p.z;
            for (int k = 0; k < 9; ++k) info[k] = (k % 4 == 0) ? 1.0e2 : 0.0;
        }
        cd.estimated = 1;
        cd.carry_count = 0;
        store_hot(a.hot + vi, mu, info);
        a.tab[h].count = 1;
        return;
    }
    if (cd.estimated && cd.num_points > a.max_pts) return;  // :145-147 frozen
    const int nc = cd.carry_count;
    const int total = nc + (int)c;
    if (total > a.min_pts) {
        if (!cd.estimated) {  // :149-153
            mean_cov_seq(carry, nc, a.pts, a.idx_sorted, s, c, mu, cd.sigma);
            double S[9];
            for (int k = 0; k < 9; ++k) S[k] = cd.sigma[k] + ((k % 4 == 0) ? 1.0e-3 : 0.0);
            inv3_sym_reg(S, info);
            cd.estimated = 1;
        } else {  // :154-178 running merge + eigen clamp
            double cm[3], cv[9], nm[3], nv[9], om[3];
            mean_cov_seq(carry, nc, a.pts, a.idx_sorted, s, c, cm, cv);
            const NdtHot& oh = a.hot[vi];
            om[0] = oh.mu[0]; om[1] = oh.mu[1]; om[2] = oh.mu[2];
            const double m = (double)cd.num_points, n = (double)total;
            for (int k = 0; k < 3; ++k) nm[k] = (m * om[k] + n * cm[k]) / (m + n);
            for (int x = 0; x < 3; ++x)
                for (int y = 0; y < 3; ++y)
                    nv[x * 3 + y] = (m * (cd.sigma[x * 3 + y] + (om[x] - nm[x]) * (om[y] - nm[y])) + n * (cv[x * 3 + y] + (cm[x] - nm[x]) * (cm[y] - nm[y]))) / (m + n);
            for (int k = 0; k < 3; ++k) mu[k] = nm[k];
            for (int k = 0; k < 9; ++k) cd.sigma[k] = nv[k];
            cd.num_points += total;
            double lam[3], V[9];
            sym_eig3_dev(cd.sigma, lam, V);
            if (lam[1] < lam[0] * 1e-3) lam[1] = lam[0] * 1e-3;
            if (lam[2] < lam[0] * 1e-3) lam[2] = lam[0] * 1e-3;
            for (int x = 0; x < 3; ++x)
                for (int y = 0; y < 3; ++y)
                    info[x * 3 + y] = V[x * 3 + 0] * V[y * 3 + 0] / lam[0] + V[x * 3 + 1] * V[y * 3 + 1] / lam[1] + V[x * 3 + 2] * V[y * 3 + 2] / lam[2];
        }
        cd.carry_count = 0;
        store_hot(a.hot + vi, mu, info);
        a.tab[h].count = 1;
    } else {  // keep the points for a later estimate
        for (unsigned k = 0; k < c; ++k) {
            const float4 p = a.pts[a.idx_sorted[s + k]];
            carry[(nc + k) * 3 + 0] = (double)p.x;
            carry[(nc + k) * 3 + 1] = (double)p.y;
            carry[(nc + k) * 3 + 2] = (double)p.z;
        }
        cd.carry_count = total;
    }
}

// ---- LRU bookkeeping (incremental_ndt.h:193-214) -------------------------------------------------------------------------------
// which touched voxels exist already: how many are to be created, how many existing ones are touched
__global__ void ndt_lookup_kernel(int runs, const unsigned long long* __restrict__ run_keys, const HashSlot* __restrict__ tab, unsigned mask,
                                  int* __restrict__ run_vi, int* __restrict__ touch_run, int* counters) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= runs) return;
    unsigned vi, est;
    if (table_find(tab, mask, run_keys[r], vi, est)) {
        run_vi[r] = (int)vi;
        touch_run[vi] = r;
        atomicAdd(counters + NdtMap::kTouched, 1);
    } else {
        run_vi[r] = -1;
        atomicAdd(counters + NdtMap::kCreations, 1);
    }
}
__global__ void ndt_live_kernel(const NdtCold* __restrict__ cold, int hi_water, unsigned long long* __restrict__ stamps, unsigned* __restrict__ vis,
                                int* cursor) {
    const int vi = blockIdx.x * blockDim.x + threadIdx.x;
    if (vi >= hi_water || !cold[vi].alive) return;
    const int pos = atomicAdd(cursor, 1);
    stamps[pos] = cold[vi].stamp;
    vis[pos] = (unsigned)vi;
}
// first point of this call that touches candidate k (0xffffffff: none)
__global__ void ndt_cand_kernel(const unsigned* __restrict__ vis_sorted, int K, const int* __restrict__ touch_run, const unsigned* __restrict__ starts,
                                const unsigned* __restrict__ idx_sorted, unsigned* __restrict__ out) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= K) return;
    const int r = touch_run[vis_sorted[k]];
    out[k] = r >= 0 ? idx_sorted[starts[r]] : 0xffffffffu;
}
__global__ void ndt_create_times_kernel(int runs, const int* __restrict__ run_vi, const unsigned* __restrict__ starts,
                                        const unsigned* __restrict__ idx_sorted, unsigned* __restrict__ out, int* cursor) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= runs || run_vi[r] >= 0) return;
    out[atomicAdd(cursor, 1)] = idx_sorted[starts[r]];
}
__global__ void ndt_evict_kernel(const unsigned* __restrict__ victim_pos, const unsigned char* __restrict__ recreated, int n,
                                 const unsigned* __restrict__ vis_sorted, NdtCold* __restrict__ cold, int* __restrict__ free_list, int free_base,
                                 const int* __restrict__ touch_run, int* __restrict__ run_vi) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned vi = vis_sorted[victim_pos[i]];
    cold[vi].alive = 0;
    free_list[free_base + i] = (int)vi;
    if (recreated[i]) run_vi[touch_run[vi]] = -1;  // touched again later in the call: created anew, empty (:197-201)
}
__global__ void ndt_table_rebuild_kernel(const NdtCold* __restrict__ cold, int hi_water, HashSlot* tab, unsigned mask) {
    const int vi = blockIdx.x * blockDim.x + threadIdx.x;
    if (vi >= hi_water || !cold[vi].alive) return;
    bool created;  // the live keys are distinct
    HashSlot& slot = tab[table_claim(tab, mask, cold[vi].key, created)];
    slot.start = (unsigned)vi;
    slot.count = cold[vi].estimated ? 1u : 0u;
}
__global__ void ndt_dump_keys_kernel(const NdtCold* __restrict__ cold, int hi_water, unsigned long long* __restrict__ out, int* cursor) {
    const int vi = blockIdx.x * blockDim.x + threadIdx.x;
    if (vi >= hi_water || !cold[vi].alive) return;
    out[atomicAdd(cursor, 1)] = cold[vi].key;
}
__device__ __forceinline__ int unpack21(unsigned long long k, int shift) {
    const int c = (int)((k >> shift) & 0x1fffffu);
    return (c & 0x100000) ? c - 0x200000 : c;  // 21-bit two's complement
}
__global__ void ndt_dump_voxels_kernel(const NdtCold* __restrict__ cold, const NdtHot* __restrict__ hot, int hi_water, fls_ndt_voxel* __restrict__ out,
                                       int* cursor) {
    const int vi = blockIdx.x * blockDim.x + threadIdx.x;
    if (vi >= hi_water || !cold[vi].alive) return;
    const NdtCold& c = cold[vi];
    fls_ndt_voxel v;
    v.key[0] = unpack21(c.key, 42);
    v.key[1] = unpack21(c.key, 21);
    v.key[2] = unpack21(c.key, 0);
    v.estimated = c.estimated;
    v.num_points = c.num_points;
    v.carry_count = c.carry_count;
    for (int k = 0; k < 3; ++k) v.mu[k] = c.estimated ? hot[vi].mu[k] : 0.0;  // the hot record is written by the first estimate
    for (int k = 0; k < 6; ++k) v.info[k] = c.estimated ? hot[vi].info[k] : 0.0;
    out[atomicAdd(cursor, 1)] = v;
}

// ---- K2: NDT residual kernel -----------------------------------------------------------------------------------
// Source point i's terms at the pose s_pose (row-major R, t) into the sums `acc`: the seven-voxel probe, the outlier gate and
// J^T L J, -J^T L e, chi (incremental_ndt.h:255-275).  The Gauss-Newton loop and the information evaluation (fls_info.cuh) both call it.
__device__ __forceinline__ void ndt_point(const NdtArgs& a, int i, const double* s_pose, double (&acc)[kNumAcc]) {
    const float4 sp = a.src[i];
    const double px = sp.x, py = sp.y, pz = sp.z;
    const double* R = s_pose;
    const double qx = xform_row_dd(R[0], R[1], R[2], s_pose[9], px, py, pz);  // incremental_ndt.h:255
    const double qy = xform_row_dd(R[3], R[4], R[5], s_pose[10], px, py, pz);
    const double qz = xform_row_dd(R[6], R[7], R[8], s_pose[11], px, py, pz);
    const int kx = ndt_coord(qx, a.map.inv_voxel), ky = ndt_coord(qy, a.map.inv_voxel), kz = ndt_coord(qz, a.map.inv_voxel);  // :256
    double L0 = 0, L1 = 0, L2 = 0, L3 = 0, L4 = 0, L5 = 0;  // sum of information matrices (sym)
    double w0 = 0, w1 = 0, w2 = 0, chis = 0;
    int cnt = 0, hits = 0;
#pragma unroll 1
    for (int s = 0; s < 7; ++s) {  // stencil order of :122-127 = first 7 entries of c_stencil
        const unsigned long long key = pack_key(kx + c_stencil[s][0], ky + c_stencil[s][1], kz + c_stencil[s][2]);
        unsigned vi, est;
        if (!table_find(a.map.tab, a.map.mask, key, vi, est)) continue;
        ++hits;
        if (!est) continue;  // voxel exists but ndt_estimated_ is false (:263)
        const double2* hp = reinterpret_cast<const double2*>(a.map.hot + vi);
        const double2 h0 = __ldg(hp), h1 = __ldg(hp + 1), h2 = __ldg(hp + 2), h3 = __ldg(hp + 3), h4 = __ldg(hp + 4);
        const double ex = qx - h0.x, ey = qy - h0.y, ez = qz - h1.x;
        const double ixx = h1.y, ixy = h2.x, ixz = h2.y, iyy = h3.x, iyz = h3.y, izz = h4.x;
        const double ux = ixx * ex + ixy * ey + ixz * ez;
        const double uy = ixy * ex + iyy * ey + iyz * ez;
        const double uz = ixz * ex + iyz * ey + izz * ez;
        const double chi = ex * ux + ey * uy + ez * uz;
        if (isnan(chi) || chi > a.outlier_thres) continue;  // :267-271
        L0 += ixx; L1 += ixy; L2 += ixz; L3 += iyy; L4 += iyz; L5 += izz;
        w0 += ux; w1 += uy; w2 += uz;
        chis += chi;
        ++cnt;
    }
    acc[kAccHits] += (double)hits;
    acc[kAccCand] += (double)cnt;
    if (cnt > 0) {
        // B = -R * hat(p)  (3x3), J = [B | I]  (:273-275);  H = [[B^T L B, B^T L],[L B, L]],  err = -[B^T w ; w]
        double B[3][3];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const double r0 = R[r * 3 + 0], r1 = R[r * 3 + 1], r2 = R[r * 3 + 2];
            B[r][0] = -(r1 * pz - r2 * py);
            B[r][1] = -(r2 * px - r0 * pz);
            B[r][2] = -(r0 * py - r1 * px);
        }
        double LB[3][3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            LB[0][c] = L0 * B[0][c] + L1 * B[1][c] + L2 * B[2][c];
            LB[1][c] = L1 * B[0][c] + L3 * B[1][c] + L4 * B[2][c];
            LB[2][c] = L2 * B[0][c] + L4 * B[1][c] + L5 * B[2][c];
        }
        // upper triangle in dx = [dθ(0..2), dt(3..5)] order
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = r; c < 3; ++c) acc[tri6(r, c)] += B[0][r] * LB[0][c] + B[1][r] * LB[1][c] + B[2][r] * LB[2][c];
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) acc[tri6(r, 3 + c)] += LB[c][r];  // (B^T L)[r][c] = (L B)[c][r], L symmetric
        acc[tri6(3, 3)] += L0; acc[tri6(3, 4)] += L1; acc[tri6(3, 5)] += L2;
        acc[tri6(4, 4)] += L3; acc[tri6(4, 5)] += L4; acc[tri6(5, 5)] += L5;
#pragma unroll
        for (int r = 0; r < 3; ++r) acc[21 + r] -= (B[0][r] * w0 + B[1][r] * w1 + B[2][r] * w2);
        acc[24] -= w0; acc[25] -= w1; acc[26] -= w2;
        acc[kAccValid] += (double)cnt;
        acc[kAccRes] += chis;
    }
}

// One persistent launch runs every Gauss-Newton iteration of a Match (gn_handover, fls_gn.cuh): grid-stride over the
// points, per-thread sums, CTA row, last-CTA fold + solve + release.
template <int BLOCK>
__device__ __forceinline__ void ndt_gn_loop(const NdtArgs& a, const GnLoopCtl& ctl, const int cta, const int ncta) {
    __shared__ double s_pose[12];
    if (threadIdx.x < 9) s_pose[threadIdx.x] = __ldcg(&a.state->R[threadIdx.x]);
    else if (threadIdx.x < 12) s_pose[threadIdx.x] = __ldcg(&a.state->t[threadIdx.x - 9]);
    __syncthreads();
    for (int it = 0; it < ctl.gp.max_iterations; ++it) {  // the hand-over leaves the next pose in s_pose
    double acc[kNumAcc];
#pragma unroll
    for (int k = 0; k < kNumAcc; ++k) acc[k] = 0.0;

    for (int i = cta * BLOCK + threadIdx.x; i < a.n; i += ncta * BLOCK) ndt_point(a, i, s_pose, acc);
    if (gn_handover<BLOCK>(acc, ctl, it, s_pose, cta, ncta)) break;
    }
}

template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) ndt_gn_kernel(NdtArgs a, GnLoopCtl ctl) {
    ndt_gn_loop<BLOCK>(a, ctl, (int)blockIdx.x, (int)gridDim.x);
}

template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) ndt_gn_batch_kernel(const GnBatchItem<NdtArgs>* __restrict__ items, int n_scans) {
    gn_batch_loop<BLOCK>(items, n_scans, [](const NdtArgs& a, const GnLoopCtl& ctl, int cta, int ncta) { ndt_gn_loop<BLOCK>(a, ctl, cta, ncta); });
}

}  // namespace

// FLS_FLAG_INFORMATION: the loop's per-point term (fls_info.cuh), W = the voxel information, counted per point-voxel pair
template <>
struct InfoTerm<NdtArgs> {
    static constexpr int kBlock = 256, kLanes = 1;
    static __host__ __device__ int count(const NdtArgs& a) { return a.n; }
    static __device__ __forceinline__ void point(const NdtArgs& a, int i, const double* pose, const float*, int, unsigned, double (&acc)[kNumAcc]) {
        ndt_point(a, i, pose, acc);
    }
};

static int ndt_grid(int n, int device) {
    return clamp_grid((n + kNdtBlock - 1) / kNdtBlock, coresident_ctas((const void*)ndt_gn_kernel<kNdtBlock>, kNdtBlock, 0, device));
}
static void launch_ndt_loop(const NdtArgs& a, const GnLoopCtl& ctl, int grid, cudaStream_t st) {
    launch_cooperative(ndt_gn_kernel<kNdtBlock>, grid, kNdtBlock, 0, st, a, ctl);
}

static int ndt_max_grid(int device) { return coresident_ctas((const void*)ndt_gn_batch_kernel<kNdtBlock>, kNdtBlock, 0, device); }
static void launch_ndt_batch(const GnBatchItem<NdtArgs>* d_items, int n_scans, int grid, cudaStream_t st) {
    launch_cooperative(ndt_gn_batch_kernel<kNdtBlock>, grid, kNdtBlock, 0, st, d_items, n_scans);
}

void NdtMap::configure(double voxel_size, int min_points, int max_points, long long cap) {
    voxel = voxel_size;
    inv_voxel = 1.0 / voxel_size;
    min_pts = min_points;
    max_pts = max_points;
    capacity = cap;
}

int NdtMap::add_cloud(const float4* d_cloud, size_t n, float leaf, bool first_scan, Call& c) {
    if (n == 0) return FLS_OK;
    const cudaStream_t st = c.stream;
    filtered.reserve(n);
    const size_t nf = voxel_grid_device(d_cloud, n, leaf, filtered.p, scratch, c);  // :186
    if (nf == 0) return FLS_OK;
    if (table.slots == 0) {  // first use: size everything by the configured capacity
        table.size_for((size_t)capacity, 2);
        hot.reserve((size_t)capacity);
        cold.reserve((size_t)capacity);
        carry.reserve((size_t)capacity * (size_t)(min_pts > 0 ? min_pts : 1) * 3);
        counter.reserve(kCounters);
        FLS_CUDA(cudaMemsetAsync(counter.p, 0, kCounters * sizeof(int), st));
        table.clear(c);
    }
    BuildScratch& sc = scratch;
    sc.reserve_runs<unsigned long long>(nf);
    ndt_keys_kernel<<<grid_for(nf, 256), 256, 0, st>>>(filtered.p, nf, inv_voxel, sc.keys.p, sc.idx.p);
    sc.sort_pairs<unsigned long long>(nf, 63, c);
    const int runs = sc.encode_runs<unsigned long long>(nf, c);
    sc.run_starts(runs, c);
    // ---- LRU bookkeeping: which touched voxels exist, how many are created, who has to go first --------------------------------
    const int hi_water0 = hi_water;
    run_vi.reserve((size_t)runs + 1);
    touch_run.reserve((size_t)capacity + 1);
    free_list.reserve((size_t)capacity + 1);
    FLS_CUDA(cudaMemsetAsync(counter.p + kOverflow, 0, (kCounters - kOverflow) * sizeof(int), st));
    if (hi_water0 > 0) FLS_CUDA(cudaMemsetAsync(touch_run.p, 0xff, sizeof(int) * (size_t)hi_water0, st));
    ndt_lookup_kernel<<<grid_for(runs, 256), 256, 0, st>>>(runs, sc.uniq.p, table.buf.p, table.mask, run_vi.p, touch_run.p, counter.p);
    int hc[kCounters] = {};
    FLS_CUDA(cudaMemcpyAsync(hc, counter.p, sizeof(hc), cudaMemcpyDeviceToHost, st));
    c.sync();
    c.launches += 1;
    const int n_new = hc[kCreations], n_touched = hc[kTouched];
    ++call_no;
    // upstream: after every creation `if (data_.size() >= capacity_) pop_back()` (:203-206) — the list never holds `capacity` voxels
    if ((long long)n_vox + n_new >= capacity) {
        const int rc = evict_lru(runs, n_new, n_touched, c);
        if (rc != FLS_OK) return rc;
    }
    NdtUpdateArgs ua;
    ua.pts = filtered.p;
    ua.idx_sorted = sc.idx_sorted.p;
    ua.run_keys = sc.uniq.p;
    ua.starts = sc.starts.p;
    ua.counts = sc.counts.p;
    ua.runs = runs;
    ua.tab = table.buf.p;
    ua.mask = table.mask;
    ua.hot = hot.p;
    ua.cold = cold.p;
    ua.carry = carry.p;
    ua.counter = counter.p;
    ua.free_list = free_list.p;
    ua.n_free = n_free;
    ua.call_hi = call_no << 32;
    ua.capacity = capacity;
    ua.min_pts = min_pts;
    ua.max_pts = max_pts;
    ua.first_scan = first_scan ? 1 : 0;
    FLS_CUDA(cudaMemsetAsync(counter.p + kOverflow, 0, 2 * sizeof(int), st));  // overflow flag, free-stack cursor
    ndt_update_kernel<<<grid_for(runs, 128), 128, 0, st>>>(ua, counter.p + kOverflow);
    int h[3] = {0, 0, 0};  // up to the free-stack cursor
    FLS_CUDA(cudaMemcpyAsync(h, counter.p, 3 * sizeof(int), cudaMemcpyDeviceToHost, st));
    c.sync();
    c.launches += 6;
    hi_water = h[kHiWater];
    n_free -= h[kFreeCursor] < n_free ? h[kFreeCursor] : n_free;  // the creations popped that many indices off the free stack
    n_vox += (size_t)n_new;
    if (h[kOverflow]) return FLS_ERR_CAPACITY;
    return FLS_OK;
}

// Evicts what upstream's sequential insert would evict during this call (exact, including a victim that is touched again later in
// the call): candidates = live voxels by ascending stamp, simulated on the host against the creation times of the new voxels.
int NdtMap::evict_lru(int runs, int n_new, int n_touched, Call& c) {
    const cudaStream_t st = c.stream;
    BuildScratch& sc = scratch;
    const int hw = hi_water;
    const size_t n_live = n_vox;
    if (n_live == 0) return FLS_ERR_CAPACITY;  // the first cloud alone overflows the capacity: upstream dereferences an erased voxel (:216-220)
    ndt_live_kernel<<<grid_for(hw, 256), 256, 0, st>>>(cold.p, hw, eviction.stamps.reserve(n_live + 1), eviction.ids.reserve(n_live + 1),
                                                       counter.p + kLiveCursor);
    ndt_create_times_kernel<<<grid_for(runs, 256), 256, 0, st>>>(runs, run_vi.p, sc.starts.p, sc.idx_sorted.p, sc.k32b.reserve((size_t)n_new + 1),
                                                                counter.p + kCreateCursor);
    c.launches += 2;
    const int rc = eviction.run((int)n_live, sc.k32b.p, n_new, n_touched, n_live, capacity, sc.cub_tmp, c,
                                [&](const unsigned* vis_sorted, int K, unsigned* out) {
                                    ndt_cand_kernel<<<grid_for(K, 256), 256, 0, st>>>(vis_sorted, K, touch_run.p, sc.starts.p, sc.idx_sorted.p, out);
                                });
    if (rc != FLS_OK) return rc;
    const int n_victims = (int)eviction.n_victims;
    n_vox = n_vox + eviction.n_recreated - eviction.n_victims;
    if (n_victims == 0) return FLS_OK;
    // victims -> free list, their keys out of the table (rebuild: open addressing has no cheap delete)
    ndt_evict_kernel<<<grid_for(n_victims, 128), 128, 0, st>>>(eviction.victims.p, eviction.recreated.p, n_victims, eviction.ids_sorted.p, cold.p,
                                                              free_list.p, n_free, touch_run.p, run_vi.p);
    n_free += n_victims;
    table.clear(c);
    ndt_table_rebuild_kernel<<<grid_for(hw, 256), 256, 0, st>>>(cold.p, hw, table.buf.p, table.mask);
    c.launches += 2;
    return FLS_OK;
}

size_t NdtMap::dump_keys(unsigned long long* h_out, size_t cap, cudaStream_t st) {
    if (n_vox == 0 || hi_water == 0) return 0;
    scratch.keys.reserve(n_vox + 1);
    FLS_CUDA(cudaMemsetAsync(counter.p + kDumpCursor, 0, sizeof(int), st));
    ndt_dump_keys_kernel<<<grid_for(hi_water, 256), 256, 0, st>>>(cold.p, hi_water, scratch.keys.p, counter.p + kDumpCursor);
    int n = 0;
    FLS_CUDA(cudaMemcpyAsync(&n, counter.p + kDumpCursor, sizeof(int), cudaMemcpyDeviceToHost, st));
    FLS_CUDA(cudaStreamSynchronize(st));
    const size_t m = (size_t)n < cap ? (size_t)n : cap;
    FLS_CUDA(cudaMemcpy(h_out, scratch.keys.p, sizeof(unsigned long long) * m, cudaMemcpyDeviceToHost));
    return m;
}

void NdtMap::dump_voxels(std::vector<fls_ndt_voxel>& out, cudaStream_t st) {
    out.clear();
    if (n_vox == 0 || hi_water == 0) return;
    DevBuf<fls_ndt_voxel> d;
    d.reserve(n_vox + 1);
    FLS_CUDA(cudaMemsetAsync(counter.p + kDumpCursor, 0, sizeof(int), st));
    ndt_dump_voxels_kernel<<<grid_for(hi_water, 256), 256, 0, st>>>(cold.p, hot.p, hi_water, d.p, counter.p + kDumpCursor);
    int n = 0;
    FLS_CUDA(cudaMemcpyAsync(&n, counter.p + kDumpCursor, sizeof(int), cudaMemcpyDeviceToHost, st));
    FLS_CUDA(cudaStreamSynchronize(st));
    out.resize((size_t)n);
    if (n) FLS_CUDA(cudaMemcpy(out.data(), d.p, sizeof(fls_ndt_voxel) * (size_t)n, cudaMemcpyDeviceToHost));
}

// ---- IncrementalNDT ----------------------------------------------------------------------------------------------

class NdtPlugin final : public Plugin {
    NdtMap map;
    bool first_scan = true;  // flag_first_scan_ (incremental_ndt.h:394)
    DevBuf<float4> scan;     // VoxelGridCloud of the source(s) (:232)
    DevBuf<float4> ins;      // Match-internal insert: the filtered scan moved by the input guess

  public:
    explicit NdtPlugin(Handle& handle) : Plugin(handle, kOrdered) {
        map.configure(h.cfg.ndt_voxel_size, h.cfg.ndt_min_points_in_voxel, h.cfg.ndt_max_points_in_voxel, h.cfg.ndt_capacity);
    }

    int add_cloud(const float4* d_cloud, size_t n, const float4*, size_t) override {
        const fls_config& cfg = h.cfg;
        const int rc = map.add_cloud(d_cloud, n, cfg.source_cloud_filter_size, first_scan, h.call);
        if (cfg.localization_mode && rc == FLS_OK) {
            // kdtree_flann_.setInputCloud(cloud_world) — the voxel-filtered cloud (incremental_ndt.h:188-190)
            const size_t nf = voxel_grid_device(d_cloud, n, cfg.source_cloud_filter_size, map.filtered.p, map.scratch, h.call);
            h.set_fit_cloud(map.filtered.p, nf);
        }
        first_scan = cfg.localization_mode != 0;  // :222-226
        return rc;
    }

    int match(const float4* d_in, size_t n_in, const float4*, size_t, double* T, int* converged, fls_match_stats* st) override {
        const fls_config& cfg = h.cfg;
        if (map.n_vox == 0) return FLS_ERR_NO_MAP;  // CHECK(!grids_.empty())
        scan.reserve(n_in);
        const size_t n = voxel_grid_device(d_in, n_in, cfg.source_cloud_filter_size, scan.p, h.scratch, h.call);  // :232
        const int ni = (int)n;
        const int grid = ndt_grid(ni, cfg.device);
        double T_in[16];
        std::memcpy(T_in, T, sizeof(T_in));
        NdtArgs a;
        a.src = scan.p;
        a.n = ni;
        a.map = map.view();
        a.outlier_thres = cfg.ndt_outlier_thres;
        a.state = h.state.p;
        // roofline accounting (SURVEY.md §8d, K2): 16 B source point + 7 x 16 B slot probes per point-iteration,
        // 80 B voxel record per estimated voxel hit; the 6x6 sums are fused (no per-point output).
        h.match_single(FLS_NDT, cfg.ndt_min_effective_pts, grid, 16 + 16LL * 7, 80, scan.p, n, n, T, converged, st, a,
                       [&](const GnLoopCtl& ctl) { launch_ndt_loop(a, ctl, grid, h.call.stream); });
        if (!h.h_state.p->failed && !cfg.localization_mode) {
            // :326-330 — the scan enters the map transformed by the INPUT guess T, not the optimised pose  [quirk 6]
            ins.reserve(n);
            launch_transform_f(scan.p, n, T_in, ins.p, h.call.stream);
            h.call.launches++;
            return h.inserted(add_cloud(ins.p, n, nullptr, 0), st);
        }
        return FLS_OK;
    }

    // n_scans independent IncrementalNDT::Match calls against the same (static) map in ONE cooperative launch (ndt_gn_batch_kernel —
    // one sub-grid and one persistent Gauss-Newton loop per scan).  Localization semantics only: the map is not modified
    // (incremental_ndt.h:222-226, flag_first_scan_ stays set).
    int match_batch(int B, const void* const* scans, const size_t* n_in, size_t host_stride, double* T, int* converged,
                    fls_match_stats* st) override {
        const float4* d_scans[kMaxBatch];
        const int rc = h.begin_batch(B, scans, n_in, host_stride, d_scans, st);
        if (rc != FLS_OK) return rc;
        if (B == 1) return match(d_scans[0], n_in[0], nullptr, 0, T, converged, st);
        const fls_config& cfg = h.cfg;
        if (map.n_vox == 0) return FLS_ERR_NO_MAP;
        // VoxelGridCloud of every distinct source (incremental_ndt.h:232)
        size_t off[kMaxBatch], ns[kMaxBatch];
        const int rf = h.filter_batch(B, d_scans, n_in, cfg.source_cloud_filter_size, scan, off, ns);
        if (rf != FLS_OK) return rf;
        const NdtView view = map.view();
        return h.match_subgrids<NdtArgs>(FLS_NDT, cfg.ndt_min_effective_pts, B, ns, kNdtBlock, ndt_max_grid(cfg.device), 16 + 16LL * 7, 80,
                                         scan.p + off[0], ns[0], T, converged, st,
                                         [&](int s, NdtArgs& a) {
                                             a.src = scan.p + off[s];
                                             a.n = (int)ns[s];
                                             a.map = view;
                                             a.outlier_thres = cfg.ndt_outlier_thres;
                                             a.state = h.state.p + s;
                                         },
                                         [&](const GnBatchItem<NdtArgs>* d_items, int grid) { launch_ndt_batch(d_items, B, grid, h.call.stream); });
    }

    void map_info(fls_map_info* out) const override {
        out->n_voxels = (long long)map.n_vox;
        out->table_slots = (long long)map.table.slots;
        out->bytes = (long long)map.bytes();
    }

    int voxel_keys(std::vector<unsigned long long>& packed, size_t cap, size_t* n) override {
        FLS_CUDA(cudaSetDevice(h.cfg.device));
        packed.resize(cap + 1);
        packed.resize(map.dump_keys(packed.data(), cap, h.call.stream));
        *n = map.n_vox;
        return FLS_OK;
    }

    int ndt_voxels(std::vector<fls_ndt_voxel>& out) override {
        FLS_CUDA(cudaSetDevice(h.cfg.device));
        map.dump_voxels(out, h.call.stream);
        return FLS_OK;
    }
};

std::unique_ptr<Plugin> make_ndt_plugin(Handle& h) { return std::make_unique<NdtPlugin>(h); }

}  // namespace fls
