// fls_reloc.cu — GetFitnessScore of many poses of one cloud, and relocalization from a coarse pose (fls_relocalize).
//
// pose_score_kernel is the one fitness path of the library: for P poses of one cloud it returns, per pose, the sum of the fp32 squared
// 1-NN distances <= max_range (in fp64) and how many there are.  A CTA stages a tile of the cloud in shared memory once and sweeps
// PPC poses over it; each pose's partial of that tile is reduced in a fixed tree, written to its own slot, and a second kernel adds
// the tiles of every pose in index order.  No atomics: every result is reproducible bit for bit and independent of scheduling.
// GetFitnessScore (Handle::fitness) is its one-pose-per-CTA form; relocalization scores its whole hypothesis grid with 8 poses per
// CTA, keeps the best by a stable radix sort of the scores, refines them with the plug-in's batch Match and scores the refined poses
// with the same one-pose-per-CTA form that a later fls_fitness runs.
#include <cfloat>
#include <cmath>
#include <cstring>

#include <cub/device/device_radix_sort.cuh>

#include "fls_handle.h"

namespace fls {

namespace {

constexpr int kScoreBlock = 256;

// nearest map point within the 27-cell neighbourhood; returns false when the neighbourhood is empty
__device__ __forceinline__ bool grid_nn1(const GridView& g, float qx, float qy, float qz, float& best_d, unsigned& best_j, unsigned& n_cand,
                                         unsigned& n_hits) {
    best_d = INFINITY;
    best_j = 0xffffffffu;
    n_cand = 0;
    n_hits = 0;
    const float ux = __fmul_rn(qx, g.inv_cell), uy = __fmul_rn(qy, g.inv_cell), uz = __fmul_rn(qz, g.inv_cell);
    const int kx = (int)floorf(ux), ky = (int)floorf(uy), kz = (int)floorf(uz);
    const float cell = 1.0f / g.inv_cell;  // not g.cell: the two can differ in the last bit
#pragma unroll 1
    for (int s = 0; s < 27; ++s) {
        const int cx = kx + c_stencil[s][0], cy = ky + c_stencil[s][1], cz = kz + c_stencil[s][2];
        // lower bound of the distance from q to the cell box, in metres (conservative by 0.1 %)
        const float ax = fmaxf(0.f, fmaxf((float)cx - ux, ux - (float)(cx + 1)));
        const float ay = fmaxf(0.f, fmaxf((float)cy - uy, uy - (float)(cy + 1)));
        const float az = fmaxf(0.f, fmaxf((float)cz - uz, uz - (float)(cz + 1)));
        const float lb = (ax * ax + ay * ay + az * az) * cell * cell * 0.998f;
        if (lb > best_d) continue;
        unsigned start, count;
        if (!table_find(g.tab, g.mask, pack_key(cx, cy, cz), start, count)) continue;
        n_cand += count;
        n_hits += 1;
#pragma unroll 1
        for (unsigned j = start; j < start + count; ++j) {
            const float4 p = __ldg(g.pts + j);
            const float d = dist2_ref(p.x, p.y, p.z, qx, qy, qz);
            if (d < best_d) {
                best_d = d;
                best_j = j;
            }
        }
    }
    return best_j != 0xffffffffu;
}

struct ScoreArgs {
    GridView g;
    const float4* __restrict__ src;
    int n;
    const double* __restrict__ poses;  // [P][12]: row-major R, then t (fp64; cast to float here, as TransformPointCloud does)
    int P;
    float max_range;
    int n_tiles;
    double* __restrict__ part_sum;  // [P][n_tiles]
    unsigned* __restrict__ part_cnt;
};

// grid (ceil(P / PPC), min(n_tiles, 65535)): CTA (x, y) scores poses x*PPC .. x*PPC+PPC-1 on tiles y, y + gridDim.y, ... of TILE
// points each, one partial per (pose, tile)
template <int PPC, int TILE>
__global__ void __launch_bounds__(kScoreBlock) pose_score_kernel(ScoreArgs a) {
    constexpr int TPP = kScoreBlock / PPC;  // threads per pose
    __shared__ float4 s_pts[TILE];
    __shared__ double s_sum[kScoreBlock];
    __shared__ unsigned s_cnt[kScoreBlock];
    const int sub = threadIdx.x % TPP;
    const int pose = blockIdx.x * PPC + threadIdx.x / TPP;
    float r[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) r[k] = pose < a.P ? (float)__ldg(a.poses + (size_t)pose * 12 + k) : 0.f;
    for (int tile = blockIdx.y; tile < a.n_tiles; tile += gridDim.y) {  // uniform across the CTA
        const size_t base = (size_t)tile * TILE;
        const int m = (int)min((size_t)TILE, (size_t)a.n - base);
        for (int i = threadIdx.x; i < m; i += kScoreBlock) s_pts[i] = a.src[base + i];
        double sum = 0.0;
        unsigned cnt = 0;
        __syncthreads();
        if (pose < a.P) {
#pragma unroll 1
            for (int i = sub; i < m; i += TPP) {
                const float4 sp = s_pts[i];
                const float qx = xform_row_f(r[0], r[1], r[2], r[9], sp.x, sp.y, sp.z);
                const float qy = xform_row_f(r[3], r[4], r[5], r[10], sp.x, sp.y, sp.z);
                const float qz = xform_row_f(r[6], r[7], r[8], r[11], sp.x, sp.y, sp.z);
                float d2;
                unsigned j, nc, nh;
                if (grid_nn1(a.g, qx, qy, qz, d2, j, nc, nh) && d2 <= a.max_range) {
                    sum += (double)d2;
                    cnt += 1;
                }
            }
        }
        s_sum[threadIdx.x] = sum;
        s_cnt[threadIdx.x] = cnt;
        __syncthreads();  // also: every read of s_pts is done before the next tile overwrites it
#pragma unroll
        for (int o = TPP / 2; o > 0; o >>= 1) {  // fixed tree inside each pose's group of threads
            if (sub < o) {
                s_sum[threadIdx.x] += s_sum[threadIdx.x + o];
                s_cnt[threadIdx.x] += s_cnt[threadIdx.x + o];
            }
            __syncthreads();
        }
        if (sub == 0 && pose < a.P) {
            a.part_sum[(size_t)pose * a.n_tiles + tile] = s_sum[threadIdx.x];
            a.part_cnt[(size_t)pose * a.n_tiles + tile] = s_cnt[threadIdx.x];
        }
    }
}

// per pose: the tiles in order -> {sum, count}; with keys: also the coarse score, its sort key (the bits of a non-negative double
// order as the values do) and the identity permutation
__global__ void pose_score_reduce_kernel(const double* __restrict__ part_sum, const unsigned* __restrict__ part_cnt, int P, int n_tiles, int m,
                                         float max_range, double* __restrict__ sum_out, unsigned* __restrict__ cnt_out, double* __restrict__ score,
                                         unsigned long long* __restrict__ key, unsigned* __restrict__ idx) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    double s = 0.0;
    unsigned c = 0;
    for (int t = 0; t < n_tiles; ++t) {
        s += part_sum[(size_t)p * n_tiles + t];
        c += part_cnt[(size_t)p * n_tiles + t];
    }
    if (sum_out) {
        sum_out[p] = s;
        cnt_out[p] = c;
    }
    if (score) {
        const double v = (s + (double)(m - (int)c) * (double)max_range) / (double)m;
        score[p] = v;
        key[p] = (unsigned long long)__double_as_longlong(v);
        idx[p] = (unsigned)p;
    }
}

// the hypothesis grid of fls_relocalize (fls_b200.h): pose p in fp64, row-major R | t
struct RelocGridArgs {
    double R[9], t[3];  // the guess
    double xy_step, yaw_step;
    int I, K, k0, n_yaw;  // yaw offsets k0 .. K
    int P;
};
__global__ void reloc_poses_kernel(RelocGridArgs g, double* __restrict__ poses) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= g.P) return;
    const int nx = 2 * g.I + 1;
    const int ky = p % g.n_yaw, ix = (p / g.n_yaw) % nx, jy = p / (g.n_yaw * nx);
    const double psi = __dmul_rn((double)(g.k0 + ky), g.yaw_step);
    const double c = cos(psi), s = sin(psi);
    double* o = poses + (size_t)p * 12;
    for (int j = 0; j < 3; ++j) {
        const double a = g.R[j], b = g.R[3 + j];
        o[j] = __dsub_rn(__dmul_rn(c, a), __dmul_rn(s, b));
        o[3 + j] = __dadd_rn(__dmul_rn(s, a), __dmul_rn(c, b));
        o[6 + j] = g.R[6 + j];
    }
    o[9] = __dadd_rn(g.t[0], __dmul_rn((double)(ix - g.I), g.xy_step));
    o[10] = __dadd_rn(g.t[1], __dmul_rn((double)(jy - g.I), g.xy_step));
    o[11] = g.t[2];
}

// the selected hypotheses: {index, coarse score, pose} records, read back in one copy
struct RelocPick {
    long long index;
    double score;
    double pose[12];
};
__global__ void reloc_pick_kernel(const unsigned* __restrict__ idx_sorted, const double* __restrict__ score, const double* __restrict__ poses, int n,
                                  RelocPick* __restrict__ out) {
    const int r = threadIdx.x;
    if (r >= n) return;
    const unsigned i = idx_sorted[r];
    out[r].index = i;
    out[r].score = score[i];
    for (int k = 0; k < 12; ++k) out[r].pose[k] = poses[(size_t)i * 12 + k];
}

constexpr int kFitTile = kScoreBlock;  // GetFitnessScore: one pose per CTA, one point per thread
constexpr int kCoarseTile = 2048;      // the hypothesis grid: 8 poses per CTA over 2048 staged points (32 KB)
constexpr int kCoarsePoses = 8;

void pose_score_launch(bool coarse, const GridView& g, const float4* d_src, int n, const double* d_poses, int P, float max_range, double* part_sum,
                       unsigned* part_cnt, cudaStream_t st) {
    ScoreArgs a{g, d_src, n, d_poses, P, max_range, 0, part_sum, part_cnt};
    const int tile = coarse ? kCoarseTile : kFitTile, ppc = coarse ? kCoarsePoses : 1;
    a.n_tiles = (n + tile - 1) / tile;
    const dim3 grid((unsigned)((P + ppc - 1) / ppc), (unsigned)(a.n_tiles < 65535 ? a.n_tiles : 65535));
    if (coarse) pose_score_kernel<kCoarsePoses, kCoarseTile><<<grid, kScoreBlock, 0, st>>>(a);
    else pose_score_kernel<1, kFitTile><<<grid, kScoreBlock, 0, st>>>(a);
    FLS_CUDA(cudaGetLastError());
}

}  // namespace

// ---- GetFitnessScore ---------------------------------------------------------------------------------------------------------
// The fit grid is the search grid over the fit cloud with cells of sqrt(max_range): every point within the gate lies in the 27 cells
// around a query.  Rebuilt when the cloud or max_range changed (one wait).
int Handle::fit_grid_for(float max_range, int* waits) {
    if (fit_grid_version == fit_cloud_version && fit_grid_range == max_range) return FLS_OK;
    fit_grid.res = std::sqrt(max_range) * 1.001f;
    const int rc = fit_grid.build(fit_pts, fit_cloud_n, scratch, stream, &launches);
    if (rc != FLS_OK) return rc;
    if (waits) ++*waits;
    fit_grid_version = fit_cloud_version;
    fit_grid_range = max_range;
    return FLS_OK;
}

// GetFitnessScore (icp_optimized.h:191-215 upstream) of the last Match's source cloud at P poses (row-major R | t records in fit_pose):
// enqueues {sum, count} of every pose into fit_out; the grid must be current
void Handle::fitness_enqueue(const float4* d_src, size_t n, int P, float max_range) {
    const size_t tiles = (n + kFitTile - 1) / kFitTile;
    fit_part_sum.reserve((size_t)P * tiles + 1);
    fit_part_cnt.reserve((size_t)P * tiles + 1);
    fit_out.reserve((size_t)P);
    fit_cnt.reserve((size_t)P);
    pose_score_launch(false, fit_grid.view(), d_src, (int)n, fit_pose.p, P, max_range, fit_part_sum.p, fit_part_cnt.p, stream);
    pose_score_reduce_kernel<<<grid_for((size_t)P, 64), 64, 0, stream>>>(fit_part_sum.p, fit_part_cnt.p, P, (int)tiles, 0, max_range, fit_out.p, fit_cnt.p,
                                                                         nullptr, nullptr, nullptr);
    launches += 2;
}

static void pose_rows(const double* T, double* o) {  // column-major Mat4d -> row-major R | t
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) o[r * 3 + c] = T[c * 4 + r];
        o[9 + r] = T[12 + r];
    }
}

static float fitness_of(double sum, unsigned cnt) { return cnt > 0 ? (float)(sum / (double)cnt) : FLT_MAX; }

int Handle::fitness(float max_range, float* score) {
    *score = FLT_MAX;  // FloatNaN / "no inliers" upstream
    // no cloud to search: LoamFull (loam_full_kdtree.h:206-208), NDT / iVox outside localization mode, or no map yet
    if (fit_cloud_n == 0 || last_src == nullptr || last_src_n == 0 || !(max_range > 0.f)) return FLS_OK;
    begin_call();
    const int rc = fit_grid_for(max_range, nullptr);
    if (rc != FLS_OK) return rc;
    double pose[12];
    pose_rows(T_final, pose);
    fit_pose.reserve(12);
    FLS_CUDA(cudaMemcpyAsync(fit_pose.p, pose, sizeof(pose), cudaMemcpyHostToDevice, stream));
    fitness_enqueue(last_src, last_src_n, 1, max_range);
    double sum = 0;
    unsigned cnt = 0;
    FLS_CUDA(cudaMemcpyAsync(&sum, fit_out.p, sizeof(sum), cudaMemcpyDeviceToHost, stream));
    FLS_CUDA(cudaMemcpyAsync(&cnt, fit_cnt.p, sizeof(cnt), cudaMemcpyDeviceToHost, stream));
    end_call(nullptr);
    *score = fitness_of(sum, cnt);
    return FLS_OK;
}

// ---- relocalization ------------------------------------------------------------------------------------------------------------
int reloc_grid(const fls_reloc_cfg& c, RelocGrid* g) {
    auto bad = [](double v) { return !(v > 0.0) || !std::isfinite(v); };
    if (!(c.xy_radius >= 0.0) || !std::isfinite(c.xy_radius) || !(c.yaw_range >= 0.0) || !std::isfinite(c.yaw_range)) return FLS_ERR_INVALID_ARG;
    if ((c.xy_radius > 0.0 && bad(c.xy_step)) || (c.yaw_range > 0.0 && bad(c.yaw_step))) return FLS_ERR_INVALID_ARG;
    if (bad(c.coarse_leaf) || bad(c.max_range) || std::isnan(c.accept_fitness) || c.n_refine < 1 || c.n_refine > kMaxBatch) return FLS_ERR_INVALID_ARG;
    const double kPi = 3.14159265358979323846;
    const double fi = c.xy_radius > 0.0 ? std::floor(c.xy_radius / c.xy_step + 1e-9) : 0.0;
    const double fk = c.yaw_range > 0.0 ? std::floor(std::fmin(c.yaw_range, kPi) / c.yaw_step + 1e-9) : 0.0;
    if (fi > 1024.0 || fk > (double)kRelocMaxHypotheses) return FLS_ERR_INVALID_ARG;
    g->I = (int)fi;
    g->K = (int)fk;
    g->k0 = -g->K;
    if (c.yaw_range >= kPi && g->K > 0 && 2.0 * g->K * c.yaw_step >= 2.0 * kPi - 1e-9) g->k0 = -g->K + 1;  // -K would repeat +K
    g->n_yaw = g->K - g->k0 + 1;
    const long long nx = 2LL * g->I + 1;
    const long long P = nx * nx * g->n_yaw;
    if (P > kRelocMaxHypotheses) return FLS_ERR_INVALID_ARG;
    g->P = P;
    return FLS_OK;
}

int Handle::relocalize(const float4* d_scan, size_t n, const fls_reloc_cfg& c, const RelocGrid& gr, double* T, fls_reloc_result* out, double* refined_T,
                       int32_t* refined_converged, float* refined_fitness, int64_t* refined_index, double* coarse_scores, size_t coarse_cap) {
    std::memset(out, 0, sizeof(*out));
    out->n_hypotheses = gr.P;
    out->best_hypothesis = -1;
    out->fitness = FLT_MAX;
    out->coarse_score = FLT_MAX;
    int L = 0, W = 0;  // launches and waits of the whole call
    auto account = [&] {
        out->gpu_launches = L + launches;
        out->host_waits = W;
    };
    // ---- coarse cloud and the fit grid ---------------------------------------------------------------------------------------------
    reloc_coarse.reserve(n + 1);
    const size_t m = voxel_grid_device(d_scan, n, c.coarse_leaf, reloc_coarse.p, scratch, stream, &launches, &W);
    if (m == 0) {  // an empty scan: nothing to score or refine, and a later fls_fitness scores the empty cloud
        last_src = d_scan;
        last_src_n = 0;
        account();
        return FLS_OK;
    }
    int rc = fit_grid_for(c.max_range, &W);
    if (rc != FLS_OK) return rc;
    // ---- the hypotheses, their coarse scores and the n_refine best -----------------------------------------------------------------
    const int P = (int)gr.P;
    const int nr = P < c.n_refine ? P : c.n_refine;
    RelocGridArgs ga;
    pose_rows(T, ga.R);
    for (int k = 0; k < 3; ++k) ga.t[k] = T[12 + k];
    ga.xy_step = gr.I ? c.xy_step : 0.0;  // an unused step may be anything
    ga.yaw_step = gr.K ? c.yaw_step : 0.0;
    ga.I = gr.I;
    ga.K = gr.K;
    ga.k0 = gr.k0;
    ga.n_yaw = gr.n_yaw;
    ga.P = P;
    const size_t tiles = (m + kCoarseTile - 1) / kCoarseTile;
    reloc_poses.reserve((size_t)P * 12);
    reloc_part_sum.reserve((size_t)P * tiles);
    reloc_part_cnt.reserve((size_t)P * tiles);
    reloc_score.reserve((size_t)P);
    reloc_key.reserve((size_t)P * 2);
    reloc_idx.reserve((size_t)P * 2);
    reloc_pick.reserve(sizeof(RelocPick) * kMaxBatch);
    reloc_poses_kernel<<<grid_for((size_t)P, 128), 128, 0, stream>>>(ga, reloc_poses.p);
    pose_score_launch(true, fit_grid.view(), reloc_coarse.p, (int)m, reloc_poses.p, P, c.max_range, reloc_part_sum.p, reloc_part_cnt.p, stream);
    pose_score_reduce_kernel<<<grid_for((size_t)P, 128), 128, 0, stream>>>(reloc_part_sum.p, reloc_part_cnt.p, P, (int)tiles, (int)m, c.max_range, nullptr,
                                                                           nullptr, reloc_score.p, reloc_key.p, reloc_idx.p);
    // stable LSD radix sort of (score bits, index): equal scores keep index order
    unsigned long long* keys_out = reloc_key.p + P;
    unsigned* idx_out = reloc_idx.p + P;
    cub_pass(scratch.cub_tmp, [&](void* tmp, size_t& bytes) {
        return cub::DeviceRadixSort::SortPairs(tmp, bytes, reloc_key.p, keys_out, reloc_idx.p, idx_out, P, 0, 64, stream);
    });
    RelocPick* d_pick = reinterpret_cast<RelocPick*>(reloc_pick.p);
    reloc_pick_kernel<<<1, kMaxBatch, 0, stream>>>(idx_out, reloc_score.p, reloc_poses.p, nr, d_pick);
    FLS_CUDA(cudaGetLastError());
    L += 5;
    RelocPick pick[kMaxBatch];
    FLS_CUDA(cudaMemcpyAsync(pick, d_pick, sizeof(RelocPick) * (size_t)nr, cudaMemcpyDeviceToHost, stream));
    const size_t n_cs = coarse_scores ? (coarse_cap < (size_t)P ? coarse_cap : (size_t)P) : 0;
    if (n_cs) FLS_CUDA(cudaMemcpyAsync(coarse_scores, reloc_score.p, sizeof(double) * n_cs, cudaMemcpyDeviceToHost, stream));
    FLS_CUDA(cudaStreamSynchronize(stream));
    ++W;
    // ---- refinement: the plug-in's batch Match of the picks, the same scan nr times ------------------------------------------------
    double Tr[kMaxBatch * 16];
    int conv[kMaxBatch];
    const void* scans[kMaxBatch];
    size_t ns[kMaxBatch];
    for (int r = 0; r < nr; ++r) {
        double* Ts = Tr + 16 * r;
        for (int i = 0; i < 3; ++i) {
            for (int j = 0; j < 3; ++j) Ts[j * 4 + i] = pick[r].pose[i * 3 + j];
            Ts[12 + i] = pick[r].pose[9 + i];
        }
        Ts[3] = Ts[7] = Ts[11] = 0.0;
        Ts[15] = 1.0;
        scans[r] = d_scan;
        ns[r] = n;
    }
    L += launches;
    rc = plugin->match_batch(nr, scans, ns, 0, Tr, conv, nullptr);  // begins its own call
    L += launches;
    W += waits;
    launches = 0;
    if (rc != FLS_OK) return rc;
    // ---- fitness of every refined pose on the cloud fls_fitness reads after that Match, in one launch -------------------------------
    double rows[kMaxBatch * 12];
    for (int r = 0; r < nr; ++r) pose_rows(Tr + 16 * r, rows + 12 * r);
    fit_pose.reserve((size_t)nr * 12);
    FLS_CUDA(cudaMemcpyAsync(fit_pose.p, rows, sizeof(double) * 12 * (size_t)nr, cudaMemcpyHostToDevice, stream));
    float fit[kMaxBatch];
    for (int r = 0; r < nr; ++r) fit[r] = FLT_MAX;
    if (last_src && last_src_n) {
        fitness_enqueue(last_src, last_src_n, nr, c.max_range);
        double sums[kMaxBatch];
        unsigned cnts[kMaxBatch];
        FLS_CUDA(cudaMemcpyAsync(sums, fit_out.p, sizeof(double) * (size_t)nr, cudaMemcpyDeviceToHost, stream));
        FLS_CUDA(cudaMemcpyAsync(cnts, fit_cnt.p, sizeof(unsigned) * (size_t)nr, cudaMemcpyDeviceToHost, stream));
        FLS_CUDA(cudaStreamSynchronize(stream));
        ++W;
        for (int r = 0; r < nr; ++r) fit[r] = fitness_of(sums[r], cnts[r]);
    }
    // ---- choice: the converged pose of lowest fitness (ties: rank), else the lowest fitness -----------------------------------------
    int best = -1;
    for (int pass = 0; pass < 2 && best < 0; ++pass)
        for (int r = 0; r < nr; ++r)
            if ((pass == 1 || conv[r]) && (best < 0 || fit[r] < fit[best])) best = r;
    std::memcpy(T, Tr + 16 * best, 16 * sizeof(double));
    std::memcpy(T_final, T, sizeof(T_final));  // a later fls_fitness scores the chosen pose on last_src
    out->n_refined = nr;
    out->best_rank = best;
    out->best_hypothesis = pick[best].index;
    out->converged = conv[best] ? 1 : 0;
    out->fitness = fit[best];
    out->coarse_score = (float)pick[best].score;
    out->accepted = (conv[best] && fit[best] < c.accept_fitness) ? 1 : 0;
    for (int r = 0; r < nr; ++r) {
        if (refined_T) std::memcpy(refined_T + 16 * r, Tr + 16 * r, 16 * sizeof(double));
        if (refined_converged) refined_converged[r] = conv[r];
        if (refined_fitness) refined_fitness[r] = fit[r];
        if (refined_index) refined_index[r] = pick[r].index;
    }
    account();
    return FLS_OK;
}

}  // namespace fls
