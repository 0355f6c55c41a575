// fls_reloc.cu — GetFitnessScore of many poses of one cloud, and relocalization from a coarse pose (fls_relocalize, and its exact
// branch and bound over a whole local map, fls_relocalize_wide).
//
// pose_score_kernel sweeps P poses over one cloud: a CTA stages a tile of the cloud in shared memory once and sweeps PPC poses over
// it; each pose's partial of that tile is reduced in a fixed tree and written to its own slot.  What a point adds is its term's:
// FitTerm makes it the one fitness path of the library (per pose the sum of the fp32 squared 1-NN distances <= max_range, in fp64,
// and how many there are; a second kernel adds the tiles of every pose in index order), BoundTerm the lower bound of the branch and
// bound.  No atomics: every result is reproducible bit for bit and independent of scheduling.  GetFitnessScore (Handle::fitness) is
// the one-pose-per-CTA form; relocalization scores hypotheses with 8 poses per CTA, keeps the best by a stable radix sort of the
// scores, refines them with the plug-in's batch Match and scores the refined poses with the same one-pose-per-CTA form that a later
// fls_fitness runs.
#include <cfloat>
#include <cmath>
#include <cstring>
#include <string>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

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

// A term of pose_score_kernel: pose(p) reads what slot p (< P) needs, add(pose, point, sum, cnt) adds one point's contribution;
// only a term with kCounts counts points, and only its kernel keeps counts in shared memory.
template <class Term>
struct SweepArgs {
    Term t;
    const float4* __restrict__ src;
    int n, P, n_tiles;
    double* __restrict__ part_sum;    // [P][n_tiles]
    unsigned* __restrict__ part_cnt;  // [P][n_tiles] when Term::kCounts
};

// grid (ceil(P / PPC), min(n_tiles, 65535)): CTA (x, y) sweeps poses x*PPC .. x*PPC+PPC-1 over tiles y, y + gridDim.y, ... of TILE
// points each, one partial per (pose, tile)
template <int PPC, int TILE, class Term>
__global__ void __launch_bounds__(kScoreBlock) pose_score_kernel(SweepArgs<Term> a) {
    constexpr int TPP = kScoreBlock / PPC;  // threads per pose
    __shared__ float4 s_pts[TILE];
    __shared__ double s_sum[kScoreBlock];
    __shared__ unsigned s_cnt[Term::kCounts ? kScoreBlock : 1];
    const int sub = threadIdx.x % TPP;
    const int pose = blockIdx.x * PPC + threadIdx.x / TPP;
    typename Term::Pose q;
    if (pose < a.P) q = a.t.pose(pose);
    for (int tile = blockIdx.y; tile < a.n_tiles; tile += gridDim.y) {  // uniform across the CTA
        const size_t base = (size_t)tile * TILE;
        const int m = (int)min((size_t)TILE, (size_t)a.n - base);
        for (int i = threadIdx.x; i < m; i += kScoreBlock) s_pts[i] = a.src[base + i];
        double sum = 0.0;
        unsigned cnt = 0;
        __syncthreads();
        if (pose < a.P) {
#pragma unroll 1
            for (int i = sub; i < m; i += TPP) a.t.add(q, s_pts[i], sum, cnt);
        }
        s_sum[threadIdx.x] = sum;
        if constexpr (Term::kCounts) s_cnt[threadIdx.x] = cnt;
        __syncthreads();  // also: every read of s_pts is done before the next tile overwrites it
#pragma unroll
        for (int o = TPP / 2; o > 0; o >>= 1) {  // fixed tree inside each pose's group of threads
            if (sub < o) {
                s_sum[threadIdx.x] += s_sum[threadIdx.x + o];
                if constexpr (Term::kCounts) s_cnt[threadIdx.x] += s_cnt[threadIdx.x + o];
            }
            __syncthreads();
        }
        if (sub == 0 && pose < a.P) {
            a.part_sum[(size_t)pose * a.n_tiles + tile] = s_sum[threadIdx.x];
            if constexpr (Term::kCounts) a.part_cnt[(size_t)pose * a.n_tiles + tile] = s_cnt[threadIdx.x];
        }
    }
}

// GetFitnessScore's term: the pose from a row-major R | t table; a point's fp32 squared 1-NN distance, added and counted when it is
// within max_range
struct FitTerm {
    static constexpr bool kCounts = true;
    GridView g;
    const double* __restrict__ poses;  // [P][12]: row-major R, then t (fp64; cast to float here, as TransformPointCloud does)
    float max_range;
    struct Pose {
        float r[12];
    };
    __device__ __forceinline__ Pose pose(int p) const {
        Pose q;
#pragma unroll
        for (int k = 0; k < 12; ++k) q.r[k] = (float)__ldg(poses + (size_t)p * 12 + k);
        return q;
    }
    __device__ __forceinline__ void add(const Pose& q, float4 sp, double& sum, unsigned& cnt) const {
        const float* r = q.r;
        const float qx = xform_row_f(r[0], r[1], r[2], r[9], sp.x, sp.y, sp.z);
        const float qy = xform_row_f(r[3], r[4], r[5], r[10], sp.x, sp.y, sp.z);
        const float qz = xform_row_f(r[6], r[7], r[8], r[11], sp.x, sp.y, sp.z);
        float d2;
        unsigned j, nc, nh;
        if (grid_nn1(g, qx, qy, qz, d2, j, nc, nh) && d2 <= max_range) {
            sum += (double)d2;
            cnt += 1;
        }
    }
};

// per pose: the tiles in order -> {sum, count} (sum_out), or the coarse score's sort key (the bits of a non-negative double order as
// the values do) and, when ids is given, the id of the pose's node (nodes null: base + p), which at level 0 is its leaf
__global__ void pose_score_reduce_kernel(const double* __restrict__ part_sum, const unsigned* __restrict__ part_cnt, int P, int n_tiles, int m,
                                         float max_range, double* __restrict__ sum_out, unsigned* __restrict__ cnt_out,
                                         unsigned long long* __restrict__ key, const long long* __restrict__ nodes, long long base,
                                         unsigned long long* __restrict__ ids) {
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
        return;
    }
    const double v = (s + (double)(m - (int)c) * (double)max_range) / (double)m;
    key[p] = (unsigned long long)__double_as_longlong(v);
    if (ids) ids[p] = (unsigned long long)(nodes ? nodes[p] : base + p);
}

// the hypothesis grids of fls_relocalize (fls_b200.h) around G guesses: leaf g * P + p is pose p of guess g's grid, in fp64, row-major
// R | t.  The guesses live in a device table, not in this struct: BoundTerm carries it by value into every sweep's kernel argument.
struct RelocGridArgs {
    const double* __restrict__ guess;  // [G][12]: row-major R, then t
    double xy_step, yaw_step;
    int I, K, k0;  // yaw offsets k0 .. K
    long long n_yaw, P;  // P: hypotheses per guess
};
// leaf `leaf` of the grids: the one formula of every search, so that a hypothesis has the same bits in each
__device__ __forceinline__ void reloc_leaf_pose(const RelocGridArgs& g, long long leaf, double* o) {
    const long long gi = leaf / g.P, p = leaf - gi * g.P;
    const double* R = g.guess + gi * 12;
    const double* t = R + 9;
    const long long nx = 2LL * g.I + 1;
    const long long ky = p % g.n_yaw, ix = (p / g.n_yaw) % nx, jy = p / (g.n_yaw * nx);
    const double psi = __dmul_rn((double)(g.k0 + ky), g.yaw_step);
    const double c = cos(psi), s = sin(psi);
    for (int j = 0; j < 3; ++j) {
        const double a = __ldg(R + j), b = __ldg(R + 3 + j);
        o[j] = __dsub_rn(__dmul_rn(c, a), __dmul_rn(s, b));
        o[3 + j] = __dadd_rn(__dmul_rn(s, a), __dmul_rn(c, b));
        o[6 + j] = __ldg(R + 6 + j);
    }
    o[9] = __dadd_rn(__ldg(t), __dmul_rn((double)(ix - g.I), g.xy_step));
    o[10] = __dadd_rn(__ldg(t + 1), __dmul_rn((double)(jy - g.I), g.xy_step));
    o[11] = __ldg(t + 2);
}
// the selected hypotheses: {index, coarse score, pose} records, read back in one copy
struct RelocPick {
    long long index;
    double score;
    double pose[12];
};
// the n best after the sort: {leaf index, score, pose}
__global__ void reloc_pick_kernel(const unsigned long long* __restrict__ key_sorted, const unsigned long long* __restrict__ leaf_sorted,
                                  RelocGridArgs g, int n, RelocPick* __restrict__ out) {
    const int r = threadIdx.x;
    if (r >= n) return;
    out[r].index = (long long)leaf_sorted[r];
    out[r].score = __longlong_as_double((long long)key_sorted[r]);
    reloc_leaf_pose(g, (long long)leaf_sorted[r], out[r].pose);
}

constexpr int kFitTile = kScoreBlock;  // GetFitnessScore: one pose per CTA, one point per thread
constexpr int kCoarseTile = 2048;      // relocalization: 8 poses per CTA over 2048 staged points (32 KB)
constexpr int kCoarsePoses = 8;

template <bool kCoarse, class Term>
void pose_score_launch(const Term& t, const float4* d_src, int n, int P, double* part_sum, unsigned* part_cnt, cudaStream_t st) {
    constexpr int tile = kCoarse ? kCoarseTile : kFitTile, ppc = kCoarse ? kCoarsePoses : 1;
    const SweepArgs<Term> a{t, d_src, n, P, (n + tile - 1) / tile, part_sum, part_cnt};
    const dim3 grid((unsigned)((P + ppc - 1) / ppc), (unsigned)(a.n_tiles < 65535 ? a.n_tiles : 65535));
    pose_score_kernel<ppc, tile, Term><<<grid, kScoreBlock, 0, st>>>(a);
    FLS_CUDA(cudaGetLastError());
}

}  // namespace

// ---- GetFitnessScore ---------------------------------------------------------------------------------------------------------
// The fit grid is the search grid over the fit cloud with cells of sqrt(max_range): every point within the gate lies in the 27 cells
// around a query.  Rebuilt when the cloud or max_range changed (one wait).
int Handle::fit_grid_for(float max_range) {
    if (fit_grid_version == fit_cloud_version && fit_grid_range == max_range) return FLS_OK;
    fit_grid.res = std::sqrt(max_range) * 1.001f;
    const int rc = fit_grid.build(fit_pts, fit_cloud_n, scratch, call);
    if (rc != FLS_OK) return rc;
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
    pose_score_launch<false>(FitTerm{fit_grid.view(), fit_pose.p, max_range}, d_src, (int)n, P, fit_part_sum.p, fit_part_cnt.p, call.stream);
    pose_score_reduce_kernel<<<grid_for((size_t)P, 64), 64, 0, call.stream>>>(fit_part_sum.p, fit_part_cnt.p, P, (int)tiles, 0, max_range, fit_out.p,
                                                                              fit_cnt.p, nullptr, nullptr, 0, nullptr);
    call.launches += 2;
}

static float fitness_of(double sum, unsigned cnt) { return cnt > 0 ? (float)(sum / (double)cnt) : FLT_MAX; }

int Handle::fitness(float max_range, float* score) {
    *score = FLT_MAX;  // FloatNaN / "no inliers" upstream
    // no cloud to search: LoamFull (loam_full_kdtree.h:206-208), NDT / iVox outside localization mode, or no map yet
    if (fit_cloud_n == 0 || last_src == nullptr || last_src_n == 0 || !(max_range > 0.f)) return FLS_OK;
    begin_call();
    const int rc = fit_grid_for(max_range);
    if (rc != FLS_OK) return rc;
    const GnPose pose = gn_pose(T_final);
    fit_pose.reserve(12);
    FLS_CUDA(cudaMemcpyAsync(fit_pose.p, &pose, sizeof(pose), cudaMemcpyHostToDevice, call.stream));
    fitness_enqueue(last_src, last_src_n, 1, max_range);
    double sum = 0;
    unsigned cnt = 0;
    FLS_CUDA(cudaMemcpyAsync(&sum, fit_out.p, sizeof(sum), cudaMemcpyDeviceToHost, call.stream));
    FLS_CUDA(cudaMemcpyAsync(&cnt, fit_cnt.p, sizeof(cnt), cudaMemcpyDeviceToHost, call.stream));
    call.end(nullptr);
    *score = fitness_of(sum, cnt);
    return FLS_OK;
}

// ---- relocalization ------------------------------------------------------------------------------------------------------------
int reloc_grid(const fls_reloc_cfg& c, RelocGrid* g, bool wide) {
    const double max_i = wide ? 32767.0 : 1024.0;
    const long long max_p = wide ? kRelocWideMaxHypotheses : kRelocMaxHypotheses;
    auto bad = [](double v) { return !(v > 0.0) || !std::isfinite(v); };
    if (!(c.xy_radius >= 0.0) || !std::isfinite(c.xy_radius) || !(c.yaw_range >= 0.0) || !std::isfinite(c.yaw_range)) return FLS_ERR_INVALID_ARG;
    if ((c.xy_radius > 0.0 && bad(c.xy_step)) || (c.yaw_range > 0.0 && bad(c.yaw_step))) return FLS_ERR_INVALID_ARG;
    if (bad(c.coarse_leaf) || bad(c.max_range) || std::isnan(c.accept_fitness) || c.n_refine < 1 || c.n_refine > kMaxBatch) return FLS_ERR_INVALID_ARG;
    const double kPi = 3.14159265358979323846;
    const double fi = c.xy_radius > 0.0 ? std::floor(c.xy_radius / c.xy_step + 1e-9) : 0.0;
    const double fk = c.yaw_range > 0.0 ? std::floor(std::fmin(c.yaw_range, kPi) / c.yaw_step + 1e-9) : 0.0;
    if (fi > max_i || fk > (double)(max_p / 2)) return FLS_ERR_INVALID_ARG;  // K > max_p / 2 gives more than max_p yaws
    g->I = (int)fi;
    g->K = (int)fk;
    g->k0 = -g->K;
    if (c.yaw_range >= kPi && g->K > 0 && 2.0 * g->K * c.yaw_step >= 2.0 * kPi - 1e-9) g->k0 = -g->K + 1;  // -K would repeat +K
    g->n_yaw = (long long)g->K - g->k0 + 1;
    const long long nx = 2LL * g->I + 1;
    if (nx * nx > max_p / g->n_yaw) return FLS_ERR_INVALID_ARG;  // P > max_p, without overflow
    const long long P = nx * nx * g->n_yaw;
    g->P = P;
    return FLS_OK;
}

// The tail of the search: the plug-in's batch Match of the nr picks, GetFitnessScore of every refined pose and Init's choice rule.
// out has its defaults.
static int reloc_refine(Handle& h, const float4* d_scan, size_t n, const fls_reloc_cfg& c, const RelocPick* pick, int nr, double* T,
                        fls_reloc_result* out, double* refined_T, int32_t* refined_converged, float* refined_fitness, int64_t* refined_index) {
    // ---- refinement: the plug-in's batch Match of the picks, the same scan nr times ------------------------------------------------
    double Tr[kMaxBatch * 16];
    int conv[kMaxBatch];
    const void* scans[kMaxBatch];
    size_t ns[kMaxBatch];
    for (int r = 0; r < nr; ++r) {
        gn_pose_T(pick[r].pose, pick[r].pose + 9, Tr + 16 * r);
        scans[r] = d_scan;
        ns[r] = n;
    }
    const Call before = h.call;  // the Match begins a call of its own: this call's counts go on after it
    const int rc = h.plugin->match_batch(nr, scans, ns, 0, Tr, conv, nullptr);
    h.call.launches += before.launches;
    h.call.waits += before.waits;
    h.call.h2d += before.h2d;
    h.call.d2h += before.d2h;
    if (rc != FLS_OK) return rc;
    // ---- fitness of every refined pose on the cloud fls_fitness reads after that Match, in one launch -------------------------------
    GnPose rows[kMaxBatch];
    for (int r = 0; r < nr; ++r) rows[r] = gn_pose(Tr + 16 * r);
    h.fit_pose.reserve((size_t)nr * 12);
    FLS_CUDA(cudaMemcpyAsync(h.fit_pose.p, rows, sizeof(GnPose) * (size_t)nr, cudaMemcpyHostToDevice, h.call.stream));
    float fit[kMaxBatch];
    for (int r = 0; r < nr; ++r) fit[r] = FLT_MAX;
    if (h.last_src && h.last_src_n) {
        h.fitness_enqueue(h.last_src, h.last_src_n, nr, c.max_range);
        double sums[kMaxBatch];
        unsigned cnts[kMaxBatch];
        FLS_CUDA(cudaMemcpyAsync(sums, h.fit_out.p, sizeof(double) * (size_t)nr, cudaMemcpyDeviceToHost, h.call.stream));
        FLS_CUDA(cudaMemcpyAsync(cnts, h.fit_cnt.p, sizeof(unsigned) * (size_t)nr, cudaMemcpyDeviceToHost, h.call.stream));
        h.call.sync();
        for (int r = 0; r < nr; ++r) fit[r] = fitness_of(sums[r], cnts[r]);
    }
    // ---- choice: the converged pose of lowest fitness (ties: rank), else the lowest fitness -----------------------------------------
    int best = -1;
    for (int pass = 0; pass < 2 && best < 0; ++pass)
        for (int r = 0; r < nr; ++r)
            if ((pass == 1 || conv[r]) && (best < 0 || fit[r] < fit[best])) best = r;
    std::memcpy(T, Tr + 16 * best, 16 * sizeof(double));
    std::memcpy(h.T_final, T, sizeof(h.T_final));  // a later fls_fitness scores the chosen pose on last_src
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
    out->gpu_launches = h.call.launches;
    out->host_waits = h.call.waits;
    return FLS_OK;
}

namespace {

// ---- fls_relocalize_wide: exact branch and bound over the hypothesis grid ------------------------------------------------------
// A node of level l is an aligned block of 2^l x 2^l x 2^l leaves (hypotheses) in (x, y, yaw) index space, clipped at the grid's
// edges; its id orders the blocks as the leaves are ordered (yaw fastest, then x, then y), so a level-0 node is a leaf.  A node is
// evaluated at one representative leaf: the one 2^(l-1) past its low corner in each index, or the last one where the block is clipped.
// With G guesses a node never spans two grids: node g * N_l + b is block b of guess g's grid, N_l the blocks of one grid at level l.
//
// The bound.  Let q_i be scan point p_i moved by the representative as the score kernel moves it (the fp64 pose cast to float,
// xform_row_f), and b_i a lower bound on the distance from q_i to the fit cloud (the lattice below).  A leaf of the node moves p_i to
// q'_i with |q'_i - q_i| <= delta_i = dt + dpsi * |(R_guess p_i)_xy| + eps_i, where dt = xy_step * sqrt(hx^2 + hy^2) bounds the
// translation offset (hx, hy, hk: the largest index offsets from the representative to a leaf of the node), and dpsi = hk * yaw_step
// bounds the turn: the leaves share z, roll and pitch, and |Rz(a) v - Rz(b) v| = 2 |sin((a - b) / 2)| |v_xy| <= |a - b| |v_xy|.
// eps_i covers the floats.  A transform row is ((r0 x + r1 y) + r2 z) + t in fp32 with r and t the fp64 pose rounded once: with
// u = 2^-24, |r| <= 1 and the rotation rows of the leaves rounded in fp64 (2^-53, far below u), each of the five roundings and the
// two casts is at most u (|p|_1 + |t|) to first order, so a coordinate is within 7u (|p|_1 + |t|_inf) of the exact value and the
// point within 7 sqrt(3) u (...) < 13u (...); for two poses 26u, taken as 32u (|p_i|_1 + tau) with tau the largest |t| coordinate of
// any leaf.  dist2_ref's three roundings on differences and three on products and sums give d2_f >= d^2 (1 - 6u) to first order,
// so sqrt(d2_f) >= d - 3u d; the term below only differs from max_range when d < sqrt(max_range) (1 + 4u), so 8u sqrt(max_range)
// covers it.  The lattice lookup and the bound itself run in fp64, whose roundings (2^-53 relative) the factor 32 absorbs.  So
// every leaf's fp32 squared 1-NN distance of p_i is at least max(0, b_i - delta_i)^2, and GetFitnessScore's gated sum of the leaf,
// sum_i min(d2_i, max_range) (an outlier or a point without a neighbour counts max_range), is at least
//   LB = sum_i min(max(0, b_i - delta_i)^2, max_range)        (in fp64).
// Both sums are fp64 sums of up to 2^30 non-negative terms in different orders: their rounding is below m 2^-53 < 1.2e-7 of the
// sum, so a node is pruned only when LB / m > U (1 + kPruneMargin).
// Over G guesses the bound takes w_i = max_g |(R_g p_i)_xy| and tau over every guess's leaves: both only make delta_i larger than
// the one guess g of the node needs, so LB stays a lower bound of every leaf of every grid (for G = 1 both are the values above).
//
// U is the n-th smallest exact score among the distinct leaves scored so far: the representatives of the start level (the lowest
// level with at most 2^20 nodes over all guesses) are all scored exactly, and no later level scores any (those reps would repeat leaves already
// scored or be scored again at level 0; the start level's U already comes from up to 2^20 leaves spread over the whole grid).  A
// node is kept iff LB / m <= U (1 + margin): every leaf scoring <= U keeps all its ancestors, so the n best leaves of the whole grid,
// and every tie at the n-th score, reach level 0, where all survivors are scored exactly and sorted on (score bits, leaf index).
constexpr long long kWideChunk = 1LL << 20;  // nodes of the start level, and of one launch at any level
constexpr long long kWideCap = 1LL << 23;    // survivors of one level; more is FLS_ERR_CAPACITY
constexpr double kPruneMargin = 1e-6;
constexpr double kU = 1.0 / 16777216.0;  // unit roundoff of fp32
constexpr size_t kLatticeCells = 1u << 25;
constexpr int kLatticeLine = 65535;  // cells per axis at most: the per-line stacks of the transform are 16-bit
constexpr unsigned kEdtInf = 0xffffffffu;

struct LatticeView {
    const unsigned short* v;
    int nx, ny, nz;
    double ox, oy, oz, h, inv_h, q;
};

// blocks per axis of n leaves at level l
__host__ __device__ inline long long level_blocks(long long n, int l) { return (n + (1LL << l) - 1) >> l; }

// representative index and largest offset to any index of block b at level l of an axis of n leaves
__device__ inline long long block_rep(long long b, int l, long long n, int& h) {
    const long long lo = b << l, hi = min(lo + (1LL << l), n) - 1;
    const long long r = l ? min(lo + (1LL << (l - 1)), hi) : lo;
    h = (int)max(r - lo, hi - r);
    return r;
}

// node id -> (guess, block of that guess's grid at level l in yaw, x, y)
struct NodeIdx {
    long long g, bk, bx, by;
};
__device__ inline NodeIdx node_idx(long long id, int l, long long nx, long long nk) {
    const long long nbk = level_blocks(nk, l), nbx = level_blocks(nx, l), b = id % (nbk * nbx * nbx);
    return {id / (nbk * nbx * nbx), b % nbk, (b / nbk) % nbx, b / (nbk * nbx)};
}

struct NodeRep {
    long long leaf;
    int hx, hy, hk;
};
__device__ inline NodeRep node_rep(long long id, int l, long long nx, long long nk) {
    const NodeIdx d = node_idx(id, l, nx, nk);
    NodeRep r;
    const long long rk = block_rep(d.bk, l, nk, r.hk), rx = block_rep(d.bx, l, nx, r.hx), ry = block_rep(d.by, l, nx, r.hy);
    r.leaf = (d.g * nx + ry) * nx * nk + rx * nk + rk;
    return r;
}

__global__ void reloc_iota_kernel(long long* __restrict__ out, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = i;
}

// poses of the representatives of N nodes of level l (nodes null: node i is base + i)
__global__ void reloc_rep_poses_kernel(RelocGridArgs g, const long long* __restrict__ nodes, long long base, int N, int l, double* __restrict__ poses) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    reloc_leaf_pose(g, node_rep(nodes ? nodes[i] : base + i, l, 2LL * g.I + 1, g.n_yaw).leaf, poses + (size_t)i * 12);
}

// pose_score_kernel's term of LB (derived at the head of this section): the pose of a node's representative, and per point
// min(max(0, b_i - delta_i)^2, max_range).  The points are the coarse cloud with w = max over the guesses of |(R_g p)_xy| rounded up
// (reloc_slack_points_kernel).
struct BoundTerm {
    static constexpr bool kCounts = false;
    LatticeView lat;
    RelocGridArgs g;
    const long long* __restrict__ nodes;
    int level;
    double eps0, eps1, max_range;  // eps_i = eps0 + eps1 |p_i|_1
    struct Pose {
        float r[12];
        double dt, dpsi, ex, ey, ez;  // delta_i's node terms, and the far corner of the lattice's box
    };
    __device__ __forceinline__ Pose pose(int i) const {
        const NodeRep nr = node_rep(nodes[i], level, 2LL * g.I + 1, g.n_yaw);
        double p[12];
        reloc_leaf_pose(g, nr.leaf, p);
        Pose q;
#pragma unroll
        for (int k = 0; k < 12; ++k) q.r[k] = (float)p[k];
        q.dt = g.xy_step * sqrt((double)nr.hx * nr.hx + (double)nr.hy * nr.hy);
        q.dpsi = (double)nr.hk * g.yaw_step;
        q.ex = lat.ox + lat.nx * lat.h, q.ey = lat.oy + lat.ny * lat.h, q.ez = lat.oz + lat.nz * lat.h;
        return q;
    }
    __device__ __forceinline__ void add(const Pose& q, float4 sp, double& sum, unsigned&) const {
        const float* r = q.r;
        const LatticeView& L = lat;
        const double qx = xform_row_f(r[0], r[1], r[2], r[9], sp.x, sp.y, sp.z);
        const double qy = xform_row_f(r[3], r[4], r[5], r[10], sp.x, sp.y, sp.z);
        const double qz = xform_row_f(r[6], r[7], r[8], r[11], sp.x, sp.y, sp.z);
        // b_i: the distance to the lattice's box, and the lattice value of the cell of q's projection onto the box (the
        // projection onto a convex set: |q - p|^2 >= |q - q*|^2 + |q* - p|^2 for every fit point p in the box)
        const double dx = fmax(0.0, fmax(L.ox - qx, qx - q.ex)), dy = fmax(0.0, fmax(L.oy - qy, qy - q.ey)), dz = fmax(0.0, fmax(L.oz - qz, qz - q.ez));
        const int cx = (int)fmin(fmax((qx - L.ox) * L.inv_h, 0.0), L.nx - 1.0);
        const int cy = (int)fmin(fmax((qy - L.oy) * L.inv_h, 0.0), L.ny - 1.0);
        const int cz = (int)fmin(fmax((qz - L.oz) * L.inv_h, 0.0), L.nz - 1.0);
        const double lv = (double)__ldg(L.v + ((size_t)cz * L.ny + cy) * L.nx + cx) * L.q;
        const double b = sqrt(dx * dx + dy * dy + dz * dz + lv * lv);
        const double delta = q.dt + q.dpsi * (double)sp.w + eps0 + eps1 * ((double)fabsf(sp.x) + (double)fabsf(sp.y) + (double)fabsf(sp.z));
        const double e = fmax(0.0, b - delta);
        sum += fmin(e * e, max_range);
    }
};

// per node: LB / m against U (the n-th smallest sorted score bits at *u_key) -> how many children it passes to level l - 1
__global__ void reloc_keep_kernel(const double* __restrict__ part, int N, int n_tiles, int m, const unsigned long long* __restrict__ u_key,
                                  const long long* __restrict__ nodes, int l, long long nx, long long nk, int* __restrict__ n_children) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    double lb = 0.0;
    for (int t = 0; t < n_tiles; ++t) lb += part[(size_t)i * n_tiles + t];
    const double U = __longlong_as_double((long long)*u_key);
    int k = 0;
    if (lb / (double)m <= U * (1.0 + kPruneMargin)) {
        const NodeIdx d = node_idx(nodes[i], l, nx, nk);
        const long long ck = level_blocks(nk, l - 1), cx = level_blocks(nx, l - 1);
        k = (int)((min(2 * d.bk + 2, ck) - 2 * d.bk) * (min(2 * d.bx + 2, cx) - 2 * d.bx) * (min(2 * d.by + 2, cx) - 2 * d.by));
    }
    n_children[i] = k;
}

// the children of the kept nodes of level l, at their offsets in the level l - 1 list (in the same guess)
__global__ void reloc_children_kernel(const long long* __restrict__ nodes, const int* __restrict__ n_children, const int* __restrict__ offset, int N,
                                      int l, long long nx, long long nk, long long* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N || n_children[i] == 0) return;
    const NodeIdx d = node_idx(nodes[i], l, nx, nk);
    const long long ck = level_blocks(nk, l - 1), cx = level_blocks(nx, l - 1);
    long long* o = out + offset[i];
    for (long long y = 2 * d.by; y < min(2 * d.by + 2, cx); ++y)
        for (long long x = 2 * d.bx; x < min(2 * d.bx + 2, cx); ++x)
            for (long long k = 2 * d.bk; k < min(2 * d.bk + 2, ck); ++k) *o++ = ((d.g * cx + y) * cx + x) * ck + k;
}

// ---- the lower-bound distance lattice -------------------------------------------------------------------------------------------
// Cells of pitch h over the fit cloud's bounding box.  An exact squared Euclidean distance transform between cell centres (in cells,
// three separable passes of Meijster's integer lower envelope, one thread per line) gives D(c) to the nearest occupied cell.  A point
// x of cell c and a fit point p of cell c' are at least the distance between the two cell boxes apart, h sqrt(sum_k max(0, |c_k -
// c'_k| - 1)^2) = h min over the 27 neighbours c + s (s in {-1, 0, 1}^3) of |c + s - c'|, and the neighbour that attains it lies
// between c and c', inside the box; so the cell stores h sqrt(min_s D(c + s)), rounded down to quanta of h / 64 in 16 bits.  Values
// saturate at 1024 h, which covers sqrt(max_range) (<= 4 h) plus a slack of about 1000 cells; a larger slack makes its term zero
// anyway.  h = sqrt(max_range) / 4, doubled until the box has at most 2^25 cells and at most 65535 along each axis.

// one block: the bounding box of the fit cloud, as {min x, y, z, max x, y, z}
__global__ void lattice_bbox_kernel(const float4* __restrict__ pts, size_t n, float* __restrict__ box) {
    __shared__ float s[6][256];
    float v[6] = {INFINITY, INFINITY, INFINITY, -INFINITY, -INFINITY, -INFINITY};
    for (size_t i = threadIdx.x; i < n; i += blockDim.x) {
        const float4 p = pts[i];
        v[0] = fminf(v[0], p.x), v[1] = fminf(v[1], p.y), v[2] = fminf(v[2], p.z);
        v[3] = fmaxf(v[3], p.x), v[4] = fmaxf(v[4], p.y), v[5] = fmaxf(v[5], p.z);
    }
    for (int k = 0; k < 6; ++k) s[k][threadIdx.x] = v[k];
    __syncthreads();
    for (int o = blockDim.x / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o)
            for (int k = 0; k < 6; ++k) s[k][threadIdx.x] = k < 3 ? fminf(s[k][threadIdx.x], s[k][threadIdx.x + o]) : fmaxf(s[k][threadIdx.x], s[k][threadIdx.x + o]);
        __syncthreads();
    }
    if (threadIdx.x < 6) box[threadIdx.x] = s[threadIdx.x][0];
}

__global__ void lattice_mark_kernel(const float4* __restrict__ pts, size_t n, LatticeView L, unsigned* __restrict__ d) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 p = pts[i];
    const int cx = (int)fmin(fmax(floor(((double)p.x - L.ox) * L.inv_h), 0.0), L.nx - 1.0);
    const int cy = (int)fmin(fmax(floor(((double)p.y - L.oy) * L.inv_h), 0.0), L.ny - 1.0);
    const int cz = (int)fmin(fmax(floor(((double)p.z - L.oz) * L.inv_h), 0.0), L.nz - 1.0);
    d[((size_t)cz * L.ny + cy) * L.nx + cx] = 0u;
}

// one pass of the separable transform along `axis`: out(u) = min_i (u - i)^2 + in(i) on every line, exact in integers (kEdtInf: no
// fit point yet; a finite value saturates below it, which keeps it a lower bound).  s and t: per-line stacks at the line's own cells.
__global__ void lattice_edt_kernel(const unsigned* __restrict__ in, unsigned* __restrict__ out, unsigned short* __restrict__ s,
                                   unsigned short* __restrict__ t, int nx, int ny, int nz, int axis) {
    const long long line = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    long long base, stride;
    int n;
    if (axis == 0) {
        if (line >= (long long)ny * nz) return;
        base = line * nx, stride = 1, n = nx;
    } else if (axis == 1) {
        if (line >= (long long)nx * nz) return;
        base = (line / nx) * nx * ny + line % nx, stride = nx, n = ny;
    } else {
        if (line >= (long long)nx * ny) return;
        base = line, stride = (long long)nx * ny, n = nz;
    }
    constexpr long long kInf = 1LL << 40;
    auto g = [&](long long i) -> long long {
        const unsigned v = in[base + i * stride];
        return v == kEdtInf ? kInf : (long long)v;
    };
    auto f = [&](long long x, long long i) { return (x - i) * (x - i) + g(i); };
    auto S = [&](long long k) -> unsigned short& { return s[base + k * stride]; };
    auto Tt = [&](long long k) -> unsigned short& { return t[base + k * stride]; };
    long long q = 0;
    S(0) = 0;
    Tt(0) = 0;
    for (long long u = 1; u < n; ++u) {
        while (q >= 0 && f(Tt(q), S(q)) > f(Tt(q), u)) --q;
        if (q < 0) {
            q = 0;
            S(0) = (unsigned short)u;
        } else {
            const long long i = S(q), num = u * u - i * i + g(u) - g(i), den = 2 * (u - i);
            const long long w = 1 + (num >= 0 ? num / den : -((-num + den - 1) / den));  // 1 + floor(num / den)
            if (w < n) {
                ++q;
                S(q) = (unsigned short)u;
                Tt(q) = (unsigned short)w;
            }
        }
    }
    for (long long u = n - 1; u >= 0; --u) {
        const long long d = f(u, S(q));
        out[base + u * stride] = d >= kInf ? kEdtInf : (unsigned)min(d, (long long)kEdtInf - 1);
        if (u == Tt(q)) --q;
    }
}

__global__ void lattice_store_kernel(const unsigned* __restrict__ d, int nx, int ny, int nz, double h, double q, unsigned short* __restrict__ v) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)nx * ny * nz) return;
    const int x = (int)(i % nx), y = (int)((i / nx) % ny), z = (int)(i / ((size_t)nx * ny));
    unsigned m = kEdtInf;
    for (int dz = max(z - 1, 0); dz <= min(z + 1, nz - 1); ++dz)
        for (int dy = max(y - 1, 0); dy <= min(y + 1, ny - 1); ++dy)
            for (int dx = max(x - 1, 0); dx <= min(x + 1, nx - 1); ++dx) m = min(m, d[((size_t)dz * ny + dy) * nx + dx]);
    // fp64 roundings of the square root and the products: taken off with a relative 2^-40 before rounding down
    const double b = sqrt((double)m) * h * (1.0 - 0x1p-40);
    v[i] = (unsigned short)fmin(floor(b / q), 65535.0);
}

// per scan point: its coordinates and max over the G guesses of |(R_g p)_xy| rounded up, the node-independent part of the slack
__global__ void reloc_slack_points_kernel(const float4* __restrict__ src, int n, const double* __restrict__ guess, int G, float4* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 p = src[i];
    double w = 0.0;
    for (int g = 0; g < G; ++g) {
        const double* R = guess + 12 * g;
        const double vx = R[0] * p.x + R[1] * p.y + R[2] * p.z, vy = R[3] * p.x + R[4] * p.y + R[5] * p.z;
        const double v = sqrt(vx * vx + vy * vy);
        w = g ? fmax(w, v) : v;
    }
    out[i] = make_float4(p.x, p.y, p.z, __double2float_ru(w));
}

}  // namespace

// Relocalization's state on a handle, made by its first call: the guess table, the coarse cloud and its copy with each point's slack
// term, a launch's poses and partials, sort keys and leaf ids (an unsorted and a sorted half each), the node lists of a level and the next with their
// child counts and offsets, U's sort key, the picks, the lower-bound lattice of the fit cloud, and the levels of the last wide search.
struct Reloc {
    DevBuf<float4> coarse, slack_pts;
    DevBuf<double> guess, poses, part_sum;
    DevBuf<unsigned> part_cnt;
    DevBuf<unsigned long long> key, leaf, u;
    DevBuf<long long> nodes, next;
    DevBuf<int> count;
    DevBuf<RelocPick> pick;
    LatticeView lat{};
    DevBuf<unsigned short> lat_v;
    unsigned long long lat_version = ~0ull;
    float lat_range = -1.f;
    std::vector<long long> levels;  // nodes evaluated per level of the last fls_relocalize_wide call, from its start level down to 0

    int lattice_for(Handle& hd, float max_range);
};

void RelocFree::operator()(Reloc* r) const { delete r; }

int Handle::relocalize_levels(int64_t* out, int capacity) const {
    const int n = reloc ? (int)reloc->levels.size() : 0;
    for (int i = 0; i < n && i < capacity; ++i) out[i] = reloc->levels[i];
    return n;
}

// The lattice of the current fit cloud and max_range, rebuilt like fit_grid (two waits when it is: the bounding box, and the end of
// the build before its scratch is freed).
int Reloc::lattice_for(Handle& hd, float max_range) {
    if (lat_version == hd.fit_cloud_version && lat_range == max_range) return FLS_OK;
    const cudaStream_t stream = hd.call.stream;
    DevBuf<float> box;
    box.reserve(6);
    lattice_bbox_kernel<<<1, 256, 0, stream>>>(hd.fit_pts, hd.fit_cloud_n, box.p);
    float b[6];
    FLS_CUDA(cudaMemcpyAsync(b, box.p, sizeof(b), cudaMemcpyDeviceToHost, stream));
    hd.call.sync();
    double h = std::sqrt((double)max_range) / 4.0;
    long long n[3];
    for (;; h *= 2.0) {
        for (int k = 0; k < 3; ++k) n[k] = (long long)std::floor(((double)b[3 + k] - (double)b[k]) / h) + 1;
        if (n[0] * n[1] * n[2] <= (long long)kLatticeCells && n[0] <= kLatticeLine && n[1] <= kLatticeLine && n[2] <= kLatticeLine) break;
    }
    const size_t cells = (size_t)(n[0] * n[1] * n[2]);
    DevBuf<unsigned> d0, d1;
    DevBuf<unsigned short> s, t;
    d0.reserve(cells), d1.reserve(cells), s.reserve(cells), t.reserve(cells);
    lat_v.reserve(cells);
    lat = {lat_v.p, (int)n[0], (int)n[1], (int)n[2], b[0], b[1], b[2], h, 1.0 / h, h / 64.0};
    FLS_CUDA(cudaMemsetAsync(d0.p, 0xff, cells * sizeof(unsigned), stream));
    lattice_mark_kernel<<<grid_for(hd.fit_cloud_n, 256), 256, 0, stream>>>(hd.fit_pts, hd.fit_cloud_n, lat, d0.p);
    const long long lines[3] = {n[1] * n[2], n[0] * n[2], n[0] * n[1]};
    lattice_edt_kernel<<<grid_for((size_t)lines[0], 128), 128, 0, stream>>>(d0.p, d1.p, s.p, t.p, lat.nx, lat.ny, lat.nz, 0);
    lattice_edt_kernel<<<grid_for((size_t)lines[1], 128), 128, 0, stream>>>(d1.p, d0.p, s.p, t.p, lat.nx, lat.ny, lat.nz, 1);
    lattice_edt_kernel<<<grid_for((size_t)lines[2], 128), 128, 0, stream>>>(d0.p, d1.p, s.p, t.p, lat.nx, lat.ny, lat.nz, 2);
    lattice_store_kernel<<<grid_for(cells, 256), 256, 0, stream>>>(d1.p, lat.nx, lat.ny, lat.nz, h, lat.q, lat_v.p);
    FLS_CUDA(cudaGetLastError());
    hd.call.sync();  // the scratch above is freed on return
    hd.call.launches += 6;
    lat_version = hd.fit_cloud_version;
    lat_range = max_range;
    return FLS_OK;
}

int Handle::relocalize(const float4* d_scan, size_t n, const fls_reloc_cfg& c, const RelocGrid& gr, bool wide, const double* guesses, int G, double* T,
                       fls_reloc_result* out, double* refined_T, int32_t* refined_converged, float* refined_fitness, int64_t* refined_index,
                       double* coarse_scores, size_t coarse_cap, int64_t* evaluations) {
    if (!reloc) reloc.reset(new Reloc);
    Reloc& s = *reloc;
    const cudaStream_t stream = call.stream;
    long long evals = 0;
    if (evaluations) *evaluations = 0;
    if (wide) s.levels.clear();
    std::memset(out, 0, sizeof(*out));
    const long long P = (long long)G * gr.P, nx = 2LL * gr.I + 1, nk = gr.n_yaw;  // every grid's hypotheses; one grid's axes
    out->n_hypotheses = P;
    out->best_hypothesis = -1;
    out->fitness = FLT_MAX;
    out->coarse_score = FLT_MAX;
    // ---- coarse cloud and the fit grid; an empty coarse cloud ends the call: nothing to score or refine, and a later fls_fitness
    // scores the empty cloud --------------------------------------------------------------------------------------------------------
    s.coarse.reserve(n + 1);
    const size_t m = voxel_grid_device(d_scan, n, c.coarse_leaf, s.coarse.p, scratch, call);
    if (m == 0) {
        if (T != guesses) std::memcpy(T, guesses, 16 * sizeof(double));
        last_src = d_scan;
        last_src_n = 0;
        out->gpu_launches = call.launches;
        out->host_waits = call.waits;
        return FLS_OK;
    }
    int rc = fit_grid_for(c.max_range);
    if (rc != FLS_OK) return rc;
    GnPose rows[kMaxBatch];
    for (int g = 0; g < G; ++g) rows[g] = gn_pose(guesses + 16 * g);
    s.guess.reserve((size_t)G * 12);
    FLS_CUDA(cudaMemcpyAsync(s.guess.p, rows, sizeof(GnPose) * (size_t)G, cudaMemcpyHostToDevice, stream));
    RelocGridArgs ga;
    ga.guess = s.guess.p;
    ga.xy_step = gr.I ? c.xy_step : 0.0;  // an unused step may be anything
    ga.yaw_step = gr.K ? c.yaw_step : 0.0;
    ga.I = gr.I;
    ga.K = gr.K;
    ga.k0 = gr.k0;
    ga.n_yaw = gr.n_yaw;
    ga.P = gr.P;
    // ---- the start level: the lowest with at most 2^20 nodes over all guesses (level 0 on every grid fls_relocalize accepts) -------
    const int nr = P < c.n_refine ? (int)P : c.n_refine;
    auto level_nodes = [&](int l) { return G * level_blocks(nx, l) * level_blocks(nx, l) * level_blocks(nk, l); };
    int ls = 0;
    while (level_nodes(ls) > kWideChunk) ++ls;
    long long N = level_nodes(ls);
    const size_t tiles = (m + kCoarseTile - 1) / kCoarseTile;
    auto reserve_chunk = [&](size_t k) {  // a launch's poses and partials
        s.poses.reserve(k * 12);
        s.part_sum.reserve(k * tiles);
        s.part_cnt.reserve(k * tiles);
    };
    s.pick.reserve(kMaxBatch);
    // exact scores of the representatives of N_ nodes of level l (nodes null: node i is i) -> their sort keys, and their node ids
    // when ids is given
    auto exact = [&](const long long* nodes, long long N_, int l, unsigned long long* keys, unsigned long long* ids) {
        for (long long o = 0; o < N_; o += kWideChunk) {
            const int k = (int)(N_ - o < kWideChunk ? N_ - o : kWideChunk);
            const long long* chunk = nodes ? nodes + o : nullptr;
            reserve_chunk((size_t)k);
            reloc_rep_poses_kernel<<<grid_for((size_t)k, 128), 128, 0, stream>>>(ga, chunk, o, k, l, s.poses.p);
            pose_score_launch<true>(FitTerm{fit_grid.view(), s.poses.p, c.max_range}, s.coarse.p, (int)m, k, s.part_sum.p, s.part_cnt.p, stream);
            pose_score_reduce_kernel<<<grid_for((size_t)k, 128), 128, 0, stream>>>(s.part_sum.p, s.part_cnt.p, k, (int)tiles, (int)m, c.max_range, nullptr,
                                                                                   nullptr, keys + o, chunk, o, ids ? ids + o : nullptr);
            call.launches += 3;
        }
        evals += N_;
    };
    // ---- the descent from the start level to level 1 (fls_relocalize_wide past 2^20 hypotheses) ------------------------------------
    if (ls > 0) {
        rc = s.lattice_for(*this, c.max_range);
        if (rc != FLS_OK) return rc;
        s.nodes.reserve((size_t)N);
        reloc_iota_kernel<<<grid_for((size_t)N, 256), 256, 0, stream>>>(s.nodes.p, N);
        ++call.launches;
        // U: the nr-th smallest score of the start level's representatives
        s.key.reserve((size_t)N * 2);
        exact(s.nodes.p, N, ls, s.key.p, nullptr);
        cub_pass(scratch.cub_tmp, [&](void* tmp, size_t& bytes) {
            return cub::DeviceRadixSort::SortKeys(tmp, bytes, s.key.p, s.key.p + N, (int)N, 0, 64, stream);
        });
        ++call.launches;
        s.u.reserve(1);
        FLS_CUDA(cudaMemcpyAsync(s.u.p, s.key.p + N + nr - 1, sizeof(unsigned long long), cudaMemcpyDeviceToDevice, stream));
        // the slack's float terms (derivation above): tau, the largest translation coordinate of any leaf of any guess
        double tau = 0.0;
        for (int g = 0; g < G; ++g) {
            const double* t = rows[g].t;
            const double tg = std::fmax(std::fmax(std::fabs(t[0]), std::fabs(t[1])) + gr.I * ga.xy_step, std::fabs(t[2]));
            tau = g ? std::fmax(tau, tg) : tg;
        }
        s.slack_pts.reserve(m);
        reloc_slack_points_kernel<<<grid_for(m, 256), 256, 0, stream>>>(s.coarse.p, (int)m, s.guess.p, G, s.slack_pts.p);
        ++call.launches;
        BoundTerm bound{s.lat, ga, nullptr, 0, 32.0 * kU * tau + 8.0 * kU * std::sqrt((double)c.max_range), 32.0 * kU, c.max_range};
        for (int l = ls; l >= 1; --l) {
            s.count.reserve((size_t)N * 2);
            int* cnt = s.count.p;
            int* off = s.count.p + N;
            for (long long o = 0; o < N; o += kWideChunk) {
                const int k = (int)(N - o < kWideChunk ? N - o : kWideChunk);
                reserve_chunk((size_t)k);
                bound.nodes = s.nodes.p + o;
                bound.level = l;
                pose_score_launch<true>(bound, s.slack_pts.p, (int)m, k, s.part_sum.p, nullptr, stream);
                reloc_keep_kernel<<<grid_for((size_t)k, 128), 128, 0, stream>>>(s.part_sum.p, k, (int)tiles, (int)m, s.u.p, s.nodes.p + o, l, nx, nk, cnt + o);
                call.launches += 2;
            }
            evals += N;
            s.levels.push_back(N);
            cub_pass(scratch.cub_tmp, [&](void* tmp, size_t& bytes) { return cub::DeviceScan::ExclusiveSum(tmp, bytes, cnt, off, (int)N, stream); });
            int last[2];
            FLS_CUDA(cudaMemcpyAsync(last, cnt + N - 1, sizeof(int), cudaMemcpyDeviceToHost, stream));
            FLS_CUDA(cudaMemcpyAsync(last + 1, off + N - 1, sizeof(int), cudaMemcpyDeviceToHost, stream));
            call.sync();
            ++call.launches;
            const long long next = (long long)last[0] + last[1];
            if (next > kWideCap) {
                set_last_error(std::string(G > 1 ? "fls_relocalize_multi: " : "fls_relocalize_wide: ") + std::to_string(next) +
                               " nodes survive at level " + std::to_string(l - 1));
                out->gpu_launches = call.launches;
                out->host_waits = call.waits;
                return FLS_ERR_CAPACITY;
            }
            s.next.reserve((size_t)next);
            reloc_children_kernel<<<grid_for((size_t)N, 128), 128, 0, stream>>>(s.nodes.p, cnt, off, (int)N, l, nx, nk, s.next.p);
            ++call.launches;
            std::swap(s.nodes.p, s.next.p);
            std::swap(s.nodes.cap, s.next.cap);
            N = next;
        }
    }
    // ---- level 0: every leaf left scored exactly, a stable sort on (score bits, leaf index g * P + p), the n best ---------------------
    // A descent's survivors are scored into the upper halves and first sorted into leaf order; a grid scored whole is in leaf order.
    s.key.reserve((size_t)N * 2);
    s.leaf.reserve((size_t)N * 2);
    unsigned long long *key = s.key.p, *leaf = s.leaf.p, *key2 = key + N, *leaf2 = leaf + N;
    exact(ls ? s.nodes.p : nullptr, N, 0, ls ? key2 : key, ls ? leaf2 : leaf);
    if (wide) s.levels.push_back(N);
    int bits = 1;
    while ((1LL << bits) < P) ++bits;
    auto by_leaf = [&](void* tmp, size_t& bytes) { return cub::DeviceRadixSort::SortPairs(tmp, bytes, leaf2, leaf, key2, key, (int)N, 0, bits, stream); };
    auto by_key = [&](void* tmp, size_t& bytes) { return cub::DeviceRadixSort::SortPairs(tmp, bytes, key, key2, leaf, leaf2, (int)N, 0, 64, stream); };
    if (ls > 0) {
        cub_reserve(scratch.cub_tmp, by_leaf, by_key);
        cub_run(scratch.cub_tmp, by_leaf);
        ++call.launches;
    } else {
        cub_reserve(scratch.cub_tmp, by_key);
    }
    cub_run(scratch.cub_tmp, by_key);
    reloc_pick_kernel<<<1, kMaxBatch, 0, stream>>>(key2, leaf2, ga, nr, s.pick.p);
    FLS_CUDA(cudaGetLastError());
    call.launches += 2;
    RelocPick pick[kMaxBatch];
    FLS_CUDA(cudaMemcpyAsync(pick, s.pick.p, sizeof(RelocPick) * (size_t)nr, cudaMemcpyDeviceToHost, stream));
    // fls_relocalize's coarse scores: the unsorted keys hold their bits
    const size_t n_cs = coarse_scores ? (coarse_cap < (size_t)P ? coarse_cap : (size_t)P) : 0;
    if (n_cs) FLS_CUDA(cudaMemcpyAsync(coarse_scores, key, sizeof(double) * n_cs, cudaMemcpyDeviceToHost, stream));
    call.sync();
    if (evaluations) *evaluations = evals;
    return reloc_refine(*this, d_scan, n, c, pick, nr, T, out, refined_T, refined_converged, refined_fitness, refined_index);
}

}  // namespace fls
