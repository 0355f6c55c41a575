// fls_p2plane.cu — K1 (+ fused K6), generation 8: the whole LoamPointToPlaneIVOX Gauss-Newton loop as ONE persistent kernel with a
// CTA barrier per visit.  It serves the single Match (fls_match / fls_match_device); batches run on generation 9
// (fls_p2plane_v9.cu), which shares the per-point arithmetic (fls_knn.cuh, fls_plane.cuh).  This file also holds the per-batch query
// preparation (one kernel: state init + tile-local locality sort), the Match-internal insertion rule of mapping mode and the k-NN test entry.
//
// Per source point and iteration it fuses what LoamPointToPlaneIVOX::PlanerMatch / ::SumCoefficient do
// (include/registration/loam_point_to_plane_ivox.h:256-340 upstream): transform with the current pose, bounded
// 5-NN in the iVox map, least-squares plane through the 5 neighbours (normal equations, column-pivoted Householder QR as the
// fallback, fp64), validity / near-point gates, J (6) and |d|, and the 21+6+2 Gauss-Newton sums; the scan's folding CTA reduces
// the CTA rows in a fixed order, solves the 6x6 system, updates the pose and applies the stop rule (:167-203), then publishes the
// next pose.  No host round trip inside a Match.
//
// Mapping onto the GPU
//   * grid = the CTAs the scan's chunks need (one 24-warp CTA per SM, 768 threads, 80 registers) + the folding CTA, launched
//     cooperatively only to guarantee co-residency; the scheduling unit is the WARP: warp w of CTA c works on 32-point chunk
//     (c, w) of every scan of the visit group, a static round-robin (consecutive chunks stay in one CTA: Morton neighbours share
//     candidate runs in L1);
//   * a visit = one Gauss-Newton iteration of up to 8 scans: poses in (LL records), chunks, one __syncthreads, CTA rows out (LL
//     records, no fence, no atomic); only the scan's folding CTA waits for the other rows — 24 warps x 8 loads in flight sweep
//     them until every tag matches, sums in a fixed order (bitwise reproducible for a given grid), gn_step, next pose out;
//   * queries are processed in Morton order of their voxel (sorted once per Match), so the lanes of a warp share
//     centre voxels: the table probe and the candidate stream are the same addresses -> L1 broadcast, no divergence;
//   * k-NN = 1 probe of the centre table + a streaming scan of that centre's contiguous stencil list (fls_ivox.cuh),
//     top-6 kept as quantised 32-bit keys with integer min/max, exact comparator for ambiguous queries (fls_knn.cuh);
//   * the 29 sums are accumulated warp-transposed: each lane stages {J, |d|, flags} in shared memory and lane k then
//     owns sum k (32 FMAs on broadcast LDS) — one register pair of accumulator state instead of 62, no shuffles;
//   * state that survives across iterations [quirk 1, SURVEY.md §7]: upstream resets the valid flags once per Match
//     and sums every flagged point, so a point valid earlier but rejected now keeps contributing its stale H_i, g_i:
//     a 32-byte record {J[6], |d|} per valid point (two float4 arrays) + a flag byte, re-read only on the stale path.
#include <cooperative_groups.h>

#include <cub/cub.cuh>

#include "fls_gn.cuh"
#include "fls_ivox.cuh"
#include "fls_kernels.h"
#include "fls_knn.cuh"
#include "fls_plane.cuh"

namespace fls {
namespace {

// IVoxMap::GetClosestPoint through the stencil lists: one probe of the centre table, then a streaming scan of the
// contiguous candidate run (already in the reference's visit order).  Indices refer to `lists`.
__device__ __forceinline__ void knn5_stream(const IvoxView& m, float qx, float qy, float qz, Top5& nn, unsigned& n_cand) {
    nn.init();
    n_cand = 0;
    const unsigned long long key = pack_key(ivox_coord(qx, m.inv_res), ivox_coord(qy, m.inv_res), ivox_coord(qz, m.inv_res));
    unsigned start, count;
    if (!table_find(m.ctab, m.cmask, key, start, count)) return;
    n_cand = count;
    const float4* __restrict__ L = m.lists + start;
    const float r2 = m.max_range2;
    // A run is ~4 cache lines and the scan below touches them one after the other; when a line is not on chip yet (first
    // touch of a voxel in this Match) that would be one exposed HBM round trip per line.  Requesting the rest of the run
    // up front overlaps them (lanes that share a run issue the same addresses: one request).
    {
        const char* pl = reinterpret_cast<const char*>(L);
        const unsigned bytes = count * 16u;
        for (unsigned off = 128u; off < bytes; off += 128u) asm volatile("prefetch.global.L2 [%0];" ::"l"(pl + off));
    }
    if (count > 64u) {  // position does not fit the 6-bit field
        knn5_exact(L, start, count, r2, qx, qy, qz, nn);
        return;
    }
    Top6q t;
    t.init();
    unsigned j = 0;
    bool amb;
    if (m.fast_knn) {
        // every candidate of the stencil is provably inside max_range (host check, fls_api.cu), so the range test is
        // dropped, and the distance may be contracted to FMAs: it then differs from the reference rounding by <= 2 ulp,
        // which can only reorder keys whose 26-bit prefixes are equal or adjacent — those queries take the exact path
#pragma unroll 1
        for (; j + 4 <= count; j += 4) {
            const float4 p0 = __ldg(L + j), p1 = __ldg(L + j + 1), p2 = __ldg(L + j + 2), p3 = __ldg(L + j + 3);
            t.push((__float_as_uint(dist2_fast(p0.x, p0.y, p0.z, qx, qy, qz)) & 0xffffffc0u) | j);
            t.push((__float_as_uint(dist2_fast(p1.x, p1.y, p1.z, qx, qy, qz)) & 0xffffffc0u) | (j + 1));
            t.push((__float_as_uint(dist2_fast(p2.x, p2.y, p2.z, qx, qy, qz)) & 0xffffffc0u) | (j + 2));
            t.push((__float_as_uint(dist2_fast(p3.x, p3.y, p3.z, qx, qy, qz)) & 0xffffffc0u) | (j + 3));
        }
#pragma unroll 1
        for (; j < count; ++j) {
            const float4 p = __ldg(L + j);
            t.push((__float_as_uint(dist2_fast(p.x, p.y, p.z, qx, qy, qz)) & 0xffffffc0u) | j);
        }
        amb = ((t.k1 >> 6) - (t.k0 >> 6) <= 1u && t.k1 != 0xffffffffu) || ((t.k5 >> 6) - (t.k4 >> 6) <= 1u && t.k5 != 0xffffffffu);
    } else {
#pragma unroll 1
        for (; j + 4 <= count; j += 4) {
            const float4 p0 = __ldg(L + j), p1 = __ldg(L + j + 1), p2 = __ldg(L + j + 2), p3 = __ldg(L + j + 3);
            const float e0 = dist2_ref(p0.x, p0.y, p0.z, qx, qy, qz);
            const float e1 = dist2_ref(p1.x, p1.y, p1.z, qx, qy, qz);
            const float e2 = dist2_ref(p2.x, p2.y, p2.z, qx, qy, qz);
            const float e3 = dist2_ref(p3.x, p3.y, p3.z, qx, qy, qz);
            t.push(qkey(e0, r2, j));
            t.push(qkey(e1, r2, j + 1));
            t.push(qkey(e2, r2, j + 2));
            t.push(qkey(e3, r2, j + 3));
        }
#pragma unroll 1
        for (; j < count; ++j) {
            const float4 p = __ldg(L + j);
            t.push(qkey(dist2_ref(p.x, p.y, p.z, qx, qy, qz), r2, j));
        }
        amb = ((t.k0 >> 6) == (t.k1 >> 6) && t.k1 != 0xffffffffu) || ((t.k4 >> 6) == (t.k5 >> 6) && t.k5 != 0xffffffffu);
    }
    if (amb) {
        knn5_exact(L, start, count, r2, qx, qy, qz, nn);
        return;
    }
    // fewer than 5 in range leaves the tail at the sentinel ("not full")
    nn.k0 = (t.k0 != 0xffffffffu) ? start + (t.k0 & 63u) : 0xffffffffu;
    nn.k1 = (t.k1 != 0xffffffffu) ? start + (t.k1 & 63u) : 0xffffffffu;
    nn.k2 = (t.k2 != 0xffffffffu) ? start + (t.k2 & 63u) : 0xffffffffu;
    nn.k3 = (t.k3 != 0xffffffffu) ? start + (t.k3 & 63u) : 0xffffffffu;
    nn.k4 = (t.k4 != 0xffffffffu) ? start + (t.k4 & 63u) : 0xffffffffu;
}

// Geometry of one source point against the map: returns true when the point produces a valid residual.
__device__ __forceinline__ bool p2plane_point(const IvoxView& map, const float4 sp, const double* __restrict__ pose /*R[9], t[3]*/,
                                              double plane_thres, double (&J)[6], double& ad, unsigned& n_cand, unsigned& n_fallback) {
    const float qx = xform_row_d(pose[0], pose[1], pose[2], pose[9], (double)sp.x, (double)sp.y, (double)sp.z);
    const float qy = xform_row_d(pose[3], pose[4], pose[5], pose[10], (double)sp.x, (double)sp.y, (double)sp.z);
    const float qz = xform_row_d(pose[6], pose[7], pose[8], pose[11], (double)sp.x, (double)sp.y, (double)sp.z);
    Top5 nn;
    knn5_stream(map, qx, qy, qz, nn, n_cand);
    n_fallback = 0;
    if (!nn.full()) return false;  // fewer than 5 neighbours (:271-273)
    const unsigned js[5] = {nn.idx(nn.k0), nn.idx(nn.k1), nn.idx(nn.k2), nn.idx(nn.k3), nn.idx(nn.k4)};
    return plane_term(map.lists, js, sp, qx, qy, qz, pose, plane_thres, J, ad, n_fallback);
}

// columns of the per-point staging record
constexpr int kRecAd = 6, kRecValid = 7, kRecCand = 8, kRecHits = 9, kRecOne = 10, kRecW = 12;

constexpr int kVisitGroup = 8;  // most scans whose chunks a warp works through between two CTA barriers

template <int BLOCK, int MINB>
__global__ void __launch_bounds__(BLOCK, MINB) p2plane_gn_kernel(P2PlaneLoopArgs a) {
    constexpr int W = BLOCK / 32;
    constexpr int V = kVisitGroup < W ? kVisitGroup : W;
    extern __shared__ __align__(16) unsigned char s_dyn[];
    double (*s_rec)[32][kRecW] = reinterpret_cast<double (*)[32][kRecW]>(s_dyn);  // [W][32][kRecW] per-lane staging records
    double (*s_part)[W][32] = reinterpret_cast<double (*)[W][32]>(s_dyn + sizeof(double) * W * 32 * kRecW);  // [V][W][32] per scan of the group: every warp's 32 sums
    __shared__ double s_pose[V][12];
    __shared__ double s_red[W][32];      // fold scratch of the folding CTA
    __shared__ int s_stop[V];
    __shared__ unsigned char s_iter[kMaxBatch];  // iterations this CTA has completed of every scan (255 = scan finished)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int G = (int)gridDim.x, cta = (int)blockIdx.x;
    const int n_warps = G * W;

    // which product of record columns lane k accumulates: sum_k = sgn * sum_p rec[p][ca] * rec[p][cb]
    int ca = kRecOne, cb = kRecOne;
    double sgn = 1.0;
    if (lane < 21) {
        int r = 0, k = lane;
        while (k >= 6 - r) { k -= 6 - r; ++r; }
        ca = r;
        cb = r + k;
    } else if (lane < 27) {
        ca = lane - 21; cb = kRecAd; sgn = -1.0;  // g = sum -J |d|
    } else if (lane == kAccValid) {
        ca = kRecValid;
    } else if (lane == kAccRes) {
        ca = kRecAd;
    } else if (lane == kAccCand) {
        ca = kRecCand;
    } else if (lane == kAccHits) {
        ca = kRecHits;
    } else {
        sgn = 0.0;
    }
    if (threadIdx.x < kMaxBatch) s_iter[threadIdx.x] = 0;
    __syncthreads();

    // One launch serves a batch of independent scans and EVERY CTA works on EVERY scan: the grid sweeps the scans round-
    // robin, one Gauss-Newton iteration of each scan per visit, up to V scans per visit.  Inside a visit a warp works
    // through its chunk of every scan of the group back to back — the CTA barrier that ends the visit then waits for the
    // slowest SUM of V chunks instead of V times for the slowest chunk.  A visit ends with this CTA's rows of partial sums
    // going out as LL records; only a scan's folding CTA waits for the other rows, solves and publishes the next pose —
    // everybody else moves straight on, and by the time the sweep returns to a scan its pose has long been published.  The
    // hand-over latency of one scan is hidden behind the work on the others; finished scans drop out of the sweep, so the
    // remaining ones come round faster (no static partition of the SMs, no idle CTAs).
    // With a single scan the sweep degenerates to: work, publish, wait for the pose.
    int n_left = a.n_scans;
    int next = 0;  // where the sweep continues
    while (n_left > 0) {
        // ---- the group: the next (up to V) unfinished scans in round-robin order (uniform: s_iter is shared) -------------
        int gs[V], git[V], nv = 0;
        for (int k = 0; k < a.n_scans && nv < V; ++k) {
            const int s = (next + k) % a.n_scans;
            const int it = s_iter[s];
            if (it == 255) continue;
            gs[nv] = s;
            git[nv] = it;
            ++nv;
        }
        next = (gs[nv - 1] + 1) % a.n_scans;
        // ---- poses of this visit: the prep kernel's state for iteration 0, afterwards the LL record published by the
        // scan's folder at the end of iteration it-1 (12 values + the stop word); 16 threads per scan of the group
        {
            const int v = threadIdx.x >> 4, k = threadIdx.x & 15;
            if (v < nv && k < 13) {
                const P2PlaneScan* __restrict__ sc = a.scans + gs[v];
                if (git[v] == 0) {
                    if (k < 9) s_pose[v][k] = __ldcg(&sc->state->R[k]);
                    else if (k < 12) s_pose[v][k] = __ldcg(&sc->state->t[k - 9]);
                    else s_stop[v] = 0;
                } else {
                    const unsigned ptag = sc->tag_base | (unsigned)git[v];
                    const uint4* ll = sc->ll_pose;
                    double val;
                    while (!ll_load(ll + k, ptag, val)) __nanosleep(100);
                    if (k < 12) s_pose[v][k] = val;
                    else s_stop[v] = val != 0.0;
                }
            }
        }
        __syncthreads();
        bool live[V];
#pragma unroll
        for (int v = 0; v < V; ++v) {
            live[v] = v < nv && !s_stop[v];
            if (v < nv && s_stop[v]) {  // uniform: the scan finished with iteration it-1
                if (threadIdx.x == 0) s_iter[gs[v]] = 255;
                --n_left;
            }
        }
        // ---- work: this warp's chunks of every live scan of the group, no barrier in between ---------------------------
#pragma unroll 1
        for (int v = 0; v < nv; ++v) {
            if (!live[v]) continue;
            const int s = gs[v];
            const P2PlaneScan* __restrict__ sc = a.scans + s;
            const int folder = s % G;
            const int n = sc->n;
            const int n_chunks = (n + 31) >> 5;  // warp-sized chunks
            const float4* __restrict__ src = sc->src;
            float4* __restrict__ rec0 = sc->rec0;
            float4* __restrict__ rec1 = sc->rec1;
            unsigned char* __restrict__ flags = sc->flags;
            // the folder takes the last block of chunks: it is the CTA that stays idle when the scan has fewer chunks than
            // the grid has warps (p2plane_grid adds one CTA for that purpose)
            const int slot = (cta - folder - 1 + G) % G;
            const double* pose = s_pose[v];

            double acc = 0.0;  // lane k's running sum over every chunk of this warp
            // warp-granular work loop, static round-robin over 32-point chunks: no barrier, no atomics inside
            // (consecutive chunks stay in one CTA: Morton neighbours share candidate lists in L1 — spreading them over SMs
            //  for balance was measured 35 % slower; letting the CTA's warps pull the V x W chunk lists of a visit from a
            //  shared counter was measured too: 709 vs 704 us per 8-scan launch, no gain)
            for (int chunk = slot * W + warp; chunk < n_chunks; chunk += n_warps) {
                const int i = (chunk << 5) + lane;
                double J[6] = {0, 0, 0, 0, 0, 0}, ad = 0.0, vflag = 0.0;
                unsigned n_cand = 0, n_fb = 0;
                if (i < n) {
                    const float4 sp = src[i];
                    bool use = p2plane_point(a.map, sp, pose, a.plane_thres, J, ad, n_cand, n_fb);
                    if (use) {
                        rec0[i] = make_float4((float)J[0], (float)J[1], (float)J[2], (float)J[3]);
                        rec1[i] = make_float4((float)J[4], (float)J[5], (float)ad, 1.0f);
                        flags[i] = 1;
                    } else if (flags[i]) {  // stale contribution [quirk 1]
                        const float4 r0 = rec0[i], r1 = rec1[i];
                        J[0] = r0.x; J[1] = r0.y; J[2] = r0.z; J[3] = r0.w; J[4] = r1.x; J[5] = r1.y;
                        ad = r1.z;
                        use = true;
                    } else {
#pragma unroll
                        for (int k = 0; k < 6; ++k) J[k] = 0.0;
                        ad = 0.0;
                    }
                    vflag = use ? 1.0 : 0.0;
                }
                double* rec = s_rec[warp][lane];
#pragma unroll
                for (int k = 0; k < 6; ++k) rec[k] = J[k];
                rec[kRecAd] = ad;
                rec[kRecValid] = vflag;
                rec[kRecCand] = (double)n_cand;
                rec[kRecHits] = (double)n_fb;  // points that took the QR path (diagnostic; reported as hits_total)
                rec[kRecOne] = 1.0;
                __syncwarp();
#pragma unroll 8
                for (int p = 0; p < 32; ++p) acc += s_rec[warp][p][ca] * s_rec[warp][p][cb];
                __syncwarp();
            }
            s_part[v][warp][lane] = acc * sgn;
        }
        __syncthreads();
        // ---- CTA rows: warp v publishes the row of the group's v-th scan — LL records, no fence, no atomic ---------------
        if (warp < nv && live[warp]) {
            const P2PlaneScan* __restrict__ sc = a.scans + gs[warp];
            double val = 0;
#pragma unroll
            for (int w = 0; w < W; ++w) val += s_part[warp][w][lane];
            ll_store(sc->rows + (size_t)cta * 32 + lane, val, sc->tag_base | (unsigned)(git[warp] + 1));
        }
        // ---- folds: for the scans of the group this CTA is the folder of -------------------------------------------------
#pragma unroll 1
        for (int v = 0; v < nv; ++v) {
            if (!live[v] || cta != gs[v] % G) continue;  // uniform per CTA
            const P2PlaneScan* __restrict__ sc = a.scans + gs[v];
            GnState* const state = sc->state;
            const int it = git[v];
            const unsigned tag = sc->tag_base | (unsigned)(it + 1);
            uint4* const rows = sc->rows;
            // warp w owns rows w, w+W, ...; every sweep re-reads all of them (independent loads, one L2 round trip) until
            // each carries this iteration's tag, then the sums are taken in a fixed order — bitwise reproducible, and the
            // fold is finished one sweep after the slowest CTA's row lands
            GnPre pre;
            if (threadIdx.x == 0) gn_load(state, pre);  // off the critical path: the state is stable until gn_step below
            const int nrows = G;
            double sum;
            for (;;) {
                bool ok = true;
                double a0 = 0, a1 = 0, a2 = 0, a3 = 0;
                int r = warp;
                for (; r + 7 * W < nrows; r += 8 * W) {  // 8 independent 16-byte loads in flight per lane
                    double v0, v1, v2, v3, v4, v5, v6, v7;
                    const bool k0 = ll_load(rows + (size_t)r * 32 + lane, tag, v0);
                    const bool k1 = ll_load(rows + (size_t)(r + W) * 32 + lane, tag, v1);
                    const bool k2 = ll_load(rows + (size_t)(r + 2 * W) * 32 + lane, tag, v2);
                    const bool k3 = ll_load(rows + (size_t)(r + 3 * W) * 32 + lane, tag, v3);
                    const bool k4 = ll_load(rows + (size_t)(r + 4 * W) * 32 + lane, tag, v4);
                    const bool k5 = ll_load(rows + (size_t)(r + 5 * W) * 32 + lane, tag, v5);
                    const bool k6 = ll_load(rows + (size_t)(r + 6 * W) * 32 + lane, tag, v6);
                    const bool k7 = ll_load(rows + (size_t)(r + 7 * W) * 32 + lane, tag, v7);
                    ok = ok && k0 && k1 && k2 && k3 && k4 && k5 && k6 && k7;
                    a0 += v0; a1 += v1; a2 += v2; a3 += v3;
                    a0 += v4; a1 += v5; a2 += v6; a3 += v7;
                }
                for (; r + 3 * W < nrows; r += 4 * W) {
                    double v0, v1, v2, v3;
                    const bool k0 = ll_load(rows + (size_t)r * 32 + lane, tag, v0);
                    const bool k1 = ll_load(rows + (size_t)(r + W) * 32 + lane, tag, v1);
                    const bool k2 = ll_load(rows + (size_t)(r + 2 * W) * 32 + lane, tag, v2);
                    const bool k3 = ll_load(rows + (size_t)(r + 3 * W) * 32 + lane, tag, v3);
                    ok = ok && k0 && k1 && k2 && k3;
                    a0 += v0; a1 += v1; a2 += v2; a3 += v3;
                }
                for (; r < nrows; r += W) {
                    double v0;
                    ok = ok && ll_load(rows + (size_t)r * 32 + lane, tag, v0);
                    a0 += v0;
                }
                sum = (a0 + a1) + (a2 + a3);
                if (__all_sync(0xffffffffu, ok)) break;
                __nanosleep(100);
            }
            s_red[warp][lane] = sum;
            __syncthreads();
            if (warp == 0) {
                double t = 0;
#pragma unroll
                for (int w = 0; w < W; ++w) t += s_red[w][lane];
                __syncwarp();
                s_red[0][lane] = t;
                __syncwarp();
                if (lane == 0) gn_step_pre(state, pre, s_red[0], a.gp, sc->log, a.log_cap, sc->ll_pose, tag, sc->result);
            }
            __syncthreads();  // s_red is reused by the next fold
        }
        if (threadIdx.x == 0)
            for (int v = 0; v < nv; ++v)
                if (live[v]) s_iter[gs[v]] = (unsigned char)(git[v] + 1);
        __syncthreads();  // s_part / s_pose / s_stop / s_iter are reused by the next visit
    }
}

// ---- query ordering --------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned spread_bits3(unsigned v) {  // up to 10 bits -> every 3rd bit
    v &= 0x3ffu;
    v = (v | (v << 16)) & 0x030000ffu;
    v = (v | (v << 8)) & 0x0300f00fu;
    v = (v | (v << 4)) & 0x030c30c3u;
    v = (v | (v << 2)) & 0x09249249u;
    return v;
}

// Per-batch preparation in ONE launch: for every scan initialise its GN state from the caller's pose, clear the per-point
// valid flags [quirk 1: reset once per Match] and `zero` (the v9 chunk tickets), and write every scan in locality order.
// Each block owns a tile of kOrderTile consecutive points of one scan and sorts it in shared memory by the key of the voxel each
// point falls into at its initial pose: the 3-D Morton code of the low 4 bits per axis (an 8 m cube) and 2 more bits each of
// x and y (wrap-around beyond that only costs locality, never correctness).  Lanes of a warp then share centre voxels; a
// voxel whose points fall into two tiles is visited from two chunks.  The order is a fixed function of the input (block radix
// sort, ties in the sort's fixed order), so the per-point records and the single-scan kernel's sums stay reproducible.
constexpr int kOrdThreads = 512, kOrdItems = kOrderTile / kOrdThreads;

__global__ void __launch_bounds__(kOrdThreads) p2plane_prep_kernel(const float4* const* __restrict__ scan_ptrs, const int* __restrict__ offsets,
                                                                   const int* __restrict__ tile_off, int n_scans, const PoseArg* __restrict__ poses,
                                                                   float inv_res, unsigned* __restrict__ zero, int n_zero,
                                                                   unsigned char* __restrict__ flags, GnState* __restrict__ states,
                                                                   float4* __restrict__ dst, const HashSlot* __restrict__ ctab, unsigned cmask,
                                                                   const float4* __restrict__ lists) {
    using Sort = cub::BlockRadixSort<unsigned, kOrdThreads, kOrdItems, unsigned>;
    __shared__ typename Sort::TempStorage s_sort;
    if (blockIdx.x == 0) {
        if ((int)threadIdx.x < n_scans) {
            GnState* s = states + threadIdx.x;
            const PoseArg& pose = poses[threadIdx.x];
            for (int k = 0; k < 9; ++k) s->R[k] = s->R0[k] = s->Rprev[k] = pose.R[k];
            for (int k = 0; k < 3; ++k) s->t[k] = s->t0[k] = s->tprev[k] = pose.t[k];
            s->last_rot = s->last_pos = 0.0;
            s->sum_res = 0;
            s->cand_total = s->hits_total = 0;
            s->n_valid = 0;
            s->iter = 0;
            s->done = 0;
            s->converged = 0;
            s->failed = 0;
        }
        for (int k = threadIdx.x; k < n_zero; k += blockDim.x) zero[k] = 0;
    }
    const int tile = (int)blockIdx.x;
    if (tile >= __ldg(tile_off + n_scans)) return;  // the one block of an empty batch
    int sid = 0;  // scan of this tile (block-uniform)
    {
        int lo = 0, hi = n_scans;
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (__ldg(tile_off + mid) <= tile) lo = mid;
            else hi = mid;
        }
        sid = lo;
    }
    const int first = __ldg(offsets + sid) + (tile - __ldg(tile_off + sid)) * kOrderTile;  // batch position of the tile
    const int n_here = min(kOrderTile, __ldg(offsets + sid + 1) - first);
    const float4* __restrict__ src = scan_ptrs[sid] + (first - __ldg(offsets + sid));
    const PoseArg& pose = poses[sid];
    unsigned key[kOrdItems], pos[kOrdItems];
#pragma unroll
    for (int k = 0; k < kOrdItems; ++k) {  // striped: item k of thread t is point k * kOrdThreads + t of the tile (coalesced)
        const int q = k * kOrdThreads + (int)threadIdx.x;
        pos[k] = (unsigned)q;
        key[k] = 1u << 16;  // past the tile's end: a 17th key bit sorts it behind every real point, never written
        if (q < n_here) {
            flags[first + q] = 0;
            const float4 sp = src[q];
            const float qx = xform_row_d(__ldg(&pose.R[0]), __ldg(&pose.R[1]), __ldg(&pose.R[2]), __ldg(&pose.t[0]), sp.x, sp.y, sp.z);
            const float qy = xform_row_d(__ldg(&pose.R[3]), __ldg(&pose.R[4]), __ldg(&pose.R[5]), __ldg(&pose.t[1]), sp.x, sp.y, sp.z);
            const float qz = xform_row_d(__ldg(&pose.R[6]), __ldg(&pose.R[7]), __ldg(&pose.R[8]), __ldg(&pose.t[2]), sp.x, sp.y, sp.z);
            const unsigned kx = (unsigned)ivox_coord(qx, inv_res), ky = (unsigned)ivox_coord(qy, inv_res), kz = (unsigned)ivox_coord(qz, inv_res);
            const unsigned lo = spread_bits3(kx & 15u) | (spread_bits3(ky & 15u) << 1) | (spread_bits3(kz & 15u) << 2);  // 12 bits
            const unsigned hx = (kx >> 4) & 3u, hy = (ky >> 4) & 3u;
            key[k] = lo | (((hx & 1u) | ((hy & 1u) << 1) | ((hx & 2u) << 1) | ((hy & 2u) << 2)) << 12);
            // Warm L2 for the first iteration: the candidate run of the voxel this point starts in is requested now and arrives
            // while the tile is sorted (the GN kernel is latency-bound on exactly these lines when they come from HBM).  One
            // lane per distinct voxel of the warp issues the prefetches.
            if (ctab) {
                const unsigned long long vkey = pack_key((int)kx, (int)ky, (int)kz);
                const unsigned peers = __match_any_sync(__activemask(), vkey);
                if ((int)(__ffs(peers) - 1) == (int)(threadIdx.x & 31)) {
                    unsigned start, count;
                    if (table_find(ctab, cmask, vkey, start, count)) {
                        const char* p = reinterpret_cast<const char*>(lists + start);
                        const unsigned bytes = count * 16u;
                        for (unsigned off = 0; off < bytes; off += 128u) asm volatile("prefetch.global.L2 [%0];" ::"l"(p + off));
                        asm volatile("prefetch.global.L2 [%0];" ::"l"(p + bytes - 1));
                    }
                }
            }
        }
    }
    Sort(s_sort).SortBlockedToStriped(key, pos, 0, 17);
#pragma unroll
    for (int k = 0; k < kOrdItems; ++k) {  // sorted position k * kOrdThreads + t: coalesced stores
        const int r = k * kOrdThreads + (int)threadIdx.x;
        if (r < n_here) dst[first + r] = src[pos[k]];
    }
}

__global__ void ivox_knn_test_kernel(IvoxView map, const float4* __restrict__ q, int n, float4* __restrict__ out, int* __restrict__ found) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 p = q[i];
    Top5 nn;
    unsigned nc;
    knn5_stream(map, p.x, p.y, p.z, nn, nc);
    const unsigned js[5] = {nn.idx(nn.k0), nn.idx(nn.k1), nn.idx(nn.k2), nn.idx(nn.k3), nn.idx(nn.k4)};
    int f = 0;
    for (int k = 0; k < 5; ++k) {
        if (js[k] != 0xffffffffu) {
            out[(size_t)i * 5 + k] = map.lists[js[k]];
            ++f;
        } else {
            out[(size_t)i * 5 + k] = make_float4(0, 0, 0, 0);
        }
    }
    found[i] = f;
}

// LoamPointToPlaneIVOX::AddCloudToLocalMap, the Match-internal call (loam_point_to_plane_ivox.h:79-128 upstream): every
// body-frame point is moved to the map with the FINAL pose and then kept or dropped by looking at the 5 neighbours its
// last PlanerMatch found (those were searched at the pose BEFORE the last update — GnState::Rprev/tprev) and at the
// centre of the 0.5 m cell it falls into:  class 2 ("no need to down-sample": nearest neighbour outside the cell in all
// three axes), class 1 (no cached neighbour closer to the cell centre than the point itself), class 0 (dropped)  [quirk 8].
__global__ void ivox_insert_rule_kernel(IvoxView map, const float4* __restrict__ src, int n, PoseArg prev, PoseArg fin, double filter,
                                        unsigned char* __restrict__ cls, float4* __restrict__ world) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 sp = src[i];
    const float qx = xform_row_d(prev.R[0], prev.R[1], prev.R[2], prev.t[0], (double)sp.x, (double)sp.y, (double)sp.z);
    const float qy = xform_row_d(prev.R[3], prev.R[4], prev.R[5], prev.t[1], (double)sp.x, (double)sp.y, (double)sp.z);
    const float qz = xform_row_d(prev.R[6], prev.R[7], prev.R[8], prev.t[2], (double)sp.x, (double)sp.y, (double)sp.z);
    Top5 nn;
    unsigned nc;
    knn5_stream(map, qx, qy, qz, nn, nc);
    const float wx = xform_row_d(fin.R[0], fin.R[1], fin.R[2], fin.t[0], (double)sp.x, (double)sp.y, (double)sp.z);
    const float wy = xform_row_d(fin.R[3], fin.R[4], fin.R[5], fin.t[1], (double)sp.x, (double)sp.y, (double)sp.z);
    const float wz = xform_row_d(fin.R[6], fin.R[7], fin.R[8], fin.t[2], (double)sp.x, (double)sp.y, (double)sp.z);
    world[i] = make_float4(wx, wy, wz, sp.w);
    const unsigned js[5] = {nn.k0, nn.k1, nn.k2, nn.k3, nn.k4};
    if (js[0] == 0xffffffffu) {  // no cached neighbour at all (:93-96)
        cls[i] = 1;
        return;
    }
    const double pv[3] = {(double)wx, (double)wy, (double)wz};
    double c[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) c[a] = (floor(pv[a] / filter) + 0.5) * filter;  // :97-99
    const float4 n0 = __ldg(map.lists + js[0]);
    const double half = 0.5 * filter;
    if (fabs((double)n0.x - c[0]) > half && fabs((double)n0.y - c[1]) > half && fabs((double)n0.z - c[2]) > half) {  // :103-108
        cls[i] = 2;
        return;
    }
    bool need = true;
    const double dist = (pv[0] - c[0]) * (pv[0] - c[0]) + (pv[1] - c[1]) * (pv[1] - c[1]) + (pv[2] - c[2]) * (pv[2] - c[2]);
    if (js[4] != 0xffffffffu) {  // NUM_MATCH_POINTS cached neighbours (:113)
#pragma unroll
        for (int r = 0; r < 5; ++r) {
            const float4 m = __ldg(map.lists + js[r]);
            const double ex = (double)m.x - c[0], ey = (double)m.y - c[1], ez = (double)m.z - c[2];
            if (ex * ex + ey * ey + ez * ez < dist + 1.0e-6) need = false;  // :114-120
        }
    }
    cls[i] = need ? 1 : 0;
}

// stable two-class compaction: class-1 points first, then class-2 points, both in input order (:126-127)
__global__ void ivox_insert_keys_kernel(const unsigned char* __restrict__ cls, int n, unsigned long long* __restrict__ ones) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) ones[i] = (cls[i] == 1 ? 1ull : 0ull) | (cls[i] == 2 ? (1ull << 32) : 0ull);
}
__global__ void ivox_insert_scatter_kernel(const unsigned char* __restrict__ cls, const unsigned long long* __restrict__ excl, int n,
                                           const float4* __restrict__ world, float4* __restrict__ out, unsigned long long* __restrict__ total) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned long long last = excl[n - 1] + ((cls[n - 1] == 1 ? 1ull : 0ull) | (cls[n - 1] == 2 ? (1ull << 32) : 0ull));
    const unsigned n1 = (unsigned)(last & 0xffffffffull);
    if (i == 0) *total = last;
    const unsigned char c = cls[i];
    if (c == 1) out[(unsigned)(excl[i] & 0xffffffffull)] = world[i];
    else if (c == 2) out[n1 + (unsigned)(excl[i] >> 32)] = world[i];
}

// One 768-thread CTA per SM: 24 resident warps (<= 80 registers).
constexpr int kMinB = 1;
size_t p2plane_smem() {
    constexpr int W = kP2PlaneBlock / 32, V = kVisitGroup < W ? kVisitGroup : W;
    return (size_t)W * 32 * kRecW * sizeof(double) + (size_t)V * W * 32 * sizeof(double);
}

}  // namespace

int p2plane_chunks(int n) { return (n + 31) / 32; }

int p2plane_grid(int n, int device) {
    const int W = kP2PlaneBlock / 32;
    const int need = (p2plane_chunks(n) + W - 1) / W;
    // + the folding CTA (stays without chunks when there is room)
    return clamp_grid(need + 1, coresident_ctas((const void*)p2plane_gn_kernel<kP2PlaneBlock, kMinB>, kP2PlaneBlock, p2plane_smem(), device));
}

void launch_p2plane_loop(const P2PlaneLoopArgs& a, int grid, cudaStream_t st) {
    launch_cooperative(p2plane_gn_kernel<kP2PlaneBlock, kMinB>, grid, kP2PlaneBlock, p2plane_smem(), st, a);
}

// Per-batch preparation: state init, flag and ticket reset and the locality order of every scan, in one launch of one block per
// tile (one block for an empty batch).
void prepare_queries(const float4* const* d_scan_ptrs, const int* d_offsets, const int* d_tile_off, int n_tiles, int n_scans,
                     const PoseArg* d_poses, GnState* d_states, const IvoxView& map, unsigned char* d_flags, float4* d_sorted,
                     unsigned* d_zero, int n_zero, cudaStream_t st, int* launches) {
    p2plane_prep_kernel<<<n_tiles > 0 ? n_tiles : 1, kOrdThreads, 0, st>>>(d_scan_ptrs, d_offsets, d_tile_off, n_scans, d_poses, map.inv_res, d_zero,
                                                                          n_zero, d_flags, d_states, d_sorted, map.ctab, map.cmask, map.lists);
    if (launches) *launches += 1;
}

// Returns the number of points selected for insertion (class 1 then class 2, input order) in d_out; synchronises the stream.
size_t select_ivox_inserts(const IvoxView& map, const float4* d_src, int n, const double* R_prev, const double* t_prev, const double* R_fin,
                           const double* t_fin, double filter, float4* d_world, float4* d_out, BuildScratch& sc, cudaStream_t st, int* launches) {
    if (n <= 0) return 0;
    PoseArg prev, fin;
    for (int k = 0; k < 9; ++k) {
        prev.R[k] = R_prev[k];
        fin.R[k] = R_fin[k];
    }
    for (int k = 0; k < 3; ++k) {
        prev.t[k] = t_prev[k];
        fin.t[k] = t_fin[k];
    }
    sc.minmax.reserve((size_t)n / 4 + 16);  // class bytes
    unsigned char* cls = reinterpret_cast<unsigned char*>(sc.minmax.p);
    sc.keys.reserve((size_t)n + 1);
    sc.keys_sorted.reserve((size_t)n + 1);
    const int g = (n + 127) / 128;
    ivox_insert_rule_kernel<<<g, 128, 0, st>>>(map, d_src, n, prev, fin, filter, cls, d_world);
    ivox_insert_keys_kernel<<<(n + 255) / 256, 256, 0, st>>>(cls, n, sc.keys.p);
    size_t tb = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, tb, sc.keys.p, sc.keys_sorted.p, n, st);
    sc.cub_tmp.reserve(tb + 256);
    tb = sc.cub_tmp.cap;
    FLS_CUDA(cub::DeviceScan::ExclusiveSum(sc.cub_tmp.p, tb, sc.keys.p, sc.keys_sorted.p, n, st));
    unsigned long long* d_total = sc.keys.p + n;  // spare slot
    ivox_insert_scatter_kernel<<<(n + 255) / 256, 256, 0, st>>>(cls, sc.keys_sorted.p, n, d_world, d_out, d_total);
    unsigned long long total = 0;
    FLS_CUDA(cudaMemcpyAsync(&total, d_total, sizeof(total), cudaMemcpyDeviceToHost, st));
    FLS_CUDA(cudaStreamSynchronize(st));
    if (launches) *launches += 4;
    return (size_t)(total & 0xffffffffull) + (size_t)(total >> 32);
}

void launch_ivox_knn_test(const IvoxView& map, const float4* d_q, int n, float4* d_out, int* d_found, cudaStream_t st) {
    if (n <= 0) return;
    ivox_knn_test_kernel<<<(n + 127) / 128, 128, 0, st>>>(map, d_q, n, d_out, d_found);
}

}  // namespace fls
