// fls_p2plane.cu — K1 (+ fused K6), generation 8: the whole LoamPointToPlaneIVOX Gauss-Newton loop of ONE scan as one persistent
// kernel with a CTA barrier per iteration.  It serves the single Match (fls_match / fls_match_device); batches run on generation 9
// (fls_p2plane_v9.cu), which shares the per-point arithmetic (fls_knn.cuh, fls_plane.cuh).  This file also holds the per-batch query
// preparation (one kernel: every scan's gn_state_init + tile-local locality sort), the Match-internal insertion rule of mapping mode, the
// k-NN test entry and the plug-in's host half (IvoxPlugin: its iVox map, its per-batch table and watchdog word, AddCloudToLocalMap, and
// the single and batch Match on v8 / v9 over the shared host half of a Match in Handle).
//
// Per source point and iteration it fuses what LoamPointToPlaneIVOX::PlanerMatch / ::SumCoefficient do
// (include/registration/loam_point_to_plane_ivox.h:256-340 upstream): transform with the current pose, bounded
// 5-NN in the iVox map, least-squares plane through the 5 neighbours (normal equations, column-pivoted Householder QR as the
// fallback, fp64), validity / near-point gates, J (6) and |d|, and the 21+6+2 Gauss-Newton sums; the folding CTA reduces
// the CTA rows in a fixed order, solves the 6x6 system, updates the pose and applies the stop rule (:167-203), then publishes the
// next pose.  No host round trip inside a Match.
//
// Mapping onto the GPU
//   * grid = the CTAs the scan's chunks need (one 24-warp CTA per SM, 768 threads, 80 registers) + the folding CTA, launched
//     cooperatively only to guarantee co-residency; the scheduling unit is the WARP: warp w of CTA c works on 32-point chunk
//     (c, w), a static round-robin (consecutive chunks stay in one CTA: Morton neighbours share candidate runs in L1);
//   * an iteration = chunks, then the shared hand-over (gn_handover_rows, fls_gn.cuh): one __syncthreads, CTA row out (LL
//     records, no fence, no atomic); only CTA 0 waits for the other rows — 24 warps x 8 loads in flight sweep them until every
//     tag matches, sums in a fixed order (bitwise reproducible for a given grid), gn_step, next pose out, every CTA polls it;
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

#include <algorithm>

#include <cub/cub.cuh>

#include "fls_gn.cuh"
#include "fls_handle.h"
#include "fls_info.cuh"
#include "fls_ivox.cuh"
#include "fls_knn.cuh"
#include "fls_plane.cuh"

namespace fls {

static constexpr int kP2PlaneBlock = 768;  // shape of the single-scan kernel: one 24-warp CTA per SM

// whole-loop arguments of the single-scan kernel (generation 8)
struct P2PlaneArgs {
    IvoxView map;
    double plane_thres;
    const float4* src;  // body-frame scan in Morton order of the query voxel (prepare_queries), packed float4
    int n;
    float4* rec0;  // persistent per-point record: J0..J3
    float4* rec1;  //                              J4, J5, |d|, 1
    unsigned char* flags;
};

// queries of a batch are put in locality order in tiles of this many consecutive points; a tile never spans two scans
static constexpr int kOrderTile = 8192;
inline int order_tiles(int n) { return (n + kOrderTile - 1) / kOrderTile; }

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

template <int BLOCK, int MINB>
__global__ void __launch_bounds__(BLOCK, MINB) p2plane_gn_kernel(P2PlaneArgs a, GnLoopCtl ctl) {
    constexpr int W = BLOCK / 32;
    extern __shared__ __align__(16) unsigned char s_dyn[];
    double (*s_rec)[32][kRecW] = reinterpret_cast<double (*)[32][kRecW]>(s_dyn);  // [W][32][kRecW] per-lane staging records
    __shared__ double s_red[W][kAccStride];  // every warp's 32 sums
    __shared__ int s_stop;
    __shared__ double s_pose[12];
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
    // iteration 0 starts from the state the prep kernel wrote; gn_handover_rows leaves every later pose in s_pose
    if (threadIdx.x < 12) s_pose[threadIdx.x] = threadIdx.x < 9 ? __ldcg(&ctl.state->R[threadIdx.x]) : __ldcg(&ctl.state->t[threadIdx.x - 9]);
    __syncthreads();
    const int n_chunks = (a.n + 31) >> 5;  // warp-sized chunks
    // CTA 0 folds, so it takes the last block of chunks: it is the CTA that stays idle when the scan has fewer chunks than
    // the grid has warps (p2plane_grid adds one CTA for that purpose)
    const int slot = (cta - 1 + G) % G;
    for (int it = 0;; ++it) {  // ends on the stop word, which gn_step raises at max_iterations at the latest
        double acc = 0.0;  // lane k's running sum over every chunk of this warp
        // warp-granular work loop, static round-robin over 32-point chunks: no barrier, no atomics inside
        // (consecutive chunks stay in one CTA: Morton neighbours share candidate lists in L1 — spreading them over SMs
        //  for balance was measured 35 % slower)
        for (int chunk = slot * W + warp; chunk < n_chunks; chunk += n_warps) {
            const int i = (chunk << 5) + lane;
            double J[6] = {0, 0, 0, 0, 0, 0}, ad = 0.0, vflag = 0.0;
            unsigned n_cand = 0, n_fb = 0;
            if (i < a.n) {
                const float4 sp = a.src[i];
                bool use = p2plane_point(a.map, sp, s_pose, a.plane_thres, J, ad, n_cand, n_fb);
                if (use) {
                    a.rec0[i] = make_float4((float)J[0], (float)J[1], (float)J[2], (float)J[3]);
                    a.rec1[i] = make_float4((float)J[4], (float)J[5], (float)ad, 1.0f);
                    a.flags[i] = 1;
                } else if (a.flags[i]) {  // stale contribution [quirk 1]
                    const float4 r0 = a.rec0[i], r1 = a.rec1[i];
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
        s_red[warp][lane] = acc * sgn;
        if (gn_handover_rows<BLOCK>(s_red, s_stop, ctl, ctl.tag_base | (unsigned)(it + 1), s_pose)) break;
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
// sort, ties in the sort's fixed order), so the per-point records and the single-scan kernel's sums stay reproducible.  A single
// Match is the batch of one; its kernel starts from the state written here.
constexpr int kOrdThreads = 512, kOrdItems = kOrderTile / kOrdThreads;

__global__ void __launch_bounds__(kOrdThreads) p2plane_prep_kernel(const float4* const* __restrict__ scan_ptrs, const int* __restrict__ offsets,
                                                                   const int* __restrict__ tile_off, int n_scans, const GnPose* __restrict__ poses,
                                                                   float inv_res, unsigned* __restrict__ zero, int n_zero,
                                                                   unsigned char* __restrict__ flags, GnState* __restrict__ states,
                                                                   float4* __restrict__ dst, const HashSlot* __restrict__ ctab, unsigned cmask,
                                                                   const float4* __restrict__ lists) {
    using Sort = cub::BlockRadixSort<unsigned, kOrdThreads, kOrdItems, unsigned>;
    __shared__ typename Sort::TempStorage s_sort;
    if (blockIdx.x == 0) {
        if ((int)threadIdx.x < n_scans) gn_state_init(states + threadIdx.x, poses[threadIdx.x]);
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
    const GnPose& pose = poses[sid];
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
__global__ void ivox_insert_rule_kernel(IvoxView map, const float4* __restrict__ src, int n, GnPose prev, GnPose fin, double filter,
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
size_t p2plane_smem() { return (size_t)(kP2PlaneBlock / 32) * 32 * kRecW * sizeof(double); }

}  // namespace

// FLS_FLAG_INFORMATION: the loops' per-point term (p2plane_point, fls_info.cuh), W = 1, over the scan in its locality order; the
// evaluation reads map, plane_thres, src and n, never the persistent records
template <>
struct InfoTerm<P2PlaneArgs> {
    static constexpr int kBlock = 256, kLanes = 1;
    static __host__ __device__ int count(const P2PlaneArgs& a) { return a.n; }
    static __device__ __forceinline__ void point(const P2PlaneArgs& a, int i, const double* pose, const float*, int, unsigned, double (&acc)[kNumAcc]) {
        double J[6], ad = 0.0;
        unsigned n_cand, n_fb;
        if (p2plane_point(a.map, a.src[i], pose, a.plane_thres, J, ad, n_cand, n_fb)) info_add_J(J, ad, acc);
    }
};

// CTAs that serve a scan of n points: its warp-sized (32-point) chunks / warps per CTA, + the folder, <= co-resident
static int p2plane_grid(int n, int device) {
    const int W = kP2PlaneBlock / 32;
    const int need = ((n + 31) / 32 + W - 1) / W;
    // + the folding CTA (stays without chunks when there is room)
    return clamp_grid(need + 1, coresident_ctas((const void*)p2plane_gn_kernel<kP2PlaneBlock, kMinB>, kP2PlaneBlock, p2plane_smem(), device));
}

static void launch_p2plane_loop(const P2PlaneArgs& a, const GnLoopCtl& ctl, int grid, cudaStream_t st) {
    launch_cooperative(p2plane_gn_kernel<kP2PlaneBlock, kMinB>, grid, kP2PlaneBlock, p2plane_smem(), st, a, ctl);
}

// The per-batch table of a LOAM-iVox Match, staged in pinned memory and sent with one copy
struct IvoxBatchTable {
    GnPose pose[kMaxBatch];        // the pose each scan starts from
    int off[kMaxBatch + 4];        // [n_scans + 1]: the scans' positions in the batch
    int tile_off[kMaxBatch + 4];   // [n_scans + 1]: prefix sums of order_tiles(n) over the scans
    P2PlaneScan desc[kMaxBatch];   // the v9 kernel's scan descriptors
    const float4* ptr[kMaxBatch];  // device pointers of the scans
};

// Per-batch preparation: state init, flag and ticket reset and the locality order of every scan, in one launch of one block per
// tile (one block for an empty batch).  d_tbl: the batch's table on the device; d_zero[n_zero]: words zeroed on the way (v9 tickets).
static void prepare_queries(const IvoxBatchTable* d_tbl, int n_tiles, int n_scans, GnState* d_states, const IvoxView& map, unsigned char* d_flags,
                            float4* d_sorted, unsigned* d_zero, int n_zero, Call& c) {
    p2plane_prep_kernel<<<n_tiles > 0 ? n_tiles : 1, kOrdThreads, 0, c.stream>>>(d_tbl->ptr, d_tbl->off, d_tbl->tile_off, n_scans, d_tbl->pose,
                                                                                map.inv_res, d_zero, n_zero, d_flags, d_states, d_sorted, map.ctab,
                                                                                map.cmask, map.lists);
    c.launches += 1;
}

// The Match-internal AddCloudToLocalMap of mapping mode: classifies and compacts the points that enter the map (d_world, d_out: n
// records).  Returns the number of points selected for insertion (class 1 then class 2, input order) in d_out; waits once.
static size_t select_ivox_inserts(const IvoxView& map, const float4* d_src, int n, const GnPose& prev, const GnPose& fin, double filter, float4* d_world,
                                  float4* d_out, BuildScratch& sc, Call& c) {
    if (n <= 0) return 0;
    const cudaStream_t st = c.stream;
    sc.minmax.reserve((size_t)n / 4 + 16);  // class bytes
    unsigned char* cls = reinterpret_cast<unsigned char*>(sc.minmax.p);
    sc.keys.reserve((size_t)n + 1);
    sc.keys_sorted.reserve((size_t)n + 1);
    const int g = (n + 127) / 128;
    ivox_insert_rule_kernel<<<g, 128, 0, st>>>(map, d_src, n, prev, fin, filter, cls, d_world);
    ivox_insert_keys_kernel<<<(n + 255) / 256, 256, 0, st>>>(cls, n, sc.keys.p);
    cub_pass(sc.cub_tmp, [&](void* tmp, size_t& bytes) { return cub::DeviceScan::ExclusiveSum(tmp, bytes, sc.keys.p, sc.keys_sorted.p, n, st); });
    unsigned long long* d_total = sc.keys.p + n;  // spare slot
    ivox_insert_scatter_kernel<<<(n + 255) / 256, 256, 0, st>>>(cls, sc.keys_sorted.p, n, d_world, d_out, d_total);
    unsigned long long total = 0;
    FLS_CUDA(cudaMemcpyAsync(&total, d_total, sizeof(total), cudaMemcpyDeviceToHost, st));
    c.sync();
    c.launches += 4;
    return (size_t)(total & 0xffffffffull) + (size_t)(total >> 32);
}

// ---- LoamPointToPlaneIVOX ------------------------------------------------------------------------------------

class IvoxPlugin final : public Plugin {
    IvoxMap map;
    DevBuf<float4> queries;     // the scans of the batch in locality order (prepare_queries)
    DevBuf<float4> rec0, rec1;  // persistent per-point {J, |d|} records
    DevBuf<unsigned char> flags;
    DevBuf<unsigned> tickets;   // chunk ticket counters of the v9 kernel (dynamic work distribution)
    DevBuf<float4> ins_world, ins;  // Match-internal insert: the scan at its final pose, the points that enter the map
    PinnedBuf<unsigned char> h_tbl;  // the per-batch table (IvoxBatchTable), staged ...
    DevBuf<unsigned char> d_tbl;     // ... and its device copy
    // watchdog word of the last batch launch, read back with the states (pinned: a copy into pageable memory would make the enqueue
    // wait for the kernel)
    PinnedBuf<unsigned> h_abort;
    std::vector<size_t> pend_n;     // scans of the batch in flight (empty: none)
    bool pend_v9 = false;

    IvoxView view() const {
        const float max_range2 = h.cfg.ivox_max_range * h.cfg.ivox_max_range;
        // a query and a candidate of its stencil differ by at most 2*res per axis with a non-zero offset and res otherwise:
        // d^2 <= 12 res^2 for the full 26-neighbourhood
        const unsigned fast_knn = 12.0 * 1.01 * (double)map.res * (double)map.res < (double)max_range2 ? 1u : 0u;
        return {map.pts_sorted.p, map.table.buf.p, map.table.mask, map.inv_res, max_range2, map.n_stencil, map.lists.p, map.ctab.buf.p, map.ctab.mask,
                fast_knn};
    }
    int append(const float4* d, size_t n) { return map.append_and_build(d, n, h.cfg.ivox_capacity, h.call); }

    // everything of a batch up to the asynchronous read-back of the states: nothing here waits for the device
    int enqueue(int B, const float4* const* d_scans, const size_t* n, const double* T) {
        if (map.n_pts == 0) return FLS_ERR_NO_MAP;
        const int device = h.cfg.device;
        cudaStream_t stream = h.call.stream;
        int off[kMaxBatch + 1];
        off[0] = 0;
        int grid = 1;
        // K1 generations: the dataflow kernel (v9: TMA-staged runs, work ring, DMMA sums — fls_p2plane_v9.cu) serves batches; a single
        // Match runs on the barrier kernel (v8, this file) whose one-chunk-per-warp round has the shorter hand-over (DESIGN.md §3.1 has
        // the H100 numbers)
        const bool use_v9 = B > 1;
        for (int s = 0; s < B; ++s) {
            if (n[s] > 0x3fffffffull || (long long)off[s] + (long long)n[s] > 0x7ffffff0ll) return FLS_ERR_INVALID_ARG;
            off[s + 1] = off[s] + (int)n[s];
            const int g = use_v9 ? p2plane_v9_grid((int)n[s], device) : p2plane_grid((int)n[s], device);
            if (g > grid) grid = g;
        }
        const int n_total = off[B];
        const size_t nt = (size_t)n_total;
        rec0.reserve(nt + 1);
        rec1.reserve(nt + 1);
        flags.reserve(nt + 1);
        queries.reserve(nt + 1);
        // one LL row per CTA + one LL pose record per scan (+ the group rows of v9)
        const unsigned tag_base = h.next_ll_epoch((size_t)B * grid * 32 + (size_t)B * kLlPoseLen + (size_t)B * 16 * 32);
        // ---- the per-batch table -------------------------------------------------------------------------------------------
        IvoxBatchTable& t = *reinterpret_cast<IvoxBatchTable*>(h_tbl.reserve(sizeof(IvoxBatchTable)));
        const IvoxBatchTable* d_t = reinterpret_cast<const IvoxBatchTable*>(d_tbl.reserve(sizeof(IvoxBatchTable)));
        // scan s's control block: its rows of grid x 32 LL records, then its LL pose record after every scan's rows
        uint4* pose_base = h.ll_rows.p + (size_t)B * grid * 32;
        auto ctl = [&](int s) {
            return h.loop_ctl(s, FLS_P2PLANE_IVOX, 50, tag_base, h.ll_rows.p + (size_t)s * grid * 32, pose_base + (size_t)s * kLlPoseLen);
        };
        t.tile_off[0] = 0;
        for (int s = 0; s < B; ++s) {
            t.pose[s] = gn_pose(T + 16 * s);
            t.off[s] = off[s];
            t.tile_off[s + 1] = t.tile_off[s] + order_tiles((int)n[s]);
            t.ptr[s] = d_scans[s];
            const GnLoopCtl c = ctl(s);
            P2PlaneScan& d = t.desc[s];
            d.src = queries.p + off[s];
            d.n = (int)n[s];
            d.tag_base = c.tag_base;
            d.state = c.state;
            d.rec0 = rec0.p + off[s];
            d.rec1 = rec1.p + off[s];
            d.flags = flags.p + off[s];
            d.rows = c.ll_rows;
            d.ll_pose = c.ll_pose;
            d.log = c.log;
            d.result = c.result;
            d.grows = pose_base + (size_t)B * kLlPoseLen + (size_t)s * 16 * 32;
        }
        t.off[B] = off[B];
        FLS_CUDA(cudaMemcpyAsync(d_tbl.p, &t, sizeof(t), cudaMemcpyHostToDevice, stream));
        h.call.h2d += (long long)sizeof(t);
        // chunk tickets of v9's dynamic work distribution: one counter per (scan, iteration) + the watchdog's abort word, zeroed by
        // the prep kernel
        const int ticket_stride = h.cfg.max_iterations + 2;
        const int n_tickets = use_v9 ? B * ticket_stride + 4 : 0;
        if (use_v9) tickets.reserve((size_t)n_tickets);
        // ONE prep kernel for the whole batch (state init, flag and ticket reset): every tile of a scan ends up in Morton order of the
        // voxel its points fall into at the initial pose (locality only: the sums are order-free up to fp64 rounding, and the
        // persistent per-point records live in the same order for the whole Match)
        prepare_queries(d_t, t.tile_off[B], B, h.state.p, view(), flags.p, queries.p, use_v9 ? tickets.p : nullptr, n_tickets, h.call);
        P2PlaneLoopArgs a;
        a.map = view();
        a.plane_thres = h.cfg.point_to_planar_thres;
        a.gp = h.gn_params(FLS_P2PLANE_IVOX, 50);
        a.log_cap = h.log_cap;
        a.scans = d_t->desc;
        a.n_scans = B;
        a.tickets = nullptr;
        a.ticket_stride = 0;
        a.abort_word = nullptr;
        // roofline accounting (SURVEY.md §8d, K1 — the REFERENCE algorithm's traffic): 16 B source point + n_stencil x 16 B
        // slot probes + 32 B persistent record per point-iteration, 16 B per map record resident in the stencil voxels.
        h.gn_launch(16 + 16LL * a.map.n_stencil + 32, 16, d_scans[0], n[0], [&] {
            if (use_v9) {
                a.ticket_stride = ticket_stride;
                a.tickets = tickets.p;
                a.abort_word = tickets.p + (size_t)B * a.ticket_stride;
                launch_p2plane_v9(a, grid, stream);
            } else {  // the single scan: the same buffers as scan 0's descriptor above
                const P2PlaneArgs one{a.map, a.plane_thres, queries.p, (int)n[0], rec0.p, rec1.p, flags.p};
                launch_p2plane_loop(one, ctl(0), grid, stream);
            }
        });
        if (h.info_on) {
            P2PlaneArgs info_args[kMaxBatch];
            for (int s = 0; s < B; ++s) info_args[s] = {a.map, a.plane_thres, queries.p + off[s], (int)n[s], nullptr, nullptr, nullptr};
            enqueue_information(h, info_args, B);
        }
        // ---- read back: every scan's state (+ its iteration log) ----------------------------------------------------------
        h.read_back(B);
        *h_abort.p = 0;
        if (use_v9) FLS_CUDA(cudaMemcpyAsync(h_abort.p, a.abort_word, sizeof(unsigned), cudaMemcpyDeviceToHost, stream));
        pend_n.assign(n, n + B);
        pend_v9 = use_v9;
        return FLS_OK;
    }

    // waits for the batch enqueued last and unpacks its results
    int finish(double* T, int* converged, fls_match_stats* st) {
        const int B = (int)pend_n.size();
        if (B < 1) return FLS_ERR_INVALID_ARG;
        h.call.end(st);
        if (pend_v9 && *h_abort.p) {
            pend_n.clear();
            set_last_error("p2plane_v9_kernel: watchdog — a wait loop gave up after 4 s (hand-over protocol error)");
            return FLS_ERR_CUDA;
        }
        h.unpack(B, pend_n.data(), T, converged, st);
        pend_n.clear();
        return FLS_OK;
    }

    // The whole LoamPointToPlaneIVOX Match of `B` independent scans in one persistent launch; a single Match is the batch of one.
    int run(int B, const float4* const* d_scans, const size_t* n, double* T, int* converged, fls_match_stats* st) {
        const int rc = enqueue(B, d_scans, n, T);
        if (rc != FLS_OK) return rc;
        return finish(T, converged, st);
    }

  public:
    explicit IvoxPlugin(Handle& handle) : Plugin(handle, kPlanar) {
        static const int counts[4] = {1, 7, 19, 27};
        map.set_resolution(h.cfg.ivox_resolution);
        map.incremental = !h.cfg.localization_mode;  // mapping mode: the map grows by small inserts
        map.n_stencil = counts[h.cfg.ivox_nearby];
        h_abort.reserve(1);
    }

    // external non-first insert in mapping mode: relies on Match-internal caches upstream
    int add_check() const override { return !h.cfg.localization_mode && map.n_pts != 0 ? FLS_ERR_UNSUPPORTED : FLS_OK; }

    int add_cloud(const float4* d, size_t n, const float4*, size_t) override {
        const int chk = add_check();
        if (chk != FLS_OK) return chk;
        if (h.cfg.localization_mode) map.clear();  // loam_point_to_plane_ivox.h:64-69 upstream: map re-created per call
        const int rc = append(d, n);
        if (h.cfg.localization_mode) h.set_fit_cloud(d, n);  // :134-138 kd-tree over the raw planar cloud
        return rc;
    }

    int match(const float4* d_src, size_t n, const float4*, size_t, double* T, int* converged, fls_match_stats* st) override {
        const float4* scans[1] = {d_src};
        const size_t ns[1] = {n};
        int conv = 0;
        const int rc = run(1, scans, ns, T, &conv, st);
        if (rc != FLS_OK) return rc;
        if (converged) *converged = conv;
        const GnState& s = h.h_state.p[0];
        if (s.converged && !h.cfg.localization_mode) {
            // :205-206 — the scan enters the map through the cached-5-NN rule (body-frame points, final pose T)  [quirk 8]
            GnPose prev;
            std::copy(s.Rprev, s.Rprev + 9, prev.R);
            std::copy(s.tprev, s.tprev + 3, prev.t);
            ins.reserve(n + 1);
            ins_world.reserve(n + 1);
            const size_t n_add = select_ivox_inserts(view(), d_src, (int)n, prev, gn_pose(T), 0.5 /* filter_size_map_min_ (:351) */, ins_world.p,
                                                     ins.p, h.scratch, h.call);
            return h.inserted(append(ins.p, n_add), st);
        }
        return FLS_OK;
    }

    int match_batch(int B, const void* const* scans, const size_t* n, size_t host_stride, double* T, int* converged,
                    fls_match_stats* st) override {
        const float4* ptrs[kMaxBatch];
        const int rc = h.begin_batch(B, scans, n, host_stride, ptrs, st);
        if (rc != FLS_OK) return rc;
        return B == 1 ? match(ptrs[0], n[0], nullptr, 0, T, converged, st) : run(B, ptrs, n, T, converged, st);
    }

    int batch_begin(int B, const void* const* scans, const size_t* n, size_t host_stride, const double* T) override {
        const float4* ptrs[kMaxBatch];
        const int rc = h.begin_batch(B, scans, n, host_stride, ptrs, nullptr);
        if (rc != FLS_OK) return rc;
        return enqueue(B, ptrs, n, T);
    }
    int batch_end(double* T, int* converged, fls_match_stats* st) override { return finish(T, converged, st); }
    int batch_pending() const override { return (int)pend_n.size(); }

    void map_info(fls_map_info* out) const override {
        out->n_points = (long long)map.n_pts;
        out->n_voxels = (long long)map.n_vox;
        out->table_slots = map.n_pts ? (long long)map.table.slots : 0;
        out->bytes = (long long)map.bytes();
        out->incremental_inserts = (long long)map.n_incremental;
        out->full_builds = (long long)map.n_full;
    }

    int voxel_keys(std::vector<unsigned long long>& packed, size_t cap, size_t* n) override {
        FLS_CUDA(cudaSetDevice(h.cfg.device));
        packed.resize(cap + 1);
        packed.resize(map.dump_keys(packed.data(), cap, h.call.stream));
        *n = map.n_vox;
        return FLS_OK;
    }

    int map_points(float* xyzi, size_t cap, size_t* n) override {
        FLS_CUDA(cudaSetDevice(h.cfg.device));
        FLS_CUDA(cudaStreamSynchronize(h.call.stream));
        const size_t m = map.n_pts < cap ? map.n_pts : cap;
        if (m) FLS_CUDA(cudaMemcpy(xyzi, map.pts_all.p, m * sizeof(float4), cudaMemcpyDeviceToHost));
        *n = map.n_pts;
        return FLS_OK;
    }

    int ivox_knn(const void* queries_in, size_t n, size_t stride, float* out_pts, int32_t* out_count) override {
        if (map.n_pts == 0) return FLS_ERR_NO_MAP;
        h.begin_call();
        const float4* dq = h.upload(queries_in, n, stride, h.src);
        DevBuf<float4> d_out;
        DevBuf<int> d_found;
        d_out.reserve(n * 5);
        d_found.reserve(n);
        if (n > 0) ivox_knn_test_kernel<<<(unsigned)((n + 127) / 128), 128, 0, h.call.stream>>>(view(), dq, (int)n, d_out.p, d_found.p);
        FLS_CUDA(cudaMemcpyAsync(out_pts, d_out.p, n * 5 * sizeof(float4), cudaMemcpyDeviceToHost, h.call.stream));
        FLS_CUDA(cudaMemcpyAsync(out_count, d_found.p, n * sizeof(int), cudaMemcpyDeviceToHost, h.call.stream));
        h.call.end(nullptr);
        return FLS_OK;
    }

    // fls_ivox_add_points: IVoxMap::AddPoints on the map as it is (no localization-mode re-creation)
    int ivox_add_points(const void* pts, size_t n, size_t stride) override {
        h.begin_call();
        const int rc = append(h.upload(pts, n, stride, h.up_cloud), n);
        h.call.end(nullptr);
        return rc;
    }
};

std::unique_ptr<Plugin> make_ivox_plugin(Handle& h) { return std::make_unique<IvoxPlugin>(h); }

}  // namespace fls
