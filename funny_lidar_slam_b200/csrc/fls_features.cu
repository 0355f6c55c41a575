// fls_features.cu — K4: LOAM edge / planar feature extraction on the projector's arrays.
//
// loam::FeatureExtractor::ExtractFeatures (src/loam/feature_extractor.cpp:35-222 upstream) =
//   SelectValidPoints (:64-118)  — occlusion / parallel-beam masks          -> feat_point_kernel (one thread per point)
//   ComputeRoughness  (:46-61)   — 11-tap range curvature                   -> feat_point_kernel
//   SelectFeatures    (:120-222) — per ring, 6 blocks: sort by roughness, greedy corner pick (<= 20, suppress +-5),
//                                  greedy planar suppression, emit every non-corner  -> feat_ring_kernel (one CTA per ring)
// Rings are independent (index gap 11 between rows, pointcloud_projector.cpp:115,131); blocks of a ring are not
// (suppression and the inclusive `block_end` visit bleed into the next block [quirk 10]), so a CTA walks its 6 blocks in
// order: bitonic sort of (roughness, position) in shared memory by the whole CTA — the composite key makes the unstable
// upstream std::sort deterministic exactly as the oracle pins it — then the two greedy passes by one thread on
// shared-memory state (they are sequential by definition: every pick changes the validity of later candidates).
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "fls_frontend.h"

namespace fls {
namespace {

// per-point meta byte: bit0 valid, bit1 corner, bits 2-4 forward suppression reach, bits 5-7 backward reach
__device__ __forceinline__ int col_gap_ok(const int* __restrict__ col, int a, int b) { return abs(col[a] - col[b]) <= 10; }

__global__ void feat_point_kernel(const float* __restrict__ depth, const int* __restrict__ col, int n, float* __restrict__ rough,
                                  unsigned char* __restrict__ meta) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    // roughness (:46-61): left-to-right fp32 sum, then - 10*d, squared; no FMA contraction
    float r = 0.f;
    if (k >= 5 && k < n - 5) {
        float s = __fadd_rn(depth[k - 5], depth[k - 4]);
        s = __fadd_rn(s, depth[k - 3]);
        s = __fadd_rn(s, depth[k - 2]);
        s = __fadd_rn(s, depth[k - 1]);
        s = __fadd_rn(s, depth[k + 1]);
        s = __fadd_rn(s, depth[k + 2]);
        s = __fadd_rn(s, depth[k + 3]);
        s = __fadd_rn(s, depth[k + 4]);
        s = __fadd_rn(s, depth[k + 5]);
        s = __fsub_rn(s, __fmul_rn(10.0f, depth[k]));
        r = __fmul_rn(s, s);
    }
    rough[k] = r;
    // validity (:64-118) in gather form: k is cleared by an occlusion found at i in [k, k+5] (near side, clears i-5..i),
    // by one found at i in [k-6, k-1] (far side, clears i+1..i+6), or by the parallel-beam test at k itself
    bool valid = !(k < 5 || k >= n - 6);
    const int lo = 5, hi = n - 6;  // i ranges over [lo, hi)
    if (valid) {
        for (int i = max(k, lo); i <= k + 5 && i < hi; ++i) {
            if (abs(col[i + 1] - col[i]) < 10 && (double)__fsub_rn(depth[i], depth[i + 1]) > 0.3) valid = false;
        }
        for (int i = max(k - 6, lo); i <= k - 1 && i < hi; ++i) {
            if (abs(col[i + 1] - col[i]) < 10 && !((double)__fsub_rn(depth[i], depth[i + 1]) > 0.3) &&
                (double)__fsub_rn(depth[i + 1], depth[i]) > 0.3)
                valid = false;
        }
        if (k >= lo && k < hi) {
            const float d1 = fabsf(__fsub_rn(depth[k - 1], depth[k])), d2 = fabsf(__fsub_rn(depth[k + 1], depth[k]));
            const double lim = 0.02 * (double)depth[k];
            if ((double)d1 > lim && (double)d2 > lim) valid = false;
        }
    } else if (k >= 5 && k < n - 6) {
        valid = false;
    }
    // points outside [5, n-6) are invalid but may still be cleared again harmlessly; occlusions can also clear them
    int fwd = 0, bwd = 0;
    if (k >= 5 && k < n - 5) {
        while (fwd < 5 && k + fwd + 1 < n && col_gap_ok(col, k + fwd + 1, k + fwd)) ++fwd;
        while (bwd < 5 && k - bwd - 1 >= 0 && col_gap_ok(col, k - bwd - 1, k - bwd)) ++bwd;
    }
    meta[k] = (unsigned char)((valid ? 1 : 0) | (fwd << 2) | (bwd << 5));
}

struct RingArgs {
    const float* __restrict__ rough;
    const unsigned char* __restrict__ meta;
    const int* __restrict__ row_start;
    const int* __restrict__ row_end;
    int n_rows;
    int n;
    float corner_thr, planar_thr;
    int lpad;      // power-of-two capacity of the sort buffer (>= longest block)
    int lcap;      // longest block + 16: capacity of the block-local visit tables
    int ring_cap;  // longest ring
    int max_rounds;  // parallel rounds per greedy pass before one thread finishes the rest in visit order
    unsigned long long* __restrict__ sorted;  // [n] per-block ascending (roughness bits << 32 | point index), written by feat_sort_kernel
    int* __restrict__ corner_out;             // [n_rows][120]
    int* __restrict__ corner_cnt;             // [n_rows]
    int* __restrict__ planar_out;             // ring r writes at planar_off[r]
    const int* __restrict__ planar_off;
    int* __restrict__ planar_cnt;
};

// K4a: the six per-ring sorts do not depend on the greedy state, so every (ring, block) sorts in its own CTA.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) feat_sort_kernel(RingArgs a) {
    extern __shared__ unsigned char smem[];
    unsigned long long* skey = reinterpret_cast<unsigned long long*>(smem);
    const int r = blockIdx.y, b = blockIdx.x;
    const int rs = a.row_start[r], re = a.row_end[r];
    const int len = (re - rs) / 6;  // C integer division (:129)
    const int bs = rs + b * len, be = rs + (b + 1) * len;
    if (bs >= be) return;
    const int L = be - bs;
    int lp = 1;
    while (lp < L) lp <<= 1;
    for (int i = threadIdx.x; i < lp; i += BLOCK)
        skey[i] = (i < L) ? (((unsigned long long)__float_as_uint(a.rough[bs + i]) << 32) | (unsigned)(bs + i)) : ~0ull;
    __syncthreads();
    for (int k = 2; k <= lp; k <<= 1) {  // bitonic sort, ascending
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < lp; i += BLOCK) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const unsigned long long x = skey[i], y = skey[ixj];
                    const bool up = ((i & k) == 0);
                    if ((x > y) == up) {
                        skey[i] = y;
                        skey[ixj] = x;
                    }
                }
            }
            __syncthreads();
        }
    }
    for (int i = threadIdx.x; i < L; i += BLOCK) a.sorted[bs + i] = skey[i];
}

enum : unsigned char { kDead = 0, kUndecided = 1, kPicked = 2 };

// exclusive prefix sum of one int per thread over the CTA; `total` = sum over all threads
template <int BLOCK>
__device__ __forceinline__ int block_excl_scan(int v, int* s_warp /*[BLOCK/32]*/, int& total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    __syncthreads();  // s_warp may still be read from a previous call
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    int base = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < BLOCK / 32; ++w) {
        const int c = s_warp[w];
        if (w < warp) base += c;
        tot += c;
    }
    total = tot;
    return base + inc - v;
}

// The greedy passes of SelectFeatures visit candidates in a fixed order and a pick only suppresses points at most 5
// positions away, so the outcome of visit v depends only on earlier visits within +-5 positions whose reach covers it.
// Every CTA round decides all visits whose earlier neighbours are decided (the parallel form of a sequential greedy
// independent set: same picks, bit for bit); a monotone roughness ramp degenerates to one decision per round, so after
// `max_rounds` one thread finishes the rest in visit order.
//   vpos[v]  ring-local position of visit v,  rank[q] visit number of block-local position q (INT_MAX: not visited),
//   stat[q]  kDead / kUndecided / kPicked,     m[]     ring-local meta bytes (reach bits are constant during a pass)
template <int BLOCK>
__device__ __forceinline__ void greedy_rounds(int nvis, const int* vpos, const int* rank, volatile unsigned char* stat, const unsigned char* m,
                                              int base_li /*ring-local position of block-local 0*/, int span, int max_rounds) {
    auto decide = [&](int v) -> int {  // kDead / kPicked / kUndecided (= wait)
        const int li = vpos[v], q0 = li - base_li;
        bool wait = false, dead = false;
#pragma unroll
        for (int d = -5; d <= 5; ++d) {
            if (d == 0) continue;
            const int q = q0 + d;
            if (q < 0 || q >= span) continue;
            if (rank[q] >= v) continue;  // not visited before v
            const unsigned char mm = m[li + d];
            const int reach = d < 0 ? ((mm >> 2) & 7) : ((mm >> 5) & 7);  // neighbour before v: its forward reach; after: backward
            if ((d < 0 ? -d : d) > reach) continue;
            const unsigned char s = stat[q];
            dead |= (s == kPicked);
            wait |= (s == kUndecided);
        }
        return dead ? kDead : (wait ? kUndecided : kPicked);
    };
    int rounds = 0;
    bool more;
    do {
        bool und = false;
        for (int v = threadIdx.x; v < nvis; v += BLOCK) {
            const int q0 = vpos[v] - base_li;
            if (stat[q0] != kUndecided) continue;
            const int s = decide(v);
            if (s == kUndecided) und = true;
            else stat[q0] = (unsigned char)s;
        }
        more = __syncthreads_or(und);
    } while (more && ++rounds < max_rounds);
    if (more) {
        if (threadIdx.x == 0)
            for (int v = 0; v < nvis; ++v) {
                const int q0 = vpos[v] - base_li;
                if (stat[q0] == kUndecided) stat[q0] = (unsigned char)decide(v);  // every earlier visit is decided by now
            }
        __syncthreads();
    }
}

__device__ __forceinline__ void suppress(unsigned char* m, int li) {
    const int fwd = (m[li] >> 2) & 7, bwd = (m[li] >> 5) & 7;
    for (int k = 1; k <= fwd; ++k) m[li + k] &= ~1;
    for (int k = 1; k <= bwd; ++k) m[li - k] &= ~1;
}

// K4b: one CTA per ring walks its six blocks in order (suppression and the inclusive `block_end` visit bleed into the
// next block [quirk 10]); inside a block everything is CTA-parallel.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) feat_ring_kernel(RingArgs a) {
    extern __shared__ unsigned char smem[];
    int* rank = reinterpret_cast<int*>(smem);                                // [lcap]
    int* vpos = rank + a.lcap;                                               // [lcap]
    unsigned char* stat = reinterpret_cast<unsigned char*>(vpos + a.lcap);  // [lcap]
    unsigned char* m = stat + a.lcap;                                        // [ring_cap]
    __shared__ int s_warp[BLOCK / 32];
    __shared__ int s_cut;
    const int r = blockIdx.x;
    const int rs = a.row_start[r], re = a.row_end[r];
    const int p0 = rs - 5;             // first point of the ring
    const int ring_len = re + 6 - p0;  // points of the ring
    int n_corner = 0, n_planar = 0;
    int* pout = a.planar_out + a.planar_off[r];
    if (ring_len > 0 && ring_len <= a.ring_cap) {
        for (int i = threadIdx.x; i < ring_len; i += BLOCK) m[i] = a.meta[p0 + i];
        const int len = (re - rs) / 6;  // C integer division (:129)
        for (int b = 0; b < 6; ++b) {
            const int bs = rs + b * len, be = rs + (b + 1) * len;
            if (bs >= be) continue;
            const int L = be - bs;
            const int base = bs - 5, span = L + 11;  // block-local window: positions bs-5 .. be+5
            const int base_li = base - p0;
            const unsigned long long* sk = a.sorted + bs;
            const float rough_be = a.rough[be];

            // ---- corner pass (:145-182): visit `be` (unsorted element of the next block), then the sorted block from the top
            // while roughness > threshold; the 21st pick ends the pass untouched.
            if (threadIdx.x == 0) s_cut = -1;
            for (int q = threadIdx.x; q < span; q += BLOCK) rank[q] = 0x7fffffff;
            __syncthreads();
            {
                int cut = -1;  // highest sorted slot that fails `roughness > threshold` — the descending walk stops there
                for (int i = threadIdx.x; i < L; i += BLOCK)
                    if (!(__uint_as_float((unsigned)(sk[i] >> 32)) > a.corner_thr)) cut = i;
                if (cut >= 0) atomicMax(&s_cut, cut);
            }
            __syncthreads();
            const int first = s_cut + 1;        // sorted slots first..L-1 are visited, top first
            const int nvis_c = 1 + (L - first);  // visit 0 is `be`
            for (int v = threadIdx.x; v < nvis_c; v += BLOCK) {
                const int idx = (v == 0) ? be : (int)(unsigned)sk[L - v];
                const float rg = (v == 0) ? rough_be : __uint_as_float((unsigned)(sk[L - v] >> 32));
                const int li = idx - p0, q = li - base_li;
                vpos[v] = li;
                rank[q] = v;
                stat[q] = (rg > a.corner_thr && (m[li] & 1)) ? kUndecided : kDead;
            }
            __syncthreads();
            greedy_rounds<BLOCK>(nvis_c, vpos, rank, stat, m, base_li, span, a.max_rounds);
            {
                const int chunk = (nvis_c + BLOCK - 1) / BLOCK;
                const int v0 = threadIdx.x * chunk, v1 = min(nvis_c, v0 + chunk);
                int cnt = 0;
                for (int v = v0; v < v1; ++v) cnt += (stat[vpos[v] - base_li] == kPicked);
                int total;
                int pr = block_excl_scan<BLOCK>(cnt, s_warp, total);
                for (int v = v0; v < v1; ++v) {
                    const int li = vpos[v], q = li - base_li;
                    if (stat[q] != kPicked) continue;
                    if (pr < 20) {
                        m[li] = (unsigned char)((m[li] | 2) & ~1);  // own byte only; neighbours are cleared after the barrier
                        a.corner_out[r * 120 + n_corner + pr] = li + p0;
                    } else {
                        stat[q] = kDead;  // beyond the limit: never picked, state untouched
                    }
                    ++pr;
                }
                n_corner += min(total, 20);
                __syncthreads();
                for (int v = v0; v < v1; ++v) {
                    const int li = vpos[v];
                    if (stat[li - base_li] == kPicked) suppress(m, li);
                }
                __syncthreads();
            }

            // ---- planar pass (:184-217): ascending through the sorted block, then `be`; every visited non-corner is emitted
            const int nvis_p = L + 1;
            for (int v = threadIdx.x; v < nvis_p; v += BLOCK) {
                const int idx = (v == L) ? be : (int)(unsigned)sk[v];
                const float rg = (v == L) ? rough_be : __uint_as_float((unsigned)(sk[v] >> 32));
                const int li = idx - p0, q = li - base_li;
                vpos[v] = li;
                rank[q] = v;
                stat[q] = ((m[li] & 1) && rg < a.planar_thr) ? kUndecided : kDead;
            }
            __syncthreads();
            greedy_rounds<BLOCK>(nvis_p, vpos, rank, stat, m, base_li, span, a.max_rounds);
            {
                const int chunk = (nvis_p + BLOCK - 1) / BLOCK;
                const int v0 = threadIdx.x * chunk, v1 = min(nvis_p, v0 + chunk);
                for (int v = v0; v < v1; ++v) {
                    const int li = vpos[v];
                    if (stat[li - base_li] == kPicked) {
                        m[li] &= ~1;
                        suppress(m, li);  // every writer clears bit 0 only: order-free
                    }
                }
                int cnt = 0;
                for (int v = v0; v < v1; ++v) cnt += !(m[vpos[v]] & 2);  // corner bits are final since the barrier above
                int total;
                int off = block_excl_scan<BLOCK>(cnt, s_warp, total);
                for (int v = v0; v < v1; ++v)
                    if (!(m[vpos[v]] & 2)) pout[n_planar + off++] = vpos[v] + p0;
                n_planar += total;
                __syncthreads();
            }
        }
    }
    if (threadIdx.x == 0) {
        a.corner_cnt[r] = n_corner;
        a.planar_cnt[r] = n_planar;
    }
}

__global__ void ring_offsets_kernel(const int* __restrict__ row_start, const int* __restrict__ row_end, int n_rows, int* __restrict__ off) {
    // capacity of ring r's planar segment: 6 * (len + 1)
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        int acc = 0;
        for (int r = 0; r < n_rows; ++r) {
            off[r] = acc;
            const int len = (row_end[r] - row_start[r]) / 6;
            acc += len > 0 ? 6 * (len + 1) : 0;
        }
        off[n_rows] = acc;
    }
}

// Exclusive scan of the 2V segment counts [corner counts of rings 0..V-1][planar counts of rings 0..V-1] (one CTA): segment g's
// records go to position off[g] of the compacted index list; totals = {n_corner, n_planar}.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) feat_scan_kernel(const int* __restrict__ cnt, int n_rows, int* __restrict__ off, int* __restrict__ totals) {
    __shared__ int s_warp[BLOCK / 32];
    const int m = 2 * n_rows;
    int carry = 0;
    for (int base = 0; base < m; base += BLOCK) {
        const int i = base + threadIdx.x;
        int total;
        const int ex = block_excl_scan<BLOCK>(i < m ? cnt[i] : 0, s_warp, total);
        if (i < m) off[i] = carry + ex;
        carry += total;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        totals[0] = off[n_rows];
        totals[1] = carry - off[n_rows];
    }
}

// Emission in upstream's order (feature_extractor.cpp:147-157 corners, :184-216 planar points; rings in order): CTA column
// g < V copies ring g's corner picks (corner_out[g*120 ..]), g >= V ring g-V's planar points (planar_out + planar_off[g-V]),
// to position off[g] of the index list and / or of its class's cloud.  blockIdx.y splits long segments.
__global__ void feat_emit_kernel(const int* __restrict__ corner_out, const int* __restrict__ planar_out, const int* __restrict__ planar_off,
                                 const int* __restrict__ cnt, const int* __restrict__ off, int n_rows, const float4* __restrict__ ordered,
                                 int* __restrict__ idx_out, float4* __restrict__ corner_cloud, float4* __restrict__ planar_cloud) {
    const int g = blockIdx.x;
    const bool corner = g < n_rows;
    const int r = corner ? g : g - n_rows;
    const int* src = corner ? corner_out + (size_t)r * 120 : planar_out + planar_off[r];
    const int c = cnt[g], o = off[g];
    float4* cloud = corner ? corner_cloud : planar_cloud;
    const int co = corner ? o : o - off[n_rows];  // planar points start at n_corner in the index list, at 0 in their cloud
    for (int k = blockIdx.y * blockDim.x + threadIdx.x; k < c; k += gridDim.y * blockDim.x) {
        const int i = src[k];
        if (idx_out) idx_out[o + k] = i;
        if (cloud) cloud[co + k] = ordered[i];
    }
}

// The kernels' dynamic shared-memory limits are per device and per function (every caller of enqueue_features holds its
// workspace lock already; raise_smem_limit's lock is taken last and alone).
void ensure_feat_smem(int device, size_t smem_sort, size_t smem_ring) {
    raise_smem_limit((const void*)feat_sort_kernel<256>, smem_sort, device);
    raise_smem_limit((const void*)feat_sort_kernel<1024>, smem_sort, device);
    raise_smem_limit((const void*)feat_ring_kernel<256>, smem_ring, device);
    raise_smem_limit((const void*)feat_ring_kernel<1024>, smem_ring, device);
}

template <int BLOCK>
void launch_feat(const RingArgs& a, size_t smem_sort, size_t smem_ring, cudaStream_t st) {
    feat_sort_kernel<BLOCK><<<dim3(6, a.n_rows), BLOCK, smem_sort, st>>>(a);
    feat_ring_kernel<BLOCK><<<a.n_rows, BLOCK, smem_ring, st>>>(a);
}

struct FeatWorkspace : Workspace {
    cudaEvent_t k0 = nullptr, k1 = nullptr;  // around the kernels (created on first use)
    DevBuf<float> d_depth;
    DevBuf<int> d_col, d_rows, d_idx;
    FeatStage s;
    PinnedBuf<int> h_out;  // [n_corner, n_planar][indices]
};

}  // namespace

int plan_features(const int* row_start, const int* row_end, int n_rows, size_t n, FeatPlan& p) {
    std::memset(&p, 0, sizeof(p));
    if (n < 12 || n_rows <= 0) return FLS_OK;
    int max_len = 0, max_ring = 0;
    long long planar_cap = 0;
    for (int r = 0; r < n_rows; ++r) {
        const int len = (row_end[r] - row_start[r]) / 6;
        if (len > max_len) max_len = len;
        const int ring = row_end[r] + 6 - (row_start[r] - 5);
        if (ring > max_ring) max_ring = ring;
        if (len > 0 && (row_start[r] < 5 || row_end[r] + 6 > (int)n)) return FLS_ERR_INVALID_ARG;
        planar_cap += len > 0 ? 6LL * (len + 1) : 0;
    }
    int lpad = 1;
    while (lpad < max_len) lpad <<= 1;
    const int lcap = max_len + 16;
    p.smem_sort = (size_t)lpad * 8;
    p.smem_ring = (size_t)lcap * 9 + (size_t)(max_ring > 0 ? max_ring : 1) + 16;
    // block or ring too long for the shared-memory working set (DESIGN.md "limits")
    if (p.smem_sort > 200 * 1024 || p.smem_ring > 200 * 1024) return FLS_ERR_UNSUPPORTED;
    p.active = true;
    p.n = (int)n;
    p.n_rows = n_rows;
    p.max_len = max_len;
    p.max_ring = max_ring;
    p.lpad = lpad;
    p.lcap = lcap;
    p.planar_cap = (size_t)planar_cap;
    return FLS_OK;
}

const int* enqueue_features(FeatStage& s, const FeatPlan& p, int device, const float* d_depth, const int* d_col, const int* d_rows, float corner_thr,
                            float planar_thr, const float4* d_ordered, int* d_idx, float4* d_corner, float4* d_planar, cudaStream_t st) {
    const int V = p.n_rows;
    const size_t n = (size_t)p.n;
    // d_out: [corner picks V*120][counts 2V][offsets 2V][planar_off V+1][totals 2][planar picks]
    const size_t o_cnt = (size_t)V * 120, o_off = o_cnt + 2 * (size_t)V, o_poff = o_off + 2 * (size_t)V, o_tot = o_poff + V + 1, o_planar = o_tot + 2;
    s.rough.reserve(n);
    s.meta.reserve(n);
    s.sorted.reserve(n);
    s.out.reserve(o_planar + p.planar_cap + 8);
    ensure_feat_smem(device, p.smem_sort, p.smem_ring);
    int* out = s.out.p;
    feat_point_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_depth, d_col, (int)n, s.rough.p, s.meta.p);
    ring_offsets_kernel<<<1, 32, 0, st>>>(d_rows, d_rows + V, V, out + o_poff);
    RingArgs a;
    a.rough = s.rough.p;
    a.meta = s.meta.p;
    a.row_start = d_rows;
    a.row_end = d_rows + V;
    a.n_rows = V;
    a.n = (int)n;
    a.corner_thr = corner_thr;
    a.planar_thr = planar_thr;
    a.lpad = p.lpad;
    a.lcap = p.lcap;
    a.ring_cap = p.max_ring;
    a.max_rounds = 96;
    if (const char* e = std::getenv("FLS_FEAT_MAX_ROUNDS")) a.max_rounds = std::atoi(e) > 0 ? std::atoi(e) : 1;
    a.sorted = s.sorted.p;
    a.corner_out = out;
    a.corner_cnt = out + o_cnt;
    a.planar_cnt = out + o_cnt + V;
    a.planar_off = out + o_poff;
    a.planar_out = out + o_planar;
    if (p.max_len > 512) launch_feat<1024>(a, p.smem_sort, p.smem_ring, st);
    else launch_feat<256>(a, p.smem_sort, p.smem_ring, st);
    feat_scan_kernel<1024><<<1, 1024, 0, st>>>(out + o_cnt, V, out + o_off, out + o_tot);
    const size_t seg_cap = std::max<size_t>(120, 6 * ((size_t)p.max_len + 1));  // longest segment a ring can emit
    const unsigned split = (unsigned)std::min<size_t>((seg_cap + 1023) / 1024, 64);
    feat_emit_kernel<<<dim3(2 * V, split), 256, 0, st>>>(out, out + o_planar, out + o_poff, out + o_cnt, out + o_off, V, d_ordered, d_idx, d_corner,
                                                         d_planar);
    FLS_CUDA(cudaGetLastError());
    return out + o_tot;
}

// Host driver of fls_extract_features.  Returns fls_status; fills corner_idx / planar_idx (host) in the reference's emission order.
int extract_features_device(int device, const float* depth, const int* col, size_t n, const int* row_start, const int* row_end, int n_rows,
                            float corner_thr, float planar_thr, int* corner_idx, size_t* n_corner, int* planar_idx, size_t* n_planar,
                            fls_match_stats* stats) {
    *n_corner = 0;
    *n_planar = 0;
    if (n < 12 || n_rows <= 0) return FLS_OK;
    FeatPlan p;
    const int prc = plan_features(row_start, row_end, n_rows, n, p);
    if (prc != FLS_OK) return prc;
    return with_workspace<FeatWorkspace>(device, [&](FeatWorkspace& w) -> int {
        if (!w.k1) {
            FLS_CUDA(cudaEventCreate(&w.k0));
            FLS_CUDA(cudaEventCreate(&w.k1));
        }
        Call& c = w.call;
        const cudaStream_t st = c.stream;
        const size_t idx_cap = (size_t)n_rows * 120 + p.planar_cap;
        w.d_depth.reserve(n);
        w.d_col.reserve(n);
        w.d_rows.reserve((size_t)n_rows * 2);
        w.d_idx.reserve(idx_cap);
        int* const h_out = w.h_out.reserve(idx_cap + 2);
        c.begin();
        FLS_CUDA(cudaMemcpyAsync(w.d_depth.p, depth, n * 4, cudaMemcpyHostToDevice, st));
        FLS_CUDA(cudaMemcpyAsync(w.d_col.p, col, n * 4, cudaMemcpyHostToDevice, st));
        FLS_CUDA(cudaMemcpyAsync(w.d_rows.p, row_start, n_rows * 4, cudaMemcpyHostToDevice, st));
        FLS_CUDA(cudaMemcpyAsync(w.d_rows.p + n_rows, row_end, n_rows * 4, cudaMemcpyHostToDevice, st));
        c.h2d += (long long)(n * 8 + (size_t)n_rows * 8);
        FLS_CUDA(cudaEventRecord(w.k0, st));
        const int* d_tot = enqueue_features(w.s, p, device, w.d_depth.p, w.d_col.p, w.d_rows.p, corner_thr, planar_thr, nullptr, w.d_idx.p, nullptr,
                                            nullptr, st);
        c.launches += kFeatLaunches;
        FLS_CUDA(cudaEventRecord(w.k1, st));
        FLS_CUDA(cudaMemcpyAsync(h_out, d_tot, 2 * sizeof(int), cudaMemcpyDeviceToHost, st));
        c.sync();  // the two counts size the read-back
        const size_t nc = (size_t)h_out[0], np = (size_t)h_out[1];
        if (nc + np) FLS_CUDA(cudaMemcpyAsync(h_out + 2, w.d_idx.p, (nc + np) * 4, cudaMemcpyDeviceToHost, st));
        c.d2h += (long long)(2 + nc + np) * 4;
        c.end(stats);
        std::memcpy(corner_idx, h_out + 2, nc * 4);
        std::memcpy(planar_idx, h_out + 2 + nc, np * 4);
        *n_corner = nc;
        *n_planar = np;
        if (stats) {
            FLS_CUDA(cudaEventElapsedTime(&stats->kernel_ms, w.k0, w.k1));
            stats->kernel_launches = kFeatLaunches;
            stats->n_source = (long long)n;
            // algorithmic bytes: depth + col in, roughness/meta/sort keys written and read once, indices out
            stats->algo_bytes = feature_algo_bytes(n, nc, np);
        }
        return FLS_OK;
    });
}

}  // namespace fls
