// fls_p2plane_v9.cu — K1 (+ fused K6), generation 9: the LoamPointToPlaneIVOX Gauss-Newton loops of a whole batch as ONE
// persistent, barrier-free dataflow kernel whose candidate runs arrive in shared memory through the bulk-copy engine (TMA).
//
// What it computes is unchanged (include/registration/loam_point_to_plane_ivox.h:141-340, src/ivox_map/ivox_map.cpp:6-37
// upstream; see fls_p2plane.cu for the per-point arithmetic and its rounding rules).  What changed is how the machine is
// driven — ncu on the previous generation showed a latency-bound kernel (issue active 32 %, long scoreboard 40 % and CTA
// barrier 26 % of the warp time), so this one removes both stalls:
//
//   * Roles.  A CTA (one per SM: 132 on an H100 SXM) has W compute warps, one SERVER warp and one FOLDER warp; nothing in the loop
//     is a CTA-wide barrier.  Compute warps walk the same sequence of (scan, iteration) items — iteration `it` of every
//     live scan, round-robin — each at its own pace.
//   * TMA-staged candidates, double-buffered per warp.  For its NEXT 32-point chunk a warp loads the source points,
//     transforms them with that item's pose, probes the centre table and has one lane per DISTINCT candidate run issue a
//     `cp.async.bulk` (global -> shared, completion on the warp's mbarrier) into the other stage buffer; then it works on
//     the CURRENT chunk out of shared memory (LDS.128 candidate stream, neighbour gathers).  The L2 / HBM latency of the
//     run fetch is behind a whole chunk of arithmetic instead of in front of every 4-candidate loop trip.
//   * 29 sums on the fp64 tensor cores.  Each lane stages X = [J(6), |d|, valid] in the (now free) stage buffer and eight
//     DMMA m8n8k4 accumulate X X^T for the 32 points of the chunk: H, g, sum|d| and n_valid are entries of that 8x8.
//   * Hand-over.  A warp that finished its chunks of (scan, it) deposits its 32 sums in shared memory and bumps a counter;
//     the server warp adds the W deposits in warp order and publishes the CTA row as LL records (fls_gn.cuh).  The folder
//     warp of CTA (scan mod grid) collects the rows as they land (stash in shared memory, sum in row order -> bitwise
//     reproducible), runs gn_step and publishes the next pose as LL records; every server polls it into its CTA's pose
//     cache, where the compute warps find it.  With a batch in flight the hand-over of one scan is hidden behind the work
//     on the others, and no warp ever waits for another warp's chunk.
#include <cooperative_groups.h>

#include "fls_gn.cuh"
#include "fls_ivox.cuh"
#include "fls_kernels.h"
#include "fls_knn.cuh"
#include "fls_plane.cuh"

namespace fls {
namespace {

constexpr int kSlots = 8;                 // (scan, iteration) items a CTA may have open at once: scan s uses slot s mod 8
constexpr int kRegWords = 6;               // q (3), run start, run length, offset in the stage buffer
constexpr int kXStride = 9;               // doubles per staged X record (conflict-free STS.64)

__device__ __forceinline__ unsigned long long globaltimer_ns9() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// ---- watchdog: a protocol error must end the launch, never hang the device ------------------------------------------------
// Every wait loop calls this about once per microsecond of waiting; a wait of more than kWatchdogNs raises the launch's abort word
// (global memory, zeroed before the launch) and every loop of every warp leaves.  The host reports FLS_ERR_CUDA.
constexpr unsigned long long kWatchdogNs = 4000000000ull;
struct Watchdog {
    unsigned long long t0 = 0;
    unsigned n = 0;
    __device__ __forceinline__ bool expired(unsigned* abort_word) {
        if ((++n & 1023u) != 0u) return false;
        if (*reinterpret_cast<volatile unsigned*>(abort_word)) return true;
        const unsigned long long t = globaltimer_ns9();
        if (!t0) t0 = t;
        if (t - t0 > kWatchdogNs) {
            atomicExch(abort_word, 1u);
            return true;
        }
        return false;
    }
    __device__ __forceinline__ void reset() {
        t0 = 0;
        n = 0;
    }
};

// ---- shared-memory primitives (PTX) ------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(bar),
        "r"(parity)
        : "memory");
}
// bulk copy global -> shared (the TMA engine; SASS UBLKCP), completion counted in bytes on `bar`
__device__ __forceinline__ void bulk_g2s(unsigned dst, const void* src, unsigned bytes, unsigned bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ float4 lds128(unsigned addr) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ unsigned ld_acquire_smem(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.cta.shared.u32 %0, [%1];" : "=r"(v) : "r"(smem_u32(p)) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_smem(unsigned* p, unsigned v) {
    asm volatile("st.release.cta.shared.u32 [%0], %1;" ::"r"(smem_u32(p)), "r"(v) : "memory");
}
__device__ __forceinline__ void red_release_add_smem(unsigned* p, unsigned v) {
    asm volatile("red.release.cta.shared.add.u32 [%0], %1;" ::"r"(smem_u32(p)), "r"(v) : "memory");
}
// D(8x8) += A(8x4) B(4x8) in fp64 on the tensor cores; lane (r = lane/4, c = lane%4) holds A[r][c], B[c][r], D[r][2c..2c+1]
__device__ __forceinline__ void dmma884(double& d0, double& d1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};" : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}

// ---- shared-memory layout ----------------------------------------------------------------------------------------------
template <int W, int CAP>
struct V9Smem {
    static constexpr size_t o_stage = 0;                                                   // [W][2][CAP] float4
    static constexpr size_t o_dep = o_stage + (size_t)W * 2 * CAP * 16;                    // [kSlots][W][32] doubles: every warp's sums of the slot's open item
    static constexpr size_t o_pose = o_dep + sizeof(double) * kSlots * W * 32;             // [kSlots][16] doubles
    static constexpr size_t o_tot = o_pose + sizeof(double) * kSlots * 16;                 // [32] doubles (folder)
    static constexpr size_t o_pre = o_tot + sizeof(double) * 32;                           // GnPre (folder)
    static constexpr size_t o_regs = o_pre + ((sizeof(GnPre) + 15) / 16) * 16;             // [W][2][kRegWords][32] words: ChunkRegs of a prefetched chunk
    static constexpr size_t o_bar = o_regs + sizeof(unsigned) * W * 2 * kRegWords * 32;    // [W][2] mbarriers
    static constexpr size_t o_ctl = o_bar + sizeof(unsigned long long) * W * 2;            // V9Ctl
    static constexpr size_t o_desc = o_ctl + 16 * ((sizeof(unsigned) * (4 + 8 + 8 + 4 + 256) + 15) / 16);  // [n_scans] P2PlaneScan (sized at launch)
    static constexpr size_t bytes = o_desc;
};
struct V9Ctl {
    unsigned ring_head;    // next ring position to hand out (compute warps)
    unsigned ring_tail;    // positions published (server)
    unsigned quit;         // every scan is finished
    unsigned pad;
    unsigned done[kSlots];    // chunks of the slot's open item completed by this CTA
    unsigned opened[kSlots];  // (it << 8 | scan) + 1 of the latest item the server opened in the slot (monotone in pass order)
    unsigned fin_lo, fin_hi;  // scans the server has seen stop
    unsigned pad2[2];
    unsigned ring[256];       // (scan << 26) | chunk
};

// Where the (r, 2c + e) entry of the chunk's X X^T goes in the row of 32 sums (-1: not needed), and its sign.
__device__ __forceinline__ int dep_index(int r, int col) {
    if (r < 6 && col < 6) return col >= r ? tri6(r, col) : -1;
    if (r < 6 && col == 6) return 21 + r;  // g = -sum J |d|
    if (r == 6 && col == 7) return kAccRes;
    if (r == 7 && col == 7) return kAccValid;
    if (r == 7 && col == 0) return kAccCand;  // overwritten with the candidate counter at deposit time
    if (r == 7 && col == 1) return kAccHits;
    return -1;
}

// quantised top-6 scan of a candidate run; see fls_p2plane.cu knn5_stream for the semantics.
// Hot path: every lane's run sits in this warp's stage buffer (LDS.128) and the map allows the contracted distance.
// CHAINS = 2 keeps two independent selection ladders (even / odd candidates) and merges them at the end.
template <int CHAINS>
__device__ __forceinline__ bool knn_scan_hot(unsigned Ls, unsigned count, float qx, float qy, float qz, Top6q& t) {
    Top6q u;
    t.init();
    if (CHAINS == 2) u.init();
    unsigned j = 0;
#pragma unroll 1
    for (; j + 4 <= count; j += 4) {
        const float4 p0 = lds128(Ls + j * 16u), p1 = lds128(Ls + j * 16u + 16u), p2 = lds128(Ls + j * 16u + 32u), p3 = lds128(Ls + j * 16u + 48u);
        t.push((__float_as_uint(dist2_fast(p0.x, p0.y, p0.z, qx, qy, qz)) & 0xffffffc0u) | j);
        if (CHAINS == 2) u.push((__float_as_uint(dist2_fast(p1.x, p1.y, p1.z, qx, qy, qz)) & 0xffffffc0u) | (j + 1));
        else t.push((__float_as_uint(dist2_fast(p1.x, p1.y, p1.z, qx, qy, qz)) & 0xffffffc0u) | (j + 1));
        t.push((__float_as_uint(dist2_fast(p2.x, p2.y, p2.z, qx, qy, qz)) & 0xffffffc0u) | (j + 2));
        if (CHAINS == 2) u.push((__float_as_uint(dist2_fast(p3.x, p3.y, p3.z, qx, qy, qz)) & 0xffffffc0u) | (j + 3));
        else t.push((__float_as_uint(dist2_fast(p3.x, p3.y, p3.z, qx, qy, qz)) & 0xffffffc0u) | (j + 3));
    }
#pragma unroll 1
    for (; j < count; ++j) {
        const float4 p = lds128(Ls + j * 16u);
        t.push((__float_as_uint(dist2_fast(p.x, p.y, p.z, qx, qy, qz)) & 0xffffffc0u) | j);
    }
    if (CHAINS == 2) {
        t.push(u.k0); t.push(u.k1); t.push(u.k2); t.push(u.k3); t.push(u.k4); t.push(u.k5);
    }
    return ((t.k1 >> 6) - (t.k0 >> 6) <= 1u && t.k1 != 0xffffffffu) || ((t.k5 >> 6) - (t.k4 >> 6) <= 1u && t.k5 != 0xffffffffu);
}
// Everything else, out of line: `L` is a generic pointer — shared memory for the lanes whose run was staged, `lists` (global)
// for the lanes whose run did not fit the stage buffer: one loop for both, so a warp with mixed lanes does not diverge.
__device__ __noinline__ bool knn_scan_any(const float4* L, unsigned count, float r2, float qx, float qy, float qz, bool fast, Top6q& t) {
    t.init();
    unsigned j = 0;
#pragma unroll 1
    for (; j + 4 <= count; j += 4) {
        const float4 p0 = L[j], p1 = L[j + 1], p2 = L[j + 2], p3 = L[j + 3];
        if (fast) {
            t.push((__float_as_uint(dist2_fast(p0.x, p0.y, p0.z, qx, qy, qz)) & 0xffffffc0u) | j);
            t.push((__float_as_uint(dist2_fast(p1.x, p1.y, p1.z, qx, qy, qz)) & 0xffffffc0u) | (j + 1));
            t.push((__float_as_uint(dist2_fast(p2.x, p2.y, p2.z, qx, qy, qz)) & 0xffffffc0u) | (j + 2));
            t.push((__float_as_uint(dist2_fast(p3.x, p3.y, p3.z, qx, qy, qz)) & 0xffffffc0u) | (j + 3));
        } else {
            t.push(qkey(dist2_ref(p0.x, p0.y, p0.z, qx, qy, qz), r2, j));
            t.push(qkey(dist2_ref(p1.x, p1.y, p1.z, qx, qy, qz), r2, j + 1));
            t.push(qkey(dist2_ref(p2.x, p2.y, p2.z, qx, qy, qz), r2, j + 2));
            t.push(qkey(dist2_ref(p3.x, p3.y, p3.z, qx, qy, qz), r2, j + 3));
        }
    }
#pragma unroll 1
    for (; j < count; ++j) {
        const float4 p = L[j];
        if (fast) t.push((__float_as_uint(dist2_fast(p.x, p.y, p.z, qx, qy, qz)) & 0xffffffc0u) | j);
        else t.push(qkey(dist2_ref(p.x, p.y, p.z, qx, qy, qz), r2, j));
    }
    if (fast) return ((t.k1 >> 6) - (t.k0 >> 6) <= 1u && t.k1 != 0xffffffffu) || ((t.k5 >> 6) - (t.k4 >> 6) <= 1u && t.k5 != 0xffffffffu);
    return ((t.k0 >> 6) == (t.k1 >> 6) && t.k1 != 0xffffffffu) || ((t.k4 >> 6) == (t.k5 >> 6) && t.k5 != 0xffffffffu);
}

// reference comparator over a run behind a generic pointer (positions relative to the run)
__device__ __noinline__ void knn5_exact_any(const float4* L, unsigned count, float r2, float qx, float qy, float qz, Top5& nn) {
    nn.init();
#pragma unroll 1
    for (unsigned j = 0; j < count; ++j) {
        const float4 p = L[j];
        const float d = dist2_ref(p.x, p.y, p.z, qx, qy, qz);
        const bool in = d < r2;  // d < max_range^2 (voxel_grid_node.cpp:27 upstream)
        nn.push(in ? d : INFINITY, in ? j : 0xffffffffu);
    }
}

// what the prefetch stage leaves in registers for the compute stage of the same chunk
struct ChunkRegs {
    float qx, qy, qz;     // transformed with the item's pose, rounded to float (:265-266 upstream)
    unsigned start;       // candidate run in `lists` (count == 0: the point has no candidates)
    unsigned count;
    unsigned off;         // record offset of the run inside the stage buffer; 0xffffffff: not staged (read from global)
};

// The folder's solve, out of line: inlined, its arrays share stack slots with the compute warps' `J` and keep it in local
// memory.  `p` by value: a reference would take the kernel parameter's address and copy all of it to the stack.
__device__ __noinline__ void gn_step_v9(GnState* s, const GnPre& q, const double* tot, const GnParams p, fls_iter_log* log, int log_cap,
                                        uint4* ll_pose, unsigned ll_tag, double* result) {
    gn_step_pre(s, q, tot, p, log, log_cap, ll_pose, ll_tag, result);
}

// ---- the kernel ----------------------------------------------------------------------------------------------------------
constexpr int kRing = 256;  // entries of the CTA's work ring (power of two)
// refill policy of the server warp: with several scans open it keeps kRefillQuarters / 4 x W chunks drawn and not done, and the
// second-oldest open scan draws 1 / kSecondShareDiv of what the oldest does
constexpr int kRefillQuarters = 12;
constexpr int kSecondShareDiv = 4;

template <int W, int CAP>
__global__ void __launch_bounds__((W + 2) * 32, 1) p2plane_v9_kernel(P2PlaneLoopArgs a) {
    extern __shared__ __align__(128) unsigned char smem[];
    using L = V9Smem<W, CAP>;
    constexpr int kStageBytes = CAP * 16;
    double* const s_dep = reinterpret_cast<double*>(smem + L::o_dep);
    double* const s_pose = reinterpret_cast<double*>(smem + L::o_pose);
    double* const s_tot = reinterpret_cast<double*>(smem + L::o_tot);
    GnPre* const s_pre = reinterpret_cast<GnPre*>(smem + L::o_pre);
    unsigned* const s_regs = reinterpret_cast<unsigned*>(smem + L::o_regs);
    unsigned long long* const s_bar = reinterpret_cast<unsigned long long*>(smem + L::o_bar);
    V9Ctl* const ctl = reinterpret_cast<V9Ctl*>(smem + L::o_ctl);
    P2PlaneScan* const s_desc = reinterpret_cast<P2PlaneScan*>(smem + L::o_desc);

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int G = (int)gridDim.x, cta = (int)blockIdx.x;
    const int B = a.n_scans;

    for (int k = threadIdx.x; k < (int)(sizeof(V9Ctl) / 4); k += blockDim.x) reinterpret_cast<unsigned*>(ctl)[k] = 0;
    for (int k = threadIdx.x; k < kSlots * W * 32; k += blockDim.x) s_dep[k] = 0.0;
    if (threadIdx.x < W * 2) mbar_init(smem_u32(s_bar + threadIdx.x), 1);
    for (int k = threadIdx.x; k < B * (int)(sizeof(P2PlaneScan) / 8); k += blockDim.x)  // scan descriptors: read on every item
        reinterpret_cast<unsigned long long*>(s_desc)[k] = reinterpret_cast<const unsigned long long*>(a.scans)[k];
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    fence_proxy_async_smem();
    __syncthreads();  // the only CTA-wide barrier of the kernel

    if (warp < W) {
        // =============================== compute warp ======================================================================
        // Pops (scan, chunk) entries from the CTA's ring — whatever the server has queued, from whichever scan has a pose —
        // prefetches the entry after the one it is about to compute, and adds each chunk's sums to its own row of the
        // scan's slot.  It never waits for another warp: only for an empty ring.
        unsigned char* const stage_base = smem + L::o_stage + (size_t)warp * 2 * kStageBytes;
        const unsigned stage_u32 = smem_u32(stage_base);
        const unsigned bar_u32 = smem_u32(s_bar + warp * 2);
        const float r2 = a.map.max_range2;
        const bool fast = a.map.fast_knn != 0;
        // targets of this lane's two DMMA outputs in the row of 32 sums
        const int dr = lane >> 2, dc = lane & 3;
        const int dep0 = dep_index(dr, 2 * dc), dep1 = dep_index(dr, 2 * dc + 1);
        unsigned ph = 0;  // bit s: parity the next wait on stage s expects

        // ---- prefetch stage: source points, transform, table probe, one bulk copy per distinct run ----------------------
        auto prefetch = [&](unsigned entry, int stg) {
            ChunkRegs cr;
            const int s = (int)(entry >> 26), chunk = (int)(entry & 0x3ffffffu);
            const P2PlaneScan* sc = s_desc + s;
            const double* pose = s_pose + (s & (kSlots - 1)) * 16;
            const int n = sc->n;
            const int i = (chunk << 5) + lane;
            cr.count = 0;
            cr.start = 0;
            cr.off = 0xffffffffu;
            cr.qx = cr.qy = cr.qz = 0.f;
            if (i < n) {
                const float4 sp = __ldg(sc->src + i);
                cr.qx = xform_row_d(pose[0], pose[1], pose[2], pose[9], (double)sp.x, (double)sp.y, (double)sp.z);
                cr.qy = xform_row_d(pose[3], pose[4], pose[5], pose[10], (double)sp.x, (double)sp.y, (double)sp.z);
                cr.qz = xform_row_d(pose[6], pose[7], pose[8], pose[11], (double)sp.x, (double)sp.y, (double)sp.z);
                const unsigned long long key =
                    pack_key(ivox_coord(cr.qx, a.map.inv_res), ivox_coord(cr.qy, a.map.inv_res), ivox_coord(cr.qz, a.map.inv_res));
                unsigned st, cn;
                if (table_find(a.map.ctab, a.map.cmask, key, st, cn)) {
                    cr.start = st;
                    cr.count = cn;
                }
            }
            // lanes that share a run stage it once: the lowest lane of each group of equal `start` is its leader
            const bool stageable = cr.count > 0u && cr.count <= (unsigned)CAP;
            const unsigned gkey = stageable ? cr.start : (0xffffff00u | (unsigned)lane);
            const unsigned peers = __match_any_sync(0xffffffffu, gkey);
            const int leader = __ffs(peers) - 1;
            const unsigned mine = (stageable && leader == lane) ? cr.count : 0u;
            unsigned incl = mine;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned t = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += t;
            }
            const unsigned excl = incl - mine;
            const bool fits = mine > 0u && excl + mine <= (unsigned)CAP;
            const unsigned bytes = __reduce_add_sync(0xffffffffu, fits ? mine * 16u : 0u);
            const unsigned l_off = __shfl_sync(0xffffffffu, fits ? excl : 0xffffffffu, leader);
            cr.off = stageable ? l_off : 0xffffffffu;
            const unsigned bar = bar_u32 + (unsigned)stg * 8u;
            if (lane == 0) {
                if (bytes) mbar_arrive_expect_tx(bar, bytes);
                else mbar_arrive(bar);
            }
            __syncwarp();
            if (fits) bulk_g2s(stage_u32 + (unsigned)stg * kStageBytes + excl * 16u, a.map.lists + cr.start, mine * 16u, bar);
            // the chunk's registers wait in shared memory until its compute stage (keeps them out of the register file while
            // the previous chunk is being computed)
            unsigned* rg = s_regs + ((size_t)warp * 2 + stg) * kRegWords * 32 + lane;
            rg[0] = __float_as_uint(cr.qx); rg[32] = __float_as_uint(cr.qy); rg[64] = __float_as_uint(cr.qz);
            rg[96] = cr.start; rg[128] = cr.count; rg[160] = cr.off;
            // a run that is not staged (the chunk's distinct runs exceed the buffer) is at least requested into L2
            if (cr.count > 0u && cr.off == 0xffffffffu) {
                const char* pl = reinterpret_cast<const char*>(a.map.lists + cr.start);
                const unsigned nb = cr.count * 16u;
                for (unsigned o = 0; o < nb; o += 128u) asm volatile("prefetch.global.L2 [%0];" ::"l"(pl + o));
            }
        };

        // ---- compute stage ------------------------------------------------------------------------------------------------
        auto compute = [&](unsigned entry, int stg) {
            ChunkRegs cr;
            {
                const unsigned* rg = s_regs + ((size_t)warp * 2 + stg) * kRegWords * 32 + lane;
                cr.qx = __uint_as_float(rg[0]); cr.qy = __uint_as_float(rg[32]); cr.qz = __uint_as_float(rg[64]);
                cr.start = rg[96]; cr.count = rg[128]; cr.off = rg[160];
            }
            const int s = (int)(entry >> 26), chunk = (int)(entry & 0x3ffffffu);
            const int slot = s & (kSlots - 1);
            const P2PlaneScan* sc = s_desc + s;
            const double* pose = s_pose + slot * 16;
            const int n = sc->n;
            const int i = (chunk << 5) + lane;
            unsigned char* const buf = stage_base + (size_t)stg * kStageBytes;
            float4 sp = make_float4(0.f, 0.f, 0.f, 0.f);
            unsigned char was_valid = 0;
            if (i < n) {
                sp = __ldg(sc->src + i);   // the line was fetched by the prefetch stage
                // [quirk 1] asked for now, needed after the plane fit.  Chunks move between SMs from one iteration to the next
                // (dynamic tickets), so the per-point state is read from L2, never from this SM's L1
                was_valid = __ldcg(sc->flags + i);
            }
            mbar_wait(bar_u32 + (unsigned)stg * 8u, (ph >> stg) & 1u);
            ph ^= 1u << stg;
            double J[6] = {0, 0, 0, 0, 0, 0}, ad = 0.0, vflag = 0.0;
            unsigned n_fb = 0;
            // every lane's run in the stage buffer with positions that fit the 6-bit key: the scan reads it with LDS
            const bool all_staged = __all_sync(0xffffffffu, cr.count == 0u || (cr.count <= 64u && cr.off != 0xffffffffu));
            if (i < n) {
                bool use = false;
                if (cr.count > 0u) {
                    // generic pointer to the run: this warp's stage buffer when it was staged, `lists` otherwise
                    const float4* P = (cr.off != 0xffffffffu) ? reinterpret_cast<const float4*>(buf) + cr.off : a.map.lists + cr.start;
                    unsigned js[5];
                    bool full = false, exact = cr.count > 64u;
                    if (!exact) {
                        Top6q t;
                        bool amb;
                        if (all_staged && fast) {
                            const unsigned Ls = stage_u32 + (unsigned)stg * kStageBytes + cr.off * 16u;
                            amb = knn_scan_hot<1>(Ls, cr.count, cr.qx, cr.qy, cr.qz, t);
                        } else {
                            Top6q ta;  // the out-of-line scan's result goes through memory; `t` stays in registers
                            amb = knn_scan_any(P, cr.count, r2, cr.qx, cr.qy, cr.qz, fast, ta);
                            t = ta;
                        }
                        if (amb) {
                            exact = true;
                        } else {
                            full = t.k4 != 0xffffffffu;
                            js[0] = t.k0 & 63u; js[1] = t.k1 & 63u; js[2] = t.k2 & 63u; js[3] = t.k3 & 63u; js[4] = t.k4 & 63u;
                        }
                    }
                    if (exact) {  // positions that do not fit the key, or a tie the quantised keys cannot resolve: reference comparator
                        Top5 nn;
                        knn5_exact_any(P, cr.count, r2, cr.qx, cr.qy, cr.qz, nn);
                        full = nn.full();
                        js[0] = nn.k0; js[1] = nn.k1; js[2] = nn.k2; js[3] = nn.k3; js[4] = nn.k4;
                    }
                    if (full)  // fewer than 5 neighbours: skipped (:271-273)
                        use = plane_term<false>(P, js, sp, cr.qx, cr.qy, cr.qz, pose, a.plane_thres, J, ad, n_fb);
                }
                if (use) {
                    sc->rec0[i] = make_float4((float)J[0], (float)J[1], (float)J[2], (float)J[3]);
                    sc->rec1[i] = make_float4((float)J[4], (float)J[5], (float)ad, 1.0f);
                    sc->flags[i] = 1;
                } else if (was_valid) {  // stale contribution [quirk 1]
                    const float4 r0 = __ldcg(sc->rec0 + i), r1 = __ldcg(sc->rec1 + i);
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
            const unsigned cand = __reduce_add_sync(0xffffffffu, cr.count);
            const unsigned hits = __reduce_add_sync(0xffffffffu, n_fb);
            // ---- 29 sums of the chunk on the fp64 tensor cores: stage X (the candidates are no longer needed), 8 DMMA ------
            __syncwarp();
            double* const xs = reinterpret_cast<double*>(buf);
            {
                double* x = xs + lane * kXStride;
#pragma unroll
                for (int k = 0; k < 6; ++k) x[k] = J[k];
                x[6] = ad;
                x[7] = vflag;
            }
            __syncwarp();
            double d0 = 0.0, d1 = 0.0;
#pragma unroll
            for (int m = 0; m < 8; ++m) {
                const double v = xs[(4 * m + dc) * kXStride + dr];
                dmma884(d0, d1, v, v);
            }
            __syncwarp();
            fence_proxy_async_smem();  // the next bulk copy into this buffer must not pass these generic-proxy accesses
            // ---- into this warp's row of the scan's slot (nobody else writes it; the server reads it when the item closes) ---
            {
                double* dst = s_dep + ((size_t)slot * W + warp) * 32;
                if (dr < 6 && dc == 3) d0 = -d0;  // column 6: g = -sum J |d|
                if (lane == 28) {
                    d0 = (double)cand;
                    d1 = (double)hits;
                }
                if (dep0 >= 0) dst[dep0] += d0;
                if (dep1 >= 0) dst[dep1] += d1;
                __syncwarp();
                if (lane == 0) red_release_add_smem(&ctl->done[slot], 1u);
            }
        };

        // One call site per stage (they inline): the entry after the current one is reserved and — when the server has already
        // published it — prefetched before the current chunk is computed.
        unsigned cur = 0, nxt = 0, res = 0;
        int cur_stg = 0, nxt_stg = 0, pstg = 0;
        bool cur_pending = false, nxt_ready = false, have_res = false;
        for (;;) {
            if (!have_res) {  // reserve the next position of the ring (positions are handed out once: nothing is lost)
                unsigned v = 0;
                if (lane == 0) v = atomicAdd(&ctl->ring_head, 1u);
                res = __shfl_sync(0xffffffffu, v, 0);
                have_res = true;
            }
            if (!nxt_ready) {
                bool avail = (int)(ld_acquire_smem(&ctl->ring_tail) - res) > 0;
                if (!avail && !cur_pending) {  // nothing to compute meanwhile: wait for the server (or for the end)
                    unsigned ns = 32;
                    Watchdog wd;
                    for (;;) {
                        avail = (int)(ld_acquire_smem(&ctl->ring_tail) - res) > 0;
                        if (avail || ld_acquire_smem(&ctl->quit)) break;
                        if (wd.expired(a.abort_word)) break;
                        __nanosleep(ns);
                        if (ns < 256) ns <<= 1;
                    }
                    if (!avail) break;  // quit: every scan is finished
                }
                if (avail) {
                    nxt = ctl->ring[res & (kRing - 1)];
                    nxt_stg = pstg;
                    pstg ^= 1;
                    prefetch(nxt, nxt_stg);
                    nxt_ready = true;
                    have_res = false;
                }
            }
            if (cur_pending) {
                compute(cur, cur_stg);
                cur_pending = false;
            }
            if (nxt_ready) {
                cur = nxt;
                cur_stg = nxt_stg;
                cur_pending = true;
                nxt_ready = false;
            }
        }
    } else if (warp == W) {
        // =============================== server warp: the CTA's scheduler ===================================================
        // slot k serves scans k, k + 8, ... (one open item per slot).  Per slot: wait for the pose of (scan, it) -> open:
        // draw chunk tickets from the scan's global counter in small blocks and queue them on the ring while the compute
        // warps have less than ~W entries ahead -> when the counter is exhausted and every chunk this CTA drew is done: add
        // the W warp rows in warp order, publish the CTA row (LL), clear the rows -> next item of the slot.
        int rs[kSlots], rit[kSlots], rph[kSlots];  // scan, iteration, phase: 0 wait pose, 1 open, 2 dead
        unsigned acq[kSlots];                      // chunks this CTA drew for the open item
        bool exh[kSlots];                          // the item's ticket counter is exhausted
        unsigned oseq[kSlots];                     // order in which the items opened
        unsigned n_opened = 0;
        auto oseq_of = [&](int q) -> unsigned {
            unsigned v = 0;
#pragma unroll
            for (int k = 0; k < kSlots; ++k)
                if (k == q) v = oseq[k];
            return v;
        };
        unsigned long long fin = 0;
        int live = 0;
#pragma unroll
        for (int k = 0; k < kSlots; ++k) {
            rs[k] = k;
            rit[k] = 0;
            rph[k] = k < B ? 0 : 2;
            acq[k] = 0;
            exh[k] = false;
            oseq[k] = 0;
            if (k < B) ++live;
        }
        unsigned tail = 0;
        Watchdog wd;
        while (live > 0) {
            bool progress = false;
            // ---- pose records: all waiting slots polled with independent loads ---------------------------------------------
            double pv[kSlots];
            bool pok[kSlots];
#pragma unroll
            for (int k = 0; k < kSlots; ++k) {
                pv[k] = 0.0;
                pok[k] = false;
                if (rph[k] == 0) {
                    const P2PlaneScan* sc = s_desc + rs[k];
                    if (rit[k] == 0) {  // the prep kernel's state (written before this launch)
                        if (lane < 9) pv[k] = __ldcg(&sc->state->R[lane]);
                        else if (lane < 12) pv[k] = __ldcg(&sc->state->t[lane - 9]);
                        pok[k] = true;
                    } else if (lane < 13) {
                        pok[k] = ll_load(sc->ll_pose + lane, sc->tag_base | (unsigned)rit[k], pv[k]);
                    } else {
                        pok[k] = true;
                    }
                }
            }
            {
                bool any_pose = false;
#pragma unroll
                for (int k = 0; k < kSlots; ++k) any_pose = any_pose || (rph[k] == 0 && __all_sync(0xffffffffu, pok[k]));
                // acquire side of the hand-over chain: what other SMs wrote before a pose was published (per-point records) is
                // visible to this CTA's compute warps before they see the pose
                if (any_pose) __threadfence();
            }
#pragma unroll
            for (int k = 0; k < kSlots; ++k) {
                if (rph[k] != 0) continue;
                if (!__all_sync(0xffffffffu, pok[k])) continue;
                progress = true;
                const double stopv = __shfl_sync(0xffffffffu, pv[k], 12);
                const bool stop = rit[k] > 0 && stopv != 0.0;
                if (!stop) {
                    if (lane < 12) s_pose[k * 16 + lane] = pv[k];
                    __syncwarp();
                    rph[k] = 1;
                    acq[k] = 0;
                    exh[k] = false;
                    oseq[k] = n_opened++;
                    if (lane == 0) st_release_smem(&ctl->opened[k], (((unsigned)rit[k] << 8) | (unsigned)rs[k]) + 1u);
                } else {
                    // the scan is finished: the slot moves on to its next live scan (pass order: iteration-major)
                    fin |= 1ull << rs[k];
                    if (lane == 0) {
                        if (rs[k] < 32) st_release_smem(&ctl->fin_lo, (unsigned)fin);
                        else st_release_smem(&ctl->fin_hi, (unsigned)(fin >> 32));
                    }
                    bool any = false;
                    for (int s = k; s < B; s += kSlots) any = any || !((fin >> s) & 1ull);
                    if (!any) {
                        rph[k] = 2;
                        --live;
                    } else {
                        do {
                            rs[k] += kSlots;
                            if (rs[k] >= B) {
                                rs[k] = k;
                                ++rit[k];
                            }
                        } while ((fin >> rs[k]) & 1ull);
                    }
                }
            }
            // ---- refill: this CTA holds at most 2 W chunks that are drawn and not done (one being computed and one prefetched
            // per warp) — drawing more would only take work away from CTAs that run dry; lane k draws for slot k, so one
            // round trip of the atomics serves every open slot
            {
                unsigned outstanding = 0;
                int n_open = 0;
#pragma unroll
                for (int k = 0; k < kSlots; ++k) {
                    if (rph[k] == 1) outstanding += acq[k] - ld_acquire_smem(&ctl->done[k]);
                    n_open += (rph[k] == 1 && !exh[k]) ? 1 : 0;
                }
                // (with several scans in flight one more chunk per warp waits on the ring: the refill takes a server pass)
                const int target = n_open > 1 ? (kRefillQuarters * W) / 4 : 2 * W;
                if (n_open > 0 && (int)outstanding < target) {
                    const int want = target - (int)outstanding;
                    // Oldest item first: the scans of a batch start in phase, and drawing from all of them at the same rate keeps
                    // them in phase — they would all reach their hand-over together and leave the machine without work.  Served in
                    // the order they opened, the first scan's hand-over runs while the others are worked on.  The second oldest gets
                    // a quarter so that the ring does not run dry when the oldest is exhausted between two passes.
                    int k1 = -1, k2 = -1;
#pragma unroll
                    for (int k = 0; k < kSlots; ++k) {
                        if (rph[k] == 1 && !exh[k]) {
                            if (k1 < 0 || (int)(oseq[k] - oseq_of(k1)) < 0) {
                                k2 = k1;
                                k1 = k;
                            } else if (k2 < 0 || (int)(oseq[k] - oseq_of(k2)) < 0) {
                                k2 = k;
                            }
                        }
                    }
                    const int kb1 = want, kb2 = want / kSecondShareDiv > 0 ? want / kSecondShareDiv : 1;
                    int kb = 0;
                    unsigned base = 0;
                    int my_n = 0, my_s = 0;
#pragma unroll
                    for (int k = 0; k < kSlots; ++k) {
                        if (lane == k && (k == k1 || k == k2)) {
                            kb = k == k1 ? kb1 : kb2;
                            my_s = rs[k];
                            my_n = (s_desc[rs[k]].n + 31) >> 5;
                            base = atomicAdd(a.tickets + (size_t)rs[k] * a.ticket_stride + rit[k], (unsigned)kb);
                        }
                    }
                    // valid tickets of lane k's block: [base, min(base + kb, n))
                    int cnt = 0;
                    if (kb > 0 && my_n > 0) {
                        const int hi = (int)base + kb < my_n ? (int)base + kb : my_n;
                        cnt = hi > (int)base ? hi - (int)base : 0;
                    }
                    const bool now_exh = kb > 0 && (int)base + kb >= my_n;  // (kb > 0: this lane drew; an EMPTY scan is exhausted by its first draw)
                    unsigned incl = (unsigned)cnt;
#pragma unroll
                    for (int o = 1; o < kSlots; o <<= 1) {
                        const unsigned t = __shfl_up_sync(0xffffffffu, incl, o);
                        if (lane >= o) incl += t;
                    }
                    const unsigned total = __shfl_sync(0xffffffffu, incl, kSlots - 1);
                    const unsigned excl = incl - (unsigned)cnt;
                    for (int j = 0; j < cnt; ++j) {
                        ctl->ring[(tail + excl + (unsigned)j) & (kRing - 1)] = ((unsigned)my_s << 26) | (base + (unsigned)j);
                        // the source points of a queued chunk are requested into this SM's L1 now: the compute warp that pops the
                        // entry a few microseconds later finds them there (its prefetch stage executes in order and would wait)
                        const char* sp = reinterpret_cast<const char*>(s_desc[my_s].src + ((size_t)(base + (unsigned)j) << 5));
#pragma unroll
                        for (int l = 0; l < 4; ++l) asm volatile("prefetch.global.L1 [%0];" ::"l"(sp + 128 * l));
                    }
#pragma unroll
                    for (int k = 0; k < kSlots; ++k) {
                        const unsigned c = __shfl_sync(0xffffffffu, (unsigned)cnt, k);
                        const bool e = __shfl_sync(0xffffffffu, now_exh ? 1u : 0u, k) != 0u;
                        if (rph[k] == 1 && !exh[k] && (k == k1 || k == k2)) {
                            acq[k] += c;
                            if (e) exh[k] = true;
                        }
                    }
                    __syncwarp();
                    tail += total;
                    if (lane == 0) st_release_smem(&ctl->ring_tail, tail);
                    progress = progress || total > 0u;  // an empty draw is not progress (the watchdog must see a stuck item)
                }
            }
            // ---- close: counter exhausted and every chunk drawn here is done -> CTA row (warp order), LL store, rows cleared ----
            bool closing[kSlots];
            {
                bool any_close = false;
#pragma unroll
                for (int k = 0; k < kSlots; ++k) {
                    closing[k] = rph[k] == 1 && exh[k] && ld_acquire_smem(&ctl->done[k]) == acq[k];
                    any_close = any_close || closing[k];
                }
                // release side: the compute warps' per-point records of the closing items (seen through `done`) are visible
                // gpu-wide before the rows are
                if (any_close) __threadfence();
            }
#pragma unroll
            for (int k = 0; k < kSlots; ++k) {
                if (!closing[k]) continue;
                progress = true;
                const P2PlaneScan* sc = s_desc + rs[k];
                double* dep = s_dep + (size_t)k * W * 32 + lane;
                double v = 0.0;
#pragma unroll
                for (int w = 0; w < W; ++w) {
                    v += dep[w * 32];
                    dep[w * 32] = 0.0;
                }
                ll_store(sc->rows + (size_t)cta * 32 + lane, v, sc->tag_base | (unsigned)(rit[k] + 1));
                __syncwarp();
                if (lane == 0) ctl->done[k] = 0;
                // next item of the slot: its next live scan, wrapping into the next iteration
                do {
                    rs[k] += kSlots;
                    if (rs[k] >= B) {
                        rs[k] = k;
                        ++rit[k];
                    }
                } while ((fin >> rs[k]) & 1ull);
                rph[k] = 0;
            }
            if (progress) {
                wd.reset();
            } else {
                if (wd.expired(a.abort_word)) break;
                __nanosleep(64);
            }
        }
        __syncwarp();
        if (lane == 0) st_release_smem(&ctl->quit, 1u);
    } else {
        // =============================== folder warp: rows -> group rows -> totals -> gn_step -> next pose =================
        // Two-level fold (one warp has 16 loads = one L2 round trip in flight, so one warp folding every CTA row in sequence pays
        // a round trip per 16 rows):
        //   * the folder warp of every kGroup-th CTA (a group leader) adds the CTA rows of its group in CTA order and publishes
        //     a group row;
        //   * the folder warp of CTA fold_cta(scan) adds the group rows in group order, runs gn_step and publishes the next pose.
        // Fixed orders on both levels: the totals are bitwise reproducible for a given grid.  Items are visited in pass order
        // (iteration-major); whether (scan, it) exists is learnt from the server of the same CTA (`opened` / `fin`).
        constexpr int kGroup = 12;
        const int NG = (G + kGroup - 1) / kGroup;
        const bool leader = cta % kGroup == 0;
        auto fold_cta = [&](int sx) -> int { return (sx * kGroup + 1) % G; };
        bool any_mine = false;
        for (int sx = 0; sx < B; ++sx) any_mine = any_mine || fold_cta(sx) == cta;
        if (!leader && !any_mine) return;
        unsigned long long fin = 0;
        int left = B;
        Watchdog wd;
        bool aborted = false;
        for (int it = 0; left > 0 && !aborted; ++it) {
            for (int sx = 0; sx < B && left > 0 && !aborted; ++sx) {
                if ((fin >> sx) & 1ull) continue;
                const bool mine = fold_cta(sx) == cta;
                const int slot = sx & (kSlots - 1);
                const unsigned key = (((unsigned)it << 8) | (unsigned)sx) + 1u;
                bool stopped = false;
                for (;;) {  // does the item exist?
                    const unsigned f = sx < 32 ? ld_acquire_smem(&ctl->fin_lo) : ld_acquire_smem(&ctl->fin_hi);
                    if ((f >> (sx & 31)) & 1u) {
                        stopped = true;
                        break;
                    }
                    if (ld_acquire_smem(&ctl->opened[slot]) >= key) {
                        // a LATER item of the slot may be what was opened (scans k, k + 8, ... share slot k): then either this item
                        // was opened and closed before (rows exist) or the scan stopped — the server sets `fin` before it opens
                        // anything later, so a second look at `fin` tells which
                        const unsigned f2 = sx < 32 ? ld_acquire_smem(&ctl->fin_lo) : ld_acquire_smem(&ctl->fin_hi);
                        if ((f2 >> (sx & 31)) & 1u) stopped = true;
                        break;
                    }
                    if (wd.expired(a.abort_word)) {
                        aborted = true;
                        break;
                    }
                    __nanosleep(64);
                }
                if (aborted) break;
                wd.reset();
                if (stopped) {
                    fin |= 1ull << sx;
                    --left;
                    continue;
                }
                const P2PlaneScan* sc = s_desc + sx;
                const unsigned tag = sc->tag_base | (unsigned)(it + 1);
                if (leader) {  // ---- level 1: the rows of CTAs [cta, cta + kGroup) -> group row cta / kGroup
                    const uint4* const rows = sc->rows + (size_t)cta * 32 + lane;
                    const int nr = G - cta < kGroup ? G - cta : kGroup;
                    double v[kGroup];
                    for (;;) {
                        bool ok = true;
#pragma unroll
                        for (int q = 0; q < kGroup; ++q) {
                            v[q] = 0.0;
                            if (q < nr) ok = ll_load(rows + (size_t)q * 32, tag, v[q]) && ok;
                        }
                        if (__all_sync(0xffffffffu, ok)) break;
                        if (wd.expired(a.abort_word)) {
                            aborted = true;
                            break;
                        }
                        __nanosleep(64);
                    }
                    if (aborted) break;
                    wd.reset();
                    double acc = 0.0;
#pragma unroll
                    for (int q = 0; q < kGroup; ++q) acc += v[q];
                    ll_store(sc->grows + (size_t)(cta / kGroup) * 32 + lane, acc, tag);
                }
                if (mine) {  // ---- level 2: group rows -> totals -> solve
                    GnState* const state = sc->state;
                    if (lane == 0) gn_load(state, *s_pre);  // stable until gn_step below
                    const uint4* const grows = sc->grows + lane;
                    double v[16];
                    for (;;) {
                        bool ok = true;
#pragma unroll
                        for (int q = 0; q < 16; ++q) {
                            v[q] = 0.0;
                            if (q < NG) ok = ll_load(grows + (size_t)q * 32, tag, v[q]) && ok;
                        }
                        if (__all_sync(0xffffffffu, ok)) break;
                        if (wd.expired(a.abort_word)) {
                            aborted = true;
                            break;
                        }
                        __nanosleep(64);
                    }
                    if (aborted) break;
                    wd.reset();
                    double acc = 0.0;
#pragma unroll
                    for (int q = 0; q < 16; ++q) acc += v[q];
                    s_tot[lane] = acc;
                    __threadfence();  // rows in -> pose out: keeps the chain of the per-point records causal across SMs
                    __syncwarp();
                    int stop = 0;
                    if (lane == 0) {
                        gn_step_v9(state, *s_pre, s_tot, a.gp, sc->log, a.log_cap, sc->ll_pose, tag, sc->result);
                        stop = state->done;  // written by this thread just now
                    }
                    stop = __shfl_sync(0xffffffffu, stop, 0);
                    __syncwarp();
                    if (stop) {  // (the server of this CTA will see the stop word too; no need to wait for it)
                        fin |= 1ull << sx;
                        --left;
                    }
                }
            }
        }
    }
}

// 14 compute warps (+ server + folder: 512 threads) with a stage buffer of 352 candidates per warp and stage
constexpr int kV9Warps = 14, kV9Cap = 352;
constexpr size_t kV9Smem = V9Smem<kV9Warps, kV9Cap>::bytes + sizeof(P2PlaneScan) * kMaxBatch;

}  // namespace

// CTAs that serve a batch whose largest scan has n points: one per SM, fewer when there are not enough chunks to go round
int p2plane_v9_grid(int n_max, int device) {
    raise_smem_limit((const void*)p2plane_v9_kernel<kV9Warps, kV9Cap>, kV9Smem, device);
    const int W = kV9Warps;
    const int need = ((n_max + 31) / 32 + W - 1) / W;
    const int sms = device_sms(device);
    return clamp_grid(need, sms < 192 ? sms : 192);  // the second fold level holds 16 group rows of 12 CTAs
}

void launch_p2plane_v9(const P2PlaneLoopArgs& a, int grid, cudaStream_t st) {
    launch_cooperative(p2plane_v9_kernel<kV9Warps, kV9Cap>, grid, (kV9Warps + 2) * 32, kV9Smem, st, a);
}

}  // namespace fls
