// fls_place.cu — Scan Context on the keyframe store (include/fls_b200.h, fls_keyframes_detect_loop / _place_query): the descriptors
// of the stored keyframes, cached per keyframe, and the exact search of every candidate at every column shift.
//   sc_bin_kernel       one block per tile of kTile points of one cloud: the block bins its points into a shared copy of the cloud's
//                       cells with atomicMax on the f2ord encoding, then merges the non-empty cells into the descriptor the same way;
//                       a max is exact in any order, so the cells do not depend on the schedule
//   sc_finalize_kernel  one thread per (descriptor, column): the empty sentinel (0) becomes 0.f, f2ord values become their floats, and
//                       the column's fp64 norm is written
//   sc_search_kernel    one block per tile of candidates, staged in shared memory as fp64 with the query: one thread per (candidate,
//                       shift) evaluates d_s in the fixed order of the header (columns ascending, rings ascending), then one thread per
//                       candidate takes the first minimum over the shifts and writes the sort key of (D, id)
//   sort                stable radix sort of (key, id) (BuildScratch) — ties stay in id order
//   sc_pick_kernel      the first k records, read back in one copy
#include <algorithm>
#include <cmath>
#include <cstring>

#include "fls_atan.cuh"
#include "fls_place.h"
#include "fls_voxel.cuh"

namespace fls {
namespace {

constexpr int kThreads = 256;
constexpr double kTwoPi = 6.283185307179586476925;
constexpr double kPi = 3.141592653589793238463;
constexpr int kMaxCells = 4096;
constexpr size_t kSearchSmem = 96 * 1024;  // two blocks per SM
constexpr int kMaxSearchTile = 16;

struct ScGeom {
    int n_rings, n_sectors, n_cells;
    float z_offset;
    double R;
};
struct ScSeg {  // one cloud of a pass (16 B)
    const float4* pts;
    unsigned count;
    unsigned slot;
};
struct ScTile {  // up to kTile consecutive points of one cloud
    unsigned seg, begin;
};

// the cell of a point, or -1 when it is not binned
__device__ __forceinline__ int sc_cell(const float4 p, const ScGeom& g) {
    if (!isfinite(p.x) || !isfinite(p.y) || !isfinite(p.z)) return -1;
    const double x = p.x, y = p.y;
    const double r = __dsqrt_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)));
    if (!(r < g.R)) return -1;
    const int ring = min(g.n_rings - 1, (int)floor(__ddiv_rn(__dmul_rn(r, (double)g.n_rings), g.R)));
    double th = (double)atan2f_pinned(p.y, p.x);
    if (th < 0.0) th = __dadd_rn(th, kTwoPi);
    const int sector = min(g.n_sectors - 1, (int)floor(__ddiv_rn(__dmul_rn(th, (double)g.n_sectors), kTwoPi)));
    return ring * g.n_sectors + sector;
}

__global__ void __launch_bounds__(kThreads) sc_bin_kernel(const ScSeg* __restrict__ segs, const ScTile* __restrict__ tiles, ScGeom g,
                                                          unsigned* __restrict__ cells) {
    __shared__ unsigned s_cell[kMaxCells];
    const ScTile t = tiles[blockIdx.x];
    const ScSeg sg = segs[t.seg];
    for (int i = threadIdx.x; i < g.n_cells; i += kThreads) s_cell[i] = 0u;
    __syncthreads();
    const unsigned end = min(t.begin + (unsigned)kTile, sg.count);
    for (unsigned j = t.begin + threadIdx.x; j < end; j += kThreads) {
        const float4 p = sg.pts[j];
        const int c = sc_cell(p, g);
        if (c >= 0) atomicMax(&s_cell[c], f2ord(__fadd_rn(p.z, g.z_offset)));
    }
    __syncthreads();
    unsigned* out = cells + (size_t)sg.slot * g.n_cells;
    for (int i = threadIdx.x; i < g.n_cells; i += kThreads)
        if (s_cell[i]) atomicMax(out + i, s_cell[i]);
}

__global__ void sc_finalize_kernel(unsigned* __restrict__ cells, double* __restrict__ norms, size_t first, size_t n, ScGeom g) {
    const size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (t >= n * g.n_sectors) return;
    const size_t slot = first + t / g.n_sectors;
    const int j = (int)(t % g.n_sectors);
    unsigned* c = cells + slot * g.n_cells + j;
    double s = 0.0;
    for (int r = 0; r < g.n_rings; ++r) {
        const unsigned u = c[r * g.n_sectors];
        const float v = u ? ord2f(u) : 0.f;
        c[r * g.n_sectors] = __float_as_uint(v);
        s = __dadd_rn(s, __dmul_rn((double)v, (double)v));
    }
    norms[slot * g.n_sectors + j] = __dsqrt_rn(s);
}

// shared memory of one search block: [query norms | candidate norms | d_s | query cells | candidate cells], all fp64
__host__ __device__ inline size_t search_smem(int tile, const ScGeom& g) {
    return sizeof(double) * ((size_t)g.n_sectors * (1 + 2 * tile) + (size_t)g.n_cells * (1 + tile));
}

__global__ void __launch_bounds__(kThreads) sc_search_kernel(const float* __restrict__ desc, const double* __restrict__ norms, size_t q_slot,
                                                             unsigned n_cand, int tile, ScGeom g, unsigned long long* __restrict__ keys,
                                                             unsigned* __restrict__ ids, double* __restrict__ dist, int* __restrict__ shift) {
    extern __shared__ double smem[];
    const int S = g.n_sectors, NC = g.n_cells;
    double* qn = smem;
    double* cn = qn + S;
    double* ds = cn + (size_t)tile * S;
    double* q = ds + (size_t)tile * S;
    double* cc = q + NC;
    const unsigned c0 = blockIdx.x * (unsigned)tile;
    const int nc = (int)min((unsigned)tile, n_cand - c0);
    const float* qd = desc + q_slot * NC;
    for (int i = threadIdx.x; i < NC; i += kThreads) q[i] = (double)qd[i];
    for (int i = threadIdx.x; i < S; i += kThreads) qn[i] = norms[q_slot * S + i];
    const float* cd = desc + (size_t)c0 * NC;
    for (int i = threadIdx.x; i < nc * NC; i += kThreads) cc[i] = (double)cd[i];
    for (int i = threadIdx.x; i < nc * S; i += kThreads) cn[i] = norms[(size_t)c0 * S + i];
    __syncthreads();
    for (int it = threadIdx.x; it < nc * S; it += kThreads) {
        const int c = it / S, s = it - c * S;
        const double* C = cc + (size_t)c * NC;
        const double* Cn = cn + (size_t)c * S;
        double sum = 0.0;
        int E = 0;
        int col = s;
        for (int j = 0; j < S; ++j) {
            const double a = qn[j], b = Cn[col];
            if (a != 0.0 && b != 0.0) {
                double dot = 0.0;
                for (int r = 0; r < g.n_rings; ++r) dot = __dadd_rn(dot, __dmul_rn(q[r * S + j], C[r * S + col]));
                sum = __dadd_rn(sum, __ddiv_rn(dot, __dmul_rn(a, b)));
                ++E;
            }
            if (++col == S) col = 0;
        }
        ds[it] = E ? __dsub_rn(1.0, __ddiv_rn(sum, (double)E)) : 1.0;
    }
    __syncthreads();
    if (threadIdx.x < nc) {
        const int c = threadIdx.x;
        double best = ds[(size_t)c * S];
        int bs = 0;
        for (int s = 1; s < S; ++s)
            if (ds[(size_t)c * S + s] < best) {
                best = ds[(size_t)c * S + s];
                bs = s;
            }
        const unsigned id = c0 + c;
        const unsigned long long b = (unsigned long long)__double_as_longlong(best);
        keys[id] = (b >> 63) ? ~b : (b | 0x8000000000000000ull);  // order-preserving: a rounded cosine sum can leave D just below 0
        ids[id] = id;
        dist[id] = best;
        shift[id] = bs;
    }
}

__global__ void sc_pick_kernel(const unsigned* __restrict__ ids_sorted, const double* __restrict__ dist, const int* __restrict__ shift, int n,
                               int n_sectors, fls_place_match* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned id = ids_sorted[i];
    const int s = shift[id];
    double yaw = __dmul_rn((double)s, __ddiv_rn(kTwoPi, (double)n_sectors));
    if (yaw > kPi) yaw = __dsub_rn(yaw, kTwoPi);
    out[i] = fls_place_match{(int64_t)id, dist[id], yaw, s, 0};
}

inline size_t align16(size_t n) { return (n + 15) & ~size_t(15); }

ScGeom geom(const fls_sc_cfg& c) { return ScGeom{c.n_rings, c.n_sectors, c.n_rings * c.n_sectors, c.z_offset, (double)c.max_radius}; }

// grows b to at least `want` elements, keeping its first `keep`.  The cudaFree of the old buffer waits for the device (so also for
// the copy): a host wait outside the call's count, taken only when the cache grows.
template <class T>
void grow_keep(DevBuf<T>& b, size_t want, size_t keep, cudaStream_t st) {
    if (want <= b.cap) return;
    T* p = nullptr;
    FLS_CUDA(cudaMalloc(&p, want * sizeof(T)));
    const cudaError_t e = keep ? cudaMemcpyAsync(p, b.p, keep * sizeof(T), cudaMemcpyDeviceToDevice, st) : cudaSuccess;
    if (e != cudaSuccess) cudaFree(p);
    FLS_CUDA(e);
    b.release();
    b.p = p;
    b.cap = want;
}

}  // namespace

bool sc_cfg_ok(const fls_sc_cfg& c) {
    return c.n_rings >= 1 && c.n_rings <= 64 && c.n_sectors >= 1 && c.n_sectors <= 360 && c.n_rings * c.n_sectors <= kMaxCells &&
           std::isfinite(c.max_radius) && c.max_radius > 0.f && std::isfinite(c.z_offset);
}

size_t PlaceIndex::describe(const fls_sc_cfg& c, const float4* arena, const std::vector<unsigned long long>& begin, const std::vector<unsigned>& count,
                          const float4* d_query, size_t n_query, bool with_query, Call& call) {
    if (std::memcmp(&c, &cfg, sizeof(c)) != 0) {  // bitwise: z_offset -0.0 and +0.0 give different cells for z = -0.0
        cfg = c;
        described = 0;
    }
    const size_t K = count.size(), first = described, last = K + (with_query ? 1 : 0);
    if (first == last) return 0;
    const cudaStream_t st = call.stream;
    const size_t NC = n_cells(), S = (size_t)cfg.n_sectors;
    // descriptors the buffers hold at this cfg: they were sized for the cfg of their last growth, which may have had fewer cells
    const size_t held = std::min(cells.cap / NC, norms.cap / S);
    if (last > held) {
        const size_t want = std::max(last, std::max<size_t>(2 * held, 64));
        grow_keep(cells, want * NC, described * NC, st);
        grow_keep(norms, want * S, described * S, st);
    }
    // one upload: [segments | tiles]
    const size_t n_segs = last - first;
    size_t n_tiles = 0, n_pts = with_query ? n_query : 0;
    for (size_t k = first; k < K; ++k) {
        n_tiles += (count[k] + kTile - 1) / kTile;
        n_pts += count[k];
    }
    if (with_query) n_tiles += (n_query + kTile - 1) / kTile;
    const size_t off_tiles = align16(n_segs * sizeof(ScSeg)), bytes = off_tiles + n_tiles * sizeof(ScTile);
    const ScGeom g = geom(cfg);
    FLS_CUDA(cudaMemsetAsync(cells.p + first * NC, 0, n_segs * NC * sizeof(unsigned), st));
    ++call.launches;
    if (n_tiles) {
        unsigned char* h = h_table.reserve(bytes);
        ScSeg* hs = reinterpret_cast<ScSeg*>(h);
        ScTile* ht = reinterpret_cast<ScTile*>(h + off_tiles);
        size_t t = 0;
        for (size_t i = 0; i < n_segs; ++i) {
            const size_t slot = first + i;
            const bool q = slot == K;
            hs[i] = ScSeg{q ? d_query : arena + begin[slot], q ? (unsigned)n_query : count[slot], (unsigned)slot};
            for (unsigned j = 0; j < hs[i].count; j += kTile) ht[t++] = ScTile{(unsigned)i, j};
        }
        table.reserve(bytes);
        FLS_CUDA(cudaMemcpyAsync(table.p, h, bytes, cudaMemcpyHostToDevice, st));
        call.h2d += (long long)bytes;
        sc_bin_kernel<<<(unsigned)n_tiles, kThreads, 0, st>>>(reinterpret_cast<const ScSeg*>(table.p),
                                                               reinterpret_cast<const ScTile*>(table.p + off_tiles), g, cells.p);
        FLS_CUDA(cudaGetLastError());
        ++call.launches;
    }
    sc_finalize_kernel<<<grid_for(n_segs * S, 128), 128, 0, st>>>(cells.p, norms.p, first, n_segs, g);
    FLS_CUDA(cudaGetLastError());
    ++call.launches;
    described = K;
    return n_pts;
}

void PlaceIndex::search(size_t q, size_t n_cand, size_t n_out, fls_place_match* h_out, Call& call, int device) {
    const cudaStream_t st = call.stream;
    const ScGeom g = geom(cfg);
    const size_t base = search_smem(0, g), per = search_smem(1, g) - base;
    const int tile = (int)std::min<size_t>(kMaxSearchTile, std::max<size_t>(1, (kSearchSmem - base) / per));
    const size_t smem = search_smem(tile, g);
    raise_smem_limit((const void*)sc_search_kernel, smem, device);
    sc.reserve_runs<unsigned long long>(n_cand);
    dist.reserve(n_cand);
    shift.reserve(n_cand);
    pick.reserve(n_out);
    sc_search_kernel<<<grid_for(n_cand, tile), kThreads, smem, st>>>(desc(0), norms.p, q, (unsigned)n_cand, tile, g, sc.keys.p, sc.idx.p, dist.p,
                                                                     shift.p);
    FLS_CUDA(cudaGetLastError());
    sc.sort_pairs<unsigned long long>(n_cand, 64, call);
    sc_pick_kernel<<<grid_for(n_out, 128), 128, 0, st>>>(sc.idx_sorted.p, dist.p, shift.p, (int)n_out, cfg.n_sectors, pick.p);
    FLS_CUDA(cudaGetLastError());
    FLS_CUDA(cudaMemcpyAsync(h_out, pick.p, n_out * sizeof(fls_place_match), cudaMemcpyDeviceToHost, st));
    call.launches += 3;
}

}  // namespace fls
