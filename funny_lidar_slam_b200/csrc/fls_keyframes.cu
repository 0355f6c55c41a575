// fls_keyframes.cu — the device-resident keyframe store and its map assembly (include/fls_b200.h, fls_keyframes_*).
//
// Upstream rebuilds a point map from its keyframes at three sites, all with the same primitive: for each selected keyframe
// VoxelGridCloud(cloud, leaf) -> TransformPointCloud(., pose) -> concatenate, then optionally one more VoxelGridCloud over the
// result (System::SaveMap, src/slam/system.cpp:310-316; System::VisualizeGlobalMap, :884-892; LoopClosure::GetSubMap,
// src/slam/loop_closure.cpp:217-230).  Here the per-keyframe filters of a whole selection run as ONE segmented voxel grid:
//   kf_bbox_kernel      per-segment bounding boxes (tiles of kTile points, one atomicMin / atomicMax per block and axis)
//   kf_keys_kernel      per-segment grid parameters (inv, min_b, div_b, the INT_MAX fallback) derived on the device from those boxes;
//                       key = segment << 32 | cell id (a segment that overflows keys its points by input position instead)
//   voxel-runs pass     stable radix sort of (key, arena index), run-length encode, exclusive scan (BuildScratch, CUB) — plumbing only
//   kf_centroid_kernel  one centroid per run (fp32 sums in input order), transformed by its segment's pose as it is written
// The sort is stable and the segment is the key's high half, so the output is segment-major with cells ascending inside each
// segment — the order of upstream's `+=` loop — and every centroid is summed in input order, as fls_voxelgrid.cu does (both share
// fls_voxel.cuh).  The host waits once for the run count and once at the end, plus the two waits of the final voxel_grid_device pass
// when there is one: the count does not depend on the number of keyframes.
#include <algorithm>
#include <cstring>
#include <mutex>
#include <new>
#include <vector>

#include "fls_maps.h"
#include "fls_place.h"
#include "fls_voxel.cuh"

namespace fls {
namespace {

constexpr int kThreads = 256;

struct KfSeg {                    // one keyframe of the selection (64 B)
    float rt[12];                 // R row-major, then t — cast to float on the host, as TransformPointCloud does
    unsigned long long arena_begin;
    unsigned count;
    unsigned pad;
};
struct KfTile {                   // up to kTile consecutive points of one segment (16 B)
    unsigned seg;
    unsigned local_begin;         // first point of the tile inside its segment
    unsigned long long out_begin; // its position in the concatenated selection
};

__global__ void __launch_bounds__(kThreads) kf_bbox_kernel(const float4* __restrict__ arena, const KfSeg* __restrict__ segs,
                                                           const KfTile* __restrict__ tiles, MinMaxOrd* __restrict__ mm) {
    const KfTile t = tiles[blockIdx.x];
    const unsigned long long base = segs[t.seg].arena_begin;
    const unsigned end = min(t.local_begin + (unsigned)kTile, segs[t.seg].count);
    float v[6] = {INFINITY, INFINITY, INFINITY, -INFINITY, -INFINITY, -INFINITY};
    for (unsigned j = t.local_begin + threadIdx.x; j < end; j += kThreads) {
        const float4 p = arena[base + j];
        v[0] = fminf(v[0], p.x); v[3] = fmaxf(v[3], p.x);
        v[1] = fminf(v[1], p.y); v[4] = fmaxf(v[4], p.y);
        v[2] = fminf(v[2], p.z); v[5] = fmaxf(v[5], p.z);
    }
    for (int o = 16; o > 0; o >>= 1) {
        for (int k = 0; k < 3; ++k) v[k] = fminf(v[k], __shfl_xor_sync(0xffffffffu, v[k], o));
        for (int k = 3; k < 6; ++k) v[k] = fmaxf(v[k], __shfl_xor_sync(0xffffffffu, v[k], o));
    }
    __shared__ float s[kThreads / 32][6];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0)
        for (int k = 0; k < 6; ++k) s[warp][k] = v[k];
    __syncthreads();
    if (threadIdx.x < 6) {
        const int k = threadIdx.x;
        float r = s[0][k];
        for (int w = 1; w < kThreads / 32; ++w) r = k < 3 ? fminf(r, s[w][k]) : fmaxf(r, s[w][k]);
        if (k < 3) atomicMin(&mm[t.seg].mn[k], f2ord(r));
        else atomicMax(&mm[t.seg].mx[k - 3], f2ord(r));
    }
}

__global__ void __launch_bounds__(kThreads) kf_keys_kernel(const float4* __restrict__ arena, const KfSeg* __restrict__ segs,
                                                           const KfTile* __restrict__ tiles, const MinMaxOrd* __restrict__ mm, float inv,
                                                           unsigned long long* __restrict__ keys, unsigned* __restrict__ vals) {
    const KfTile t = tiles[blockIdx.x];
    const unsigned long long base = segs[t.seg].arena_begin;
    const unsigned end = min(t.local_begin + (unsigned)kTile, segs[t.seg].count);
    const VgParams g = vg_params(mm[t.seg], inv);
    const unsigned long long hi = (unsigned long long)t.seg << 32;
    for (unsigned j = t.local_begin + threadIdx.x; j < end; j += kThreads) {
        const unsigned long long a = base + j;
        // an overflowing segment keeps its points in input order: one run per point
        const unsigned cell = g.overflow ? j : vg_cell_id(arena[a], inv, g);
        const unsigned long long o = t.out_begin + (j - t.local_begin);
        keys[o] = hi | cell;
        vals[o] = (unsigned)a;
    }
}

__global__ void kf_centroid_kernel(const float4* __restrict__ arena, const KfSeg* __restrict__ segs, const MinMaxOrd* __restrict__ mm, float inv,
                                   const unsigned long long* __restrict__ uniq, const unsigned* __restrict__ vals_sorted,
                                   const unsigned* __restrict__ starts, const unsigned* __restrict__ counts, int runs, float4* __restrict__ out) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= runs) return;
    const unsigned seg = (unsigned)(uniq[r] >> 32);
    const unsigned s = starts[r], c = counts[r];
    float4 p;
    if (vg_params(mm[seg], inv).overflow) {
        p = arena[vals_sorted[s]];  // PCL copies the input: the bits are kept (a one-point centroid would turn -0.0 into +0.0)
    } else {
        VgCentroid acc;
        for (unsigned k = 0; k < c; ++k) acc.add(__ldg(arena + vals_sorted[s + k]));
        p = acc.mean(c);
    }
    const float* q = segs[seg].rt;
    out[r] = make_float4(xform_row_f(q[0], q[1], q[2], q[9], p.x, p.y, p.z), xform_row_f(q[3], q[4], q[5], q[10], p.x, p.y, p.z),
                         xform_row_f(q[6], q[7], q[8], q[11], p.x, p.y, p.z), p.w);
}

inline size_t align16(size_t n) { return (n + 15) & ~size_t(15); }

}  // namespace

struct KeyframeStore {
    int device = 0;
    size_t capacity = 0, used = 0;
    std::mutex mu;
    Call call;
    float4* arena = nullptr;
    std::vector<unsigned long long> begin;  // per keyframe id: first arena record
    std::vector<unsigned> count;            // per keyframe id: records
    // per-call scratch
    DevBuf<unsigned char> table, raw;
    PinnedBuf<unsigned char> h_table;  // staging of the per-call table
    DevBuf<float4> cat, fin;
    BuildScratch sc;  // segmented pass (keys, keys_sorted, uniq, idx, idx_sorted, counts, starts, cub_tmp, num_runs)
    BuildScratch vg;  // final voxel_grid_device pass
    PlaceIndex place;                 // Scan Context descriptors (fls_place.cu)
    DevBuf<float4> query;             // a host scan query, uploaded
    PinnedBuf<unsigned char> h_out;   // read-back of the place entries

    KeyframeStore(int dev, size_t cap) : device(dev), capacity(cap) {
        try {
            FLS_CUDA(cudaSetDevice(device));
            FLS_CUDA(cudaStreamCreateWithFlags(&call.stream, cudaStreamNonBlocking));
            FLS_CUDA(cudaEventCreate(&call.e0));
            FLS_CUDA(cudaEventCreate(&call.e1));
            FLS_CUDA(cudaMalloc(&arena, capacity * sizeof(float4)));
        } catch (...) {
            release();
            throw;
        }
    }
    ~KeyframeStore() { release(); }
    void release() {
        h_table.release();
        h_out.release();
        if (arena) cudaFree(arena);
        if (call.e0) cudaEventDestroy(call.e0);
        if (call.e1) cudaEventDestroy(call.e1);
        if (call.stream) cudaStreamDestroy(call.stream);
        arena = nullptr;
        call.e0 = call.e1 = nullptr;
        call.stream = nullptr;
    }

    int add(long long id, const void* pts, size_t n, size_t stride, bool on_device) {
        std::lock_guard<std::mutex> lk(mu);
        if (id != (long long)count.size()) return FLS_ERR_INVALID_ARG;
        if (n > capacity - used) return FLS_ERR_CAPACITY;
        if (n) {
            FLS_CUDA(cudaSetDevice(device));
            call.begin();
            float4* dst = arena + used;
            if (on_device) {
                FLS_CUDA(cudaMemcpyAsync(dst, pts, n * sizeof(float4), cudaMemcpyDeviceToDevice, call.stream));
            } else {
                upload_records(pts, n, stride, dst, raw, call);
            }
            call.sync();
        }
        begin.push_back(used);
        count.push_back((unsigned)n);
        used += n;
        return FLS_OK;
    }

    int assemble(const int64_t* ids, size_t K, const double* T, float leaf, float final_leaf, const float4* d_base, size_t n_base, float* out,
                 float4* d_out, size_t capacity_out, size_t* n_out, fls_match_stats* stats) {
        std::lock_guard<std::mutex> lk(mu);
        for (size_t k = 0; k < K; ++k)
            if (ids[k] < 0 || ids[k] >= (int64_t)count.size()) return FLS_ERR_INVALID_ARG;
        size_t N = 0, n_tiles = 0;
        for (size_t k = 0; k < K; ++k) {
            N += count[ids[k]];
            n_tiles += (count[ids[k]] + kTile - 1) / kTile;
        }
        if (N > 0x7fffffffull) {  // CUB's item counts are int
            *n_out = 0;
            return FLS_ERR_CAPACITY;
        }
        FLS_CUDA(cudaSetDevice(device));
        const cudaStream_t stream = call.stream;
        const float inv = 1.0f / leaf;
        const bool final_pass = final_leaf > 0.f;
        call.begin();
        size_t runs = 0;
        const KfSeg* d_segs = nullptr;
        const MinMaxOrd* d_mm = nullptr;
        if (N > 0) {
            // one upload: [segments | empty bounding boxes | tiles]
            const size_t off_mm = align16(K * sizeof(KfSeg)), off_tiles = align16(off_mm + K * sizeof(MinMaxOrd));
            const size_t bytes = off_tiles + n_tiles * sizeof(KfTile);
            unsigned char* h = h_table.reserve(bytes);
            KfSeg* hs = reinterpret_cast<KfSeg*>(h);
            MinMaxOrd* hm = reinterpret_cast<MinMaxOrd*>(h + off_mm);
            KfTile* ht = reinterpret_cast<KfTile*>(h + off_tiles);
            size_t t = 0;
            unsigned long long o = 0;
            for (size_t k = 0; k < K; ++k) {
                const double* M = T + 16 * k;  // column-major: R(r,c) = M[c*4+r]
                KfSeg& sg = hs[k];
                for (int r = 0; r < 3; ++r) {
                    for (int c = 0; c < 3; ++c) sg.rt[r * 3 + c] = (float)M[c * 4 + r];
                    sg.rt[9 + r] = (float)M[12 + r];
                }
                sg.arena_begin = begin[ids[k]];
                sg.count = count[ids[k]];
                sg.pad = 0;
                for (int a = 0; a < 3; ++a) {
                    hm[k].mn[a] = 0xffffffffu;
                    hm[k].mx[a] = 0u;
                }
                for (unsigned j = 0; j < sg.count; j += kTile) ht[t++] = KfTile{(unsigned)k, j, o + j};
                o += sg.count;
            }
            table.reserve(bytes);
            FLS_CUDA(cudaMemcpyAsync(table.p, h, bytes, cudaMemcpyHostToDevice, stream));
            call.h2d += (long long)bytes;
            d_segs = reinterpret_cast<const KfSeg*>(table.p);
            MinMaxOrd* mm = reinterpret_cast<MinMaxOrd*>(table.p + off_mm);
            d_mm = mm;
            const KfTile* d_tiles = reinterpret_cast<const KfTile*>(table.p + off_tiles);

            sc.reserve_runs<unsigned long long>(N);
            kf_bbox_kernel<<<(unsigned)n_tiles, kThreads, 0, stream>>>(arena, d_segs, d_tiles, mm);
            kf_keys_kernel<<<(unsigned)n_tiles, kThreads, 0, stream>>>(arena, d_segs, d_tiles, mm, inv, sc.keys.p, sc.idx.p);
            FLS_CUDA(cudaGetLastError());
            // the cell id takes the low 32 bits, the segment the next 16 (all 32 beyond 65536 keyframes): a fixed bit range keeps the
            // sort's passes, and so the launches, the same for every selection size
            sc.sort_pairs<unsigned long long>(N, K <= 65536 ? 48 : 64, call);
            runs = (size_t)sc.encode_runs<unsigned long long>(N, call);
            call.d2h += (long long)sizeof(int);
            call.launches += 4;
        }
        const size_t R = n_base + runs;
        if (!final_pass && R > capacity_out) {
            *n_out = R;
            return FLS_ERR_CAPACITY;
        }
        // the concatenation [base | segments]: straight into the caller's device buffer when it is the result
        float4* catp = (!final_pass && d_out) ? d_out : cat.reserve(std::max<size_t>(R, 1));
        if (n_base) FLS_CUDA(cudaMemcpyAsync(catp, d_base, n_base * sizeof(float4), cudaMemcpyDeviceToDevice, stream));
        if (runs) {
            sc.run_starts((int)runs, call);
            kf_centroid_kernel<<<grid_for(runs, 128), 128, 0, stream>>>(arena, d_segs, d_mm, inv, sc.uniq.p, sc.idx_sorted.p, sc.starts.p,
                                                                        sc.counts.p, (int)runs, catp + n_base);
            FLS_CUDA(cudaGetLastError());
            call.launches += 2;
        }
        size_t m = R;
        const float4* res = catp;
        if (final_pass && R) {
            fin.reserve(R);
            m = voxel_grid_device(catp, R, final_leaf, fin.p, vg, call);
            res = fin.p;
        }
        if (m > capacity_out) {
            *n_out = m;
            return FLS_ERR_CAPACITY;
        }
        if (m && d_out && res != d_out) FLS_CUDA(cudaMemcpyAsync(d_out, res, m * sizeof(float4), cudaMemcpyDeviceToDevice, stream));
        if (m && out) {
            FLS_CUDA(cudaMemcpyAsync(out, res, m * sizeof(float4), cudaMemcpyDeviceToHost, stream));
            call.d2h += (long long)(m * sizeof(float4));
        }
        call.end(stats);
        *n_out = m;
        if (stats) {
            stats->iterations = call.waits;
            stats->n_source = (int64_t)N;
            stats->n_valid = (int64_t)runs;
        }
        return FLS_OK;
    }

    // fls_keyframes_scan_context
    int scan_context(const fls_sc_cfg& cfg, const int64_t* ids, size_t n_ids, float* desc) {
        std::lock_guard<std::mutex> lk(mu);
        for (size_t k = 0; k < n_ids; ++k)
            if (ids[k] < 0 || ids[k] >= (int64_t)count.size()) return FLS_ERR_INVALID_ARG;
        FLS_CUDA(cudaSetDevice(device));
        call.begin();
        place.describe(cfg, arena, begin, count, nullptr, 0, false, call);
        const size_t nc = place.n_cells();
        float* h = reinterpret_cast<float*>(h_out.reserve(std::max<size_t>(n_ids * nc * sizeof(float), 1)));
        for (size_t k = 0; k < n_ids; ++k)
            FLS_CUDA(cudaMemcpyAsync(h + k * nc, place.desc((size_t)ids[k]), nc * sizeof(float), cudaMemcpyDeviceToHost, call.stream));
        call.sync();
        if (n_ids) std::memcpy(desc, h, n_ids * nc * sizeof(float));
        return FLS_OK;
    }

    // fls_keyframes_detect_loop (query_id >= 0) and fls_keyframes_place_query(_device) (query_id < 0: the scan pts)
    int place_match(const fls_sc_cfg& cfg, int64_t query_id, int64_t min_span, const void* pts, size_t n, size_t stride, bool on_device, size_t k,
                    fls_place_match* out, size_t* n_found, float* query_desc, fls_match_stats* stats) {
        std::lock_guard<std::mutex> lk(mu);
        const size_t K = count.size();
        const bool scan = query_id < 0;
        if (!scan && query_id >= (int64_t)K) return FLS_ERR_INVALID_ARG;
        const size_t n_cand = scan ? K : (size_t)std::max<int64_t>(0, query_id - min_span);  // ids with query_id - id > min_span
        const size_t n_out = std::min(k, n_cand);
        FLS_CUDA(cudaSetDevice(device));
        call.begin();
        const float4* d_query = nullptr;
        if (scan && n) {
            if (on_device) {
                d_query = reinterpret_cast<const float4*>(pts);
            } else {
                query.reserve(n);
                upload_records(pts, n, stride, query.p, raw, call);
                d_query = query.p;
            }
        }
        const size_t n_read = place.describe(cfg, arena, begin, count, d_query, n, scan, call);
        const size_t q = scan ? K : (size_t)query_id, nc = place.n_cells();
        const size_t off_desc = (n_out * sizeof(fls_place_match) + 15) & ~size_t(15);
        unsigned char* h = h_out.reserve(off_desc + nc * sizeof(float));
        if (n_cand) {
            place.search(q, n_cand, n_out, reinterpret_cast<fls_place_match*>(h), call, device);
            call.d2h += (long long)(n_out * sizeof(fls_place_match));
        }
        if (query_desc) {
            FLS_CUDA(cudaMemcpyAsync(h + off_desc, place.desc(q), nc * sizeof(float), cudaMemcpyDeviceToHost, call.stream));
            call.d2h += (long long)(nc * sizeof(float));
        }
        call.end(stats);
        if (n_out) std::memcpy(out, h, n_out * sizeof(fls_place_match));
        if (query_desc) std::memcpy(query_desc, h + off_desc, nc * sizeof(float));
        *n_found = n_out;
        if (stats) {
            stats->iterations = call.waits;
            stats->n_source = (int64_t)n_read;
            stats->n_valid = (int64_t)n_cand;
        }
        return FLS_OK;
    }
};

}  // namespace fls

extern "C" {

int fls_keyframes_create(int device, size_t capacity_points, fls_keyframes** out) {
    if (!out) return FLS_ERR_INVALID_ARG;
    *out = nullptr;
    if (capacity_points == 0 || capacity_points > 0xffffffffull) return FLS_ERR_INVALID_ARG;
    if (fls::check_device(device) != FLS_OK) return FLS_ERR_NO_DEVICE;
    FLS_TRY
    *out = reinterpret_cast<fls_keyframes*>(new fls::KeyframeStore(device, capacity_points));
    return FLS_OK;
    FLS_CATCH
}

void fls_keyframes_destroy(fls_keyframes* s) {
    fls::KeyframeStore* k = reinterpret_cast<fls::KeyframeStore*>(s);
    if (!k) return;
    cudaSetDevice(k->device);
    delete k;
}

int fls_keyframes_add(fls_keyframes* s, int64_t id, const void* pts, size_t n, size_t stride_bytes) {
    if (!s || (!pts && n) || !fls::stride_ok(stride_bytes)) return FLS_ERR_INVALID_ARG;
    FLS_TRY
    return reinterpret_cast<fls::KeyframeStore*>(s)->add(id, pts, n, stride_bytes, false);
    FLS_CATCH
}

int fls_keyframes_add_device(fls_keyframes* s, int64_t id, const void* d_pts, size_t n) {
    if (!s || (!d_pts && n)) return FLS_ERR_INVALID_ARG;
    FLS_TRY
    return reinterpret_cast<fls::KeyframeStore*>(s)->add(id, d_pts, n, FLS_LAYOUT_PACKED, true);
    FLS_CATCH
}

int fls_keyframes_count(fls_keyframes* s, size_t* n_keyframes, size_t* n_points) {
    fls::KeyframeStore* k = reinterpret_cast<fls::KeyframeStore*>(s);
    if (!k) return FLS_ERR_INVALID_ARG;
    FLS_TRY
    std::lock_guard<std::mutex> lk(k->mu);
    if (n_keyframes) *n_keyframes = k->count.size();
    if (n_points) *n_points = k->used;
    return FLS_OK;
    FLS_CATCH
}

int fls_keyframes_assemble(fls_keyframes* s, const int64_t* ids, size_t n_ids, const double* T_colmajor, float leaf, float final_leaf,
                           const void* d_base, size_t n_base, float* out, float* d_out, size_t capacity, size_t* n_out, fls_match_stats* stats) {
    if (!n_out) return FLS_ERR_INVALID_ARG;
    *n_out = 0;
    if (!s || (n_ids && (!ids || !T_colmajor)) || !(leaf > 0.f) || final_leaf != final_leaf || (n_base && !d_base)) return FLS_ERR_INVALID_ARG;
    if (!out && !d_out && capacity) return FLS_ERR_INVALID_ARG;
    if (n_base && d_out) {  // the base is read while the output is written
        const uintptr_t b0 = (uintptr_t)d_base, b1 = b0 + n_base * 16, o0 = (uintptr_t)d_out, o1 = o0 + capacity * 16;
        if (b0 < o1 && o0 < b1) return FLS_ERR_INVALID_ARG;
    }
    FLS_TRY
    return reinterpret_cast<fls::KeyframeStore*>(s)->assemble(ids, n_ids, T_colmajor, leaf, final_leaf, reinterpret_cast<const float4*>(d_base),
                                                              n_base, out, reinterpret_cast<float4*>(d_out), capacity, n_out, stats);
    FLS_CATCH
}

int fls_keyframes_scan_context(fls_keyframes* s, const fls_sc_cfg* cfg, const int64_t* ids, size_t n_ids, float* desc) {
    if (!s || !cfg || !fls::sc_cfg_ok(*cfg) || (n_ids && (!ids || !desc))) return FLS_ERR_INVALID_ARG;
    FLS_TRY
    return reinterpret_cast<fls::KeyframeStore*>(s)->scan_context(*cfg, ids, n_ids, desc);
    FLS_CATCH
}

int fls_keyframes_detect_loop(fls_keyframes* s, const fls_sc_cfg* cfg, int64_t query_id, int64_t min_span, size_t k, fls_place_match* out,
                              size_t* n_found, fls_match_stats* stats) {
    if (!n_found) return FLS_ERR_INVALID_ARG;
    *n_found = 0;
    if (!s || !cfg || !fls::sc_cfg_ok(*cfg) || k < 1 || !out || query_id < 0 || min_span < 0) return FLS_ERR_INVALID_ARG;
    FLS_TRY
    return reinterpret_cast<fls::KeyframeStore*>(s)->place_match(*cfg, query_id, min_span, nullptr, 0, 0, false, k, out, n_found, nullptr, stats);
    FLS_CATCH
}

int fls_keyframes_place_query(fls_keyframes* s, const fls_sc_cfg* cfg, const void* pts, size_t n, size_t stride_bytes, size_t k,
                              fls_place_match* out, size_t* n_found, float* query_desc, fls_match_stats* stats) {
    if (!n_found) return FLS_ERR_INVALID_ARG;
    *n_found = 0;
    if (!s || !cfg || !fls::sc_cfg_ok(*cfg) || k < 1 || !out || (!pts && n) || n > 0xffffffffull || !fls::stride_ok(stride_bytes))
        return FLS_ERR_INVALID_ARG;
    FLS_TRY
    return reinterpret_cast<fls::KeyframeStore*>(s)->place_match(*cfg, -1, 0, pts, n, stride_bytes, false, k, out, n_found, query_desc, stats);
    FLS_CATCH
}

int fls_keyframes_place_query_device(fls_keyframes* s, const fls_sc_cfg* cfg, const void* d_pts, size_t n, size_t k, fls_place_match* out,
                                     size_t* n_found, float* query_desc, fls_match_stats* stats) {
    if (!n_found) return FLS_ERR_INVALID_ARG;
    *n_found = 0;
    if (!s || !cfg || !fls::sc_cfg_ok(*cfg) || k < 1 || !out || (!d_pts && n) || n > 0xffffffffull) return FLS_ERR_INVALID_ARG;
    FLS_TRY
    return reinterpret_cast<fls::KeyframeStore*>(s)->place_match(*cfg, -1, 0, d_pts, n, FLS_LAYOUT_PACKED, true, k, out, n_found, query_desc,
                                                                 stats);
    FLS_CATCH
}

}  // extern "C"
