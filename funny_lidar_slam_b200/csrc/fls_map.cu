// fls_map.cu — device-side construction of the point grids (iVox map IvoxMap, search grid SearchGrid): K8, batch form.
//
// IVoxMap::AddPoints (src/ivox_map/ivox_map.cpp:122-143 upstream) inserts points one by one into an
// unordered_map of std::list nodes.  Here a whole cloud is inserted at once:
//   key (Morton of round(p/res); floor(p/res) in a SearchGrid) -> stable radix sort -> gather -> run-length encode -> scan -> hash insert,
// then the iVox map materialises its per-centre stencil lists (see fls_ivox.cuh).
// The stable sort keeps insertion order inside a voxel, so the k-NN tie order matches a sequential insert.
// LRU eviction (capacity_, ivox_map.cpp:133-136) is emulated exactly: every point carries its insertion stamp, the stamp of a
// voxel's last point is its position in upstream's list, and the sequential insert of a call is simulated on the host against
// the candidates (IvoxMap::evict_lru).  window_add keeps the sliding-window local map of the ICP and kd-tree LOAM plug-ins on top
// of a SearchGrid.
// Shared with the NDT map (fls_ndt.cu): VoxelTable, the open-addressing table of every map, and LruEviction, the exact-LRU
// eviction pass around lru_simulate.
#include <cub/cub.cuh>

#include <algorithm>
#include <cstdlib>
#include <functional>
#include <queue>
#include <vector>

#include "fls_ivox.cuh"
#include "fls_maps.h"

namespace fls {

bool lru_simulate(size_t size0, size_t capacity, const std::vector<unsigned>& cand_first_touch, std::vector<unsigned> create_times,
                  std::vector<unsigned>& victims, std::vector<unsigned char>& recreated) {
    victims.clear();
    recreated.clear();
    // creation events in time order; a victim that is touched later in the call adds one (it is created again, empty)
    std::priority_queue<unsigned, std::vector<unsigned>, std::greater<unsigned>> events(std::greater<unsigned>(), std::move(create_times));
    size_t size = size0, ci = 0;
    while (!events.empty()) {
        const unsigned t = events.top();
        events.pop();
        ++size;
        if (size < capacity) continue;
        // pop_back(): the oldest voxel that has not been moved to the front by an earlier point of this call
        while (ci < cand_first_touch.size() && cand_first_touch[ci] < t) ++ci;
        if (ci >= cand_first_touch.size()) return false;
        const unsigned ft = cand_first_touch[ci];
        victims.push_back((unsigned)ci);
        recreated.push_back(ft != 0xffffffffu ? 1 : 0);
        if (ft != 0xffffffffu) events.push(ft);
        ++ci;
        --size;
    }
    return true;
}

size_t lru_candidate_bound(size_t n_vox, int n_new, int n_touched, long long capacity, size_t n_cand) {
    const long long e0 = (long long)n_vox + n_new - (capacity - 1);
    const size_t K = (size_t)(e0 > 0 ? e0 : 0) + 2 * (size_t)n_touched + 64;
    return K < n_cand ? K : n_cand;
}

int LruEviction::run(int n_cand, const unsigned* d_create, int n_create, int n_touched, size_t size0, long long capacity,
                     DevBuf<unsigned char>& cub_tmp, Call& c, const std::function<void(const unsigned*, int, unsigned*)>& write_first) {
    const cudaStream_t st = c.stream;
    stamps_sorted.reserve((size_t)n_cand + 1);
    ids_sorted.reserve((size_t)n_cand + 1);
    cub_pass(cub_tmp, [&](void* tmp, size_t& bytes) {
        return cub::DeviceRadixSort::SortPairs(tmp, bytes, stamps.p, stamps_sorted.p, ids.p, ids_sorted.p, n_cand, 0, 64, st);
    });
    const size_t K = lru_candidate_bound(size0, n_create, n_touched, capacity, (size_t)n_cand);
    first_touch.reserve(K + 1);
    write_first(ids_sorted.p, (int)K, first_touch.p);
    c.launches += 3;  // the sort counts two
    h_first.resize(K);
    h_create.resize((size_t)n_create);
    FLS_CUDA(cudaMemcpyAsync(h_first.data(), first_touch.p, sizeof(unsigned) * K, cudaMemcpyDeviceToHost, st));
    if (n_create) FLS_CUDA(cudaMemcpyAsync(h_create.data(), d_create, sizeof(unsigned) * (size_t)n_create, cudaMemcpyDeviceToHost, st));
    c.sync();
    if (!lru_simulate(size0, (size_t)capacity, h_first, h_create, h_victims, h_recreated)) return FLS_ERR_CAPACITY;
    n_victims = h_victims.size();
    n_recreated = (size_t)std::count(h_recreated.begin(), h_recreated.end(), 1);
    if (n_victims == 0) return FLS_OK;
    victims.reserve(n_victims + 1);
    recreated.reserve(n_victims + 1);
    FLS_CUDA(cudaMemcpyAsync(victims.p, h_victims.data(), sizeof(unsigned) * n_victims, cudaMemcpyHostToDevice, st));
    FLS_CUDA(cudaMemcpyAsync(recreated.p, h_recreated.data(), n_victims, cudaMemcpyHostToDevice, st));
    return FLS_OK;
}

BuildScratch::BuildScratch() {
    if (cudaMallocHost(&h_num_runs, sizeof(int)) != cudaSuccess) {  // no device / out of pinned memory: a plain allocation still works as a copy target
        cudaGetLastError();
        h_num_runs = static_cast<int*>(std::malloc(sizeof(int)));
        pinned = false;
    }
}
BuildScratch::~BuildScratch() {
    if (h_num_runs) {
        if (pinned) cudaFreeHost(h_num_runs);
        else std::free(h_num_runs);
    }
}

namespace {

// the key arrays of the voxel-runs pass by key type: unsorted, sorted, one per run
template <class K>
struct RunKeys {
    DevBuf<K>&in, &sorted, &uniq;
};
RunKeys<unsigned long long> run_keys(BuildScratch& sc, unsigned long long) { return {sc.keys, sc.keys_sorted, sc.uniq}; }
RunKeys<unsigned> run_keys(BuildScratch& sc, unsigned) { return {sc.k32a, sc.k32b, sc.uniq32}; }
template <class K>
auto encode_pass(BuildScratch& sc, int n, cudaStream_t st) {
    return [&sc, n, st](void* tmp, size_t& bytes) {
        const RunKeys<K> k = run_keys(sc, K());
        return cub::DeviceRunLengthEncode::Encode(tmp, bytes, k.sorted.p, k.uniq.p, sc.counts.p, sc.num_runs.p, n, st);
    };
}
auto starts_pass(BuildScratch& sc, int n, cudaStream_t st) {
    return [&sc, n, st](void* tmp, size_t& bytes) { return cub::DeviceScan::ExclusiveSum(tmp, bytes, sc.counts.p, sc.starts.p, n, st); };
}

}  // namespace

template <class K>
void BuildScratch::reserve_runs(size_t n) {
    const RunKeys<K> k = run_keys(*this, K());
    k.in.reserve(n);
    k.sorted.reserve(n);
    k.uniq.reserve(n);
    idx.reserve(n);
    idx_sorted.reserve(n);
    counts.reserve(n);
    starts.reserve(n);
    num_runs.reserve(2);
}

template <class K>
void BuildScratch::sort_pairs(size_t n, int end_bit, Call& c) {
    const cudaStream_t st = c.stream;
    const RunKeys<K> k = run_keys(*this, K());
    auto sort = [&](void* tmp, size_t& bytes) {
        return cub::DeviceRadixSort::SortPairs(tmp, bytes, k.in.p, k.sorted.p, idx.p, idx_sorted.p, (int)n, 0, end_bit, st);
    };
    cub_reserve(cub_tmp, sort, encode_pass<K>(*this, (int)n, st), starts_pass(*this, (int)n, st));
    cub_run(cub_tmp, sort);
}

template <class K>
int BuildScratch::encode_runs(size_t n, Call& c) {
    cub_run(cub_tmp, encode_pass<K>(*this, (int)n, c.stream));
    FLS_CUDA(cudaMemcpyAsync(h_num_runs, num_runs.p, sizeof(int), cudaMemcpyDeviceToHost, c.stream));
    c.sync();
    return *h_num_runs;
}

void BuildScratch::run_starts(int runs, Call& c) { cub_run(cub_tmp, starts_pass(*this, runs, c.stream)); }

template void BuildScratch::reserve_runs<unsigned long long>(size_t);
template void BuildScratch::reserve_runs<unsigned>(size_t);
template void BuildScratch::sort_pairs<unsigned long long>(size_t, int, Call&);
template void BuildScratch::sort_pairs<unsigned>(size_t, int, Call&);
template int BuildScratch::encode_runs<unsigned long long>(size_t, Call&);
template int BuildScratch::encode_runs<unsigned>(size_t, Call&);

namespace {

// Morton keys of the voxels of round(p * inv_res) (iVox) or floor(p * inv_res) (search grid)
template <bool kFloor>
__global__ void voxel_keys_kernel(const float4* __restrict__ pts, size_t n, float inv_res, unsigned long long* __restrict__ keys,
                                  unsigned* __restrict__ idx) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 p = pts[i];
    keys[i] = kFloor ? morton_key(floor_coord(p.x, inv_res), floor_coord(p.y, inv_res), floor_coord(p.z, inv_res))
                     : morton_key(ivox_coord(p.x, inv_res), ivox_coord(p.y, inv_res), ivox_coord(p.z, inv_res));
    idx[i] = (unsigned)i;
}

__global__ void gather_kernel(const float4* __restrict__ src, const unsigned* __restrict__ idx, size_t n, float4* __restrict__ dst) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i < n) dst[i] = src[idx[i]];
}

__global__ void table_clear_kernel(HashSlot* tab, size_t slots) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i < slots) {
        tab[i].key = kEmptyKey;
        tab[i].start = 0;
        tab[i].count = 0;
    }
}

__device__ __forceinline__ void table_insert(HashSlot* tab, unsigned mask, unsigned long long key, unsigned start, unsigned count) {
    bool created;
    HashSlot& slot = tab[table_claim(tab, mask, key, created)];
    slot.start = start;
    slot.count = count;
}

// one thread per occupied voxel (run of equal Morton codes)
__global__ void ivox_insert_kernel(const unsigned long long* __restrict__ run_morton, const unsigned* __restrict__ starts,
                                   const unsigned* __restrict__ counts, int n_runs, HashSlot* tab, unsigned mask) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= n_runs) return;
    int x, y, z;
    morton_decode(run_morton[v], x, y, z);
    table_insert(tab, mask, pack_key(x, y, z), starts[v], counts[v]);
}

// ---- LRU bookkeeping (ivox_map.cpp:122-143) ----------------------------------------------------------------------------
__global__ void ivox_stamp_kernel(unsigned long long* __restrict__ stamps, size_t n, unsigned long long call_hi) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i < n) stamps[i] = call_hi | (unsigned long long)i;
}
// per voxel of the sorted order (old points first inside a voxel: the sort is stable and the new points have the highest
// indices): how many points it held before the call, the stamp of the last of them (its LRU position), the first point of this
// call that touches it.  cnt[0] candidates (voxels that existed), cnt[1] creations, cnt[2] existing voxels touched by the call.
__global__ void ivox_run_info_kernel(int runs, const unsigned* __restrict__ starts, const unsigned* __restrict__ counts,
                                     const unsigned* __restrict__ idx_sorted, const unsigned long long* __restrict__ stamp_all, unsigned n_old,
                                     unsigned* __restrict__ nold_out, unsigned* __restrict__ first_out, unsigned long long* __restrict__ cand_stamp,
                                     unsigned* __restrict__ cand_run, unsigned* __restrict__ create_times, int* cnt) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= runs) return;
    const unsigned s = starts[r], c = counts[r];
    unsigned lo = 0, hi = c;  // first position whose point is new
    while (lo < hi) {
        const unsigned mid = (lo + hi) >> 1;
        if (idx_sorted[s + mid] < n_old) lo = mid + 1;
        else hi = mid;
    }
    const unsigned first = lo < c ? idx_sorted[s + lo] - n_old : 0xffffffffu;
    nold_out[r] = lo;
    first_out[r] = first;
    if (lo > 0) {
        const int pos = atomicAdd(cnt, 1);
        cand_stamp[pos] = stamp_all[idx_sorted[s + lo - 1]];
        cand_run[pos] = (unsigned)r;
        if (lo < c) atomicAdd(cnt + 2, 1);
    } else {
        create_times[atomicAdd(cnt + 1, 1)] = first;
    }
}
__global__ void ivox_cand_kernel(const unsigned* __restrict__ runs_sorted, int K, const unsigned* __restrict__ first, unsigned* __restrict__ out) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < K) out[k] = first[runs_sorted[k]];
}
// one warp per victim: its points from before the call are dropped
__global__ void ivox_kill_kernel(const unsigned* __restrict__ victim_pos, int n_victims, const unsigned* __restrict__ runs_sorted,
                                 const unsigned* __restrict__ starts, const unsigned* __restrict__ nold, const unsigned* __restrict__ idx_sorted,
                                 unsigned char* __restrict__ keep) {
    const int v = (int)((blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (v >= n_victims) return;
    const unsigned r = runs_sorted[victim_pos[v]];
    const unsigned s = starts[r], m = nold[r];
    for (unsigned k = lane; k < m; k += 32) keep[idx_sorted[s + k]] = 0;
}
__global__ void table_dump_kernel(const HashSlot* __restrict__ tab, size_t slots, unsigned long long* __restrict__ out, int* cursor) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i < slots && tab[i].key != kEmptyKey) out[atomicAdd(cursor, 1)] = tab[i].key;
}

// ---- stencil lists ---------------------------------------------------------------------------------------------------
__global__ void center_keys_kernel(const unsigned long long* __restrict__ run_morton, int n_runs, int n_stencil,
                                   unsigned long long* __restrict__ out) {
    const size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (t >= (size_t)n_runs * n_stencil) return;
    const int v = (int)(t / n_stencil), s = (int)(t % n_stencil);
    int x, y, z;
    morton_decode(run_morton[v], x, y, z);
    // the stencil is symmetric: voxel v is in the stencil of centre c  <=>  c = v - offset
    out[t] = morton_key(x - c_stencil[s][0], y - c_stencil[s][1], z - c_stencil[s][2]);
}

__global__ void list_count_kernel(const unsigned long long* __restrict__ centers, int n_centers, int n_stencil, const HashSlot* __restrict__ tab,
                                  unsigned mask, unsigned* __restrict__ ccount) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n_centers) return;
    int x, y, z;
    morton_decode(centers[c], x, y, z);
    unsigned tot = 0;
    for (int s = 0; s < n_stencil; ++s) {
        unsigned st, cnt;
        if (table_find(tab, mask, pack_key(x + c_stencil[s][0], y + c_stencil[s][1], z + c_stencil[s][2]), st, cnt)) tot += cnt;
    }
    ccount[c] = tot;
}

// one warp per centre: concatenate the points of its stencil voxels in visit order; lane 0 publishes the centre slot
__global__ void list_fill_kernel(const unsigned long long* __restrict__ centers, int n_centers, int n_stencil, const HashSlot* __restrict__ tab,
                                 unsigned mask, const float4* __restrict__ pts, const unsigned* __restrict__ cstart,
                                 const unsigned* __restrict__ ccount, float4* __restrict__ lists, HashSlot* ctab, unsigned cmask) {
    const int c = (int)((blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (c >= n_centers) return;
    int x, y, z;
    morton_decode(centers[c], x, y, z);
    unsigned off = cstart[c];
    for (int s = 0; s < n_stencil; ++s) {
        unsigned st, cnt;
        if (!table_find(tab, mask, pack_key(x + c_stencil[s][0], y + c_stencil[s][1], z + c_stencil[s][2]), st, cnt)) continue;
        for (unsigned k = lane; k < cnt; k += 32) lists[off + k] = pts[st + k];
        off += cnt;
    }
    if (lane == 0) table_insert(ctab, cmask, pack_key(x, y, z), cstart[c], ccount[c]);
}

// ---- incremental insertion (log-structured): touched voxels and the centres around them are rewritten at the end of the arrays ----
// per touched voxel (run of the NEW points): where it lives now, how long it becomes
__global__ void inc_plan_kernel(const unsigned long long* __restrict__ run_morton, const unsigned* __restrict__ add_counts, int n_runs,
                                const HashSlot* __restrict__ tab, unsigned mask, unsigned* __restrict__ old_start, unsigned* __restrict__ old_count,
                                unsigned* __restrict__ new_count, int* n_created) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= n_runs) return;
    int x, y, z;
    morton_decode(run_morton[v], x, y, z);
    unsigned st = 0, cnt = 0;
    if (!table_find(tab, mask, pack_key(x, y, z), st, cnt)) {
        cnt = 0;
        atomicAdd(n_created, 1);
    }
    old_start[v] = st;
    old_count[v] = cnt;
    new_count[v] = cnt + add_counts[v];
}
// one warp per touched voxel: its old points, then the new ones in input order, move to the end of the point array
__global__ void inc_move_kernel(const unsigned long long* __restrict__ run_morton, int n_runs, const unsigned* __restrict__ old_start,
                                const unsigned* __restrict__ old_count, const unsigned* __restrict__ add_start, const unsigned* __restrict__ add_count,
                                const unsigned* __restrict__ new_off, unsigned base, const unsigned* __restrict__ idx_sorted,
                                const float4* __restrict__ pts_new, float4* __restrict__ pts, HashSlot* tab, unsigned mask) {
    const int v = (int)((blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (v >= n_runs) return;
    const unsigned dst = base + new_off[v], oc = old_count[v], os = old_start[v], ac = add_count[v], as = add_start[v];
    for (unsigned k = lane; k < oc; k += 32) pts[dst + k] = pts[os + k];
    for (unsigned k = lane; k < ac; k += 32) pts[dst + oc + k] = pts_new[idx_sorted[as + k]];
    if (lane == 0) {
        int x, y, z;
        morton_decode(run_morton[v], x, y, z);
        table_insert(tab, mask, pack_key(x, y, z), dst, oc + ac);
    }
}
__global__ void add_base_kernel(unsigned* __restrict__ a, int n, unsigned base) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) a[i] += base;
}
// how many of the affected centres are not in the centre table yet
__global__ void inc_new_centres_kernel(const unsigned long long* __restrict__ centers, int n, const HashSlot* __restrict__ ctab, unsigned cmask,
                                       const unsigned* __restrict__ ccount, int* counters /*[0] new centres, [1..2] old list records (u64)*/) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n) return;
    int x, y, z;
    morton_decode(centers[c], x, y, z);
    unsigned st, cnt;
    if (!table_find(ctab, cmask, pack_key(x, y, z), st, cnt)) atomicAdd(counters, 1);
    else atomicAdd(reinterpret_cast<unsigned long long*>(counters + 2), (unsigned long long)cnt);
}

__global__ void repack_kernel(const unsigned char* __restrict__ raw, size_t n, size_t stride, float4* __restrict__ out) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* f = reinterpret_cast<const float*>(raw + i * stride);
    float4 p;
    p.x = f[0];
    p.y = f[1];
    p.z = f[2];
    p.w = f[4];  // pcl::PointXYZI keeps intensity at byte 16
    out[i] = p;
}

__global__ void transform_f_kernel(const float4* __restrict__ in, size_t n, float r0, float r1, float r2, float r3, float r4, float r5, float r6,
                                   float r7, float r8, float t0, float t1, float t2, float4* __restrict__ out) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 p = in[i];
    out[i] = make_float4(xform_row_f(r0, r1, r2, t0, p.x, p.y, p.z), xform_row_f(r3, r4, r5, t1, p.x, p.y, p.z),
                         xform_row_f(r6, r7, r8, t2, p.x, p.y, p.z), p.w);
}

// pcl::transformPoint / pcl::transformPointCloud with a double transform: fp64 R·p + t, stored back as fp32
__global__ void transform_d_kernel(const float4* __restrict__ in, size_t n, double r0, double r1, double r2, double r3, double r4, double r5,
                                   double r6, double r7, double r8, double t0, double t1, double t2, float4* __restrict__ out) {
    const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 p = in[i];
    out[i] = make_float4(xform_row_d(r0, r1, r2, t0, (double)p.x, (double)p.y, (double)p.z),
                         xform_row_d(r3, r4, r5, t1, (double)p.x, (double)p.y, (double)p.z),
                         xform_row_d(r6, r7, r8, t2, (double)p.x, (double)p.y, (double)p.z), p.w);
}

}  // namespace

void launch_transform_d(const float4* d_in, size_t n, const double* T, float4* d_out, cudaStream_t st) {
    if (n == 0) return;
    transform_d_kernel<<<grid_for(n, 256), 256, 0, st>>>(d_in, n, T[0], T[4], T[8], T[1], T[5], T[9], T[2], T[6], T[10], T[12], T[13], T[14], d_out);
}

static void launch_repack(const unsigned char* d_raw, size_t n, size_t stride, float4* d_out, cudaStream_t st) {
    if (n == 0) return;
    repack_kernel<<<grid_for(n, 256), 256, 0, st>>>(d_raw, n, stride, d_out);
}

void upload_records(const void* pts, size_t n, size_t stride, float4* dst, DevBuf<unsigned char>& staging, Call& c) {
    if (n == 0) return;
    const cudaStream_t st = c.stream;
    if (stride == FLS_LAYOUT_PACKED) {
        FLS_CUDA(cudaMemcpyAsync(dst, pts, n * 16, cudaMemcpyHostToDevice, st));
    } else {
        staging.reserve(n * stride);  // stream order: the previous repack out of `staging` has run before this copy lands
        FLS_CUDA(cudaMemcpyAsync(staging.p, pts, n * stride, cudaMemcpyHostToDevice, st));
        launch_repack(staging.p, n, stride, dst, st);
        FLS_CUDA(cudaGetLastError());
        ++c.launches;
    }
    c.h2d += (long long)(n * stride);
}

void launch_transform_f(const float4* d_in, size_t n, const double* T, float4* d_out, cudaStream_t st) {
    if (n == 0) return;
    // T column-major: R(r,c) = T[c*4+r]
    transform_f_kernel<<<grid_for(n, 256), 256, 0, st>>>(d_in, n, (float)T[0], (float)T[4], (float)T[8], (float)T[1], (float)T[5], (float)T[9],
                                                        (float)T[2], (float)T[6], (float)T[10], (float)T[12], (float)T[13], (float)T[14], d_out);
}

// The build steps IvoxMap and SearchGrid share.  keys -> stable sort -> gather into dst (room for n) -> run-length encode ->
// starts: the n points at pts in voxel-contiguous order; returns the voxel count.
template <bool kFloor>
static int sorted_runs(const float4* pts, size_t n, float inv_res, float4* dst, BuildScratch& sc, Call& c) {
    sc.reserve_runs<unsigned long long>(n);
    voxel_keys_kernel<kFloor><<<grid_for(n, 256), 256, 0, c.stream>>>(pts, n, inv_res, sc.keys.p, sc.idx.p);
    sc.sort_pairs<unsigned long long>(n, 63, c);
    gather_kernel<<<grid_for(n, 256), 256, 0, c.stream>>>(pts, sc.idx_sorted.p, n, dst);
    const int runs = sc.encode_runs<unsigned long long>(n, c);
    sc.run_starts(runs, c);
    c.launches += 6;
    return runs;
}

void VoxelTable::size_for(size_t n, size_t factor, bool grow_only) {
    size_t want = 1024;
    while (want < factor * n) want <<= 1;
    if (!grow_only || want > slots) slots = want;
    buf.reserve(slots);
    mask = (unsigned)(slots - 1);
}

void VoxelTable::clear(Call& c) {
    table_clear_kernel<<<grid_for(slots, 256), 256, 0, c.stream>>>(buf.p, slots);
    FLS_CUDA(cudaGetLastError());
    ++c.launches;
}

// the table (sized) over the runs of sorted_runs
static void fill_table(VoxelTable& table, int runs, const BuildScratch& sc, Call& c) {
    table.clear(c);
    ivox_insert_kernel<<<grid_for(runs, 256), 256, 0, c.stream>>>(sc.uniq.p, sc.starts.p, sc.counts.p, runs, table.buf.p, table.mask);
    FLS_CUDA(cudaGetLastError());
    c.launches += 1;
}

int SearchGrid::build(const float4* d_cloud, size_t n, BuildScratch& sc, Call& c) {
    n_pts = n_vox = 0;
    if (n == 0) return FLS_OK;
    if (n > 0xfffffff0ull) return FLS_ERR_INVALID_ARG;
    pts_sorted.reserve(n);
    const int runs = sorted_runs<true>(d_cloud, n, 1.0f / res, pts_sorted.p, sc, c);
    table.size_for((size_t)runs, 2);
    fill_table(table, runs, sc, c);
    n_pts = n;
    n_vox = (size_t)runs;
    return FLS_OK;
}

// Incremental insert (mapping mode): cost proportional to the inserted points and the centres around the voxels they touch
// (<= n_stencil per voxel), not to the map.  Touched voxels are rewritten — old points, then the new ones in input order — at the
// end of the point array and their table slots redirected; every centre whose stencil contains a touched voxel gets a fresh run
// at the end of `lists` (same visit order as a full build: stencil order, insertion order inside a voxel) and its centre slot
// redirected.  The space left behind is garbage until the next full build, which happens when the slack runs out, when a table
// would exceed its load factor, when the garbage outweighs the live data, or when the LRU has to evict.
// Returns 1 when the caller has to take the full path instead.
int IvoxMap::append_incremental(const float4* d_new, size_t n_new, long long capacity, Call& c) {
    if (!incremental || n_pts == 0 || n_new == 0) return 1;
    const cudaStream_t st = c.stream;
    BuildScratch& sc = scratch;
    const size_t S = (size_t)n_stencil;
    // new points -> voxel runs (stable: input order inside a voxel)
    sc.reserve_runs<unsigned long long>(n_new);
    sc.num_runs.reserve(4);
    voxel_keys_kernel<false><<<grid_for(n_new, 256), 256, 0, st>>>(d_new, n_new, inv_res, sc.keys.p, sc.idx.p);
    sc.sort_pairs<unsigned long long>(n_new, 63, c);
    const int T = sc.encode_runs<unsigned long long>(n_new, c);  // touched voxels
    sc.run_starts(T, c);
    // plan: old location / length of every touched voxel, how many are created
    inc_old_start.reserve((size_t)T + 1);
    inc_old_count.reserve((size_t)T + 1);
    inc_new_count.reserve((size_t)T + 1);
    inc_new_off.reserve((size_t)T + 1);
    inc_cnt.reserve(8);
    FLS_CUDA(cudaMemsetAsync(inc_cnt.p, 0, 8 * sizeof(int), st));
    inc_plan_kernel<<<grid_for((size_t)T, 256), 256, 0, st>>>(sc.uniq.p, sc.counts.p, T, table.buf.p, table.mask, inc_old_start.p, inc_old_count.p,
                                                            inc_new_count.p, inc_cnt.p);
    // sized by sort_pairs: the same scan over n_new >= T items
    cub_run(sc.cub_tmp, [&](void* tmp, size_t& bytes) { return cub::DeviceScan::ExclusiveSum(tmp, bytes, inc_new_count.p, inc_new_off.p, T, st); });
    // affected centres: every centre whose stencil contains a touched voxel
    const size_t n_keys = (size_t)T * S;
    ckeys.reserve(n_keys);
    ckeys_sorted.reserve(n_keys);
    cuniq.reserve(n_keys);
    center_keys_kernel<<<grid_for(n_keys, 256), 256, 0, st>>>(sc.uniq.p, T, n_stencil, ckeys.p);
    auto sort = [&](void* tmp, size_t& bytes) { return cub::DeviceRadixSort::SortKeys(tmp, bytes, ckeys.p, ckeys_sorted.p, (int)n_keys, 0, 63, st); };
    auto unique = [&](void* tmp, size_t& bytes) {
        return cub::DeviceSelect::Unique(tmp, bytes, ckeys_sorted.p, cuniq.p, sc.num_runs.p + 1, (int)n_keys, st);
    };
    cub_reserve(sc.cub_tmp, sort, unique);
    cub_run(sc.cub_tmp, sort);
    cub_run(sc.cub_tmp, unique);
    int hc[8];
    unsigned last_off = 0, last_cnt = 0;
    int n_aff = 0;
    FLS_CUDA(cudaMemcpyAsync(hc, inc_cnt.p, 8 * sizeof(int), cudaMemcpyDeviceToHost, st));
    FLS_CUDA(cudaMemcpyAsync(&last_off, inc_new_off.p + (T - 1), sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    FLS_CUDA(cudaMemcpyAsync(&last_cnt, inc_new_count.p + (T - 1), sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    FLS_CUDA(cudaMemcpyAsync(&n_aff, sc.num_runs.p + 1, sizeof(int), cudaMemcpyDeviceToHost, st));
    c.sync();
    c.launches += 9;
    const int n_created = hc[0];
    const size_t moved = (size_t)last_off + last_cnt;  // points of the rewritten voxels
    // has to take the full path: eviction, no room, table load
    if (capacity > 0 && (long long)n_vox + n_created >= capacity) return 1;
    if (pts_end + moved > pts_sorted.cap) return 1;
    if (2 * (n_vox + (size_t)n_created) > table.slots) return 1;
    // voxels first (the centre runs are gathered from their new locations)
    inc_move_kernel<<<grid_for((size_t)T * 32, 256), 256, 0, st>>>(sc.uniq.p, T, inc_old_start.p, inc_old_count.p, sc.starts.p, sc.counts.p, inc_new_off.p,
                                                                 (unsigned)pts_end, sc.idx_sorted.p, d_new, pts_sorted.p, table.buf.p, table.mask);
    // centre runs
    ccount.reserve((size_t)n_aff + 1);
    cstart.reserve((size_t)n_aff + 1);
    list_count_kernel<<<grid_for((size_t)n_aff, 128), 128, 0, st>>>(cuniq.p, n_aff, n_stencil, table.buf.p, table.mask, ccount.p);
    FLS_CUDA(cudaMemsetAsync(inc_cnt.p, 0, 8 * sizeof(int), st));
    inc_new_centres_kernel<<<grid_for((size_t)n_aff, 256), 256, 0, st>>>(cuniq.p, n_aff, ctab.buf.p, ctab.mask, ccount.p, inc_cnt.p);
    cub_pass(sc.cub_tmp, [&](void* tmp, size_t& bytes) { return cub::DeviceScan::ExclusiveSum(tmp, bytes, ccount.p, cstart.p, n_aff, st); });
    unsigned l_off = 0, l_cnt = 0;
    FLS_CUDA(cudaMemcpyAsync(hc, inc_cnt.p, 8 * sizeof(int), cudaMemcpyDeviceToHost, st));
    FLS_CUDA(cudaMemcpyAsync(&l_off, cstart.p + (n_aff - 1), sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    FLS_CUDA(cudaMemcpyAsync(&l_cnt, ccount.p + (n_aff - 1), sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    c.sync();
    const size_t run_total = (size_t)l_off + l_cnt;
    const int n_new_centres = hc[0];
    unsigned long long old_records = 0;
    std::memcpy(&old_records, hc + 2, sizeof(old_records));
    c.launches += 5;
    // From here on the point array and the occupied table are already updated; if the lists do not fit, the caller's full build
    // regenerates everything from pts_all (which it extends itself), so nothing is lost.
    if (lists_end + run_total > lists.cap || lists_end + run_total > 0xfffffff0ull) return 1;
    if (4 * (n_centers + (size_t)n_new_centres) > ctab.slots) return 1;
    add_base_kernel<<<grid_for((size_t)n_aff, 256), 256, 0, st>>>(cstart.p, n_aff, (unsigned)lists_end);
    list_fill_kernel<<<grid_for((size_t)n_aff * 32, 256), 256, 0, st>>>(cuniq.p, n_aff, n_stencil, table.buf.p, table.mask, pts_sorted.p, cstart.p, ccount.p,
                                                                       lists.p, ctab.buf.p, ctab.mask);
    FLS_CUDA(cudaGetLastError());
    c.launches += 2;
    // bookkeeping
    pts_end += moved;
    pts_garbage += moved - n_new;  // the old copies of the rewritten voxels
    lists_end += run_total;
    lists_garbage += (size_t)old_records;
    n_pts += n_new;
    n_vox += (size_t)n_created;
    n_centers += (size_t)n_new_centres;
    n_list += run_total - (size_t)old_records;
    ++n_incremental;
    return FLS_OK;
}

int IvoxMap::append_and_build(const float4* d_new, size_t n_new, long long capacity, Call& c) {
    // mapping mode: append without touching the rest of the map whenever that is possible
    if (incremental && n_pts > 0 && n_new > 0 && (lists_garbage < n_list + (n_list >> 1)) && (pts_garbage < 2 * n_pts)) {
        // pts_all / stamp_all first (the full path and the LRU read them)
        const size_t n_old0 = n_pts, n0 = n_old0 + n_new;
        if (n0 <= pts_all.cap && (capacity <= 0 || n0 <= stamp_all.cap)) {
            FLS_CUDA(cudaMemcpyAsync(pts_all.p + n_old0, d_new, n_new * sizeof(float4), cudaMemcpyDeviceToDevice, c.stream));
            if (capacity > 0) {
                ++call_no;
                ivox_stamp_kernel<<<grid_for(n_new, 256), 256, 0, c.stream>>>(stamp_all.p + n_old0, n_new, call_no << 32);
            }
            const int rc = append_incremental(d_new, n_new, capacity, c);
            if (rc == FLS_OK) return FLS_OK;
            if (rc < 0) return rc;
            // full path below: pts_all / stamp_all already hold the new points
            return build_full(n_old0, n0, capacity, c, /*appended=*/true);
        }
    }
    return build_full(n_pts, n_pts + n_new, capacity, c, false, d_new, n_new);
}

int IvoxMap::build_full(size_t n_old, size_t n_in, long long capacity, Call& c, bool appended, const float4* d_new, size_t n_new) {
    size_t n = n_in;
    if (n == 0) return FLS_OK;
    const cudaStream_t st = c.stream;
    if (n > 0xfffffff0ull) return FLS_ERR_INVALID_ARG;
    const bool lru = capacity > 0;
    // grow pts_all (and the insertion stamps) preserving the old contents
    if (n > pts_all.cap) {
        DevBuf<float4> bigger;
        bigger.reserve(incremental ? 3 * n : n + n / 2);
        if (n_old) FLS_CUDA(cudaMemcpyAsync(bigger.p, pts_all.p, n_old * sizeof(float4), cudaMemcpyDeviceToDevice, st));
        c.sync();
        std::swap(bigger.p, pts_all.p);
        std::swap(bigger.cap, pts_all.cap);
    }
    if (lru && n > stamp_all.cap) {
        DevBuf<unsigned long long> bigger;
        bigger.reserve(incremental ? 3 * n : n + n / 2);
        if (n_old) FLS_CUDA(cudaMemcpyAsync(bigger.p, stamp_all.p, n_old * sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st));
        c.sync();
        std::swap(bigger.p, stamp_all.p);
        std::swap(bigger.cap, stamp_all.cap);
    }
    if (!appended) {
        if (n_new) FLS_CUDA(cudaMemcpyAsync(pts_all.p + n_old, d_new, n_new * sizeof(float4), cudaMemcpyDeviceToDevice, st));
        if (lru && n_new) {
            ++call_no;
            ivox_stamp_kernel<<<grid_for(n_new, 256), 256, 0, st>>>(stamp_all.p + n_old, n_new, call_no << 32);
        }
    }
    // mapping mode: room for the voxels the incremental inserts rewrite; buffers grow geometrically (a cudaFree + cudaMalloc of a
    // few hundred MB costs milliseconds — more than the build itself)
    if (incremental) {
        if (n + n / 2 + 65536 > pts_sorted.cap) pts_sorted.reserve(3 * n + 65536);
    } else {
        pts_sorted.reserve(n);
    }
    int runs = sorted_runs<false>(pts_all.p, n, inv_res, pts_sorted.p, scratch, c);
    if (lru && (long long)runs >= capacity) {
        // IVoxMap::AddPoints would have evicted the LRU tail while inserting (ivox_map.cpp:133-136): drop those voxels' old points
        size_t n_after = n;
        const int rc = evict_lru(n_old, n, runs, capacity, c, &n_after);
        if (rc != FLS_OK) return rc;
        n = n_after;
        runs = sorted_runs<false>(pts_all.p, n, inv_res, pts_sorted.p, scratch, c);  // n only shrank: pts_sorted has room
    }
    table.size_for((size_t)runs, incremental ? 4 : 2, incremental);  // mapping mode: room for the voxels to come
    fill_table(table, runs, scratch, c);
    n_pts = n;
    n_vox = (size_t)runs;
    pts_end = n;
    pts_garbage = 0;
    ++n_full;
    return build_stencil_lists(c);
}

// Exact LRU of IVoxMap::AddPoints for this call (see lru_simulate): a voxel's position in upstream's list is the insertion time of
// its last point, so the stamps of the points are all the state there is.  Victims lose every point they held before the call;
// one that is touched again later in the call keeps this call's points (it is created anew).  Compacts pts_all / stamp_all.
int IvoxMap::evict_lru(size_t n_old, size_t n, int runs, long long capacity, Call& c, size_t* n_after) {
    const cudaStream_t st = c.stream;
    BuildScratch& sc = scratch;
    if (n_vox == 0) return FLS_ERR_CAPACITY;  // the first cloud alone overflows the capacity
    lru_first.reserve((size_t)runs + 1);
    lru_nold.reserve((size_t)runs + 1);
    lru_cnt.reserve(4);
    FLS_CUDA(cudaMemsetAsync(lru_cnt.p, 0, 4 * sizeof(int), st));
    ivox_run_info_kernel<<<grid_for(runs, 256), 256, 0, st>>>(runs, sc.starts.p, sc.counts.p, sc.idx_sorted.p, stamp_all.p, (unsigned)n_old, lru_nold.p,
                                                            lru_first.p, eviction.stamps.reserve((size_t)runs + 1),
                                                            eviction.ids.reserve((size_t)runs + 1), sc.k32b.reserve(n + 1), lru_cnt.p);
    ++c.launches;
    int hc[4] = {0, 0, 0, 0};
    FLS_CUDA(cudaMemcpyAsync(hc, lru_cnt.p, 4 * sizeof(int), cudaMemcpyDeviceToHost, st));
    c.sync();
    const int n_cand = hc[0], n_create = hc[1], n_touched = hc[2];
    if (n_cand == 0) return FLS_ERR_CAPACITY;
    const int rc = eviction.run(n_cand, sc.k32b.p, n_create, n_touched, n_vox, capacity, sc.cub_tmp, c,
                                [&](const unsigned* runs_sorted, int K, unsigned* out) {
                                    ivox_cand_kernel<<<grid_for(K, 256), 256, 0, st>>>(runs_sorted, K, lru_first.p, out);
                                });
    if (rc != FLS_OK) return rc;
    *n_after = n;
    if (eviction.n_victims == 0) return FLS_OK;
    // flags: 1 = keep; the victims' points from before this call go
    lru_flags.reserve(n + 1);
    FLS_CUDA(cudaMemsetAsync(lru_flags.p, 1, n, st));
    ivox_kill_kernel<<<grid_for(eviction.n_victims * 32, 256), 256, 0, st>>>(eviction.victims.p, (int)eviction.n_victims, eviction.ids_sorted.p, sc.starts.p,
                                                                            lru_nold.p, sc.idx_sorted.p, lru_flags.p);
    // stable compaction of the points and their stamps (pts_sorted / keys are rebuilt by the second sort anyway: use them as targets)
    sc.keys.reserve(n + 1);
    auto keep_pts = [&](void* tmp, size_t& bytes) {
        return cub::DeviceSelect::Flagged(tmp, bytes, pts_all.p, lru_flags.p, pts_sorted.p, sc.num_runs.p, (int)n, st);
    };
    auto keep_stamps = [&](void* tmp, size_t& bytes) {
        return cub::DeviceSelect::Flagged(tmp, bytes, stamp_all.p, lru_flags.p, sc.keys.p, sc.num_runs.p, (int)n, st);
    };
    cub_reserve(sc.cub_tmp, keep_pts, keep_stamps);
    cub_run(sc.cub_tmp, keep_pts);
    cub_run(sc.cub_tmp, keep_stamps);
    FLS_CUDA(cudaMemcpyAsync(sc.h_num_runs, sc.num_runs.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    c.sync();
    const size_t kept = (size_t)*sc.h_num_runs;
    FLS_CUDA(cudaMemcpyAsync(pts_all.p, pts_sorted.p, kept * sizeof(float4), cudaMemcpyDeviceToDevice, st));
    FLS_CUDA(cudaMemcpyAsync(stamp_all.p, sc.keys.p, kept * sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st));
    c.launches += 4;
    *n_after = kept;
    return FLS_OK;
}

size_t IvoxMap::dump_keys(unsigned long long* h_out, size_t cap, cudaStream_t st) {
    // packed keys of the occupied voxels, from the table (tests)
    if (n_vox == 0) return 0;
    scratch.keys.reserve(n_vox + 1);
    scratch.num_runs.reserve(2);
    FLS_CUDA(cudaMemsetAsync(scratch.num_runs.p, 0, sizeof(int), st));
    table_dump_kernel<<<grid_for(table.slots, 256), 256, 0, st>>>(table.buf.p, table.slots, scratch.keys.p, scratch.num_runs.p);
    int n = 0;
    FLS_CUDA(cudaMemcpyAsync(&n, scratch.num_runs.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    FLS_CUDA(cudaStreamSynchronize(st));
    const size_t m = (size_t)n < cap ? (size_t)n : cap;
    FLS_CUDA(cudaMemcpy(h_out, scratch.keys.p, sizeof(unsigned long long) * m, cudaMemcpyDeviceToHost));
    return m;
}

int IvoxMap::build_stencil_lists(Call& c) {
    const cudaStream_t st = c.stream;
    BuildScratch& sc = scratch;
    const size_t S = (size_t)n_stencil;
    const size_t n_keys = n_vox * S;
    const size_t total = n_pts * S;  // every point lands in exactly S lists (symmetric stencil)
    if (total > 0xfffffff0ull || n_keys > 0x7ffffff0ull) return FLS_ERR_CAPACITY;
    ckeys.reserve(n_keys);
    ckeys_sorted.reserve(n_keys);
    cuniq.reserve(n_keys);
    center_keys_kernel<<<grid_for(n_keys, 256), 256, 0, st>>>(sc.uniq.p, (int)n_vox, n_stencil, ckeys.p);
    auto sort = [&](void* tmp, size_t& bytes) { return cub::DeviceRadixSort::SortKeys(tmp, bytes, ckeys.p, ckeys_sorted.p, (int)n_keys, 0, 63, st); };
    auto unique = [&](void* tmp, size_t& bytes) {
        return cub::DeviceSelect::Unique(tmp, bytes, ckeys_sorted.p, cuniq.p, sc.num_runs.p, (int)n_keys, st);
    };
    cub_reserve(sc.cub_tmp, sort, unique);
    cub_run(sc.cub_tmp, sort);
    cub_run(sc.cub_tmp, unique);
    FLS_CUDA(cudaMemcpyAsync(sc.h_num_runs, sc.num_runs.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    c.sync();
    const int nc = *sc.h_num_runs;
    ccount.reserve((size_t)nc);
    cstart.reserve((size_t)nc);
    list_count_kernel<<<grid_for((size_t)nc, 128), 128, 0, st>>>(cuniq.p, nc, n_stencil, table.buf.p, table.mask, ccount.p);
    cub_pass(sc.cub_tmp, [&](void* tmp, size_t& bytes) { return cub::DeviceScan::ExclusiveSum(tmp, bytes, ccount.p, cstart.p, nc, st); });
    // load factor <= 0.25: the centre table is probed once per point-iteration and a long linear-probing chain stalls
    // a whole warp, so it is kept sparser than the occupied table
    ctab.size_for((size_t)nc, incremental ? 8 : 4, incremental);
    if (incremental) {  // mapping mode: room for the runs the incremental inserts append, geometric growth
        if (2 * total + 1048576 > lists.cap) lists.reserve(4 * total + 1048576);
    } else {
        lists.reserve(total);
    }
    ctab.clear(c);
    list_fill_kernel<<<grid_for((size_t)nc * 32, 256), 256, 0, st>>>(cuniq.p, nc, n_stencil, table.buf.p, table.mask, pts_sorted.p, cstart.p, ccount.p,
                                                                     lists.p, ctab.buf.p, ctab.mask);
    FLS_CUDA(cudaGetLastError());
    n_centers = (size_t)nc;
    n_list = total;
    lists_end = total;
    lists_garbage = 0;
    c.launches += 6;
    // the transient key arrays are the largest buffers of the build; give them back
    if (!incremental) {
        ckeys.release();
        ckeys_sorted.release();
    }
    return FLS_OK;
}

int window_add(WindowMap& w, const float4* d_cloud, size_t n, size_t window, float leaf, bool filter_always, bool replace, BuildScratch& sc,
               Call& call) {
    const cudaStream_t st = call.stream;
    const float4* merged = d_cloud;
    size_t n_merged = n;
    size_t depth = 1;
    if (!replace) {
        std::unique_ptr<WindowMap::Cloud> c(new WindowMap::Cloud());
        c->buf.reserve(n);
        if (n) FLS_CUDA(cudaMemcpyAsync(c->buf.p, d_cloud, n * sizeof(float4), cudaMemcpyDeviceToDevice, st));
        c->n = n;
        w.deque.push_back(std::move(c));
        if (w.deque.size() > window) {
            call.sync();  // the evicted buffer may still feed a copy in flight
            w.deque.pop_front();
        }
        n_merged = 0;
        for (auto& q : w.deque) n_merged += q->n;
        w.merged.reserve(n_merged);
        size_t off = 0;
        for (auto& q : w.deque) {
            if (q->n) FLS_CUDA(cudaMemcpyAsync(w.merged.p + off, q->buf.p, q->n * sizeof(float4), cudaMemcpyDeviceToDevice, st));
            off += q->n;
        }
        merged = w.merged.p;
        depth = w.deque.size();
    }
    w.cloud.reserve(n_merged);
    if (filter_always || depth > 5) {
        w.n = voxel_grid_device(merged, n_merged, leaf, w.cloud.p, sc, call);
    } else {
        if (n_merged) FLS_CUDA(cudaMemcpyAsync(w.cloud.p, merged, n_merged * sizeof(float4), cudaMemcpyDeviceToDevice, st));
        w.n = n_merged;
    }
    return w.grid.build(w.cloud.p, w.n, sc, call);
}

}  // namespace fls
