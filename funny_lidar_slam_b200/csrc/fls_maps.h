// fls_maps.h — host-side owners of the device-resident map structures (SearchGrid, IvoxMap, NdtMap, WindowMap).  Every builder runs
// on the stream of the Call it is given and counts its launches and waits into it.
#pragma once
#include <deque>
#include <functional>
#include <memory>
#include <vector>

#include "fls_common.cuh"

namespace fls {

// Exact emulation of upstream's LRU policy for one insert call (IVoxMap::AddPoints, ivox_map.cpp:122-143; IncrementalNDT::
// AddCloudToLocalMap, incremental_ndt.h:193-214): points are inserted one after the other, a touched voxel moves to the front,
// a created voxel is pushed to the front and — when the size then reaches `capacity` — the tail is popped.
//   cand_first_touch[i]: candidates = voxels that existed before the call, oldest first; value = index of the first point of
//                        this call that touches it (0xffffffff: untouched)
//   create_times       : index of the point that creates each new voxel (any order)
// Output: victims (positions in the candidate list) in eviction order, and for each whether the voxel is touched again later in
// the call (it is then re-created empty).  Returns false when the candidates run out (the call alone overflows the capacity).
bool lru_simulate(size_t size0, size_t capacity, const std::vector<unsigned>& cand_first_touch, std::vector<unsigned> create_times,
                  std::vector<unsigned>& victims, std::vector<unsigned char>& recreated);

// How many of the n_cand oldest candidates lru_simulate needs for a call that creates n_new voxels in a map of n_vox, n_touched
// of the candidates being touched by the call.  Without cascades n_vox + n_new - (capacity - 1) voxels go; every candidate the
// simulation skips was touched in this call, and each touched victim is re-created and can push out one more, so 2 * n_touched
// (plus a margin) covers both.  Capped at n_cand.
size_t lru_candidate_bound(size_t n_vox, int n_new, int n_touched, long long capacity, size_t n_cand);

// The exact-LRU eviction pass of IvoxMap and NdtMap (fls_map.cu).  The map writes one (stamp, id) pair per candidate to stamps / ids
// and the creation times of its new voxels to a device array; run() sorts the candidates by stamp, has the map write the first touch
// of the K oldest (lru_candidate_bound) through `write_first`, runs lru_simulate and leaves the victims on the device: victims[i] is
// a position in ids_sorted, recreated[i] whether that voxel is created anew later in the call.  FLS_ERR_CAPACITY: the call alone
// overflows the capacity.
struct LruEviction {
    DevBuf<unsigned long long> stamps, stamps_sorted;
    DevBuf<unsigned> ids, ids_sorted, first_touch, victims;
    DevBuf<unsigned char> recreated;
    size_t n_victims = 0, n_recreated = 0;
    std::vector<unsigned> h_first, h_create, h_victims;
    std::vector<unsigned char> h_recreated;
    // write_first(ids_sorted, K, out) enqueues one kernel on c.stream that writes the first touch of candidates 0..K-1 to out[0..K-1]
    int run(int n_cand, const unsigned* d_create, int n_create, int n_touched, size_t size0, long long capacity, DevBuf<unsigned char>& cub_tmp,
            Call& c, const std::function<void(const unsigned*, int, unsigned*)>& write_first);
};

// Scratch shared by the sort / run-length passes of every map build and of the voxel-grid filter.
// The voxel-runs pass puts n keyed points in voxel-contiguous order: a stable radix sort of (key, point index) over key bits
// [0, end_bit), a run-length encode of the sorted keys, and the exclusive sum of the run lengths (each run's first sorted
// position).  Keys K = unsigned long long go keys -> keys_sorted -> uniq, keys K = unsigned go k32a -> k32b -> uniq32; both
// sort idx -> idx_sorted and write counts and starts.  It is split in steps so that a caller can work between them:
//   reserve_runs<K>(n)          the arrays, before the caller's key kernel fills the keys and idx
//   sort_pairs<K>(n, end_bit)   sizes cub_tmp once for sort, encode and sum over n, then sorts
//   encode_runs<K>(n)           encodes and returns the run count, read through h_num_runs after one wait
//   run_starts(runs)            the exclusive sum of the run lengths
struct BuildScratch {
    DevBuf<unsigned long long> keys, keys_sorted, uniq;
    DevBuf<unsigned> idx, idx_sorted, counts, starts, k32a, k32b, uniq32;
    DevBuf<unsigned char> cub_tmp;
    DevBuf<float> minmax;
    DevBuf<int> num_runs;
    int* h_num_runs = nullptr;  // pinned (plain memory when the pinned allocation failed)
    bool pinned = true;
    BuildScratch();
    ~BuildScratch();
    template <class K>
    void reserve_runs(size_t n);
    template <class K>
    void sort_pairs(size_t n, int end_bit, Call& c);
    template <class K>
    int encode_runs(size_t n, Call& c);
    void run_starts(int runs, Call& c);
};

// K7: VoxelGridCloud on the device.  d_out must hold n records; returns the output count.
size_t voxel_grid_device(const float4* d_pts, size_t n, float leaf, float4* d_out, BuildScratch& sc, Call& c);

// Open-addressing table of HashSlot {key, start, count}, linear probing: table_find reads it, table_claim inserts (fls_common.cuh).
// A power of two of at least 1024 slots.
struct VoxelTable {
    DevBuf<HashSlot> buf;
    unsigned mask = 0;
    size_t slots = 0;
    // room for n keys at `factor` slots per key; grow_only (mapping mode) keeps a larger table as it is, for the keys to come
    void size_for(size_t n, size_t factor, bool grow_only = false);
    void clear(Call& c);  // every slot empty; one kernel
};

// Uniform search grid over a cloud for the exact 1-NN of IcpOptimized / GetFitnessScore and the exact 5-NN of the kd-tree LOAM
// plug-ins: cells of floor(p/res), the cloud in cell-contiguous order and an open-addressing table of {key, start, count}.
struct GridView {  // what the search kernels read
    const float4* __restrict__ pts;    // cell-contiguous points
    const HashSlot* __restrict__ tab;  // floor-keyed occupied-cell table
    unsigned mask;
    float inv_cell, cell;
    unsigned n_pts;
};
struct SearchGrid {
    float res = 0.5f;
    size_t n_pts = 0, n_vox = 0;
    DevBuf<float4> pts_sorted;
    VoxelTable table;
    // rebuilds the grid over the n points at d_cloud (an empty cloud leaves it empty and launches nothing); returns fls_status
    int build(const float4* d_cloud, size_t n, BuildScratch& sc, Call& c);
    GridView view() const { return {pts_sorted.p, table.buf.p, table.mask, 1.0f / res, res, (unsigned)n_pts}; }
    size_t bytes() const { return pts_sorted.bytes() + table.buf.bytes(); }
};

// iVox map: voxels of round(p/res) (IVoxMap::Pos2Grid), voxel-contiguous float4 points + open-addressing table of
// {key, start, count} (see fls_ivox.cuh).
//
// The build also materialises, for every "centre" voxel (occupied, or within the stencil of an
// occupied voxel), the concatenation of the points of its stencil voxels in the reference's visit order — the exact
// candidate sequence IVoxMap::GetClosestPoint walks — as one contiguous float4 run, plus a second table
// {centre key -> run start, run length}.  A k-NN query is then ONE table probe and ONE streaming scan
// (HBM is spent to buy bandwidth-friendly access: ~n_stencil x the point array).
struct IvoxMap {
    float res = 0.5f, inv_res = 2.0f;
    int n_stencil = 1;  // voxels per stencil: 1, 7, 19 or 27
    size_t n_pts = 0, n_vox = 0;
    DevBuf<float4> pts_all;     // insertion order (kept so incremental adds can rebuild)
    DevBuf<unsigned long long> stamp_all;  // per point of pts_all: (AddPoints call << 32) | position in that call — LRU state (capacity > 0 only)
    unsigned long long call_no = 0;
    DevBuf<unsigned> lru_first, lru_nold;  // per run of the build: first point of the call that touches it, points from before the call
    DevBuf<unsigned char> lru_flags;       // per point: kept by the eviction
    DevBuf<int> lru_cnt;                   // ivox_run_info_kernel's candidates, creations, touched candidates
    LruEviction eviction;
    DevBuf<float4> pts_sorted;  // voxel-contiguous, Morton order
    VoxelTable table;           // occupied voxels
    // stencil lists
    size_t n_centers = 0, n_list = 0;
    DevBuf<float4> lists;
    VoxelTable ctab;
    DevBuf<unsigned long long> ckeys, ckeys_sorted, cuniq;
    DevBuf<unsigned> ccount, cstart;
    BuildScratch scratch;

    void set_resolution(float r) {
        res = r;
        inv_res = 1.0f / r;
    }
    void clear() { n_pts = n_vox = n_centers = n_list = 0; }
    int evict_lru(size_t n_old, size_t n, int runs, long long capacity, Call& c, size_t* n_after);
    size_t dump_keys(unsigned long long* h_out, size_t cap, cudaStream_t st);  // packed keys of the occupied voxels (tests)
    // append n points that are already on the device (packed float4) and rebuild; returns fls_status
    int append_and_build(const float4* d_new, size_t n_new, long long capacity, Call& c);
    int build_full(size_t n_old, size_t n_in, long long capacity, Call& c, bool appended, const float4* d_new = nullptr, size_t n_new = 0);
    int append_incremental(const float4* d_new, size_t n_new, long long capacity, Call& c);
    // log-structured state of the incremental path (mapping mode)
    bool incremental = false;          // set by the owner: the map grows by small inserts (mapping mode)
    size_t pts_end = 0, pts_garbage = 0;      // used part of pts_sorted, dead records in it
    size_t lists_end = 0, lists_garbage = 0;  // used part of lists, dead records in it
    size_t n_incremental = 0, n_full = 0;     // how many inserts took which path
    DevBuf<unsigned> inc_old_start, inc_old_count, inc_new_count, inc_new_off;
    DevBuf<int> inc_cnt;  // created voxels, then new centres and (u64 at [2]) the records of the centre runs they replace
    int build_stencil_lists(Call& c);
    size_t bytes() const { return pts_all.bytes() + pts_sorted.bytes() + table.buf.bytes() + lists.bytes() + ctab.buf.bytes(); }
};

// ---- NDT voxel map ------------------------------------------------------------------------------------------
// Hot record read by the residual kernel: mean + symmetric information matrix (upper triangle), 80 bytes.
struct __align__(16) NdtHot {
    double mu[3];
    double info[6];  // xx, xy, xz, yy, yz, zz
    double pad;
};
// Cold per-voxel state used only by AddCloudToLocalMap / UpdateVoxel (incremental_ndt.h:130-179 upstream)
struct NdtCold {
    double sigma[9];
    int num_points;   // VoxelData::num_points_
    int carry_count;  // points buffered and not yet consumed by an estimate (<= min_points_in_voxel)
    int estimated;
    int alive;                  // 0 once the voxel has been evicted (its index is on the free list)
    unsigned long long key;     // packed voxel key (table rebuild after evictions)
    unsigned long long stamp;   // last touch: (AddCloudToLocalMap call << 32) | index of the touching point in that call's cloud —
                                // the position of the voxel in upstream's LRU list (incremental_ndt.h:193-214)
};
// table slot: {packed key, voxel index, estimated flag}
struct NdtView {
    const HashSlot* __restrict__ tab;
    const NdtHot* __restrict__ hot;
    unsigned mask;
    double inv_voxel;
};

struct NdtMap {
    double voxel = 1.0, inv_voxel = 1.0;
    int min_pts = 5, max_pts = 50;
    long long capacity = 100000;
    size_t n_vox = 0;
    VoxelTable table;  // {key, voxel index, estimated flag}, sized once for 2 x capacity
    DevBuf<NdtHot> hot;
    DevBuf<NdtCold> cold;
    DevBuf<double> carry;  // [capacity][min_pts][3]
    DevBuf<float4> filtered;
    // device counters: voxel indices handed out, overflow flag, free-stack cursor, this call's creations and touched voxels, cursors
    enum Counter { kHiWater, kOverflow, kFreeCursor, kCreations, kTouched, kLiveCursor, kCreateCursor, kDumpCursor, kCounters };
    DevBuf<int> counter;
    DevBuf<int> free_list;         // indices of evicted voxels, reused by the next creations
    int n_free = 0;
    int hi_water = 0;              // voxel indices handed out so far
    unsigned long long call_no = 0;  // AddCloudToLocalMap calls so far (high half of the LRU stamps)
    DevBuf<int> run_vi;            // per touched voxel of a call: its index, -1 = to be created
    DevBuf<int> touch_run;         // per voxel index: the run that touches it in this call, -1 = none
    LruEviction eviction;
    BuildScratch scratch;

    void configure(double voxel_size, int min_points, int max_points, long long cap);
    // evict the LRU tail exactly as upstream's sequential insert would (incremental_ndt.h:203-206), n_vox net of it; called by add_cloud
    int evict_lru(int runs, int n_new, int n_touched, Call& c);
    // packed voxel keys of the live voxels (tests); returns how many
    size_t dump_keys(unsigned long long* h_out, size_t cap, cudaStream_t st);
    // every live voxel with its mean, information and counters, in device order (tests)
    void dump_voxels(std::vector<fls_ndt_voxel>& out, cudaStream_t st);
    // VoxelGridCloud(cloud, leaf) then insert/update voxels; `first_scan` = flag_first_scan_ upstream
    int add_cloud(const float4* d_cloud, size_t n, float leaf, bool first_scan, Call& c);
    NdtView view() const {
        NdtView v;
        v.tab = table.buf.p;
        v.hot = hot.p;
        v.mask = table.mask;
        v.inv_voxel = inv_voxel;
        return v;
    }
    size_t bytes() const { return table.buf.bytes() + hot.bytes() + cold.bytes() + carry.bytes(); }
};

// Sliding window of clouds -> VoxelGrid -> exact search grid: the local map of IcpOptimized (cloud_deque_ / local_map_ptr_,
// icp_optimized.h:173-187, 246) and of the kd-tree LOAM plug-ins (planar_cloud_deque_ / corner_cloud_deque_)
struct WindowMap {
    struct Cloud {
        DevBuf<float4> buf;
        size_t n = 0;
    };
    std::deque<std::unique_ptr<Cloud>> deque;
    DevBuf<float4> merged;  // concatenation of the window
    DevBuf<float4> cloud;   // what upstream builds the kd-tree on
    size_t n = 0;
    SearchGrid grid;        // over `cloud`
};
// Adds a device cloud to w (replace: the window is that cloud alone) and rebuilds it.  filter_always false: VoxelGrid(leaf) only
// once the window holds more than 5 clouds (loam_full_kdtree.h:91-99).
int window_add(WindowMap& w, const float4* d_cloud, size_t n, size_t window, float leaf, bool filter_always, bool replace, BuildScratch& sc,
               Call& call);

// K4: LOAM feature extraction on the projector's arrays (host in / host out); see fls_features.cu
int extract_features_device(int device, const float* depth, const int* col, size_t n, const int* row_start, const int* row_end, int n_rows,
                            float corner_thr, float planar_thr, int* corner_idx, size_t* n_corner, int* planar_idx, size_t* n_planar,
                            fls_match_stats* stats);

// PCD v0.7 files of x y z [intensity] clouds (fls_localmap.cu)
int pcd_read(const char* path, std::vector<float>& xyzi, std::string& err);
int pcd_write(const char* path, const float* xyzi, size_t n, std::string& err);

// repack caller records (stride >= 20, intensity at byte 16) into packed float4 on the device
int project_device(int device, const void* raw, const int* ring, const float* time, const fls_imu_buffer* imu, const double* vel, size_t n, size_t stride,
                   int V, int H, float h_res, float min_d, float max_d, float* ordered_out, float* depth_out, int* col_out, int* row_start, int* row_end,
                   size_t* n_out);
// PreProcessing::Run, non-feature branch (preprocessing.cpp:181-225): raw x,y,z,intensity,time records -> ordered + planar clouds (host)
// `vel`: NULL, or the body velocity of fls_preprocess_motion (rotation only when all zero)
int preprocess_device(int device, const float* raw_xyzit, size_t n, const fls_imu_buffer* imu, const double* vel, float min_d, float max_d, int jump_span,
                      float leaf, float* ordered_out, size_t* n_ordered, float* planar_out, size_t* n_planar);
// Copies n host records of `stride` bytes (stride_ok) to packed float4 at dst on c.stream: one copy when they are packed already, else
// a copy to `staging` and one repack kernel.  Counts the bytes copied and the kernel.
void upload_records(const void* pts, size_t n, size_t stride, float4* dst, DevBuf<unsigned char>& staging, Call& c);
// TransformPointCloud(cloud, Mat4d) with R, t cast to float first (pointcloud_utility.h:141-158 upstream); T column-major
void launch_transform_f(const float4* d_in, size_t n, const double* T_colmajor, float4* d_out, cudaStream_t st);
void launch_transform_d(const float4* d_in, size_t n, const double* T_colmajor, float4* d_out, cudaStream_t st);

}  // namespace fls
