// fls_maps.h — host-side owners of the device-resident map structures.
#pragma once
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

// scratch shared by the sort / run-length passes of every map build and of the voxel-grid filter
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
};

// K7: VoxelGridCloud on the device.  d_out must hold n records; returns the output count.  `waits` (optional) counts the
// stream synchronisations the call made.
size_t voxel_grid_device(const float4* d_pts, size_t n, float leaf, float4* d_out, BuildScratch& sc, cudaStream_t st, int* launches,
                         int* waits = nullptr);

// Point grid: voxel-contiguous float4 points + open-addressing table of {key, start, count} (see fls_ivox.cuh).
// key_mode 0: round(p/res)  — IVoxMap::Pos2Grid (iVox map of the LOAM plug-in)
// key_mode 1: floor(p/res)  — uniform search grid under the bounded exact 1-NN of IcpOptimized / GetFitnessScore
//
// With n_stencil > 0 the build also materialises, for every "centre" voxel (occupied, or within the stencil of an
// occupied voxel), the concatenation of the points of its stencil voxels in the reference's visit order — the exact
// candidate sequence IVoxMap::GetClosestPoint walks — as one contiguous float4 run, plus a second table
// {centre key -> run start, run length}.  A k-NN query is then ONE table probe and ONE streaming scan
// (HBM is spent to buy bandwidth-friendly access: ~n_stencil x the point array).
struct IvoxMap {
    float res = 0.5f, inv_res = 2.0f;
    int key_mode = 0;
    int n_stencil = 0;  // 0: no stencil lists (ICP / fitness grids)
    size_t n_pts = 0, n_vox = 0;
    unsigned mask = 0;
    DevBuf<float4> pts_all;     // insertion order (kept so incremental adds can rebuild)
    DevBuf<unsigned long long> stamp_all;  // per point of pts_all: (AddPoints call << 32) | position in that call — LRU state (capacity > 0 only)
    unsigned long long call_no = 0;
    DevBuf<unsigned> lru_old, lru_first, lru_nold, lru_vals, lru_vals_sorted;
    DevBuf<unsigned long long> lru_keys, lru_keys_sorted;
    DevBuf<unsigned char> lru_flags;
    DevBuf<int> lru_cnt;
    DevBuf<float4> pts_sorted;  // voxel-contiguous, Morton order
    DevBuf<HashSlot> table;     // occupied voxels
    // stencil lists
    size_t n_centers = 0, n_list = 0;
    unsigned cmask = 0;
    DevBuf<float4> lists;
    DevBuf<HashSlot> ctab;
    DevBuf<unsigned long long> ckeys, ckeys_sorted, cuniq;
    DevBuf<unsigned> ccount, cstart;
    BuildScratch scratch;
    int launches = 0;

    void set_resolution(float r) {
        res = r;
        inv_res = 1.0f / r;
    }
    void clear() { n_pts = n_vox = n_centers = n_list = 0; }
    int sort_and_runs(size_t n, cudaStream_t st, int* runs_out);
    int evict_lru(size_t n_old, size_t n, int runs, long long capacity, cudaStream_t st, size_t* n_after);
    size_t dump_keys(unsigned long long* h_out, size_t cap, cudaStream_t st);  // packed keys of the occupied voxels (tests)
    // append n points that are already on the device (packed float4) and rebuild; returns fls_status
    int append_and_build(const float4* d_new, size_t n_new, long long capacity, cudaStream_t st);
    int build_full(size_t n_old, size_t n_in, long long capacity, cudaStream_t st, bool appended, const float4* d_new = nullptr, size_t n_new = 0);
    int append_incremental(const float4* d_new, size_t n_new, long long capacity, cudaStream_t st);
    // log-structured state of the incremental path (mapping mode)
    bool incremental = false;          // set by the owner: the map grows by small inserts (mapping mode)
    size_t pts_end = 0, pts_garbage = 0;      // used part of pts_sorted, dead records in it
    size_t lists_end = 0, lists_garbage = 0;  // used part of lists, dead records in it
    size_t n_incremental = 0, n_full = 0;     // how many inserts took which path
    DevBuf<unsigned> inc_old_start, inc_old_count, inc_new_count, inc_new_off;
    int build_stencil_lists(cudaStream_t st);
    size_t bytes() const { return pts_all.bytes() + pts_sorted.bytes() + table.bytes() + lists.bytes() + ctab.bytes(); }
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
    unsigned mask = 0;
    size_t slots = 0;
    DevBuf<HashSlot> table;
    DevBuf<NdtHot> hot;
    DevBuf<NdtCold> cold;
    DevBuf<double> carry;  // [capacity][min_pts][3]
    DevBuf<float4> filtered;
    DevBuf<int> counter;  // device voxel counter (high-water mark of allocated indices), overflow flag, free-list cursor, creations
    DevBuf<int> free_list;         // indices of evicted voxels, reused by the next creations
    int n_free = 0;
    int hi_water = 0;              // voxel indices handed out so far
    unsigned long long call_no = 0;  // AddCloudToLocalMap calls so far (high half of the LRU stamps)
    DevBuf<int> run_vi;            // per touched voxel of a call: its index, -1 = to be created
    DevBuf<int> touch_run;         // per voxel index: the run that touches it in this call, -1 = none
    DevBuf<unsigned long long> lru_keys, lru_keys_sorted;
    DevBuf<unsigned> lru_vals, lru_vals_sorted;
    std::vector<int> h_buf;
    BuildScratch scratch;
    int launches = 0;

    void configure(double voxel_size, int min_points, int max_points, long long cap);
    // evict the LRU tail exactly as upstream's sequential insert would (incremental_ndt.h:203-206); called by add_cloud
    int evict_lru(int runs, int n_new, int n_touched, cudaStream_t st, int* n_victims, int* n_recreated);
    // packed voxel keys of the live voxels (tests); returns how many
    size_t dump_keys(unsigned long long* h_out, size_t cap, cudaStream_t st);
    // every live voxel with its mean, information and counters, in device order (tests)
    void dump_voxels(std::vector<fls_ndt_voxel>& out, cudaStream_t st);
    // VoxelGridCloud(cloud, leaf) then insert/update voxels; `first_scan` = flag_first_scan_ upstream
    int add_cloud(const float4* d_cloud, size_t n, float leaf, bool first_scan, cudaStream_t st);
    NdtView view() const {
        NdtView v;
        v.tab = table.p;
        v.hot = hot.p;
        v.mask = mask;
        v.inv_voxel = inv_voxel;
        return v;
    }
    size_t bytes() const { return table.bytes() + hot.bytes() + cold.bytes() + carry.bytes(); }
};

// K4: LOAM feature extraction on the projector's arrays (host in / host out); see fls_features.cu
int extract_features_device(int device, const float* depth, const int* col, size_t n, const int* row_start, const int* row_end, int n_rows,
                            float corner_thr, float planar_thr, int* corner_idx, size_t* n_corner, int* planar_idx, size_t* n_planar,
                            fls_match_stats* stats);

// PCD v0.7 files of x y z [intensity] clouds (fls_localmap.cu)
int pcd_read(const char* path, std::vector<float>& xyzi, std::string& err);
int pcd_write(const char* path, const float* xyzi, size_t n, std::string& err);

// repack caller records (stride >= 20, intensity at byte 16) into packed float4 on the device
int project_device(int device, const void* raw, const int* ring, const float* time, const fls_imu_buffer* imu, size_t n, size_t stride, int V, int H,
                   float h_res, float min_d, float max_d, float* ordered_out, float* depth_out, int* col_out, int* row_start, int* row_end,
                   size_t* n_out);
// PreProcessing::Run, non-feature branch (preprocessing.cpp:181-225): raw x,y,z,intensity,time records -> ordered + planar clouds (host)
int preprocess_device(int device, const float* raw_xyzit, size_t n, const fls_imu_buffer* imu, float min_d, float max_d, int jump_span, float leaf,
                      float* ordered_out, size_t* n_ordered, float* planar_out, size_t* n_planar);
// Copies n host records of `stride` bytes (stride_ok) to packed float4 at dst on st: one copy when they are packed already, else a
// copy to `staging` and one repack kernel.  Adds the bytes copied to *h2d and the kernel to *launches.
void upload_records(const void* pts, size_t n, size_t stride, float4* dst, DevBuf<unsigned char>& staging, cudaStream_t st, long long* h2d,
                    int* launches);
// TransformPointCloud(cloud, Mat4d) with R, t cast to float first (pointcloud_utility.h:141-158 upstream); T column-major
void launch_transform_f(const float4* d_in, size_t n, const double* T_colmajor, float4* d_out, cudaStream_t st);
void launch_transform_d(const float4* d_in, size_t n, const double* T_colmajor, float4* d_out, cudaStream_t st);

}  // namespace fls
