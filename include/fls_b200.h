/*
 * fls_b200.h — C ABI of the H100-native (sm_90a) scan-matching frontend.
 *
 * Drop-in boundary for funny_lidar_slam's registration plug-in interface.  Every entry point is what
 * a thin `RegistrationInterface` adapter (funny_lidar_slam_b200/shim/b200_registration.h, see
 * INTEGRATION.md) binds; citations are relative to the reference tree (zm0612/funny_lidar_slam):
 *
 *   fls_create / fls_destroy   <- plug-in constructors selected by mode string in
 *                                 FrontEnd::InitMatcher (src/slam/frontend.cpp:30-88) and
 *                                 Localization::InitMatcher (src/slam/localization.cpp:43-92)
 *   fls_add_cloud              <- RegistrationInterface::AddCloudToLocalMap
 *                                 (include/registration/registration_interface.h:17)
 *   fls_match                  <- RegistrationInterface::Match (registration_interface.h:13)
 *   fls_fitness                <- RegistrationInterface::GetFitnessScore (registration_interface.h:19)
 *   fls_extract_features       <- loam::FeatureExtractor::ExtractFeatures
 *                                 (include/loam/feature_extractor.h:22, src/loam/feature_extractor.cpp:35-44)
 *   fls_project / _imu         <- loam::PointcloudProjector::Project (src/loam/pointcloud_projector.cpp:32-133)
 *   fls_preprocess             <- PreProcessing::Run range gate + LidarDistortionCorrector::ProcessPoint + jump span + VoxelGrid
 *                                 (src/slam/preprocessing.cpp:181-225, src/lidar/lidar_distortion_corrector.cpp:37-64)
 *   fls_voxel_grid             <- VoxelGridCloud (include/common/pointcloud_utility.h:216-224,263-271)
 *   fls_preprocess_loam        <- PreProcessing::Run, LoamFull branch: Project + ExtractFeatures + corner / planar VoxelGrid
 *                                 (src/slam/preprocessing.cpp:226-237)
 *   fls_convert_cloud          <- PreProcessing::ConvertMessageToCloud + ComputePointOffsetTime + GetLidarPointMinMaxOffsetTime
 *                                 (src/slam/preprocessing.cpp:262-571) and the scan's time window (:86-104)
 *   fls_preprocess_device /    <- fls_preprocess / fls_preprocess_loam reading a cloud already in device memory
 *   fls_preprocess_loam_device
 *   fls_keyframes_*            <- the keyframe-map loops of System::SaveMap (src/slam/system.cpp:299-341),
 *                                 System::VisualizeGlobalMap (src/slam/system.cpp:847-896) and
 *                                 LoopClosure::GetSubMap (src/slam/loop_closure.cpp:179-231)
 *
 * Conventions
 *   * Points are read from caller memory as {float x, y, z, <pad>, intensity ...} records `stride_bytes`
 *     apart: stride 32 with intensity at byte offset 16 is pcl::PointXYZI (the reference's cloud type,
 *     include/common/data_type.h:29-30); stride 16 is packed {x, y, z, intensity}.  Use FLS_LAYOUT_*.
 *   * Poses are Eigen `Mat4d` memory: 16 doubles, COLUMN-major (include/common/data_type.h:55).
 *   * All functions return 0 on success or a negative fls_status; nothing aborts, nothing throws
 *     (the reference's only runtime failure signal is `Match` returning false, frontend.cpp:208-210).
 *   * A handle is used from one thread at a time (the reference calls every plug-in method from the
 *     single frontend / localization thread: src/slam/system.cpp:52-53,68-69).  Each handle owns one CUDA
 *     stream; fls_match is synchronous with respect to the caller.
 */
#ifndef FLS_B200_H
#define FLS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FLS_ABI_VERSION 1

typedef struct fls_handle fls_handle;

typedef enum {
    FLS_OK = 0,
    FLS_ERR_INVALID_ARG = -1,   /* null pointer, bad stride, sentinel ("NaN") parameter left unset */
    FLS_ERR_CUDA = -2,          /* a CUDA runtime call failed; fls_last_error() has the text */
    FLS_ERR_NO_DEVICE = -3,     /* no sm_90 device visible — the product has NO CPU fallback */
    FLS_ERR_UNSUPPORTED = -4,   /* method / mode not implemented by this build */
    FLS_ERR_NO_MAP = -5,        /* Match before AddCloudToLocalMap (reference: CHECK(!grids_.empty())) */
    FLS_ERR_CAPACITY = -6,      /* voxel count would exceed the LRU capacity (eviction not emulated on device) */
    FLS_ERR_TOO_FEW_POINTS = -7 /* reference: CHECK_GT(ordered_cloud_.size(), 10u) icp_optimized.h:55 */
} fls_status;

/* Mode strings of include/common/constant_variable.h:21-25, in the same order as SURVEY.md §8b. */
typedef enum {
    FLS_ICP_P2P = 0,      /* kIcpOptimized       -> IcpOptimized<double>          */
    FLS_NDT = 1,          /* kIncrementalNDT     -> IncrementalNDT                */
    FLS_P2PLANE_IVOX = 2, /* kPointToPlane_IVOX  -> LoamPointToPlaneIVOX<double>  */
    FLS_P2PLANE_KNN = 3,  /* kPointToPlane_KdTree-> LoamPointToPlaneKdtree<double>*/
    FLS_LOAM_FULL = 4     /* kLoamFull_KdTree    -> LoamFull<double>              */
} fls_method;

/* IVoxMap::NearbyType (include/ivox_map/ivox_map.h:24-29) */
typedef enum { FLS_NEARBY_CENTER = 0, FLS_NEARBY6 = 1, FLS_NEARBY18 = 2, FLS_NEARBY26 = 3 } fls_nearby;

/* point record layouts accepted by every `stride_bytes` argument */
#define FLS_LAYOUT_PCL_XYZI 32u /* pcl::PointXYZI: x,y,z,pad | intensity,pad,pad,pad */
#define FLS_LAYOUT_PACKED 16u   /* x,y,z,intensity */

/* All constructor arguments of the five plug-ins (same names as the reference's ctor parameters). */
typedef struct {
    int32_t method;            /* fls_method */
    int32_t device;            /* CUDA device ordinal */
    int32_t localization_mode; /* is_localization_mode: Match never modifies the map */
    int32_t max_iterations;    /* opti_iter_num / max_iterations / max_iteration */
    double position_converge_thres;
    double rotation_converge_thres;

    /* LoamPointToPlaneIVOX / LoamPointToPlaneKdtree / LoamFull (loam_point_to_plane_ivox.h:36-58) */
    double point_to_planar_thres;
    float ivox_resolution;    /* 0.5  (loam_point_to_plane_ivox.h:55) */
    int32_t ivox_nearby;      /* FLS_NEARBY18 (:56) */
    int64_t ivox_capacity;    /* 1000000 voxels (ivox_map.h:35) */
    float ivox_max_range;     /* 5.0 (ivox_map.h:58) */
    int32_t ivox_k;           /* 5 (ivox_map.h:57) */

    /* IncrementalNDT (incremental_ndt.h:22-26) */
    double ndt_voxel_size;
    double ndt_outlier_thres;
    int32_t ndt_min_points_in_voxel;
    int32_t ndt_max_points_in_voxel;
    int32_t ndt_min_effective_pts;
    int32_t ndt_capacity;

    /* IcpOptimized (icp_optimized.h:24-27) */
    double icp_max_correspond_distance;
    double rot_thre_add_cloud;
    double dist_thre_add_cloud;
    int32_t local_map_size;

    /* shared down-sampling leafs */
    float source_cloud_filter_size; /* ICP / NDT: VoxelGridCloud at the top of Match */
    float map_cloud_filter_size;    /* ICP / kd-tree maps */

    /* LoamFull (loam_full_kdtree.h:33-44) */
    double point_search_thres;
    double line_ratio_thres;
    float corner_map_filter_size;
    int32_t corner_local_map_size;

    uint32_t flags; /* FLS_FLAG_* */
    uint32_t reserved[7];
} fls_config;

#define FLS_FLAG_ITER_LOG 1u /* keep per-iteration H, g, dx, n_valid, sum_res for fls_get_iter_log */
#define FLS_FLAG_PROFILE 2u  /* bracket the fused Gauss-Newton launch of a Match with CUDA events (fills kernel_ms / kernel_launches) */

typedef struct {
    int32_t iterations;   /* GN iterations executed */
    int32_t converged;    /* the bool Match returns */
    int64_t n_source;     /* points entering the GN loop (after Match's own VoxelGridCloud where the plug-in has one) */
    int64_t n_valid;      /* number_valid_planar_ / effective_num of the last executed iteration */
    double sum_residual;  /* overall_res_planar_ / total_res of the last executed iteration */
    float gpu_ms;         /* device time of this call's kernels (CUDA events on the handle's stream) */
    int32_t gpu_launches; /* kernels of this library launched by the call */
    int64_t h2d_bytes;    /* bytes copied host->device by the call */
    int64_t d2h_bytes;    /* bytes copied device->host by the call */
    float kernel_ms;      /* FLS_FLAG_PROFILE: device time of the fused Gauss-Newton launch (all executed iterations) */
    int32_t kernel_launches; /* FLS_FLAG_PROFILE: how many launches kernel_ms covers (1: one launch runs every iteration) */
    int64_t algo_bytes;   /* FLS_FLAG_PROFILE: algorithmic bytes those launches moved (DESIGN.md "roofline accounting") */
} fls_match_stats;  /* valid only when the call returned FLS_OK */

typedef struct {
    double H[36]; /* row-major 6x6 (symmetric) */
    double g[6];
    double dx[6];
    double sum_residual;
    int64_t n_valid;
} fls_iter_log;

typedef struct {
    int64_t n_points;    /* map points resident on the device */
    int64_t n_voxels;    /* occupied voxels (iVox / NDT) or grid cells (ICP) */
    int64_t table_slots; /* open-addressing table size */
    int64_t bytes;       /* device bytes held by the map */
    int64_t incremental_inserts; /* LOAM-iVox mapping mode: inserts that only rewrote the touched voxels and the centres around them */
    int64_t full_builds;         /* ... and inserts (incl. the first) that rebuilt table + stencil lists from all points */
} fls_map_info;

/* Fill `cfg` with the parameter set the reference ships for `method` (config YAMLs; SURVEY.md App. B). */
int fls_config_default(fls_config* cfg, int method);

int fls_create(const fls_config* cfg, fls_handle** out);
void fls_destroy(fls_handle* h);

/* AddCloudToLocalMap.  `n_clouds` is the initializer_list arity (1, or 2 = {planar, corner} for LoamFull).
 * Clouds are in the map frame. */
int fls_add_cloud(fls_handle* h, int n_clouds, const void* const* pts, const size_t* n, size_t stride_bytes);

/* Match.  Pass the PointcloudCluster members the plug-in reads (include/lidar/pointcloud_cluster.h:13-26):
 * ordered_cloud_ (ICP, NDT), planar_cloud_ (P2PLANE_*), corner_cloud_ + planar_cloud_ (LOAM_FULL); unused
 * ones may be NULL/0.  T is in-out and written even when *converged == 0 (icp_optimized.h:152,
 * incremental_ndt.h:307,334, loam_point_to_plane_ivox.h:198). */
int fls_match(fls_handle* h, const void* ordered, size_t n_ordered, const void* planar, size_t n_planar, const void* corner, size_t n_corner,
              size_t stride_bytes, double T_colmajor[16], int* converged, fls_match_stats* stats);

/* Same as fls_match but the scan is already resident in device memory as packed float4 {x,y,z,i}
 * (the `value` leg of bench.py).  `d_points` is a device pointer on the handle's device.  The LOAM plug-ins keep the pointer for a
 * later fls_fitness (the source cloud of the last Match, as upstream keeps source_cloud_ptr_): the buffer must stay valid and
 * unchanged until the next Match on the handle, or fls_fitness must not be called.  `stats` (here and in every Match entry) is
 * meaningful only when the call returns FLS_OK. */
int fls_match_device(fls_handle* h, const void* d_points, size_t n, double T_colmajor[16], int* converged, fls_match_stats* stats);

/* fls_match with the three PointcloudCluster clouds already in device memory on the handle's device (packed float4 {x,y,z,i}); the
 * plug-in reads the same clouds as in fls_match (unused ones may be NULL/0).  This is the device-resident Match of FLS_LOAM_FULL, which
 * reads two clouds (fls_match_device takes one and returns FLS_ERR_UNSUPPORTED for it), e.g. straight from fls_preprocess_loam's
 * device outputs.  The LOAM plug-ins keep the planar pointer for a later fls_fitness, as in fls_match_device: the buffer must stay
 * valid and unchanged until the next Match on the handle, or fls_fitness must not be called. */
int fls_match_cluster_device(fls_handle* h, const void* d_ordered, size_t n_ordered, const void* d_planar, size_t n_planar, const void* d_corner,
                             size_t n_corner, double T_colmajor[16], int* converged, fls_match_stats* stats);

/* GetFitnessScore(max_range): FLT_MAX when unsupported / no inliers, as upstream. */
int fls_fitness(fls_handle* h, float max_range, float* score);

/* Batched Match for throughput (the benchmark entry SURVEY.md §8b names): `n_scans` (<= 64) independent scans, each with its
 * own in-out pose T[s*16 .. s*16+15], converged[s] and stats[s], matched against the same map in ONE persistent launch.
 * Implemented for FLS_P2PLANE_IVOX (one persistent work-queue kernel for the batch) and FLS_NDT (one cooperative launch, a
 * sub-grid and a Gauss-Newton loop per scan); more than one scan requires localization_mode (Match must not modify the map).
 * For the LOAM-iVox plug-in the entry reads the planar clouds, for NDT the ordered clouds of the scans.
 * Call-level figures (gpu_ms, gpu_launches, byte counts, kernel_ms) are reported in stats[0]; per-scan fields everywhere.
 * Results are identical to n_scans separate fls_match calls.  The _device variant takes device pointers to packed float4 scans. */
int fls_match_batch(fls_handle* h, int n_scans, const void* const* planar, const size_t* n, size_t stride_bytes, double* T_colmajor,
                    int* converged, fls_match_stats* stats);
/* fls_match_batch in two halves, so that a caller with two handles overlaps the host->device copy of one batch with the kernels of
 * the other: _begin enqueues the copies, the matching and the read-back on the handle's stream and returns without waiting (the
 * host buffers — pinned, to be asynchronous — and `n` must stay valid until _end); _end waits and fills T / converged / stats like
 * fls_match_batch.  FLS_P2PLANE_IVOX in localization mode; one batch in flight per handle. */
int fls_match_batch_begin(fls_handle* h, int n_scans, const void* const* planar, const size_t* n, size_t stride_bytes, const double* T_colmajor);
int fls_match_batch_begin_device(fls_handle* h, int n_scans, const void* const* d_planar, const size_t* n, const double* T_colmajor);
int fls_match_batch_end(fls_handle* h, double* T_colmajor, int* converged, fls_match_stats* stats);
int fls_match_batch_device(fls_handle* h, int n_scans, const void* const* d_planar, const size_t* n, double* T_colmajor, int* converged,
                           fls_match_stats* stats);

/* Device-side results for a consumer that lives on the GPU (the per-batch NCCL all-gather of poses, SURVEY.md §8e): once set,
 * every Match additionally writes, for scan s of the call, 18 doubles at d_results + 18*s — the column-major Mat4d pose
 * (what T receives), converged (0/1), iterations — from inside the Gauss-Newton kernel when the scan stops; the buffer is
 * complete when the Match call returns.  `capacity_scans` bounds s; NULL unsets.  The buffer is owned by the caller and must
 * stay valid until unset or the handle is destroyed. */
int fls_set_result_buffer_device(fls_handle* h, double* d_results, size_t capacity_scans);

/* per-iteration log of the last fls_match (needs FLS_FLAG_ITER_LOG; batch: scan 0); returns the number of entries written */
int fls_get_iter_log(const fls_handle* h, fls_iter_log* out, int capacity);
/* the same for scan `scan` of the last Match call (the batch entries of FLS_P2PLANE_IVOX and FLS_NDT keep one log per scan);
 * FLS_ERR_INVALID_ARG when `scan` is not below that call's n_scans; a Match that fails after its launch leaves no log */
int fls_get_iter_log_scan(const fls_handle* h, int scan, fls_iter_log* out, int capacity);

int fls_get_map_info(const fls_handle* h, fls_map_info* out);
/* Keys (x, y, z voxel coordinates, int32 triples) of the voxels the map currently holds, in no particular order: FLS_NDT
 * (IncrementalNDT::grids_, incremental_ndt.h:393) and FLS_P2PLANE_IVOX (IVoxMap::grids_map_, ivox_map.h:70).  Introspection for the
 * LRU parity tests; writes at most `capacity` triples and returns the voxel count in *n. */
int fls_get_voxel_keys(fls_handle* h, int32_t* keys_xyz, size_t capacity, size_t* n);
/* One live voxel of the FLS_NDT map (IncrementalNDT::VoxelData, incremental_ndt.h:65-85 upstream).  mu and info are what Match
 * reads: the mean and the symmetrised information matrix (xx, xy, xz, yy, yz, zz); both are zero while estimated == 0, as in a
 * fresh VoxelData.  num_points is num_points_; carry_count the points buffered for a later estimate (points_.size(); 0 once the
 * voxel is frozen past max_points_in_voxel, whose later points upstream keeps but never reads). */
typedef struct {
    int32_t key[3];
    int32_t estimated;
    int32_t num_points;
    int32_t carry_count;
    double mu[3];
    double info[6];
} fls_ndt_voxel;
/* Every live voxel of the FLS_NDT map, sorted by key (x, then y, then z).  Read-only introspection for the map parity tests; writes at
 * most `capacity` records and returns the voxel count in *n.  FLS_ERR_UNSUPPORTED for other plug-ins. */
int fls_get_ndt_voxels(fls_handle* h, fls_ndt_voxel* out, size_t capacity, size_t* n);

/* Test hook: one Gauss-Newton step (the 6x6 solve, pose update and stop rule every persistent Match kernel runs after its sums) on
 * N independent cases, one device thread per case, in one launch on the handle's device and stream.  Read-only: the handle's map
 * and state are untouched.  A case is the pre-step state of a loop, the parameters of fls_config that the step reads, and the
 * reduced totals of one iteration in the kernels' layout: 21 upper-triangular entries of H (row by row), 6 of g, the sum of
 * residuals, n_valid and two traffic counters. */
typedef struct {
    int32_t method;         /* fls_method */
    int32_t max_iterations;
    int32_t min_effective;  /* NDT: ndt_min_effective_pts; the LOAM plug-ins: 50 */
    int32_t iter;           /* iterations executed before this step */
    double rot_thres, pos_thres;
    double R[9];            /* row-major rotation before the step */
    double t[3];
    double last_rot, last_pos; /* LOAM: the dx norms of the previous iteration (0 before iteration 0) */
    double tot[31];         /* H (21), g (6), valid count, sum of residuals, candidates, table hits */
} fls_gn_step_case;
typedef struct {
    double R[9], t[3];      /* state after the step (row-major R) */
    double dx[6], H[36], g[6];
    double last_rot, last_pos;
    double published[13];   /* what the step published for the other CTAs: R[9], t[3], stop word (1.0 / 0.0) */
    double result[18];      /* the result record (fls_set_result_buffer_device layout); NaN where the step wrote none */
    double det_spd;         /* product of the LDL^T pivots when the fast path accepted the system, else 0 */
    int64_t n_valid;
    int32_t iter, converged, failed, done;
    int32_t spd;            /* the register LDL^T fast path accepted the system (else the pivoting solver ran) */
    int32_t published_ok;   /* every published record carried the iteration's tag */
} fls_gn_step_out;
int fls_gn_step_probe(fls_handle* h, const fls_gn_step_case* cases, size_t n, fls_gn_step_out* out);
/* The points the FLS_P2PLANE_IVOX map holds (packed x, y, z, intensity), in insertion order; at most `capacity` points are written, the
 * count is returned in *n.  Introspection for the map parity tests. */
int fls_get_map_points(fls_handle* h, float* xyzi, size_t capacity, size_t* n);

/* Test hook: IVoxMap::GetClosestPoint for a batch of map-frame queries (packed float4 host arrays).
 * out_pts receives n*k packed points (unused slots zero), out_count the number found per query. */
/* IVoxMap::AddPoints (include/ivox_map/ivox_map.h:44, src/ivox_map/ivox_map.cpp:122-143): the points enter the FLS_P2PLANE_IVOX map as
 * they are (map frame, no insertion rule), in order, with upstream's LRU policy at `ivox_capacity`.  The map of a handle in
 * localization mode is otherwise replaced by fls_add_cloud; this entry appends. */
int fls_ivox_add_points(fls_handle* h, const void* pts, size_t n, size_t stride_bytes);
int fls_ivox_knn(fls_handle* h, const void* queries, size_t n, size_t stride_bytes, int k, float* out_pts, int32_t* out_count);

/* VoxelGridCloud on the device: `out` must hold n packed float4 records; *n_out receives the count. */
int fls_voxel_grid(int device, const void* pts, size_t n, size_t stride_bytes, float leaf, float* out, size_t* n_out);

/* LOAM feature extraction on the projector's arrays (PointcloudCluster::point_depth_vec_, point_col_index_vec_,
 * row_start_index_vec_, row_end_index_vec_).  corner_idx / planar_idx receive indices into the ordered cloud in
 * the reference's emission order; capacities: corner >= 120*V, planar >= n + 6*V. */
typedef struct {
    float corner_threshold;
    float planar_threshold;
    int32_t device;
    int32_t reserved;
} fls_feature_cfg;
int fls_extract_features(const fls_feature_cfg* cfg, const float* depth, const int32_t* col, size_t n, const int32_t* row_start,
                         const int32_t* row_end, int32_t n_rows, int32_t* corner_idx, size_t* n_corner, int32_t* planar_idx, size_t* n_planar,
                         fls_match_stats* stats);

/* PointcloudProjector::Project (src/loam/pointcloud_projector.cpp:32-133): raw cloud + ring per point (firing order) ->
 * ordered_cloud_ (packed float4, capacity n_rows*n_cols), point_depth_vec_ / point_col_index_vec_ (n_rows*n_cols entries, the
 * first *n_ordered meaningful), row_start_index_vec_ / row_end_index_vec_ (n_rows).  Without an IMU buffer the de-skew of :100-103
 * is the identity; fls_project_imu below applies it. */
int fls_project(int device, const void* raw, const int32_t* ring, size_t n, size_t stride_bytes, int32_t n_rows, int32_t n_cols,
                float horizontal_resolution, float min_distance, float max_distance, float* ordered, float* depth, int32_t* col,
                int32_t* row_start, int32_t* row_end, size_t* n_ordered);

/* Localization mode, the map side (Localization::LoadLocalMap, src/slam/localization.cpp:364-410, and its callers :127-135, :216-224):
 * fls_set_global_map keeps the global map resident in device memory; fls_update_local_map(T) re-cuts the local map — a +-100 m
 * pcl::CropBox around the translation of T, input order kept — when there is none yet or the pose is within 50 m of one of its
 * edges, and hands it to AddCloudToLocalMap of the handle's plug-in without a host round trip.  *updated = 1 when a new local map
 * was cut (need_update_local_map_), *n_local its size (0: LoadLocalMap returned an empty cloud; the matcher's map is untouched). */
int fls_set_global_map(fls_handle* h, const void* pts, size_t n, size_t stride_bytes);
int fls_update_local_map(fls_handle* h, const double T_colmajor[16], int* updated, size_t* n_local);

/* PCD v0.7 files as pcl::io::loadPCDFile / savePCDFileBinary read and write them for x y z intensity clouds
 * (include/common/keyframe.h:24-74, src/slam/localization.cpp:283-300): fls_pcd_read fills at most `capacity` packed
 * x, y, z, intensity records (DATA ascii or binary; extra fields are skipped, a missing intensity reads 0) and returns the point
 * count of the file in *n; fls_pcd_write writes DATA binary. */
int fls_pcd_read(const char* path, float* xyzi, size_t capacity, size_t* n);
int fls_pcd_write(const char* path, const float* xyzi, size_t n);

/* IMU orientation samples around a scan — what LidarDistortionCorrector reads through its DataSearcher<IMUData>
 * (include/lidar/lidar_distortion_corrector.h:11-48, src/lidar/lidar_distortion_corrector.cpp:19-64): time stamps in microseconds,
 * ascending (equal neighbours allowed; a stamp followed by a smaller one is rejected with FLS_ERR_INVALID_ARG, where upstream's
 * downward scan would pick some pair anyway; so is a null time or quaternion array when n_imu > 0), unit quaternions in Eigen coefficient order x, y, z, w, the reference time of the scan (SetRefTime) and the
 * lidar -> imu extrinsic (column-major 4x4).  n_imu == 0 (or a NULL pointer to the struct): no de-skew, points pass unchanged. */
typedef struct {
    const uint64_t* imu_time_us;
    const double* imu_quat_xyzw;
    size_t n_imu;
    uint64_t ref_time_us;
    double T_lidar_to_imu[16];
} fls_imu_buffer;

/* PreProcessing::Run, the branch of the plug-ins that take no features (src/slam/preprocessing.cpp:181-225): per raw point
 * {x, y, z, intensity, time-relative-to-ref [s]} (5 floats, firing order): range gate [min_distance, max_distance], IMU de-skew
 * (a point whose time is outside the IMU buffer is dropped), ordered_cloud_ = every kept point, planar_cloud_ = the kept points
 * whose RAW index is a multiple of jump_span, then pcl::VoxelGrid(planar_leaf).  Outputs: packed x, y, z, intensity records,
 * each buffer with room for n points.  When ref_time_us is outside the IMU buffer upstream skips the scan: both counts are 0. */
int fls_preprocess(int device, const float* raw_xyzit, size_t n, const fls_imu_buffer* imu, float min_distance, float max_distance,
                   int32_t jump_span, float planar_leaf, float* ordered, size_t* n_ordered, float* planar, size_t* n_planar);

/* fls_project with the per-point de-skew of pointcloud_projector.cpp:100-103: `time` holds the time of every raw point relative to
 * ref_time_us [s].  A point whose time is outside the IMU buffer does not claim its cell; the depth of a cell stays the range of
 * the raw point (:57, :105). */
int fls_project_imu(int device, const void* raw, const int32_t* ring, const float* time, size_t n, size_t stride_bytes, const fls_imu_buffer* imu,
                    int32_t n_rows, int32_t n_cols, float horizontal_resolution, float min_distance, float max_distance, float* ordered,
                    float* depth, int32_t* col, int32_t* row_start, int32_t* row_end, size_t* n_ordered);

/* PreProcessing::Run, the LoamFull branch (src/slam/preprocessing.cpp:226-237), in one device call: fls_project_imu (range gate,
 * projection, de-skew) -> fls_extract_features -> corner_cloud_ = VoxelGrid(corner_leaf), planar_cloud_ = VoxelGrid(planar_leaf).
 * The outputs are bit-identical to that chain of per-stage calls with the features gathered from ordered_cloud_ in between; no point
 * data returns to the host between the stages.  Inputs are those of fls_project_imu (`time` may be NULL without de-skew; imu == NULL
 * or n_imu == 0: no de-skew; a reference time outside the IMU buffer gives empty clouds).  Outputs, packed x, y, z, intensity:
 * `corner` / `planar` on the host and `d_corner` / `d_planar` in device memory on cfg->device; any of the four may be NULL, not all.
 * Capacities: corner >= 120 * n_rows records, planar >= n_rows * n_cols records.  A ring or block too long for the feature kernels'
 * shared memory returns FLS_ERR_UNSUPPORTED with both counts 0 and no output written.  stats: gpu_ms, gpu_launches, h2d_bytes,
 * d2h_bytes, n_source = n, algo_bytes (sum of the three stages). */
typedef struct {
    int32_t device;
    int32_t n_rows, n_cols;       /* LidarModel vertical_scan_num_ / horizon_scan_num_ */
    float horizontal_resolution;  /* radians per column */
    float min_distance, max_distance;
    float corner_threshold, planar_threshold; /* frontend/feature/corner_thres, planar_thres */
    float corner_leaf, planar_leaf;           /* frontend/feature/corner_voxel_filter_size, planar_voxel_filter_size */
    uint32_t reserved[4];
} fls_loam_frontend_cfg;
int fls_preprocess_loam(const fls_loam_frontend_cfg* cfg, const void* raw, const int32_t* ring, const float* time, size_t n, size_t stride_bytes,
                        const fls_imu_buffer* imu, float* corner, float* planar, float* d_corner, float* d_planar, size_t* n_corner,
                        size_t* n_planar, fls_match_stats* stats);

/* ---- PreProcessing::ConvertMessageToCloud on the device (src/slam/preprocessing.cpp:262-571) ---- */

/* LidarModel::LidarSensorType (include/lidar/lidar_model.h:25), same order */
typedef enum {
    FLS_LIDAR_VELODYNE = 0,
    FLS_LIDAR_OUSTER = 1,
    FLS_LIDAR_LIVOX_AVIA = 2,
    FLS_LIDAR_ROBOSENSE = 3,
    FLS_LIDAR_LEISHEN = 4,
    FLS_LIDAR_LIVOX_MID_360 = 5,
    FLS_LIDAR_NONE = 6
} fls_lidar_type;

/* sensor_msgs/PointField datatypes */
#define FLS_PF_INT8 1u
#define FLS_PF_UINT8 2u
#define FLS_PF_INT16 3u
#define FLS_PF_UINT16 4u
#define FLS_PF_INT32 5u
#define FLS_PF_UINT32 6u
#define FLS_PF_FLOAT32 7u
#define FLS_PF_FLOAT64 8u

typedef struct {
    const char* name; /* NUL-terminated */
    uint32_t offset;
    uint32_t datatype; /* FLS_PF_* */
    uint32_t count;
    uint32_t reserved;
} fls_point_field;

/* sensor_msgs/PointCloud2.  `data` holds height * row_step bytes: host memory, or a device pointer on cfg->device when
 * data_on_device is 1.  stamp_us is header.stamp.toNSec() / 1000, the stamp pcl_conversions gives the PCL cloud. */
typedef struct {
    const void* data;
    int32_t data_on_device;
    uint32_t height, width, point_step, row_step;
    int32_t is_dense, is_bigendian;
    uint32_t n_fields;
    const fls_point_field* fields;
    uint64_t stamp_us;
    uint32_t reserved[4];
} fls_pointcloud2;

typedef struct {
    int32_t device;
    int32_t lidar_type;       /* fls_lidar_type */
    int32_t n_rows;           /* LidarModel vertical_scan_num_ */
    float lower_angle, v_res; /* LidarModel lower_angle_ / v_res_, read for FLS_LIDAR_NONE only */
    double time_scale;        /* lidar_point_time_scale_ (include/slam/config_parameters.h:69) */
    uint32_t reserved[4];
} fls_convert_cfg;

/* What PreProcessing::Run derives from the converted cloud before the IMU gate (preprocessing.cpp:86-104). */
typedef struct {
    uint64_t stamp_us;          /* header.stamp of the converted cloud (RoboSense: uint64(first kept timestamp * 1e6), :376) */
    uint64_t start_us, end_us;  /* cloud_start_timestamp / cloud_end_timestamp after the one-sided widening of :100-104 */
    float min_time, max_time;   /* GetLidarPointMinMaxOffsetTime (:554-571) */
    int32_t valid;              /* 0 when no point is kept: the other fields are 0 and stamp_us is the message's */
    int32_t recomputed;         /* ComputePointOffsetTime (:513-552) replaced the offsets (the last point's time was <= 0) */
    uint32_t reserved[2];
} fls_convert_result;

/* ConvertMessageToCloud: pcl::fromROSMsg into the sensor's point type (a struct field reads the first message field with its name,
 * datatype and a count of 0 or 1, else 0), the sensor's filter (NaN removal when not dense, the Livox Avia line / tag filter, the
 * ring of FLS_LIDAR_NONE from elevation), ring and time, and ComputePointOffsetTime(cloud, 10.0) when the last kept point's time is
 * <= 0.  Outputs, *n records: packed float4 {x, y, z, intensity}, int32 ring, float time, on the host (xyzi / ring / time) and / or in
 * device memory on cfg->device (d_*); any of the six may be NULL.  Capacities: width * height records.  The host copies cover the whole
 * capacity (the call waits once, at its end).  An empty message or one with no kept point returns FLS_OK with *n = 0 and
 * result->valid = 0.  FLS_ERR_INVALID_ARG when a field does not fit in point_step or row_step < width * point_step;
 * FLS_ERR_UNSUPPORTED for a big-endian message.  stats: gpu_ms, gpu_launches, h2d_bytes, d2h_bytes, n_source, algo_bytes. */
int fls_convert_cloud(const fls_convert_cfg* cfg, const fls_pointcloud2* msg, float* xyzi, int32_t* ring, float* time, float* d_xyzi,
                      int32_t* d_ring, float* d_time, size_t* n, fls_convert_result* result, fls_match_stats* stats);

/* fls_preprocess_loam on a cloud already in device memory on cfg->device (e.g. fls_convert_cloud's device outputs): packed float4
 * d_xyzi, int32 d_ring and float d_time (may be NULL without de-skew).  Nothing is uploaded but the IMU buffer; the stages and the
 * outputs are those of fls_preprocess_loam on the same records. */
int fls_preprocess_loam_device(const fls_loam_frontend_cfg* cfg, const float* d_xyzi, const int32_t* d_ring, const float* d_time, size_t n,
                               const fls_imu_buffer* imu, float* corner, float* planar, float* d_corner, float* d_planar, size_t* n_corner,
                               size_t* n_planar, fls_match_stats* stats);

/* fls_preprocess on a cloud already in device memory on `device`: packed float4 d_xyzi and float d_time (relative time [s]; may be
 * NULL without de-skew).  ordered_cloud_ goes to `ordered` (host) and / or `d_ordered` (device), planar_cloud_ to `planar` and / or
 * `d_planar`; each needs room for n records and any of the four may be NULL, not all (the counts are returned either way).  Outputs equal fls_preprocess's on the same
 * records; the planar device output is what fls_match_device takes. */
int fls_preprocess_device(int device, const float* d_xyzi, const float* d_time, size_t n, const fls_imu_buffer* imu, float min_distance,
                          float max_distance, int32_t jump_span, float planar_leaf, float* ordered, float* d_ordered, size_t* n_ordered, float* planar,
                          float* d_planar, size_t* n_planar);

/* ---- Keyframe maps on the device: System::SaveMap, System::VisualizeGlobalMap, LoopClosure::GetSubMap ---- */

/* A device-resident store of keyframe clouds (the ordered_cloud_ every KeyFrame keeps, include/common/keyframe.h:31-74), separate from
 * any fls_handle: upstream reads keyframes from the loop-closure thread, the visualization thread and the save-map service, none of
 * which owns a matcher.  The store owns one CUDA stream and a mutex; calls from several host threads are serialized.  Clouds are held
 * as packed float4 {x, y, z, intensity} in one arena of `capacity_points` records, fixed at creation.  Poses are not stored: every
 * assemble call takes the current poses of its selection (upstream re-optimises them after each loop closure, system.cpp:711-717). */
typedef struct fls_keyframes fls_keyframes;

/* capacity_points in [1, 2^32 - 1]; FLS_ERR_NO_DEVICE when `device` is not a visible CUDA device. */
int fls_keyframes_create(int device, size_t capacity_points, fls_keyframes** out);
void fls_keyframes_destroy(fls_keyframes* s);
/* Append keyframe `id`'s ordered cloud, as System keeps keyframes_ indexed by id (include/slam/system.h:187): ids are dense and
 * appended in order, so `id` must equal the current count (else FLS_ERR_INVALID_ARG).  FLS_ERR_CAPACITY when the arena cannot take n
 * more records (the store does not grow).  An empty cloud is a valid keyframe.  _add reads host records `stride_bytes` apart
 * (FLS_LAYOUT_*); _add_device copies n packed float4 records from device memory on the store's device, e.g. the ordered or planar
 * output of fls_preprocess_loam_device, so the cloud never passes through the host.  Both return once the copy is complete. */
int fls_keyframes_add(fls_keyframes* s, int64_t id, const void* pts, size_t n, size_t stride_bytes);
int fls_keyframes_add_device(fls_keyframes* s, int64_t id, const void* d_pts, size_t n);
/* number of keyframes and of arena records in use (either pointer may be NULL) */
int fls_keyframes_count(fls_keyframes* s, size_t* n_keyframes, size_t* n_points);
/* map = [base] ++ concat_k TransformPointCloud(VoxelGridCloud(cloud[ids[k]], leaf), T[k]);  if final_leaf > 0: map = VoxelGridCloud(map,
 * final_leaf).  This is the loop of System::SaveMap (src/slam/system.cpp:310-316, leaf = final_leaf = 0.3), of one round of
 * System::VisualizeGlobalMap (src/slam/system.cpp:884-892, base = the running global_map, leaf = final_leaf = the visualization
 * resolution) and of LoopClosure::GetSubMap (src/slam/loop_closure.cpp:217-230, leaf 0.2, no final pass).
 *   ids / T_colmajor: n_ids keyframe ids (below the count; repeats allowed) and their poses, 16 doubles each (Eigen Mat4d memory).
 *       The transform is TransformPointCloud's (include/common/pointcloud_utility.h:141-158): R and t cast to float first.
 *   Each keyframe is filtered on its own; one whose extent overflows at `leaf` (PCL's dx*dy*dz > INT_MAX) keeps its points unchanged
 *       and in input order, as PCL does.  The output is in selection order and, within a keyframe, in ascending cell order.
 *   d_base / n_base: optional device records (packed float4, on the store's device) placed before the keyframes; they must not overlap
 *       d_out.  Two caller buffers used in turn carry a running global map from one round to the next.
 *   final_leaf: <= 0 for no final pass.
 *   out (host) and / or d_out (device, on the store's device) receive the map; `capacity` is the room of each given buffer in records.
 *       *n_out always receives the size of the map; when it exceeds `capacity` the call returns FLS_ERR_CAPACITY and writes nothing
 *       (with both buffers NULL and capacity 0 this is a size query).
 * Device inputs (d_base) must be complete when the call is made.  The number of host waits and kernel launches does not depend on
 * n_ids.  stats (optional): gpu_ms, gpu_launches, h2d_bytes, d2h_bytes, n_source = records entering the per-keyframe pass, n_valid =
 * records after it, iterations = the host waits (stream synchronisations) of the call.  FLS_ERR_CAPACITY also when the selection
 * holds more than 2^31 - 1 records. */
int fls_keyframes_assemble(fls_keyframes* s, const int64_t* ids, size_t n_ids, const double* T_colmajor, float leaf, float final_leaf,
                           const void* d_base, size_t n_base, float* out, float* d_out, size_t capacity, size_t* n_out, fls_match_stats* stats);

const char* fls_strerror(int status);
const char* fls_last_error(void); /* thread-local text of the last CUDA failure */
int fls_abi_version(void);
int fls_device_count(void);

#ifdef __cplusplus
}
#endif
#endif /* FLS_B200_H */
