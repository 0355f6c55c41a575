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
 *   fls_*_motion               <- the five de-skewing entries above with the sensor's translation over the sweep added (not
 *                                 upstream: lidar_distortion_corrector.cpp:34 leaves it as a TODO)
 *   fls_keyframes_*            <- the keyframe-map loops of System::SaveMap (src/slam/system.cpp:299-341),
 *                                 System::VisualizeGlobalMap (src/slam/system.cpp:847-896) and
 *                                 LoopClosure::GetSubMap (src/slam/loop_closure.cpp:179-231)
 *   fls_relocalize / _device   <- Localization::Init's Match + GetFitnessScore(2.0) < 1.0 (src/slam/localization.cpp:135-140),
 *                                 searching an x-y-yaw grid around the given pose
 *   fls_relocalize_wide /      <- the same over a whole local map (up to 2^31 hypotheses), by exact branch and bound
 *   _wide_device
 *   fls_relocalize_multi /     <- the same around up to 64 guesses at once (the top-k candidates of fls_keyframes_place_query),
 *   _multi_device                 ranked together in one search and refined by one batch Match
 *   fls_keyframes_detect_loop  <- LoopClosure::DetectByFeature (src/slam/loop_closure.cpp:62-64, a stub upstream), by Scan Context
 *   fls_keyframes_place_query  <- the keyframe a scan was taken near, and its yaw: the guess of fls_relocalize without a clicked pose
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
    FLS_ERR_CAPACITY = -6,      /* voxel count would exceed the LRU capacity (eviction not emulated on device); also fls_relocalize_wide */
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
#define FLS_FLAG_INFORMATION 4u /* evaluate every Match's information matrix at its returned pose for fls_get_information */

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

/* FLS_FLAG_INFORMATION: how well a scan constrains the pose T_final its Match returned (DESIGN.md §3.13).  The terms are those the
 * plug-in's Gauss-Newton iteration builds from a fresh correspondence search at T_final (same neighbour search, gates, residual
 * and weight W; LoamFull: its planar and corner terms); a point without a correspondence adds nothing.  In the fusion
 * parameterization: order [dtheta; dp], T_final perturbed as R <- R * Exp(dtheta), p <- p + dp (p in the world frame):
 *   H = sum J_i^T W_i J_i,   g = sum J_i^T W_i r_i.
 * Scaling H to a covariance is the caller's choice: NDT's residual is already Mahalanobis (W = the voxel information), the LOAM
 * and ICP residuals are metres with W = 1. */
typedef struct {
    double H[36];         /* row-major 6x6, symmetric */
    double g[6];
    double sum_residual;  /* LOAM: sum |d|, NDT: sum of e^T W e, ICP: sum ||e|| over the contributing terms */
    int64_t n_valid;      /* contributing terms: points (LOAM, ICP; LoamFull: planar + corner), point-voxel pairs (NDT) */
    int32_t valid;        /* 1: the record belongs to the last Match call; 0: no record (see fls_get_information) */
    int32_t pad;
} fls_information;

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
 * Implemented for FLS_P2PLANE_IVOX (one persistent work-queue kernel for the batch) and for FLS_NDT, FLS_ICP_P2P and
 * FLS_P2PLANE_KNN (one cooperative launch, a sub-grid and a Gauss-Newton loop per scan); more than one scan requires
 * localization_mode (Match must not modify the map), and a batch of one is fls_match.  The LOAM-iVox and kd-tree point-to-plane
 * plug-ins read each scan as its planar cloud, NDT and ICP as its ordered cloud (voxel-filtered once per distinct (pointer, count)).
 * FLS_ICP_P2P: FLS_ERR_TOO_FEW_POINTS when any scan has 10 points or fewer and FLS_ERR_NO_MAP before a map, both before anything is
 * uploaded or launched (T untouched).  FLS_LOAM_FULL reads two clouds per scan: FLS_ERR_UNSUPPORTED for any n_scans, no side effect.
 * After a batch, fls_fitness scores scan 0's final pose on scan 0's source.
 * Call-level figures (gpu_ms, gpu_launches, byte counts, kernel_ms) are reported in stats[0]; per-scan fields everywhere.
 * Results equal n_scans separate fls_match calls: the same converged flag, iterations and n_valid, poses within fp64 rounding (a
 * sub-grid folds its CTA rows in another order than a whole grid).  The _device variant takes device pointers to packed float4 scans. */
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

/* Relocalization from a coarse pose (Localization::Init's "2D Pose Estimate", src/slam/localization.cpp:114-169 upstream, which runs
 * one Match from the clicked pose and accepts it when it converges and GetFitnessScore(2.0) < 1.0).
 *
 * Hypotheses.  With I = floor(xy_radius / xy_step + 1e-9) (0 when xy_radius == 0) and K = floor(min(yaw_range, pi) / yaw_step + 1e-9)
 * (0 when yaw_range == 0), the yaw offsets are psi_k = k * yaw_step for k = -K..K, except that k = -K is left out when yaw_range >= pi
 * and 2 K yaw_step >= 2 pi - 1e-9 (it would repeat +K: the full circle without a duplicate).  Hypothesis (j, i, k) is, in fp64,
 *   R = Rz(psi_k) * R_guess   (row 0: c*g0 - s*g1, row 1: s*g0 + c*g1, row 2: g2, no fused multiply-add)
 *   t = t_guess + (i * xy_step, j * xy_step, 0)        for i, j = -I..I,
 * so z, roll and pitch stay those of the guess.  Index order: yaw fastest, then x (i), then y (j): index = ((j+I)*(2I+1) + (i+I))*n_yaw + k'.
 * Coarse score.  C = VoxelGridCloud(scan, coarse_leaf) with m points; d2 = the fp32 squared distance of each point, moved by the
 * hypothesis cast to float (as fls_fitness moves it), to its nearest fit-cloud point; a point is an inlier when d2 <= max_range.
 * score = (sum of inlier d2 + (m - inliers) * max_range) / m: GetFitnessScore's sum with every outlier counted at the gate.
 * Selection: the n_refine smallest scores, ties to the lower index.  Refinement: one fls_match_batch_device of those poses, the same
 * device scan n_refine times (n_refine == 1: a plain Match).  Fitness: GetFitnessScore(max_range) of each refined pose on the cloud
 * fls_fitness reads after that Match.  Choice: the converged refined pose with the lowest fitness (ties: the better coarse rank), or
 * the lowest fitness when none converged; accepted = converged && fitness < accept_fitness.  T receives the chosen pose even when it
 * is not accepted, as upstream (:160-163).  Afterwards fls_fitness(max_range) returns the reported fitness and a Match behaves as
 * after a plain Match; the map is not modified.  Every score is reproducible bit for bit from call to call.
 *
 * `scan` is the cloud the plug-in's Match reads (planar for FLS_P2PLANE_IVOX, ordered for FLS_NDT), host records of stride_bytes;
 * fls_relocalize_device takes packed float4 device records, which must stay valid until the next Match (as in fls_match_device).
 * Optional outputs, in refinement rank order (rank 0 = best coarse score): refined_T [n_refine*16] column-major poses after the
 * Match, refined_converged, refined_fitness and refined_index (grid index of the start pose) [n_refine]; coarse_scores receives
 * the first min(coarse_cap, n_hypotheses) scores in index order.  An empty scan (or an empty coarse cloud) refines nothing: T is
 * left as given, fitness = FLT_MAX, accepted = 0.  out->host_waits and out->gpu_launches count the call's stream synchronisations
 * and launches: 5 waits for FLS_P2PLANE_IVOX and 7 for FLS_NDT, one more when the fit grid is rebuilt for a new map or max_range.
 * FLS_P2PLANE_IVOX and FLS_NDT in localization mode; FLS_ERR_UNSUPPORTED (no side effect) otherwise; FLS_ERR_NO_MAP before a map;
 * FLS_ERR_INVALID_ARG for a NaN, zero or negative step, leaf or range where it is used, n_refine outside 1..64, more than 2^20
 * hypotheses, or while a batch from fls_match_batch_begin is in flight on the handle.  The step must lie inside the convergence
 * basin of the plug-in's Match: about 1 m and 10 degrees for FLS_P2PLANE_IVOX, 0.5 m and 5 degrees or finer for FLS_NDT. */
typedef struct {
    double xy_radius;      /* hypotheses at guess + (i*xy_step, j*xy_step, 0), |i|,|j| <= floor(xy_radius/xy_step) */
    double xy_step;        /* > 0 (ignored when xy_radius == 0) */
    double yaw_range;      /* yaw offsets k*yaw_step, |k*yaw_step| <= yaw_range; >= pi: the full circle, no duplicate offset */
    double yaw_step;       /* > 0 (ignored when yaw_range == 0) */
    float coarse_leaf;     /* VoxelGridCloud leaf of the scan used for the coarse scores (> 0) */
    float max_range;       /* GetFitnessScore's max_range, for both stages: 2.0 in Localization::Init (:138) */
    float accept_fitness;  /* accepted = converged && fitness < accept_fitness: 1.0 upstream (:140) */
    int32_t n_refine;      /* 1..64 best coarse hypotheses refined by one batch Match */
} fls_reloc_cfg;

typedef struct {
    int64_t n_hypotheses;     /* hypotheses scored */
    int64_t best_hypothesis;  /* grid index of the returned pose's start hypothesis (-1 when nothing was refined) */
    int32_t n_refined;
    int32_t best_rank;        /* its rank among the refined (0 = best coarse score) */
    int32_t converged;
    int32_t accepted;
    float fitness;            /* GetFitnessScore(max_range) at the returned pose */
    float coarse_score;       /* its coarse score */
    int32_t host_waits;       /* stream synchronisations of the call */
    int32_t gpu_launches;
} fls_reloc_result;

int fls_relocalize(fls_handle* h, const void* scan, size_t n, size_t stride_bytes, const fls_reloc_cfg* cfg, double T_colmajor[16],
                   fls_reloc_result* out, double* refined_T, int32_t* refined_converged, float* refined_fitness, int64_t* refined_index,
                   double* coarse_scores, size_t coarse_cap);
int fls_relocalize_device(fls_handle* h, const void* d_scan, size_t n, const fls_reloc_cfg* cfg, double T_colmajor[16], fls_reloc_result* out,
                          double* refined_T, int32_t* refined_converged, float* refined_fitness, int64_t* refined_index, double* coarse_scores,
                          size_t coarse_cap);

/* Relocalization over a whole local map: the hypotheses of fls_relocalize's grid searched by exact branch and bound on the device.
 * It takes the same fls_reloc_cfg, defines the same grid and returns what fls_relocalize would return for that cfg without its
 * 2^20 cap: T, every field of *out, and the refined arrays (the same n_refine hypotheses in the same order, hence the same Match,
 * fitness and choice).  In place of coarse_scores, *evaluations (optional) receives the number of pose evaluations the search ran:
 * lower bounds plus exact scores, against out->n_hypotheses for the exhaustive search.
 *
 * The search.  Aligned blocks of 2^l x 2^l x 2^l hypotheses (x, y, yaw indices) are evaluated at one representative each, from the
 * lowest level with at most 2^20 blocks down to single hypotheses; all representatives of that start level are scored exactly,
 * and U is the n_refine-th smallest of those scores.  A block is dropped when a lower bound on the coarse score of every hypothesis
 * in it exceeds U by a relative 1e-6: the score at the representative, with each point's distance to the fit cloud read from a
 * lower-bound distance lattice and reduced by how far the block's other hypotheses can move that point (plus fp32 rounding).  Every
 * hypothesis that scores at most U survives, so the selection is exact, ties included.  Grids of at most 2^20 hypotheses start at
 * single hypotheses and score every one, as fls_relocalize does.  DESIGN.md §3.11 gives the bound and the lattice.
 *
 * Caps: at most 2^31 hypotheses and floor(xy_radius / xy_step) <= 32767 (else FLS_ERR_INVALID_ARG).  FLS_ERR_CAPACITY when more
 * than 2^23 blocks survive one level, before any Match runs (T, the map and fls_fitness are then as before the call): a map and scan
 * so featureless that most of a very large grid cannot be told apart from the best.  The lattice is built by the first call past 2^20
 * hypotheses after the map or max_range changes (two more waits); its pitch is sqrt(max_range) / 4, coarser when the map's bounding box would exceed
 * 2^25 cells.  Waits: those of fls_relocalize, plus one per level above the start of the descent; launches: those of fls_relocalize
 * on a grid of at most 2^20 hypotheses, and past it growing with the number of levels and of 2^20-block chunks.  Everything else —
 * plug-ins, modes, argument checks, the empty scan, the state left for fls_fitness and Match — is fls_relocalize's. */
int fls_relocalize_wide(fls_handle* h, const void* scan, size_t n, size_t stride_bytes, const fls_reloc_cfg* cfg, double T_colmajor[16],
                        fls_reloc_result* out, double* refined_T, int32_t* refined_converged, float* refined_fitness, int64_t* refined_index,
                        int64_t* evaluations);
int fls_relocalize_wide_device(fls_handle* h, const void* d_scan, size_t n, const fls_reloc_cfg* cfg, double T_colmajor[16], fls_reloc_result* out,
                               double* refined_T, int32_t* refined_converged, float* refined_fitness, int64_t* refined_index, int64_t* evaluations);
/* The nodes the last fls_relocalize_wide call on h reached at each level, from its start level down to single hypotheses (the start
 * level: all its blocks; below: the children of the blocks kept one level up; 0 levels after an empty scan or a failed call before
 * the search).  Writes min(capacity, levels) values and returns the number of levels, or FLS_ERR_INVALID_ARG. */
int fls_relocalize_wide_levels(const fls_handle* h, int64_t* nodes, int capacity);

/* Relocalization from several coarse poses in one search: the grids that fls_relocalize defines for cfg around each of G = n_guesses
 * guesses (1..64; guess g is the column-major pose at guesses_colmajor + 16 g), searched as one grid of G * P hypotheses.  Hypothesis
 * g * P + p is hypothesis p of guess g's grid (P: the hypotheses of one grid), with the coarse score fls_relocalize gives it on guess
 * g, bit for bit; out->n_hypotheses = G * P, and best_hypothesis and refined_index use this index (the guess is index / P).  The
 * selection (the n_refine smallest scores of all grids, ties to the lower index), the one batch Match of the picks, the fitness and
 * the choice are fls_relocalize's.  The search is fls_relocalize_wide's exact branch and bound over all grids together: one
 * pruning threshold, the n_refine-th best score of any guess, and a lower bound that holds for every guess's hypotheses; a block
 * never spans two guesses.  When G * P <= 2^20 it scores every hypothesis.  *evaluations and fls_relocalize_wide_levels report the
 * search as for fls_relocalize_wide, and launches and waits are those of fls_relocalize_wide with the same node counts: on at most
 * 2^20 hypotheses in all they do not depend on G.
 *
 * T is output only: it receives the chosen pose, or guess 0 after an empty scan or an empty coarse cloud.  Grids are not merged
 * where they overlap (identical guesses tie, and the lower index wins); a grid off the map scores max_range and is not picked.
 * Caps: G * P <= 2^31 and floor(xy_radius / xy_step) <= 32767.  FLS_ERR_INVALID_ARG, in addition to fls_relocalize_wide's cases,
 * for a NULL guesses_colmajor, n_guesses outside 1..64, a non-finite entry of any guess, or G * P > 2^31.  FLS_ERR_CAPACITY,
 * plug-ins, modes, FLS_ERR_NO_MAP, the batch-in-flight refusal, the empty scan and the state left for fls_fitness and Match are
 * fls_relocalize_wide's; a refused call leaves T and the handle as they were. */
int fls_relocalize_multi(fls_handle* h, const void* scan, size_t n, size_t stride_bytes, const fls_reloc_cfg* cfg, const double* guesses_colmajor,
                         int32_t n_guesses, double T_colmajor[16], fls_reloc_result* out, double* refined_T, int32_t* refined_converged,
                         float* refined_fitness, int64_t* refined_index, int64_t* evaluations);
int fls_relocalize_multi_device(fls_handle* h, const void* d_scan, size_t n, const fls_reloc_cfg* cfg, const double* guesses_colmajor,
                                int32_t n_guesses, double T_colmajor[16], fls_reloc_result* out, double* refined_T, int32_t* refined_converged,
                                float* refined_fitness, int64_t* refined_index, int64_t* evaluations);

/* Device-side results for a consumer that lives on the GPU (the per-batch NCCL all-gather of poses, SURVEY.md §8e): once set,
 * every Match additionally writes, for scan s of the call, 18 doubles at d_results + 18*s — the column-major Mat4d pose
 * (what T receives), converged (0/1), iterations — from inside the Gauss-Newton kernel when the scan stops; the buffer is
 * complete when the Match call returns.  `capacity_scans` bounds s; NULL unsets.  The buffer is owned by the caller and must
 * stay valid until unset or the handle is destroyed. */
int fls_set_result_buffer_device(fls_handle* h, double* d_results, size_t capacity_scans);

/* per-iteration log of the last fls_match (needs FLS_FLAG_ITER_LOG; batch: scan 0); returns the number of entries written */
int fls_get_iter_log(const fls_handle* h, fls_iter_log* out, int capacity);
/* the same for scan `scan` of the last Match call (the batch entries of FLS_P2PLANE_IVOX, FLS_NDT,
 * FLS_ICP_P2P and FLS_P2PLANE_KNN keep one log per scan);
 * FLS_ERR_INVALID_ARG when `scan` is not below that call's n_scans; a Match that fails after its launch leaves no log */
int fls_get_iter_log_scan(const fls_handle* h, int scan, fls_iter_log* out, int capacity);

/* the information record of scan `scan` of the last Match call (fls_information).  out->valid = 0 when the handle was created
 * without FLS_FLAG_INFORMATION, before its first Match, after a Match call that returned an error, between
 * fls_match_batch_begin and _end, and after any relocalization call (whose internal Matches do not evaluate).
 * FLS_ERR_INVALID_ARG when `scan` is not below the n_scans of the call that left records (1 when there are none). */
int fls_get_information_scan(const fls_handle* h, int scan, fls_information* out);
int fls_get_information(const fls_handle* h, fls_information* out); /* scan 0 */

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

/* ---- De-skew with the sensor's translation (not upstream: LidarDistortionCorrector de-skews rotation only,
 *      src/lidar/lidar_distortion_corrector.cpp:34 "TODO: add translation") ----
 *
 * Each de-skewing entry has a _motion sibling with one more argument, velocity_imu: the body's velocity [m/s] expressed in the
 * IMU frame at ref_time_us, taken as constant over the sweep.  A kept point becomes
 *     p_corr = q_ref^-1 q(t) (R_li p + t_li) + v * dt
 * where t = ref_time_us + trunc_i64(rel_time * 1e6) is the integer microsecond stamp the interpolation uses and dt_us = t - ref_time_us
 * as a signed count.  Rounding, pinned: each coordinate is (float)(rot_k + v[k] * dt) with dt = (double)dt_us * 1.0e-6, every
 * product and sum rounded to nearest in fp64 (no fused multiply-add), and rot_k the fp64 value the parent entry rounds to float.
 *   * velocity_imu == NULL, or all three components exactly +-0: the term is skipped (not added as +0.0), and every output is
 *     bit-identical to the parent entry's.
 *   * a NaN or infinite component: FLS_ERR_INVALID_ARG before anything, counts included, is written.
 *   * no IMU samples (imu == NULL or n_imu == 0): no de-skew at all, velocity_imu is ignored.
 * Everything else is the parent's: the range gate, the points outside the IMU buffer dropped, the empty result when ref_time_us is
 * outside the buffer, and the projector's cell depth and column, which stay those of the raw point. */
int fls_preprocess_motion(int device, const float* raw_xyzit, size_t n, const fls_imu_buffer* imu, float min_distance, float max_distance,
                          int32_t jump_span, float planar_leaf, float* ordered, size_t* n_ordered, float* planar, size_t* n_planar,
                          const double velocity_imu[3]);
int fls_preprocess_device_motion(int device, const float* d_xyzi, const float* d_time, size_t n, const fls_imu_buffer* imu, float min_distance,
                                 float max_distance, int32_t jump_span, float planar_leaf, float* ordered, float* d_ordered, size_t* n_ordered,
                                 float* planar, float* d_planar, size_t* n_planar, const double velocity_imu[3]);
int fls_project_imu_motion(int device, const void* raw, const int32_t* ring, const float* time, size_t n, size_t stride_bytes, const fls_imu_buffer* imu,
                           int32_t n_rows, int32_t n_cols, float horizontal_resolution, float min_distance, float max_distance, float* ordered,
                           float* depth, int32_t* col, int32_t* row_start, int32_t* row_end, size_t* n_ordered, const double velocity_imu[3]);
int fls_preprocess_loam_motion(const fls_loam_frontend_cfg* cfg, const void* raw, const int32_t* ring, const float* time, size_t n, size_t stride_bytes,
                               const fls_imu_buffer* imu, float* corner, float* planar, float* d_corner, float* d_planar, size_t* n_corner,
                               size_t* n_planar, fls_match_stats* stats, const double velocity_imu[3]);
int fls_preprocess_loam_device_motion(const fls_loam_frontend_cfg* cfg, const float* d_xyzi, const int32_t* d_ring, const float* d_time, size_t n,
                                      const fls_imu_buffer* imu, float* corner, float* planar, float* d_corner, float* d_planar, size_t* n_corner,
                                      size_t* n_planar, fls_match_stats* stats, const double velocity_imu[3]);

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

/* ---- Place recognition on the keyframe store: Scan Context (G. Kim, A. Kim, IROS 2018), DESIGN.md §3.12 ----
 *
 * Descriptor of a cloud (packed x, y, z, intensity in the sensor frame, z up): an n_rings x n_sectors fp32 matrix, row-major.  Each
 * point with finite x, y and z, every operation rounded on its own (no FMA):
 *   r = sqrt(x*x + y*y) in fp64 (x, y widened from float); kept only if r < R (R = max_radius)
 *   ring = min(n_rings - 1, floor((r * n_rings) / R)) in fp64
 *   th = (double)atan2f(y, x) (the pinned atan2f of fls_atan.cuh), plus 2*pi when th < 0
 *   sector = min(n_sectors - 1, floor((th * n_sectors) / (2*pi)))
 *   cell = max over its points of (float)(z + z_offset) (-0.0 < +0.0); 0 for a cell without a point.
 * Distance of query Q to candidate C: column norms are fp64 sums over rings in ring order, then sqrt.  For each shift s in
 * [0, n_sectors), over the columns j (ascending) where both |Q_j| and |C_(j+s) mod n_sectors| are non-zero, E_s of them:
 *   cos_j = dot_j / (|Q_j| * |C_(j+s)|), dot_j an fp64 sum over rings in ring order;  d_s = 1 - (sum_j cos_j) / E_s  (1 when E_s = 0)
 * D = min_s d_s, ties to the smallest s; yaw = s * (2*pi / n_sectors), minus 2*pi when above pi.  A query taken where the candidate
 * was, with the sensor turned by +psi about z, has its best shift near psi / (2*pi / n_sectors): Rz(yaw) maps query-frame points into
 * the candidate frame, and T_candidate * Rz(yaw) is the query's coarse pose.  Results are ordered by (D, id) ascending, the same bits
 * from call to call. */
typedef struct {
    int32_t n_rings;   /* 1..64, 20 in the paper */
    int32_t n_sectors; /* 1..360, 60 in the paper; n_rings * n_sectors <= 4096 */
    float max_radius;  /* finite, > 0: 80 m in the paper */
    float z_offset;    /* finite: added to z before the maximum (2 m: the sensor height, so ground cells are near zero) */
} fls_sc_cfg;

typedef struct {
    int64_t id;       /* keyframe id */
    double distance;  /* D */
    double yaw;       /* rad, in (-pi, pi] */
    int32_t shift;    /* the best shift s */
    int32_t reserved;
} fls_place_match;

/* The descriptors of keyframes ids[0 .. n_ids) (below the count), n_rings * n_sectors floats each, one after another. */
int fls_keyframes_scan_context(fls_keyframes* s, const fls_sc_cfg* cfg, const int64_t* ids, size_t n_ids, float* desc);
/* LoopClosure::DetectByFeature: the query is stored keyframe query_id, the candidates the ids with query_id - id > min_span (the span
 * rule of CheckCandidateKeyFrames, src/slam/loop_closure.cpp:171, min_span = skip_near_keyframe_threshold).  FLS_ERR_INVALID_ARG when
 * query_id is not below the keyframe count or min_span < 0.  *n_found = min(k, candidates), possibly 0; out has room for k records.
 * The library applies no distance threshold: the caller does. */
int fls_keyframes_detect_loop(fls_keyframes* s, const fls_sc_cfg* cfg, int64_t query_id, int64_t min_span, size_t k, fls_place_match* out,
                              size_t* n_found, fls_match_stats* stats);
/* The query is a scan (host records stride_bytes apart, FLS_LAYOUT_*; _device: n packed float4 on the store's device, complete when
 * the call is made), the candidates every stored keyframe.  query_desc (optional, n_rings * n_sectors floats) receives its descriptor. */
int fls_keyframes_place_query(fls_keyframes* s, const fls_sc_cfg* cfg, const void* pts, size_t n, size_t stride_bytes, size_t k,
                              fls_place_match* out, size_t* n_found, float* query_desc, fls_match_stats* stats);
int fls_keyframes_place_query_device(fls_keyframes* s, const fls_sc_cfg* cfg, const void* d_pts, size_t n, size_t k, fls_place_match* out,
                                     size_t* n_found, float* query_desc, fls_match_stats* stats);
/* Common to the three: k >= 1; a bad cfg, k or pointer returns FLS_ERR_INVALID_ARG before any device work.  The store keeps one
 * descriptor per keyframe for the cfg of the last call; each call first describes the keyframes added since (all of them after a cfg
 * change) in one segmented pass.  Launches: that pass (a memset, a binning kernel when it reads a point, a finalize; nothing when
 * there is nothing to describe), the host query's repack when its stride is not 16, and the search, sort and pick (none without a
 * candidate).  One host wait (stream synchronisation); a call that grows the descriptor cache also frees its old buffers, and that
 * cudaFree waits for the device (the cache doubles, so this happens a logarithmic number of times).  None of this depends on the
 * keyframe count.  stats (optional): gpu_ms, gpu_launches, h2d_bytes,
 * d2h_bytes, n_source = points the pass read, n_valid = candidates, iterations = the host waits of the call. */

const char* fls_strerror(int status);
const char* fls_last_error(void); /* thread-local text of the last CUDA failure */
int fls_abi_version(void);
int fls_device_count(void);

#ifdef __cplusplus
}
#endif
#endif /* FLS_B200_H */
