"""ctypes mirror of include/fls_b200.h (struct layouts + enums).  No library is loaded here."""
from __future__ import annotations

import ctypes as C

FLS_ABI_VERSION = 1

# fls_status
FLS_OK = 0
FLS_ERR_INVALID_ARG = -1
FLS_ERR_CUDA = -2
FLS_ERR_NO_DEVICE = -3
FLS_ERR_UNSUPPORTED = -4
FLS_ERR_NO_MAP = -5
FLS_ERR_CAPACITY = -6
FLS_ERR_TOO_FEW_POINTS = -7

# fls_method — mode strings of include/common/constant_variable.h:21-25 upstream
FLS_ICP_P2P = 0
FLS_NDT = 1
FLS_P2PLANE_IVOX = 2
FLS_P2PLANE_KNN = 3
FLS_LOAM_FULL = 4
METHOD_BY_MODE_STRING = {
    "IcpOptimized": FLS_ICP_P2P,
    "IncrementalNDT": FLS_NDT,
    "PointToPlane_IVOX": FLS_P2PLANE_IVOX,
    "PointToPlane_KdTree": FLS_P2PLANE_KNN,
    "LoamFull_KdTree": FLS_LOAM_FULL,
}

FLS_NEARBY_CENTER, FLS_NEARBY6, FLS_NEARBY18, FLS_NEARBY26 = 0, 1, 2, 3
FLS_LAYOUT_PCL_XYZI = 32
FLS_LAYOUT_PACKED = 16
FLS_FLAG_ITER_LOG = 1
FLS_FLAG_PROFILE = 2
FLS_FLAG_INFORMATION = 4


class FlsConfig(C.Structure):
    _fields_ = [
        ("method", C.c_int32), ("device", C.c_int32), ("localization_mode", C.c_int32), ("max_iterations", C.c_int32),
        ("position_converge_thres", C.c_double), ("rotation_converge_thres", C.c_double),
        ("point_to_planar_thres", C.c_double), ("ivox_resolution", C.c_float), ("ivox_nearby", C.c_int32),
        ("ivox_capacity", C.c_int64), ("ivox_max_range", C.c_float), ("ivox_k", C.c_int32),
        ("ndt_voxel_size", C.c_double), ("ndt_outlier_thres", C.c_double), ("ndt_min_points_in_voxel", C.c_int32),
        ("ndt_max_points_in_voxel", C.c_int32), ("ndt_min_effective_pts", C.c_int32), ("ndt_capacity", C.c_int32),
        ("icp_max_correspond_distance", C.c_double), ("rot_thre_add_cloud", C.c_double), ("dist_thre_add_cloud", C.c_double),
        ("local_map_size", C.c_int32),
        ("source_cloud_filter_size", C.c_float), ("map_cloud_filter_size", C.c_float),
        ("point_search_thres", C.c_double), ("line_ratio_thres", C.c_double), ("corner_map_filter_size", C.c_float),
        ("corner_local_map_size", C.c_int32),
        ("flags", C.c_uint32), ("reserved", C.c_uint32 * 7),
    ]


class FlsMatchStats(C.Structure):
    _fields_ = [
        ("iterations", C.c_int32), ("converged", C.c_int32), ("n_source", C.c_int64), ("n_valid", C.c_int64),
        ("sum_residual", C.c_double), ("gpu_ms", C.c_float), ("gpu_launches", C.c_int32), ("h2d_bytes", C.c_int64),
        ("d2h_bytes", C.c_int64), ("kernel_ms", C.c_float), ("kernel_launches", C.c_int32), ("algo_bytes", C.c_int64),
    ]


class FlsIterLog(C.Structure):
    _fields_ = [("H", C.c_double * 36), ("g", C.c_double * 6), ("dx", C.c_double * 6), ("sum_residual", C.c_double),
                ("n_valid", C.c_int64)]


class FlsInformation(C.Structure):
    _fields_ = [("H", C.c_double * 36), ("g", C.c_double * 6), ("sum_residual", C.c_double), ("n_valid", C.c_int64),
                ("valid", C.c_int32), ("pad", C.c_int32)]


class FlsMapInfo(C.Structure):
    _fields_ = [("n_points", C.c_int64), ("n_voxels", C.c_int64), ("table_slots", C.c_int64), ("bytes", C.c_int64),
                ("incremental_inserts", C.c_int64), ("full_builds", C.c_int64)]


class FlsNdtVoxel(C.Structure):
    _fields_ = [("key", C.c_int32 * 3), ("estimated", C.c_int32), ("num_points", C.c_int32), ("carry_count", C.c_int32),
                ("mu", C.c_double * 3), ("info", C.c_double * 6)]


class FlsGnStepCase(C.Structure):
    _fields_ = [("method", C.c_int32), ("max_iterations", C.c_int32), ("min_effective", C.c_int32), ("iter", C.c_int32),
                ("rot_thres", C.c_double), ("pos_thres", C.c_double), ("R", C.c_double * 9), ("t", C.c_double * 3),
                ("last_rot", C.c_double), ("last_pos", C.c_double), ("tot", C.c_double * 31)]


class FlsGnStepOut(C.Structure):
    _fields_ = [("R", C.c_double * 9), ("t", C.c_double * 3), ("dx", C.c_double * 6), ("H", C.c_double * 36), ("g", C.c_double * 6),
                ("last_rot", C.c_double), ("last_pos", C.c_double), ("published", C.c_double * 13), ("result", C.c_double * 18),
                ("det_spd", C.c_double), ("n_valid", C.c_int64), ("iter", C.c_int32), ("converged", C.c_int32), ("failed", C.c_int32),
                ("done", C.c_int32), ("spd", C.c_int32), ("published_ok", C.c_int32)]


class FlsRelocCfg(C.Structure):
    _fields_ = [("xy_radius", C.c_double), ("xy_step", C.c_double), ("yaw_range", C.c_double), ("yaw_step", C.c_double),
                ("coarse_leaf", C.c_float), ("max_range", C.c_float), ("accept_fitness", C.c_float), ("n_refine", C.c_int32)]


class FlsRelocResult(C.Structure):
    _fields_ = [("n_hypotheses", C.c_int64), ("best_hypothesis", C.c_int64), ("n_refined", C.c_int32), ("best_rank", C.c_int32),
                ("converged", C.c_int32), ("accepted", C.c_int32), ("fitness", C.c_float), ("coarse_score", C.c_float),
                ("host_waits", C.c_int32), ("gpu_launches", C.c_int32)]


class FlsScCfg(C.Structure):
    """fls_sc_cfg: the Scan Context descriptor's shape (include/fls_b200.h)"""
    _fields_ = [("n_rings", C.c_int32), ("n_sectors", C.c_int32), ("max_radius", C.c_float), ("z_offset", C.c_float)]


class FlsPlaceMatch(C.Structure):
    _fields_ = [("id", C.c_int64), ("distance", C.c_double), ("yaw", C.c_double), ("shift", C.c_int32), ("reserved", C.c_int32)]


class FlsFeatureCfg(C.Structure):
    _fields_ = [("corner_threshold", C.c_float), ("planar_threshold", C.c_float), ("device", C.c_int32), ("reserved", C.c_int32)]


class FlsLoamFrontendCfg(C.Structure):
    _fields_ = [("device", C.c_int32), ("n_rows", C.c_int32), ("n_cols", C.c_int32), ("horizontal_resolution", C.c_float),
                ("min_distance", C.c_float), ("max_distance", C.c_float), ("corner_threshold", C.c_float), ("planar_threshold", C.c_float),
                ("corner_leaf", C.c_float), ("planar_leaf", C.c_float), ("reserved", C.c_uint32 * 4)]


def default_config(method: int, **overrides) -> FlsConfig:
    """Python twin of fls_config_default(): the parameter sets the reference ships (SURVEY.md App. B):
    config/localization/config_turing.yaml:48-53 (P2PLANE_IVOX), config/mapping/config_nclt_ndt.yaml:42-51 (NDT),
    config/localization/config_nclt_icp.yaml:42-48 (ICP)."""
    c = FlsConfig()
    c.method = method
    c.device = 0
    c.localization_mode = 1
    c.max_iterations = 10
    c.position_converge_thres = 0.01
    c.rotation_converge_thres = 0.01
    c.point_to_planar_thres = 0.1
    c.ivox_resolution = 0.5
    c.ivox_nearby = FLS_NEARBY18
    c.ivox_capacity = 1000000
    c.ivox_max_range = 5.0
    c.ivox_k = 5
    c.ndt_voxel_size = 1.0
    c.ndt_outlier_thres = 5.0
    c.ndt_min_points_in_voxel = 5
    c.ndt_max_points_in_voxel = 50
    c.ndt_min_effective_pts = 50
    c.ndt_capacity = 100000
    c.icp_max_correspond_distance = 1.0
    c.rot_thre_add_cloud = 0.2
    c.dist_thre_add_cloud = 1.0
    c.local_map_size = 50
    c.source_cloud_filter_size = 0.2
    c.map_cloud_filter_size = 0.4
    c.point_search_thres = 1.0
    c.line_ratio_thres = 3.0
    c.corner_map_filter_size = 0.2
    c.corner_local_map_size = 50
    if method == FLS_NDT:
        c.max_iterations = 30
        c.position_converge_thres = 0.005
        c.rotation_converge_thres = 0.005
        c.source_cloud_filter_size = 0.2
    elif method == FLS_ICP_P2P:
        c.max_iterations = 30
        c.position_converge_thres = 0.005
        c.rotation_converge_thres = 0.005
        c.source_cloud_filter_size = 0.4
        c.map_cloud_filter_size = 0.4
    elif method == FLS_P2PLANE_KNN:
        c.max_iterations = 8
        c.position_converge_thres = 0.005
        c.rotation_converge_thres = 0.005
        c.map_cloud_filter_size = 0.5
    elif method == FLS_LOAM_FULL:
        c.max_iterations = 30
        c.position_converge_thres = 0.01
        c.rotation_converge_thres = 0.05
        c.point_to_planar_thres = 0.2
        c.map_cloud_filter_size = 0.4
    for k, v in overrides.items():
        if not hasattr(c, k):
            raise AttributeError(f"fls_config has no field {k!r}")
        setattr(c, k, v)
    return c


# fls_lidar_type — LidarModel::LidarSensorType (include/lidar/lidar_model.h:25 upstream), same order
FLS_LIDAR_VELODYNE, FLS_LIDAR_OUSTER, FLS_LIDAR_LIVOX_AVIA, FLS_LIDAR_ROBOSENSE, FLS_LIDAR_LEISHEN, FLS_LIDAR_LIVOX_MID_360, FLS_LIDAR_NONE = range(7)
LIDAR_TYPE_BY_NAME = {"velodyne": FLS_LIDAR_VELODYNE, "ouster": FLS_LIDAR_OUSTER, "livox_avia": FLS_LIDAR_LIVOX_AVIA, "robosense": FLS_LIDAR_ROBOSENSE,
                      "leishen": FLS_LIDAR_LEISHEN, "livox_mid_360": FLS_LIDAR_LIVOX_MID_360, "none": FLS_LIDAR_NONE}
# sensor_msgs/PointField datatypes
FLS_PF_INT8, FLS_PF_UINT8, FLS_PF_INT16, FLS_PF_UINT16, FLS_PF_INT32, FLS_PF_UINT32, FLS_PF_FLOAT32, FLS_PF_FLOAT64 = range(1, 9)


class FlsPointField(C.Structure):
    _fields_ = [("name", C.c_char_p), ("offset", C.c_uint32), ("datatype", C.c_uint32), ("count", C.c_uint32), ("reserved", C.c_uint32)]


class FlsPointCloud2(C.Structure):
    """sensor_msgs/PointCloud2 (fls_pointcloud2)."""
    _fields_ = [("data", C.c_void_p), ("data_on_device", C.c_int32), ("height", C.c_uint32), ("width", C.c_uint32), ("point_step", C.c_uint32),
                ("row_step", C.c_uint32), ("is_dense", C.c_int32), ("is_bigendian", C.c_int32), ("n_fields", C.c_uint32),
                ("fields", C.POINTER(FlsPointField)), ("stamp_us", C.c_uint64), ("reserved", C.c_uint32 * 4)]


class FlsConvertCfg(C.Structure):
    _fields_ = [("device", C.c_int32), ("lidar_type", C.c_int32), ("n_rows", C.c_int32), ("lower_angle", C.c_float), ("v_res", C.c_float),
                ("time_scale", C.c_double), ("reserved", C.c_uint32 * 4)]


class FlsConvertResult(C.Structure):
    _fields_ = [("stamp_us", C.c_uint64), ("start_us", C.c_uint64), ("end_us", C.c_uint64), ("min_time", C.c_float), ("max_time", C.c_float),
                ("valid", C.c_int32), ("recomputed", C.c_int32), ("reserved", C.c_uint32 * 2)]
