"""Loader of the product library libfls_b200.so (C ABI: include/fls_b200.h).  No fallback of any kind:
a missing library or a missing GPU raises."""
from __future__ import annotations

import ctypes as C
import os

from ._abi import (FlsConfig, FlsConvertCfg, FlsConvertResult, FlsFeatureCfg, FlsIterLog, FlsLoamFrontendCfg, FlsMapInfo, FlsMatchStats,
                   FlsPointCloud2)

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "libfls_b200.so")
_lib = None

EXPORTS = [
    "fls_abi_version", "fls_device_count", "fls_last_error", "fls_strerror", "fls_config_default", "fls_create", "fls_destroy",
    "fls_add_cloud", "fls_match", "fls_match_device", "fls_fitness", "fls_get_iter_log", "fls_get_iter_log_scan", "fls_get_map_info", "fls_ivox_knn",
    "fls_voxel_grid", "fls_extract_features", "fls_project", "fls_match_batch", "fls_match_batch_device",
    "fls_set_result_buffer_device", "fls_get_voxel_keys", "fls_get_map_points", "fls_ivox_add_points", "fls_preprocess", "fls_project_imu", "fls_match_batch_begin", "fls_match_batch_begin_device", "fls_match_batch_end", "fls_set_global_map", "fls_update_local_map",
    "fls_pcd_read", "fls_pcd_write", "fls_preprocess_loam", "fls_match_cluster_device", "fls_convert_cloud", "fls_preprocess_loam_device",
    "fls_preprocess_device", "fls_keyframes_create", "fls_keyframes_destroy", "fls_keyframes_add", "fls_keyframes_add_device",
    "fls_keyframes_count", "fls_keyframes_assemble", "fls_get_ndt_voxels",
]


class FlsError(RuntimeError):
    def __init__(self, status: int, where: str):
        L = lib()
        msg = L.fls_strerror(status).decode()
        extra = L.fls_last_error().decode()
        super().__init__(f"{where}: {msg} [{status}]" + (f" — {extra}" if extra and status == -2 else ""))
        self.status = status


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing — build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(funny_lidar_slam_b200 has no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    vp, sz, i32, f32 = C.c_void_p, C.c_size_t, C.c_int32, C.c_float
    L.fls_abi_version.restype = C.c_int
    L.fls_device_count.restype = C.c_int
    L.fls_last_error.restype = C.c_char_p
    L.fls_strerror.restype = C.c_char_p
    L.fls_strerror.argtypes = [C.c_int]
    L.fls_config_default.argtypes = [C.POINTER(FlsConfig), C.c_int]
    L.fls_create.argtypes = [C.POINTER(FlsConfig), C.POINTER(vp)]
    L.fls_destroy.argtypes = [vp]
    L.fls_destroy.restype = None
    L.fls_add_cloud.argtypes = [vp, C.c_int, C.POINTER(vp), C.POINTER(sz), sz]
    L.fls_match.argtypes = [vp, vp, sz, vp, sz, vp, sz, sz, vp, C.POINTER(C.c_int), C.POINTER(FlsMatchStats)]
    L.fls_match_device.argtypes = [vp, vp, sz, vp, C.POINTER(C.c_int), C.POINTER(FlsMatchStats)]
    L.fls_match_cluster_device.argtypes = [vp, vp, sz, vp, sz, vp, sz, vp, C.POINTER(C.c_int), C.POINTER(FlsMatchStats)]
    L.fls_preprocess_loam.argtypes = [C.POINTER(FlsLoamFrontendCfg), vp, vp, vp, sz, sz, vp, vp, vp, vp, vp, C.POINTER(sz), C.POINTER(sz),
                                      C.POINTER(FlsMatchStats)]
    L.fls_preprocess_loam_device.argtypes = [C.POINTER(FlsLoamFrontendCfg), vp, vp, vp, sz, vp, vp, vp, vp, vp, C.POINTER(sz), C.POINTER(sz),
                                             C.POINTER(FlsMatchStats)]
    L.fls_preprocess_device.argtypes = [C.c_int, vp, vp, sz, vp, f32, f32, i32, f32, vp, vp, C.POINTER(sz), vp, vp, C.POINTER(sz)]
    L.fls_convert_cloud.argtypes = [C.POINTER(FlsConvertCfg), C.POINTER(FlsPointCloud2), vp, vp, vp, vp, vp, vp, C.POINTER(sz),
                                    C.POINTER(FlsConvertResult), C.POINTER(FlsMatchStats)]
    L.fls_match_batch.argtypes = [vp, C.c_int, C.POINTER(vp), C.POINTER(sz), sz, vp, C.POINTER(C.c_int), C.POINTER(FlsMatchStats)]
    L.fls_match_batch_device.argtypes = [vp, C.c_int, C.POINTER(vp), C.POINTER(sz), vp, C.POINTER(C.c_int), C.POINTER(FlsMatchStats)]
    L.fls_set_result_buffer_device.argtypes = [vp, vp, sz]
    L.fls_match_batch_begin.argtypes = [vp, C.c_int, C.POINTER(vp), C.POINTER(sz), sz, vp]
    L.fls_match_batch_begin_device.argtypes = [vp, C.c_int, C.POINTER(vp), C.POINTER(sz), vp]
    L.fls_set_global_map.argtypes = [vp, vp, sz, sz]
    L.fls_update_local_map.argtypes = [vp, vp, C.POINTER(C.c_int), C.POINTER(sz)]
    L.fls_pcd_read.argtypes = [C.c_char_p, vp, sz, C.POINTER(sz)]
    L.fls_pcd_write.argtypes = [C.c_char_p, vp, sz]
    L.fls_match_batch_end.argtypes = [vp, vp, C.POINTER(C.c_int), C.POINTER(FlsMatchStats)]
    L.fls_fitness.argtypes = [vp, f32, C.POINTER(f32)]
    L.fls_get_iter_log.argtypes = [vp, C.POINTER(FlsIterLog), C.c_int]
    L.fls_get_iter_log_scan.argtypes = [vp, C.c_int, C.POINTER(FlsIterLog), C.c_int]
    L.fls_get_map_info.argtypes = [vp, C.POINTER(FlsMapInfo)]
    L.fls_get_voxel_keys.argtypes = [vp, vp, sz, C.POINTER(sz)]
    L.fls_get_map_points.argtypes = [vp, vp, sz, C.POINTER(sz)]
    L.fls_get_ndt_voxels.argtypes = [vp, vp, sz, C.POINTER(sz)]
    L.fls_ivox_knn.argtypes = [vp, vp, sz, sz, C.c_int, vp, vp]
    L.fls_ivox_add_points.argtypes = [vp, vp, sz, sz]
    L.fls_voxel_grid.argtypes = [C.c_int, vp, sz, sz, f32, vp, C.POINTER(sz)]
    L.fls_extract_features.argtypes = [C.POINTER(FlsFeatureCfg), vp, vp, sz, vp, vp, i32, vp, C.POINTER(sz), vp, C.POINTER(sz),
                                       C.POINTER(FlsMatchStats)]
    L.fls_keyframes_create.argtypes = [C.c_int, sz, C.POINTER(vp)]
    L.fls_keyframes_destroy.argtypes = [vp]
    L.fls_keyframes_destroy.restype = None
    L.fls_keyframes_add.argtypes = [vp, C.c_int64, vp, sz, sz]
    L.fls_keyframes_add_device.argtypes = [vp, C.c_int64, vp, sz]
    L.fls_keyframes_count.argtypes = [vp, C.POINTER(sz), C.POINTER(sz)]
    L.fls_keyframes_assemble.argtypes = [vp, vp, sz, vp, f32, f32, vp, sz, vp, vp, sz, C.POINTER(sz), C.POINTER(FlsMatchStats)]
    for name in EXPORTS:
        getattr(L, name)  # AttributeError if the ABI drifted
    if L.fls_abi_version() != 1:
        raise ImportError("libfls_b200.so ABI version mismatch")
    _lib = L
    return _lib


def check(status: int, where: str) -> None:
    if status != 0:
        raise FlsError(status, where)
