"""ctypes front end of the conversion oracle (oracle_convert/libfls_oracle_convert.so): ConvertMessageToCloud, ComputePointOffsetTime,
GetLidarPointMinMaxOffsetTime and the stamps (orc_convert.h), and the pinned atan2f.  TEST INFRASTRUCTURE ONLY, like oracle/pyoracle.py."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from funny_lidar_slam_b200._abi import FlsConvertCfg, FlsConvertResult, FlsPointCloud2

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libfls_oracle_convert.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            subprocess.check_call(["make", "-C", _HERE, "-s"], env={**os.environ})
        L = C.CDLL(_SO)
        vp, sz, f32 = C.c_void_p, C.c_size_t, C.c_float
        L.orc_atan2f_pinned.restype = f32
        L.orc_atan2f_pinned.argtypes = [f32, f32]
        L.orc_atan2f_pinned_batch.argtypes = [vp, vp, sz, vp]
        L.orc_convert_cloud.argtypes = [C.POINTER(FlsConvertCfg), C.POINTER(FlsPointCloud2), vp, vp, vp, C.POINTER(sz), C.POINTER(FlsConvertResult)]
        _lib = L
    return _lib


def atan2f(y, x) -> np.ndarray:
    """The pinned std::atan2(float, float), elementwise over float32 arrays."""
    y = np.ascontiguousarray(y, np.float32).reshape(-1)
    x = np.ascontiguousarray(x, np.float32).reshape(-1)
    out = np.empty_like(y)
    lib().orc_atan2f_pinned_batch(y.ctypes.data_as(C.c_void_p), x.ctypes.data_as(C.c_void_p), len(y), out.ctypes.data_as(C.c_void_p))
    return out


def convert_message(msg, lidar_type: int, n_rows: int, time_scale: float, lower_angle: float = 0.0, v_res: float = 0.0) -> dict:
    """The oracle of features.convert_message on a host message (features.PointCloud2); same keys."""
    from funny_lidar_slam_b200.features import convert_cfg
    cfg = convert_cfg(lidar_type, n_rows, time_scale, lower_angle, v_res)
    cap = max(msg.width * msg.height, 1)
    xyzi, ring, time = np.zeros((cap, 4), np.float32), np.zeros(cap, np.int32), np.zeros(cap, np.float32)
    m, keep = msg.struct()
    n = C.c_size_t(0)
    res = FlsConvertResult()
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    lib().orc_convert_cloud(C.byref(cfg), C.byref(m), vp(xyzi), vp(ring), vp(time), C.byref(n), C.byref(res))
    k = n.value
    return dict(n=k, xyzi=xyzi[:k].copy(), ring=ring[:k].copy(), time=time[:k].copy(), stamp_us=res.stamp_us, start_us=res.start_us,
                end_us=res.end_us, min_time=res.min_time, max_time=res.max_time, valid=bool(res.valid), recomputed=bool(res.recomputed))
