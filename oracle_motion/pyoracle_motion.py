"""ctypes front end of the velocity-aware de-skew oracle (oracle_motion/libfls_oracle_motion.so, orc_motion.h): pre-processing and
projection with p_corr = q_ref^-1 q(t) (R_li p + t_li) + v * dt.  NOT UPSTREAM (upstream de-skews rotation only).  TEST INFRASTRUCTURE
ONLY, like oracle/pyoracle.py, whose argument conventions it shares: `imu` is dict(t_us, q_xyzw, ref_time_us, T_lidar_to_imu) or None,
`velocity` three floats [m/s] in the IMU frame at ref_time or None (rotation only)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle.pyoracle import _f4, _imu_args, _p

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libfls_oracle_motion.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            subprocess.check_call(["make", "-C", _HERE, "-s"], env={**os.environ})
        L = C.CDLL(_SO)
        vp, sz, f32, i32 = C.c_void_p, C.c_size_t, C.c_float, C.c_int
        L.orc_preprocess_motion.restype = sz
        L.orc_preprocess_motion.argtypes = [vp, sz, vp, vp, sz, C.c_uint64, vp, vp, f32, f32, i32, f32, vp, vp, C.POINTER(sz)]
        L.orc_project_imu_motion.restype = sz
        L.orc_project_imu_motion.argtypes = [vp, vp, vp, sz, vp, vp, sz, C.c_uint64, vp, vp, i32, i32, f32, f32, f32, vp, vp, vp, vp, vp]
        _lib = L
    return _lib


def _vel(velocity):
    if velocity is None:
        return None, None
    v = np.ascontiguousarray(velocity, np.float64).reshape(3)
    return _p(v), v


def preprocess(raw_xyzit, imu, velocity, min_d, max_d, jump_span, leaf):
    """oracle.pyoracle.preprocess with the translation term; returns (ordered, planar) as (n,4) float32."""
    raw = np.ascontiguousarray(raw_xyzit, np.float32)
    n = len(raw)
    ordered = np.zeros((max(n, 1), 4), np.float32)
    planar = np.zeros((max(n, 1), 4), np.float32)
    npl = C.c_size_t(0)
    pt, pq, m, ref, pT, keep = _imu_args(imu)
    pv, keep_v = _vel(velocity)
    no = lib().orc_preprocess_motion(_p(raw), n, pt, pq, m, ref, pT, pv, float(min_d), float(max_d), int(jump_span), float(leaf), _p(ordered),
                                     _p(planar), C.byref(npl))
    return ordered[:no].copy(), planar[:npl.value].copy()


def project_imu(raw, ring, time, imu, velocity, V, H, h_res, min_d, max_d):
    """oracle.pyoracle.project_imu with the translation term; same dict."""
    raw = _f4(raw)
    ring = np.ascontiguousarray(ring, np.int32)
    time = np.ascontiguousarray(time, np.float32)
    ordered = np.zeros((V * H, 4), np.float32)
    depth = np.zeros(V * H, np.float32)
    col = np.zeros(V * H, np.int32)
    rs = np.zeros(V, np.int32)
    re = np.zeros(V, np.int32)
    pt, pq, m, ref, pT, keep = _imu_args(imu)
    pv, keep_v = _vel(velocity)
    n = lib().orc_project_imu_motion(_p(raw), _p(ring), _p(time), len(raw), pt, pq, m, ref, pT, pv, V, H, float(h_res), float(min_d), float(max_d),
                                     _p(ordered), _p(depth), _p(col), _p(rs), _p(re))
    return dict(ordered=ordered[:n].copy(), depth=depth, col=col, row_start=rs, row_end=re, n=n)


def preprocess_loam(raw, ring, time, imu, velocity, V, H, h_res, min_d, max_d, corner_thr, planar_thr, corner_leaf, planar_leaf):
    """The LoamFull branch on the oracle: project_imu (with the term) -> extract_features -> gather -> voxel_grid x 2."""
    from oracle import pyoracle as orc
    pr = project_imu(raw, ring, time, imu, velocity, V, H, h_res, min_d, max_d)
    ci, pi, _ = orc.extract_features(pr["depth"], pr["col"], pr["n"], pr["row_start"], pr["row_end"], corner_thr, planar_thr)
    return orc.voxel_grid(pr["ordered"][ci], corner_leaf), orc.voxel_grid(pr["ordered"][pi], planar_leaf)
