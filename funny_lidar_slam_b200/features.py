"""Host-side mirror of loam::FeatureExtractor (include/loam/feature_extractor.h:15-45 upstream) over the C ABI.

`FeatureExtractor(corner_thr, planar_thr).ExtractFeatures(cluster)` fills cluster.corner_cloud / cluster.planar_cloud
from the projector's arrays exactly as upstream's ExtractFeatures(PointcloudCluster&) does, and also keeps the
index lists (into ordered_cloud) it was built from.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._abi import FlsFeatureCfg, FlsLoamFrontendCfg, FlsMatchStats
from ._lib import check, lib
from .registration import PointcloudCluster


class FeatureExtractor:
    def __init__(self, corner_thr: float, planar_thr: float, lidar_horizontal_scan: int = 0, lidar_vertical_scan: int = 0, device: int = 0):
        self.cfg = FlsFeatureCfg(float(corner_thr), float(planar_thr), int(device), 0)
        self.last_stats = FlsMatchStats()
        self.corner_idx = np.zeros(0, np.int32)
        self.planar_idx = np.zeros(0, np.int32)

    def extract_indices(self, depth, col, n: int, row_start, row_end):
        depth = np.ascontiguousarray(depth, np.float32)
        col = np.ascontiguousarray(col, np.int32)
        rs = np.ascontiguousarray(row_start, np.int32)
        re = np.ascontiguousarray(row_end, np.int32)
        V = len(rs)
        ci = np.zeros(120 * V + 16, np.int32)
        pi = np.zeros(n + 6 * V + 16, np.int32)
        nc, npl = C.c_size_t(0), C.c_size_t(0)
        st = FlsMatchStats()
        rc = lib().fls_extract_features(C.byref(self.cfg), depth.ctypes.data_as(C.c_void_p), col.ctypes.data_as(C.c_void_p), n,
                                        rs.ctypes.data_as(C.c_void_p), re.ctypes.data_as(C.c_void_p), V, ci.ctypes.data_as(C.c_void_p),
                                        C.byref(nc), pi.ctypes.data_as(C.c_void_p), C.byref(npl), C.byref(st))
        check(rc, "fls_extract_features")
        self.last_stats = st
        self.corner_idx, self.planar_idx = ci[:nc.value].copy(), pi[:npl.value].copy()
        return self.corner_idx, self.planar_idx

    def ExtractFeatures(self, cluster: PointcloudCluster) -> None:
        n = len(cluster.ordered_cloud)
        ci, pi = self.extract_indices(cluster.point_depth_vec, cluster.point_col_index_vec, n, cluster.row_start_index_vec,
                                      cluster.row_end_index_vec)
        cluster.corner_cloud = np.ascontiguousarray(cluster.ordered_cloud[ci])
        cluster.planar_cloud = np.ascontiguousarray(cluster.ordered_cloud[pi])


class PointcloudProjector:
    """Host-side mirror of loam::PointcloudProjector (include/loam/pointcloud_projector.h upstream): `Project(cluster)`
    reads cluster.extra["raw_cloud"] ((n,4) xyzi or (n,8) pcl records, firing order) and cluster.extra["ring"] and
    fills ordered_cloud / point_depth_vec / point_col_index_vec / row_start_index_vec / row_end_index_vec.
    Without an IMU buffer the de-skew step of upstream is the identity; project_imu() below applies it."""

    def __init__(self, lidar_horizontal_scan: int, lidar_vertical_scan: int, lidar_horizontal_resolution: float, min_distance: float,
                 max_distance: float, device: int = 0):
        self.H, self.V = int(lidar_horizontal_scan), int(lidar_vertical_scan)
        self.h_res, self.min_d, self.max_d = float(lidar_horizontal_resolution), float(min_distance), float(max_distance)
        self.device = int(device)

    def project_arrays(self, raw, ring):
        raw = np.ascontiguousarray(raw, np.float32)
        if raw.ndim != 2 or raw.shape[1] not in (4, 8):
            raise ValueError("raw cloud must be (n,4) packed xyzi or (n,8) pcl records")
        ring = np.ascontiguousarray(ring, np.int32)
        cells = self.V * self.H
        ordered = np.zeros((cells, 4), np.float32)
        depth = np.zeros(cells, np.float32)
        col = np.zeros(cells, np.int32)
        rs = np.zeros(self.V, np.int32)
        re = np.zeros(self.V, np.int32)
        n_out = C.c_size_t(0)
        vp = lambda a: a.ctypes.data_as(C.c_void_p)
        rc = lib().fls_project(self.device, vp(raw), vp(ring), C.c_size_t(len(raw)), C.c_size_t(raw.shape[1] * 4), self.V, self.H,
                               C.c_float(self.h_res), C.c_float(self.min_d), C.c_float(self.max_d), vp(ordered), vp(depth), vp(col), vp(rs),
                               vp(re), C.byref(n_out))
        check(rc, "fls_project")
        return dict(ordered=ordered[:n_out.value].copy(), depth=depth, col=col, row_start=rs, row_end=re, n=n_out.value)

    def Project(self, cluster: PointcloudCluster) -> None:
        out = self.project_arrays(cluster.extra["raw_cloud"], cluster.extra["ring"])
        cluster.ordered_cloud = out["ordered"]
        cluster.point_depth_vec = out["depth"]
        cluster.point_col_index_vec = out["col"]
        cluster.row_start_index_vec = out["row_start"]
        cluster.row_end_index_vec = out["row_end"]


class ImuBuffer(C.Structure):
    """fls_imu_buffer (include/fls_b200.h): IMU orientation samples of a scan for the de-skew."""
    _fields_ = [("imu_time_us", C.c_void_p), ("imu_quat_xyzw", C.c_void_p), ("n_imu", C.c_size_t), ("ref_time_us", C.c_uint64),
                ("T_lidar_to_imu", C.c_double * 16)]


def _imu_struct(imu):
    """imu: dict(t_us (m,) uint64, q_xyzw (m,4) float64, ref_time_us int, T_lidar_to_imu (4,4)) or None -> (struct or None, keep-alive)."""
    if imu is None:
        return None, ()
    t = np.ascontiguousarray(imu["t_us"], np.uint64)
    q = np.ascontiguousarray(imu["q_xyzw"], np.float64)
    T = np.ascontiguousarray(np.asarray(imu["T_lidar_to_imu"], np.float64).T).reshape(-1)  # column-major
    b = ImuBuffer()
    b.imu_time_us = t.ctypes.data
    b.imu_quat_xyzw = q.ctypes.data
    b.n_imu = len(t)
    b.ref_time_us = int(imu["ref_time_us"])
    for k in range(16):
        b.T_lidar_to_imu[k] = float(T[k])
    return b, (t, q)


def preprocess(raw_xyzit, imu, min_distance, max_distance, jump_span, planar_leaf, device: int = 0):
    """PreProcessing::Run, the branch without features (src/slam/preprocessing.cpp:181-225 upstream), on the device:
    returns (ordered_cloud, planar_cloud) as (n,4) float32."""
    raw = np.ascontiguousarray(raw_xyzit, np.float32)
    if raw.ndim != 2 or raw.shape[1] != 5:
        raise ValueError("raw cloud must be (n,5): x, y, z, intensity, relative time")
    n = len(raw)
    ordered = np.zeros((max(n, 1), 4), np.float32)
    planar = np.zeros((max(n, 1), 4), np.float32)
    no, npl = C.c_size_t(0), C.c_size_t(0)
    b, keep = _imu_struct(imu)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = lib().fls_preprocess(int(device), vp(raw), C.c_size_t(n), C.byref(b) if b is not None else None, C.c_float(min_distance),
                              C.c_float(max_distance), int(jump_span), C.c_float(planar_leaf), vp(ordered), C.byref(no), vp(planar), C.byref(npl))
    check(rc, "fls_preprocess")
    return ordered[:no.value].copy(), planar[:npl.value].copy()


def project_imu(projector: "PointcloudProjector", raw, ring, time, imu):
    """PointcloudProjector::Project with the de-skew of pointcloud_projector.cpp:100-103."""
    raw = np.ascontiguousarray(raw, np.float32)
    ring = np.ascontiguousarray(ring, np.int32)
    time = np.ascontiguousarray(time, np.float32)
    cells = projector.V * projector.H
    ordered = np.zeros((cells, 4), np.float32)
    depth = np.zeros(cells, np.float32)
    col = np.zeros(cells, np.int32)
    rs = np.zeros(projector.V, np.int32)
    re = np.zeros(projector.V, np.int32)
    n_out = C.c_size_t(0)
    b, keep = _imu_struct(imu)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = lib().fls_project_imu(projector.device, vp(raw), vp(ring), vp(time), C.c_size_t(len(raw)), C.c_size_t(raw.shape[1] * 4),
                               C.byref(b) if b is not None else None, projector.V, projector.H, C.c_float(projector.h_res), C.c_float(projector.min_d),
                               C.c_float(projector.max_d), vp(ordered), vp(depth), vp(col), vp(rs), vp(re), C.byref(n_out))
    check(rc, "fls_project_imu")
    return dict(ordered=ordered[:n_out.value].copy(), depth=depth, col=col, row_start=rs, row_end=re, n=n_out.value)


class LoamFrontEnd:
    """PreProcessing::Run, the LoamFull branch (src/slam/preprocessing.cpp:226-237 upstream), in one device call
    (fls_preprocess_loam): projection with de-skew, feature extraction and the corner / planar voxel filters.
    `Process(cluster)` reads cluster.extra["raw_cloud"] ((n,4) xyzi or (n,8) pcl records, firing order), ["ring"], ["time"]
    (seconds relative to the scan's reference time; only read with an IMU buffer) and, optionally, ["imu"], and fills cluster.corner_cloud / planar_cloud,
    as upstream's branch fills the PointcloudCluster."""

    def __init__(self, lidar_horizontal_scan: int, lidar_vertical_scan: int, lidar_horizontal_resolution: float, min_distance: float,
                 max_distance: float, corner_thr: float, planar_thr: float, corner_leaf: float, planar_leaf: float, device: int = 0):
        self.cfg = FlsLoamFrontendCfg(int(device), int(lidar_vertical_scan), int(lidar_horizontal_scan), float(lidar_horizontal_resolution),
                                      float(min_distance), float(max_distance), float(corner_thr), float(planar_thr), float(corner_leaf),
                                      float(planar_leaf))
        self.last_stats = FlsMatchStats()
        self.last_counts = (0, 0)

    def run(self, raw, ring, time, imu=None, device_out=None, host_out: bool = True):
        """Returns (corner, planar) as (n,4) float32.  device_out=(d_corner, d_planar): device addresses on the configured device
        (capacities 120*V and V*H records) that receive the same clouds; with host_out=False only those are written and (None, None)
        is returned.  self.last_counts holds (n_corner, n_planar), self.last_stats the call's fls_match_stats."""
        raw = np.ascontiguousarray(raw, np.float32)
        if raw.ndim != 2 or raw.shape[1] not in (4, 8):
            raise ValueError("raw cloud must be (n,4) packed xyzi or (n,8) pcl records")
        ring = np.ascontiguousarray(ring, np.int32)
        time = np.ascontiguousarray(time, np.float32) if time is not None else None  # needed only to de-skew
        if len(ring) != len(raw) or (time is not None and len(time) != len(raw)):
            raise ValueError("ring and time need one entry per raw point")
        V, H = self.cfg.n_rows, self.cfg.n_cols
        corner = np.zeros((120 * V, 4), np.float32) if host_out else None
        planar = np.zeros((V * H, 4), np.float32) if host_out else None
        d_c, d_p = (int(device_out[0]), int(device_out[1])) if device_out is not None else (0, 0)
        nc, npl = C.c_size_t(0), C.c_size_t(0)
        st = FlsMatchStats()
        b, keep = _imu_struct(imu)
        vp = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
        rc = lib().fls_preprocess_loam(C.byref(self.cfg), vp(raw), vp(ring), vp(time), len(raw), raw.shape[1] * 4, C.byref(b) if b is not None else None,
                                       vp(corner), vp(planar), C.c_void_p(d_c) if d_c else None, C.c_void_p(d_p) if d_p else None, C.byref(nc),
                                       C.byref(npl), C.byref(st))
        check(rc, "fls_preprocess_loam")
        self.last_stats = st
        self.last_counts = (nc.value, npl.value)
        if not host_out:
            return None, None
        return corner[:nc.value].copy(), planar[:npl.value].copy()

    def Process(self, cluster: PointcloudCluster) -> None:
        e = cluster.extra
        cluster.corner_cloud, cluster.planar_cloud = self.run(e["raw_cloud"], e["ring"], e.get("time"), e.get("imu"))


def preprocess_loam(raw, ring, time, imu, lidar_horizontal_scan, lidar_vertical_scan, lidar_horizontal_resolution, min_distance, max_distance,
                    corner_thr, planar_thr, corner_leaf, planar_leaf, device: int = 0, device_out=None):
    """PreProcessing::Run's LoamFull branch on the device (fls_preprocess_loam): returns (corner_cloud, planar_cloud) as (n,4) float32;
    with device_out=(d_corner, d_planar) the same clouds are also written to those device buffers."""
    fe = LoamFrontEnd(lidar_horizontal_scan, lidar_vertical_scan, lidar_horizontal_resolution, min_distance, max_distance, corner_thr, planar_thr,
                      corner_leaf, planar_leaf, device)
    return fe.run(raw, ring, time, imu, device_out)
