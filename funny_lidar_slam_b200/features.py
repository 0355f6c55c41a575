"""Host-side mirror of loam::FeatureExtractor (include/loam/feature_extractor.h:15-45 upstream) over the C ABI.

`FeatureExtractor(corner_thr, planar_thr).ExtractFeatures(cluster)` fills cluster.corner_cloud / cluster.planar_cloud
from the projector's arrays exactly as upstream's ExtractFeatures(PointcloudCluster&) does, and also keeps the
index lists (into ordered_cloud) it was built from.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._abi import (FLS_PF_FLOAT32, FLS_PF_FLOAT64, FLS_PF_INT8, FLS_PF_INT16, FLS_PF_INT32, FLS_PF_UINT8, FLS_PF_UINT16, FLS_PF_UINT32, FlsConvertCfg,
                   FlsConvertResult, FlsFeatureCfg, FlsLoamFrontendCfg, FlsMatchStats, FlsPointCloud2, FlsPointField)
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


def _velocity(velocity):
    """velocity: None (rotation-only de-skew, the parent entry) or three floats [m/s], the body velocity in the IMU frame at the scan's
    reference time (a *_motion entry) -> (ctypes double[3] or None)."""
    if velocity is None:
        return None
    v = np.asarray(velocity, np.float64).reshape(-1)
    if v.shape != (3,):
        raise ValueError("velocity must hold three components")
    return (C.c_double * 3)(*[float(x) for x in v])


def _entry(name, velocity):
    """The library entry `name`, or its _motion sibling with the velocity appended when one is given."""
    v = _velocity(velocity)
    if v is None:
        return getattr(lib(), name), (), name
    return getattr(lib(), name + "_motion"), (v,), name + "_motion"


def preprocess(raw_xyzit, imu, min_distance, max_distance, jump_span, planar_leaf, device: int = 0, velocity=None):
    """PreProcessing::Run, the branch without features (src/slam/preprocessing.cpp:181-225 upstream), on the device:
    returns (ordered_cloud, planar_cloud) as (n,4) float32.  velocity (three floats [m/s], IMU frame at ref_time; not upstream) also
    de-skews the sensor's translation over the sweep (fls_preprocess_motion); None de-skews rotation only."""
    raw = np.ascontiguousarray(raw_xyzit, np.float32)
    if raw.ndim != 2 or raw.shape[1] != 5:
        raise ValueError("raw cloud must be (n,5): x, y, z, intensity, relative time")
    n = len(raw)
    ordered = np.zeros((max(n, 1), 4), np.float32)
    planar = np.zeros((max(n, 1), 4), np.float32)
    no, npl = C.c_size_t(0), C.c_size_t(0)
    b, keep = _imu_struct(imu)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    fn, extra, name = _entry("fls_preprocess", velocity)
    rc = fn(int(device), vp(raw), C.c_size_t(n), C.byref(b) if b is not None else None, C.c_float(min_distance), C.c_float(max_distance),
            int(jump_span), C.c_float(planar_leaf), vp(ordered), C.byref(no), vp(planar), C.byref(npl), *extra)
    check(rc, name)
    return ordered[:no.value].copy(), planar[:npl.value].copy()


def project_imu(projector: "PointcloudProjector", raw, ring, time, imu, velocity=None):
    """PointcloudProjector::Project with the de-skew of pointcloud_projector.cpp:100-103; with `velocity` (see preprocess) the
    translation too (fls_project_imu_motion)."""
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
    fn, extra, name = _entry("fls_project_imu", velocity)
    rc = fn(projector.device, vp(raw), vp(ring), vp(time), C.c_size_t(len(raw)), C.c_size_t(raw.shape[1] * 4), C.byref(b) if b is not None else None,
            projector.V, projector.H, C.c_float(projector.h_res), C.c_float(projector.min_d), C.c_float(projector.max_d), vp(ordered), vp(depth),
            vp(col), vp(rs), vp(re), C.byref(n_out), *extra)
    check(rc, name)
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

    def run(self, raw, ring, time, imu=None, device_out=None, host_out: bool = True, velocity=None):
        """Returns (corner, planar) as (n,4) float32.  velocity: see preprocess (fls_preprocess_loam_motion when given).  device_out=(d_corner, d_planar): device addresses on the configured device
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
        fn, extra, name = _entry("fls_preprocess_loam", velocity)
        rc = fn(C.byref(self.cfg), vp(raw), vp(ring), vp(time), len(raw), raw.shape[1] * 4, C.byref(b) if b is not None else None, vp(corner),
                vp(planar), C.c_void_p(d_c) if d_c else None, C.c_void_p(d_p) if d_p else None, C.byref(nc), C.byref(npl), C.byref(st), *extra)
        check(rc, name)
        self.last_stats = st
        self.last_counts = (nc.value, npl.value)
        if not host_out:
            return None, None
        return corner[:nc.value].copy(), planar[:npl.value].copy()

    def run_device(self, d_xyzi: int, d_ring: int, d_time: int, n: int, imu=None, device_out=None, host_out: bool = True, velocity=None):
        """run() on a cloud already in device memory on the configured device (fls_preprocess_loam_device): d_xyzi (n packed float4),
        d_ring (n int32) and d_time (n float, 0 without de-skew) are device addresses, e.g. convert_message's device outputs."""
        V, H = self.cfg.n_rows, self.cfg.n_cols
        corner = np.zeros((120 * V, 4), np.float32) if host_out else None
        planar = np.zeros((V * H, 4), np.float32) if host_out else None
        d_c, d_p = (int(device_out[0]), int(device_out[1])) if device_out is not None else (0, 0)
        nc, npl = C.c_size_t(0), C.c_size_t(0)
        st = FlsMatchStats()
        b, keep = _imu_struct(imu)
        vp = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
        dp = lambda a: C.c_void_p(int(a)) if a else None
        fn, extra, name = _entry("fls_preprocess_loam_device", velocity)
        rc = fn(C.byref(self.cfg), dp(d_xyzi), dp(d_ring), dp(d_time), int(n), C.byref(b) if b is not None else None, vp(corner), vp(planar), dp(d_c),
                dp(d_p), C.byref(nc), C.byref(npl), C.byref(st), *extra)
        check(rc, name)
        self.last_stats = st
        self.last_counts = (nc.value, npl.value)
        if not host_out:
            return None, None
        return corner[:nc.value].copy(), planar[:npl.value].copy()

    def Process(self, cluster: PointcloudCluster) -> None:
        e = cluster.extra
        cluster.corner_cloud, cluster.planar_cloud = self.run(e["raw_cloud"], e["ring"], e.get("time"), e.get("imu"), velocity=e.get("velocity"))


def preprocess_loam(raw, ring, time, imu, lidar_horizontal_scan, lidar_vertical_scan, lidar_horizontal_resolution, min_distance, max_distance,
                    corner_thr, planar_thr, corner_leaf, planar_leaf, device: int = 0, device_out=None, velocity=None):
    """PreProcessing::Run's LoamFull branch on the device (fls_preprocess_loam): returns (corner_cloud, planar_cloud) as (n,4) float32;
    with device_out=(d_corner, d_planar) the same clouds are also written to those device buffers.  velocity: see preprocess."""
    fe = LoamFrontEnd(lidar_horizontal_scan, lidar_vertical_scan, lidar_horizontal_resolution, min_distance, max_distance, corner_thr, planar_thr,
                      corner_leaf, planar_leaf, device)
    return fe.run(raw, ring, time, imu, device_out, velocity=velocity)


def preprocess_device(d_xyzi: int, d_time: int, n: int, imu, min_distance, max_distance, jump_span, planar_leaf, device: int = 0, device_out=None,
                      host_out: bool = True, velocity=None):
    """preprocess() on a cloud already in device memory (fls_preprocess_device): d_xyzi (n packed float4) and d_time (n float, 0 without
    de-skew) are device addresses.  Returns (ordered_cloud, planar_cloud) as (n,4) float32 (None, None with host_out=False);
    device_out=(d_ordered, d_planar), each with room for n records (0: not written), receives the same clouds; the ordered cloud may go
    nowhere (host_out=False, d_ordered 0).  The counts are in
    the returned clouds or, without host outputs, in preprocess_device.last_counts.  velocity: see preprocess."""
    cap = max(int(n), 1)
    ordered = np.zeros((cap, 4), np.float32) if host_out else None
    planar = np.zeros((cap, 4), np.float32) if host_out else None
    d_o, d_p = (int(device_out[0]), int(device_out[1])) if device_out is not None else (0, 0)
    no, npl = C.c_size_t(0), C.c_size_t(0)
    b, keep = _imu_struct(imu)
    vp = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    dp = lambda a: C.c_void_p(int(a)) if a else None
    fn, extra, name = _entry("fls_preprocess_device", velocity)
    rc = fn(int(device), dp(d_xyzi), dp(d_time), int(n), C.byref(b) if b is not None else None, float(min_distance), float(max_distance), int(jump_span),
            float(planar_leaf), vp(ordered), dp(d_o), C.byref(no), vp(planar), dp(d_p), C.byref(npl), *extra)
    check(rc, name)
    preprocess_device.last_counts = (no.value, npl.value)
    if not host_out:
        return None, None
    return ordered[:no.value].copy(), planar[:npl.value].copy()


preprocess_device.last_counts = (0, 0)

# numpy scalar type -> sensor_msgs/PointField datatype
_PF_BY_DTYPE = {np.dtype(np.int8): FLS_PF_INT8, np.dtype(np.uint8): FLS_PF_UINT8, np.dtype(np.int16): FLS_PF_INT16, np.dtype(np.uint16): FLS_PF_UINT16,
                np.dtype(np.int32): FLS_PF_INT32, np.dtype(np.uint32): FLS_PF_UINT32, np.dtype(np.float32): FLS_PF_FLOAT32,
                np.dtype(np.float64): FLS_PF_FLOAT64}


class PointCloud2:
    """sensor_msgs/PointCloud2 as the library reads it: `data` (bytes / uint8 array of height * row_step bytes, or a device address with
    data_on_device=True), the layout, and the PointField table as (name, offset, datatype, count) tuples.  stamp_us is
    header.stamp.toNSec() / 1000."""

    def __init__(self, data, fields, width, height=1, point_step=None, row_step=None, is_dense=True, is_bigendian=False, stamp_us=0,
                 data_on_device=False):
        self.fields = [(str(n), int(o), int(d), int(c)) for n, o, d, c in fields]
        self.width, self.height = int(width), int(height)
        self.point_step = int(point_step)
        self.row_step = int(row_step) if row_step is not None else self.width * self.point_step
        self.is_dense, self.is_bigendian = bool(is_dense), bool(is_bigendian)
        self.stamp_us = int(stamp_us)
        self.data_on_device = bool(data_on_device)
        self.data = int(data) if data_on_device else np.frombuffer(bytes(data), np.uint8) if not isinstance(data, np.ndarray) else \
            np.ascontiguousarray(data).view(np.uint8).reshape(-1)

    @classmethod
    def from_records(cls, rec: np.ndarray, **kw):
        """A message from a numpy structured array (1-D: one row; 2-D: organized), one PointField per named scalar field of its dtype
        (offsets and itemsize as the dtype has them, e.g. np.dtype({'names': ..., 'formats': ..., 'offsets': ..., 'itemsize': ...}))."""
        rec = np.ascontiguousarray(rec)
        h, w = (1, rec.shape[0]) if rec.ndim == 1 else rec.shape
        fields = [(n, rec.dtype.fields[n][1], _PF_BY_DTYPE[rec.dtype.fields[n][0]], 1) for n in rec.dtype.names]
        return cls(rec.view(np.uint8).reshape(-1), fields, w, h, rec.dtype.itemsize, **kw)

    def struct(self):
        """(fls_pointcloud2, keep-alive)"""
        names = [C.c_char_p(n.encode()) for n, _, _, _ in self.fields]
        tab = (FlsPointField * max(len(self.fields), 1))()
        for k, (n, o, d, c) in enumerate(self.fields):
            tab[k] = FlsPointField(names[k].value, o, d, c, 0)
        m = FlsPointCloud2()
        m.data = self.data if self.data_on_device else (self.data.ctypes.data if self.data.size else None)
        m.data_on_device = int(self.data_on_device)
        m.height, m.width, m.point_step, m.row_step = self.height, self.width, self.point_step, self.row_step
        m.is_dense, m.is_bigendian = int(self.is_dense), int(self.is_bigendian)
        m.n_fields = len(self.fields)
        m.fields = C.cast(tab, C.POINTER(FlsPointField))
        m.stamp_us = self.stamp_us
        return m, (names, tab, self.data)


def convert_cfg(lidar_type: int, n_rows: int, time_scale: float, lower_angle: float = 0.0, v_res: float = 0.0, device: int = 0) -> FlsConvertCfg:
    c = FlsConvertCfg()
    c.device, c.lidar_type, c.n_rows = int(device), int(lidar_type), int(n_rows)
    c.lower_angle, c.v_res, c.time_scale = float(lower_angle), float(v_res), float(time_scale)
    return c


def convert_message(msg: PointCloud2, lidar_type: int, n_rows: int, time_scale: float, lower_angle: float = 0.0, v_res: float = 0.0,
                    device: int = 0, device_out=None, host_out: bool = True):
    """PreProcessing::ConvertMessageToCloud on the device (fls_convert_cloud, src/slam/preprocessing.cpp:262-571 upstream).  Returns a dict:
    xyzi (n,4) float32, ring (n,) int32, time (n,) float32 (None with host_out=False), n, and the scan's time window: stamp_us,
    start_us, end_us, min_time, max_time, valid, recomputed, stats.  device_out=(d_xyzi, d_ring, d_time): device addresses with room for
    width * height records that receive the same arrays (0: not written)."""
    cap = msg.width * msg.height
    cfg = convert_cfg(lidar_type, n_rows, time_scale, lower_angle, v_res, device)
    xyzi = np.zeros((max(cap, 1), 4), np.float32) if host_out else None
    ring = np.zeros(max(cap, 1), np.int32) if host_out else None
    time = np.zeros(max(cap, 1), np.float32) if host_out else None
    d = [int(a) for a in device_out] if device_out is not None else [0, 0, 0]
    m, keep = msg.struct()
    n = C.c_size_t(0)
    res = FlsConvertResult()
    st = FlsMatchStats()
    vp = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    dp = lambda a: C.c_void_p(a) if a else None
    rc = lib().fls_convert_cloud(C.byref(cfg), C.byref(m), vp(xyzi), vp(ring), vp(time), dp(d[0]), dp(d[1]), dp(d[2]), C.byref(n), C.byref(res),
                                 C.byref(st))
    check(rc, "fls_convert_cloud")
    k = n.value
    out = dict(n=k, stamp_us=res.stamp_us, start_us=res.start_us, end_us=res.end_us, min_time=res.min_time, max_time=res.max_time,
               valid=bool(res.valid), recomputed=bool(res.recomputed), stats=st)
    out.update(xyzi=xyzi[:k].copy(), ring=ring[:k].copy(), time=time[:k].copy()) if host_out else out.update(xyzi=None, ring=None, time=None)
    return out
