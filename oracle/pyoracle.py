"""ctypes front end of the CPU oracle (oracle/libfls_oracle.so).

ORACLE — TEST INFRASTRUCTURE ONLY, parity unpinned (see oracle/orc_math.h).  Importable only from tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from funny_lidar_slam_b200._abi import FlsConfig, FlsIterLog, FlsMatchStats

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libfls_oracle.so")
_lib = None


def build(force: bool = False) -> str:
    if force or not os.path.exists(_SO) or any(
            os.path.getmtime(os.path.join(_HERE, f)) > os.path.getmtime(_SO) for f in os.listdir(_HERE) if f.endswith((".h", ".cpp"))):
        subprocess.check_call(["make", "-C", _HERE, "-s"], env={**os.environ})
    return _SO


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            build()
        L = C.CDLL(_SO)
        vp, sz, f32, i32, dbl = C.c_void_p, C.c_size_t, C.c_float, C.c_int, C.c_double
        L.orc_num_threads.restype = i32
        L.orc_fast_atan2f.restype = f32
        L.orc_fast_atan2f.argtypes = [f32, f32]
        L.orc_solve6_lu.restype = dbl
        L.orc_voxel_grid.restype = sz
        L.orc_voxel_grid.argtypes = [vp, sz, sz, f32, vp]
        L.orc_transform_d.argtypes = [vp, sz, vp, vp]
        L.orc_transform_f.argtypes = [vp, sz, vp, vp]
        L.orc_knn_build.restype = vp
        L.orc_knn_build.argtypes = [vp, sz, f32]
        L.orc_knn_search.argtypes = [vp, vp, sz, i32, vp, vp, vp]
        L.orc_knn_free.argtypes = [vp]
        L.orc_ivox_create.restype = vp
        L.orc_ivox_create.argtypes = [f32, i32, sz]
        L.orc_ivox_add.argtypes = [vp, vp, sz]
        L.orc_ivox_closest.argtypes = [vp, vp, sz, i32, f32, vp, vp]
        L.orc_ivox_num_voxels.restype = sz
        L.orc_ivox_num_voxels.argtypes = [vp]
        L.orc_ivox_num_points.restype = sz
        L.orc_ivox_num_points.argtypes = [vp]
        L.orc_ivox_free.argtypes = [vp]
        L.orc_reg_create.restype = vp
        L.orc_reg_create.argtypes = [C.POINTER(FlsConfig)]
        L.orc_reg_free.argtypes = [vp]
        L.orc_reg_add_cloud.argtypes = [vp, vp, sz, sz]
        L.orc_reg_match.argtypes = [vp, vp, sz, sz, vp, C.POINTER(i32), C.POINTER(FlsMatchStats), C.POINTER(dbl)]
        L.orc_reg_get_iter_log.argtypes = [vp, C.POINTER(FlsIterLog), i32]
        L.orc_reg_add_cloud2.argtypes = [vp, vp, sz, vp, sz, sz]
        L.orc_reg_match2.argtypes = [vp, vp, sz, vp, sz, sz, vp, C.POINTER(i32), C.POINTER(FlsMatchStats), C.POINTER(dbl)]
        L.orc_reg_map_copy.restype = sz
        L.orc_reg_map_copy.argtypes = [vp, i32, vp, sz]
        L.orc_reg_fitness.restype = f32
        L.orc_reg_fitness.argtypes = [vp, f32]
        L.orc_reg_map_voxels.restype = sz
        L.orc_reg_map_voxels.argtypes = [vp]
        L.orc_reg_map_points.restype = sz
        L.orc_reg_map_points.argtypes = [vp]
        L.orc_reg_ndt_dump.restype = sz
        L.orc_reg_ndt_dump.argtypes = [vp, vp, vp, vp, vp, vp, vp]
        L.orc_project.restype = sz
        L.orc_project.argtypes = [vp, vp, sz, i32, i32, f32, f32, f32, vp, vp, vp, vp, vp]
        L.orc_preprocess.restype = sz
        L.orc_preprocess.argtypes = [vp, sz, vp, vp, sz, C.c_uint64, vp, f32, f32, i32, f32, vp, vp, C.POINTER(sz)]
        L.orc_project_imu.restype = sz
        L.orc_project_imu.argtypes = [vp, vp, vp, sz, vp, vp, sz, C.c_uint64, vp, i32, i32, f32, f32, f32, vp, vp, vp, vp, vp]
        L.orc_extract_features.argtypes = [vp, vp, sz, vp, vp, i32, f32, f32, vp, C.POINTER(sz), vp, C.POINTER(sz), C.POINTER(dbl)]
        _lib = L
    return _lib


def _f4(a) -> np.ndarray:
    a = np.ascontiguousarray(a, dtype=np.float32)
    assert a.ndim == 2 and a.shape[1] == 4
    return a


def _p(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def num_threads() -> int:
    return lib().orc_num_threads()


def set_num_threads(n: int) -> None:
    lib().orc_set_num_threads(int(n))


# ---- math ---------------------------------------------------------------------------------------------
def so3_exp(v):
    v = np.ascontiguousarray(v, np.float64)
    R = np.empty(9)
    lib().orc_so3_exp(_p(v), _p(R))
    return R.reshape(3, 3)


def se3_exp(v):
    v = np.ascontiguousarray(v, np.float64)
    T = np.empty(16)
    lib().orc_se3_exp(_p(v), _p(T))
    return T.reshape(4, 4)


def rot_to_rpy(R):
    R = np.ascontiguousarray(R, np.float64)
    o = np.empty(3)
    lib().orc_rot_to_rpy(_p(R), _p(o))
    return o


def fast_atan2f(y, x) -> float:
    return float(lib().orc_fast_atan2f(float(y), float(x)))


def lstsq53(A, b):
    A = np.ascontiguousarray(A, np.float64)
    b = np.ascontiguousarray(b, np.float64)
    x = np.empty(3)
    lib().orc_lstsq53(_p(A), _p(b), _p(x))
    return x


def solve6_fullpiv(H, g):
    H = np.ascontiguousarray(H, np.float64)
    g = np.ascontiguousarray(g, np.float64)
    x = np.empty(6)
    lib().orc_solve6_fullpiv(_p(H), _p(g), _p(x))
    return x


def solve6_lu(H, g):
    H = np.ascontiguousarray(H, np.float64)
    g = np.ascontiguousarray(g, np.float64)
    x = np.zeros(6)
    det = lib().orc_solve6_lu(_p(H), _p(g), _p(x))
    return x, det


def sym_eig3(S):
    S = np.ascontiguousarray(S, np.float64)
    lam, V = np.empty(3), np.empty(9)
    lib().orc_sym_eig3(_p(S), _p(lam), _p(V))
    return lam, V.reshape(3, 3)


# ---- clouds -------------------------------------------------------------------------------------------
def voxel_grid(pts, leaf: float) -> np.ndarray:
    pts = _f4(pts)
    out = np.empty_like(pts)
    n = lib().orc_voxel_grid(_p(pts), len(pts), 16, float(leaf), _p(out))
    return out[:n].copy()


def transform_d(pts, T) -> np.ndarray:
    pts = _f4(pts)
    Tc = np.ascontiguousarray(np.asarray(T, np.float64).T)  # column-major memory
    out = np.empty_like(pts)
    lib().orc_transform_d(_p(pts), len(pts), _p(Tc), _p(out))
    return out


def transform_f(pts, T) -> np.ndarray:
    pts = _f4(pts)
    Tc = np.ascontiguousarray(np.asarray(T, np.float64).T)
    out = np.empty_like(pts)
    lib().orc_transform_f(_p(pts), len(pts), _p(Tc), _p(out))
    return out


class ExactKnn:
    def __init__(self, pts, cell: float = 1.0):
        pts = _f4(pts)
        self._h = lib().orc_knn_build(_p(pts), len(pts), float(cell))

    def search(self, q, k: int):
        q = _f4(q)
        idx = np.full((len(q), k), -1, np.int32)
        d2 = np.full((len(q), k), np.inf, np.float32)
        found = np.zeros(len(q), np.int32)
        lib().orc_knn_search(self._h, _p(q), len(q), k, _p(idx), _p(d2), _p(found))
        return idx, d2, found

    def __del__(self):
        if getattr(self, "_h", None):
            lib().orc_knn_free(self._h)
            self._h = None


class IVox:
    def __init__(self, resolution=0.5, nearby=2, capacity=1000000):
        self._h = lib().orc_ivox_create(float(resolution), int(nearby), int(capacity))

    def add(self, pts):
        pts = _f4(pts)
        lib().orc_ivox_add(self._h, _p(pts), len(pts))

    def closest(self, q, K=5, max_range=5.0):
        q = _f4(q)
        out = np.zeros((len(q), K, 4), np.float32)
        found = np.zeros(len(q), np.int32)
        lib().orc_ivox_closest(self._h, _p(q), len(q), K, float(max_range), _p(out), _p(found))
        return out, found

    @property
    def num_voxels(self):
        return lib().orc_ivox_num_voxels(self._h)

    @property
    def num_points(self):
        return lib().orc_ivox_num_points(self._h)

    def __del__(self):
        if getattr(self, "_h", None):
            lib().orc_ivox_free(self._h)
            self._h = None


class Registration:
    """Oracle twin of funny_lidar_slam_b200.registration.Registration (same call shapes)."""

    def __init__(self, cfg: FlsConfig):
        self.cfg = cfg
        self._h = lib().orc_reg_create(C.byref(cfg))
        if not self._h:
            raise ValueError(f"oracle does not implement method {cfg.method}")
        self.last_seconds = 0.0

    def add_cloud(self, pts, corner=None):
        """One cloud for ICP / NDT / point-to-plane; (planar, corner) for LoamFull."""
        pts = _f4(pts)
        if corner is not None:
            corner = _f4(corner)
            rc = lib().orc_reg_add_cloud2(self._h, _p(pts), len(pts), _p(corner), len(corner), 16)
        else:
            rc = lib().orc_reg_add_cloud(self._h, _p(pts), len(pts), 16)
        if rc != 0:
            raise ValueError("wrong number of clouds for this plug-in")

    def match(self, pts, T, corner=None):
        pts = _f4(pts)
        Tc = np.ascontiguousarray(np.asarray(T, np.float64).T).copy()
        conv = C.c_int(0)
        st = FlsMatchStats()
        sec = C.c_double(0)
        if corner is not None:
            corner = _f4(corner)
            rc = lib().orc_reg_match2(self._h, _p(pts), len(pts), _p(corner), len(corner), 16, _p(Tc), C.byref(conv), C.byref(st), C.byref(sec))
        else:
            rc = lib().orc_reg_match(self._h, _p(pts), len(pts), 16, _p(Tc), C.byref(conv), C.byref(st), C.byref(sec))
        if rc != 0:
            raise ValueError("wrong number of clouds for this plug-in")
        self.last_seconds = sec.value
        return bool(conv.value), Tc.T.copy(), st

    def map_copy(self, which=0):
        """Current local map of the kd-tree plug-ins / ICP (which=1: LoamFull's corner map)."""
        n = lib().orc_reg_map_copy(self._h, int(which), None, 0)
        out = np.zeros((max(n, 1), 4), np.float32)
        lib().orc_reg_map_copy(self._h, int(which), _p(out), n)
        return out[:n]

    def iter_log(self, cap=64):
        buf = (FlsIterLog * cap)()
        n = lib().orc_reg_get_iter_log(self._h, buf, cap)
        return [dict(H=np.array(b.H).reshape(6, 6), g=np.array(b.g), dx=np.array(b.dx), sum_residual=b.sum_residual, n_valid=b.n_valid)
                for b in buf[:n]]

    def fitness(self, max_range: float) -> float:
        return float(lib().orc_reg_fitness(self._h, float(max_range)))

    @property
    def map_voxels(self):
        return lib().orc_reg_map_voxels(self._h)

    @property
    def map_points(self):
        return lib().orc_reg_map_points(self._h)

    def ndt_dump(self):
        n = self.map_voxels
        keys = np.zeros((n, 3), np.int32)
        mu = np.zeros((n, 3))
        info = np.zeros((n, 9))
        est = np.zeros(n, np.int32)
        m = lib().orc_reg_ndt_dump(self._h, _p(keys), _p(mu), _p(info), _p(est), None, None)
        return keys[:m], mu[:m], info[:m].reshape(-1, 3, 3), est[:m]

    def ndt_voxels(self):
        """Every NDT voxel in LRU order (front first): key (n,3), mu (n,3), info (n,3,3), estimated, num_points and pending (the
        points_ buffer, incremental_ndt.h:78 upstream) per voxel."""
        n = self.map_voxels
        keys, mu, info = np.zeros((n, 3), np.int32), np.zeros((n, 3)), np.zeros((n, 9))
        est, num, pend = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.int32)
        m = lib().orc_reg_ndt_dump(self._h, _p(keys), _p(mu), _p(info), _p(est), _p(num), _p(pend))
        return dict(key=keys[:m], mu=mu[:m], info=info[:m].reshape(-1, 3, 3), estimated=est[:m], num_points=num[:m], pending=pend[:m])

    def __del__(self):
        if getattr(self, "_h", None):
            lib().orc_reg_free(self._h)
            self._h = None


def project(raw, ring, V, H, h_res, min_d, max_d):
    raw = _f4(raw)
    ring = np.ascontiguousarray(ring, np.int32)
    ordered = np.zeros((V * H, 4), np.float32)
    depth = np.zeros(V * H, np.float32)
    col = np.zeros(V * H, np.int32)
    rs = np.zeros(V, np.int32)
    re = np.zeros(V, np.int32)
    n = lib().orc_project(_p(raw), _p(ring), len(raw), V, H, float(h_res), float(min_d), float(max_d), _p(ordered), _p(depth), _p(col), _p(rs), _p(re))
    return dict(ordered=ordered[:n].copy(), depth=depth, col=col, row_start=rs, row_end=re, n=n)


def _imu_args(imu):
    if imu is None:
        return None, None, 0, 0, _p(np.eye(4).T.copy()), ()
    t = np.ascontiguousarray(imu["t_us"], np.uint64)
    q = np.ascontiguousarray(imu["q_xyzw"], np.float64)
    T = np.ascontiguousarray(np.asarray(imu["T_lidar_to_imu"], np.float64).T)  # column-major
    return _p(t), _p(q), len(t), int(imu["ref_time_us"]), _p(T), (t, q, T)


def preprocess(raw_xyzit, imu, min_d, max_d, jump_span, leaf):
    """preprocessing.cpp:181-225 (non-feature branch): range gate + IMU de-skew + jump span + voxel filter.
    raw_xyzit: (n,5) float32 x,y,z,intensity,relative time [s]; imu: dict(t_us, q_xyzw, ref_time_us, T_lidar_to_imu) or None."""
    raw = np.ascontiguousarray(raw_xyzit, np.float32)
    n = len(raw)
    ordered = np.zeros((max(n, 1), 4), np.float32)
    planar = np.zeros((max(n, 1), 4), np.float32)
    npl = C.c_size_t(0)
    pt, pq, m, ref, pT, keep = _imu_args(imu)
    no = lib().orc_preprocess(_p(raw), n, pt, pq, m, ref, pT, float(min_d), float(max_d), int(jump_span), float(leaf), _p(ordered), _p(planar),
                              C.byref(npl))
    return ordered[:no].copy(), planar[:npl.value].copy()


def project_imu(raw, ring, time, imu, V, H, h_res, min_d, max_d):
    """pointcloud_projector.cpp:32-133 with the per-point de-skew of :100-103."""
    raw = _f4(raw)
    ring = np.ascontiguousarray(ring, np.int32)
    time = np.ascontiguousarray(time, np.float32)
    ordered = np.zeros((V * H, 4), np.float32)
    depth = np.zeros(V * H, np.float32)
    col = np.zeros(V * H, np.int32)
    rs = np.zeros(V, np.int32)
    re = np.zeros(V, np.int32)
    pt, pq, m, ref, pT, keep = _imu_args(imu)
    n = lib().orc_project_imu(_p(raw), _p(ring), _p(time), len(raw), pt, pq, m, ref, pT, V, H, float(h_res), float(min_d), float(max_d), _p(ordered),
                              _p(depth), _p(col), _p(rs), _p(re))
    return dict(ordered=ordered[:n].copy(), depth=depth, col=col, row_start=rs, row_end=re, n=n)


def extract_features(depth, col, n, row_start, row_end, corner_thr=1.0, planar_thr=0.1):
    depth = np.ascontiguousarray(depth, np.float32)
    col = np.ascontiguousarray(col, np.int32)
    rs = np.ascontiguousarray(row_start, np.int32)
    re = np.ascontiguousarray(row_end, np.int32)
    V = len(rs)
    ci = np.zeros(120 * V + 16, np.int32)
    pi = np.zeros(n + 6 * V + 16, np.int32)
    nc, npl = C.c_size_t(0), C.c_size_t(0)
    sec = C.c_double(0)
    lib().orc_extract_features(_p(depth), _p(col), n, _p(rs), _p(re), V, float(corner_thr), float(planar_thr), _p(ci), C.byref(nc), _p(pi),
                               C.byref(npl), C.byref(sec))
    return ci[:nc.value].copy(), pi[:npl.value].copy(), sec.value
