"""Every C entry that takes a device index rejects an unusable one the same way: FLS_ERR_NO_DEVICE, and no output written.  An index is
usable when it names a visible CUDA device; runs with or without a GPU (the indices below are never usable)."""
import ctypes as C

import numpy as np
import pytest

from funny_lidar_slam_b200 import _abi, _lib
from funny_lidar_slam_b200._abi import FlsFeatureCfg, FlsLoamFrontendCfg, FlsPointCloud2, FlsPointField
from funny_lidar_slam_b200.features import convert_cfg

SENTINEL = 7
FAKE_DEVICE_PTR = C.c_void_p(0x1000)  # never dereferenced: the device check fails first
f32, sz = C.c_float, C.c_size_t


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def _outs(*shapes, dtype=np.float32):
    return [np.full(s, SENTINEL, dtype) for s in shapes]


def _written(*outs):
    return any(np.any(o != SENTINEL) for o in outs)


# each case calls one entry with valid arguments on `device` and returns (status, whether it wrote an output: a handle, points or indices)
def _create(L, device):
    cfg = _abi.default_config(_abi.FLS_P2PLANE_IVOX)
    cfg.device = device
    h = C.c_void_p(SENTINEL)
    rc = L.fls_create(C.byref(cfg), C.byref(h))
    return rc, h.value is not None


def _keyframes_create(L, device):
    s = C.c_void_p(SENTINEL)
    rc = L.fls_keyframes_create(device, 1000, C.byref(s))
    return rc, s.value is not None


def _voxel_grid(L, device):
    pts = np.arange(16, dtype=np.float32).reshape(4, 4)
    (out,) = _outs((4, 4))
    n = sz(SENTINEL)
    rc = L.fls_voxel_grid(device, _vp(pts), 4, 16, 0.5, _vp(out), C.byref(n))
    return rc, _written(out) or n.value != SENTINEL


def _project(L, device, imu):
    raw = np.arange(16, dtype=np.float32).reshape(4, 4) + 2.0
    ring = np.zeros(4, np.int32)
    time = np.zeros(4, np.float32)
    ordered, depth = _outs((16, 4), 16)
    col, rs, re = _outs(16, 2, 2, dtype=np.int32)
    n = sz(SENTINEL)
    geom = (2, 8, f32(0.78), f32(1.0), f32(50.0), _vp(ordered), _vp(depth), _vp(col), _vp(rs), _vp(re), C.byref(n))
    if imu:
        rc = L.fls_project_imu(device, _vp(raw), _vp(ring), _vp(time), sz(4), sz(16), None, *geom)
    else:
        rc = L.fls_project(device, _vp(raw), _vp(ring), sz(4), sz(16), *geom)
    return rc, _written(ordered, depth, col, rs, re)


def _preprocess(L, device):
    raw = np.arange(20, dtype=np.float32).reshape(4, 5) + 2.0
    ordered, planar = _outs((4, 4), (4, 4))
    no, npl = sz(SENTINEL), sz(SENTINEL)
    rc = L.fls_preprocess(device, _vp(raw), sz(4), None, f32(1.0), f32(50.0), 4, f32(0.5), _vp(ordered), C.byref(no), _vp(planar), C.byref(npl))
    return rc, _written(ordered, planar)


def _preprocess_device(L, device):
    ordered, planar = _outs((4, 4), (4, 4))
    no, npl = sz(SENTINEL), sz(SENTINEL)
    rc = L.fls_preprocess_device(device, FAKE_DEVICE_PTR, None, 4, None, 1.0, 50.0, 4, 0.5, _vp(ordered), None, C.byref(no), _vp(planar), None,
                                 C.byref(npl))
    return rc, _written(ordered, planar)


def _loam_cfg(device):
    return FlsLoamFrontendCfg(device, 16, 1800, 0.0035, 2.0, 80.0, 1.0, 0.1, 0.2, 0.4)


def _preprocess_loam(L, device):
    raw = np.arange(16, dtype=np.float32).reshape(4, 4) + 2.0
    ring = np.zeros(4, np.int32)
    corner, planar = _outs((4, 4), (4, 4))
    nc, npl = sz(SENTINEL), sz(SENTINEL)
    cfg = _loam_cfg(device)
    rc = L.fls_preprocess_loam(C.byref(cfg), _vp(raw), _vp(ring), None, 4, 16, None, _vp(corner), _vp(planar), None, None, C.byref(nc), C.byref(npl),
                               None)
    return rc, _written(corner, planar)


def _preprocess_loam_device(L, device):
    corner, planar = _outs((4, 4), (4, 4))
    nc, npl = sz(SENTINEL), sz(SENTINEL)
    cfg = _loam_cfg(device)
    rc = L.fls_preprocess_loam_device(C.byref(cfg), FAKE_DEVICE_PTR, FAKE_DEVICE_PTR, None, 4, None, _vp(corner), _vp(planar), None, None, C.byref(nc),
                                      C.byref(npl), None)
    return rc, _written(corner, planar)


def _extract_features(L, device):
    n, rows = 64, 2
    depth = np.full(n, 5.0, np.float32)
    col = np.arange(n, dtype=np.int32)
    rs = np.array([5, 37], np.int32)
    re = np.array([26, 58], np.int32)
    ci, pi = _outs(n, n, dtype=np.int32)
    nc, npl = sz(SENTINEL), sz(SENTINEL)
    cfg = FlsFeatureCfg(0.1, 1.0, device, 0)
    rc = L.fls_extract_features(C.byref(cfg), _vp(depth), _vp(col), n, _vp(rs), _vp(re), rows, _vp(ci), C.byref(nc), _vp(pi), C.byref(npl), None)
    return rc, _written(ci, pi)


def _convert_cloud(L, device):
    data = np.arange(16, dtype=np.float32).reshape(4, 4)
    fields = (FlsPointField * 4)(*[FlsPointField(name, 4 * k, 7, 1, 0) for k, name in enumerate([b"x", b"y", b"z", b"intensity"])])
    msg = FlsPointCloud2(_vp(data).value, 0, 1, 4, 16, 64, 1, 0, 4, fields, 1)
    xyzi = _outs((4, 4))[0]
    n = sz(SENTINEL)
    res = _abi.FlsConvertResult()
    cfg = convert_cfg(_abi.FLS_LIDAR_VELODYNE, 16, 1.0, device=device)
    rc = L.fls_convert_cloud(C.byref(cfg), C.byref(msg), _vp(xyzi), None, None, None, None, None, C.byref(n), C.byref(res), None)
    return rc, _written(xyzi)


ENTRIES = {
    "fls_create": _create,
    "fls_keyframes_create": _keyframes_create,
    "fls_voxel_grid": _voxel_grid,
    "fls_project": lambda L, d: _project(L, d, imu=False),
    "fls_project_imu": lambda L, d: _project(L, d, imu=True),
    "fls_preprocess": _preprocess,
    "fls_preprocess_device": _preprocess_device,
    "fls_preprocess_loam": _preprocess_loam,
    "fls_preprocess_loam_device": _preprocess_loam_device,
    "fls_extract_features": _extract_features,
    "fls_convert_cloud": _convert_cloud,
}


@pytest.mark.parametrize("entry", sorted(ENTRIES))
def test_unusable_device_index_is_rejected_without_output(entry):
    L = _lib.lib()
    ndev = L.fls_device_count()
    for device in (-1, ndev, 64):
        rc, written = ENTRIES[entry](L, device)
        assert rc == _abi.FLS_ERR_NO_DEVICE, (entry, device, rc)
        assert not written, (entry, device)
