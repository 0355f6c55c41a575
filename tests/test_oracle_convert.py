"""The conversion oracle (oracle_convert/orc_convert.h) against a literal Python restatement of ConvertMessageToCloud,
ComputePointOffsetTime, GetLidarPointMinMaxOffsetTime and the stamps (src/slam/preprocessing.cpp:86-104, 262-571 upstream) on every
sensor type and edge; the pinned atan2f against a correctly rounded reference; the layouts of the new ABI structs; and the argument
checks of fls_convert_cloud and the device-input pre-processing entries, which fail before any device is touched."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

from funny_lidar_slam_b200._abi import (FLS_ERR_INVALID_ARG, FLS_ERR_NO_DEVICE, FLS_ERR_UNSUPPORTED, FLS_LIDAR_LIVOX_AVIA, FLS_LIDAR_LIVOX_MID_360,
                                        FLS_LIDAR_NONE, FLS_LIDAR_OUSTER, FLS_LIDAR_ROBOSENSE, FLS_LIDAR_VELODYNE, FlsConvertCfg, FlsConvertResult,
                                        FlsPointCloud2, FlsPointField)
from tests import convert_msgs as cm

f32 = np.float32


# ---- the restatement ---------------------------------------------------------------------------------------------------------
def _from_ros_msg(msg, lidar_type):
    """pcl::fromROSMsg: every struct field of the point type reads the first message field with its name, datatype and count 0 or 1."""
    want = {"x": 7, "y": 7, "z": 7, "intensity": 7}
    want.update({FLS_LIDAR_VELODYNE: {"ring": 4, "time": 7}, FLS_LIDAR_OUSTER: {"t": 6, "ring": 2},
                 FLS_LIDAR_ROBOSENSE: {"ring": 4, "timestamp": 8}, 4: {"ring": 4, "timestamp": 8},
                 FLS_LIDAR_LIVOX_MID_360: {"tag": 2, "line": 2, "timestamp": 8}, FLS_LIDAR_LIVOX_AVIA: {"time": 6, "line": 2, "tag": 2},
                 FLS_LIDAR_NONE: {}}[lidar_type])
    np_type = {2: np.uint8, 4: np.uint16, 6: np.uint32, 7: np.float32, 8: np.float64}
    data = np.asarray(msg.data, np.uint8)
    pts = []
    for row in range(msg.height):
        for c in range(msg.width):
            base = row * msg.row_step + c * msg.point_step
            p = {}
            for name, dt in want.items():
                src = next((o for n, o, d, k in msg.fields if n == name and d == dt and k in (0, 1)), None)
                p[name] = np_type[dt](0) if src is None else data[base + src:base + src + np.dtype(np_type[dt]).itemsize].view(np_type[dt])[0]
            pts.append(p)
    return pts


def _finite(p):
    return math.isfinite(p["x"]) and math.isfinite(p["y"]) and math.isfinite(p["z"])


def _compute_point_offset_time(cloud, n_rows, yaw_of):
    lidar_omega = 2.0 * math.pi * 10.0
    is_first, yaw_first, time_last = [True] * n_rows, [0.0] * n_rows, [f32(0)] * n_rows
    for i, p in enumerate(cloud):
        ring = p["ring"]
        if ring >= n_rows:
            continue
        yaw = float(yaw_of[i])
        if is_first[ring]:
            yaw_first[ring], is_first[ring], time_last[ring] = yaw, False, f32(0)
            continue
        if yaw <= yaw_first[ring]:
            p["time"] = f32((yaw_first[ring] - yaw) / lidar_omega)
        else:
            p["time"] = f32((yaw_first[ring] - yaw + 2.0 * math.pi) / lidar_omega)
        if p["time"] < time_last[ring]:
            p["time"] = f32(p["time"] + f32(2.0 * math.pi / lidar_omega))
        time_last[ring] = p["time"]


def restate(msg, lidar_type, n_rows, time_scale, lower_angle=0.0, v_res=0.0):
    """ConvertMessageToCloud (:262-511) -> GetLidarPointMinMaxOffsetTime (:554-571) -> the stamps (:86-104), loop for loop."""
    from oracle import pyoracle as orc
    from oracle_convert import pyoracle_convert as orcc
    src = _from_ros_msg(msg, lidar_type)
    stamp, recomputed, cloud = msg.stamp_us, False, []
    if lidar_type in (FLS_LIDAR_VELODYNE, FLS_LIDAR_OUSTER, 4, FLS_LIDAR_ROBOSENSE, FLS_LIDAR_LIVOX_MID_360):
        if not msg.is_dense:
            src = [p for p in src if _finite(p)]
        if src:
            ts0 = float(src[0].get("timestamp", 0.0))
            if lidar_type == FLS_LIDAR_ROBOSENSE:
                stamp = int(ts0 * 1.0e6)
            for p in src:
                q = dict(x=p["x"], y=p["y"], z=p["z"], intensity=p["intensity"])
                if lidar_type == FLS_LIDAR_VELODYNE:
                    q.update(ring=int(p["ring"]) & 0xff, time=f32(float(p["time"]) * time_scale))
                elif lidar_type == FLS_LIDAR_OUSTER:
                    q.update(ring=int(p["ring"]), time=f32(float(p["t"]) * time_scale))
                elif lidar_type == 4:
                    q.update(ring=int(p["ring"]) & 0xff, time=f32(float(p["timestamp"]) * time_scale))
                elif lidar_type == FLS_LIDAR_ROBOSENSE:
                    q.update(ring=int(p["ring"]) & 0xff, time=f32((float(p["timestamp"]) - ts0) * time_scale))
                else:
                    q.update(ring=0, time=f32((float(p["timestamp"]) - ts0) * time_scale))
                cloud.append(q)
            if lidar_type == FLS_LIDAR_VELODYNE and cloud[-1]["time"] <= f32(0):
                yaw = orcc.atan2f([p["y"] for p in cloud], [p["x"] for p in cloud])
                _compute_point_offset_time(cloud, n_rows, yaw)
                recomputed = True
    elif lidar_type == FLS_LIDAR_LIVOX_AVIA:
        for p in src:
            if p["line"] < 6 and (int(p["tag"]) & 0x30) in (0x10, 0x00):
                cloud.append(dict(x=p["x"], y=p["y"], z=p["z"], intensity=p["intensity"], ring=0, time=f32(float(p["time"]) * time_scale)))
    else:
        for p in src:
            if not _finite(p):
                continue
            xy = np.sqrt(f32(p["x"] * p["x"]) + f32(p["y"] * p["y"]), dtype=f32)
            v = f32(f32(f32(orc.fast_atan2f(p["z"], xy)) + f32(lower_angle)) / f32(v_res))
            row = int(np.trunc(v)) + (int(np.sign(v)) if abs(float(v) - float(np.trunc(v))) >= 0.5 else 0)  # std::round: half away from 0
            if row >= n_rows or row < 0:
                continue
            cloud.append(dict(x=p["x"], y=p["y"], z=p["z"], intensity=p["intensity"], ring=row & 0xff, time=f32(0)))
        if cloud and cloud[-1]["time"] <= f32(0):
            yaw = orcc.atan2f([p["y"] for p in cloud], [p["x"] for p in cloud])
            _compute_point_offset_time(cloud, n_rows, yaw)
            recomputed = True
    out = dict(n=len(cloud), xyzi=np.array([[p["x"], p["y"], p["z"], p["intensity"]] for p in cloud], f32).reshape(-1, 4),
               ring=np.array([p["ring"] for p in cloud], np.int32), time=np.array([p["time"] for p in cloud], f32),
               stamp_us=stamp, valid=bool(cloud), recomputed=recomputed, start_us=0, end_us=0, min_time=0.0, max_time=0.0)
    if cloud:
        mn = mx = cloud[0]["time"]
        for p in cloud:
            if p["time"] < mn:
                mn = p["time"]
            if p["time"] > mx:
                mx = p["time"]

        def trunc(v):  # static_cast<int64_t>, x86-64: INT64_MIN for NaN / out of range
            return int(v) if math.isfinite(v) and -2.0 ** 63 <= v < 2.0 ** 63 else -2 ** 63
        start = (stamp + trunc(float(mn) * 1.0e6)) % 2 ** 64
        end = (stamp + trunc(float(mx) * 1.0e6)) % 2 ** 64
        if stamp < start:
            start = stamp
        elif stamp > end:
            end = stamp
        out.update(start_us=start, end_us=end, min_time=float(mn), max_time=float(mx))
    return out


def _bits(v):
    """float32 bit patterns with every NaN made the same: a NaN's payload is not part of the result (x86 propagates an operand's
    payload, the GPU returns the canonical NaN), its position is."""
    v = np.array(v, f32, ndmin=1)
    return np.where(np.isnan(v), np.uint32(0x7fc00000), v.view(np.uint32))


def same(a, b, keys=("n", "stamp_us", "valid", "recomputed", "start_us", "end_us")):
    """Bit-identical arrays and window (-0 != +0; NaN == NaN whatever its payload)."""
    for k in keys:
        assert a[k] == b[k], (k, a[k], b[k])
    for k in ("min_time", "max_time"):
        assert np.array_equal(_bits(a[k]), _bits(b[k])), (k, a[k], b[k])
    assert np.array_equal(_bits(a["xyzi"]), _bits(b["xyzi"]))
    assert np.array_equal(a["ring"], b["ring"])
    assert np.array_equal(_bits(a["time"]), _bits(b["time"]))


CASES = cm.cases(n=1500)


@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_oracle_equals_literal_restatement(name):
    from oracle_convert import pyoracle_convert as orcc
    _, msg, kw = next(c for c in CASES if c[0] == name)
    same(orcc.convert_message(msg, **kw), restate(msg, **kw))


def test_cases_cover_the_branches():
    from oracle_convert import pyoracle_convert as orcc
    got = {name: orcc.convert_message(msg, **kw) for name, msg, kw in CASES}
    assert got["velodyne_no_time"]["recomputed"] and not got["velodyne"]["recomputed"]
    assert got["none"]["recomputed"] and got["none"]["n"] > 1000
    assert np.all(got["ouster_ring_u16_reads_0"]["ring"] == 0)
    assert got["velodyne_time_f64_reads_0"]["recomputed"]  # the float64 time reads 0: the offsets are recomputed
    assert got["velodyne_ring_u16_ge_256"]["ring"].max() > 200
    assert 0 < got["avia"]["n"] < 1500 and got["none_rows_out_of_range"]["n"] < got["none"]["n"]
    assert got["velodyne_nan_dense0"]["n"] < 1500 and got["velodyne_nan_dense1"]["n"] == 1500
    assert got["robosense_nan_first_dense0"]["stamp_us"] == int((1.7e9) * 1e6)
    assert math.isnan(got["velodyne_nan_first_time"]["min_time"]) and math.isnan(got["velodyne_nan_first_time"]["max_time"])
    assert np.signbit(np.float32(got["velodyne_signed_zero_times"]["min_time"]))
    # skipped rings keep their (zero) time during the recompute
    r = got["velodyne_no_time_ring_ge_n_rows"]
    assert np.all(r["time"][r["ring"] >= 12] == 0) and np.any(r["time"][r["ring"] < 12] > 0)
    for k in ("velodyne_empty", "robosense_all_nan", "none_all_nan", "avia_nothing_kept"):
        assert got[k]["n"] == 0 and not got[k]["valid"] and got[k]["stamp_us"] == cm.STAMP_US


# the rotation sense of a real Velodyne needs the scan to carry state: identity maps after a +2 pi / omega (state 1)
CARRY_CASES = ["velodyne_cw_no_time", "velodyne_cw_no_time_ring_ge_n_rows", "none_cw"]


@pytest.mark.parametrize("name", CARRY_CASES)
def test_clockwise_cases_carry_state_through_the_scan(name):
    from oracle_convert import pyoracle_convert as orcc
    _, msg, kw = next(c for c in CASES if c[0] == name)
    got = orcc.convert_message(msg, **kw)
    assert got["recomputed"]
    h = cm.offset_maps(got["xyzi"], got["ring"], kw["n_rows"], orcc.atan2f(got["xyzi"][:, 1], got["xyzi"][:, 0]))
    assert h["identity"] > got["n"] // 2 and h["identity_carrying_1"] > 20 and h["const0"] + h["const1"] > 10, h
    # the offsets after a ring's first yaw is passed again are the ones that got the +2 pi / omega
    assert got["max_time"] > 0.1


# ---- the pinned atan2f ---------------------------------------------------------------------------------------------------------
def _boundary_pairs(rng, m):
    """Octant boundaries (|y| = |x| +- a few ulps), the axes, signed zeros, infinities, subnormals and tiny / huge ratios."""
    x = rng.uniform(1e-3, 1e3, m).astype(f32)
    sgn = lambda k: rng.choice(np.array([-1, 1], f32), k)
    ys = [x * sgn(m)]
    for d in (1, 2, 3, 17):
        ys.append(np.nextafter(x, np.float32(np.inf)) if d == 1 else (x.view(np.int32) + d).view(f32))
        ys.append((x.view(np.int32) - d).view(f32))
    y = np.concatenate(ys)
    xx = np.tile(x, len(ys)) * np.concatenate([sgn(m) for _ in ys])
    special = np.array([0.0, -0.0, np.inf, -np.inf, 1.0, -1.0, 1e-45, -1e-45, 1e-40, 3.4e38, -3.4e38, 1.17549435e-38], f32)
    sy, sx = np.meshgrid(special, special)
    sub = (rng.integers(1, 2 ** 23, m).astype(np.int32)).view(f32) * sgn(m)
    yy = np.concatenate([y, sy.ravel(), sub, rng.uniform(-1, 1, m).astype(f32)])
    xs = np.concatenate([xx, sx.ravel(), rng.uniform(-5, 5, m).astype(f32), sub * f32(1e-10)])
    return yy, xs


def _certified_reference(y, x):
    """float32(atan2) correctly rounded: float64 atan2 (libm, within 1 ulp of fp64) decides every case whose result is not within 2^-45
    relative of a float32 rounding boundary; mpmath at 60 digits decides the others."""
    import mpmath
    mpmath.mp.dps = 60
    d = np.arctan2(y.astype(np.float64), x.astype(np.float64))
    r = d.astype(f32)
    lo = np.nextafter(r, np.float32(-np.inf)).astype(np.float64)
    hi = np.nextafter(r, np.float32(np.inf)).astype(np.float64)
    mid_lo, mid_hi = (lo + r.astype(np.float64)) / 2, (hi + r.astype(np.float64)) / 2
    tol = np.abs(d) * 2.0 ** -45 + 1e-300
    unsure = np.isfinite(d) & ((np.abs(d - mid_lo) < tol) | (np.abs(d - mid_hi) < tol) | (np.abs(r) < 1.2e-38))
    for i in np.flatnonzero(unsure):
        # mpmath has no signed zero: the sign of atan2 is the sign of y, as float64 atan2 has it
        r[i] = np.copysign(f32(float(mpmath.atan2(mpmath.mpf(float(y[i])), mpmath.mpf(float(x[i]))))), d[i])
    return r, int(unsure.sum())


def test_pinned_atan2f_is_correctly_rounded():
    from oracle_convert import pyoracle_convert as orcc
    rng = np.random.default_rng(2024)
    n = 700_000
    y = np.concatenate([(rng.standard_normal(n) * 10 ** rng.uniform(-6, 6, n)).astype(f32), _boundary_pairs(rng, 20_000)[0]])
    x = np.concatenate([(rng.standard_normal(n) * 10 ** rng.uniform(-6, 6, n)).astype(f32), _boundary_pairs(rng, 20_000)[1]])
    pts, _, _, _ = cm.scan(sensor="hdl64")
    y = np.concatenate([y, pts[:, 1]])
    x = np.concatenate([x, pts[:, 0]])
    assert len(y) >= 1_000_000
    got = orcc.atan2f(y, x)
    ref, n_mp = _certified_reference(y, x)
    bad = np.flatnonzero(got.view(np.uint32) != ref.view(np.uint32))
    assert len(bad) == 0, [(float(y[i]), float(x[i]), float(got[i]), float(ref[i])) for i in bad[:10]]
    # a direct mpmath check on a sample, and the IEEE special values
    import mpmath
    for i in rng.choice(len(y), 3000, replace=False):
        if np.isfinite(y[i]) and np.isfinite(x[i]):
            assert got[i] == f32(float(mpmath.atan2(mpmath.mpf(float(y[i])), mpmath.mpf(float(x[i]))))), (y[i], x[i])  # -0 == 0 here
    a = lambda yy, xx: orcc.atan2f([yy], [xx])[0]
    pi = f32(np.pi)
    assert np.signbit(a(-0.0, 1.0)) and a(-0.0, 1.0) == 0 and a(0.0, -0.0) == pi and a(-0.0, -0.0) == -pi and a(0.0, 0.0) == 0
    assert a(1.0, 0.0) == f32(np.pi / 2) and a(-1.0, -0.0) == -f32(np.pi / 2) and a(2.0, -3.0e38) == pi
    assert a(np.inf, np.inf) == f32(np.pi / 4) and a(-np.inf, -np.inf) == -f32(3 * np.pi / 4) and np.isnan(a(np.nan, 1.0))


# ---- ABI layout and argument checks (no device needed) -------------------------------------------------------------------------
def test_convert_structs_match_header(tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no C compiler")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    checks = [("fls_point_field", FlsPointField, ("offset", "datatype", "count")),
              ("fls_pointcloud2", FlsPointCloud2, ("data_on_device", "height", "width", "point_step", "row_step", "is_dense", "is_bigendian",
                                                   "n_fields", "fields", "stamp_us", "reserved")),
              ("fls_convert_cfg", FlsConvertCfg, ("lidar_type", "n_rows", "lower_angle", "v_res", "time_scale", "reserved")),
              ("fls_convert_result", FlsConvertResult, ("start_us", "end_us", "min_time", "max_time", "valid", "recomputed", "reserved"))]
    body = "".join(f'  printf("%zu\\n", sizeof({s}));\n' + "".join(f'  printf("%zu\\n", offsetof({s}, {f}));\n' for f in fs) for s, _, fs in checks)
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "fls_b200.h"\nint main(void) {\n' + body + "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.check_call([gcc, "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    want = []
    for _, cls, fs in checks:
        want += [C.sizeof(cls)] + [getattr(cls, f).offset for f in fs]
    assert got == want
    assert (C.sizeof(FlsPointField), C.sizeof(FlsPointCloud2), C.sizeof(FlsConvertCfg), C.sizeof(FlsConvertResult)) == (24, 72, 48, 48)


def test_convert_argument_checks():
    from funny_lidar_slam_b200._lib import lib
    from funny_lidar_slam_b200.features import PointCloud2, convert_cfg
    L = lib()
    rec = cm.records(FLS_LIDAR_VELODYNE, *cm.scan(n=64))
    out = np.zeros((64, 4), np.float32)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)

    def call(msg, cfg=None, outs=True, n=True, res=True):
        m, keep = msg.struct()
        nn, rr = C.c_size_t(5), FlsConvertResult()
        cfg = convert_cfg(FLS_LIDAR_VELODYNE, 16, 1.0) if cfg is None else cfg
        rr.valid = 7
        rc = L.fls_convert_cloud(C.byref(cfg) if cfg is not False else None, C.byref(m), vp(out) if outs else None, None, None, None, None, None,
                                 C.byref(nn) if n else None, C.byref(rr) if res else None, None)
        return rc, rr.valid

    good = cm.message(rec)
    assert call(good, cfg=False)[0] == FLS_ERR_INVALID_ARG
    assert call(good, n=False)[0] == FLS_ERR_INVALID_ARG and call(good, res=False)[0] == FLS_ERR_INVALID_ARG
    assert call(good, outs=False)[0] == FLS_ERR_INVALID_ARG
    assert call(good, cfg=convert_cfg(7, 16, 1.0))[0] == FLS_ERR_INVALID_ARG
    assert call(good, cfg=convert_cfg(FLS_LIDAR_VELODYNE, 0, 1.0))[0] == FLS_ERR_INVALID_ARG
    assert call(good, cfg=convert_cfg(FLS_LIDAR_VELODYNE, 16, float("nan")))[0] == FLS_ERR_INVALID_ARG
    assert call(good, cfg=convert_cfg(FLS_LIDAR_NONE, 16, 1.0, 0.26, 0.0))[0] == FLS_ERR_INVALID_ARG  # v_res unset
    assert call(good, cfg=convert_cfg(FLS_LIDAR_NONE, 16, 1.0, 3.4e38, 0.03))[0] == FLS_ERR_INVALID_ARG  # lower_angle sentinel
    f = good.fields
    # a field that does not fit in point_step, row_step < width * point_step: invalid, nothing written
    bad_field = PointCloud2(good.data, f + [("extra", 30, 8, 1)], good.width, 1, 32, stamp_us=1)
    assert call(bad_field) == (FLS_ERR_INVALID_ARG, 7)
    bad_count = PointCloud2(good.data, f[:-1] + [("time", 24, 7, 3)], good.width, 1, 32, stamp_us=1)
    assert call(bad_count) == (FLS_ERR_INVALID_ARG, 7)
    short_rows = PointCloud2(good.data, f, good.width, 1, 32, row_step=32 * good.width - 1, stamp_us=1)
    assert call(short_rows) == (FLS_ERR_INVALID_ARG, 7)
    big_endian = PointCloud2(good.data, f, good.width, 1, 32, is_bigendian=True, stamp_us=1)
    assert call(big_endian) == (FLS_ERR_UNSUPPORTED, 7)
    assert np.all(out == 0)
    if L.fls_device_count() < 1:
        assert call(good)[0] == FLS_ERR_NO_DEVICE


def test_device_input_entries_argument_checks():
    from funny_lidar_slam_b200._abi import FlsLoamFrontendCfg
    from funny_lidar_slam_b200._lib import lib
    L = lib()
    nc, npl = C.c_size_t(3), C.c_size_t(3)
    out = np.zeros((64, 4), np.float32)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    cfg = FlsLoamFrontendCfg(0, 16, 1800, 0.0035, 2.0, 80.0, 1.0, 0.1, 0.2, 0.4)
    fake = C.c_void_p(0x1000)  # never dereferenced: every call below fails its checks first
    assert L.fls_preprocess_loam_device(None, fake, fake, None, 4, None, vp(out), vp(out), None, None, C.byref(nc), C.byref(npl), None) == FLS_ERR_INVALID_ARG
    assert L.fls_preprocess_loam_device(C.byref(cfg), None, fake, None, 4, None, vp(out), vp(out), None, None, C.byref(nc), C.byref(npl), None) == FLS_ERR_INVALID_ARG
    assert L.fls_preprocess_loam_device(C.byref(cfg), fake, None, None, 4, None, vp(out), vp(out), None, None, C.byref(nc), C.byref(npl), None) == FLS_ERR_INVALID_ARG
    assert L.fls_preprocess_loam_device(C.byref(cfg), fake, fake, None, 4, None, None, None, None, None, C.byref(nc), C.byref(npl), None) == FLS_ERR_INVALID_ARG
    assert (nc.value, npl.value) == (0, 0)
    bad = FlsLoamFrontendCfg(0, 16, 1800, 0.0035, 2.0, 80.0, 1.0, 0.1, 0.0, 0.4)
    assert L.fls_preprocess_loam_device(C.byref(bad), fake, fake, None, 4, None, vp(out), vp(out), None, None, C.byref(nc), C.byref(npl), None) == FLS_ERR_INVALID_ARG
    no, npl2 = C.c_size_t(3), C.c_size_t(3)
    args = lambda **kw: [kw.get("dev", 0), kw.get("x", fake), None, 4, None, C.c_float(2.0), C.c_float(80.0), kw.get("jump", 1), C.c_float(kw.get("leaf", 0.4)),
                         kw.get("o", vp(out)), None, C.byref(no), kw.get("p", vp(out)), None, C.byref(npl2)]
    assert L.fls_preprocess_device(*args(x=None)) == FLS_ERR_INVALID_ARG
    assert L.fls_preprocess_device(*args(jump=0)) == FLS_ERR_INVALID_ARG
    assert L.fls_preprocess_device(*args(leaf=0.0)) == FLS_ERR_INVALID_ARG
    assert L.fls_preprocess_device(*args(o=None, p=None)) == FLS_ERR_INVALID_ARG
    assert (no.value, npl2.value) == (0, 0)
    if L.fls_device_count() < 1:
        assert L.fls_preprocess_device(*args()) == FLS_ERR_NO_DEVICE
