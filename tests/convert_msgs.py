"""PointCloud2 messages for the conversion tests: the seven sensor types in their ROS drivers' layouts, built from a synthetic scan with
numpy structured dtypes (explicit offsets and itemsize), and the edge cases of ConvertMessageToCloud."""
import numpy as np

from funny_lidar_slam_b200 import synth
from funny_lidar_slam_b200._abi import (FLS_LIDAR_LEISHEN, FLS_LIDAR_LIVOX_AVIA, FLS_LIDAR_LIVOX_MID_360, FLS_LIDAR_NONE, FLS_LIDAR_OUSTER,
                                        FLS_LIDAR_ROBOSENSE, FLS_LIDAR_VELODYNE)
from funny_lidar_slam_b200.features import PointCloud2

STAMP_US = 1_700_000_000_123_456
# (names, formats, offsets, itemsize) of each driver's point, and lidar_point_time_scale for its time unit
LAYOUTS = {
    FLS_LIDAR_VELODYNE: ((["x", "y", "z", "intensity", "ring", "time"], ["<f4", "<f4", "<f4", "<f4", "<u2", "<f4"], [0, 4, 8, 16, 20, 24], 32), 1.0),
    FLS_LIDAR_OUSTER: ((["x", "y", "z", "intensity", "t", "reflectivity", "ring", "ambient", "range"],
                        ["<f4", "<f4", "<f4", "<f4", "<u4", "<u2", "u1", "<u2", "<u4"], [0, 4, 8, 16, 20, 24, 26, 28, 32], 48), 1e-9),
    FLS_LIDAR_ROBOSENSE: ((["x", "y", "z", "intensity", "ring", "timestamp"], ["<f4", "<f4", "<f4", "<f4", "<u2", "<f8"], [0, 4, 8, 12, 16, 24], 32), 1.0),
    FLS_LIDAR_LEISHEN: ((["x", "y", "z", "intensity", "ring", "timestamp"], ["<f4", "<f4", "<f4", "<f4", "<u2", "<f8"], [0, 4, 8, 12, 16, 24], 32), 1.0),
    FLS_LIDAR_LIVOX_MID_360: ((["x", "y", "z", "intensity", "tag", "line", "timestamp"], ["<f4", "<f4", "<f4", "<f4", "u1", "u1", "<f8"],
                               [0, 4, 8, 12, 16, 17, 18], 26), 1e-9),
    FLS_LIDAR_LIVOX_AVIA: ((["x", "y", "z", "intensity", "time", "line", "tag"], ["<f4", "<f4", "<f4", "<f4", "<u4", "u1", "u1"], [0, 4, 8, 12, 16, 20, 21], 24), 1e-9),
    FLS_LIDAR_NONE: ((["x", "y", "z", "intensity"], ["<f4", "<f4", "<f4", "<f4"], [0, 4, 8, 16], 32), 1.0),
}
ALL_TYPES = list(LAYOUTS)
TYPE_NAMES = {FLS_LIDAR_VELODYNE: "velodyne", FLS_LIDAR_OUSTER: "ouster", FLS_LIDAR_ROBOSENSE: "robosense", FLS_LIDAR_LEISHEN: "leishen",
              FLS_LIDAR_LIVOX_MID_360: "mid360", FLS_LIDAR_LIVOX_AVIA: "avia", FLS_LIDAR_NONE: "none"}
NONE_LOWER, NONE_VRES = float(np.float32(np.deg2rad(15.0))), float(np.float32(np.deg2rad(2.0)))  # VLP-16: -15..15 deg, 2 deg apart


def dtype_of(lidar_type, layout=None):
    names, formats, offsets, itemsize = layout or LAYOUTS[lidar_type][0]
    return np.dtype({"names": names, "formats": formats, "offsets": offsets, "itemsize": itemsize})


def scan(sensor="vlp16", pose_index=3, seed=7, n=None):
    """A synthetic scan in firing order (column-major over rings): points (n,4), ring, col, cols."""
    world = synth.make_world()
    sc = synth.make_scan(world, synth.trajectory(8)[pose_index], sensor, seed=seed)
    order = np.lexsort((sc["ring"], sc["col"]))
    pts, ring, col = sc["points"][order], sc["ring"][order].astype(np.int64), sc["col"][order].astype(np.int64)
    if n is not None:
        pts, ring, col = pts[:n], ring[:n], col[:n]
    return pts, ring, col, synth.SENSORS[sensor].cols


def clockwise_scan(sensor="vlp16", pose_index=3, seed=7, col_step=1, extra=0.08):
    """A scan with a real Velodyne's sense of rotation and more than one revolution per ring: the synthetic scan mirrored (y -> -y, so
    the yaw falls with firing order), the first `extra` of every ring's revolution fired again at its end (slightly moved), and 5 % of
    the points rotated by up to three columns either way (a point below its predecessor).  ComputePointOffsetTime then carries
    time_last from point to point (identity maps) and, after a ring passes its first yaw, carries the +2 pi / omega (state 1)."""
    pts, ring, col, cols = scan(sensor, pose_index, seed)
    keep = col % col_step == 0
    pts, ring, col = pts[keep].copy(), ring[keep], col[keep]
    pts[:, 1] = -pts[:, 1]
    again = col < extra * cols
    pts2 = pts[again].copy()
    pts2[:, :3] *= np.float32(1.002)
    pts = np.concatenate([pts, pts2])
    ring = np.concatenate([ring, ring[again]])
    col = np.concatenate([col, col[again] + cols])
    rng = np.random.default_rng(seed + 11)
    k = rng.choice(len(pts), len(pts) // 20, replace=False)
    a = rng.uniform(-3, 3, len(k)) * 2 * np.pi / cols
    x, y = pts[k, 0].astype(np.float64), pts[k, 1].astype(np.float64)
    pts[k, 0], pts[k, 1] = (x * np.cos(a) - y * np.sin(a)).astype(np.float32), (x * np.sin(a) + y * np.cos(a)).astype(np.float32)
    return pts, ring, col, cols


def offset_maps(xyzi, ring, n_rows, yaw):
    """The 2-state maps of ComputePointOffsetTime (preprocessing.cpp:523-551) over a converted cloud, replayed in cloud order with the
    given yaws: counts of constant-0, swap, identity and constant-1 maps of the points after a ring's first, and of identity maps
    whose state before is 1 (a +2 pi / omega carried on by the scan)."""
    omega = 2.0 * np.pi * 10.0
    P = np.float32(2.0 * np.pi / omega)
    yf, prev, state = {}, {}, {}
    hist = dict(const0=0, swap=0, identity=0, const1=0, identity_carrying_1=0)
    names = {0: "const0", 1: "swap", 2: "identity", 3: "const1"}

    def base(r, y):
        d = yf[r] - y
        return np.float32((d if y <= yf[r] else d + 2.0 * np.pi) / omega)
    for i in range(len(xyzi)):
        r = int(ring[i])
        if r >= n_rows:
            continue
        y = float(yaw[i])
        if r not in yf:
            yf[r], prev[r], state[r] = y, None, 0
            continue
        b = base(r, y)
        v0 = np.float32(0) if prev[r] is None else base(r, prev[r])
        v1 = np.float32(0) if prev[r] is None else np.float32(v0 + P)
        m = int(b < v0) | (int(b < v1) << 1)
        hist[names[m]] += 1
        if m == 2 and state[r] == 1:
            hist["identity_carrying_1"] += 1
        state[r] = (m >> state[r]) & 1
        prev[r] = y
    return hist


def records(lidar_type, pts, ring, col, cols, with_time=True, dtype=None, seed=1):
    """The driver record of every point.  Times: 0.1 s per revolution, in the unit of the type's time scale."""
    rng = np.random.default_rng(seed)
    rec = np.zeros(len(pts), dtype or dtype_of(lidar_type))
    names = rec.dtype.names
    for k, f in enumerate(("x", "y", "z", "intensity")):
        if f in names:
            rec[f] = pts[:, k]
    frac = col / float(cols) * 0.1
    if "ring" in names:
        rec["ring"] = ring
    if lidar_type == FLS_LIDAR_VELODYNE and "time" in names and with_time:
        rec["time"] = frac.astype(np.float32)
    if lidar_type == FLS_LIDAR_OUSTER:
        rec["t"] = (frac * 1e9).astype(np.uint32)
        if "reflectivity" in names:
            rec["reflectivity"] = 7
    if lidar_type == FLS_LIDAR_ROBOSENSE:
        rec["timestamp"] = 1.7e9 + frac
    if lidar_type == FLS_LIDAR_LEISHEN:
        rec["timestamp"] = frac
    if lidar_type == FLS_LIDAR_LIVOX_MID_360:
        rec["timestamp"] = 1.7e18 + np.round(frac * 1e9)
        rec["line"] = ring % 4
        rec["tag"] = rng.integers(0, 256, len(pts))
    if lidar_type == FLS_LIDAR_LIVOX_AVIA:
        rec["time"] = (frac * 1e9).astype(np.uint32)
        rec["line"] = ring % 8                       # lines 6, 7 are dropped
        rec["tag"] = rng.integers(0, 256, len(pts))  # every (tag & 0x30) class
    return rec


def message(rec, lidar_type=None, **kw):
    kw.setdefault("stamp_us", STAMP_US)
    return PointCloud2.from_records(rec, **kw)


def convert_kwargs(lidar_type, n_rows=16):
    kw = dict(lidar_type=lidar_type, n_rows=n_rows, time_scale=LAYOUTS[lidar_type][1])
    if lidar_type == FLS_LIDAR_NONE:
        kw.update(lower_angle=NONE_LOWER, v_res=NONE_VRES)
    return kw


def cases(n=None):
    """(name, message, convert kwargs) for every sensor type and edge the conversion must reproduce."""
    pts, ring, col, cols = scan(n=n)
    out = []
    for t in ALL_TYPES:
        out.append((f"{TYPE_NAMES[t]}", message(records(t, pts, ring, col, cols)), convert_kwargs(t)))
    V = FLS_LIDAR_VELODYNE
    # Velodyne without a time field: ComputePointOffsetTime; with one, but rings beyond n_rows (skipped, keep their time)
    vel_nt = dtype_of(V, (["x", "y", "z", "intensity", "ring"], ["<f4"] * 4 + ["<u2"], [0, 4, 8, 16, 20], 24))
    out.append(("velodyne_no_time", message(records(V, pts, ring, col, cols, dtype=vel_nt)), convert_kwargs(V)))
    out.append(("velodyne_no_time_ring_ge_n_rows", message(records(V, pts, ring, col, cols, dtype=vel_nt)), convert_kwargs(V, n_rows=12)))
    # shuffled field order, extra fields, padding and an odd point_step (unaligned floats)
    shuf = dtype_of(V, (["ring", "pad", "time", "intensity", "z", "x", "y", "extra"], ["<u2", "u1", "<f4", "<f4", "<f4", "<f4", "<f4", "<f8"],
                        [0, 2, 3, 7, 11, 15, 19, 23], 33))
    out.append(("velodyne_shuffled_odd_step", message(records(V, pts, ring, col, cols, dtype=shuf)), convert_kwargs(V)))
    # datatype-mismatched fields read 0: a float64 time and an Ouster uint16 ring
    mism = dtype_of(V, (["x", "y", "z", "intensity", "ring", "time"], ["<f4"] * 4 + ["<u2", "<f8"], [0, 4, 8, 12, 16, 24], 32))
    out.append(("velodyne_time_f64_reads_0", message(records(V, pts, ring, col, cols, dtype=mism)), convert_kwargs(V)))
    O = FLS_LIDAR_OUSTER
    o16 = dtype_of(O, (["x", "y", "z", "intensity", "t", "ring"], ["<f4"] * 4 + ["<u4", "<u2"], [0, 4, 8, 16, 20, 24], 32))
    out.append(("ouster_ring_u16_reads_0", message(records(O, pts, ring, col, cols, dtype=o16)), convert_kwargs(O)))
    # uint16 rings >= 256 go through the uint8 cast
    big = records(V, pts, ring, col, cols)
    big["ring"] = big["ring"].astype(np.uint32) * 37 + 250
    out.append(("velodyne_ring_u16_ge_256", message(big), convert_kwargs(V)))
    big_nt = records(V, pts, ring, col, cols, dtype=vel_nt)
    big_nt["ring"] = (big_nt["ring"].astype(np.uint32) + 254) % 300
    out.append(("velodyne_no_time_ring_u16_ge_256", message(big_nt), convert_kwargs(V)))
    # organized cloud with row_step padding (16 rows)
    m = len(pts) // 16 * 16
    org = records(V, pts[:m], ring[:m], col[:m], cols).reshape(16, -1)
    padded = np.zeros((16, org.shape[1] * 32 + 40), np.uint8)
    padded[:, :org.shape[1] * 32] = org.view(np.uint8).reshape(16, -1)
    f = [(n, org.dtype.fields[n][1], d, 1) for n, d in zip(org.dtype.names, (7, 7, 7, 7, 4, 7))]
    out.append(("velodyne_organized_row_step", PointCloud2(padded.reshape(-1), f, org.shape[1], 16, 32, org.shape[1] * 32 + 40, stamp_us=STAMP_US),
                convert_kwargs(V)))
    # NaNs: removed when not dense, kept when dense (for every type that removes them, and None / Avia)
    rng = np.random.default_rng(5)
    nan_idx = np.sort(rng.choice(len(pts), len(pts) // 10, replace=False))
    for t in ALL_TYPES:
        for dense in (False, True):
            r = records(t, pts, ring, col, cols)
            r["x"][nan_idx[::2]] = np.nan
            r["z"][nan_idx[1::2]] = np.inf
            out.append((f"{TYPE_NAMES[t]}_nan_dense{int(dense)}", message(r, is_dense=dense), convert_kwargs(t)))
    # a NaN first RoboSense point: the times and the stamp are relative to the first KEPT point
    rs = records(FLS_LIDAR_ROBOSENSE, pts, ring, col, cols)
    rs["y"][0] = np.nan
    rs["timestamp"][0] = 1.6e9
    for dense in (False, True):
        out.append((f"robosense_nan_first_dense{int(dense)}", message(rs, is_dense=dense), convert_kwargs(FLS_LIDAR_ROBOSENSE)))
    # Velodyne, dense with NaNs and no time field: NaN yaws in the offsets
    vn = records(V, pts, ring, col, cols, dtype=vel_nt)
    vn["x"][nan_idx] = np.nan
    out.append(("velodyne_no_time_dense_nan", message(vn, is_dense=True), convert_kwargs(V)))
    # a NaN first time stays the minimum and the maximum
    vt = records(V, pts, ring, col, cols)
    vt["time"][0] = np.nan
    out.append(("velodyne_nan_first_time", message(vt), convert_kwargs(V)))
    # signed zeros: the earliest of equal extremes wins
    vz = records(V, pts, ring, col, cols)
    vz["time"][:] = np.where(np.arange(len(pts)) % 3 == 0, -0.0, 0.0).astype(np.float32)
    vz["time"][-1] = 0.05
    out.append(("velodyne_signed_zero_times", message(vz), convert_kwargs(V)))
    # a real Velodyne's sense of rotation, more than one revolution per ring: time_last carried through the segmented scan
    cw = clockwise_scan(col_step=16 if n is not None else 1)
    out.append(("velodyne_cw_no_time", message(records(V, *cw, dtype=vel_nt)), convert_kwargs(V)))
    out.append(("velodyne_cw_no_time_ring_ge_n_rows", message(records(V, *cw, dtype=vel_nt)), convert_kwargs(V, n_rows=12)))
    out.append(("none_cw", message(records(FLS_LIDAR_NONE, *cw)), convert_kwargs(FLS_LIDAR_NONE)))
    # None with rows out of range (a narrow vertical window)
    out.append(("none_rows_out_of_range", message(records(FLS_LIDAR_NONE, pts, ring, col, cols)),
                dict(convert_kwargs(FLS_LIDAR_NONE), n_rows=9)))
    # empty and all-NaN messages: n = 0, result invalid
    for t in (V, FLS_LIDAR_ROBOSENSE, FLS_LIDAR_NONE):
        out.append((f"{TYPE_NAMES[t]}_empty", message(np.zeros(0, dtype_of(t))), convert_kwargs(t)))
        r = records(t, pts[:50], ring[:50], col[:50], cols)
        r["x"][:] = np.nan
        out.append((f"{TYPE_NAMES[t]}_all_nan", message(r, is_dense=False), convert_kwargs(t)))
    # Avia: no kept point
    av = records(FLS_LIDAR_LIVOX_AVIA, pts[:50], ring[:50], col[:50], cols)
    av["line"][:] = 7
    out.append(("avia_nothing_kept", message(av), convert_kwargs(FLS_LIDAR_LIVOX_AVIA)))
    return out
