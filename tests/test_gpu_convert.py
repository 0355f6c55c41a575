"""fls_convert_cloud — ConvertMessageToCloud, ComputePointOffsetTime and the time window on the device — bit for bit against the
conversion oracle on every sensor type and edge; the device-input pre-processing entries (fls_preprocess_loam_device,
fls_preprocess_device) against the host-input entries fed with the converted host arrays; and message -> device Match for LoamFull and
LOAM-iVox against the host chain and the oracle."""
import numpy as np
import pytest

from funny_lidar_slam_b200 import default_config, synth
from funny_lidar_slam_b200._abi import FLS_ERR_UNSUPPORTED, FLS_LIDAR_NONE, FLS_LIDAR_VELODYNE, FLS_LOAM_FULL, FLS_P2PLANE_IVOX
from tests import convert_msgs as cm
from tests.test_oracle_convert import same

gpu = pytest.mark.gpu
MIN_D, MAX_D = 2.0, 80.0
CORNER_THR, PLANAR_THR, CORNER_LEAF, PLANAR_LEAF = 1.0, 0.1, 0.2, 0.4
POS_TOL, ROT_TOL = 1e-4, 1e-4
CASES = cm.cases()


def _convert(msg, **kw):
    from funny_lidar_slam_b200.features import convert_message
    return convert_message(msg, **kw)


def _oracle(msg, **kw):
    from oracle_convert import pyoracle_convert as orcc
    return orcc.convert_message(msg, **kw)


def _torch_bytes(msg):
    import torch
    return torch.from_numpy(np.asarray(msg.data, np.uint8).copy()).to("cuda:0")


@gpu
@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_convert_bit_exact_vs_oracle(name):
    import torch
    from funny_lidar_slam_b200.features import PointCloud2
    _, msg, kw = next(c for c in CASES if c[0] == name)
    got, ref = _convert(msg, **kw), _oracle(msg, **kw)
    same(got, ref)
    st = got["stats"]
    cap = msg.width * msg.height
    if cap:
        assert st.n_source == cap and st.gpu_launches >= 4 and st.h2d_bytes == msg.height * msg.row_step
        assert st.d2h_bytes == cap * 24 + 4 + 48
    # device-resident message bytes and device outputs: the same records
    if cap:
        d_msg = _torch_bytes(msg)
        dm = PointCloud2(d_msg.data_ptr(), msg.fields, msg.width, msg.height, msg.point_step, msg.row_step, msg.is_dense, stamp_us=msg.stamp_us,
                         data_on_device=True)
        dx = torch.full((cap, 4), float("nan"), device="cuda:0")
        dr = torch.full((cap,), -1, dtype=torch.int32, device="cuda:0")
        dt = torch.full((cap,), float("nan"), device="cuda:0")
        torch.cuda.synchronize()
        g2 = _convert(dm, device_out=(dx.data_ptr(), dr.data_ptr(), dt.data_ptr()), host_out=False, **kw)
        assert g2["stats"].h2d_bytes == 0 and g2["stats"].d2h_bytes == 4 + 48
        k = g2["n"]
        same(dict(g2, xyzi=dx[:k].cpu().numpy(), ring=dr[:k].cpu().numpy(), time=dt[:k].cpu().numpy()), ref)


@gpu
@pytest.mark.parametrize("sensor", ["vlp16", "hdl64"])
@pytest.mark.parametrize("lidar_type", [FLS_LIDAR_VELODYNE, FLS_LIDAR_NONE])
def test_convert_clockwise_full_scans_carry_state(sensor, lidar_type):
    """Full scans with a real Velodyne's sense of rotation and more than one revolution per ring, no time field: most points carry
    time_last on (identity maps), many of them the +2 pi / omega of a ring that passed its first yaw again."""
    from oracle_convert import pyoracle_convert as orcc
    cw = cm.clockwise_scan(sensor)
    V = synth.SENSORS[sensor].lines
    if lidar_type == FLS_LIDAR_VELODYNE:
        dt = cm.dtype_of(FLS_LIDAR_VELODYNE, (["x", "y", "z", "intensity", "ring"], ["<f4"] * 4 + ["<u2"], [0, 4, 8, 16, 20], 24))
        kw = cm.convert_kwargs(FLS_LIDAR_VELODYNE, n_rows=V)
    else:
        dt = None
        kw = dict(cm.convert_kwargs(FLS_LIDAR_NONE, n_rows=V), lower_angle=cm.NONE_LOWER if V == 16 else float(np.float32(np.deg2rad(25.0))),
                  v_res=cm.NONE_VRES if V == 16 else float(np.float32(np.deg2rad(26.8 / 63))))
    msg = cm.message(cm.records(lidar_type, *cw, dtype=dt))
    got, ref = _convert(msg, **kw), _oracle(msg, **kw)
    same(got, ref)
    assert got["recomputed"] and got["n"] > 0.5 * len(cw[0])
    h = cm.offset_maps(ref["xyzi"], ref["ring"], V, orcc.atan2f(ref["xyzi"][:, 1], ref["xyzi"][:, 0]))
    assert h["identity"] > got["n"] // 2 and h["identity_carrying_1"] > 100, h


@gpu
@pytest.mark.parametrize("sensor", ["vlp16", "hdl64"])
@pytest.mark.parametrize("with_time", [True, False])
def test_convert_velodyne_full_scans(sensor, with_time):
    pts, ring, col, cols = cm.scan(sensor)
    dt = cm.dtype_of(FLS_LIDAR_VELODYNE) if with_time else cm.dtype_of(
        FLS_LIDAR_VELODYNE, (["x", "y", "z", "intensity", "ring"], ["<f4"] * 4 + ["<u2"], [0, 4, 8, 16, 20], 32))
    msg = cm.message(cm.records(FLS_LIDAR_VELODYNE, pts, ring, col, cols, dtype=dt))
    V = synth.SENSORS[sensor].lines
    kw = cm.convert_kwargs(FLS_LIDAR_VELODYNE, n_rows=V)
    got = _convert(msg, **kw)
    same(got, _oracle(msg, **kw))
    assert got["recomputed"] == (not with_time) and got["n"] == len(pts) and got["max_time"] > 0.09


@gpu
def test_big_endian_is_unsupported():
    from funny_lidar_slam_b200 import _lib
    from funny_lidar_slam_b200.features import PointCloud2
    _, msg, kw = CASES[0]
    be = PointCloud2(msg.data, msg.fields, msg.width, 1, msg.point_step, is_bigendian=True, stamp_us=1)
    with pytest.raises(_lib.FlsError) as e:
        _convert(be, **kw)
    assert e.value.status == FLS_ERR_UNSUPPORTED


# ---- device-input pre-processing entries -----------------------------------------------------------------------------------------
def _imu():
    from tests.test_oracle_deskew import make_case
    return make_case(n=1)[1]


def _converted_on_device(sensor, seed=7, pose_index=3, with_time=False):
    """A Velodyne message of the scan converted into device buffers; returns the host result too.  Without a time field the offsets are
    recomputed; the synthetic scanner turns the other way round, so nearly all of them land near the end of the sweep, beyond the
    test IMU buffer (85 ms): the de-skew cases use the time field."""
    import torch
    pts, ring, col, cols = cm.scan(sensor, pose_index=pose_index, seed=seed)
    dt = cm.dtype_of(FLS_LIDAR_VELODYNE) if with_time else cm.dtype_of(
        FLS_LIDAR_VELODYNE, (["x", "y", "z", "intensity", "ring"], ["<f4"] * 4 + ["<u2"], [0, 4, 8, 16, 20], 24))
    msg = cm.message(cm.records(FLS_LIDAR_VELODYNE, pts, ring, col, cols, dtype=dt))
    kw = cm.convert_kwargs(FLS_LIDAR_VELODYNE, n_rows=synth.SENSORS[sensor].lines)
    cap = len(pts)
    bufs = (torch.empty((cap, 4), device="cuda:0"), torch.empty(cap, dtype=torch.int32, device="cuda:0"), torch.empty(cap, device="cuda:0"))
    torch.cuda.synchronize()
    host = _convert(msg, device_out=tuple(b.data_ptr() for b in bufs), **kw)
    return msg, kw, host, bufs


def _shape(sensor):
    sn = synth.SENSORS[sensor]
    return sn.lines, sn.cols, float(np.float32(2 * np.pi / sn.cols))


@gpu
@pytest.mark.parametrize("sensor", ["vlp16", "hdl64"])
@pytest.mark.parametrize("with_imu", [False, True])
def test_preprocess_loam_device_equals_host_entry(sensor, with_imu):
    import torch
    from funny_lidar_slam_b200.features import LoamFrontEnd
    V, H, h_res = _shape(sensor)
    _, _, host, (dx, dr, dt) = _converted_on_device(sensor, with_time=with_imu)
    n = host["n"]
    imu = _imu() if with_imu else None
    fe = LoamFrontEnd(H, V, h_res, MIN_D, MAX_D, CORNER_THR, PLANAR_THR, CORNER_LEAF, PLANAR_LEAF)
    hc, hp = fe.run(host["xyzi"], host["ring"], host["time"], imu)
    h_st = fe.last_stats
    dc, dp = fe.run_device(dx.data_ptr(), dr.data_ptr(), dt.data_ptr(), n, imu)
    assert len(hc) > 50 and len(hp) > 500
    assert np.array_equal(dc, hc) and np.array_equal(dp, hp)
    st = fe.last_stats
    assert st.h2d_bytes == (h_st.h2d_bytes - n * (16 + 4 + (4 if with_imu else 0)))  # only the IMU samples go up
    # device outputs only
    oc = torch.full((120 * V, 4), float("nan"), device="cuda:0")
    op = torch.full((V * H, 4), float("nan"), device="cuda:0")
    torch.cuda.synchronize()
    assert fe.run_device(dx.data_ptr(), dr.data_ptr(), dt.data_ptr(), n, imu, device_out=(oc.data_ptr(), op.data_ptr()), host_out=False) == (None, None)
    assert fe.last_counts == (len(hc), len(hp))
    assert np.array_equal(oc[:len(hc)].cpu().numpy(), hc) and np.array_equal(op[:len(hp)].cpu().numpy(), hp)


@gpu
@pytest.mark.parametrize("sensor", ["vlp16", "hdl64"])
@pytest.mark.parametrize("with_imu", [False, True])
def test_preprocess_device_equals_host_entry(sensor, with_imu):
    import torch
    from funny_lidar_slam_b200.features import preprocess, preprocess_device
    _, _, host, (dx, _, dt) = _converted_on_device(sensor, with_time=with_imu)
    n = host["n"]
    imu = _imu() if with_imu else None
    raw = np.concatenate([host["xyzi"], host["time"][:, None]], 1)
    ho, hp = preprocess(raw, imu, MIN_D, MAX_D, 3, 0.5)
    do, dp = preprocess_device(dx.data_ptr(), dt.data_ptr(), n, imu, MIN_D, MAX_D, 3, 0.5)
    assert len(ho) > 1000 and len(hp) > 100
    assert np.array_equal(do, ho) and np.array_equal(dp, hp)
    go = torch.full((n, 4), float("nan"), device="cuda:0")
    gp = torch.full((n, 4), float("nan"), device="cuda:0")
    torch.cuda.synchronize()
    assert preprocess_device(dx.data_ptr(), dt.data_ptr(), n, imu, MIN_D, MAX_D, 3, 0.5, device_out=(go.data_ptr(), gp.data_ptr()),
                             host_out=False) == (None, None)
    assert preprocess_device.last_counts == (len(ho), len(hp))
    assert np.array_equal(go[:len(ho)].cpu().numpy(), ho) and np.array_equal(gp[:len(hp)].cpu().numpy(), hp)


# ---- message -> device Match ---------------------------------------------------------------------------------------------------
def _to_world(pts, T):
    out = pts.copy()
    out[:, :3] = (pts[:, :3].astype(np.float64) @ T[:3, :3].T + T[:3, 3]).astype(np.float32)
    return out


@gpu
def test_loam_full_stream_from_message():
    """Velodyne messages (no time field) -> fls_convert_cloud -> fls_preprocess_loam_device -> fls_match_cluster_device, all on the device,
    against the host chain on a second handle (identical) and the oracle chain (1e-4)."""
    import torch
    from funny_lidar_slam_b200.features import LoamFrontEnd
    from funny_lidar_slam_b200.registration import PointcloudCluster, Registration
    from oracle import pyoracle as orc
    V, H, h_res = _shape("vlp16")
    traj = synth.trajectory(16)
    cfg = default_config(FLS_LOAM_FULL, localization_mode=0, local_map_size=6, corner_local_map_size=4, dist_thre_add_cloud=0.5)
    dev, host, o = Registration(cfg), Registration(cfg), orc.Registration(cfg)
    fe = LoamFrontEnd(H, V, h_res, MIN_D, MAX_D, CORNER_THR, PLANAR_THR, CORNER_LEAF, PLANAR_LEAF)

    def oracle_front(conv):
        pr = orc.project_imu(conv["xyzi"], conv["ring"], conv["time"], None, V, H, h_res, MIN_D, MAX_D)
        ci, pi, _ = orc.extract_features(pr["depth"], pr["col"], pr["n"], pr["row_start"], pr["row_end"], CORNER_THR, PLANAR_THR)
        return orc.voxel_grid(pr["ordered"][ci], CORNER_LEAF), orc.voxel_grid(pr["ordered"][pi], PLANAR_LEAF)

    for k0 in (0, 2, 4, 6):
        msg, kw, conv, _ = _converted_on_device("vlp16", seed=300 + k0, pose_index=k0)
        c0, p0 = oracle_front(_oracle(msg, **kw))
        cw, pw = _to_world(c0, traj[k0]), _to_world(p0, traj[k0])
        dev.AddCloudToLocalMap([pw, cw])
        host.AddCloudToLocalMap([pw, cw])
        o.add_cloud(pw, cw)
    d_c = torch.empty((120 * V, 4), device="cuda:0")
    d_p = torch.empty((V * H, 4), device="cuda:0")
    for k in range(1, 8):
        msg, kw, conv, (dx, dr, dt) = _converted_on_device("vlp16", seed=300 + k, pose_index=k)
        fe.run_device(dx.data_ptr(), dr.data_ptr(), dt.data_ptr(), conv["n"], device_out=(d_c.data_ptr(), d_p.data_ptr()), host_out=False)
        nc, npl = fe.last_counts
        guess = synth.perturb_pose(traj[k], dpos=0.05, drot_deg=0.5, seed=k)
        Td = guess.copy()
        ok_d = dev.match_cluster_device(0, 0, d_p.data_ptr(), npl, d_c.data_ptr(), nc, Td)
        st_d = dev.last_stats
        hc, hp = fe.run(conv["xyzi"], conv["ring"], conv["time"])
        Th = guess.copy()
        ok_h = host.Match(PointcloudCluster(planar_cloud=hp, corner_cloud=hc), Th)
        st_h = host.last_stats
        assert ok_d == ok_h and np.array_equal(Td, Th), k
        assert (st_d.iterations, st_d.converged, st_d.n_valid) == (st_h.iterations, st_h.converged, st_h.n_valid), k
        oc, op = oracle_front(_oracle(msg, **kw))
        assert np.array_equal(oc, hc) and np.array_equal(op, hp), k
        ok_o, To, st_o = o.match(op, guess, corner=oc)
        assert ok_d == ok_o and st_d.iterations == st_o.iterations, k
        dtr, drr = synth.pose_error(Td, To)
        assert dtr < POS_TOL and drr < ROT_TOL, (k, dtr, drr)


@gpu
def test_loam_ivox_stream_from_message():
    """Velodyne messages (with a time field, de-skewed) -> fls_convert_cloud -> fls_preprocess_device -> fls_match_device over a stream of
    scans against a map of four key-frames, against the host chain (fls_preprocess + fls_match) on a second handle (identical) and the
    oracle chain (1e-4)."""
    import torch
    from funny_lidar_slam_b200.features import preprocess, preprocess_device
    from funny_lidar_slam_b200.registration import PointcloudCluster, Registration
    from oracle import pyoracle as orc
    traj = synth.trajectory(16)
    cfg = default_config(FLS_P2PLANE_IVOX)
    dev, host, o = Registration(cfg), Registration(cfg), orc.Registration(cfg)
    imu = _imu()
    JUMP, LEAF = 2, 0.4

    def oracle_front(msg, kw):
        ref = _oracle(msg, **kw)
        return orc.preprocess(np.concatenate([ref["xyzi"], ref["time"][:, None]], 1), imu, MIN_D, MAX_D, JUMP, LEAF)

    key = []
    for k0 in (0, 2, 4, 6):
        msg, kw, _, _ = _converted_on_device("vlp16", seed=400 + k0, pose_index=k0, with_time=True)
        key.append(_to_world(oracle_front(msg, kw)[1], traj[k0]))
    mp = np.concatenate(key)
    for reg in (dev, host):
        reg.AddCloudToLocalMap([mp])
    o.add_cloud(mp)
    for k in range(1, 8):
        msg, kw, conv, (dx, _, dt) = _converted_on_device("vlp16", seed=400 + k, pose_index=k, with_time=True)
        oo, op = oracle_front(msg, kw)
        n = conv["n"]
        d_pl = torch.empty((n, 4), device="cuda:0")
        torch.cuda.synchronize()
        preprocess_device(dx.data_ptr(), dt.data_ptr(), n, imu, MIN_D, MAX_D, JUMP, LEAF, device_out=(0, d_pl.data_ptr()), host_out=False)
        npl = preprocess_device.last_counts[1]
        ho, hp = preprocess(np.concatenate([conv["xyzi"], conv["time"][:, None]], 1), imu, MIN_D, MAX_D, JUMP, LEAF)
        assert np.array_equal(hp, op) and np.array_equal(ho, oo) and npl == len(hp), k
        guess = synth.perturb_pose(traj[k], dpos=0.05, drot_deg=0.5, seed=k)
        Td, Th = guess.copy(), guess.copy()
        ok_d = dev.match_device(d_pl.data_ptr(), npl, Td)
        st_d = dev.last_stats
        ok_h = host.Match(PointcloudCluster(planar_cloud=hp), Th)
        st_h = host.last_stats
        assert ok_d == ok_h and np.array_equal(Td, Th), k
        assert (st_d.iterations, st_d.converged, st_d.n_valid) == (st_h.iterations, st_h.converged, st_h.n_valid), k
        ok_o, To, st_o = o.match(op, guess)
        assert ok_d == ok_o and st_d.iterations == st_o.iterations, k
        dtr, drr = synth.pose_error(Td, To)
        assert dtr < POS_TOL and drr < ROT_TOL, (k, dtr, drr)
