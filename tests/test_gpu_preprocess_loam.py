"""fls_preprocess_loam — PreProcessing::Run's LoamFull branch (projection with de-skew, features, two voxel filters) in one device
call — against the oracle chain and the per-stage GPU entries, bit for bit; fls_match_cluster_device, which matches its device
outputs; and the argument checks of both entries (CPU)."""
import ctypes as C

import numpy as np
import pytest

from funny_lidar_slam_b200 import default_config, synth
from funny_lidar_slam_b200._abi import (FLS_ERR_INVALID_ARG, FLS_ERR_NO_DEVICE, FLS_ERR_UNSUPPORTED, FLS_LOAM_FULL, FlsLoamFrontendCfg,
                                        FlsMatchStats)

gpu = pytest.mark.gpu
CORNER_THR, PLANAR_THR = 1.0, 0.1     # config_nclt_loam_full.yaml: corner_thres, planar_thres
CORNER_LEAF, PLANAR_LEAF = 0.2, 0.4   # corner_voxel_filter_size, planar_voxel_filter_size
MIN_D, MAX_D = 2.0, 80.0
POS_TOL, ROT_TOL = 1e-4, 1e-4


def _shape(sensor):
    sn = synth.SENSORS[sensor]
    return sn.lines, sn.cols, float(np.float32(2 * np.pi / sn.cols))


def _raw_scan(world, pose, sensor, seed):
    """Raw cloud in firing order (column-major over rings), time = col / n_cols * 0.1 s, and a second, slightly different return
    for every 7th point (the later duplicate must lose its cell)."""
    sc = synth.make_scan(world, pose, sensor, seed=seed)
    order = np.lexsort((sc["ring"], sc["col"]))
    pts, ring, col = sc["points"][order], sc["ring"][order].astype(np.int32), sc["col"][order]
    time = (col / synth.SENSORS[sensor].cols * 0.1).astype(np.float32)
    dup = pts[::7].copy()
    dup[:, :3] *= 1.0005
    return np.concatenate([pts, dup]), np.concatenate([ring, ring[::7]]), np.concatenate([time, time[::7]])


def _imu():
    """200 Hz orientation samples that end before the sweep does (points after 85 ms are refused)."""
    from tests.test_oracle_deskew import make_case
    return make_case(n=1)[1]


def _front_end(V, H, h_res, corner_leaf=CORNER_LEAF, planar_leaf=PLANAR_LEAF):
    from funny_lidar_slam_b200.features import LoamFrontEnd
    return LoamFrontEnd(H, V, h_res, MIN_D, MAX_D, CORNER_THR, PLANAR_THR, corner_leaf, planar_leaf)


def _oracle_chain(raw, ring, time, imu, V, H, h_res, corner_leaf=CORNER_LEAF, planar_leaf=PLANAR_LEAF):
    """The same branch on the CPU oracle: project_imu -> extract_features -> gather -> voxel_grid x 2."""
    from oracle import pyoracle as orc
    pr = orc.project_imu(raw, ring, time, imu, V, H, h_res, MIN_D, MAX_D)
    ci, pi, _ = orc.extract_features(pr["depth"], pr["col"], pr["n"], pr["row_start"], pr["row_end"], CORNER_THR, PLANAR_THR)
    return orc.voxel_grid(pr["ordered"][ci], corner_leaf), orc.voxel_grid(pr["ordered"][pi], planar_leaf)


def _gpu_chain(raw, ring, time, imu, V, H, h_res):
    """The five-call chain the fused entry replaces: fls_project_imu -> fls_extract_features -> host gather -> fls_voxel_grid x 2."""
    from funny_lidar_slam_b200.features import FeatureExtractor, PointcloudProjector, project_imu
    from funny_lidar_slam_b200.registration import voxel_grid
    pr = project_imu(PointcloudProjector(H, V, h_res, MIN_D, MAX_D), raw, ring, time, imu)
    ci, pi = FeatureExtractor(CORNER_THR, PLANAR_THR).extract_indices(pr["depth"], pr["col"], pr["n"], pr["row_start"], pr["row_end"])
    return voxel_grid(pr["ordered"][ci], CORNER_LEAF), voxel_grid(pr["ordered"][pi], PLANAR_LEAF)


def _layout(raw, layout):
    from tests.conftest import to_pcl
    return to_pcl(raw) if layout == "pcl" else raw


CASES = [(s, i, l) for s in ("vlp16", "hdl64") for i in (False, True) for l in ("packed", "pcl")]


@gpu
@pytest.mark.parametrize("sensor,with_imu,layout", CASES)
def test_bit_exact_vs_oracle_chain(world, traj, sensor, with_imu, layout):
    V, H, h_res = _shape(sensor)
    raw, ring, time = _raw_scan(world, traj[3], sensor, 31)
    imu = _imu() if with_imu else None
    fe = _front_end(V, H, h_res)
    gc, gp = fe.run(_layout(raw, layout), ring, time, imu)
    oc, op = _oracle_chain(raw, ring, time, imu, V, H, h_res)
    assert len(gc) > 100 and len(gp) > 1000, (len(gc), len(gp))
    assert np.array_equal(gc, oc), (len(gc), len(oc))
    assert np.array_equal(gp, op), (len(gp), len(op))
    st = fe.last_stats
    assert st.n_source == len(raw) and st.gpu_launches > 0 and st.gpu_ms > 0
    # point data goes up once and only the two clouds (+ sizes) come back
    assert st.h2d_bytes >= raw.nbytes if layout == "packed" else st.h2d_bytes >= 2 * raw.nbytes
    assert st.d2h_bytes == 16 * (len(gc) + len(gp)) + 4 * (2 * V + 1) + 8


@gpu
@pytest.mark.parametrize("sensor,with_imu,layout", CASES)
def test_bit_exact_vs_per_stage_gpu_chain(world, traj, sensor, with_imu, layout):
    V, H, h_res = _shape(sensor)
    raw, ring, time = _raw_scan(world, traj[6], sensor, 61)
    imu = _imu() if with_imu else None
    gc, gp = _front_end(V, H, h_res).run(_layout(raw, layout), ring, time, imu)
    sc, sp = _gpu_chain(_layout(raw, layout), ring, time, imu, V, H, h_res)
    assert len(gc) > 100 and len(gp) > 1000
    assert np.array_equal(gc, sc) and np.array_equal(gp, sp)


@gpu
@pytest.mark.parametrize("sensor", ["vlp16", "hdl64"])
def test_device_outputs_equal_host_outputs(world, traj, sensor):
    import torch
    V, H, h_res = _shape(sensor)
    raw, ring, time = _raw_scan(world, traj[5], sensor, 51)
    imu = _imu()
    d_c = torch.full((120 * V, 4), float("nan"), dtype=torch.float32, device="cuda:0")
    d_p = torch.full((V * H, 4), float("nan"), dtype=torch.float32, device="cuda:0")
    torch.cuda.synchronize()
    fe = _front_end(V, H, h_res)
    gc, gp = fe.run(raw, ring, time, imu, device_out=(d_c.data_ptr(), d_p.data_ptr()))
    assert fe.last_counts == (len(gc), len(gp)) and len(gc) > 100
    assert np.array_equal(d_c[:len(gc)].cpu().numpy(), gc) and np.array_equal(d_p[:len(gp)].cpu().numpy(), gp)
    # device pair only: same counts, same records, nothing read back but the sizes
    d_c.fill_(float("nan"))
    d_p.fill_(float("nan"))
    torch.cuda.synchronize()
    assert fe.run(raw, ring, time, imu, device_out=(d_c.data_ptr(), d_p.data_ptr()), host_out=False) == (None, None)
    assert fe.last_counts == (len(gc), len(gp))
    assert fe.last_stats.d2h_bytes == 4 * (2 * V + 1) + 8
    assert np.array_equal(d_c[:len(gc)].cpu().numpy(), gc) and np.array_equal(d_p[:len(gp)].cpu().numpy(), gp)
    # one cloud on the device, the other on the host
    d_c.fill_(float("nan"))
    torch.cuda.synchronize()
    from funny_lidar_slam_b200.features import preprocess_loam
    hc, hp = preprocess_loam(raw, ring, time, imu, H, V, h_res, MIN_D, MAX_D, CORNER_THR, PLANAR_THR, CORNER_LEAF, PLANAR_LEAF,
                             device_out=(d_c.data_ptr(), 0))
    assert np.array_equal(hc, gc) and np.array_equal(hp, gp) and np.array_equal(d_c[:len(gc)].cpu().numpy(), gc)


@gpu
def test_edges(world, traj):
    V, H, h_res = _shape("vlp16")
    fe = _front_end(V, H, h_res)
    raw, ring, time = _raw_scan(world, traj[2], "vlp16", 21)
    e4, ei, ef = np.zeros((0, 4), np.float32), np.zeros(0, np.int32), np.zeros(0, np.float32)
    # empty scan, with and without an IMU buffer
    for imu in (None, _imu()):
        c, p = fe.run(e4, ei, ef, imu)
        assert len(c) == 0 and len(p) == 0
    # every point beyond max_distance
    far = raw.copy()
    far[:, :3] *= 1000.0
    c, p = fe.run(far, ring, time)
    assert len(c) == 0 and len(p) == 0
    # reference time after the last IMU sample: SetRefTime fails, no point is accepted
    imu = _imu()
    late = dict(imu, ref_time_us=int(imu["t_us"][-1]) + 10)
    c, p = fe.run(raw, ring, time, late)
    assert len(c) == 0 and len(p) == 0 and fe.last_counts == (0, 0)
    # fewer than 12 ordered points: no features
    for k in (11, 12, 40):
        sub = slice(0, 3 * k, 3)
        c, p = fe.run(raw[sub], ring[sub], time[sub])
        oc, op = _oracle_chain(raw[sub], ring[sub], time[sub], None, V, H, h_res)
        assert np.array_equal(c, oc) and np.array_equal(p, op)
        if k == 11:
            assert len(c) == 0 and len(p) == 0
    # a leaf so small that dx*dy*dz exceeds INT_MAX: PCL returns the input unchanged
    tiny = _front_end(V, H, h_res, corner_leaf=1e-4)
    c, p = tiny.run(raw, ring, time)
    oc, op = _oracle_chain(raw, ring, time, None, V, H, h_res, corner_leaf=1e-4)
    assert np.array_equal(c, oc) and np.array_equal(p, op)
    from oracle import pyoracle as orc
    pr = orc.project_imu(raw, ring, time, None, V, H, h_res, MIN_D, MAX_D)
    ci, _, _ = orc.extract_features(pr["depth"], pr["col"], pr["n"], pr["row_start"], pr["row_end"], CORNER_THR, PLANAR_THR)
    assert np.array_equal(c, pr["ordered"][ci])  # pass-through: the gathered corners themselves


def _long_ring_scan(H=150000, seed=4):
    """One ring with ~130 k occupied columns: beyond the feature kernels' shared-memory working set."""
    rng = np.random.default_rng(seed)
    n = 2 * H
    a = rng.uniform(-np.pi, np.pi, n)
    raw = np.zeros((n, 4), np.float32)
    raw[:, 0], raw[:, 1], raw[:, 2] = 10 * np.cos(a), 10 * np.sin(a), rng.normal(0, 0.1, n)
    return raw, np.zeros(n, np.int32), np.zeros(n, np.float32), 1, H, float(np.float32(2 * np.pi / H))


@gpu
def test_over_long_ring_is_unsupported_and_writes_nothing():
    from funny_lidar_slam_b200 import _lib
    from funny_lidar_slam_b200.features import FeatureExtractor, PointcloudProjector
    raw, ring, time, V, H, h_res = _long_ring_scan()
    # the per-stage extractor refuses the same ring
    pr = PointcloudProjector(H, V, h_res, MIN_D, MAX_D).project_arrays(raw, ring)
    assert pr["n"] > 100000
    with pytest.raises(_lib.FlsError) as e:
        FeatureExtractor(CORNER_THR, PLANAR_THR).extract_indices(pr["depth"], pr["col"], pr["n"], pr["row_start"], pr["row_end"])
    assert e.value.status == FLS_ERR_UNSUPPORTED
    cfg = FlsLoamFrontendCfg(0, V, H, h_res, MIN_D, MAX_D, CORNER_THR, PLANAR_THR, CORNER_LEAF, PLANAR_LEAF)
    corner = np.full((120 * V, 4), 5.0, np.float32)
    planar = np.full((V * H, 4), 5.0, np.float32)
    nc, npl = C.c_size_t(7), C.c_size_t(7)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = _lib.lib().fls_preprocess_loam(C.byref(cfg), vp(raw), vp(ring), vp(time), len(raw), 16, None, vp(corner), vp(planar), None, None,
                                        C.byref(nc), C.byref(npl), None)
    assert rc == FLS_ERR_UNSUPPORTED and nc.value == 0 and npl.value == 0
    assert np.all(corner == 5.0) and np.all(planar == 5.0)


def _to_world(pts, T):
    out = pts.copy()
    out[:, :3] = (pts[:, :3].astype(np.float64) @ T[:3, :3].T + T[:3, 3]).astype(np.float32)
    return out


@gpu
def test_loam_full_mapping_stream_from_device_front_end(world, traj):
    """Raw scan -> fls_preprocess_loam into device buffers -> fls_match_cluster_device, for nine scans of a LoamFull mapping stream
    (windows of 6 planar / 4 corner clouds, filtered from the 6th cloud on).  A second handle matching the same clouds through host
    fls_match gives identical results; the oracle chain + oracle matcher agrees to 1e-4."""
    import torch
    from funny_lidar_slam_b200.registration import PointcloudCluster, Registration
    from oracle import pyoracle as orc
    V, H, h_res = _shape("vlp16")
    cfg = default_config(FLS_LOAM_FULL, localization_mode=0, local_map_size=6, corner_local_map_size=4, dist_thre_add_cloud=0.5)
    dev, host, o = Registration(cfg), Registration(cfg), orc.Registration(cfg)
    fe = _front_end(V, H, h_res)
    for k0 in (0, 2, 4, 6):  # a well-conditioned start: four surrounding key-frames
        raw, ring, time = _raw_scan(world, traj[k0], "vlp16", 300 + k0)
        c0, p0 = fe.run(raw, ring, time)
        cw, pw = _to_world(c0, traj[k0]), _to_world(p0, traj[k0])
        dev.AddCloudToLocalMap([pw, cw])
        host.AddCloudToLocalMap([pw, cw])
        o.add_cloud(pw, cw)
    d_c = torch.empty((120 * V, 4), dtype=torch.float32, device="cuda:0")
    d_p = torch.empty((V * H, 4), dtype=torch.float32, device="cuda:0")
    torch.cuda.synchronize()
    sizes = []
    for k in range(1, 10):
        raw, ring, time = _raw_scan(world, traj[k], "vlp16", 300 + k)
        fe.run(raw, ring, time, device_out=(d_c.data_ptr(), d_p.data_ptr()), host_out=False)
        nc, npl = fe.last_counts
        guess = synth.perturb_pose(traj[k], dpos=0.05, drot_deg=0.5, seed=k)
        Td = guess.copy()
        ok_d = dev.match_cluster_device(0, 0, d_p.data_ptr(), npl, d_c.data_ptr(), nc, Td)
        st_d = dev.last_stats
        hc, hp = d_c[:nc].cpu().numpy(), d_p[:npl].cpu().numpy()
        Th = guess.copy()
        ok_h = host.Match(PointcloudCluster(planar_cloud=hp, corner_cloud=hc), Th)
        st_h = host.last_stats
        assert ok_d == ok_h and np.array_equal(Td, Th), k
        assert (st_d.iterations, st_d.converged, st_d.n_valid, st_d.n_source) == (st_h.iterations, st_h.converged, st_h.n_valid, st_h.n_source), k
        assert st_d.h2d_bytes < st_h.h2d_bytes
        assert dev.map_info().n_points == host.map_info().n_points, k
        oc, op = _oracle_chain(raw, ring, time, None, V, H, h_res)
        assert np.array_equal(oc, hc) and np.array_equal(op, hp), k
        ok_o, To, st_o = o.match(op, guess, corner=oc)
        assert ok_d == ok_o and st_d.iterations == st_o.iterations, k
        dt, dr = synth.pose_error(Td, To)
        assert dt < POS_TOL and dr < ROT_TOL, (k, dt, dr)
        sizes.append(o.map_points)
    assert max(sizes) > min(sizes)


# ---- argument checks (no device needed) ------------------------------------------------------------------------------------
def test_preprocess_loam_argument_checks():
    from funny_lidar_slam_b200._lib import lib
    L = lib()
    raw = np.zeros((4, 4), np.float32)
    ring = np.zeros(4, np.int32)
    time = np.zeros(4, np.float32)
    out = np.zeros((16 * 120, 4), np.float32)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    nc, npl = C.c_size_t(3), C.c_size_t(3)
    good = lambda **kw: FlsLoamFrontendCfg(*[kw.get(k, v) for k, v in (("device", 0), ("n_rows", 16), ("n_cols", 1800), ("h", 0.0035),
                                                                         ("min_d", 2.0), ("max_d", 80.0), ("ct", 1.0), ("pt", 0.1),
                                                                         ("cl", 0.2), ("pl", 0.4))])

    def call(cfg, stride=16, outs=(out, out, None, None), counts=True, r=raw):
        ptr = lambda a: vp(a) if a is not None else None
        return L.fls_preprocess_loam(C.byref(cfg) if cfg is not None else None, vp(r), vp(ring), vp(time), len(r), stride, None,
                                     *[ptr(a) for a in outs], C.byref(nc) if counts else None, C.byref(npl) if counts else None, None)

    assert call(None) == FLS_ERR_INVALID_ARG
    assert call(good(cl=0.0)) == FLS_ERR_INVALID_ARG
    assert call(good(pl=-1.0)) == FLS_ERR_INVALID_ARG
    assert call(good(n_rows=0)) == FLS_ERR_INVALID_ARG
    assert call(good(h=0.0)) == FLS_ERR_INVALID_ARG
    assert call(good(ct=float("inf"))) == FLS_ERR_INVALID_ARG  # FloatNaN sentinel upstream
    assert call(good(), counts=False) == FLS_ERR_INVALID_ARG
    assert call(good(), outs=(None, None, None, None)) == FLS_ERR_INVALID_ARG
    assert call(good(), stride=12) == FLS_ERR_INVALID_ARG
    assert (nc.value, npl.value) == (0, 0)  # counts are cleared once they can be written
    if L.fls_device_count() < 1:
        assert call(good()) == FLS_ERR_NO_DEVICE
        from tests.conftest import to_pcl
        assert call(good(), stride=32, r=to_pcl(raw)) == FLS_ERR_NO_DEVICE


def test_match_cluster_device_argument_checks():
    from funny_lidar_slam_b200._lib import lib
    T = np.eye(4)
    assert lib().fls_match_cluster_device(None, None, 0, None, 0, None, 0, T.ctypes.data_as(C.c_void_p), None, None) == FLS_ERR_INVALID_ARG


def test_frontend_cfg_layout_matches_header(tmp_path):
    """The ctypes mirror of fls_loam_frontend_cfg has gcc's layout of the C struct."""
    import os
    import shutil
    import subprocess
    gcc = shutil.which("gcc")
    if gcc is None:
        return
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "cfg.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "fls_b200.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu\\n", sizeof(fls_loam_frontend_cfg), offsetof(fls_loam_frontend_cfg, planar_leaf), '
                   'offsetof(fls_loam_frontend_cfg, reserved));\n  return 0;\n}\n')
    exe = tmp_path / "cfg"
    subprocess.check_call([gcc, "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(FlsLoamFrontendCfg), FlsLoamFrontendCfg.planar_leaf.offset, FlsLoamFrontendCfg.reserved.offset]
    assert C.sizeof(FlsMatchStats) == 72
