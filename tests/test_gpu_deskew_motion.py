"""The five *_motion entries (de-skew with the sensor's translation, include/fls_b200.h; not upstream): bit-exact with the velocity-aware
oracle (oracle_motion/) on the edge scenes of tests/frontend_scenes.py, host and device routes; byte-equal to their parent entries
with a NULL or all-zero velocity; the fused LoamFull front end equal to its per-stage chain; a non-finite velocity refused before
anything is written (CPU); and a sensor moving at 15 m/s, whose de-skewed sweep lies on the surfaces it hit and matches closer to
the true pose than the rotation-only one."""
import ctypes as C

import numpy as np
import pytest

from funny_lidar_slam_b200 import features
from funny_lidar_slam_b200._abi import FLS_ERR_INVALID_ARG, FlsLoamFrontendCfg, FlsMatchStats
from oracle import pyoracle as orc
from oracle_motion import pyoracle_motion as orcm
from tests import deskew_motion_ref as mref
from tests import deskew_motion_scene as ms
from tests import frontend_scenes as fs
from tests.test_oracle_deskew_motion import SPEED, VELOCITIES, check_match, check_sweep
from tests.test_oracle_frontend_edges import same_bits

gpu = pytest.mark.gpu
NZ_DESKEW, NZ_PROJECT = ms.negative_zero_scenes()  # rotation-only outputs with -0.0 coordinates
DESKEW = fs.deskew_scenes() + [NZ_DESKEW]
PROJECT = fs.project_scenes() + [NZ_PROJECT]
MOVING = {k: VELOCITIES[k] for k in ("tiny", "30", "1e6")}
CT, PT, CL, PL = 0.5, 0.05, 0.3, 0.5  # LoamFull thresholds and leaves of the edge-scene chain


def _dev(a):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")
    torch.cuda.synchronize()
    return t


def _preprocess(s, route, velocity):
    a = (s["imu"], s["min_d"], s["max_d"], s["jump"], s["leaf"])
    if route == "host":
        return features.preprocess(s["raw"], *a, velocity=velocity)
    dx, dt = _dev(s["raw"][:, :4]), _dev(s["raw"][:, 4])
    return features.preprocess_device(dx.data_ptr(), dt.data_ptr(), len(s["raw"]), *a, velocity=velocity)


def _project(s, velocity):
    pr = features.PointcloudProjector(s["H"], s["V"], s["h_res"], s["min_d"], s["max_d"])
    return features.project_imu(pr, s["raw"], s["ring"], s["time"], s["imu"], velocity=velocity)


def _loam(s, route, velocity):
    fe = features.LoamFrontEnd(s["H"], s["V"], s["h_res"], s["min_d"], s["max_d"], CT, PT, CL, PL)
    if route == "host":
        return fe.run(s["raw"], s["ring"], s["time"], s["imu"], velocity=velocity)
    dx, dr, dt = _dev(s["raw"]), _dev(s["ring"]), _dev(s["time"])
    return fe.run_device(dx.data_ptr(), dr.data_ptr(), dt.data_ptr(), len(s["raw"]), s["imu"], velocity=velocity)


def _cell_product_overflows(planar_in, leaf):
    """PCL's cell-count product d_x d_y d_z does not fit in int64.  Both voxel filters (orc_cloud.h:81, fls_voxel.cuh:59) form it as a
    signed int64 product, so there its value is undefined behaviour and the two may take different branches (the near-zero-norm
    scene at 30 and 1e6 m/s, whose 2^39 us offsets put points 1e7 m and more apart).  The velocity cases are the only ones that reach
    it; the planar cloud is left out of the comparison there on purpose."""
    d = fs.ref.voxel_grid(planar_in, leaf)[1]["d"]
    return d is not None and d[0] * d[1] * d[2] >= 2 ** 63


def _skip_empty(s, route):
    if route == "device" and len(s["raw"]) == 0:
        pytest.skip("no device array of zero points")


@gpu
@pytest.mark.parametrize("v", MOVING.values(), ids=list(MOVING))
@pytest.mark.parametrize("route", ["host", "device"])
@pytest.mark.parametrize("s", DESKEW, ids=[s["name"] for s in DESKEW])
def test_preprocess_motion_vs_oracle(s, route, v):
    _skip_empty(s, route)
    g_ord, g_pl = _preprocess(s, route, v)
    o_ord, o_pl = orcm.preprocess(s["raw"], s["imu"], v, s["min_d"], s["max_d"], s["jump"], s["leaf"])
    assert same_bits(g_ord, o_ord)
    raw_index = mref.preprocess(s["raw"], s["imu"], v, s["min_d"], s["max_d"], s["jump"], s["leaf"])["raw_index"]
    if not _cell_product_overflows(o_ord[raw_index % s["jump"] == 0], s["leaf"]):
        assert same_bits(g_pl, o_pl)


@gpu
@pytest.mark.parametrize("v", MOVING.values(), ids=list(MOVING))
@pytest.mark.parametrize("s", PROJECT, ids=[s["name"] for s in PROJECT])
def test_project_and_loam_motion_vs_oracle(s, v):
    a = (s["V"], s["H"], s["h_res"], s["min_d"], s["max_d"])
    g = _project(s, v)
    o = orcm.project_imu(s["raw"], s["ring"], s["time"], s["imu"], v, *a)
    assert g["n"] == o["n"]
    for k in ("depth", "col", "row_start", "row_end"):
        assert np.array_equal(g[k], o[k]), k
    assert same_bits(g["ordered"], o["ordered"])
    oc, op = orcm.preprocess_loam(s["raw"], s["ring"], s["time"], s["imu"], v, *a, CT, PT, CL, PL)
    for route in ("host", "device"):
        gc, gp = _loam(s, route, v)
        assert same_bits(gc, oc) and same_bits(gp, op), route


# ---- NULL and all-zero velocity: the parent entry's bytes ----------------------------------------------------------------------------
@pytest.fixture(params=["null", "zero", "signed_zero"])
def motion_entries(request, monkeypatch):
    """Route every velocity-less call of funny_lidar_slam_b200.features through the _motion sibling with this velocity argument."""
    v = {"null": None, "zero": (C.c_double * 3)(0.0, 0.0, 0.0), "signed_zero": (C.c_double * 3)(-0.0, 0.0, -0.0)}[request.param]
    real = features._entry

    def entry(name, velocity):
        return getattr(features.lib(), name + "_motion"), (v,), name + "_motion"

    return lambda: monkeypatch.setattr(features, "_entry", entry), lambda: monkeypatch.setattr(features, "_entry", real)


def _bytes_equal(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_bytes_equal(a[k], b[k]) for k in a)
    if isinstance(a, tuple):
        return len(a) == len(b) and all(_bytes_equal(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray):
        return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()
    return a == b


@gpu
@pytest.mark.parametrize("route", ["host", "device"])
@pytest.mark.parametrize("s", DESKEW, ids=[s["name"] for s in DESKEW])
def test_preprocess_zero_velocity_is_the_parent(s, route, motion_entries):
    _skip_empty(s, route)
    on, off = motion_entries
    parent = _preprocess(s, route, None)
    on()
    sibling = _preprocess(s, route, None)
    off()
    assert _bytes_equal(sibling, parent)


@gpu
@pytest.mark.parametrize("s", PROJECT, ids=[s["name"] for s in PROJECT])
def test_project_and_loam_zero_velocity_is_the_parent(s, motion_entries):
    on, off = motion_entries
    parent = (_project(s, None), _loam(s, "host", None), _loam(s, "device", None))
    on()
    sibling = (_project(s, None), _loam(s, "host", None), _loam(s, "device", None))
    off()
    assert _bytes_equal(sibling, parent)


# ---- the fused LoamFull front end against its per-stage chain --------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("sensor", ["vlp16", "hdl64"])
def test_loam_motion_equals_per_stage_motion_chain(world, traj, sensor):
    from funny_lidar_slam_b200.registration import voxel_grid
    from tests.test_gpu_preprocess_loam import CORNER_LEAF, CORNER_THR, MAX_D, MIN_D, PLANAR_LEAF, PLANAR_THR, _front_end, _imu, _raw_scan, _shape
    V, H, h_res = _shape(sensor)
    raw, ring, time = _raw_scan(world, traj[6], sensor, 61)
    imu, v = _imu(), (12.0, -3.0, 0.25)
    gc, gp = _front_end(V, H, h_res).run(raw, ring, time, imu, velocity=v)
    pr = features.project_imu(features.PointcloudProjector(H, V, h_res, MIN_D, MAX_D), raw, ring, time, imu, velocity=v)
    ci, pi = features.FeatureExtractor(CORNER_THR, PLANAR_THR).extract_indices(pr["depth"], pr["col"], pr["n"], pr["row_start"], pr["row_end"])
    assert len(gc) > 100 and len(gp) > 1000
    assert np.array_equal(gc, voxel_grid(pr["ordered"][ci], CORNER_LEAF)) and np.array_equal(gp, voxel_grid(pr["ordered"][pi], PLANAR_LEAF))
    rc, rp = _front_end(V, H, h_res).run(raw, ring, time, imu)
    assert not (len(rc) == len(gc) and np.array_equal(rc, gc))  # the term changed the clouds


# ---- a non-finite velocity (no device needed) --------------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", [(np.nan, 0.0, 0.0), (0.0, np.inf, 0.0), (1.0, 2.0, -np.inf)], ids=["nan", "inf", "-inf"])
def test_non_finite_velocity_is_refused_and_writes_nothing(bad):
    L = features.lib()
    v = (C.c_double * 3)(*bad)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    raw5, imu = fs.deskew_scenes()[0]["raw"], fs.deskew_scenes()[0]["imu"]
    b, keep = features._imu_struct(imu)
    n = len(raw5)
    out = [np.full((n, 4), 7.0, np.float32) for _ in range(4)]
    cnt = [C.c_size_t(11), C.c_size_t(12)]
    rc = L.fls_preprocess_motion(0, vp(raw5), n, C.byref(b), 2.0, 60.0, 1, 0.5, vp(out[0]), C.byref(cnt[0]), vp(out[1]), C.byref(cnt[1]), v)
    assert rc == FLS_ERR_INVALID_ARG
    rc = L.fls_preprocess_device_motion(0, vp(raw5), vp(raw5), n, C.byref(b), 2.0, 60.0, 1, 0.5, vp(out[0]), None, C.byref(cnt[0]), vp(out[1]), None,
                                        C.byref(cnt[1]), v)
    assert rc == FLS_ERR_INVALID_ARG
    V, H = 4, 64
    ring = np.zeros(n, np.int32)
    time = np.ascontiguousarray(raw5[:, 4])
    xyzi = np.ascontiguousarray(raw5[:, :4])
    depth, col, rs, re = np.full(V * H, 7.0, np.float32), np.full(V * H, 7, np.int32), np.full(V, 7, np.int32), np.full(V, 7, np.int32)
    big = np.full((V * H, 4), 7.0, np.float32)
    rc = L.fls_project_imu_motion(0, vp(xyzi), vp(ring), vp(time), n, 16, C.byref(b), V, H, 0.1, 2.0, 60.0, vp(big), vp(depth), vp(col), vp(rs), vp(re),
                                  C.byref(cnt[0]), v)
    assert rc == FLS_ERR_INVALID_ARG
    cfg = FlsLoamFrontendCfg(0, V, H, 0.1, 2.0, 60.0, 1.0, 0.1, 0.2, 0.4)
    st = FlsMatchStats()
    st.n_source = 99
    for fn in (L.fls_preprocess_loam_motion, L.fls_preprocess_loam_device_motion):
        args = [C.byref(cfg), vp(xyzi), vp(ring), vp(time), n] + ([16] if fn is L.fls_preprocess_loam_motion else [])
        rc = fn(*args, C.byref(b), vp(out[2]), vp(out[3]), None, None, C.byref(cnt[0]), C.byref(cnt[1]), C.byref(st), v)
        assert rc == FLS_ERR_INVALID_ARG
    assert all(np.all(o == 7.0) for o in out) and np.all(big == 7.0) and np.all(depth == 7.0)
    assert np.all(col == 7) and np.all(rs == 7) and np.all(re == 7)
    assert (cnt[0].value, cnt[1].value, st.n_source) == (11, 12, 99)


# ---- a sensor moving at 15 m/s -----------------------------------------------------------------------------------------------------
@gpu
def test_moving_sensor_end_to_end(world, traj):
    from funny_lidar_slam_b200 import FLS_P2PLANE_IVOX, default_config, synth
    from funny_lidar_slam_b200.registration import PointcloudCluster, Registration
    from oracle import pyoracle as orc
    s = ms.moving_sweep(world, traj[3], speed=SPEED)
    a = (s["imu"], ms.MIN_D, ms.MAX_D, ms.JUMP, ms.LEAF)
    o_mot, p_mot = features.preprocess(s["raw"], *a, velocity=s["velocity"])
    o_rot, p_rot = features.preprocess(s["raw"], *a)
    r_ord, r_pl = orcm.preprocess(s["raw"], s["imu"], s["velocity"], *a[1:])
    assert same_bits(o_mot, r_ord) and same_bits(p_mot, r_pl)
    assert same_bits(o_rot, orc.preprocess(s["raw"], *a)[0])
    check_sweep(s, o_mot, o_rot)
    mp = ms.surface_map(world, traj[3])
    guess = synth.perturb_pose(traj[3], dpos=0.2, drot_deg=1.0, seed=5)
    errs = []
    for pl in (p_mot, p_rot):
        reg = Registration(default_config(FLS_P2PLANE_IVOX))
        reg.AddCloudToLocalMap([mp])
        T = guess.copy()
        assert reg.Match(PointcloudCluster(planar_cloud=pl), T)
        errs.append(synth.pose_error(T, traj[3]))
    check_match(*errs)
