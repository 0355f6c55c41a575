"""FLS_FLAG_INFORMATION: the information record of a Match at the pose it returned, for all five plug-ins.

  * without the flag nothing changes, and with it only what it adds: poses, converged flags, iterations, n_valid and sum_residual are
    the same bits as an unflagged handle's, launches grow by exactly two per call, d2h bytes by one record per scan, h2d bytes stay;
  * in mapping mode the map after a sequence of flagged Matches is the unflagged handle's, key for key and point for point;
  * the record is the system the plug-in's next Gauss-Newton iteration would build at T_final (a one-iteration Match started there,
    FLS_FLAG_ITER_LOG), mapped to the fusion parameterization [dθ; dp], R <- R·Exp(dθ), p <- p + dp;
  * a corridor without end wall leaves the position block singular along its axis, one with an end wall does not;
  * two flagged calls give the same record bits; valid = 0 before a Match, after an error and after relocalization; a scan index
    outside the last call is refused.
"""
import ctypes as C

import numpy as np
import pytest

from funny_lidar_slam_b200 import FLS_ICP_P2P, FLS_NDT, FLS_P2PLANE_IVOX, FLS_P2PLANE_KNN, default_config
from funny_lidar_slam_b200._abi import FLS_FLAG_INFORMATION, FLS_FLAG_ITER_LOG, FLS_LOAM_FULL, FlsInformation

pytestmark = pytest.mark.gpu
METHODS = {"ivox": FLS_P2PLANE_IVOX, "ndt": FLS_NDT, "icp": FLS_ICP_P2P, "kd": FLS_P2PLANE_KNN, "full": FLS_LOAM_FULL}
REC = C.sizeof(FlsInformation)


def _reg(method, flags=0, **kw):
    from funny_lidar_slam_b200.registration import Registration
    kw.setdefault("localization_mode", 1)
    return Registration(default_config(method, flags=flags, **kw))


def _add_map(g, method, mp):
    g.AddCloudToLocalMap([mp, mp[::3].copy()] if method == FLS_LOAM_FULL else [mp])


def _cluster(method, scan):
    from funny_lidar_slam_b200.registration import PointcloudCluster
    if method in (FLS_NDT, FLS_ICP_P2P):
        return PointcloudCluster(ordered_cloud=scan)
    return PointcloudCluster(planar_cloud=scan, corner_cloud=scan[::7].copy() if method == FLS_LOAM_FULL else None)


def _match(g, method, scan, guess):
    T = guess.copy()
    ok = g.Match(_cluster(method, scan), T)
    return ok, T, g.last_stats


def _same_result(a, b):
    (ok_a, T_a, st_a), (ok_b, T_b, st_b) = a, b
    assert ok_a == ok_b and np.array_equal(T_a, T_b)
    assert st_a.iterations == st_b.iterations and st_a.n_valid == st_b.n_valid and st_a.sum_residual == st_b.sum_residual


def _counts_add(st_plain, st_flag, n_scans):
    assert st_flag.gpu_launches == st_plain.gpu_launches + 2
    assert st_flag.h2d_bytes == st_plain.h2d_bytes
    assert st_flag.d2h_bytes == st_plain.d2h_bytes + n_scans * REC


def _A(method, R):
    """The plug-in's dx = A [dθ; dp] (fls_info.cu)."""
    A = np.eye(6)
    if method == FLS_ICP_P2P:
        A = np.zeros((6, 6))
        A[0:3, 3:6] = np.eye(3)
        A[3:6, 0:3] = np.eye(3)
    elif method != FLS_NDT:
        A[0:3, 0:3] = R
    return A


@pytest.mark.parametrize("name", list(METHODS))
def test_single_match_flag_adds_only_its_record(scene16, name):
    method = METHODS[name]
    plain, flag = _reg(method), _reg(method, FLS_FLAG_INFORMATION)
    for g in (plain, flag):
        _add_map(g, method, scene16["map"])
    assert flag.information() is None  # before any Match
    a = _match(plain, method, scene16["scan"], scene16["guess"])
    b = _match(flag, method, scene16["scan"], scene16["guess"])
    _same_result(a, b)
    _counts_add(a[2], b[2], 1)
    assert plain.information() is None
    rec = flag.information()
    assert rec is not None and rec["n_valid"] > 0
    assert np.array_equal(rec["H"], rec["H"].T) and np.all(np.linalg.eigvalsh(rec["H"]) > -1e-9 * np.abs(rec["H"]).max())
    # the same call again: the same record bits
    c = _match(flag, method, scene16["scan"], scene16["guess"])
    _same_result(b, c)
    rec2 = flag.information()
    assert np.array_equal(rec["H"], rec2["H"]) and np.array_equal(rec["g"], rec2["g"])
    assert rec["n_valid"] == rec2["n_valid"] and rec["sum_residual"] == rec2["sum_residual"]


@pytest.mark.parametrize("name", ["ivox", "ndt", "icp", "kd"])
@pytest.mark.parametrize("B", [4, 64])
def test_batch_flag_adds_only_its_records(scene16, name, B):
    import torch
    method = METHODS[name]
    from funny_lidar_slam_b200 import synth
    Ts = np.stack([synth.perturb_pose(scene16["truth"], seed=k, dpos=0.2, drot_deg=2.0) for k in range(B)])
    scans = [scene16["scan"][k % 5::2].copy() for k in range(B)]
    plain, flag = _reg(method), _reg(method, FLS_FLAG_INFORMATION)
    for g in (plain, flag):
        _add_map(g, method, scene16["map"])
    ca, Ta = plain.match_batch(scans, Ts)
    sa = plain.last_batch_stats
    cb, Tb = flag.match_batch(scans, Ts)
    sb = flag.last_batch_stats
    assert np.array_equal(np.asarray(ca), np.asarray(cb))
    if method == FLS_P2PLANE_IVOX:
        # the LOAM-iVox batch kernel hands chunks out dynamically, so its sums (and poses) vary in the last bits from run to run
        # with or without the flag
        assert np.abs(Ta - Tb).max() < 1e-9
    else:
        assert np.array_equal(Ta, Tb)
        for s in range(B):
            assert sa[s].n_valid == sb[s].n_valid and sa[s].sum_residual == sb[s].sum_residual
    for s in range(B):
        assert sa[s].iterations == sb[s].iterations
    _counts_add(sa[0], sb[0], B)
    recs = [flag.information(s) for s in range(B)]
    assert all(r is not None and r["n_valid"] > 0 for r in recs)
    with pytest.raises(Exception):
        flag.information(B)
    # the device entry and begin / end: the same records bit for bit
    d = [torch.from_numpy(np.ascontiguousarray(s[:, :4] if s.shape[1] == 4 else s)).cuda() for s in scans]
    exact = method != FLS_P2PLANE_IVOX

    def same(r, q):
        if exact:
            return np.array_equal(r["H"], q["H"]) and np.array_equal(r["g"], q["g"]) and r["n_valid"] == q["n_valid"]
        return np.abs(r["H"] - q["H"]).max() <= 1e-6 * np.abs(q["H"]).max() and abs(r["n_valid"] - q["n_valid"]) <= 2

    cd, Td = flag.match_batch_device([t.data_ptr() for t in d], [len(s) for s in scans], Ts)
    assert np.abs(Td - Tb).max() <= (0 if exact else 1e-9)
    for s in range(B):
        assert same(flag.information(s), recs[s])
    if method == FLS_P2PLANE_IVOX:  # the one plug-in with fls_match_batch_begin / _end
        flag.match_batch_begin(scans, Ts)
        assert flag.information() is None  # between begin and end
        ce, Te = flag.match_batch_end()
        assert np.abs(Te - Tb).max() <= (0 if exact else 1e-9)
        for s in range(B):
            assert same(flag.information(s), recs[s])


@pytest.mark.parametrize("name", list(METHODS))
def test_record_is_the_next_iteration_at_T_final(scene16, name):
    """A one-iteration Match started at T_final searches its correspondences afresh there: its logged H and g, mapped through A,
    are the record (up to the order of the fp64 sums)."""
    method = METHODS[name]
    flag = _reg(method, FLS_FLAG_INFORMATION)
    _add_map(flag, method, scene16["map"])
    _, T, _ = _match(flag, method, scene16["scan"], scene16["guess_small"])
    rec = flag.information()
    one = _reg(method, FLS_FLAG_ITER_LOG, max_iterations=1)
    _add_map(one, method, scene16["map"])
    _match(one, method, scene16["scan"], T)
    log = one.iter_log()[0]
    A = _A(method, T[:3, :3])
    H = A.T @ log["H"] @ A
    g = -A.T @ log["g"]
    assert np.abs(rec["H"] - H).max() <= 1e-9 * np.abs(H).max()
    assert np.abs(rec["g"] - g).max() <= 1e-9 * np.abs(g).max() + 1e-12 * max(1.0, np.abs(H).max())
    if method != FLS_LOAM_FULL:  # the loop counts LoamFull's planar terms only, the record both kinds
        assert rec["n_valid"] == log["n_valid"]
        assert abs(rec["sum_residual"] - log["sum_residual"]) <= 1e-9 * abs(log["sum_residual"])
    else:
        assert rec["n_valid"] >= log["n_valid"]


@pytest.mark.parametrize("name", list(METHODS))
def test_mapping_mode_map_is_unchanged(world, traj, name):
    from funny_lidar_slam_b200 import synth
    method = METHODS[name]
    kw = dict(localization_mode=0)
    plain, flag = _reg(method, **kw), _reg(method, FLS_FLAG_INFORMATION, **kw)
    first = synth.make_scan(world, traj[0], "vlp16", seed=0)["points"]
    for g in (plain, flag):
        g.AddCloudToLocalMap([synth.transform_points(first, traj[0])] * (2 if method == FLS_LOAM_FULL else 1))
    for k in range(1, 5):
        scan = synth.make_scan(world, traj[k], "vlp16", seed=k)["points"]
        guess = synth.perturb_pose(traj[k], dpos=0.05, drot_deg=0.5)
        a = _match(plain, method, scan, guess)
        b = _match(flag, method, scan, guess)
        _same_result(a, b)
        assert flag.information() is not None
        ia, ib = plain.map_info(), flag.map_info()
        assert (ia.n_points, ia.n_voxels, ia.table_slots, ia.incremental_inserts, ia.full_builds) == \
               (ib.n_points, ib.n_voxels, ib.table_slots, ib.incremental_inserts, ib.full_builds)
        if method in (FLS_P2PLANE_IVOX, FLS_NDT):
            ka, kb = plain.voxel_keys(), flag.voxel_keys()
            assert np.array_equal(ka[np.lexsort(ka.T)], kb[np.lexsort(kb.T)])
        try:  # every plug-in that exposes its map points (LOAM-iVox)
            pa = plain.map_points()
        except Exception:
            pa = None
        if pa is None:
            with pytest.raises(Exception):
                flag.map_points()
        else:
            assert np.array_equal(pa, flag.map_points())
        if method == FLS_NDT:
            va, vb = plain.ndt_voxels(), flag.ndt_voxels()
            oa, ob = np.lexsort(va["key"].T), np.lexsort(vb["key"].T)
            for f in va:
                assert np.array_equal(va[f][oa], vb[f][ob]), f


def _corridor(end_wall):
    s = 0.2
    xs = np.arange(-10.0, 10.0 + 1e-9, s)
    zs = np.arange(-1.3, 1.5 + 1e-9, s)
    ys = np.arange(-1.8, 1.8 + 1e-9, s)
    parts = []
    for y in (-2.0, 2.0):
        X, Z = np.meshgrid(xs, zs)
        parts.append(np.stack([X.ravel(), np.full(X.size, y), Z.ravel()], 1))
    X, Y = np.meshgrid(xs, ys)
    parts.append(np.stack([X.ravel(), Y.ravel(), np.full(X.size, -1.5)], 1))  # a LOAM plane n.p + 1 = 0 cannot pass through the origin
    if end_wall:
        Y, Z = np.meshgrid(ys, zs)
        parts.append(np.stack([np.full(Y.size, 10.0), Y.ravel(), Z.ravel()], 1))
    p = np.concatenate(parts).astype(np.float32)
    return np.concatenate([p, np.ones((len(p), 1), np.float32)], 1)


@pytest.mark.parametrize("end_wall", [False, True])
def test_corridor_degeneracy(end_wall):
    cloud = _corridor(end_wall)
    g = _reg(FLS_P2PLANE_IVOX, FLS_FLAG_INFORMATION)
    g.AddCloudToLocalMap([cloud])
    T = np.eye(4)
    g.Match(_cluster(FLS_P2PLANE_IVOX, cloud), T)
    rec = g.information()
    assert rec is not None and rec["n_valid"] > 100
    P = rec["H"][3:6, 3:6]
    w, V = np.linalg.eigh(P)
    if end_wall:
        assert w[0] >= 1e-3 * w[2], w
    else:
        assert w[0] < 1e-3 * w[2], w
        axis = V[:, 0] / np.linalg.norm(V[:, 0])
        assert np.degrees(np.arccos(min(1.0, abs(axis[0])))) < 2.0, axis


def test_no_record_after_error_or_relocalization(scene16):
    from funny_lidar_slam_b200.registration import reloc_cfg
    icp = _reg(FLS_ICP_P2P, FLS_FLAG_INFORMATION)
    icp.AddCloudToLocalMap([scene16["map"]])
    _match(icp, FLS_ICP_P2P, scene16["scan"], scene16["guess"])
    assert icp.information() is not None
    with pytest.raises(Exception):  # too few points: the call fails and leaves no record
        _match(icp, FLS_ICP_P2P, scene16["scan"][:5].copy(), scene16["guess"])
    assert icp.information() is None
    full = _reg(FLS_LOAM_FULL, FLS_FLAG_INFORMATION)
    _add_map(full, FLS_LOAM_FULL, scene16["map"])
    _match(full, FLS_LOAM_FULL, scene16["scan"], scene16["guess"])
    assert full.information() is not None
    T = scene16["guess"].copy()
    with pytest.raises(Exception):  # refused before any work (LoamFull reads two clouds): no record either
        full.match_device(0, 0, T)
    assert full.information() is None
    g = _reg(FLS_NDT, FLS_FLAG_INFORMATION)
    with pytest.raises(Exception):  # no map yet
        _match(g, FLS_NDT, scene16["scan"], scene16["guess"])
    assert g.information() is None
    g.AddCloudToLocalMap([scene16["map"]])
    _match(g, FLS_NDT, scene16["scan"], scene16["guess"])
    assert g.information() is not None
    with pytest.raises(Exception):
        g.information(1)
    with pytest.raises(Exception):
        g.information(-1)
    g.relocalize(scene16["scan"], scene16["guess"], cfg=reloc_cfg(xy_radius=1.0, xy_step=1.0, yaw_range=0.1, yaw_step=0.1))
    assert g.information() is None
    _match(g, FLS_NDT, scene16["scan"], scene16["guess"])
    assert g.information() is not None
