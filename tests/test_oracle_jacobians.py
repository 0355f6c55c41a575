"""Oracle pinning (CPU), part 3: checks that share no code with the oracle.

  * ICP and NDT: the accumulated gradient of one point equals minus half the finite-difference gradient of the cost
    it linearises, under the RIGHT perturbation each plug-in applies (icp_optimized.h:135-136, incremental_ndt.h:311-313);
  * LOAM-iVox: one PlanerMatch + SumCoefficient pass restated with numpy on the brute-force k-NN of tests/ivox_ref.py;
  * LOAM-iVox mapping mode: the cached-5-NN insertion rule (loam_point_to_plane_ivox.h:79-128) restated with numpy."""
import numpy as np
import pytest

from funny_lidar_slam_b200 import FLS_ICP_P2P, FLS_NDT, FLS_P2PLANE_IVOX, default_config, synth
from funny_lidar_slam_b200._abi import FLS_FLAG_ITER_LOG
from oracle import pyoracle as orc
from tests import ivox_ref


def _hat(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])


def _exp(w):
    th = np.linalg.norm(w)
    if th == 0:
        return np.eye(3)
    K = _hat(w / th)
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def _fd(f, n=6, eps=1e-6):
    g = np.zeros(n)
    for k in range(n):
        d = np.zeros(n)
        d[k] = eps
        g[k] = (f(d) - f(-d)) / (2 * eps)
    return g


def test_icp_gradient_is_half_the_derivative_of_the_squared_error():
    """IcpOptimized: dx = [dt, dtheta], t += dt, R <- R Exp(dtheta); B = -sum J^T e with J = [I | -R p^] (:97-103)."""
    rng = np.random.default_rng(1)
    mp = np.zeros((40, 4), np.float32)
    mp[:, :3] = rng.uniform(-1, 1, (40, 3)) * 30.0
    mp[0, :3] = (5.0, 1.0, 0.5)
    T = synth.perturb_pose(np.eye(4), dpos=0.4, drot_deg=25.0, seed=6)
    pw = np.array([5.1, 1.05, 0.45])  # lands 0.12 m from map point 0, far from everything else
    ps = (T[:3, :3].T @ (pw - T[:3, 3])).astype(np.float32)
    src = np.tile(np.array([[ps[0], ps[1], ps[2], 0.0]], np.float32), (11, 1))  # CHECK_GT(size, 10u); identical points filter to one
    cfg = default_config(FLS_ICP_P2P, flags=FLS_FLAG_ITER_LOG, max_iterations=1, map_cloud_filter_size=0.05, source_cloud_filter_size=0.05)
    r = orc.Registration(cfg)
    r.add_cloud(mp)
    r.match(src, T)
    lg = r.iter_log()[0]
    assert lg["n_valid"] == 1
    m = orc.voxel_grid(mp, 0.05)[:, :3].astype(np.float64)
    m0 = m[np.argmin(np.linalg.norm(m - pw, axis=1))]
    Rf, tf = T[:3, :3].astype(np.float32), T[:3, 3].astype(np.float32)  # the transform is evaluated in fp32 (:64)
    p64 = ps.astype(np.float64)

    def half_sq(d):
        R = T[:3, :3] @ _exp(d[3:])
        t = T[:3, 3] + d[:3]
        e = R @ p64 + t - m0
        return 0.5 * e @ e

    # g = -grad(0.5 |e|^2); the fp32 evaluation of q moves e by ~1e-6, hence the tolerance
    assert np.allclose(lg["g"], -_fd(half_sq), atol=2e-5)
    e0 = (Rf @ ps + tf).astype(np.float64) - m0
    assert lg["sum_residual"] == pytest.approx(np.linalg.norm(e0), rel=2e-5)  # fp32 transform of a voxel-filtered (fp32 centroid) point
    J = np.hstack([np.eye(3), -T[:3, :3] @ _hat(p64)])
    assert np.allclose(lg["H"], J.T @ J, atol=1e-9)


def test_ndt_gradient_is_half_the_derivative_of_the_mahalanobis_cost():
    """IncrementalNDT: dx = [dtheta, dt], R <- R Exp(dtheta), t += dt; err = -sum J^T Lambda e over the hit voxels
    (incremental_ndt.h:273-304) = -1/2 grad sum e^T Lambda e."""
    rng = np.random.default_rng(3)
    cfg = default_config(FLS_NDT, flags=FLS_FLAG_ITER_LOG, max_iterations=1, ndt_min_effective_pts=1, source_cloud_filter_size=0.05,
                         ndt_outlier_thres=60.0)
    # a few voxels around (10, 4, 1): the source point sees its own voxel and up to 6 neighbours
    cl = []
    for c in ((10.5, 4.5, 1.5), (11.5, 4.5, 1.5), (10.5, 5.5, 1.5), (10.5, 4.5, 0.5)):
        cl.append(np.array(c) + np.clip(rng.normal(0, 0.25, (30, 3)), -0.45, 0.45) * (1.0, 1.0, 0.5))
    mp = np.zeros((120, 4), np.float32)
    mp[:, :3] = np.concatenate(cl)
    r = orc.Registration(cfg)
    r.add_cloud(mp)
    keys, mu, info, est = r.ndt_dump()
    T = synth.perturb_pose(np.eye(4), dpos=0.3, drot_deg=10.0, seed=8)
    pw = np.array([10.6, 4.6, 1.4])
    ps = (T[:3, :3].T @ (pw - T[:3, 3])).astype(np.float32)
    src = np.array([[ps[0], ps[1], ps[2], 0.0]], np.float32)
    r.match(src, T)
    lg = r.iter_log()[0]
    p64 = ps.astype(np.float64)
    q0 = T[:3, :3] @ p64 + T[:3, 3]
    k0 = (q0 / cfg.ndt_voxel_size).astype(np.int32)  # C truncation
    stencil = [(0, 0, 0), (-1, 0, 0), (1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, -1), (0, 0, 1)]
    hits = []
    for o in stencil:
        sel = np.where(np.all(keys == k0 + np.array(o), axis=1))[0]
        if len(sel) and est[sel[0]]:
            e = q0 - mu[sel[0]]
            if e @ info[sel[0]] @ e <= cfg.ndt_outlier_thres:
                hits.append(sel[0])
    assert lg["n_valid"] == len(hits) >= 2

    def half_cost(d):
        R = T[:3, :3] @ _exp(d[:3])
        t = T[:3, 3] + d[3:]
        q = R @ p64 + t
        return 0.5 * sum((q - mu[h]) @ info[h] @ (q - mu[h]) for h in hits)

    assert np.allclose(lg["g"], -_fd(half_cost), rtol=1e-5, atol=1e-6)
    J = np.hstack([-T[:3, :3] @ _hat(p64), np.eye(3)])
    H = sum(J.T @ info[h] @ J for h in hits)
    assert np.allclose(lg["H"], H, rtol=1e-9, atol=1e-9 * np.abs(H).max())


def _knn5_points(mp, q):
    """The 5 nearest map points of every query (IVoxMap::GetClosestPoint at the default NEARBY18, 0.5 m, 5 m), fp64 rows."""
    r = ivox_ref.knn5(mp, q, 0.5, 2, 5.0)
    return [mp[r.idx[i, :r.found[i]], :3].astype(np.float64) for i in range(len(q))]


def test_ivox_first_iteration_against_numpy(scene16):
    cfg = default_config(FLS_P2PLANE_IVOX, flags=FLS_FLAG_ITER_LOG, max_iterations=1)
    r = orc.Registration(cfg)
    mp = scene16["map"]
    r.add_cloud(mp)
    src = scene16["scan"][::40]
    T = scene16["guess_small"]
    r.match(src, T)
    lg = r.iter_log()[0]
    R, t = T[:3, :3], T[:3, 3]
    H, g, nv = np.zeros((6, 6)), np.zeros(6), 0
    qs = ivox_ref.transform(src, T)  # fp64 rows rounded to fp32, as transform_point_d
    for sp, q, A in zip(src, qs, _knn5_points(mp, qs)):
        ps = sp[:3].astype(np.float64)
        if len(A) < 5:
            continue
        c = np.linalg.lstsq(A, -np.ones(5), rcond=None)[0]
        cn = np.linalg.norm(c)
        if np.any(np.abs(A @ c + 1.0) / cn > cfg.point_to_planar_thres):
            continue
        n = c / cn
        d = (q.astype(np.float64) - A[0]) @ n
        if np.linalg.norm(ps) < 81 * d * d:
            continue
        s = 1.0 if d > 0 else -1.0
        J = np.concatenate([np.cross(R @ ps, n) * s, n * s])
        H += np.outer(J, J)
        g += -J * abs(d)
        nv += 1
    assert nv == lg["n_valid"] and nv > 100
    assert np.allclose(H, lg["H"], rtol=1e-9, atol=1e-9 * np.abs(H).max())
    assert np.allclose(g, lg["g"], rtol=1e-9, atol=1e-9)


def test_ivox_mapping_mode_insertion_rule_against_numpy(world, traj):
    """After a successful Match in mapping mode the scan enters the map through the rule of :79-128; the number of points
    the oracle adds must be what a numpy restatement of the rule selects."""
    cfg = default_config(FLS_P2PLANE_IVOX, localization_mode=0, max_iterations=1)
    first = synth.make_map_from_scans(world, traj[0:5:2], "vlp16", leaf=0.3)
    scan = synth.voxel_downsample_np(synth.make_scan(world, traj[1], "vlp16", seed=41)["points"], 0.6)
    guess = synth.perturb_pose(traj[1], dpos=0.03, drot_deg=0.3, seed=1)
    r = orc.Registration(cfg)
    r.add_cloud(first)
    n0 = r.map_points
    ok, Tf, _ = r.match(scan, guess)
    assert ok
    added = r.map_points - n0
    # the single PlanerMatch ran at the guess: its 5-NN are the cached ones
    Rf, tf = Tf[:3, :3], Tf[:3, 3]
    expect = 0
    for sp, near in zip(scan, _knn5_points(first, ivox_ref.transform(scan, guess))):
        ps = sp[:3].astype(np.float64)
        pw = (Rf @ ps + tf).astype(np.float32).astype(np.float64)
        if len(near) == 0:
            expect += 1
            continue
        c = (np.floor(pw / 0.5) + 0.5) * 0.5
        if np.all(np.abs(near[0] - c) > 0.25):
            expect += 1
            continue
        dist = np.sum((pw - c) ** 2)
        need = True
        if len(near) >= 5 and np.any(np.sum((near - c) ** 2, axis=1) < dist + 1e-6):
            need = False
        expect += int(need)
    assert 0 < added < len(scan)
    assert added == expect


def test_ndt_incremental_voxel_updates_against_python_restatement(world, traj):
    """IncrementalNDT::AddCloudToLocalMap + UpdateVoxel in mapping mode (incremental_ndt.h:130-227) restated in Python:
    first-scan estimate of every voxel, then per voxel: pending points are consumed only when MORE than min_points are
    waiting — first estimate, or running merge + eigenvalue clamp of the information matrix — and a voxel freezes once it
    has absorbed more than max_points.  Compared voxel by voxel with the oracle after a stream of overlapping scans."""
    cfg = default_config(FLS_NDT, localization_mode=0, ndt_min_points_in_voxel=5, ndt_max_points_in_voxel=50, ndt_capacity=1000000)
    o = orc.Registration(cfg)
    leaf, inv = cfg.source_cloud_filter_size, 1.0 / cfg.ndt_voxel_size
    vox, first = {}, True
    for k in range(6):
        cloud = synth.make_scan(world, traj[k // 2], "vlp16", seed=500 + k)["points"]
        T = traj[k // 2]
        cloud[:, :3] = (cloud[:, :3].astype(np.float64) @ T[:3, :3].T + T[:3, 3]).astype(np.float32)
        o.add_cloud(cloud)
        active = []
        for p in orc.voxel_grid(cloud, leaf)[:, :3].astype(np.float64):
            key = tuple((p * inv).astype(np.int32))  # C truncation [quirk 5]
            v = vox.get(key)
            if v is None:
                vox[key] = dict(pts=[p], mu=np.zeros(3), sigma=np.zeros((3, 3)), info=np.zeros((3, 3)), est=False, n=1)
            else:
                v["pts"].append(p)
                if not v["est"]:
                    v["n"] += 1
            if key not in active:
                active.append(key)
        for key in set(active):
            v = vox[key]
            P = np.array(v["pts"])
            if first:
                if len(P) > 1:
                    v["mu"], v["sigma"] = P.mean(0), np.cov(P.T, ddof=1).reshape(3, 3)
                    v["info"] = np.linalg.inv(v["sigma"] + 1e-3 * np.eye(3))
                else:
                    v["mu"], v["info"] = P[0], 100.0 * np.eye(3)
                v["est"], v["pts"] = True, []
                continue
            if v["est"] and v["n"] > cfg.ndt_max_points_in_voxel:
                continue
            if len(P) > cfg.ndt_min_points_in_voxel:
                cm, cv = P.mean(0), np.cov(P.T, ddof=1).reshape(3, 3)
                if not v["est"]:
                    v["mu"], v["sigma"] = cm, cv
                    v["info"] = np.linalg.inv(cv + 1e-3 * np.eye(3))
                    v["est"] = True
                else:
                    m, c = v["n"], len(P)
                    nm = (m * v["mu"] + c * cm) / (m + c)
                    nv = (m * (v["sigma"] + np.outer(v["mu"] - nm, v["mu"] - nm)) + c * (cv + np.outer(cm - nm, cm - nm))) / (m + c)
                    v["mu"], v["sigma"], v["n"] = nm, nv, m + c
                    lam, V = np.linalg.eigh(nv)
                    lam, V = lam[::-1].copy(), V[:, ::-1]
                    lam[1] = max(lam[1], lam[0] * 1e-3)
                    lam[2] = max(lam[2], lam[0] * 1e-3)
                    v["info"] = V @ np.diag(1.0 / lam) @ V.T
                v["pts"] = []
        first = False
    keys, mu, info, est = o.ndt_dump()
    assert len(keys) == len(vox)
    n_est = n_merged = 0
    for kk, m_, i_, e_ in zip(keys, mu, info, est):
        v = vox[tuple(kk)]
        assert bool(e_) == v["est"], kk
        if v["est"]:
            n_est += 1
            n_merged += v["n"] > 10
            assert np.allclose(m_, v["mu"], atol=1e-9), kk
            assert np.allclose(i_, v["info"], rtol=1e-6, atol=1e-6 * np.abs(v["info"]).max()), kk
    assert n_est > 500 and n_merged > 50 and n_est < len(vox)  # all three voxel states occur


def test_icp_first_iteration_against_numpy(scene16):
    """IcpOptimized::Match, iteration 0 (icp_optimized.h:57-127): VoxelGrid(source), fp32 transform with R, t cast to float,
    exact 1-NN on VoxelGrid(map), gate d^2 > max_correspond_distance [quirk 4], J = [I | -R p^], serial sums."""
    from scipy.spatial import cKDTree
    cfg = default_config(FLS_ICP_P2P, flags=FLS_FLAG_ITER_LOG, max_iterations=1)
    r = orc.Registration(cfg)
    r.add_cloud(scene16["map"])
    T = scene16["guess"]
    r.match(scene16["scan"], T)
    lg = r.iter_log()[0]
    src = orc.voxel_grid(scene16["scan"], cfg.source_cloud_filter_size)[:, :3]
    mp = orc.voxel_grid(scene16["map"], cfg.map_cloud_filter_size)[:, :3]
    Rf, tf = T[:3, :3].astype(np.float32), T[:3, 3].astype(np.float32)
    # q = R_f p + t_f in fp32, row by row in the order ((r0 x + r1 y) + r2 z) + t
    q = ((Rf[None, :, 0] * src[:, None, 0] + Rf[None, :, 1] * src[:, None, 1]) + Rf[None, :, 2] * src[:, None, 2]) + tf[None, :]
    assert q.dtype == np.float32
    tree = cKDTree(mp.astype(np.float64))
    _, nn = tree.query(q.astype(np.float64), k=1)
    d = q - mp[nn]
    d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]  # fp32 squared distance, as FLANN returns it
    keep = ~(d2.astype(np.float64) > cfg.icp_max_correspond_distance)
    H, g, res = np.zeros((6, 6)), np.zeros(6), 0.0
    R = T[:3, :3]
    for i in np.where(keep)[0]:
        e = q[i].astype(np.float64) - mp[nn[i]].astype(np.float64)
        J = np.hstack([np.eye(3), -R @ _hat(src[i].astype(np.float64))])
        H += J.T @ J
        g += -J.T @ e
        res += np.linalg.norm(e)
    assert int(keep.sum()) == lg["n_valid"] and lg["n_valid"] > 1000
    assert np.allclose(H, lg["H"], rtol=1e-9, atol=1e-9 * np.abs(H).max())
    assert np.allclose(g, lg["g"], rtol=1e-9, atol=1e-7)
    assert res == pytest.approx(lg["sum_residual"], rel=1e-9)


def test_ndt_first_iteration_against_numpy(scene16):
    """IncrementalNDT::Match, iteration 0 (incremental_ndt.h:232-304): VoxelGrid(source), fp64 q = R p + t, C-truncated key,
    7 stencil probes, chi-square gate, J = [-R p^ | I], H += J^T L J, err -= J^T L e, effective = number of accepted
    (point, voxel) pairs."""
    cfg = default_config(FLS_NDT, flags=FLS_FLAG_ITER_LOG, max_iterations=1)
    r = orc.Registration(cfg)
    r.add_cloud(scene16["map"])
    keys, mu, info, est = r.ndt_dump()
    lut = {tuple(k): i for i, k in enumerate(keys)}
    T = scene16["guess_small"]
    r.match(scene16["scan"], T)
    lg = r.iter_log()[0]
    src = orc.voxel_grid(scene16["scan"], cfg.source_cloud_filter_size)[:, :3].astype(np.float64)
    R, t = T[:3, :3], T[:3, 3]
    stencil = [(0, 0, 0), (-1, 0, 0), (1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, -1), (0, 0, 1)]
    H, g, n_eff, chi_sum = np.zeros((6, 6)), np.zeros(6), 0, 0.0
    for p in src:
        q = R @ p + t
        k0 = (q * (1.0 / cfg.ndt_voxel_size)).astype(np.int32)
        J = np.hstack([-R @ _hat(p), np.eye(3)])
        for o in stencil:
            vi = lut.get((k0[0] + o[0], k0[1] + o[1], k0[2] + o[2]))
            if vi is None or not est[vi]:
                continue
            e = q - mu[vi]
            chi = e @ info[vi] @ e
            if np.isnan(chi) or chi > cfg.ndt_outlier_thres:
                continue
            H += J.T @ info[vi] @ J
            g += -J.T @ info[vi] @ e
            n_eff += 1
            chi_sum += chi
    assert n_eff == lg["n_valid"] and n_eff > 1000
    assert np.allclose(H, lg["H"], rtol=1e-8, atol=1e-9 * np.abs(H).max())
    assert np.allclose(g, lg["g"], rtol=1e-8, atol=1e-6)
