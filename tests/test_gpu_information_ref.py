"""FLS_FLAG_INFORMATION against an independent reference (tests/info_ref.py): every record — single Match, every scan of a 4- and a
64-scan batch, and the Matches of a mapping-mode stream — is rebuilt in fp64 from T_final as the device returned it, with brute-force
correspondences (tests/ivox_ref.py, ndt_ref.py, icp_ref.py, loam_kd_ref.py) and analytic Jacobians in the fusion parameterization,
and compared with the issue's tolerances: n_valid equal, H within 1e-9 |H|, g within 1e-9 |g| + 1e-12, sum_residual 1e-9 relative.

The scene is a crop of the session map around the scan's pose and a thinned scan, so that the 50-digit plane and line fits of the
references stay affordable; at T_final some of its points pass and some fail each plug-in's gates.  The gate-edge scenes of the
first-pass tests (tests/*_scenes.py) hold the shared per-point functions to the same references at the gates themselves."""
import numpy as np
import pytest

from funny_lidar_slam_b200 import FLS_ICP_P2P, FLS_NDT, FLS_P2PLANE_IVOX, FLS_P2PLANE_KNN, default_config, synth
from funny_lidar_slam_b200._abi import FLS_FLAG_INFORMATION, FLS_LOAM_FULL
from tests import icp_ref, info_ref, ivox_ref, loam_kd_ref, ndt_ref

pytestmark = pytest.mark.gpu
METHODS = {"ivox": FLS_P2PLANE_IVOX, "ndt": FLS_NDT, "icp": FLS_ICP_P2P, "kd": FLS_P2PLANE_KNN, "full": FLS_LOAM_FULL}
F32 = np.float32


@pytest.fixture(scope="module")
def small(scene16):
    T = scene16["truth"]
    mp = scene16["map"]
    keep = np.all(np.abs(mp[:, :3].astype(np.float64) - T[:3, 3]) < 14.0, axis=1)
    scan = scene16["scan"]
    r = np.linalg.norm(scan[:, :3], axis=1)
    sc = scan[(r < 12.0)][::9].copy()
    return dict(map=mp[keep].copy(), scan=sc, truth=T)


def _reg(method, **kw):
    from funny_lidar_slam_b200.registration import Registration
    kw.setdefault("localization_mode", 1)
    return Registration(default_config(method, flags=FLS_FLAG_INFORMATION, **kw))


def _corner(scan):
    return scan[::4].copy()


def _add(g, method, mp):
    g.AddCloudToLocalMap([mp, mp[::3].copy()] if method == FLS_LOAM_FULL else [mp])


def _cluster(method, scan):
    from funny_lidar_slam_b200.registration import PointcloudCluster
    if method in (FLS_NDT, FLS_ICP_P2P):
        return PointcloudCluster(ordered_cloud=scan)
    return PointcloudCluster(planar_cloud=scan, corner_cloud=_corner(scan) if method == FLS_LOAM_FULL else None)


def _ndt_map(g, cfg):
    """The handle's NDT map as the reference's voxel dictionary (its estimation is held to ndt_ref elsewhere)."""
    ref = ndt_ref.NdtRef(cfg.ndt_voxel_size, cfg.ndt_min_points_in_voxel, cfg.ndt_max_points_in_voxel, cfg.ndt_capacity,
                         cfg.source_cloud_filter_size, True)
    v = g.ndt_voxels()
    for k in range(len(v["key"])):
        if not v["estimated"][k]:
            ref.data[tuple(int(x) for x in v["key"][k])] = ndt_ref.Voxel(estimated=False)
            continue
        ref.data[tuple(int(x) for x in v["key"][k])] = ndt_ref.Voxel(mu=np.array(v["mu"][k]), info=ndt_ref.sym6_to_3x3(v["info"][k]), estimated=True)
    return ref


def _reference(method, g, cfg, mp, scan, T):
    """The record the reference expects for `scan` matched to T against the map `mp` the Match searched (NDT: the handle's map)."""
    if method == FLS_P2PLANE_IVOX:
        ref = ivox_ref.planar_pass(mp, scan, T, cfg.point_to_planar_thres, cfg.ivox_resolution, cfg.ivox_nearby, cfg.ivox_max_range)
        return info_ref.ivox_record(ref, np.asarray(scan, F32), T)
    if method == FLS_NDT:
        from oracle import pyoracle as orc
        ref_map = _ndt_map(g, cfg)
        p = ndt_ref.ndt_pass(ref_map, scan, T, cfg.ndt_outlier_thres, cfg.source_cloud_filter_size)
        return info_ref.ndt_record(p, orc.voxel_grid(np.asarray(scan, F32), cfg.source_cloud_filter_size), T)
    if method == FLS_ICP_P2P:
        p = icp_ref.icp_pass(mp, scan, T, cfg.icp_max_correspond_distance, cfg.source_cloud_filter_size, cfg.map_cloud_filter_size)
        return info_ref.icp_record(p, T)
    full = method == FLS_LOAM_FULL
    if full:
        planar_map, corner_map, corner = mp, mp[::3].copy(), _corner(scan)
    else:
        from oracle import pyoracle as orc
        planar_map, corner_map, corner = orc.voxel_grid(np.asarray(mp, F32), cfg.map_cloud_filter_size), None, None
    p = loam_kd_ref.kd_pass(planar_map, corner_map, scan, corner, T, full, thres=cfg.point_search_thres, line_ratio=cfg.line_ratio_thres,
                            plane_thres=cfg.point_to_planar_thres)
    return info_ref.kd_record(p, np.asarray(scan, F32), None if corner is None else np.asarray(corner, F32), T)


@pytest.mark.parametrize("name", list(METHODS))
def test_single_match_against_reference(small, name):
    method = METHODS[name]
    g = _reg(method)
    _add(g, method, small["map"])
    T = synth.perturb_pose(small["truth"], dpos=0.05, drot_deg=0.5)
    g.Match(_cluster(method, small["scan"]), T)
    info_ref.assert_record(g.information(), _reference(method, g, g.cfg, small["map"], small["scan"], T), name)


@pytest.mark.parametrize("B", [4, 64])
@pytest.mark.parametrize("name", ["ivox", "ndt", "icp", "kd"])
def test_every_scan_of_a_batch_against_reference(small, name, B):
    method = METHODS[name]
    g = _reg(method)
    _add(g, method, small["map"])
    scans = [small["scan"][k % 3::3].copy() for k in range(B)]
    Ts = np.stack([synth.perturb_pose(small["truth"], seed=100 + k, dpos=0.1, drot_deg=1.0) for k in range(B)])
    _, Tf = g.match_batch(scans, Ts)
    for s in range(B):
        info_ref.assert_record(g.information(s), _reference(method, g, g.cfg, small["map"], scans[s], Tf[s]), (name, B, s))


@pytest.mark.parametrize("name", ["ivox", "ndt"])
def test_mapping_mode_against_reference(world, traj, name):
    """Mapping mode: each record against the map as it was before the Match inserted its scan (iVox: fls_get_map_points; NDT: the
    voxels), so a record that saw its own scan would fail."""
    method = METHODS[name]
    g = _reg(method, localization_mode=0)
    first = synth.make_scan(world, traj[0], "vlp16", seed=0)["points"]
    g.AddCloudToLocalMap([synth.transform_points(first, traj[0])])
    for k in range(1, 4):
        scan = synth.make_scan(world, traj[k], "vlp16", seed=k)["points"]
        scan = scan[np.linalg.norm(scan[:, :3], axis=1) < 12.0][::7].copy()
        mp = g.map_points() if method == FLS_P2PLANE_IVOX else None
        ref_map = _ndt_map(g, g.cfg) if method == FLS_NDT else None
        T = synth.perturb_pose(traj[k], dpos=0.05, drot_deg=0.5)
        g.Match(_cluster(method, scan), T)
        if method == FLS_NDT:
            from oracle import pyoracle as orc
            p = ndt_ref.ndt_pass(ref_map, scan, T, g.cfg.ndt_outlier_thres, g.cfg.source_cloud_filter_size)
            want = info_ref.ndt_record(p, orc.voxel_grid(np.asarray(scan, F32), g.cfg.source_cloud_filter_size), T)
        else:
            ref = ivox_ref.planar_pass(mp, scan, T, g.cfg.point_to_planar_thres, g.cfg.ivox_resolution, g.cfg.ivox_nearby, g.cfg.ivox_max_range)
            want = info_ref.ivox_record(ref, np.asarray(scan, F32), T)
        info_ref.assert_record(g.information(), want, (name, k))
