"""GPU parity (8f-4): the localization-mode map path — Localization::LoadLocalMap's global-map branch (localization.cpp:364-410):
resident global map, +-100 m CropBox around the pose when the pose nears an edge, handed to AddCloudToLocalMap on the device.
The crop must build the same map as the same cloud given to fls_add_cloud: both go through the plug-in's one AddCloudToLocalMap."""
import numpy as np
import pytest

from funny_lidar_slam_b200 import FLS_ICP_P2P, FLS_NDT, FLS_P2PLANE_IVOX, FLS_P2PLANE_KNN, default_config, synth

pytestmark = pytest.mark.gpu


def _crop(mp, T):
    lo = (T[:3, 3] - 100.0).astype(np.float32)
    hi = (T[:3, 3] + 100.0).astype(np.float32)
    k = np.all((mp[:, :3] >= lo) & (mp[:, :3] <= hi), axis=1)
    return mp[k]


def _map_info(g):
    m = g.map_info()
    return tuple(getattr(m, f) for f, _ in m._fields_)


@pytest.mark.parametrize("method", [FLS_P2PLANE_IVOX, FLS_NDT, FLS_ICP_P2P, FLS_P2PLANE_KNN])
def test_local_map_follows_the_pose(method):
    from funny_lidar_slam_b200.registration import PointcloudCluster, Registration
    from oracle import pyoracle as orc
    world = synth.make_world(seed=7, half=350.0, n_boxes=300, n_cyls=200, keepout=8.0)
    mp = synth.make_surface_map(world, spacing=0.6, seed=1)
    traj = synth.trajectory(400, step=1.0, scale=140.0)
    cfg = default_config(method)
    g = Registration(cfg)
    g.set_global_map(mp)
    direct = Registration(cfg)  # fed each crop through fls_add_cloud
    edge = None
    n_updates = 0
    for k in range(0, 400, 25):
        T = traj[k]
        need = edge is None or any(not (abs(T[i, 3] - edge[i]) > 50.0 and abs(T[i, 3] - edge[i + 3]) > 50.0) for i in range(3))
        upd, nl = g.update_local_map(T)
        assert upd == need, k
        if need:
            edge = np.concatenate([T[:3, 3] - 100.0, T[:3, 3] + 100.0])
            crop = _crop(mp, T)
            assert nl == len(crop), k
            n_updates += 1
            if method == FLS_P2PLANE_IVOX:
                assert g.map_info().n_points == len(crop)
                assert np.array_equal(g.map_points(), crop)  # CropBox keeps the input order
            direct.AddCloudToLocalMap([crop])
            assert _map_info(g) == _map_info(direct), k
            # Match against the cropped map == the oracle on the same crop
            o = orc.Registration(cfg)
            o.add_cloud(crop)
            scan = synth.make_scan(world, T, "vlp16", seed=900 + k)["points"]
            guess = synth.perturb_pose(T, seed=k, dpos=0.05, drot_deg=0.5)
            Tg = guess.copy()
            features = method in (FLS_P2PLANE_IVOX, FLS_P2PLANE_KNN)
            cl = PointcloudCluster(planar_cloud=scan) if features else PointcloudCluster(ordered_cloud=scan)
            ok_g = g.Match(cl, Tg)
            Td = guess.copy()
            ok_d = direct.Match(cl, Td)
            assert ok_d == ok_g and np.array_equal(Td, Tg), k
            assert direct.last_stats.iterations == g.last_stats.iterations and direct.last_stats.n_valid == g.last_stats.n_valid, k
            ok_o, To, st_o = o.match(scan, guess)
            assert ok_g == ok_o and g.last_stats.iterations == st_o.iterations, k
            if method == FLS_P2PLANE_KNN:
                assert g.last_stats.n_valid == st_o.n_valid, k
            dt, dr = synth.pose_error(Tg, To)
            assert dt < 1e-4 and dr < 1e-4, (k, dt, dr)
    assert 2 <= n_updates < 16  # re-cut a few times along the path, not at every pose
