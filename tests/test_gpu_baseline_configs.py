"""GPU parity at the REAL shape of the BASELINE.json configs (VERDICT r1 "next round" item 1), through the C ABI vs the CPU oracle:

  config 4  LoamPointToPlaneIVOX, 64-line ~108k-pt scans, batch of 8 through fls_match_batch (loam_point_to_plane_ivox.h:141-216)
  config 5  IncrementalNDT, dense 128-line scan, max_iterations = 10 with zero thresholds -> exactly 10 iterations, leaf 0.01
            pass-through (incremental_ndt.h:229-337), per-iteration H / g compared
  config 2  IncrementalNDT mapping-mode STREAM of 64-line scans: pose, iteration count and voxel count scan by scan
"""
import numpy as np
import pytest

from funny_lidar_slam_b200 import FLS_NDT, FLS_P2PLANE_IVOX, default_config, synth
from funny_lidar_slam_b200._abi import FLS_FLAG_ITER_LOG

pytestmark = pytest.mark.gpu
POS_TOL, ROT_TOL = 1e-4, 1e-4  # BASELINE.json north_star


@pytest.fixture(scope="module")
def surface_map(world):
    return synth.make_surface_map(world, spacing=0.3, seed=4321)  # ~0.6 M points: the `p2plane_ivox_64_small` bench map


def test_config4_batch8_64line_vs_oracle(world, surface_map):
    from funny_lidar_slam_b200.registration import Registration
    from oracle import pyoracle as orc
    traj = synth.trajectory(64)
    scans = [synth.make_scan(world, traj[3 + 5 * i], "hdl64", seed=100 + i)["points"] for i in range(8)]
    guesses = [synth.perturb_pose(traj[3 + 5 * i], seed=77 + i) for i in range(8)]  # 0.3 m / 3 deg, as the bench
    assert min(len(s) for s in scans) > 90000
    cfg = default_config(FLS_P2PLANE_IVOX, flags=FLS_FLAG_ITER_LOG)
    g, o = Registration(cfg), orc.Registration(cfg)
    g.AddCloudToLocalMap([surface_map])
    o.add_cloud(surface_map)
    conv, Tb = g.match_batch(scans, np.stack(guesses))
    its = []
    for s in range(8):
        ok_o, To, st_o = o.match(scans[s], guesses[s])
        st_g = g.last_batch_stats[s]
        # iteration 0 runs at the same pose on both sides: the normal equations of every scan agree to fp64 rounding
        lg, lo = g.iter_log(s), o.iter_log()
        assert len(lg) == st_g.iterations and lg[0]["n_valid"] == lo[0]["n_valid"], s
        H0 = lo[0]["H"]
        assert np.allclose(lg[0]["H"], H0, rtol=1e-9, atol=1e-9 * np.abs(H0).max()), s
        assert np.allclose(lg[0]["g"], lo[0]["g"], rtol=1e-9, atol=1e-9 * np.abs(H0).max()), s
        assert bool(conv[s]) == ok_o, s
        assert st_g.iterations == st_o.iterations, (s, st_g.iterations, st_o.iterations)
        assert abs(st_g.n_valid - st_o.n_valid) <= max(2, st_o.n_valid // 2000), (s, st_g.n_valid, st_o.n_valid)
        dt, dr = synth.pose_error(Tb[s], To)
        assert dt < POS_TOL and dr < ROT_TOL, (s, dt, dr)
        assert synth.pose_error(Tb[s], traj[3 + 5 * s])[0] < 0.1
        its.append(st_o.iterations)
    assert conv.all() and len(set(its)) > 1  # the scans of the batch really stop at different iterations


def test_config4_device_result_buffer_matches_host_results(world, surface_map):
    """fls_set_result_buffer_device: what the GN kernel writes for the all-gather equals what the call returns on the host."""
    import torch

    from funny_lidar_slam_b200 import parallel
    from funny_lidar_slam_b200.registration import Registration
    traj = synth.trajectory(64)
    scans = [synth.make_scan(world, traj[3 + 5 * i], "hdl64", seed=100 + i)["points"][:: 1 + i % 3] for i in range(4)]
    scans.append(scans[0][:30].copy())  # a failing scan (too few planes)
    guesses = [synth.perturb_pose(traj[3 + 5 * (i % 4)], seed=77 + i) for i in range(5)]
    g = Registration(default_config(FLS_P2PLANE_IVOX))
    g.AddCloudToLocalMap([surface_map])
    buf = torch.full((5 * parallel.RESULT_LEN,), -7.0, dtype=torch.float64, device="cuda:0")
    g.set_result_buffer_device(buf.data_ptr(), 5)
    conv, Tb = g.match_batch(scans, np.stack(guesses))
    got = buf.cpu().numpy().reshape(5, parallel.RESULT_LEN)
    for s in range(5):
        T, ok, it = parallel.unpack_result(got[s])
        assert np.array_equal(T, Tb[s]) and ok == bool(conv[s]) and it == g.last_batch_stats[s].iterations, s
    assert not conv[4]
    g.set_result_buffer_device(0, 0)


def test_config5_ndt_128line_exactly_10_iterations(world, surface_map):
    from funny_lidar_slam_b200.registration import PointcloudCluster, Registration
    from oracle import pyoracle as orc
    traj = synth.trajectory(16)
    scan = synth.make_scan(world, traj[5], "os128", seed=305)["points"]
    assert len(scan) > 120000
    guess = synth.perturb_pose(traj[5], seed=905, dpos=0.05, drot_deg=0.5)
    cfg = default_config(FLS_NDT, ndt_capacity=2000000, source_cloud_filter_size=0.01, max_iterations=10, position_converge_thres=0.0,
                         rotation_converge_thres=0.0, flags=FLS_FLAG_ITER_LOG)
    g, o = Registration(cfg), orc.Registration(cfg)
    g.AddCloudToLocalMap([surface_map])
    o.add_cloud(surface_map)
    assert g.map_info().n_voxels == o.map_voxels
    Tg = guess.copy()
    ok_g = g.Match(PointcloudCluster(ordered_cloud=scan), Tg)
    ok_o, To, st_o = o.match(scan, guess)
    st_g = g.last_stats
    assert ok_g and ok_o
    assert st_g.iterations == st_o.iterations == 10          # thresholds 0: never stops early (incremental_ndt.h:315)
    assert st_g.n_source == st_o.n_source == len(scan)      # leaf 0.01: pcl::VoxelGrid passes the cloud through (index overflow)
    lg, lo = g.iter_log(), o.iter_log()
    assert len(lg) == len(lo) == 10
    for it in range(10):
        assert lg[it]["n_valid"] == lo[it]["n_valid"], it
        scale = np.abs(lo[it]["H"]).max()
        assert np.allclose(lg[it]["H"], lo[it]["H"], rtol=1e-7, atol=1e-9 * scale), it
        assert np.allclose(lg[it]["g"], lo[it]["g"], rtol=1e-7, atol=1e-9 * scale), it
    dt, dr = synth.pose_error(Tg, To)
    assert dt < POS_TOL and dr < ROT_TOL, (dt, dr)
    assert synth.pose_error(Tg, traj[5])[0] < 0.02


def test_config2_ndt_64line_mapping_stream(world):
    """12-scan 64-line stream in mapping mode with the shipped parameters except the capacity (the LRU test covers that):
    every Match inserts the filtered scan at the INPUT guess (quirk 6); poses, iterations and voxel counts follow the oracle."""
    from funny_lidar_slam_b200.registration import PointcloudCluster, Registration
    from oracle import pyoracle as orc
    traj = synth.trajectory(16)
    cfg = default_config(FLS_NDT, localization_mode=0, ndt_capacity=2000000)
    g, o = Registration(cfg), orc.Registration(cfg)
    first = synth.transform_points(synth.make_scan(world, traj[0], "hdl64", seed=500)["points"], traj[0])
    g.AddCloudToLocalMap([first])
    o.add_cloud(first)
    assert g.map_info().n_voxels == o.map_voxels
    for k in range(1, 13):
        scan = synth.make_scan(world, traj[k], "hdl64", seed=500 + k)["points"]
        guess = synth.perturb_pose(traj[k], seed=600 + k, dpos=0.05, drot_deg=0.5)  # stand-in for the IMU prediction (frontend.cpp:191-205)
        Tg = guess.copy()
        ok_g = g.Match(PointcloudCluster(ordered_cloud=scan), Tg)
        ok_o, To, st_o = o.match(scan, guess)
        assert ok_g == ok_o, k
        assert g.last_stats.iterations == st_o.iterations, (k, g.last_stats.iterations, st_o.iterations)
        dt, dr = synth.pose_error(Tg, To)
        assert dt < POS_TOL and dr < ROT_TOL, (k, dt, dr)
        assert g.map_info().n_voxels == o.map_voxels, k
    assert synth.pose_error(Tg, traj[12])[0] < 0.1  # the map is built at the (perturbed) input guesses: guess-level drift
