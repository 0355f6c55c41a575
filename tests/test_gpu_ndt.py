"""GPU parity: IncrementalNDT path (K2 + K6 + K7 + K8-NDT) through the C ABI vs the CPU oracle."""
import numpy as np
import pytest

from funny_lidar_slam_b200 import FLS_NDT, default_config, synth
from funny_lidar_slam_b200._abi import FLS_FLAG_ITER_LOG

pytestmark = pytest.mark.gpu
POS_TOL, ROT_TOL = 1e-4, 1e-4


def _pair(cfg):
    from funny_lidar_slam_b200.registration import Registration
    from oracle import pyoracle as orc
    return Registration(cfg), orc.Registration(cfg)


def _cluster(scan):
    from funny_lidar_slam_b200.registration import PointcloudCluster
    return PointcloudCluster(ordered_cloud=scan)


@pytest.mark.parametrize("scene_name", ["scene16", "scene64"])
def test_match_static_map(scene_name, request):
    sc = request.getfixturevalue(scene_name)
    cfg = default_config(FLS_NDT, flags=FLS_FLAG_ITER_LOG)
    g, o = _pair(cfg)
    g.AddCloudToLocalMap([sc["map"]])
    o.add_cloud(sc["map"])
    assert g.map_info().n_voxels == o.map_voxels
    Tg = sc["guess_small"].copy()
    ok_g = g.Match(_cluster(sc["scan"]), Tg)
    ok_o, To, st_o = o.match(sc["scan"], sc["guess_small"])
    st_g = g.last_stats
    assert ok_g == ok_o and st_g.iterations == st_o.iterations
    lg, lo = g.iter_log(), o.iter_log()
    assert lg[0]["n_valid"] == lo[0]["n_valid"]
    assert np.allclose(lg[0]["H"], lo[0]["H"], rtol=1e-9, atol=1e-5)
    assert np.allclose(lg[0]["g"], lo[0]["g"], rtol=1e-9, atol=1e-5)
    dt, dr = synth.pose_error(Tg, To)
    assert dt < POS_TOL and dr < ROT_TOL, (dt, dr)
    assert synth.pose_error(Tg, sc["truth"])[0] < 0.02
    # GetFitnessScore in localization mode
    fo, fg = o.fitness(2.0), g.GetFitnessScore(2.0)
    assert abs(fg - fo) <= 1e-5 * max(1.0, abs(fo))


def test_early_out_when_too_few_effective_points(scene16):
    """effective_num < min_effective_pts: Match returns false with T = current pose (incremental_ndt.h:306-309)."""
    cfg = default_config(FLS_NDT)
    g, o = _pair(cfg)
    g.AddCloudToLocalMap([scene16["map"]])
    o.add_cloud(scene16["map"])
    far = scene16["guess"].copy()
    far[:3, 3] += 300.0
    Tg = far.copy()
    ok_g = g.Match(_cluster(scene16["scan"]), Tg)
    ok_o, To, st_o = o.match(scene16["scan"], far)
    assert ok_g is False and ok_o is False
    assert g.last_stats.iterations == st_o.iterations == 1
    assert np.allclose(Tg, To, atol=1e-12)


def test_streaming_mapping_mode(world, traj):
    """Mapping mode: every Match inserts the scan (transformed by the INPUT guess, quirk 6) and voxels follow the
    incremental UpdateVoxel rules; poses must track the oracle over a short stream."""
    cfg = default_config(FLS_NDT, localization_mode=0, max_iterations=15)
    g, o = _pair(cfg)
    first = synth.make_scan(world, traj[0], "vlp16", seed=40)["points"]
    first_w = synth.transform_points(first, traj[0])
    g.AddCloudToLocalMap([first_w])
    o.add_cloud(first_w)
    assert g.map_info().n_voxels == o.map_voxels
    Tg = traj[0].copy()
    for k in range(1, 6):
        scan = synth.make_scan(world, traj[k], "vlp16", seed=40 + k)["points"]
        # stand-in for the IMU / constant-velocity prediction of FrontEnd::Run (frontend.cpp:191-205 upstream)
        guess = synth.perturb_pose(traj[k], seed=400 + k, dpos=0.05, drot_deg=0.5)
        Tg = guess.copy()
        ok_g = g.Match(_cluster(scan), Tg)
        ok_o, To, st_o = o.match(scan, guess)
        assert ok_g == ok_o, k
        assert g.last_stats.iterations == st_o.iterations, k
        dt, dr = synth.pose_error(Tg, To)
        assert dt < POS_TOL and dr < ROT_TOL, (k, dt, dr)
        assert g.map_info().n_voxels == o.map_voxels, k
    assert synth.pose_error(Tg, traj[5])[0] < 0.05


def test_batch_equals_single_and_oracle(world, traj, scene64):
    """fls_match_batch for IncrementalNDT: one cooperative launch, a sub-grid and a Gauss-Newton loop per scan.  Every scan's
    result must equal its own single Match (same arithmetic, different CTA count -> fp64 rounding only) and the oracle."""
    cfg = default_config(FLS_NDT, flags=FLS_FLAG_ITER_LOG)
    g, o = _pair(cfg)
    g.AddCloudToLocalMap([scene64["map"]])
    o.add_cloud(scene64["map"])
    scans, guesses = [], []
    for k in range(5):
        sensor = "hdl64" if k % 2 == 0 else "vlp16"  # ragged batch: different sizes -> different sub-grids
        scans.append(synth.make_scan(world, traj[2 + k], sensor, seed=70 + k)["points"])
        guesses.append(synth.perturb_pose(traj[2 + k], seed=700 + k, dpos=0.05, drot_deg=0.5))
    oks, Ts = g.match_batch(scans, np.stack(guesses))
    sts = g.last_batch_stats
    logs = [g.iter_log(k) for k in range(5)]
    for k in range(5):
        T1 = guesses[k].copy()
        ok1 = g.Match(_cluster(scans[k]), T1)
        ok_o, To, st_o = o.match(scans[k], guesses[k])
        # iteration 0 of every scan of the batch against the oracle: same pose, same (point, voxel) pairs, the same terms
        # summed in another order.  Two fp64 sums of n terms differ by at most 2 n eps sum|term| (recursive summation); each
        # term is a few dozen flops (allow 64 n eps in all).  With every information matrix L positive semi-definite,
        # Cauchy-Schwarz bounds sum|J_a^T L J_b| by sqrt(H_aa H_bb) and sum|J_a^T L e| by sqrt(H_aa sum e^T L e), and
        # sum e^T L e is the logged sum_residual.
        lo = o.iter_log()
        assert len(logs[k]) == sts[k].iterations and logs[k][0]["n_valid"] == lo[0]["n_valid"], k
        H0, n = lo[0]["H"], lo[0]["n_valid"]
        dH = np.sqrt(np.abs(np.diag(H0)))
        tol = 64 * n * np.finfo(np.float64).eps
        assert np.all(np.abs(logs[k][0]["H"] - H0) <= tol * np.outer(dH, dH)), k
        assert np.all(np.abs(logs[k][0]["g"] - lo[0]["g"]) <= tol * dH * np.sqrt(lo[0]["sum_residual"])), k
        assert bool(oks[k]) == ok1 == ok_o, k
        assert sts[k].iterations == g.last_stats.iterations == st_o.iterations, k
        assert sts[k].n_valid == g.last_stats.n_valid == st_o.n_valid, k
        dt, dr = synth.pose_error(Ts[k], T1)
        assert dt < 1e-9 and dr < 1e-9, (k, dt, dr)
        dt, dr = synth.pose_error(Ts[k], To)
        assert dt < POS_TOL and dr < ROT_TOL, (k, dt, dr)
