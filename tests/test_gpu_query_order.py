"""GPU: the per-batch query ordering of the LOAM-iVox path (one prep kernel, scans sorted in 8192-point tiles) must neither lose
nor repeat a point, whatever the scan sizes: scan sizes around the tile size and below it, in batches run on both kernels,
checked against the CPU oracle (iterations, converged flag and n_valid are counts over every point)."""
import numpy as np
import pytest

from funny_lidar_slam_b200 import FLS_P2PLANE_IVOX, default_config, synth

pytestmark = pytest.mark.gpu


def test_tiles_keep_every_point(world, traj):
    from funny_lidar_slam_b200.registration import PointcloudCluster, Registration
    from oracle import pyoracle as orc
    mp = synth.make_map_from_scans(world, traj[0:12:2], "vlp16", leaf=0.3)
    cfg = default_config(FLS_P2PLANE_IVOX)
    g = Registration(cfg)
    g.AddCloudToLocalMap([mp])
    o = orc.Registration(cfg)
    o.add_cloud(mp)
    rng = np.random.default_rng(5)
    scans, guesses = [], []
    for j, n in enumerate([8191, 8192, 8193, 16385, 3000, 1]):
        base = synth.make_scan(world, traj[3 + j % 4], "vlp16", seed=400 + j)["points"]
        sel = np.sort(rng.choice(len(base), min(n, len(base)), replace=False))
        scans.append(np.ascontiguousarray(base[sel]))
        guesses.append(synth.perturb_pose(traj[3 + j % 4], dpos=0.1, drot_deg=1.0, seed=600 + j))
    conv, Tb = g.match_batch(scans, np.stack(guesses))
    st_b = list(g.last_batch_stats)
    for j, (sc, gs) in enumerate(zip(scans, guesses)):
        ok_o, To, st_o = o.match(sc, gs)
        assert bool(conv[j]) == ok_o and st_b[j].iterations == st_o.iterations and st_b[j].n_valid == st_o.n_valid, j
        dt, dr = synth.pose_error(Tb[j], To)
        assert dt < 1e-4 and dr < 1e-4, j
        T = gs.copy()  # the single-scan kernel orders the same way
        ok = g.Match(PointcloudCluster(planar_cloud=sc), T)
        assert ok == ok_o and g.last_stats.n_valid == st_o.n_valid and g.last_stats.iterations == st_o.iterations, j
