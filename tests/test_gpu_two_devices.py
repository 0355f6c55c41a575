"""Two devices in one process: a kernel's attributes (its dynamic shared-memory limit, its co-resident CTA count) are per device,
so a handle on device 1 must get them set for device 1 even after a handle on device 0 has set them there."""
import numpy as np
import pytest

from funny_lidar_slam_b200 import FLS_NDT, FLS_P2PLANE_IVOX, default_config, synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def two_devices():
    from funny_lidar_slam_b200._lib import lib
    n = lib().fls_device_count()
    if n < 2:
        pytest.skip(f"needs two CUDA devices, this machine shows {n}")


def _on_both(method, mp):
    from funny_lidar_slam_b200.registration import Registration
    regs = []
    for dev in (0, 1):
        g = Registration(default_config(method, device=dev))
        g.AddCloudToLocalMap([mp])
        regs.append(g)
    return regs


def _same(a, b):
    (ok0, T0, it0), (ok1, T1, it1) = a, b
    assert np.array_equal(ok0, ok1) and it0 == it1
    for P, Q in zip(np.reshape(T0, (-1, 4, 4)), np.reshape(T1, (-1, 4, 4))):
        dt, dr = synth.pose_error(P, Q)
        assert dt < 1e-9 and dr < 1e-9, (dt, dr)


def _scans(world, traj, sensor, B):
    scans = [synth.make_scan(world, traj[k % 12], sensor, seed=90 + k)["points"] for k in range(B)]
    guesses = np.stack([synth.perturb_pose(traj[k % 12], seed=900 + k, dpos=0.05, drot_deg=0.5) for k in range(B)])
    return scans, guesses


def test_loam_ivox_batch_and_single_on_two_devices(two_devices, world, traj):
    from funny_lidar_slam_b200.registration import PointcloudCluster
    mp = synth.make_map_from_scans(world, traj[0:12:2], "vlp16", leaf=0.3)
    regs = _on_both(FLS_P2PLANE_IVOX, mp)
    scans, guesses = _scans(world, traj, "vlp16", 8)
    batch, single = [], []
    for g in regs:  # device 0 first: it is the one that used to get the batch kernel's shared-memory limit
        ok, T = g.match_batch(scans, guesses)  # a batch of 8 runs on the v9 kernel
        batch.append((ok, T, [s.iterations for s in g.last_batch_stats]))
        T1 = guesses[0].copy()
        ok1 = g.Match(PointcloudCluster(planar_cloud=scans[0]), T1)  # a single Match runs on the v8 kernel
        single.append((ok1, T1, g.last_stats.iterations))
    _same(*batch)
    _same(*single)


def test_ndt_batch_on_two_devices(two_devices, world, traj):
    mp = synth.make_map_from_scans(world, traj[0:12:2], "hdl64", leaf=0.3)
    regs = _on_both(FLS_NDT, mp)
    scans, guesses = _scans(world, traj, "vlp16", 8)
    out = []
    for g in regs:
        ok, T = g.match_batch(scans, guesses)
        out.append((ok, T, [s.iterations for s in g.last_batch_stats]))
    _same(*out)
