import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    from funny_lidar_slam_b200._mem import tune_malloc
    tune_malloc()
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a) CUDA device")


def pytest_collection_modifyitems(config, items):
    """A GPU test that does not come back (a persistent kernel waiting for a hand-over that never arrives) must fail, not hang the
    box: pytest-timeout's thread method ends the process, which also ends the kernel.  (The batch kernel additionally carries a
    device-side watchdog, fls_p2plane_v9.cu.)"""
    if not config.pluginmanager.hasplugin("timeout"):
        return
    for item in items:
        if item.get_closest_marker("gpu") is not None and item.get_closest_marker("timeout") is None:
            item.add_marker(pytest.mark.timeout(240, method="thread"))


@pytest.fixture(scope="session")
def world():
    from funny_lidar_slam_b200 import synth
    return synth.make_world()


@pytest.fixture(scope="session")
def traj():
    from funny_lidar_slam_b200 import synth
    return synth.trajectory(16)


@pytest.fixture(scope="session")
def scene16(world, traj):
    """BASELINE config-1-sized data: 16-line scans + a static map built from neighbouring poses."""
    from funny_lidar_slam_b200 import synth
    scan = synth.make_scan(world, traj[5], "vlp16", seed=5)
    mp = synth.make_map_from_scans(world, traj[0:12:2], "vlp16", leaf=0.3)
    return dict(scan=scan["points"], map=mp, truth=traj[5], guess=synth.perturb_pose(traj[5]), guess_small=synth.perturb_pose(traj[5], dpos=0.05, drot_deg=0.5))


@pytest.fixture(scope="session")
def scene64(world, traj):
    from funny_lidar_slam_b200 import synth
    scan = synth.make_scan(world, traj[6], "hdl64", seed=6)
    mp = synth.make_map_from_scans(world, traj[2:12:3], "hdl64", leaf=0.3)
    return dict(scan=scan["points"], map=mp, truth=traj[6], guess=synth.perturb_pose(traj[6]), guess_small=synth.perturb_pose(traj[6], dpos=0.05, drot_deg=0.5))


def to_pcl(points: np.ndarray) -> np.ndarray:
    """(n,4) packed -> (n,8) pcl::PointXYZI records (x,y,z,1 | intensity,0,0,0)."""
    out = np.zeros((len(points), 8), np.float32)
    out[:, :3] = points[:, :3]
    out[:, 3] = 1.0
    out[:, 4] = points[:, 3]
    return out
