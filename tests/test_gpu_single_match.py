"""Single-scan Match on the persistent Gauss-Newton kernels (LOAM-iVox, NDT, ICP, kd-tree point-to-plane):

  * the packed result the kernel writes into the caller's device buffer when the loop stops (fls_set_result_buffer_device)
    equals the pose, converged flag and iteration count the call returns on the host;
  * a single LOAM-iVox Match repeated on the same input is bitwise identical: the folding CTA sums the CTA rows in a fixed
    order, so the pose, iterations, n_valid and every iteration's H, g and dx do not depend on the order the rows arrive in.

Each runs on a scan that converges, one that stops at max_iterations and a failing 30-point scan.
"""
import numpy as np
import pytest

from funny_lidar_slam_b200 import FLS_ICP_P2P, FLS_NDT, FLS_P2PLANE_IVOX, FLS_P2PLANE_KNN, default_config
from funny_lidar_slam_b200._abi import FLS_FLAG_ITER_LOG

pytestmark = pytest.mark.gpu
METHODS = {"ivox": FLS_P2PLANE_IVOX, "ndt": FLS_NDT, "icp": FLS_ICP_P2P, "kd": FLS_P2PLANE_KNN}
KINDS = ["converges", "max_iterations", "30_points"]
MAX_IT = 2


def _setup(scene16, method, kind, flags=0):
    from funny_lidar_slam_b200.registration import Registration
    extra = dict(max_iterations=MAX_IT, position_converge_thres=0.0, rotation_converge_thres=0.0) if kind == "max_iterations" else {}
    g = Registration(default_config(method, flags=flags, **extra))
    g.AddCloudToLocalMap([scene16["map"]])
    scan = scene16["scan"][:30].copy() if kind == "30_points" else scene16["scan"]
    return g, scan


def _match(g, method, scan, guess):
    from funny_lidar_slam_b200.registration import PointcloudCluster
    cl = PointcloudCluster(ordered_cloud=scan) if method in (FLS_NDT, FLS_ICP_P2P) else PointcloudCluster(planar_cloud=scan)
    T = guess.copy()
    ok = g.Match(cl, T)
    return ok, T


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("name", list(METHODS))
def test_device_result_buffer_equals_host_result(scene16, name, kind):
    import torch

    from funny_lidar_slam_b200 import parallel
    method = METHODS[name]
    g, scan = _setup(scene16, method, kind)
    buf = torch.full((parallel.RESULT_LEN,), -7.0, dtype=torch.float64, device="cuda:0")
    g.set_result_buffer_device(buf.data_ptr(), 1)
    ok, T = _match(g, method, scan, scene16["guess"])
    it = g.last_stats.iterations
    T_dev, ok_dev, it_dev = parallel.unpack_result(buf.cpu().numpy())
    g.set_result_buffer_device(0, 0)
    assert np.array_equal(T_dev, T) and ok_dev == ok and it_dev == it, (T_dev, T, ok_dev, ok, it_dev, it)
    if kind == "max_iterations":
        assert it == MAX_IT
    if kind == "30_points" and method in (FLS_P2PLANE_IVOX, FLS_P2PLANE_KNN):
        assert not ok  # fewer than 50 valid planar points


@pytest.mark.parametrize("kind", KINDS)
def test_ivox_single_match_is_bitwise_repeatable(scene16, kind):
    g, scan = _setup(scene16, FLS_P2PLANE_IVOX, kind, flags=FLS_FLAG_ITER_LOG)
    runs = []
    for _ in range(3):
        ok, T = _match(g, FLS_P2PLANE_IVOX, scan, scene16["guess"])
        st = g.last_stats
        runs.append((ok, T, st.iterations, st.n_valid, g.iter_log()))
    ok0, T0, it0, nv0, log0 = runs[0]
    assert len(log0) == it0
    if kind == "max_iterations":
        assert it0 == MAX_IT
    if kind == "30_points":
        assert not ok0
    for ok, T, it, nv, log in runs[1:]:
        assert ok == ok0 and np.array_equal(T, T0) and it == it0 and nv == nv0
        for a, b in zip(log, log0):
            assert a["n_valid"] == b["n_valid"] and a["sum_residual"] == b["sum_residual"]
            assert np.array_equal(a["H"], b["H"]) and np.array_equal(a["g"], b["g"]) and np.array_equal(a["dx"], b["dx"])
