"""GPU: iteration 0 of the kd-tree LOAM kernel (K5: LoamPointToPlaneKdtree and LoamFull) against the brute-force reference of
tests/loam_kd_ref.py (proven against the oracle by tests/test_oracle_loam_kd_edges.py) on the edge scenes of tests/loam_kd_scenes.py:
the ring search and its full-scan fallback, lanes and ties, tiny maps, LoamFull's search gate, the corner term, iteration 1 of the
stale-record scene, and the device-resident route."""
import numpy as np
import pytest

from tests import loam_kd_ref, loam_kd_scenes
from tests.test_oracle_loam_kd_edges import SCENES, reference

pytestmark = pytest.mark.gpu


def _gpu(s, max_iterations=1):
    from funny_lidar_slam_b200.registration import Registration
    g = Registration(s.config(max_iterations))
    g.AddCloudToLocalMap([s.planar_map, s.corner_map] if s.full else [s.planar_map])
    return g


def _match(g, s):
    from funny_lidar_slam_b200.registration import PointcloudCluster
    T = s.T.copy()
    g.Match(PointcloudCluster(planar_cloud=s.planar, corner_cloud=s.corner if s.full else None), T)
    return g.iter_log()


@pytest.mark.parametrize("name", list(SCENES))
def test_first_pass(name):
    s = SCENES[name]
    ref = reference(s)
    loam_kd_ref.assert_sensitive(ref)
    lg = _match(_gpu(s), s)
    loam_kd_ref.assert_matches(lg[0], ref)


def test_stale_records_at_iteration_1():
    """Iteration 1 at the GPU's own updated pose: the rejected corner and planar points contribute their iteration-0 records, each
    in its own class; every other point is evaluated again."""
    s = loam_kd_scenes.full_stale()
    lg = _match(_gpu(s, 2), s)
    r0 = reference(s)
    loam_kd_ref.assert_matches(lg[0], r0)
    r1 = reference(s, T=loam_kd_ref.next_pose(s.T, lg[0]["dx"]), prev=r0, q_ulps=1)
    assert [(t.cls, t.i) for t in r1.terms if t.stale] == [("corner", 0), ("planar", len(s.planar) - 1)]
    loam_kd_ref.assert_sensitive(r1)
    loam_kd_ref.assert_matches(lg[1], r1)


def test_cluster_device_route_equals_host_route():
    """fls_match_cluster_device on device-resident clouds gives the host route's iteration-0 log and pose, bit for bit."""
    import torch
    s = SCENES["full_corners"]
    host = _match(_gpu(s), s)[0]
    g = _gpu(s)
    d_p = torch.from_numpy(np.ascontiguousarray(s.planar, np.float32)).cuda()
    d_c = torch.from_numpy(np.ascontiguousarray(s.corner, np.float32)).cuda()
    T = s.T.copy()
    g.match_cluster_device(0, 0, d_p.data_ptr(), len(s.planar), d_c.data_ptr(), len(s.corner), T)
    dev = g.iter_log()[0]
    assert dev["n_valid"] == host["n_valid"] and dev["sum_residual"] == host["sum_residual"]
    assert np.array_equal(dev["H"], host["H"]) and np.array_equal(dev["g"], host["g"])
    loam_kd_ref.assert_matches(dev, reference(s))
