"""GPU: the IncrementalNDT map, the NDT and ICP first passes and GetFitnessScore against the brute-force references of
tests/ndt_ref.py and tests/icp_ref.py (proven against the oracle by tests/test_oracle_ndt_icp_edges.py) on the edge scenes of
tests/ndt_icp_scenes.py; batched NDT Match per scan, including a batch large enough to take the sub-grid scaling branch."""
import numpy as np
import pytest

from funny_lidar_slam_b200 import FLS_ICP_P2P, FLS_NDT, FLS_P2PLANE_IVOX, FLS_P2PLANE_KNN, default_config
from funny_lidar_slam_b200._abi import FLS_ERR_CAPACITY
from oracle import pyoracle as orc
from tests import icp_ref, ndt_icp_scenes, ndt_ref

pytestmark = pytest.mark.gpu
NDT = {s.name: s for s in ndt_icp_scenes.ndt_scenes()}
ICP = {s.name: s for s in ndt_icp_scenes.icp_scenes()}
NDT_BLOCK_CTAS = 132 * 4 * 512  # filtered points past which no H100 holds one 512-thread CTA per 512 points of every scan


def _gpu(cfg):
    from funny_lidar_slam_b200.registration import Registration
    return Registration(cfg)


def _cluster(scan):
    from funny_lidar_slam_b200.registration import PointcloudCluster
    return PointcloudCluster(ordered_cloud=scan)


def _reference(s):
    ref = ndt_ref.NdtRef(s.voxel, s.min_pts, s.max_pts, s.capacity, s.leaf, s.localization)
    for c in s.calls:
        ref.add_cloud(c)
    return ref


def test_ndt_map_dump_follows_the_stream():
    """fls_get_ndt_voxels after every AddCloudToLocalMap call of the mapping stream: keys, estimated, num_points and carry_count
    exact; mu and information within the reference's bounds — carry, first estimate, merge, clamp, freeze and an LRU eviction whose
    victim is created again in the same call."""
    s = ndt_icp_scenes.ndt_stream()
    g = _gpu(s.config())
    ref = ndt_ref.NdtRef(s.voxel, s.min_pts, s.max_pts, s.capacity, s.leaf, s.localization)
    for k, c in enumerate(s.calls):
        g.AddCloudToLocalMap([c])
        ref.add_cloud(c)
        got = g.ndt_voxels()
        assert g.map_info().n_voxels == len(ref.data), k
        ndt_ref.assert_dump_matches(got, ref.dump())


@pytest.mark.parametrize("name", list(NDT))
def test_ndt_map_dump_and_first_pass(name):
    s = NDT[name]
    g = _gpu(s.config())
    for c in s.calls:
        g.AddCloudToLocalMap([c])
    ref = _reference(s)
    ndt_ref.assert_dump_matches(g.ndt_voxels(), ref.dump())
    p = ndt_ref.ndt_pass(ref, s.scan, s.T, s.thres)
    ndt_ref.assert_gates_clear(p)
    ndt_ref.assert_sensitive(p)
    T = s.T.copy()
    g.Match(_cluster(s.scan), T)
    lg = g.iter_log()[0]
    ndt_ref.assert_matches(lg["H"], lg["g"], lg["n_valid"], p)


def test_ndt_capacity_overflow_in_one_call_is_an_error():
    """A single AddCloudToLocalMap call that creates more voxels than ndt_capacity: upstream keeps evicting (and then reads an erased
    voxel); the library reports FLS_ERR_CAPACITY."""
    from funny_lidar_slam_b200._lib import FlsError
    s = ndt_icp_scenes.ndt_stream(capacity=8)
    g = _gpu(s.config())
    g.AddCloudToLocalMap([s.calls[0]])
    with pytest.raises(FlsError) as e:
        g.AddCloudToLocalMap([s.calls[5]])
    assert e.value.status == FLS_ERR_CAPACITY


def _batch_scans(rng, B, big=False):
    """B scans around the ndt_axes map: scene scans, empty and one-point scans, and (big) 5000 filtered points per scan."""
    base = [NDT["ndt_axes"].scan, NDT["ndt_chi_single"].scan]
    scans = []
    for k in range(B):
        if B == 64 and k % 16 == 5:
            scans.append(np.zeros((0, 4), np.float32))
        elif B == 64 and k % 16 == 6:
            scans.append(base[0][:1].copy())
        elif big:
            pts = np.zeros((5000, 4), np.float32)
            pts[:, :3] = rng.uniform(-2.0, 2.0, (5000, 3))
            scans.append(pts)
        else:
            scans.append(base[k % 2].copy())
    return scans


@pytest.mark.parametrize("B,big", [(2, False), (9, False), (64, False), (64, True)], ids=["b2", "b9", "b64", "b64_scaled"])
def test_ndt_batch_iteration0_per_scan(B, big):
    """Iteration 0 of every scan of a batch equals its own single Match to 1e-9, and the reference where the scan is a scene scan.
    The big batch holds more filtered points than 132 SMs x 4 CTAs x 512 threads, so its sub-grids are provably scaled down."""
    s = NDT["ndt_axes"]
    cfg = s.config()
    g = _gpu(cfg)
    g.AddCloudToLocalMap([s.calls[0]])
    ref = _reference(s)
    rng = np.random.default_rng(100 + B)
    scans = _batch_scans(rng, B, big)
    n_f = [len(orc.voxel_grid(sc, s.leaf)) if len(sc) else 0 for sc in scans]
    if big:
        assert sum(n_f) > NDT_BLOCK_CTAS
    Ts = np.stack([np.eye(4)] * B)
    g.match_batch(scans, Ts)
    logs = [g.iter_log(k)[0] for k in range(B)]
    for k in range(B):
        one = dict(H=np.zeros((6, 6)), g=np.zeros(6), n_valid=0)  # an empty scan: nothing to sum
        if len(scans[k]):
            g.Match(_cluster(scans[k]), np.eye(4))
            one = g.iter_log()[0]
        assert logs[k]["n_valid"] == one["n_valid"], k
        scale = max(1.0, float(np.max(np.abs(one["H"]))))
        assert np.max(np.abs(logs[k]["H"] - one["H"])) <= 1e-9 * scale, k
        assert np.max(np.abs(logs[k]["g"] - one["g"])) <= 1e-9 * max(1.0, float(np.max(np.abs(one["g"])))), k
        if not big and len(scans[k]) > 1:
            p = ndt_ref.ndt_pass(ref, scans[k], np.eye(4), s.thres)
            ndt_ref.assert_matches(logs[k]["H"], logs[k]["g"], logs[k]["n_valid"], p)


@pytest.mark.parametrize("name", list(ICP))
def test_icp_first_pass(name):
    s = ICP[name]
    g = _gpu(s.config())
    g.AddCloudToLocalMap([s.map])
    T = s.T.copy()
    g.Match(_cluster(s.scan), T)
    lg = g.iter_log()[0]
    p = icp_ref.icp_pass(s.map, s.scan, s.T, s.max_corr, 0.01, 0.01)
    icp_ref.assert_sensitive(p)
    if not s.ties:
        icp_ref.assert_gates_clear(p, tie_ok=False)
        icp_ref.assert_matches(lg["H"], lg["g"], lg["n_valid"], p)
        return
    # a tie: the GPU's neighbour must be one of the tied points; g[0:3] = -(q - m) names it
    assert lg["n_valid"] == p.n_valid == 1
    mp = orc.voxel_grid(s.map, 0.01)
    m = p.q[0].astype(np.float64) + np.asarray(lg["g"][:3])
    hit = [j for j in p.nn.ties[0] if np.allclose(mp[j, :3], m, atol=1e-9)]
    assert len(hit) == 1, (m, mp[p.nn.ties[0], :3])


def _fitness_case(method):
    mp, sc = ndt_icp_scenes.fitness_scene()
    scan = np.vstack([sc] * 4)  # Match refuses ten points or fewer before filtering
    if method == FLS_ICP_P2P:
        cfg = default_config(method, max_iterations=1, icp_max_correspond_distance=0.1, source_cloud_filter_size=0.01, map_cloud_filter_size=0.01)
        return cfg, mp, scan, orc.voxel_grid(mp, 0.01), orc.voxel_grid(scan, 0.01)
    if method == FLS_NDT:  # no effective point at all: Match stops at iteration 0 with the pose untouched
        cfg = default_config(method, max_iterations=1, source_cloud_filter_size=0.01, ndt_min_effective_pts=1 << 30)
        return cfg, mp, scan, orc.voxel_grid(mp, 0.01), orc.voxel_grid(scan, 0.01)
    # the LOAM plug-ins: a planar patch matched at its own pose; the fitness tree holds the map (filtered for the kd-tree plug-in)
    rng = np.random.default_rng(31)
    pm = np.zeros((400, 4), np.float32)
    pm[:, :2] = rng.uniform(-3, 3, (400, 2))
    pm[:, 2] = rng.normal(0, 0.01, 400)
    ps = pm[::7].copy()
    ps[:, :3] += np.float32(0.02)
    cfg = default_config(method, max_iterations=1, map_cloud_filter_size=0.01)
    tree = orc.voxel_grid(pm, 0.01) if method == FLS_P2PLANE_KNN else pm
    return cfg, pm, ps, tree, ps


@pytest.mark.parametrize("method", [FLS_ICP_P2P, FLS_NDT, FLS_P2PLANE_KNN, FLS_P2PLANE_IVOX], ids=["icp", "ndt", "p2plane_knn", "loam_ivox"])
def test_fitness_equals_brute_force(method):
    from funny_lidar_slam_b200.registration import PointcloudCluster
    cfg, mp, scan, tree, src = _fitness_case(method)
    g = _gpu(cfg)
    g.AddCloudToLocalMap([mp])
    T = np.eye(4)
    cl = PointcloudCluster(ordered_cloud=scan) if method in (FLS_ICP_P2P, FLS_NDT) else PointcloudCluster(planar_cloud=scan)
    g.Match(cl, T)
    exact = method in (FLS_ICP_P2P, FLS_NDT)
    if exact:
        assert np.array_equal(T, np.eye(4))  # nothing corresponds: the pose stays and the fitness gates are exact
    for r in (1.0, 2.0, 0.5):
        want, _, gate = icp_ref.fitness(tree, src, T, r)
        if not exact:  # a moved pose rounds the query in another order: no inlier may sit within rounding of the gate
            assert np.all(np.abs(gate) > 64), r
        got = g.GetFitnessScore(r)
        assert abs(got - want) <= 1e-6 * max(1.0, abs(want)), (r, got, want)
