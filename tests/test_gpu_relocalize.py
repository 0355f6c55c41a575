"""fls_relocalize on the device, for LOAM-iVox and NDT in localization mode: the degenerate search is Localization::Init's single Match,
the coarse scores and the selection match the reference (tests/reloc_ref.py), every refined pose is the Match it replaces, a guess
metres and tens of degrees off is recovered within 0.05 m / 0.5 degrees, and the call is deterministic and leaves the handle as a
Match would."""
import numpy as np
import pytest

from funny_lidar_slam_b200 import _abi, synth
from funny_lidar_slam_b200._lib import FlsError
from funny_lidar_slam_b200.registration import PointcloudCluster, Registration, voxel_grid
from tests import reloc_ref

pytestmark = pytest.mark.gpu

FLT_MAX = float(np.finfo(np.float32).max)
METHODS = [_abi.FLS_P2PLANE_IVOX, _abi.FLS_NDT]


def _rz(deg):
    a = np.deg2rad(deg)
    R = np.eye(4)
    R[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
    return R


@pytest.fixture(scope="module")
def scene():
    world = synth.make_world(seed=1234)
    T_true = synth.trajectory(40)[10]
    mp = synth.make_surface_map(world, spacing=0.5, seed=11)
    keep = np.all(np.abs(mp[:, :2] - T_true[:2, 3].astype(np.float32)) <= 40.0, axis=1)
    scan = synth.make_scan(world, T_true, "vlp16", seed=21)["points"]
    return dict(map=np.ascontiguousarray(mp[keep]), scan=scan, T_true=T_true, guess=_off(T_true, 3.3, -2.6, 33.0))


def _off(T, dx, dy, yaw_deg):
    """T moved by (dx, dy) metres and turned by yaw_deg about the vertical"""
    out = T.copy()
    out[:3, :3] = _rz(yaw_deg)[:3, :3] @ T[:3, :3]
    out[:3, 3] += [dx, dy, 0.0]
    return out


def _handle(scene, method, **kw):
    g = Registration(_abi.default_config(method, flags=_abi.FLS_FLAG_ITER_LOG, **kw))
    g.AddCloudToLocalMap([scene["map"]])
    return g


def _cluster(method, scan):
    return PointcloudCluster(ordered_cloud=scan) if method == _abi.FLS_NDT else PointcloudCluster(planar_cloud=scan)


def _fit_cloud(scene, method):
    return voxel_grid(scene["map"], 0.2) if method == _abi.FLS_NDT else scene["map"]  # the cloud GetFitnessScore searches


@pytest.mark.parametrize("method", METHODS)
def test_degenerate_search_is_the_single_match(scene, method):
    g = _handle(scene, method)
    guess = synth.perturb_pose(scene["T_true"], seed=3, dpos=0.3, drot_deg=2.0)
    r = g.relocalize(scene["scan"], guess, xy_radius=0.0, yaw_range=0.0, n_refine=1)
    assert r.n_hypotheses == 1 and r.n_refined == 1 and r.best_hypothesis == 0
    iters = len(g.iter_log(0))
    T = guess.copy()
    ok = g.Match(_cluster(method, scene["scan"]), T)
    assert np.array_equal(r.T, T) and r.converged == ok and iters == g.last_stats.iterations
    assert r.fitness == g.GetFitnessScore(2.0)
    assert r.accepted == (ok and r.fitness < 1.0)


@pytest.mark.parametrize("method", METHODS)
def test_coarse_scores_selection_and_refinement_match_the_reference(scene, method):
    g = _handle(scene, method)
    cfg = dict(xy_radius=2.0, xy_step=1.0, yaw_range=np.deg2rad(30.0), yaw_step=np.deg2rad(10.0), coarse_leaf=1.0, max_range=2.0, n_refine=8)
    H = reloc_ref.hypotheses(scene["guess"], cfg["xy_radius"], cfg["xy_step"], cfg["yaw_range"], cfg["yaw_step"])
    r = g.relocalize(scene["scan"], scene["guess"], coarse_scores=len(H), **cfg)
    assert r.n_hypotheses == len(H) == 175
    iters = [len(g.iter_log(k)) for k in range(r.n_refined)]
    coarse = voxel_grid(scene["scan"], 1.0)
    ref = reloc_ref.coarse_scores(_fit_cloud(scene, method), coarse, H, 2.0)
    decided = ref.gate_ulps > 4.0
    print(f"coarse: {len(coarse)} points, {int((~decided).sum())} of {len(H)} hypotheses within 4 ulps of the gate (reported, not asserted)")
    rel = np.abs(r.coarse_scores - ref.score) / ref.score
    assert np.all(rel[decided] <= 1e-9), rel[decided].max()
    # selection, wherever the score gaps on both sides of a rank decide it
    order, gaps = reloc_ref.select(r.coarse_scores, r.n_refined)
    ref_order, ref_gaps = reloc_ref.select(ref.score, r.n_refined)
    assert list(r.refined_index) == list(order)
    for k in range(r.n_refined):
        tol = 1e-9 * ref.score[ref_order[k]]
        if ref_gaps[k] > tol and (k == 0 or ref_gaps[k - 1] > tol):
            assert r.refined_index[k] == ref_order[k], k
    # refinement: each refined pose is the Match from its start pose, and its fitness the GetFitnessScore after it
    for k in range(r.n_refined):
        T = H[r.refined_index[k]].copy()
        ok = g.Match(_cluster(method, scene["scan"]), T)
        assert np.max(np.abs(T - r.refined_T[k])) <= 1e-9, k
        assert ok == r.refined_converged[k] and g.last_stats.iterations == iters[k], k
        assert g.GetFitnessScore(2.0) == r.refined_fitness[k], k
    # the choice rule
    conv = np.flatnonzero(r.refined_converged)
    pool = conv if len(conv) else np.arange(r.n_refined)
    best = pool[np.lexsort((pool, r.refined_fitness[pool]))[0]]
    assert r.best_rank == best and r.fitness == r.refined_fitness[best] and np.array_equal(r.T, r.refined_T[best])


# (plug-in, guess offset, grid step).  The step is what each plug-in's Match converges from: LOAM-iVox comes in from about a metre
# and ten degrees, NDT (1 m voxels, outlier gate 5.0) only from decimetres, so its search uses 0.5 m and 5 degrees.
RECOVERY = [(_abi.FLS_P2PLANE_IVOX, (3.3, -2.6, 33.0), 1.0, 10.0), (_abi.FLS_NDT, (5.4, 4.3, 95.0), 0.5, 5.0)]


@pytest.mark.parametrize("method,offset,step,yaw_step", RECOVERY)
def test_recovers_a_pose_metres_and_degrees_off(scene, method, offset, step, yaw_step):
    g = _handle(scene, method)
    guess = _off(scene["T_true"], *offset)
    T = guess.copy()
    ok = g.Match(_cluster(method, scene["scan"]), T)
    plain = ok and g.GetFitnessScore(2.0) < 1.0
    dt0, dr0 = synth.pose_error(T, scene["T_true"])
    r = g.relocalize(scene["scan"], guess, xy_radius=8.0, xy_step=step, yaw_range=np.pi, yaw_step=np.deg2rad(yaw_step), n_refine=64)
    dt, dr = synth.pose_error(r.T, scene["T_true"])
    print(f"plain Match: accepted={plain} error {dt0:.2f} m {np.rad2deg(dr0):.1f} deg | relocalize: {r.n_hypotheses} hypotheses, rank "
          f"{r.best_rank}, fitness {r.fitness:.4f}, error {dt:.4f} m {np.rad2deg(dr):.3f} deg, {r.host_waits} waits, {r.gpu_launches} launches")
    # Init's single Match from this guess lands metres away.  In these scenes upstream's rule (converged, fitness < 1.0) accepts that
    # wrong pose (its fitness is ~0.12-0.17: GetFitnessScore averages inliers only, and the ground always has some), so the test holds
    # the plain Match to being wrong, whether accepted or not, and the relocalized pose to being right.
    assert dt0 > 1.0
    assert r.accepted and r.converged and r.fitness < 1.0
    assert dt < 0.05 and np.rad2deg(dr) < 0.5
    # the handle afterwards: fls_fitness scores the chosen pose, and a Match from it converges
    assert g.GetFitnessScore(2.0) == r.fitness
    T2 = r.T.copy()
    assert g.Match(_cluster(method, scene["scan"]), T2)


@pytest.mark.parametrize("method", METHODS)
def test_deterministic_and_device_entry_equals_host(scene, method):
    import torch
    g = _handle(scene, method)
    kw = dict(xy_radius=3.0, xy_step=1.0, yaw_range=np.pi, yaw_step=np.deg2rad(15.0), n_refine=16)
    a = g.relocalize(scene["scan"], scene["guess"], coarse_scores=1 << 20, **kw)
    b = g.relocalize(scene["scan"], scene["guess"], coarse_scores=1 << 20, **kw)
    d = torch.from_numpy(scene["scan"]).cuda()
    torch.cuda.synchronize()
    c = g.relocalize_device(d.data_ptr(), d.shape[0], scene["guess"], coarse_scores=1 << 20, **kw)
    assert len(a.coarse_scores) == a.n_hypotheses == 7 * 7 * 24
    # the coarse stage is bitwise reproducible; the refinement is the batch Match, whose sums may run in another order from call to
    # call (its bar against single Matches: poses 1e-9, converged equal)
    for o in (b, c):
        assert o.coarse_scores.tobytes() == a.coarse_scores.tobytes()
        assert list(o.refined_index) == list(a.refined_index) and np.array_equal(o.refined_converged, a.refined_converged)
        assert np.max(np.abs(o.refined_T - a.refined_T)) <= 1e-9
        assert (o.best_hypothesis, o.converged, o.accepted) == (a.best_hypothesis, a.converged, a.accepted)
        assert np.max(np.abs(o.T - a.T)) <= 1e-9 and abs(o.fitness - a.fitness) <= 1e-5 * a.fitness


@pytest.mark.parametrize("method", METHODS)
def test_edges_no_inliers_and_empty_scan(scene, method):
    g = _handle(scene, method)
    far = scene["guess"].copy()
    far[:3, 3] += [1000.0, 0.0, 0.0]
    r = g.relocalize(scene["scan"], far, xy_radius=1.0, yaw_range=0.0, n_refine=4, coarse_scores=9)
    assert np.all(r.coarse_scores == np.float32(2.0))  # every point counted at the gate
    assert list(r.refined_index) == [0, 1, 2, 3]
    assert r.fitness == FLT_MAX and not r.accepted
    e = g.relocalize(np.zeros((0, 4), np.float32), scene["guess"], n_refine=4)
    assert e.fitness == FLT_MAX and not e.accepted and e.n_refined == 0 and np.array_equal(e.T, scene["guess"])
    assert g.GetFitnessScore(2.0) == FLT_MAX


def test_unsupported_plugins_and_modes_leave_the_handle_untouched(scene):
    for method in (_abi.FLS_ICP_P2P, _abi.FLS_P2PLANE_KNN):
        g = _handle(scene, method)
        cl = PointcloudCluster(ordered_cloud=scene["scan"]) if method == _abi.FLS_ICP_P2P else PointcloudCluster(planar_cloud=scene["scan"])
        g0 = synth.perturb_pose(scene["T_true"], seed=5, dpos=0.2, drot_deg=1.0)
        Ta = g0.copy()
        g.Match(cl, Ta)
        with pytest.raises(FlsError) as ei:
            g.relocalize(scene["scan"], g0)
        assert ei.value.status == _abi.FLS_ERR_UNSUPPORTED
        Tb = g0.copy()
        g.Match(cl, Tb)
        assert np.array_equal(Ta, Tb)
    for method in METHODS:  # mapping mode: a Match after the refused call is the Match of a handle that never saw it
        a, b = (_handle(scene, method, localization_mode=0) for _ in range(2))
        with pytest.raises(FlsError) as ei:
            a.relocalize(scene["scan"], scene["guess"])
        assert ei.value.status == _abi.FLS_ERR_UNSUPPORTED
        g0 = synth.perturb_pose(scene["T_true"], seed=6, dpos=0.2, drot_deg=1.0)
        Ta, Tb = g0.copy(), g0.copy()
        oka, okb = a.Match(_cluster(method, scene["scan"]), Ta), b.Match(_cluster(method, scene["scan"]), Tb)
        assert oka == okb and np.array_equal(Ta, Tb)
        assert a.map_info().n_voxels == b.map_info().n_voxels
    g = Registration(_abi.default_config(_abi.FLS_NDT))
    with pytest.raises(FlsError) as ei:
        g.relocalize(scene["scan"], scene["guess"])
    assert ei.value.status == _abi.FLS_ERR_NO_MAP
    g = _handle(scene, _abi.FLS_P2PLANE_IVOX)
    for bad in (dict(n_refine=0), dict(n_refine=65), dict(xy_step=0.0), dict(coarse_leaf=float("nan")), dict(max_range=-1.0),
                dict(xy_radius=600.0)):
        with pytest.raises(FlsError) as ei:
            g.relocalize(scene["scan"], scene["guess"], **bad)
        assert ei.value.status == _abi.FLS_ERR_INVALID_ARG, bad
