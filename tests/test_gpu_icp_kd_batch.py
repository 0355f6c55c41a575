"""GPU: fls_match_batch for IcpOptimized and LoamPointToPlaneKdtree — one cooperative launch, a sub-grid and a Gauss-Newton loop per
scan.  Every scan of a batch against its own single Match, the CPU oracle and the brute-force references of tests/icp_ref.py and
tests/loam_kd_ref.py; sub-grid sizing on both sides of the scale-down; the kd-tree plug-in's per-scan stale records; the refusals and
the per-scan outputs."""
import numpy as np
import pytest

from funny_lidar_slam_b200 import FLS_ICP_P2P, FLS_LOAM_FULL, FLS_P2PLANE_KNN, default_config, synth
from funny_lidar_slam_b200._abi import (FLS_ERR_NO_MAP, FLS_ERR_TOO_FEW_POINTS, FLS_ERR_UNSUPPORTED, FLS_FLAG_ITER_LOG, FLS_FLAG_PROFILE)
from oracle import pyoracle as orc
from tests import icp_ref, loam_kd_ref, loam_kd_scenes, ndt_icp_scenes
from tests.ndt_icp_scenes import _cloud
from tests.test_oracle_loam_kd_edges import reference as kd_reference

pytestmark = pytest.mark.gpu
POS_TOL, ROT_TOL = 1e-4, 1e-4
METHODS = [FLS_ICP_P2P, FLS_P2PLANE_KNN]
IDS = ["icp", "kd"]
PER_CTA = {FLS_ICP_P2P: 64, FLS_P2PLANE_KNN: 32}  # queries per CTA of the batch kernels (512 / 8 and 256 / 8 lanes)
BLOCK = {FLS_ICP_P2P: 512, FLS_P2PLANE_KNN: 256}
EPS = np.finfo(np.float64).eps


def _gpu(cfg):
    from funny_lidar_slam_b200.registration import Registration
    return Registration(cfg)


def _cluster(method, scan):
    from funny_lidar_slam_b200.registration import PointcloudCluster
    return PointcloudCluster(ordered_cloud=scan) if method == FLS_ICP_P2P else PointcloudCluster(planar_cloud=scan)


def _single(g, method, scan, T0):
    """One fls_match of `scan` from T0: (converged, T, stats, log)."""
    T = np.array(T0, np.float64, copy=True)
    ok = g.Match(_cluster(method, scan), T)
    return ok, T, g.last_stats, g.iter_log()


def _n_source(method, cfg, scan):
    """Points the Gauss-Newton loop runs over: the voxel-filtered scan (ICP) or the planar cloud as given (kd-tree)."""
    if method == FLS_ICP_P2P:
        return len(orc.voxel_grid(scan, cfg.source_cloud_filter_size)) if len(scan) else 0
    return len(scan)


def _assert_sum_bound(a, b, n, k):
    """Iteration logs a and b sum the same terms in another order.  Two fp64 sums of n terms differ by at most 2 n eps sum|term|
    (recursive summation), each term a few dozen flops (64 n eps in all).  H = sum J^T J, so Cauchy-Schwarz bounds sum|J_a J_b| by
    sqrt(H_aa H_bb) and sum|J_a r| by sqrt(H_aa) sqrt(sum r^2) <= sqrt(H_aa) sum|r|, and sum|r| is the logged sum_residual (ICP:
    the error norms, kd-tree: the plane distances)."""
    assert a["n_valid"] == b["n_valid"], k
    dH = np.sqrt(np.abs(np.diag(b["H"])))
    tol = 64 * max(n, 1) * EPS
    assert np.all(np.abs(a["H"] - b["H"]) <= tol * np.outer(dH, dH)), k
    assert np.all(np.abs(a["g"] - b["g"]) <= tol * dH * max(b["sum_residual"], 0.0)), k


def _assert_single(oks, Ts, sts, logs, k, one, n):
    ok1, T1, st1, lg1 = one
    assert bool(oks[k]) == ok1, k
    assert sts[k].iterations == st1.iterations and sts[k].n_valid == st1.n_valid and sts[k].n_source == st1.n_source, k
    dt, dr = synth.pose_error(Ts[k], T1)
    assert dt < 1e-9 and dr < 1e-9, (k, dt, dr)
    assert len(logs[k]) == len(lg1), k
    if len(lg1):
        _assert_sum_bound(logs[k][0], lg1[0], n, k)


# ---- 1. synthetic batches against single Matches and the oracle ---------------------------------------------------------------
@pytest.mark.parametrize("method", METHODS, ids=IDS)
def test_batch_equals_single_and_oracle(world, traj, scene64, method):
    cfg = default_config(method, flags=FLS_FLAG_ITER_LOG)
    g, o = _gpu(cfg), orc.Registration(cfg)
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
        one = _single(g, method, scans[k], guesses[k])
        _assert_single(oks, Ts, sts, logs, k, one, _n_source(method, cfg, scans[k]))
        ok_o, To, st_o = o.match(scans[k], guesses[k])
        assert bool(oks[k]) == ok_o and sts[k].iterations == st_o.iterations and sts[k].n_valid == st_o.n_valid, k
        dt, dr = synth.pose_error(Ts[k], To)
        assert dt < POS_TOL and dr < ROT_TOL, (k, dt, dr)


# ---- 2. batch sizes: both sides of the sub-grid scale-down, B = 1 is the single Match, device scans = host scans -----------------
def _sized_scans(world, traj, B, method):
    """B 16-line scans with perturbed guesses; the batch of two is cut to 1500 points per scan so that it provably fits."""
    scans, guesses = [], []
    for k in range(B):
        sc = synth.make_scan(world, traj[2 + k % 8], "vlp16", seed=40 + k % 8)["points"]
        scans.append(sc[:1500].copy() if B == 2 else sc)
        guesses.append(synth.perturb_pose(traj[2 + k % 8], seed=400 + k, dpos=0.1, drot_deg=1.0))
    return scans, np.stack(guesses)


@pytest.mark.parametrize("B", [1, 2, 9, 64])
@pytest.mark.parametrize("method", METHODS, ids=IDS)
def test_batch_sizes(world, traj, scene16, method, B):
    """Every scan equals its single Match; which sizing branch a batch takes follows from its point counts: it fits when the CTAs it
    needs are at most the SM count (at least one CTA per SM is co-resident) and is scaled down when they exceed what 2048 threads per
    SM can hold.  A 64-scan ICP batch of 16-line scans needs about 71 CTAs per scan."""
    import torch
    cfg = default_config(method, flags=FLS_FLAG_ITER_LOG)
    g = _gpu(cfg)
    g.AddCloudToLocalMap([scene16["map"]])
    scans, guesses = _sized_scans(world, traj, B, method)
    ns = [_n_source(method, cfg, s) for s in scans]
    need = sum(max(1, -(-n // PER_CTA[method])) for n in ns)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if B == 2:
        assert need <= sms, need  # unscaled
    if B >= 9:
        assert need > sms * (2048 // BLOCK[method]), need  # scaled down
    oks, Ts = g.match_batch(scans, guesses)
    sts = g.last_batch_stats
    logs = [g.iter_log(k) for k in range(B)]
    d = [torch.from_numpy(np.ascontiguousarray(s)).cuda() for s in scans]
    oks_d, Ts_d = g.match_batch_device([t.data_ptr() for t in d], [len(s) for s in scans], guesses)
    assert np.array_equal(oks, oks_d) and np.array_equal(Ts, Ts_d)
    for k in range(B):
        one = _single(g, method, scans[k], guesses[k])
        _assert_single(oks, Ts, sts, logs, k, one, ns[k])
        if B == 1:  # the same path: bit for bit
            assert np.array_equal(Ts[0], one[1])
            assert all(np.array_equal(a["H"], b["H"]) and np.array_equal(a["g"], b["g"]) for a, b in zip(logs[0], one[3]))


# ---- 3. edge scenes at iteration 0, per scan of a batch -----------------------------------------------------------------------
ICP = {s.name: s for s in ndt_icp_scenes.icp_scenes()}
KD = {s.name: s for s in loam_kd_scenes.kd_scenes()}
SHIFT = np.array([0.125, -0.0625, 0.03125])  # dyadic: the shifted pose is exact in fp32


def _shifted(T):
    T = np.array(T, np.float64, copy=True)
    T[:3, 3] += SHIFT
    return T


@pytest.mark.parametrize("name", list(ICP))
def test_icp_edge_scenes_per_scan(name):
    """One scene's map; the batch holds its scan as designed, two subsets (Match refuses ten points or fewer, so each keeps more)
    and the scan at a shifted pose, each checked against icp_ref at its own pose.  Ties decide only n_valid."""
    s = ICP[name]
    g = _gpu(s.config())
    g.AddCloudToLocalMap([s.map])
    n = len(s.scan)
    scans = [s.scan, s.scan[: max(11, n // 2)].copy(), s.scan[-max(11, (2 * n) // 3):].copy(), s.scan]
    Ts = np.stack([s.T, s.T, s.T, _shifted(s.T)])
    g.match_batch(scans, Ts)
    logs = [g.iter_log(k)[0] for k in range(len(scans))]
    for k, (sc, T) in enumerate(zip(scans, Ts)):
        one = _single(g, FLS_ICP_P2P, sc, T)[3][0]
        _assert_sum_bound(logs[k], one, len(sc), k)
        p = icp_ref.icp_pass(s.map, sc, T, s.max_corr, 0.01, 0.01)
        if all(len(t) <= 1 for t in p.nn.ties):
            icp_ref.assert_matches(logs[k]["H"], logs[k]["g"], logs[k]["n_valid"], p)
        else:
            assert logs[k]["n_valid"] == p.n_valid, k


def _kd_clear(ref):
    try:
        loam_kd_ref.assert_gates_clear(ref)
        return True
    except AssertionError:
        return False


@pytest.mark.parametrize("name", list(KD))
def test_kd_edge_scenes_per_scan(name):
    """One scene's map; the batch holds its planar scan as designed, its halves and the scan at a shifted pose.  Each is checked
    against loam_kd_ref at its own pose where the reference's margins decide every choice, and against its single Match always."""
    s = KD[name]
    g = _gpu(s.config())
    g.AddCloudToLocalMap([s.planar_map])
    n = len(s.planar)
    halves = [h for h in (s.planar[: (n + 1) // 2].copy(), s.planar[(n + 1) // 2:].copy()) if len(h)]
    scans = [s.planar] + halves + [s.planar]
    Ts = np.stack([s.T] * (len(scans) - 1) + [_shifted(s.T)])
    g.match_batch(scans, Ts)
    logs = [g.iter_log(k)[0] for k in range(len(scans))]
    for k, (sc, T) in enumerate(zip(scans, Ts)):
        one = _single(g, FLS_P2PLANE_KNN, sc, T)[3][0]
        _assert_sum_bound(logs[k], one, len(sc), k)
        ref = kd_reference(loam_kd_scenes.KdScene(s.name, False, s.planar_map, sc, leaf=s.leaf, plane_thres=s.plane_thres), T=T)
        if k < len(scans) - 1 or _kd_clear(ref):
            loam_kd_ref.assert_matches(logs[k], ref)


# ---- 4. stale records stay per scan (kd-tree) ---------------------------------------------------------------------------------
def kd_stale():
    """The kd-tree point-to-plane variant of loam_kd_scenes.full_stale: plane pairs 30 m out (far enough that the |p| >= 81 d^4 rule
    keeps a 0.25 m residual) move the pose about 0.25 m along +x at iteration 0.  A planar query 0.75 m beside a small patch facing
    z fits the patch at iteration 0; once moved, two points 0.4 m above and below that plane become two of its five nearest, no
    plane fits them, and iteration 1 sums its stored term [quirk 1].  The query is the last point of the scan."""
    rng = np.random.default_rng(48)
    mp, sc = [], []
    u = np.linspace(-1.2, 1.2, 9)
    gu, gv = (a.ravel() for a in np.meshgrid(u, u, indexing="ij"))
    for axis in range(3):
        for side, want in ((-1.0, 0.24 if axis == 0 else 0.01), (1.0, 0.26 if axis == 0 else -0.01)):
            a1, a2 = [b for b in range(3) if b != axis]
            P = np.zeros((len(gu), 3))
            P[:, axis], P[:, a1], P[:, a2] = side * 30.0, gu, gv
            mp.append(P)
            Q = np.zeros((6, 3))
            Q[:, axis], Q[:, a1], Q[:, a2] = side * 30.0 - want, rng.uniform(-0.8, 0.8, 6), rng.uniform(-0.8, 0.8, 6)
            sc.append(Q)
    vp = np.array([3.0, 4.0, 3.0])
    patch = vp + np.array([[0.0, 0.0, 0.0], [0.1, 0.15, 0.0], [-0.12, 0.1, 0.0], [0.05, -0.15, 0.0], [0.12, -0.05, 0.0]])
    patch[:, 2] += rng.uniform(-0.01, 0.01, 5)
    mp += [patch, vp + np.array([[1.75, 0.1, 0.4], [1.75, -0.1, -0.4]])]
    sc.append((vp + np.array([0.75, 0.0, 0.01]))[None])
    return loam_kd_scenes.KdScene("kd_stale", False, _cloud(np.vstack(mp)), _cloud(np.vstack(sc)), leaf=0.1,
                                  targets="a planar record reused at iteration 1")


def test_stale_records_stay_per_scan():
    """A scan whose last point goes stale at iteration 1 between scans without such a point: its iteration 1 equals the reference
    with the stale term, and every other scan's log equals its single Match."""
    s = kd_stale()
    g = _gpu(s.config(2))
    g.AddCloudToLocalMap([s.planar_map])
    drivers = s.planar[:-1].copy()
    scans = [drivers, s.planar, drivers[::-1].copy()]
    g.match_batch(scans, np.stack([s.T] * 3))
    logs = [g.iter_log(k) for k in range(3)]
    r0 = kd_reference(s)
    loam_kd_ref.assert_matches(logs[1][0], r0)
    r1 = kd_reference(s, T=loam_kd_ref.next_pose(s.T, logs[1][0]["dx"]), prev=r0, q_ulps=1)
    assert [(t.cls, t.i) for t in r1.terms if t.stale] == [("planar", len(s.planar) - 1)]
    loam_kd_ref.assert_sensitive(r1)
    loam_kd_ref.assert_matches(logs[1][1], r1)
    for k in (0, 2):
        one = _single(g, FLS_P2PLANE_KNN, scans[k], s.T)[3]
        assert len(logs[k]) == len(one) == 2, k
        for a, b in zip(logs[k], one):
            _assert_sum_bound(a, b, len(scans[k]), k)


# ---- 5. refusals, and no side effect ------------------------------------------------------------------------------------------
def _status(fn):
    from funny_lidar_slam_b200._lib import FlsError
    with pytest.raises(FlsError) as e:
        fn()
    return e.value.status


def _untouched(method, cfg, mp, scan, T0, g):
    """g's next Match equals that of a handle that never saw the refused call, bit for bit."""
    f = _gpu(cfg)
    f.AddCloudToLocalMap([mp])
    a, b = _single(g, method, scan, T0), _single(f, method, scan, T0)
    assert a[0] == b[0] and np.array_equal(a[1], b[1]) and a[2].iterations == b[2].iterations


@pytest.mark.parametrize("method", METHODS, ids=IDS)
def test_refusals_leave_the_handle_untouched(scene16, method):
    scan, mp, T0 = scene16["scan"], scene16["map"], scene16["guess_small"]
    cfg = default_config(method)
    g = _gpu(cfg)
    assert _status(lambda: g.match_batch([scan, scan], np.stack([T0, T0]))) == FLS_ERR_NO_MAP
    g.AddCloudToLocalMap([mp])
    _untouched(method, cfg, mp, scan, T0, g)
    if method == FLS_ICP_P2P:  # CHECK_GT(ordered_cloud_.size(), 10u), whatever the batch size
        for scans in ([scan, scan[:10]], [scan[:10]], [scan[:3], scan]):
            assert _status(lambda: g.match_batch(scans, np.stack([T0] * len(scans)))) == FLS_ERR_TOO_FEW_POINTS
            _untouched(method, cfg, mp, scan, T0, g)
    mcfg = default_config(method, localization_mode=0)
    m = _gpu(mcfg)
    m.AddCloudToLocalMap([mp])
    assert _status(lambda: m.match_batch([scan, scan], np.stack([T0, T0]))) == FLS_ERR_UNSUPPORTED
    f = _gpu(mcfg)
    f.AddCloudToLocalMap([mp])
    a, b = _single(m, method, scan, T0), _single(f, method, scan, T0)
    assert a[0] == b[0] and np.array_equal(a[1], b[1]) and m.map_info().n_points == f.map_info().n_points


def test_loam_full_has_no_batch(scene16):
    """LoamFull reads two clouds per scan: FLS_ERR_UNSUPPORTED for any batch size, and its next Match is a fresh handle's."""
    from funny_lidar_slam_b200.registration import PointcloudCluster
    scan, mp, T0 = scene16["scan"], scene16["map"], scene16["guess_small"]
    cfg = default_config(FLS_LOAM_FULL, localization_mode=1)
    g, f = _gpu(cfg), _gpu(cfg)
    for h in (g, f):
        h.AddCloudToLocalMap([mp, mp])
    for B in (1, 2):
        assert _status(lambda: g.match_batch([scan] * B, np.stack([T0] * B))) == FLS_ERR_UNSUPPORTED
    Ta, Tb = T0.copy(), T0.copy()
    cl = PointcloudCluster(planar_cloud=scan[::4].copy(), corner_cloud=scan[1::8].copy())
    assert g.Match(cl, Ta) == f.Match(cl, Tb) and np.array_equal(Ta, Tb)


def test_empty_planar_scan_in_a_batch(scene16):
    cfg = default_config(FLS_P2PLANE_KNN, flags=FLS_FLAG_ITER_LOG)
    g = _gpu(cfg)
    g.AddCloudToLocalMap([scene16["map"]])
    empty = np.zeros((0, 4), np.float32)
    scans = [scene16["scan"], empty, scene16["scan"]]
    T0 = scene16["guess_small"]
    oks, Ts = g.match_batch(scans, np.stack([T0] * 3))
    sts = g.last_batch_stats
    ok1, T1, st1, lg1 = _single(g, FLS_P2PLANE_KNN, empty, T0)
    assert bool(oks[1]) == ok1 and sts[1].iterations == st1.iterations and sts[1].n_valid == st1.n_valid == 0
    assert np.array_equal(Ts[1], T1)


# ---- 6. per-scan outputs and handle state -------------------------------------------------------------------------------------
@pytest.mark.parametrize("method", METHODS, ids=IDS)
def test_outputs_and_handle_state(world, traj, scene16, method):
    import torch
    cfg = default_config(method, flags=FLS_FLAG_ITER_LOG | FLS_FLAG_PROFILE)
    g = _gpu(cfg)
    g.AddCloudToLocalMap([scene16["map"]])
    B = 6
    scans, guesses = _sized_scans(world, traj, B, method)
    buf = torch.full((B, 18), float("nan"), dtype=torch.float64, device="cuda")
    g.set_result_buffer_device(buf.data_ptr(), B)
    oks, Ts = g.match_batch(scans, guesses)
    rec = buf.cpu().numpy()
    sts = g.last_batch_stats
    logs = [g.iter_log(k) for k in range(B)]
    fit = g.GetFitnessScore(2.0)
    # two identical batches: the sums are fixed per sub-grid
    oks2, Ts2 = g.match_batch(scans, guesses)
    assert np.array_equal(oks, oks2) and np.max(np.abs(Ts - Ts2)) <= 1e-12
    print(f"repeated batch bitwise equal: {np.array_equal(Ts, Ts2)}")
    g.set_result_buffer_device(0, 0)
    # a single Match after the batch equals one on a fresh handle
    f = _gpu(cfg)
    f.AddCloudToLocalMap([scene16["map"]])
    a, b = _single(g, method, scans[1], guesses[1]), _single(f, method, scans[1], guesses[1])
    assert a[0] == b[0] and np.array_equal(a[1], b[1]) and a[2].iterations == b[2].iterations
    for k in range(B):
        one = _single(g, method, scans[k], guesses[k])
        if k == 0:  # GetFitnessScore after the batch scores scan 0's final pose on scan 0's source
            fit1 = g.GetFitnessScore(2.0)
            assert abs(fit - fit1) <= 1e-6 * max(1.0, abs(fit1)), (fit, fit1)
        ok1, T1, st1, lg1 = one
        n = _n_source(method, cfg, scans[k])
        _assert_single(oks, Ts, sts, logs, k, one, n)
        assert sts[k].algo_bytes == st1.algo_bytes, k
        for a, b in zip(logs[k], lg1):  # every iteration
            _assert_sum_bound(a, b, n, k)
        # the 18-double record: column-major pose, converged, iterations
        assert rec[k, 16] == float(ok1) and rec[k, 17] == st1.iterations, k
        assert np.max(np.abs(rec[k, :16].reshape(4, 4).T - T1)) < 1e-9, k
    assert sts[0].kernel_launches == 1 and all(st.kernel_launches == 0 for st in sts[1:])
