"""GPU parity: LoamPointToPlaneIVOX path (K1 + K6) through the C ABI vs the CPU oracle."""
import numpy as np
import pytest

from funny_lidar_slam_b200 import FLS_P2PLANE_IVOX, default_config, synth
from funny_lidar_slam_b200._abi import FLS_FLAG_ITER_LOG
from tests.conftest import to_pcl

pytestmark = pytest.mark.gpu

POS_TOL = 1e-4  # metres   (BASELINE.json north_star)
ROT_TOL = 1e-4  # radians


def _pair(cfg):
    from funny_lidar_slam_b200.registration import Registration
    from oracle import pyoracle as orc
    return Registration(cfg), orc.Registration(cfg)


def _assert_logs_equal(lb, l1, what):
    """A scan's iteration log from a batch equals the log of its single Match: same neighbours and planes, only the fp64
    summation order differs (1e-9 relative per iteration)."""
    assert len(lb) == len(l1), what
    for k, (a, b) in enumerate(zip(lb, l1)):
        assert a["n_valid"] == b["n_valid"], (what, k)
        sc = max(np.abs(b["H"]).max(), 1e-300)
        assert np.allclose(a["H"], b["H"], rtol=1e-9, atol=1e-9 * sc), (what, k)
        assert np.allclose(a["g"], b["g"], rtol=1e-9, atol=1e-9 * sc), (what, k)


def test_ivox_knn_matches_oracle(scene16):
    from funny_lidar_slam_b200.registration import Registration
    from oracle import pyoracle as orc
    cfg = default_config(FLS_P2PLANE_IVOX)
    g = Registration(cfg)
    g.AddCloudToLocalMap([scene16["map"]])
    iv = orc.IVox(0.5, 2, 1000000)
    iv.add(scene16["map"])
    mi = g.map_info()
    assert mi.n_points == len(scene16["map"]) and mi.n_voxels == iv.num_voxels
    q = synth.transform_points(scene16["scan"], scene16["guess"])[:6000]
    gp, gc = g.ivox_knn(q)
    op, oc = iv.closest(q, 5, 5.0)
    assert np.array_equal(gc, oc)
    full = gc == 5
    assert full.sum() > 1000
    # nearest neighbour identical; the 5-set identical up to ordering of equal-distance ties
    assert np.array_equal(gp[full][:, 0, :3], op[full][:, 0, :3])
    gs = np.sort(gp[full][:, :, :3].reshape(full.sum(), -1), axis=1)
    os_ = np.sort(op[full][:, :, :3].reshape(full.sum(), -1), axis=1)
    assert np.array_equal(gs, os_)


@pytest.mark.parametrize("layout", ["packed", "pcl"])
def test_match_config1_scene(scene16, layout):
    cfg = default_config(FLS_P2PLANE_IVOX, flags=FLS_FLAG_ITER_LOG)
    g, o = _pair(cfg)
    mp, sc = scene16["map"], scene16["scan"]
    from funny_lidar_slam_b200.registration import PointcloudCluster
    if layout == "pcl":
        g.AddCloudToLocalMap([to_pcl(mp)])
        cl = PointcloudCluster(planar_cloud=to_pcl(sc))
    else:
        g.AddCloudToLocalMap([mp])
        cl = PointcloudCluster(planar_cloud=sc)
    o.add_cloud(mp)
    Tg = scene16["guess"].copy()
    ok_g = g.Match(cl, Tg)
    ok_o, To, st_o = o.match(sc, scene16["guess"])
    st_g = g.last_stats
    assert ok_g == ok_o
    assert st_g.iterations == st_o.iterations
    dt, dr = synth.pose_error(Tg, To)
    assert dt < POS_TOL and dr < ROT_TOL, (dt, dr)
    assert abs(st_g.n_valid - st_o.n_valid) <= max(2, st_o.n_valid // 2000)
    # per-iteration normal equations
    lg, lo = g.iter_log(), o.iter_log()
    assert len(lg) == len(lo)
    H0g, H0o = lg[0]["H"], lo[0]["H"]
    assert lg[0]["n_valid"] == lo[0]["n_valid"]
    assert np.allclose(H0g, H0o, rtol=1e-9, atol=1e-9 * np.abs(H0o).max())
    assert np.allclose(lg[0]["g"], lo[0]["g"], rtol=1e-9, atol=1e-9 * np.abs(H0o).max())
    # ground truth sanity
    assert synth.pose_error(Tg, scene16["truth"])[0] < 0.02


def test_match_64line(scene64):
    cfg = default_config(FLS_P2PLANE_IVOX)
    g, o = _pair(cfg)
    g.AddCloudToLocalMap([scene64["map"]])
    o.add_cloud(scene64["map"])
    from funny_lidar_slam_b200.registration import PointcloudCluster
    Tg = scene64["guess"].copy()
    ok_g = g.Match(PointcloudCluster(planar_cloud=scene64["scan"]), Tg)
    ok_o, To, st_o = o.match(scene64["scan"], scene64["guess"])
    assert ok_g == ok_o and g.last_stats.iterations == st_o.iterations
    dt, dr = synth.pose_error(Tg, To)
    assert dt < POS_TOL and dr < ROT_TOL, (dt, dr)


def test_fitness_score_localization(scene16):
    cfg = default_config(FLS_P2PLANE_IVOX)
    g, o = _pair(cfg)
    g.AddCloudToLocalMap([scene16["map"]])
    o.add_cloud(scene16["map"])
    from funny_lidar_slam_b200.registration import PointcloudCluster
    Tg = scene16["guess"].copy()
    g.Match(PointcloudCluster(planar_cloud=scene16["scan"]), Tg)
    o.match(scene16["scan"], scene16["guess"])
    for r in (1.0, 2.0):
        fo, fg = o.fitness(r), g.GetFitnessScore(r)
        assert abs(fg - fo) <= 1e-5 * max(1.0, abs(fo)), (r, fg, fo)


def test_match_failure_paths(scene16):
    """empty scan / scan far from the map: Match returns false, T still written (loam_point_to_plane_ivox.h:198-203)."""
    cfg = default_config(FLS_P2PLANE_IVOX)
    g, o = _pair(cfg)
    g.AddCloudToLocalMap([scene16["map"]])
    o.add_cloud(scene16["map"])
    from funny_lidar_slam_b200.registration import PointcloudCluster
    far = scene16["guess"].copy()
    far[:3, 3] += 500.0
    Tg = far.copy()
    ok_g = g.Match(PointcloudCluster(planar_cloud=scene16["scan"][:500]), Tg)
    ok_o, To, _ = o.match(scene16["scan"][:500], far)
    assert ok_g is False and ok_o is False
    assert np.allclose(Tg, To, atol=1e-12)
    Tg = scene16["guess"].copy()
    assert g.Match(PointcloudCluster(planar_cloud=np.zeros((0, 4), np.float32)), Tg) is False
    assert np.allclose(Tg, scene16["guess"], atol=1e-12)


def test_mapping_mode_stream(world, traj):
    """Mapping mode (is_localization_mode=false): after every successful Match the scan enters the iVox map through the
    cached-5-NN insertion rule (loam_point_to_plane_ivox.h:79-128 upstream, [quirk 8]); poses and map growth must
    follow the oracle scan after scan."""
    from funny_lidar_slam_b200.registration import PointcloudCluster, Registration
    from oracle import pyoracle as orc
    cfg = default_config(FLS_P2PLANE_IVOX, localization_mode=0, flags=FLS_FLAG_ITER_LOG)
    g, o = Registration(cfg), orc.Registration(cfg)
    first = synth.make_map_from_scans(world, traj[0:5:2], "vlp16", leaf=0.3)
    g.AddCloudToLocalMap([first])
    o.add_cloud(first)
    assert g.map_info().n_points == o.map_points
    grown = []
    for k in range(1, 6):
        scan = synth.voxel_downsample_np(synth.make_scan(world, traj[k], "vlp16", seed=40 + k)["points"], 0.4)
        guess = synth.perturb_pose(traj[k], dpos=0.05, drot_deg=0.5, seed=k)
        Tg = guess.copy()
        ok_g = g.Match(PointcloudCluster(planar_cloud=scan), Tg)
        ok_o, To, st_o = o.match(scan, guess)
        assert ok_g and ok_o and g.last_stats.iterations == st_o.iterations, k
        dt, dr = synth.pose_error(Tg, To)
        assert dt < 1e-4 and dr < 1e-4, (k, dt, dr)
        a, b = g.map_info().n_points, o.map_points
        # the inserted points are transformed with poses that agree to ~1e-6 m: a point on a cell face or a tie in the
        # "closer to the centre" test can flip, so sizes agree to a few points per scan, not bit for bit
        assert abs(a - b) <= max(3, b // 5000), (k, a, b)
        grown.append(b)
    assert grown[-1] > grown[0] > len(first)


def test_external_add_after_first_is_rejected_in_mapping_mode(scene16):
    from funny_lidar_slam_b200._lib import FlsError
    from funny_lidar_slam_b200.registration import Registration
    g = Registration(default_config(FLS_P2PLANE_IVOX, localization_mode=0))
    g.AddCloudToLocalMap([scene16["map"]])
    with pytest.raises(FlsError):  # upstream would run the insertion rule on caches of a Match that never happened
        g.AddCloudToLocalMap([scene16["map"]])


def test_batch_equals_separate_matches(world, traj):
    """fls_match_batch: B scans with different sizes, poses and iteration counts in ONE launch — every result must be
    the one a separate Match returns (same kernel; only the number of CTAs per scan, hence the fp64 summation order,
    differs: poses agree to ~1e-12)."""
    from funny_lidar_slam_b200.registration import PointcloudCluster, Registration
    from oracle import pyoracle as orc
    mp = synth.make_map_from_scans(world, traj[0:12:2], "vlp16", leaf=0.3)
    cfg = default_config(FLS_P2PLANE_IVOX, flags=FLS_FLAG_ITER_LOG)
    g = Registration(cfg)
    g.AddCloudToLocalMap([mp])
    scans, guesses = [], []
    for k, (dp, dr, keep) in enumerate(((0.3, 3.0, 1), (0.05, 0.5, 1), (0.2, 1.0, 3), (0.1, 2.0, 1), (0.3, 0.2, 2))):
        sc = synth.make_scan(world, traj[2 + k], "vlp16", seed=70 + k)["points"][::keep]
        scans.append(np.ascontiguousarray(sc))
        guesses.append(synth.perturb_pose(traj[2 + k], dpos=dp, drot_deg=dr, seed=k))
    scans.append(scans[0][:40].copy())  # too few valid planes: Match fails, T still written
    guesses.append(guesses[0].copy())
    singles = []
    for sc, gs in zip(scans, guesses):
        T = gs.copy()
        ok = g.Match(PointcloudCluster(planar_cloud=sc), T)
        singles.append((ok, T, g.last_stats.iterations, g.last_stats.n_valid, g.iter_log()))
    conv, Tb = g.match_batch(scans, np.stack(guesses))
    its = [s.iterations for s in g.last_batch_stats]
    assert len(set(its)) > 1  # the scans really stop at different iterations
    for s, (ok, T, it, nv, log1) in enumerate(singles):
        assert bool(conv[s]) == ok and g.last_batch_stats[s].iterations == it and g.last_batch_stats[s].n_valid == nv, s
        assert np.allclose(Tb[s], T, rtol=0, atol=1e-9), s
        _assert_logs_equal(g.iter_log(s), log1, s)
    assert not conv[-1]
    # and against the oracle for one of them
    o = orc.Registration(cfg)
    o.add_cloud(mp)
    ok_o, To, _ = o.match(scans[2], guesses[2])
    dt, dr_ = synth.pose_error(Tb[2], To)
    assert dt < POS_TOL and dr_ < ROT_TOL
    # pcl layout through the batch entry
    conv2, Tb2 = g.match_batch([to_pcl(s) for s in scans], np.stack(guesses))
    # same inputs, other record layout: identical up to fp64 rounding (the batch kernel hands its chunks out dynamically, so the
    # order of the sums — not their terms — varies from launch to launch)
    assert np.allclose(Tb2, Tb, rtol=0, atol=1e-11) and np.array_equal(conv2, conv)


def test_batch_needs_static_map(scene16):
    from funny_lidar_slam_b200._lib import FlsError
    from funny_lidar_slam_b200.registration import Registration
    g = Registration(default_config(FLS_P2PLANE_IVOX, localization_mode=0))
    g.AddCloudToLocalMap([scene16["map"]])
    with pytest.raises(FlsError):
        g.match_batch([scene16["scan"], scene16["scan"]], np.stack([scene16["guess"], scene16["guess"]]))


def test_batch_stress_many_small_and_empty_scans(world, traj):
    """24 scans of very different sizes (one empty, several below the 50-valid-plane failure bar) in one launch: the sweep
    must terminate with each scan's own result — compared with separate Matches."""
    from funny_lidar_slam_b200.registration import PointcloudCluster, Registration
    mp = synth.make_map_from_scans(world, traj[0:12:2], "vlp16", leaf=0.3)
    g = Registration(default_config(FLS_P2PLANE_IVOX, flags=FLS_FLAG_ITER_LOG))
    g.AddCloudToLocalMap([mp])
    rng = np.random.default_rng(11)
    base = [synth.make_scan(world, traj[3 + k], "vlp16", seed=90 + k)["points"] for k in range(4)]
    scans, guesses = [], []
    for j in range(24):
        k = j % 4
        n = [0, 17, 40, 333, 1500, 5000, len(base[k])][j % 7]
        sel = np.sort(rng.choice(len(base[k]), n, replace=False)) if n else np.zeros(0, np.int64)
        scans.append(np.ascontiguousarray(base[k][sel]))
        guesses.append(synth.perturb_pose(traj[3 + k], dpos=0.02 + 0.01 * (j % 5), drot_deg=0.3 + 0.2 * (j % 3), seed=200 + j))
    conv, Tb = g.match_batch(scans, np.stack(guesses))
    st_b = [(s.iterations, s.n_valid, s.converged) for s in g.last_batch_stats]
    logs_b = [g.iter_log(j) for j in range(24)]
    assert not conv[0] and st_b[0][1] == 0          # the empty scan fails, nothing else is disturbed
    for j in range(24):
        T = guesses[j].copy()
        ok = g.Match(PointcloudCluster(planar_cloud=scans[j]), T)
        st = g.last_stats
        assert bool(conv[j]) == ok and st_b[j][0] == st.iterations and st_b[j][1] == st.n_valid, j
        assert np.allclose(Tb[j], T, rtol=0, atol=1e-8), j
        _assert_logs_equal(logs_b[j], g.iter_log(), j)
    assert conv.sum() >= 12


def test_batch_begin_end_on_two_handles(world, traj):
    """fls_match_batch_begin / _end: two handles with a batch in flight each (the copy of one overlaps the kernels of the other);
    results must equal fls_match_batch, and a second begin on a busy handle is refused."""
    from funny_lidar_slam_b200._lib import FlsError
    from funny_lidar_slam_b200.registration import Registration
    mp = synth.make_map_from_scans(world, traj[0:12:2], "vlp16", leaf=0.3)
    cfg = default_config(FLS_P2PLANE_IVOX)
    regs = [Registration(cfg), Registration(cfg)]
    for r in regs:
        r.AddCloudToLocalMap([mp])
    batches = []
    for b in range(4):
        scans = [synth.make_scan(world, traj[2 + (3 * b + k) % 10], "vlp16", seed=300 + 10 * b + k)["points"] for k in range(3)]
        guesses = np.stack([synth.perturb_pose(traj[2 + (3 * b + k) % 10], dpos=0.1, drot_deg=1.0, seed=500 + 10 * b + k) for k in range(3)])
        batches.append((scans, guesses))
    ref = [regs[0].match_batch(s, g) for s, g in batches]
    out = [None] * 4
    regs[0].match_batch_begin(*batches[0])
    with pytest.raises(FlsError):
        regs[0].match_batch_begin(*batches[1])
    for b in range(1, 4):
        regs[b % 2].match_batch_begin(*batches[b])
        out[b - 1] = regs[(b - 1) % 2].match_batch_end()
    out[3] = regs[1].match_batch_end()
    for b in range(4):
        assert np.array_equal(out[b][0], ref[b][0]), b
        assert np.allclose(out[b][1], ref[b][1], rtol=0, atol=1e-12), b


def test_point_without_candidates_is_skipped_not_stale(scene16):
    """The documented deviation from upstream's stale nearest_points_ (ivox_map.cpp:21-23: GetClosestPoint leaves the output vector
    untouched when the stencil is empty): a point whose stencil holds no map point contributes nothing — even when the same index
    had five neighbours in the previous Match — on the GPU exactly as in the oracle."""
    from funny_lidar_slam_b200._abi import FLS_FLAG_ITER_LOG
    from funny_lidar_slam_b200.registration import PointcloudCluster, Registration
    from oracle import pyoracle as orc
    cfg = default_config(FLS_P2PLANE_IVOX, flags=FLS_FLAG_ITER_LOG)
    g, o = Registration(cfg), orc.Registration(cfg)
    g.AddCloudToLocalMap([scene16["map"]])
    o.add_cloud(scene16["map"])
    scan = scene16["scan"]
    T = scene16["guess_small"].copy()
    assert g.Match(PointcloudCluster(planar_cloud=scan), T)  # every index now "has" neighbours upstream
    o.match(scan, scene16["guess_small"])
    far = scan.copy()
    far[::7, :3] += np.float32(900.0)  # every 7th index: far outside the map, no stencil candidate at any iteration
    kept = np.ascontiguousarray(np.delete(scan, np.s_[::7], axis=0))
    Tf, Tk = scene16["guess_small"].copy(), scene16["guess_small"].copy()
    ok_f = g.Match(PointcloudCluster(planar_cloud=far), Tf)
    st_f, log_f = g.last_stats, g.iter_log()
    ok_k = g.Match(PointcloudCluster(planar_cloud=kept), Tk)
    st_k, log_k = g.last_stats, g.iter_log()
    ok_o, To, st_o = o.match(far, scene16["guess_small"])
    assert ok_f == ok_k == ok_o and st_f.iterations == st_k.iterations == st_o.iterations
    assert st_f.n_valid == st_k.n_valid == st_o.n_valid
    for a, b in zip(log_f, log_k):  # the far points add nothing to H and g
        assert np.allclose(a["H"], b["H"], rtol=1e-9, atol=1e-6) and np.allclose(a["g"], b["g"], rtol=1e-9, atol=1e-6)
    dt, dr = synth.pose_error(Tf, To)
    assert dt < POS_TOL and dr < ROT_TOL
