"""Scan Context on the device (fls_keyframes_scan_context / _detect_loop / _place_query) against the numpy restatement of its definitions
(tests/scan_context_ref.py): descriptors bit for bit, distances to 1e-12, shifts and rankings wherever the reference decides them by
more than 1e-9; the span rule, the descriptor cache, the yaw of turned scans, a loop that distance-based detection misses under drift,
and a relocalization whose coarse pose comes from place_query instead of a click."""
import numpy as np
import pytest

from funny_lidar_slam_b200 import _abi, synth
from funny_lidar_slam_b200._lib import FlsError
from funny_lidar_slam_b200.keyframes import KeyFrameStore, place_pose, sc_cfg
from tests import scan_context_ref as ref

pytestmark = pytest.mark.gpu

SECTOR = 2 * np.pi / 60


def _same(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _store(clouds, capacity=None):
    s = KeyFrameStore(capacity or max(sum(len(c) for c in clouds), 1))
    for c in clouds:
        s.add(c)
    return s


def _rz(a):
    R = np.eye(4)
    R[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
    return R


def _wrap(a):
    return (a + np.pi) % (2 * np.pi) - np.pi


def _rel_yaw(Ta, Tb):
    """yaw of Ta^-1 Tb"""
    d = np.linalg.inv(Ta) @ Tb
    return float(np.arctan2(d[1, 0], d[0, 0]))


def _ref_desc(c, cfg):
    return ref.descriptor(c, cfg.n_rings, cfg.n_sectors, cfg.max_radius, cfg.z_offset)


def _edge_clouds():
    R = 80.0
    rng = np.random.default_rng(17)
    far = np.concatenate([rng.uniform(-300, 300, (400, 2)), rng.uniform(-3, 3, (400, 1)), np.ones((400, 1))], 1).astype(np.float32)
    far = far[np.hypot(far[:, 0], far[:, 1]) >= R]
    ring_edge = np.array([[j * R / 20, 0.0, 0.3 * j, 1] for j in range(21)] + [[0.0, -j * R / 20, -1.0, 1] for j in range(21)], np.float32)
    rays = np.array([[5, 0.0, 1, 1], [5, -0.0, 2, 1], [-5, 0.0, 3, 1], [-5, -0.0, 4, 1], [0.0, 5, 5, 1], [-0.0, 5, 6, 1], [0.0, -5, 7, 1],
                     [-0.0, -5, 8, 1], [0.0, 0.0, 9, 1], [-0.0, -0.0, 10, 1], [-0.0, 0.0, 11, 1], [0.0, -0.0, 12, 1]], np.float32)
    nonfinite = np.array([[np.nan, 1, 1, 1], [1, np.nan, 1, 1], [1, 1, np.nan, 1], [np.inf, 1, 1, 1], [1, -np.inf, 1, 1], [1, 1, np.inf, 1],
                          [3, 4, 0.5, 1]], np.float32)
    negative = np.array([[7, 3, -5.0, 1], [7.01, 3.01, -9.0, 1], [-20, -30, -2.0, 1], [-20.01, -30.01, -2.5, 1], [1, 1, -0.0, 1]], np.float32)
    mixed = np.concatenate([rays, negative, ring_edge, nonfinite])
    return dict(empty=np.zeros((0, 4), np.float32), far=far, ring_edge=ring_edge, rays=rays, nonfinite=nonfinite, negative=negative, mixed=mixed)


@pytest.fixture(scope="module")
def streams(world):
    traj = synth.trajectory(24)
    vlp = [synth.make_scan(world, traj[i], "vlp16", seed=300 + i)["points"] for i in range(0, 24, 2)]
    hdl = [synth.make_scan(world, traj[i], "hdl64", seed=400 + i)["points"] for i in range(1, 24, 4)]
    return dict(traj=traj, vlp=vlp, hdl=hdl)


# ---- descriptors ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", [sc_cfg(), sc_cfg(n_rings=64, n_sectors=64, max_radius=50.0, z_offset=-1.5), sc_cfg(n_rings=7, n_sectors=360)])
def test_descriptors_bit_exact(streams, cfg):
    clouds = streams["vlp"] + streams["hdl"] + list(_edge_clouds().values())
    s = _store(clouds)
    got = s.scan_context(range(len(clouds)), cfg)
    for i, c in enumerate(clouds):
        assert _same(got[i], _ref_desc(c, cfg)), i
    # the same cells from the scan entry, host and device
    for c in (streams["hdl"][0], _edge_clouds()["mixed"]):
        _, d = s.place_query(c, 1, cfg, return_desc=True)
        assert _same(d, _ref_desc(c, cfg))


def test_edge_clouds_hit_the_edges_of_the_definition():
    e = _edge_clouds()
    assert np.all(ref.descriptor(e["empty"]) == 0) and np.all(ref.descriptor(e["far"]) == 0)
    assert np.count_nonzero(ref.descriptor(e["ring_edge"])) > 0 and (ref.descriptor(e["negative"]) < 0).any()


def test_device_query_equals_host_query(streams):
    import torch
    s = _store(streams["vlp"])
    q = streams["hdl"][2]
    a, da = s.place_query(q, 5, return_desc=True)
    d = torch.from_numpy(q).cuda()
    torch.cuda.synchronize()
    b, db = s.place_query_device(d.data_ptr(), len(q), 5, return_desc=True)
    from tests.conftest import to_pcl
    c, dc = s.place_query(to_pcl(q), 5, return_desc=True)
    assert _same(da, db) and _same(da, dc)
    assert [bytes(x) for x in a] == [bytes(x) for x in b] == [bytes(x) for x in c]


# ---- distances, shifts, ranking -------------------------------------------------------------------------------------------------
def _check_against_reference(got, Q, Cs, ids):
    D, sh, d = ref.distances(Q, Cs)
    assert len(got) == len(ids)
    by_id = {m.id: m for m in got}
    assert sorted(by_id) == sorted(ids)
    for k, i in enumerate(ids):
        m = by_id[i]
        assert abs(m.distance - D[k]) <= 1e-12, (i, m.distance, D[k])
        two = np.sort(d[k])[:2]
        if len(two) < 2 or two[1] - two[0] > 1e-9:
            assert m.shift == sh[k], i
            assert m.yaw == pytest.approx(float(ref.yaw(sh[k], Q.shape[1])), abs=1e-15)
    order = [m.id for m in got]
    r = ref.rank(D, np.asarray(ids))
    Dr = D[r]
    for k in range(len(order)):
        lo = k == 0 or Dr[k] - Dr[k - 1] > 1e-9
        hi = k == len(order) - 1 or Dr[k + 1] - Dr[k] > 1e-9
        if lo and hi:
            assert order[k] == ids[r[k]], k
    ds = [m.distance for m in got]
    assert all(a <= b for a, b in zip(ds, ds[1:]))


@pytest.mark.parametrize("cfg", [sc_cfg(), sc_cfg(n_rings=10, n_sectors=360, max_radius=40.0), sc_cfg(n_rings=64, n_sectors=64)])
def test_distances_shifts_and_ranking_match_the_reference(world, streams, cfg):
    clouds = streams["vlp"] + streams["hdl"] + [_edge_clouds()["empty"], _edge_clouds()["mixed"]]
    s = _store(clouds)
    desc = np.stack([_ref_desc(c, cfg) for c in clouds])
    q = len(clouds) - 3  # the last HDL-64 keyframe; candidates: everything before it, empty and edge clouds after
    got = s.detect_loop(q, 0, k=1000, cfg=cfg)
    _check_against_reference(got, desc[q], desc[:q], list(range(q)))
    scan = synth.make_scan(world, streams["traj"][5] @ _rz(0.7), "vlp16", seed=9)["points"]
    got = s.place_query(scan, k=1000, cfg=cfg)
    _check_against_reference(got, _ref_desc(scan, cfg), desc, list(range(len(clouds))))
    assert s.last_stats.n_valid == len(clouds)
    # k below the candidate count: the first k of the full ranking
    top = s.place_query(scan, k=3, cfg=cfg)
    assert [bytes(x) for x in top] == [bytes(x) for x in got[:3]]


def test_empty_query_is_distance_one_everywhere(streams):
    s = _store(streams["vlp"][:4])
    got = s.place_query(np.zeros((0, 4), np.float32), k=10)
    assert [m.id for m in got] == [0, 1, 2, 3] and all(m.distance == 1.0 and m.shift == 0 for m in got)


# ---- the span rule --------------------------------------------------------------------------------------------------------------
def test_span_rule_at_its_edges(streams):
    s = _store(streams["vlp"])
    K = len(streams["vlp"])
    q = K - 1
    for span, want in ((q, 0), (q - 1, 1), (0, q), (q + 50, 0), (3, q - 3)):
        got = s.detect_loop(q, span, k=100)
        assert sorted(m.id for m in got) == list(range(want)), span
        assert s.last_stats.n_valid == want
    assert s.detect_loop(0, 0, k=5) == []
    for bad_q, span in ((K, 0), (K + 7, 0), (-1, 0), (3, -1)):
        with pytest.raises(FlsError) as e:
            s.detect_loop(bad_q, span, k=5)
        assert e.value.status == _abi.FLS_ERR_INVALID_ARG
    with pytest.raises(FlsError) as e:
        s.detect_loop(q, 0, k=0)
    assert e.value.status == _abi.FLS_ERR_INVALID_ARG
    with pytest.raises(FlsError) as e:
        s.place_query(streams["vlp"][0], k=1, cfg=sc_cfg(n_sectors=361))
    assert e.value.status == _abi.FLS_ERR_INVALID_ARG
    empty = KeyFrameStore(10)
    assert empty.place_query(streams["vlp"][0], k=3) == []


# ---- the cache ------------------------------------------------------------------------------------------------------------------
def test_cache_interleaved_adds_and_cfg_changes(streams):
    clouds = streams["vlp"] + streams["hdl"]
    fresh = _store(clouds).scan_context(range(len(clouds)))
    a, b = sc_cfg(), sc_cfg(n_rings=12, n_sectors=90, max_radius=60.0, z_offset=0.5)
    s = KeyFrameStore(sum(len(c) for c in clouds))
    for i, c in enumerate(clouds):
        s.add(c)
        if i % 3 == 0:
            s.place_query(clouds[0], 2, a)
        if i % 4 == 1:
            s.detect_loop(i, 0, 2, b)  # a cfg change re-describes every keyframe
    assert _same(s.scan_context(range(len(clouds)), a), fresh)
    want_b = np.stack([_ref_desc(c, b) for c in clouds])
    assert _same(s.scan_context(range(len(clouds)), b), want_b)
    assert _same(s.scan_context(range(len(clouds)), a), fresh)
    # z_offset -0.0 and +0.0 are different cfgs: a z = -0.0 cell differs
    z = np.array([[3.0, 4.0, -0.0, 1.0]], np.float32)
    t = _store([z])
    assert not np.signbit(t.scan_context([0], sc_cfg(z_offset=0.0))[0]).any()
    assert np.signbit(t.scan_context([0], sc_cfg(z_offset=-0.0))[0]).any()


@pytest.mark.parametrize("n_small", [8, 400])
def test_cfg_switches_on_one_store_to_larger_descriptors(streams, n_small):
    """One store switched between cfgs with more cells (64 x 64) and more sectors (7 x 360) than the one its cache was sized for,
    and back: every descriptor and every distance equals the reference.  With 400 more keyframes the cache is past its first size."""
    rng = np.random.default_rng(40 + n_small)
    clouds = streams["vlp"] + _small_clouds(rng, n_small) + [_edge_clouds()["mixed"]]
    assert len(clouds) >= 20
    s = _store(clouds)
    q = len(clouds) - 1
    for cfg in (sc_cfg(), sc_cfg(n_rings=64, n_sectors=64), sc_cfg(n_rings=7, n_sectors=360), sc_cfg(n_rings=1, n_sectors=360),
                sc_cfg(n_rings=11, n_sectors=360, max_radius=30.0, z_offset=-5.0), sc_cfg()):
        got = s.detect_loop(q, 0, k=len(clouds), cfg=cfg)
        want = np.stack([_ref_desc(c, cfg) for c in clouds])
        assert _same(s.scan_context(range(len(clouds)), cfg), want), (cfg.n_rings, cfg.n_sectors)
        _check_against_reference(got, want[q], want[:q], list(range(q)))


def _small_clouds(rng, k):
    return [np.concatenate([rng.uniform(-40, 40, (n, 2)), rng.uniform(-2, 5, (n, 1)), np.ones((n, 1))], 1).astype(np.float32)
            for n in rng.integers(300, 900, k)]


def test_launches_and_waits_do_not_depend_on_the_keyframe_count():
    rng = np.random.default_rng(21)
    q = _small_clouds(rng, 1)[0]
    counts = {}
    for K in (10, 1000):
        clouds = _small_clouds(rng, K)
        s = _store(clouds, sum(len(c) for c in clouds) + len(q))
        first = s.place_query(q, 5)
        a = (s.last_stats.gpu_launches, s.last_stats.iterations)
        again = s.place_query(q, 5)
        b = (s.last_stats.gpu_launches, s.last_stats.iterations)
        assert [bytes(x) for x in first] == [bytes(x) for x in again]  # two identical calls, identical bits
        s.detect_loop(K - 1, 2, 5)
        c = (s.last_stats.gpu_launches, s.last_stats.iterations)
        s.add(q)
        s.detect_loop(K, 2, 5)
        d = (s.last_stats.gpu_launches, s.last_stats.iterations)
        counts[K] = (a, b, c, d)
        assert a[1] == b[1] == c[1] == d[1] == 1
    assert counts[10] == counts[1000], counts


def test_queries_leave_assemble_unchanged(streams):
    clouds = streams["vlp"]
    poses = streams["traj"][0:24:2]
    s = _store(clouds)
    before = s.assemble(range(len(clouds)), poses, 0.3, 0.3)
    st0 = (s.last_stats.gpu_launches, s.last_stats.iterations)
    s.place_query(clouds[3], 4)
    s.detect_loop(len(clouds) - 1, 2, 4, sc_cfg(n_sectors=90))
    after = s.assemble(range(len(clouds)), poses, 0.3, 0.3)
    assert _same(before, after) and (s.last_stats.gpu_launches, s.last_stats.iterations) == st0


# ---- yaw --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("deg", [30.0, 90.0, 180.0, -120.0])
def test_turned_scan_finds_its_keyframe_and_yaw(world, streams, deg):
    traj = streams["traj"]
    ids = list(range(0, 24, 2))
    s = _store(streams["vlp"])
    kf = 4
    T_q = traj[ids[kf]] @ _rz(np.deg2rad(deg))
    scan = synth.make_scan(world, T_q, "vlp16", seed=77)["points"]
    got = s.place_query(scan, 3)
    assert got[0].id == kf, [(m.id, m.distance) for m in got]
    assert abs(_wrap(got[0].yaw - np.deg2rad(deg))) <= SECTOR, (got[0].yaw, deg)
    T_guess = place_pose(traj[ids[kf]], got[0].yaw)
    assert abs(_rel_yaw(T_guess, T_q)) <= SECTOR


# ---- a loop that distance-based detection misses ----------------------------------------------------------------------------
def _drifted(T, yaw_rate, scale):
    """odometry with a yaw error per keyframe and a scale error, integrated from the first pose"""
    out = [T[0].copy()]
    for i in range(1, len(T)):
        d = np.linalg.inv(T[i - 1]) @ T[i]
        d[:3, 3] *= scale
        out.append(out[-1] @ _rz(yaw_rate) @ d)
    return np.array(out)


def _detect_by_distance(poses, curr, dist_thre=10.0, span=30):
    """LoopClosure::DetectByDistance (src/slam/loop_closure.cpp:138-177 upstream), literally: GetNearKeyFramesResult then
    CheckCandidateKeyFrames; -1 is KeyFrame::kInvalidID"""
    p = poses[curr][:3, 3]
    cand = [(k, float(np.linalg.norm(p - poses[k][:3, 3]))) for k in range(len(poses))]
    cand = [c for c in cand if c[1] < dist_thre]
    cand.sort(key=lambda c: c[1])
    for k, _ in cand:
        if curr - k > span:
            return k
    return -1


def test_loop_under_drift(world):
    T = synth.trajectory(92)  # a figure 8: keyframe 0 and keyframe 91 both cross the centre, about 90 degrees apart
    drift = _drifted(T, 0.008, 1.03)
    q, span = 91, 30
    assert np.linalg.norm(drift[q][:3, 3] - drift[0][:3, 3]) > 10.0
    assert _detect_by_distance(drift, q, 10.0, span) == -1
    clouds = [synth.make_scan(world, T[i], "vlp16", seed=600 + i)["points"] for i in range(92)]
    s = _store(clouds)
    got = s.detect_loop(q, span, k=5)
    best = got[0]
    assert q - best.id > span
    assert np.linalg.norm(T[best.id][:3, 3] - T[q][:3, 3]) < 2.0, [(m.id, m.distance) for m in got]
    assert abs(_wrap(best.yaw - _rel_yaw(T[best.id], T[q]))) <= SECTOR, (best.yaw, _rel_yaw(T[best.id], T[q]))


# ---- relocalization without a click -----------------------------------------------------------------------------------------
def test_relocalization_from_place_query():
    from funny_lidar_slam_b200.registration import Registration
    world = synth.make_world(seed=1234)
    traj = synth.trajectory(40)
    T_true = traj[10]
    mp = synth.make_surface_map(world, spacing=0.5, seed=11)
    mp = np.ascontiguousarray(mp[np.all(np.abs(mp[:, :2] - T_true[:2, 3].astype(np.float32)) <= 40.0, axis=1)])
    first_pass = [i for i in range(25) if i != 10]  # the store never saw the query's pose
    s = _store([synth.make_scan(world, traj[i], "vlp16", seed=700 + i)["points"] for i in first_pass])
    scan = synth.make_scan(world, T_true @ _rz(np.deg2rad(63.0)), "vlp16", seed=21)["points"]
    T_scan = T_true @ _rz(np.deg2rad(63.0))
    best = s.place_query(scan, 1)[0]
    T_guess = place_pose(traj[first_pass[best.id]], best.yaw)
    dt0, dr0 = synth.pose_error(T_guess, T_scan)
    assert dt0 <= 3.0 and np.rad2deg(dr0) <= 20.0, (dt0, np.rad2deg(dr0))
    g = Registration(_abi.default_config(_abi.FLS_P2PLANE_IVOX))
    g.AddCloudToLocalMap([mp])
    r = g.relocalize(scan, T_guess, xy_radius=3.0, xy_step=1.0, yaw_range=np.deg2rad(20.0), yaw_step=np.deg2rad(10.0), n_refine=16)
    dt, dr = synth.pose_error(r.T, T_scan)
    print(f"place_query: keyframe {first_pass[best.id]} D={best.distance:.3f} guess off {dt0:.2f} m {np.rad2deg(dr0):.1f} deg | "
          f"relocalized off {dt:.4f} m {np.rad2deg(dr):.3f} deg, fitness {r.fitness:.3f}")
    assert r.accepted
    assert dt < 0.05 and np.rad2deg(dr) < 0.5
