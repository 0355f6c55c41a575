"""GPU parity of the LOAM-iVox mapping-mode map, bit for bit: the Match-internal insertion rule (ivox_insert_rule_kernel and its
class-1-then-class-2 compaction), the incremental insert of IvoxMap, each of its fall-backs to the full build (garbage,
slack, table load, capacity) and the LRU eviction, against the sequential references of tests/ivox_map_ref.py (proved against
the oracle in tests/test_oracle_ivox_mapping.py).  After every call the map's points in insertion order and its voxel keys
must equal the reference's bit for bit, and its 5-NN answers must have the reference's nearest neighbour and 5-NN set.  The
reference is fed the GPU's own poses, so only the map is compared."""
import numpy as np
import pytest

from funny_lidar_slam_b200 import FLS_P2PLANE_IVOX, default_config, synth
from tests import ivox_map_ref, ivox_ref

pytestmark = pytest.mark.gpu


def _gpu(**kw):
    from funny_lidar_slam_b200.registration import Registration
    return Registration(default_config(FLS_P2PLANE_IVOX, localization_mode=0, **kw))


def _match(g, scan, T):
    from funny_lidar_slam_b200.registration import PointcloudCluster
    T = np.array(T, np.float64)
    ok = g.Match(PointcloudCluster(planar_cloud=scan), T)
    return ok, T


def _queries(pts, rng, n=2000):
    """Map points moved by 0.1 m (sigma) plus map points snapped to a 1/16 m grid and lifted by 1/32 m: the latter hit exact
    rank-4/5 ties on lattice maps (the rule scene); the exact rank-0/1 ties of the incremental path come from lattice_queries."""
    q = pts[rng.integers(0, len(pts), n - n // 4)].copy()
    q[:, :3] += rng.normal(0, 0.1, (len(q), 3)).astype(np.float32)
    a = pts[rng.integers(0, len(pts), n // 4), :3].astype(np.float64)
    t = np.zeros((len(a), 4), np.float32)
    t[:, :3] = (np.round(a * 16.0) / 16.0 + 0.03125).astype(np.float32)
    return np.concatenate([q, t])


def lattice(x0, y0, z, n=16, h=0.125):
    """The n x n lattice of spacing h on the plane z (s2_exact_ties): every coordinate a multiple of 1/16."""
    g = np.arange(n) * h
    X, Y = np.meshgrid(x0 + g, y0 + g, indexing="ij")
    out = np.zeros((n * n, 4), np.float32)
    out[:, 0], out[:, 1], out[:, 2] = X.ravel(), Y.ravel(), z
    return out


def lattice_queries(x0, y0, z, n=16, h=0.125):
    """Cell centres (4 neighbours at one distance), edge centres (2, then 2 + 2) and lattice points (1, then 4) of `lattice`,
    lifted off the plane: exact ties at ranks 0/1 and 4/5 (every distance is exact in fp32)."""
    q = []
    for i in range(1, n - 2):
        for j in range(1, n - 2):
            x, y = x0 + i * h, y0 + j * h
            q += [(x + h / 2, y + h / 2, z + 0.03), (x, y + h / 2, z + h / 2), (x, y, z + 0.03125)]
    out = np.zeros((len(q), 4), np.float32)
    out[:, :3] = q
    return out


def check_map(g, ref, nearby, max_range, rng, tag, ties=None):
    """Points in insertion order and voxel keys bit for bit; 5-NN answers of about 2000 queries (and `ties`) against knn5."""
    pts = ref.points
    got = g.map_points()
    assert got.shape == pts.shape and np.array_equal(got, pts), (tag, got.shape, pts.shape)
    keys = set(map(tuple, np.asarray(g.voxel_keys(), np.int64).tolist()))
    assert keys == set(ref.voxels), tag
    assert g.map_info().n_voxels == ref.num_voxels, tag
    q = _queries(pts, rng)
    if ties is not None:
        q = np.concatenate([q, ties])
    out, cnt = g.ivox_knn(q)
    kn = ivox_ref.knn5(pts, q[:, :3], ref.res, nearby, max_range)
    assert np.array_equal(cnt, kn.found), tag
    for i in range(len(q)):
        a, b = out[i, :cnt[i]], pts[kn.idx[i, :cnt[i]]]
        # the nearest neighbour and the 5-NN set are exact (the selection re-runs knn5_exact where its quantised keys cannot tell
        # ranks 1/2 or 5/6 apart, fls_knn.cuh); the order of the other four among themselves is not part of the search's contract
        assert np.array_equal(a[:1], b[:1]) and np.array_equal(a[np.lexsort(a.T)], b[np.lexsort(b.T)]), (tag, i)


def _settle_ties(r, before, got):
    """Tied class-1 decisions take the GPU's choice (whether the point is in the appended slice); every other decision is the
    reference's.  Returns the expected slice and the number of ties."""
    t = r.ties()
    if len(t):
        app = {p.tobytes() for p in got[len(before):]}
        r.cls[t] = [1 if r.world[i].tobytes() in app else 0 for i in t]
        r.appended = np.concatenate([r.world[r.cls == 1], r.world[r.cls == 2]])
    return r.appended, len(t)


@pytest.mark.parametrize("nearby", range(4))
def test_rule_edges(nearby):
    s = ivox_map_ref.rule_scene()
    g = _gpu(max_iterations=1, ivox_nearby=nearby, ivox_max_range=1.0)
    ref = ivox_map_ref.IVoxMapRef(0.5, 10 ** 6)
    rng = np.random.default_rng(nearby)
    g.AddCloudToLocalMap([s.map])
    ref.add(s.map)
    check_map(g, ref, nearby, 1.0, rng, "first")
    ok, T = _match(g, s.scan, np.eye(4))
    assert ok and g.last_stats.n_valid >= 50
    r = ivox_map_ref.insert_rule(s.map, s.scan, np.eye(4), T, 0.5, nearby, 1.0)
    assert np.array_equal(r.world, s.scan) and len(r.ties()) == 0  # every edge met as built, none left to rounding
    got = g.map_points()
    assert np.array_equal(got[len(s.map):], r.appended), [int(c) for c in r.cls]
    ref.add(r.appended)
    check_map(g, ref, nearby, 1.0, rng, "edges")
    before = g.map_points()
    ok, T = _match(g, s.scan[list(s.probes.values())], np.eye(4))  # probes only: n_valid < 50, nothing enters
    assert not ok and np.array_equal(g.map_points(), before)
    ok, T = _match(g, s.on_map, np.eye(4))  # every point coincides with a map point: all dropped
    assert ok and np.array_equal(g.map_points(), before)
    check_map(g, ref, nearby, 1.0, rng, "unchanged")


def _stream(world, traj, nearby, res, capacity, n_scans):
    g = _gpu(max_iterations=1, ivox_nearby=nearby, ivox_resolution=res, ivox_capacity=capacity)
    ref = ivox_map_ref.IVoxMapRef(res, capacity)
    rng = np.random.default_rng(7 + nearby)
    first = synth.make_map_from_scans(world, traj[0:5:2], "vlp16", leaf=0.3)
    g.AddCloudToLocalMap([first])
    ref.add(first)
    check_map(g, ref, nearby, 5.0, rng, 0)
    ties, seen, evicted = 0, set(ref.voxels), False
    for k in range(1, n_scans + 1):
        scan = synth.voxel_downsample_np(synth.make_scan(world, traj[k], "vlp16", seed=40 + k)["points"], 0.5)
        guess = synth.perturb_pose(traj[k], dpos=0.05, drot_deg=0.5, seed=k)
        before = ref.points
        ok, T = _match(g, scan, guess)
        assert ok, k
        got = g.map_points()
        r = ivox_map_ref.insert_rule(before, scan, guess, T, res, nearby, 5.0)
        app, nt = _settle_ties(r, before, got)
        ties += nt
        ref.add(app)
        check_map(g, ref, nearby, 5.0, rng, k)
        keys = set(ref.voxels)
        evicted |= bool(seen - keys)
        seen |= keys
    return g, ties, evicted


@pytest.mark.parametrize("nearby,res", [(nb, r) for nb in range(4) for r in (0.5, 1.0)])
def test_stream_through_match(world, traj, nearby, res):
    """8 scans, one Gauss-Newton step each (the previous pose is the guess), run open loop on the GPU's poses."""
    g, ties, _ = _stream(world, traj, nearby, res, 10 ** 6, 8)
    mi = g.map_info()
    assert mi.incremental_inserts >= 5, (mi.incremental_inserts, mi.full_builds)
    print(f"rule decisions within rounding: {ties}")
    assert ties <= 2


def test_lru_through_match(world, traj):
    """A capacity the stream crosses: voxels stamped by earlier incremental inserts are evicted by later Matches."""
    first = synth.make_map_from_scans(world, traj[0:5:2], "vlp16", leaf=0.3)
    cap = int(len(set(map(tuple, ivox_ref.voxel_key(first[:, :3], 0.5).tolist()))) * 1.25) + 8
    g, ties, evicted = _stream(world, traj, 2, 0.5, cap, 12)
    assert evicted and g.map_info().incremental_inserts >= 1 and ties <= 2


def test_stream_with_full_iterations_through_twin(world, traj):
    """Default iterations: the rule searches at the pose before the last update.  A localization-mode twin seeded with the map
    as it was and run with the same iteration count must reproduce T bit for bit; the twin with one iteration fewer then gives
    that previous pose (the guess when the Match took one step)."""
    from funny_lidar_slam_b200.registration import Registration
    g = _gpu()
    ref = ivox_map_ref.IVoxMapRef(0.5, 10 ** 6)
    rng = np.random.default_rng(3)
    first = synth.make_map_from_scans(world, traj[0:5:2], "vlp16", leaf=0.3)
    g.AddCloudToLocalMap([first])
    ref.add(first)
    ties, multi = 0, 0
    for k in range(1, 6):
        scan = synth.voxel_downsample_np(synth.make_scan(world, traj[k], "vlp16", seed=40 + k)["points"], 0.5)
        guess = synth.perturb_pose(traj[k], dpos=0.05, drot_deg=0.5, seed=k)
        before = ref.points
        ok, T = _match(g, scan, guess)
        assert ok, k
        n = g.last_stats.iterations

        def twin(iters):
            if iters == 0:
                return guess
            t = Registration(default_config(FLS_P2PLANE_IVOX, localization_mode=1, max_iterations=iters))
            t.AddCloudToLocalMap([before])
            return _match(t, scan, guess)[1]
        assert np.array_equal(twin(n), T), k
        multi += n > 1
        r = ivox_map_ref.insert_rule(before, scan, twin(n - 1), T, 0.5, 2, 5.0)
        app, nt = _settle_ties(r, before, g.map_points())
        ties += nt
        ref.add(app)
        check_map(g, ref, 2, 5.0, rng, k)
    assert multi >= 3 and ties <= 2


def _phase(g, ref, chunks, rng, tag, ties=None):
    """ivox_add_points of every chunk, the map checked after each; returns the (incremental, full) insert counts of the phase."""
    mi0 = g.map_info()
    for j, c in enumerate(chunks):
        g.ivox_add_points(c)
        ref.add(c)
        check_map(g, ref, 2, 5.0, rng, (tag, j), ties)
    mi1 = g.map_info()
    return mi1.incremental_inserts - mi0.incremental_inserts, mi1.full_builds - mi0.full_builds


def _box(rng, n, lo, hi, first=0):
    out = np.zeros((n, 4), np.float32)
    out[:, :3] = rng.uniform(lo, hi, (n, 3))
    out[:, 3] = np.arange(first, first + n)
    return out


def _handle(base):
    g = _gpu()
    ref = ivox_map_ref.IVoxMapRef(0.5, 10 ** 6)
    g.AddCloudToLocalMap([base])
    ref.add(base)
    return g, ref


def test_fallback_garbage():
    """Many small inserts into the same voxels: every one rewrites them at the end of the arrays, until the old copies outweigh
    the live points and the next insert rebuilds.  The inserts are lattice points, repeated across inserts, so the rewritten
    runs are checked on exact ties decided by insertion order."""
    rng = np.random.default_rng(11)
    g, ref = _handle(_box(rng, 2000, (0.0, 0.0, 2.0), (4.0, 4.0, 3.0)))  # 1.5 m above the lattice: outside its stencils
    lat = lattice(1.0, 1.0, 0.5)
    chunks = []
    for j in range(30):
        c = lat[rng.choice(len(lat), 64, replace=False)].copy()
        c[:, 3] = 1000 + j  # copies of one lattice point told apart by the insert they came in
        chunks.append(c)
    inc, full = _phase(g, ref, chunks, rng, "garbage", lattice_queries(1.0, 1.0, 0.5))
    assert inc >= 5 and full >= 1, (inc, full)


def test_fallback_slack():
    """One insert that moves more points than the rewritten-voxel slack holds while the point array itself still has room: a
    map larger than the slack's fixed part, an insert that touches every voxel and adds 2.65 times the map."""
    rng = np.random.default_rng(12)
    base = _box(rng, 100000, (-20.0, -20.0, 0.0), (20.0, 20.0, 2.0))
    g, ref = _handle(base)
    inc, full = _phase(g, ref, [base[:500] + np.float32([0, 0, 0, 0.5])], rng, "slack-small")
    assert (inc, full) == (1, 0)
    big = np.tile(base, (3, 1))[:265000]  # every voxel touched: all old points move, plus 2.65x as many new ones
    big[:, 3] += 0.25
    inc, full = _phase(g, ref, [big], rng, "slack")
    assert (inc, full) == (0, 1)


def test_fallback_table_load():
    """One insert that creates more voxels than the occupied table has room for at its load factor."""
    rng = np.random.default_rng(13)
    g, ref = _handle(_box(rng, 20000, (0.0, 0.0, 0.0), (4.0, 4.0, 1.0)))
    inc, full = _phase(g, ref, [_box(rng, 200, (0.0, 0.0, 0.0), (4.0, 4.0, 1.0), 30000)], rng, "table-small")
    assert (inc, full) == (1, 0)
    slots = g.map_info().table_slots
    inc, full = _phase(g, ref, [_box(rng, slots, (-80.0, -80.0, -80.0), (80.0, 80.0, 80.0), 40000)], rng, "table")
    assert (inc, full) == (0, 1)


def test_capacity_crossing_with_retouched_victims(world, traj):
    """LRU eviction after incremental inserts: each round first re-touches the least recently used voxels with a small insert
    that creates none (incremental: its stamps are all that keeps those voxels alive), then crosses the capacity with a
    shuffled cloud, so victims are touched again later in the same call."""
    clouds = [synth.transform_points(synth.voxel_downsample_np(synth.make_scan(world, traj[k], "vlp16", seed=70 + k)["points"], 0.3), traj[k])
              for k in range(6)]
    n_first = len(set(map(tuple, ivox_ref.voxel_key(clouds[0][:, :3], 0.5).tolist())))
    cap = int(n_first * 1.3) + 8
    g = _gpu(ivox_capacity=cap)
    ref = ivox_map_ref.IVoxMapRef(0.5, cap)
    rng = np.random.default_rng(5)
    g.AddCloudToLocalMap([clouds[0]])
    ref.add(clouds[0])
    evicted, retouched, kept = False, False, 0
    for k, c in enumerate(clouds[1:]):
        oldest = [v[0] for v in list(ref.voxels.values())[:200]]  # one point of each of the 200 least recently used voxels
        small = np.array(oldest, np.float32)
        small[:, 3] += 0.5
        inc, full = _phase(g, ref, [small], rng, ("cap-small", k))
        assert (inc, full) == (1, 0), (k, inc, full)
        c = c[rng.permutation(len(c))]  # scattered touch times: a victim may be touched again later in the call
        before = {key: len(v) for key, v in ref.voxels.items()}
        in_call = {}
        for key in map(tuple, ivox_ref.voxel_key(c[:, :3], 0.5).tolist()):
            in_call[key] = in_call.get(key, 0) + 1
        inc, full = _phase(g, ref, [c], rng, ("cap", k))
        assert full == 1, (k, inc, full)
        after = {key: len(v) for key, v in ref.voxels.items()}
        evicted |= bool(set(before) - set(after))
        kept += sum(tuple(map(int, ivox_ref.voxel_key(p[:3], 0.5))) in after for p in small)
        # existed before the call, holds only the call's points after it: evicted, then touched again and re-created
        retouched |= any(key in after and after[key] == n_c for key, n_c in in_call.items() if key in before)
    assert evicted and retouched and kept > 0
