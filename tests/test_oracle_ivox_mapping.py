"""The oracle's mapping-mode iVox map against the sequential references of tests/ivox_map_ref.py: IVoxMap::AddPoints with LRU
eviction for every stencil, and the Match-internal insertion rule on the rule-edge scene and on scan streams.  These tests
prove the references on the CPU before the GPU tests rely on them."""
import numpy as np
import pytest

from funny_lidar_slam_b200 import FLS_P2PLANE_IVOX, default_config, synth
from oracle import pyoracle as orc
from tests import ivox_map_ref, ivox_ref


@pytest.fixture(scope="module")
def clouds(world, traj):
    return [synth.transform_points(synth.voxel_downsample_np(synth.make_scan(world, traj[k], "vlp16", seed=60 + k)["points"], 0.3), traj[k])
            for k in range(6)]


@pytest.mark.parametrize("nearby", range(4))
def test_oracle_lru_equals_sequential_reference(clouds, nearby):
    n_first = len(set(map(tuple, ivox_ref.voxel_key(clouds[0][:, :3], 0.5).tolist())))
    cap = int(n_first * 1.15) + 8
    o = orc.IVox(0.5, nearby, cap)
    ref = ivox_map_ref.IVoxMapRef(0.5, cap)
    rng = np.random.default_rng(nearby)
    seen, evicted = set(), False
    for k, c in enumerate(clouds):
        c = c[rng.permutation(len(c))]
        o.add(c)
        ref.add(c)
        assert o.num_voxels == ref.num_voxels and o.num_points == len(ref.points), k
        keys = set(ref.voxels)
        evicted |= bool(seen - keys)
        seen |= keys
        q = c[rng.integers(0, len(c), 300)] + rng.normal(0, 0.1, (300, 4)).astype(np.float32)
        out, found = o.closest(q, 5, 5.0)
        pts = ref.points
        kn = ivox_ref.knn5(pts, q[:, :3], 0.5, nearby, 5.0)
        assert np.array_equal(found, kn.found), k
        for i in range(len(q)):
            assert np.array_equal(out[i, :found[i]], pts[kn.idx[i, :kn.found[i]]]), (k, i)
    assert evicted


def _mapping_cfg(**kw):
    return default_config(FLS_P2PLANE_IVOX, localization_mode=0, **kw)


@pytest.mark.parametrize("nearby", range(4))
def test_oracle_rule_edges_equal_reference(nearby):
    s = ivox_map_ref.rule_scene()
    o = orc.Registration(_mapping_cfg(max_iterations=1, ivox_nearby=nearby, ivox_max_range=1.0))
    o.add_cloud(s.map)
    ok, T, st = o.match(s.scan, np.eye(4))
    assert ok and st.n_valid >= 50
    r = ivox_map_ref.insert_rule(s.map, s.scan, np.eye(4), T, 0.5, nearby, 1.0)
    assert np.array_equal(r.world, s.scan)  # the one step stays below fp32 rounding: every edge of the scene is met as built
    assert len(r.ties()) == 0
    ref = ivox_map_ref.IVoxMapRef(0.5, 10 ** 6)
    ref.add(s.map)
    ref.add(r.appended)
    assert o.map_points == len(ref.points) and o.map_voxels == ref.num_voxels
    assert np.array_equal(o.map_copy(), ref.lru_dump)
    cls = {k: int(r.cls[i]) for k, i in s.probes.items()}
    assert cls["none"] == cls["beyond"] == cls["axis_eq"] == 1 and cls["axis_gt"] == 2
    if nearby >= 1:
        assert cls["tie_a"] == 2 and cls["tie_b"] == 1
    if nearby >= 2:
        assert cls["eq"] == 0 and cls["eps2"] == 1
    # a Match that drops every point leaves the map as it was
    before = o.map_copy()
    ok, T, st = o.match(s.on_map, np.eye(4))
    assert ok and np.array_equal(o.map_copy(), before)


def test_rule_scene_reaches_its_edges():
    s = ivox_map_ref.rule_scene()
    for nearby in range(4):
        kn = ivox_ref.knn5(s.map, s.scan[:, :3], 0.5, nearby, 1.0)
        p = s.probes
        assert kn.run[p["none"]] == 0 and kn.found[p["none"]] == 0
        if nearby >= 1:
            assert kn.run[p["beyond"]] > 0 and kn.found[p["beyond"]] == 0
        if nearby == 3:
            assert [kn.found[p[f"few{k}"]] for k in range(1, 5)] == [1, 2, 3, 4]
        if nearby >= 2:
            assert kn.found[p["eq"]] == 5 and kn.found[p["eps2"]] == 5
        r = ivox_map_ref.insert_rule(s.map, s.scan, np.eye(4), np.eye(4), 0.5, nearby, 1.0)
        if nearby >= 1:  # rank 0 decided by visit order alone
            assert r.gap01[p["tie_a"]] == 0 and r.gap01[p["tie_b"]] == 0
        assert np.sum(r.gap45 == 0) >= 20  # corner points whose 5-NN set is decided by visit order
        assert r.axis_margin[p["axis_eq"]] == 0.0 and r.axis_margin[p["axis_gt"]] > 0.0
        if nearby >= 2:
            assert -1.1e-6 < r.near_margin[p["eq"]] < -0.9e-6 and 0.9e-6 < r.near_margin[p["eps2"]] < 1.1e-6
        assert set(r.cls.tolist()) == {0, 1, 2}
        ranks = np.flatnonzero(r.cls)
        assert np.any(np.diff(r.cls[ranks]) < 0)  # a class-2 point precedes a class-1 point in the input
        pp = ivox_ref.planar_pass(s.map, s.scan, np.eye(4), 0.1, 0.5, nearby, 1.0)
        assert pp.n_valid >= 100 and not any(pp.valid[i] for i in p.values())
        assert np.all(ivox_map_ref.insert_rule(s.map, s.on_map, np.eye(4), np.eye(4), 0.5, nearby, 1.0).cls == 0)


@pytest.mark.parametrize("nearby,res", [(0, 0.5), (1, 1.0), (2, 0.5), (3, 1.0)])
def test_oracle_stream_follows_insert_rule(world, traj, nearby, res):
    """Mapping mode with one Gauss-Newton step: the previous pose is the guess, so the rule is predicted from the oracle's own
    returned pose; its map must equal the sequential map fed with the predicted slices, voxel order and point order included."""
    o = orc.Registration(_mapping_cfg(max_iterations=1, ivox_nearby=nearby, ivox_resolution=res))
    first = synth.make_map_from_scans(world, traj[0:5:2], "vlp16", leaf=0.3)
    o.add_cloud(first)
    ref = ivox_map_ref.IVoxMapRef(res, 10 ** 6)
    ref.add(first)
    grown, ties = 0, 0
    for k in range(1, 5):
        scan = synth.voxel_downsample_np(synth.make_scan(world, traj[k], "vlp16", seed=40 + k)["points"], 0.5)
        guess = synth.perturb_pose(traj[k], dpos=0.05, drot_deg=0.5, seed=k)
        ok, T, st = o.match(scan, guess)
        assert ok, k
        r = ivox_map_ref.insert_rule(ref.points, scan, guess, T, res, nearby, 5.0)
        ties += len(r.ties())
        ref.add(r.appended)
        grown += len(r.appended)
        assert o.map_points == len(ref.points) and np.array_equal(o.map_copy(), ref.lru_dump), k
    assert grown > 0 and ties == 0
