"""The oracle's IncrementalNDT map and first NDT / ICP passes against the references of tests/ndt_ref.py and tests/icp_ref.py, on the
scenes of tests/ndt_icp_scenes.py.  These tests prove the references on the CPU before the GPU tests rely on them, and are the first
independent check of the oracle's carry, merge, clamp and freeze branches."""
import numpy as np
import pytest

from oracle import pyoracle as orc
from tests import icp_ref, ndt_icp_scenes, ndt_ref

NDT = {s.name: s for s in ndt_icp_scenes.ndt_scenes()}
ICP = {s.name: s for s in ndt_icp_scenes.icp_scenes()}


def oracle_dump(o, max_pts):
    """The oracle's voxels sorted by key, in the layout of fls_get_ndt_voxels."""
    v = o.ndt_voxels()
    order = np.lexsort(v["key"].T[::-1])
    I = v["info"][order]
    frozen = (v["estimated"][order] == 1) & (v["num_points"][order] > max_pts)
    return dict(key=v["key"][order], mu=v["mu"][order], estimated=v["estimated"][order], num_points=v["num_points"][order],
                carry_count=np.where(frozen, 0, v["pending"][order]),
                info=np.stack([I[:, 0, 0], I[:, 0, 1], I[:, 0, 2], I[:, 1, 1], I[:, 1, 2], I[:, 2, 2]], 1))


def ndt_reference(s):
    ref = ndt_ref.NdtRef(s.voxel, s.min_pts, s.max_pts, s.capacity, s.leaf, s.localization)
    for c in s.calls:
        ref.add_cloud(c)
    return ref


@pytest.mark.parametrize("name", list(NDT))
def test_oracle_ndt_first_pass_equals_reference(name):
    s = NDT[name]
    o = orc.Registration(s.config())
    for c in s.calls:
        o.add_cloud(c)
    ref = ndt_reference(s)
    ndt_ref.assert_dump_matches(oracle_dump(o, s.max_pts), ref.dump())
    o.match(s.scan, s.T)
    p = ndt_ref.ndt_pass(ref, s.scan, s.T, s.thres)
    ndt_ref.assert_gates_clear(p)
    ndt_ref.assert_sensitive(p)
    lg = o.iter_log()[0]
    ndt_ref.assert_matches(lg["H"], lg["g"], lg["n_valid"], p)
    assert p.n_valid > 0


def test_oracle_ndt_stream_equals_reference():
    """Mapping stream: the oracle's map equals the sequential reference after every AddCloudToLocalMap call, through every branch
    of UpdateVoxel and across the capacity."""
    s = ndt_icp_scenes.ndt_stream()
    o = orc.Registration(s.config())
    ref = ndt_ref.NdtRef(s.voxel, s.min_pts, s.max_pts, s.capacity, s.leaf, s.localization)
    for k, c in enumerate(s.calls):
        o.add_cloud(c)
        ref.add_cloud(c)
        d = ref.dump()
        ndt_ref.assert_dump_matches(oracle_dump(o, s.max_pts), d)
        assert o.map_voxels == len(d["key"]), k


@pytest.mark.parametrize("name", list(ICP))
def test_oracle_icp_first_pass_equals_reference(name):
    s = ICP[name]
    o = orc.Registration(s.config())
    o.add_cloud(s.map)
    o.match(s.scan, s.T)
    p = icp_ref.icp_pass(s.map, s.scan, s.T, s.max_corr, 0.01, 0.01)
    icp_ref.assert_gates_clear(p, tie_ok=s.ties)
    icp_ref.assert_sensitive(p)
    lg = o.iter_log()[0]
    icp_ref.assert_matches(lg["H"], lg["g"], lg["n_valid"], p)


def test_oracle_fitness_equals_brute_force():
    """GetFitnessScore of ICP at the identity pose (no correspondence at max_corr 0.1, so the pose stays) on the fitness scene."""
    from funny_lidar_slam_b200 import FLS_ICP_P2P, default_config
    mp, sc = ndt_icp_scenes.fitness_scene()
    o = orc.Registration(default_config(FLS_ICP_P2P, max_iterations=1, icp_max_correspond_distance=0.1, source_cloud_filter_size=0.01,
                                        map_cloud_filter_size=0.01))
    o.add_cloud(mp)
    _, T, _ = o.match(np.vstack([sc] * 4), np.eye(4))
    assert np.array_equal(T, np.eye(4))
    for r in (1.0, 2.0, 0.5):
        want, _, _ = icp_ref.fitness(orc.voxel_grid(mp, 0.01), orc.voxel_grid(np.vstack([sc] * 4), 0.01), T, r)
        assert abs(o.fitness(r) - want) <= 1e-6 * max(1.0, abs(want)), r


def test_scenes_reach_their_edges():
    """The scenes hold what they are built for: every gate has points within a few ulps on each side, every branch is taken."""
    # NDT keys: queries within a few ulps of a voxel face, on both sides, at v = 1.0 and 0.3
    for name, v in (("ndt_axes", 1.0), ("ndt_v03", 0.3)):
        s = NDT[name]
        src = orc.voxel_grid(s.scan, s.leaf)[:, :3].astype(np.float64)
        u = src * (1.0 / v)
        frac = u - np.round(u)
        near = np.abs(frac) < 1e-6
        assert np.sum(near & (frac > 0)) >= 6 and np.sum(near & (frac < 0)) >= 6, name
    s = NDT["ndt_axes"]  # truncation and floor disagree on the map and on queries
    assert np.any(np.trunc(s.calls[0][:, :3]) != np.floor(s.calls[0][:, :3])) and np.any(np.trunc(s.scan[:, :3]) != np.floor(s.scan[:, :3]))
    # chi: exactly at the threshold and on both sides, computed exactly; unestimated voxels inside the stencil
    p = ndt_ref.ndt_pass(ndt_reference(NDT["ndt_chi_single"]), NDT["ndt_chi_single"].scan, np.eye(4), 6.25)
    m = [c[2] for c in p.chi_margin if c[3] == 0.0]
    assert 0.0 in m and sum(x > 0 for x in m) >= 3 and sum(x < 0 for x in m) >= 3
    assert max(abs(x) for x in m) < 1e-3  # three fp32 ulps of the query move chi by about 3e-4
    s = NDT["ndt_unestimated"]
    assert ndt_ref.ndt_pass(ndt_reference(s), s.scan, s.T, s.thres).unestimated_hits >= 10
    s = NDT["ndt_far_5km"]
    assert np.min(np.abs(s.calls[0][:, :3])) > 4000
    # the stream: every branch, frozen voxels, the clamp, an eviction re-created in its own call
    s = ndt_icp_scenes.ndt_stream()
    ref = ndt_ref.NdtRef(s.voxel, s.min_pts, s.max_pts, s.capacity, s.leaf, s.localization)
    seen, recreated, evicted, clamped = set(), 0, 0, 0
    for c in s.calls:
        ev = ref.add_cloud(c)
        seen |= set(ev["branches"])
        recreated += len(ev["recreated"])
        evicted += len(ev["evicted"])
        assert len(ref.data) < s.capacity
    assert {"first_scan", "first_scan_single", "carry", "estimate", "merge", "frozen"} <= seen
    assert recreated >= 1 and evicted >= 5
    for v in ref.data.values():
        if v.branch in ("merge", "frozen"):
            lam = np.linalg.eigvalsh(v.sigma)
            clamped += lam[0] < 1e-3 * lam[2]
    assert clamped >= 6
    # ICP: d2 at max_corr and one fp32 ulp either side, for every threshold; ties of 8 and 4 points; nothing at the far guess
    for mc in (0.25, 1.0, 2.0):
        s = ICP[f"icp_gate_{mc}"]
        p = icp_ref.icp_pass(s.map, s.scan, s.T, mc, 0.01, 0.01)
        assert {0, 1, -1} <= set(p.gate_ulps.tolist())
    assert [len(t) for t in icp_ref.icp_pass(ICP["icp_ties"].map, ICP["icp_ties"].scan, np.eye(4), 1.0, 0.01, 0.01).nn.ties] == [8]
    assert icp_ref.icp_pass(ICP["icp_far"].map, ICP["icp_far"].scan, ICP["icp_far"].T, 1.0, 0.01, 0.01).n_valid == 0
    mp, sc = ndt_icp_scenes.fitness_scene()
    _, _, gate = icp_ref.fitness(mp, sc, np.eye(4), 1.0)
    assert {0, 1, -1} <= set(gate.tolist())
