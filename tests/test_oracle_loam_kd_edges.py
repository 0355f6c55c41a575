"""The oracle's kd-tree LOAM plug-ins (LoamPointToPlaneKdtree, LoamFull) against the brute-force reference of tests/loam_kd_ref.py on
the edge scenes of tests/loam_kd_scenes.py.  These tests prove the reference on the CPU before the GPU tests rely on it, and are the
first independent check of the oracle's corner path: its covariance, eigen-decomposition, ratio gate and point-to-line Jacobian."""
import numpy as np
import pytest

from oracle import pyoracle as orc
from tests import loam_kd_ref, loam_kd_scenes

SCENES = {s.name: s for s in loam_kd_scenes.kd_scenes() + loam_kd_scenes.full_scenes()}


def reference(s, T=None, prev=None, q_ulps=0):
    """The reference pass of scene s; the kd-tree point-to-plane map is the voxel-filtered one its tree is built on (:78)."""
    pm = s.planar_map if s.full else orc.voxel_grid(s.planar_map, s.leaf)
    return loam_kd_ref.kd_pass(pm, s.corner_map, s.planar, s.corner, s.T if T is None else T, s.full, s.thres, s.line_ratio,
                               s.plane_thres, prev, q_ulps)


def oracle_log(s, max_iterations=1):
    o = orc.Registration(s.config(max_iterations))
    if s.full:
        o.add_cloud(s.planar_map, s.corner_map)
        o.match(s.planar, s.T, corner=s.corner)
    else:
        o.add_cloud(s.planar_map)
        o.match(s.planar, s.T)
    return o.iter_log()


@pytest.mark.parametrize("name", list(SCENES))
def test_oracle_first_pass_equals_reference(name):
    s = SCENES[name]
    if not s.full:  # every map point alone in its leaf: the filtered map is the scene's map
        assert len(orc.voxel_grid(s.planar_map, s.leaf)) == len(s.planar_map)
    ref = reference(s)
    loam_kd_ref.assert_gates_clear(ref)
    loam_kd_ref.assert_sensitive(ref)
    loam_kd_ref.assert_matches(oracle_log(s)[0], ref)


def test_oracle_stale_records_equal_reference():
    """Iteration 1 of the stale scene at the oracle's own updated pose: the corner and the planar victim are rejected and contribute
    their iteration-0 records, each in its own class (the planar one counts toward n_valid, the corner one does not)."""
    s = loam_kd_scenes.full_stale()
    lg = oracle_log(s, 2)
    r0 = reference(s)
    loam_kd_ref.assert_gates_clear(r0)
    loam_kd_ref.assert_sensitive(r0)
    loam_kd_ref.assert_matches(lg[0], r0)
    r1 = reference(s, T=loam_kd_ref.next_pose(s.T, lg[0]["dx"]), prev=r0, q_ulps=1)
    stale = [(t.cls, t.i) for t in r1.terms if t.stale]
    assert stale == [("corner", 0), ("planar", len(s.planar) - 1)], stale
    loam_kd_ref.assert_sensitive(r1)
    loam_kd_ref.assert_matches(lg[1], r1)


def test_oracle_corner_decisions():
    """The oracle's corner decisions, one corner query at a time: accepted exactly where the reference's ratio margin is positive,
    and the exact ratio-3 neighbourhoods (in the rounding band) rejected."""
    for name in ("full_corners", "full_corners_far_5km"):
        s = SCENES[name]
        ref = reference(s)
        for i, ct in enumerate(ref.corner):
            one = loam_kd_scenes.KdScene(s.name, True, s.planar_map, s.planar[:0], corner_map=s.corner_map, corner=s.corner[i:i + 1])
            lg = oracle_log(one)[0]
            accepted = lg["sum_residual"] > 0
            if ct.in_band:
                assert not accepted, (name, i)  # S is exact here (dyadic deviations): lam0 == 3 lam1 and `<=` rejects
            else:
                assert accepted == ct.valid, (name, i, ct.ratio_margin)


def test_scenes_reach_their_edges():
    """Every branch the scenes are built for is reached, from the reference."""
    for name in ("kd_shells", "kd_shells_far_5km"):
        s = SCENES[name]
        pm = orc.voxel_grid(s.planar_map, s.leaf)
        ref = reference(s)
        kn = ref.knn["planar"]
        reach = [loam_kd_ref.reach(pm, ref.q["planar"][i], kn.sure[i] + kn.tied[i][:5 - len(kn.sure[i])], kn.d2[i, 4], s.cell)
                 for i in range(len(s.planar))]
        assert [r.shell5 for r in reach[:6]] == [1, 2, 3, 4, 5, 6], name
        assert [r.settle_ring for r in reach[:6]] == [1, 2, 3, 4, 5, 6], name
        assert reach[6].shell5 > loam_kd_ref.KMAX_SHELL and reach[6].settle_ring > loam_kd_ref.KMAX_SHELL, name  # the full scan
        for r in reach[7:]:  # face, edge, corner: face ~ 0, the 27-cell 5th just past the settle bound, the true 5th in ring 2
            assert r.face < 1e-3 and loam_kd_ref.SETTLE < r.r1_ratio < 1.002 and r.shell5 == 2, (name, r)
        if name.endswith("5km"):
            assert np.min(np.abs(pm[:, :3])) > 700 and np.max(np.abs(pm[:, :2])) > 4900
    # lanes: five nearest in one lane's cell; five nearest over five lanes with candidates in every lane
    s = SCENES["kd_lanes"]
    ref = reference(s)
    kn = ref.knn["planar"]
    lanes = [loam_kd_ref.reach(orc.voxel_grid(s.planar_map, s.leaf), ref.q["planar"][i], kn.sure[i] + kn.tied[i][:5 - len(kn.sure[i])], kn.d2[i, 4],
                               s.cell).lanes for i in range(2)]
    assert lanes[0] == [4] * 5 and len(set(lanes[1])) == 5, lanes
    assert {loam_kd_ref.stencil_lane(o) for o in loam_kd_scenes.STENCIL} == set(range(8))
    # ties: four at rank 1, eight at rank 5, and no other resolution-dependent term
    kn = reference(SCENES["kd_ties"]).knn["planar"]
    assert len(kn.first[0]) == 4 and len(kn.sure[0]) == 4 and len(kn.tied[0]) == 8
    # map sizes: nothing with 4 points, every query with 5 and 6
    assert reference(SCENES["kd_map4"]).n_valid == 0
    assert reference(SCENES["kd_map5"]).n_valid == 3 and reference(SCENES["kd_map6"]).n_valid == 3
    # LoamFull gate: d4 at fp32(thres) and one ulp either side; thres = 0.1 rejects fp32(0.1) itself
    for name, want in (("full_gate_1.0", [True, False, True]), ("full_gate_0.1", [False, False, True])):
        g = reference(SCENES[name]).gate["planar"]
        assert [u for _, u in g[:6]] == [0, 1, -1] * 2 and [ok for ok, _ in g[:6]] == want * 2, (name, g)
        assert all(ok for ok, _ in g[6:]), name  # the 5th across a face, just inside sqrt(thres)
    g = reference(SCENES["full_gate_far_5km"]).gate["planar"]
    assert len(g) == 3 and all(ok for ok, _ in g)
    # corners: collinear (lam1 = lam2 = 0), isotropic, lam0 = lam1, the exact ratio in the band, 2 fp32 ulps either side out of it
    for name in ("full_corners", "full_corners_far_5km"):
        c = reference(SCENES[name]).corner
        z = [1e-40 * t.lam[0] for t in c]  # zero to the reference's 50 digits
        assert c[0].valid and c[0].lam[1] < z[0] and c[0].lam[2] < z[0]
        assert not c[1].valid and c[1].lam[0] - c[1].lam[2] < z[1]
        assert not c[2].valid and c[2].lam[0] - c[2].lam[1] < z[2] and c[2].lam[2] < z[2] and c[2].lam[1] > 0.1 * c[2].lam[0]
        assert c[3].in_band and abs(c[3].ratio_margin) < z[3]
        assert c[4].valid and not c[4].in_band and not c[5].valid and not c[5].in_band
        assert 0 < c[4].ratio_margin < 1e-2 * c[4].lam[0] and 0 < -c[5].ratio_margin < 1e-2 * c[5].lam[0]
        assert c[6].valid
    assert reference(SCENES["full_on_line"]).corner[0].on_line
