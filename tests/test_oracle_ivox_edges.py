"""The oracle's LOAM-iVox k-NN and first PlanerMatch pass against the brute-force references of tests/ivox_ref.py, on the
adversarial scenes of tests/ivox_scenes.py, for every stencil and for the fast and the range-gated selection.  These
tests prove the references on the CPU before the GPU tests rely on them."""
import numpy as np
import pytest

from funny_lidar_slam_b200 import FLS_P2PLANE_IVOX, default_config
from funny_lidar_slam_b200._abi import FLS_FLAG_ITER_LOG
from oracle import pyoracle as orc
from tests import ivox_ref, ivox_scenes

SCENES = {s.name: s for s in ivox_scenes.all_scenes()}
CASES = [(name, cfg, nearby) for name, s in SCENES.items() for cfg in s.configs for nearby in range(4)]
IDS = [f"{n}-res{c[0]}-r{c[1]}-nb{k}" for n, c, k in CASES]


def oracle_knn(scene, res, max_range, nearby):
    iv = orc.IVox(res, nearby)
    iv.add(scene.map)
    out, found = iv.closest(scene.scan, 5, max_range)
    return out, found


def oracle_pass(scene, res, max_range, nearby):
    cfg = default_config(FLS_P2PLANE_IVOX, flags=FLS_FLAG_ITER_LOG, max_iterations=1, localization_mode=1, ivox_resolution=res,
                         ivox_max_range=max_range, ivox_nearby=nearby)
    r = orc.Registration(cfg)
    r.add_cloud(scene.map)
    r.match(scene.scan, np.eye(4))
    return r.iter_log()[0], cfg


@pytest.mark.parametrize("name,cfg,nearby", CASES, ids=IDS)
def test_oracle_knn_equals_brute_force(name, cfg, nearby):
    s = SCENES[name]
    ref = ivox_ref.knn5(s.map, s.scan[:, :3], cfg[0], nearby, cfg[1])
    out, found = oracle_knn(s, cfg[0], cfg[1], nearby)
    assert np.array_equal(found, ref.found)
    for i in range(len(s.scan)):
        # the oracle pins the full (d2, visit order) order: index for index, duplicates told apart by their intensity
        assert np.array_equal(out[i, :found[i], 3].astype(np.int64), ref.idx[i, :ref.found[i]]), i


@pytest.mark.parametrize("name,cfg,nearby", CASES, ids=IDS)
def test_oracle_first_pass_equals_reference(name, cfg, nearby):
    s = SCENES[name]
    lg, c = oracle_pass(s, cfg[0], cfg[1], nearby)
    ref = ivox_ref.planar_pass(s.map, s.scan, np.eye(4), c.point_to_planar_thres, cfg[0], nearby, cfg[1])
    ivox_ref.assert_gates_clear(ref)
    ivox_ref.assert_sensitive(ref)
    assert lg["n_valid"] == ref.n_valid
    ivox_ref.assert_matches(lg["H"], lg["g"], ref)


def test_scenes_reach_their_branches():
    """The scenes hold what they are built for (with the default NEARBY18 stencil unless noted)."""
    fast, gated = ivox_scenes.FAST, ivox_scenes.GATED

    def k(name, cfg=fast, nearby=2):
        s = SCENES[name]
        return ivox_ref.knn5(s.map, s.scan[:, :3], cfg[0], nearby, cfg[1])

    r = k("s1_dense_staged")
    assert np.any((r.run > 64) & (r.run <= 352))
    assert np.all(k("s1_dense_global").run > 352)
    r = k("s1_mixed_warps")
    assert np.all((r.run > 5) & (r.run <= 64)) and r.run[:32].sum() > 352
    r = k("s2_exact_ties")
    assert np.sum(r.gap01 == 0) >= 20 and np.sum(r.gap45 == 0) >= 20
    r = k("s3_near_ties")
    assert np.sum((r.gap01 >= 1) & (r.gap01 <= 64)) >= 5 and np.sum((r.gap45 >= 1) & (r.gap45 <= 64)) >= 5
    s, swapped = SCENES["s3_near_ties"], 0
    for i in range(len(s.scan)):  # ranks 1/2 on adjacent 26-bit prefixes whose contracted distances are swapped
        pre = [int(np.asarray(r.d2[i, j]).view(np.int32)) >> 6 for j in (0, 1)]
        fma = [int(np.asarray(ivox_scenes.fma_dist2(s.map[r.idx[i, j]], s.scan[i])).view(np.int32)) >> 6 for j in (0, 1)]
        swapped += pre[1] == pre[0] + 1 and fma[0] == pre[1] and fma[1] == pre[0]
    assert swapped >= 8
    for name, cfg, nb in (("s4_range_gate", gated, 2), ("s4_range_gate_coarse", ivox_scenes.GATED_COARSE, 3)):
        s = SCENES[name]
        r = k(name, cfg, nb)
        r2 = np.float32(cfg[1]) * np.float32(cfg[1])
        d = ivox_ref.dist2(s.map[:, :3], s.scan[:, None, :3])
        assert {np.sum(d == r2), np.sum(d == np.nextafter(r2, np.float32(0))), np.sum(d == np.nextafter(r2, np.float32(np.inf)))} == {3}
        assert list(r.found) == [3, 5, 5]  # 2 inner + the one below; 4 + 1; 5 closer ones
    r = k("s4_range_gate_exact", gated)
    assert r.run[0] > 64 and r.found[0] == 4
    s = SCENES["s4_range_gate_exact"]
    assert np.sum(ivox_ref.dist2(s.map[:, :3], s.scan[0, :3]) == np.float32(1.0)) == 1
    s = SCENES["s5_voxel_edges"]
    assert np.all(np.abs(np.abs(s.scan[:, :2] / 0.5) % 1.0 - 0.5) == 0.0)
    assert not np.array_equal(ivox_ref.voxel_key(s.scan[:, :3], 0.5), np.round(s.scan[:, :3] * np.float32(2.0)))
    r = k("s6_thin")
    assert list(r.found) == [1, 2, 3, 4, 0, 0] and list(r.run[-2:]) == [0, 0]
    s = SCENES["s7_plane_fit"]
    ref = ivox_ref.planar_pass(s.map, s.scan, np.eye(4))
    assert set(ref.rank[ref.rank >= 0]) == {1, 2, 3}
    pm = ref.plane_margin
    assert np.sum(np.abs(pm - 0.01) < 1e-6) == 1 and np.sum(np.abs(pm + 0.01) < 1e-6) == 1
    nm = ref.near_margin
    assert np.sum(np.abs(nm - 0.1) < 1e-3) == 1 and np.sum(np.abs(nm + 0.1) < 1e-3) == 1
    # near-collinear and far-away neighbourhoods whose normal equations lose more than 7 digits take the GPU's QR fallback
    shares = [ivox_ref.ldlt_share(s.map[ref.knn.idx[i], :3]) for i in np.nonzero(ref.rank == 3)[0]]
    assert sum(sh < 0.1 * ivox_ref.LDLT_GUARD for sh in shares) >= 6 and sum(sh > 10 * ivox_ref.LDLT_GUARD for sh in shares) >= 4


def test_oracle_honours_ivox_max_range():
    """IVox.closest and Registration both apply ivox_max_range (ivox_map.h:58 upstream), not a fixed 5 m."""
    s = ivox_scenes.s4_range_gate()
    ref = ivox_ref.knn5(s.map, s.scan[:, :3], 0.5, 2, 1.0)
    out, found = oracle_knn(s, 0.5, 1.0, 2)
    assert list(found) == list(ref.found) == [3, 5, 5]
    out5, found5 = oracle_knn(s, 0.5, 5.0, 2)
    assert list(found5) == [5, 5, 5]
    # Registration: a patch whose neighbours sit 1.2 m from the scan points is matched at max_range 5 and not at max_range 1
    rng = np.random.default_rng(5)
    mp = np.zeros((60, 4), np.float32)
    mp[:, 0] = rng.uniform(4.0, 5.0, 60)
    mp[:, 1] = rng.uniform(-0.5, 0.5, 60)
    mp[:, 2] = 0.0
    scan = np.zeros((20, 4), np.float32)
    scan[:, 0] = rng.uniform(4.2, 4.8, 20)
    scan[:, 1] = rng.uniform(-0.3, 0.3, 20)
    scan[:, 2] = 1.2  # 1.2 m above the plane: in the NEARBY26 stencil at 2 m voxels, out of range at 1 m
    got = {}
    for r_max in (5.0, 1.0):
        cfg = default_config(FLS_P2PLANE_IVOX, flags=FLS_FLAG_ITER_LOG, max_iterations=1, ivox_resolution=2.0, ivox_nearby=3,
                             ivox_max_range=r_max)
        o = orc.Registration(cfg)
        o.add_cloud(mp)
        o.match(scan, np.eye(4))
        ref = ivox_ref.planar_pass(mp, scan, np.eye(4), cfg.point_to_planar_thres, 2.0, 3, r_max)
        got[r_max] = o.iter_log()[0]["n_valid"]
        assert got[r_max] == ref.n_valid
    assert got[5.0] > 0 and got[1.0] == 0


def test_rounding_level_rank_follows_the_shared_qr_rule():
    """S7': where the remaining QR column is rounding noise, the rank is whatever the arithmetic decides.  The oracle's QR is
    colpiv_qr bit for bit (the arithmetic fls_plane.cuh shares), the GPU cannot take its LDL^T path on these neighbourhoods,
    both rank decisions occur, and the oracle's first pass equals planar_pass under that rule."""
    s = ivox_scenes.s7_rounding_rank()
    r = ivox_ref.knn5(s.map, s.scan[:, :3], 0.5, 2, 5.0)
    assert np.all(r.found == 5)
    ranks = []
    for i in range(len(s.scan)):
        A = s.map[r.idx[i], :3].astype(np.float64)
        c, rk = ivox_ref.colpiv_qr(A)
        assert np.array_equal(orc.lstsq53(A, -np.ones(5)), c), i
        assert ivox_ref.ldlt_share(A) < 0.1 * ivox_ref.LDLT_GUARD, i
        ranks.append(rk)
    assert {1, 2} <= set(ranks)
    rng = np.random.default_rng(3)  # five fp32 copies of random points in [-20, 20]^3: the decision is a coin flip
    flips = set()
    for _ in range(200):
        A = np.tile(rng.uniform(-20, 20, 3).astype(np.float32).astype(np.float64), (5, 1))
        c, rk = ivox_ref.colpiv_qr(A)
        assert np.array_equal(orc.lstsq53(A, -np.ones(5)), c)
        flips.add(rk)
    assert len(flips) >= 2
    for nearby in range(4):
        lg, cfg = oracle_pass(s, 0.5, 5.0, nearby)
        ref = ivox_ref.planar_pass(s.map, s.scan, np.eye(4), cfg.point_to_planar_thres, 0.5, nearby, 5.0, qr_rule=True)
        ivox_ref.assert_gates_clear(ref)
        ivox_ref.assert_sensitive(ref)
        assert lg["n_valid"] == ref.n_valid and ref.n_valid >= 40
        ivox_ref.assert_matches(lg["H"], lg["g"], ref)
