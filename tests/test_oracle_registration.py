"""Oracle pinning (CPU): the three registration plug-ins and the feature extractor against the committed golden
vectors (tests/golden/, produced by tests/golden/make_golden.py) and through size-independent properties —
ground-truth recovery, rigid re-framing invariance, permutation invariance, the documented quirks."""
import os

import numpy as np
import pytest

from funny_lidar_slam_b200 import FLS_ICP_P2P, FLS_NDT, FLS_P2PLANE_IVOX, default_config, synth
from funny_lidar_slam_b200._abi import FLS_FLAG_ITER_LOG
from oracle import pyoracle as orc
from tests import frontend_ref

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _run(method, scene, scan, guess, **kw):
    r = orc.Registration(default_config(method, flags=FLS_FLAG_ITER_LOG, **kw))
    r.add_cloud(scene["map"])
    ok, T, st = r.match(scan, guess)
    return r, ok, T, st


@pytest.mark.parametrize("name,method,guess_key", [("p2plane_scene16", FLS_P2PLANE_IVOX, "guess"), ("ndt_scene16", FLS_NDT, "guess_small"),
                                                   ("icp_scene16", FLS_ICP_P2P, "guess")])
def test_against_golden(scene16, name, method, guess_key):
    ref = np.load(os.path.join(GOLD, name + ".npz"))
    # the fixtures only make sense on bit-identical inputs
    assert float(np.sum(scene16["scan"].astype(np.float64))) == float(ref["scan_checksum"])
    assert float(np.sum(scene16["map"].astype(np.float64))) == float(ref["map_checksum"])
    r, ok, T, st = _run(method, scene16, scene16["scan"], scene16[guess_key])
    assert ok == bool(ref["ok"]) and st.iterations == int(ref["iters"]) and st.n_valid == int(ref["n_valid"])
    log = r.iter_log()
    assert log[0]["n_valid"] == int(ref["n_valid0"])
    assert np.allclose(log[0]["H"], ref["H0"], rtol=1e-12, atol=1e-9)
    assert np.allclose(log[0]["g"], ref["g0"], rtol=1e-12, atol=1e-9)
    assert np.allclose(T, ref["T"], atol=1e-10)


def test_features_and_voxelgrid_golden(world, traj, scene16):
    ref = np.load(os.path.join(GOLD, "features_vlp16.npz"))
    proj = synth.make_projected_scan(world, traj[7], kind="spin", sensor="vlp16", seed=12)
    assert float(np.sum(proj["depth"].astype(np.float64))) == float(ref["depth_checksum"])
    ci, pi, _ = orc.extract_features(proj["depth"], proj["col"], len(proj["ordered"]), proj["row_start"], proj["row_end"], 1.0, 0.1)
    assert np.array_equal(ci, ref["corner_idx"]) and np.array_equal(pi, ref["planar_idx"])
    vref = np.load(os.path.join(GOLD, "voxelgrid_scene16_0p4.npz"))
    vg = orc.voxel_grid(scene16["scan"], 0.4)
    assert len(vg) == int(vref["n"]) and float(np.sum(vg.astype(np.float64))) == float(vref["checksum"])
    assert np.array_equal(vg[:8], vref["first"]) and np.array_equal(vg[-8:], vref["last"])


def test_ground_truth_recovery(scene16):
    """Known ground-truth pose of the synthetic scan => recovered pose error << 1e-2 m for the well-posed estimators."""
    _, ok, T, _ = _run(FLS_P2PLANE_IVOX, scene16, scene16["scan"], scene16["guess"])
    assert ok and synth.pose_error(T, scene16["truth"])[0] < 5e-3
    _, ok, T, _ = _run(FLS_NDT, scene16, scene16["scan"], scene16["guess_small"])
    assert ok and synth.pose_error(T, scene16["truth"])[0] < 5e-3


def test_rigid_reframing_invariance(scene16):
    """Moving map and guess by the same rigid transform moves the estimate by that transform (ICP: exact k-NN,
    voxel filters excepted by choosing leafs below the data spacing)."""
    G = synth.se3([3.0, -2.0, 0.5], [0.0, 0.0, 0.3])
    sc = dict(scene16)
    kw = dict(source_cloud_filter_size=0.02, map_cloud_filter_size=0.02)
    scan = scene16["scan"][::3]
    mp = scene16["map"][::2]
    _, ok1, T1, _ = _run(FLS_ICP_P2P, dict(map=mp), scan, scene16["guess"], **kw)
    mp2 = synth.transform_points(mp, G)
    _, ok2, T2, _ = _run(FLS_ICP_P2P, dict(map=mp2), scan, G @ scene16["guess"], **kw)
    assert ok1 == ok2
    dt, dr = synth.pose_error(G @ T1, T2)
    assert dt < 2e-3 and dr < 2e-4, (dt, dr)


def test_input_order_invariance(scene16):
    """The sums are order-free up to rounding: permuting the scan changes nothing beyond ~1e-9."""
    scan = scene16["scan"][:6000]
    perm = np.random.default_rng(4).permutation(len(scan))
    _, ok1, T1, s1 = _run(FLS_P2PLANE_IVOX, scene16, scan, scene16["guess"])
    _, ok2, T2, s2 = _run(FLS_P2PLANE_IVOX, scene16, scan[perm], scene16["guess"])
    assert ok1 == ok2 and s1.iterations == s2.iterations and s1.n_valid == s2.n_valid
    assert np.allclose(T1, T2, atol=1e-9)


def test_match_writes_T_on_failure_and_returns_false(scene16):
    far = scene16["guess"].copy()
    far[:3, 3] += 400.0
    for method in (FLS_P2PLANE_IVOX, FLS_NDT):
        r, ok, T, st = _run(method, scene16, scene16["scan"][:2000], far)
        assert ok is False
        assert np.allclose(T, far, atol=1e-9)  # nothing matched: pose unchanged but still written
    # IcpOptimized: no correspondence => H = 0 => det == 0 => every iteration `continue`s, never converges
    r, ok, T, st = _run(FLS_ICP_P2P, scene16, scene16["scan"][:2000], far)
    assert ok is False and st.iterations == 30 and np.allclose(T, far, atol=1e-12)


def test_quirk_squared_distance_vs_unsquared_threshold(scene16):
    """[quirk 4] IcpOptimized compares the SQUARED nn distance with max_correspond_distance: raising the threshold from
    0.25 to 0.5 must admit points whose nn distance lies in (0.5, 0.707], not (0.25, 0.5]."""
    scan = scene16["scan"][:3000]
    counts = []
    for thr in (0.25, 0.5):
        r, ok, T, st = _run(FLS_ICP_P2P, scene16, scan, scene16["guess"], icp_max_correspond_distance=thr, max_iterations=1)
        counts.append(r.iter_log()[0]["n_valid"])
    src = orc.voxel_grid(scan, 0.4)
    q = orc.transform_f(src, scene16["guess"])
    tree = orc.ExactKnn(orc.voxel_grid(scene16["map"], 0.4))
    _, d2, _ = tree.search(q, 1)
    assert counts[0] == int(np.sum(d2[:, 0] <= 0.25)) and counts[1] == int(np.sum(d2[:, 0] <= 0.5))


def test_ndt_voxel_statistics_match_numpy(scene16):
    """First-scan / localization-mode voxels: mean, (n-1) covariance, information = (cov + 1e-3 I)^-1, single point => 100 I."""
    cfg = default_config(FLS_NDT)
    r = orc.Registration(cfg)
    r.add_cloud(scene16["map"])
    keys, mu, info, est = r.ndt_dump()
    assert np.all(est == 1) and len(keys) == r.map_voxels
    filt = orc.voxel_grid(scene16["map"], cfg.source_cloud_filter_size).astype(np.float64)
    k = (filt[:, :3] * (1.0 / cfg.ndt_voxel_size)).astype(np.int32)  # C truncation  [quirk 5]
    for vi in np.random.default_rng(2).choice(len(keys), 25, replace=False):
        pts = filt[np.all(k == keys[vi], axis=1), :3]
        assert len(pts) >= 1
        if len(pts) == 1:
            assert np.allclose(mu[vi], pts[0]) and np.allclose(info[vi], 100.0 * np.eye(3))
        else:
            assert np.allclose(mu[vi], pts.mean(0), atol=1e-9)
            cov = np.cov(pts.T, ddof=1).reshape(3, 3)
            assert np.allclose(info[vi], np.linalg.inv(cov + 1e-3 * np.eye(3)), rtol=1e-7, atol=1e-7)


def test_feature_extractor_properties(world, traj):
    proj = synth.make_projected_scan(world, traj[3], kind="spin", sensor="vlp16", seed=21)
    n = len(proj["ordered"])
    ci, pi, _ = orc.extract_features(proj["depth"], proj["col"], n, proj["row_start"], proj["row_end"], 1.0, 0.1)
    # <= 20 corners per block, 6 blocks per ring
    assert len(ci) <= 120 * proj["rows"] and len(set(ci.tolist())) == len(ci)
    # corners never reappear as planar points; every planar index lies inside some ring's [start, end] range
    assert not set(ci.tolist()) & set(pi.tolist())
    lo = np.min(proj["row_start"])
    hi = np.max(proj["row_end"])
    assert pi.min() >= lo and pi.max() <= hi
    # [quirk 10] the inclusive block_end visit duplicates the seam element between consecutive blocks
    assert len(pi) > len(set(pi.tolist()))
    # raising the corner threshold can only remove corners
    ci2, _, _ = orc.extract_features(proj["depth"], proj["col"], n, proj["row_start"], proj["row_end"], 5.0, 0.1)
    assert len(ci2) <= len(ci)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_feature_extractor_against_literal_python_restatement(seed):
    rng = np.random.default_rng(seed)
    counts = [int(c) for c in rng.integers(60, 420, 5)] + [11, 30]
    depth, col = [], []
    for c in counts:
        base = 8.0 + 4.0 * np.sin(np.arange(c) / rng.uniform(8, 30)) + rng.normal(0, 0.02, c)
        for _ in range(c // 60):  # depth jumps: occlusions both ways
            k = int(rng.integers(0, c))
            base[k:] += rng.choice([-1.0, 1.0]) * rng.uniform(0.4, 2.0)
        depth.append(np.abs(base) + 2.0)
        step = rng.choice([1, 1, 1, 2, 12], c)  # occasional column gaps > 10 break the suppression reach
        col.append(np.cumsum(step))
    depth = np.concatenate(depth).astype(np.float32)
    col = np.concatenate(col).astype(np.int32)
    n = len(depth)
    ends = np.cumsum(counts)
    rs = (ends - np.array(counts) + 5).astype(np.int32)
    re = (ends - 6).astype(np.int32)
    for ct, pt in ((1.0, 0.1), (0.05, 0.01), (0.2, 5.0)):
        oc, op, _ = orc.extract_features(depth, col, n, rs, re, ct, pt)
        lc, lp, _ = frontend_ref.features(depth, col, n, rs, re, ct, pt)
        assert np.array_equal(oc, lc), (seed, ct, pt)
        assert np.array_equal(op, lp), (seed, ct, pt)
    assert len(oc) > 0 and len(op) > 100
