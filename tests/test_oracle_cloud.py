"""Oracle pinning (CPU): the three un-vendored PCL primitives and the iVox map, against independent restatements
(numpy / scipy / brute force).  SURVEY.md §8c: the reference has no test at these boundaries."""
import numpy as np
import pytest
from scipy.spatial import cKDTree

from oracle import pyoracle as orc
from tests import frontend_ref


def test_voxel_grid_matches_independent_restatement():
    rng = np.random.default_rng(11)
    pts = np.concatenate([rng.uniform(-6, 6, (3000, 3)), rng.uniform(0, 100, (3000, 1))], 1).astype(np.float32)
    for leaf in (0.3, 0.5, 1.0):
        got = orc.voxel_grid(pts, leaf)
        want, _ = frontend_ref.voxel_grid(pts, leaf)
        assert got.shape == want.shape
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_voxel_grid_properties(scene16):
    scan = scene16["scan"]
    out = orc.voxel_grid(scan, 0.4)
    assert 0 < len(out) < len(scan)
    # idempotent up to cell re-assignment: a second pass can only merge, never grow
    assert len(orc.voxel_grid(out, 0.4)) <= len(out)
    # every centroid lies inside the bounding box
    assert np.all(out[:, :3] >= scan[:, :3].min(0) - 1e-4) and np.all(out[:, :3] <= scan[:, :3].max(0) + 1e-4)
    # leaf too small => PCL returns the input unchanged
    wide = np.array([[-500, -500, -500, 1], [500, 500, 500, 2]], np.float32)
    assert np.array_equal(orc.voxel_grid(wide, 0.01), wide)
    assert len(orc.voxel_grid(np.zeros((0, 4), np.float32), 0.5)) == 0


def test_exact_knn_matches_ckdtree(scene16):
    mp = scene16["map"][:20000]
    q = scene16["scan"][:1500].copy()
    q[:, :3] += 40.0 * (np.random.default_rng(0).random((len(q), 3)) - 0.5).astype(np.float32)  # some far queries too
    tree = orc.ExactKnn(mp, cell=1.0)
    idx, d2, found = tree.search(q, 5)
    assert np.all(found == 5)
    kd = cKDTree(mp[:, :3].astype(np.float64))
    dd, ii = kd.query(q[:, :3].astype(np.float64), k=5)
    # same neighbour sets (ties have measure zero on this data); distances are fp32 squared L2
    assert np.array_equal(np.sort(idx, 1), np.sort(ii, 1))
    assert np.allclose(d2, dd ** 2, rtol=1e-5, atol=1e-6)
    assert np.all(np.diff(d2, axis=1) >= 0)


def test_transforms_follow_the_reference_rounding():
    rng = np.random.default_rng(5)
    pts = np.concatenate([rng.uniform(-80, 80, (2000, 3)), np.ones((2000, 1))], 1).astype(np.float32)
    from funny_lidar_slam_b200 import synth
    T = synth.se3([10.5, -3.25, 1.8], [0.02, -0.01, 0.7])
    # pcl::transformPoint with a double transform: fp64 maths, one rounding
    want_d = (pts[:, :3].astype(np.float64) @ T[:3, :3].T + T[:3, 3]).astype(np.float32)
    got_d = orc.transform_d(pts, T)[:, :3]
    assert np.max(np.abs(got_d - want_d)) <= np.spacing(np.float32(100.0))
    # TransformPoint with R, t cast to float FIRST: pure fp32 maths
    Rf, tf = T[:3, :3].astype(np.float32), T[:3, 3].astype(np.float32)
    want_f = ((Rf[:, 0] * pts[:, 0:1] + Rf[:, 1] * pts[:, 1:2]) + Rf[:, 2] * pts[:, 2:3]) + tf
    got_f = orc.transform_f(pts, T)[:, :3]
    assert np.array_equal(got_f, want_f.astype(np.float32))


def _ivox_bruteforce(mp, q, res, offsets, K, max_range):
    inv = np.float32(1.0) / np.float32(res)
    key = lambda p: tuple(np.round(p[:3] * inv).astype(np.int64))  # noqa: E731  (np.round is half-to-even: avoided below)
    def rnd(v):  # std::round: half away from zero
        return np.sign(v) * np.floor(np.abs(v) + np.float32(0.5))
    keys = rnd(mp[:, :3] * inv).astype(np.int64)
    qk = rnd(q[:3] * inv).astype(np.int64)
    cand = []
    order = 0
    for off in offsets:
        sel = np.nonzero(np.all(keys == qk + off, axis=1))[0]
        loc = []
        for j in sel:
            d = mp[j, :3] - q[:3]
            d2 = np.float32(np.float32(d[0] * d[0]) + np.float32(d[1] * d[1])) + np.float32(d[2] * d[2])
            if float(d2) < float(np.float32(max_range) * np.float32(max_range)):
                loc.append((float(d2), order, j))
                order += 1
        loc.sort()
        cand += loc[:K]
    cand.sort()
    return [c[2] for c in cand[:K]]


def test_ivox_closest_matches_bruteforce(scene16):
    mp = scene16["map"][:6000]
    iv = orc.IVox(0.5, 2, 1000000)
    iv.add(mp)
    offs = np.array([(0, 0, 0), (-1, 0, 0), (1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, -1), (0, 0, 1), (1, 1, 0), (-1, 1, 0), (1, -1, 0),
                     (-1, -1, 0), (1, 0, 1), (-1, 0, 1), (1, 0, -1), (-1, 0, -1), (0, 1, 1), (0, -1, 1), (0, 1, -1), (0, -1, -1)])
    rng = np.random.default_rng(9)
    q = mp[rng.choice(len(mp), 120, replace=False)].copy()
    q[:, :3] += rng.normal(0, 0.15, (len(q), 3)).astype(np.float32)
    out, found = iv.closest(q, 5, 5.0)
    for i in range(len(q)):
        want = _ivox_bruteforce(mp, q[i], 0.5, offs, 5, 5.0)
        assert found[i] == len(want)
        assert np.array_equal(out[i, :found[i], :3], mp[want, :3])


def test_ivox_lru_capacity_eviction():
    """AddPoints evicts the least recently touched voxel once size() >= capacity (ivox_map.cpp:133-136 upstream)."""
    iv = orc.IVox(1.0, 0, 4)
    pts = np.array([[k * 1.0, 0, 0, 0] for k in range(6)], np.float32)  # 6 distinct voxels, capacity 4
    iv.add(pts)
    assert iv.num_voxels == 3  # after every insert that reaches 4 voxels the tail is dropped
    out, found = iv.closest(pts, 5, 5.0)
    assert list(found) == [0, 0, 0, 1, 1, 1]  # the three oldest voxels are gone
