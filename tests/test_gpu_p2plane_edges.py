"""LOAM-iVox kernels on the adversarial scenes of tests/ivox_scenes.py, against the brute-force references of tests/ivox_ref.py
(proved against the oracle by tests/test_oracle_ivox_edges.py), for every stencil and for the fast and the range-gated
selection:
  * v8's k-NN (fls_ivox_knn) against knn5;
  * iteration 0 of a single Match (v8) and of every scan of batches of 2, 9 and 64 scans (v9) against planar_pass;
  * every iteration of every scan of a batch against the oracle;
  * the QR rank decision on rounding-level neighbourhoods (S7') against the oracle's arithmetic;
  * the batch size limit of the C ABI."""
import ctypes as C
import functools

import numpy as np
import pytest

from funny_lidar_slam_b200 import FLS_P2PLANE_IVOX, default_config, synth
from funny_lidar_slam_b200._abi import FLS_ERR_INVALID_ARG, FLS_FLAG_ITER_LOG, FlsMatchStats
from tests import ivox_ref, ivox_scenes

pytestmark = pytest.mark.gpu

SCENES = {s.name: s for s in ivox_scenes.all_scenes()}
CASES = [(name, cfg, nearby) for name, s in SCENES.items() for cfg in s.configs for nearby in range(4)]
IDS = [f"{n}-res{c[0]}-r{c[1]}-nb{k}" for n, c, k in CASES]


def _cfg(res, max_range, nearby, **kw):
    return default_config(FLS_P2PLANE_IVOX, flags=FLS_FLAG_ITER_LOG, localization_mode=1, ivox_resolution=res, ivox_max_range=max_range,
                          ivox_nearby=nearby, **kw)


def _gpu(name, cfg, nearby, **kw):
    from funny_lidar_slam_b200.registration import Registration
    g = Registration(_cfg(cfg[0], cfg[1], nearby, **kw))
    g.AddCloudToLocalMap([SCENES[name].map])
    return g


@functools.lru_cache(maxsize=None)
def _ref(name, cfg, nearby, first=None):
    s = SCENES[name]
    scan = s.scan if first is None else s.scan[:first]
    ref = ivox_ref.planar_pass(s.map, scan, np.eye(4), 0.1, cfg[0], nearby, cfg[1])
    ivox_ref.assert_gates_clear(ref)
    ivox_ref.assert_sensitive(ref)
    return ref


def _check_pass(log0, ref, what):
    assert log0["n_valid"] == ref.n_valid, (what, log0["n_valid"], ref.n_valid)
    ivox_ref.assert_matches(log0["H"], log0["g"], ref)


@pytest.mark.parametrize("name,cfg,nearby", CASES, ids=IDS)
def test_v8_knn_equals_brute_force(name, cfg, nearby):
    """Found count identical; slot 0 identical in all four components; the 5-set identical (duplicates told apart by their
    intensity).  The order of slots 1-4 is not part of the contract: the quantised selection orders ranks 1/2 and 5/6 only."""
    s = SCENES[name]
    g = _gpu(name, cfg, nearby)
    pts, cnt = g.ivox_knn(s.scan)
    ref = ivox_ref.knn5(s.map, s.scan[:, :3], cfg[0], nearby, cfg[1])
    assert np.array_equal(cnt, ref.found)
    for i in np.nonzero(ref.found)[0]:
        assert np.array_equal(pts[i, 0], s.map[ref.idx[i, 0]]), i
        assert sorted(pts[i, :cnt[i], 3].astype(np.int64)) == sorted(ref.idx[i, :ref.found[i]]), i


@pytest.mark.parametrize("name,cfg,nearby", CASES, ids=IDS)
def test_v8_single_match_first_pass(name, cfg, nearby):
    from funny_lidar_slam_b200.registration import PointcloudCluster
    g = _gpu(name, cfg, nearby, max_iterations=1)
    g.Match(PointcloudCluster(planar_cloud=SCENES[name].scan), np.eye(4))
    _check_pass(g.iter_log()[0], _ref(name, cfg, nearby), "v8")


def _batch(name, B):
    """B copies of the scene's scan; at B = 64 an empty scan and 1-point scans are mixed in."""
    s = SCENES[name]
    scans, kinds = [], []
    for k in range(B):
        if B == 64 and k % 16 == 5:
            scans.append(s.scan[:0])
            kinds.append("empty")
        elif B == 64 and k % 16 == 9:
            scans.append(s.scan[:1])
            kinds.append("one")
        else:
            scans.append(s.scan)
            kinds.append("full")
    return scans, kinds


@pytest.mark.parametrize("B", [2, 9, 64])
@pytest.mark.parametrize("name,cfg,nearby", CASES, ids=IDS)
def test_v9_batch_first_pass(name, cfg, nearby, B):
    """Iteration 0 of every scan of a batch (v9) against the reference; the same scan at different positions of the batch
    gives the same sums to 1e-12 (only the order of the fp64 sums may differ)."""
    g = _gpu(name, cfg, nearby, max_iterations=1)
    scans, kinds = _batch(name, B)
    g.match_batch(scans, np.stack([np.eye(4)] * B))
    ref, ref1 = _ref(name, cfg, nearby), _ref(name, cfg, nearby, 1)
    first = None
    for k, kind in enumerate(kinds):
        lg = g.iter_log(k)
        assert len(lg) == 1, k
        if kind == "empty":
            assert lg[0]["n_valid"] == 0, k
            continue
        _check_pass(lg[0], ref if kind == "full" else ref1, ("v9", B, k))
        if kind == "full":
            if first is None:
                first = lg[0]
            sc = max(np.abs(first["H"]).max(), 1e-300)
            assert np.allclose(lg[0]["H"], first["H"], rtol=1e-12, atol=1e-12 * sc), k
            assert np.allclose(lg[0]["g"], first["g"], rtol=1e-12, atol=1e-12 * sc), k
    with pytest.raises(Exception):
        g.iter_log(B)  # beyond the last call's batch


def test_batch_every_iteration_against_oracle(scene16):
    """A batch of scans at different guesses with the full iteration budget: iteration 0 of every scan exactly as the oracle's
    (n_valid equal, H and g to 1e-9), every later iteration's H and g within 1e-8 wherever n_valid agrees."""
    from funny_lidar_slam_b200.registration import Registration
    from oracle import pyoracle as orc
    cfg = default_config(FLS_P2PLANE_IVOX, flags=FLS_FLAG_ITER_LOG)
    g, o = Registration(cfg), orc.Registration(cfg)
    g.AddCloudToLocalMap([scene16["map"]])
    o.add_cloud(scene16["map"])
    scans = [scene16["scan"][k::3] for k in range(3)] + [scene16["scan"][::2]]
    guesses = [synth.perturb_pose(scene16["truth"], dpos=0.02 + 0.05 * k, drot_deg=0.2 + 0.5 * k, seed=40 + k) for k in range(4)]
    g.match_batch(scans, np.stack(guesses))
    compared = 0
    for k in range(4):
        o.match(scans[k], guesses[k])
        lg, lo = g.iter_log(k), o.iter_log()
        assert len(lg) == len(lo) == g.last_batch_stats[k].iterations, k
        for it, (a, b) in enumerate(zip(lg, lo)):
            sc = np.abs(b["H"]).max()
            if it == 0:
                assert a["n_valid"] == b["n_valid"], k
                assert np.allclose(a["H"], b["H"], rtol=1e-9, atol=1e-9 * sc) and np.allclose(a["g"], b["g"], rtol=1e-9, atol=1e-9 * sc), k
            elif a["n_valid"] == b["n_valid"]:
                compared += 1
                assert np.allclose(a["H"], b["H"], rtol=1e-8, atol=1e-8 * sc), (k, it)
                assert np.allclose(a["g"], b["g"], rtol=1e-8, atol=1e-8 * sc), (k, it)
    assert compared >= 4


def test_batch_of_65_scans_is_rejected(scene16):
    """kMaxBatch = 64: both batch entries refuse 65 scans."""
    from funny_lidar_slam_b200._lib import lib
    from funny_lidar_slam_b200.registration import Registration
    g = Registration(_cfg(0.5, 5.0, 2))
    g.AddCloudToLocalMap([scene16["map"]])
    sc = np.ascontiguousarray(scene16["scan"][:100])
    B = 65
    ptrs = (C.c_void_p * B)(*([sc.ctypes.data] * B))
    ns = (C.c_size_t * B)(*([len(sc)] * B))
    T = np.ascontiguousarray(np.stack([np.eye(4)] * B))
    conv = (C.c_int * B)()
    st = (FlsMatchStats * B)()
    L = lib()
    assert L.fls_match_batch(g._h, B, ptrs, ns, 16, T.ctypes.data_as(C.c_void_p), conv, st) == FLS_ERR_INVALID_ARG
    dptrs = (C.c_void_p * B)()
    zeros = (C.c_size_t * B)()
    assert L.fls_match_batch_device(g._h, B, dptrs, zeros, T.ctypes.data_as(C.c_void_p), conv, st) == FLS_ERR_INVALID_ARG
    assert L.fls_match_batch(g._h, 64, ptrs, ns, 16, T.ctypes.data_as(C.c_void_p), conv, st) == 0  # the limit itself runs


@pytest.mark.parametrize("nearby", range(4))
def test_rounding_level_rank_equals_oracle(nearby):
    """S7': neighbourhoods whose QR rank is decided by fp64 rounding noise.  The GPU's QR shares the oracle's arithmetic
    (fls_plane.cuh, orc_math.h), so v8 single Matches and v9 batches take the same rank decision on every neighbourhood:
    iteration 0 equals planar_pass under that rule (which the oracle follows bit for bit) and the oracle's own pass."""
    from funny_lidar_slam_b200.registration import PointcloudCluster, Registration
    from oracle import pyoracle as orc
    s = ivox_scenes.s7_rounding_rank()
    cfg = _cfg(0.5, 5.0, nearby, max_iterations=1)
    ref = ivox_ref.planar_pass(s.map, s.scan, np.eye(4), cfg.point_to_planar_thres, 0.5, nearby, 5.0, qr_rule=True)
    ivox_ref.assert_gates_clear(ref)
    ivox_ref.assert_sensitive(ref)
    o = orc.Registration(cfg)
    o.add_cloud(s.map)
    o.match(s.scan, np.eye(4))
    lo = o.iter_log()[0]
    g = Registration(cfg)
    g.AddCloudToLocalMap([s.map])
    g.Match(PointcloudCluster(planar_cloud=s.scan), np.eye(4))
    logs = [("v8", g.iter_log()[0])]
    for B in (2, 9):
        g.match_batch([s.scan] * B, np.stack([np.eye(4)] * B))
        logs += [(("v9", B, k), g.iter_log(k)[0]) for k in range(B)]
    for what, lg in logs:
        _check_pass(lg, ref, what)
        assert lg["n_valid"] == lo["n_valid"], what
        ivox_ref.assert_matches(lo["H"], lo["g"], ref)
