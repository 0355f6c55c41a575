"""fls_relocalize_multi on the device, for LOAM-iVox and NDT in localization mode: with one guess it is fls_relocalize_wide; with
several, its selection is the exact n best of the union of the guesses' grids (each hypothesis scored as fls_relocalize scores it on
its own guess), on grids scored whole and on grids past 2^20 hypotheses where the descent runs; it recovers the pose when the first
guess is a wrong place; it is deterministic, its launches and waits do not grow with the number of guesses, and its refusals leave
the handle untouched.  The scenes are tests/test_gpu_relocalize.py's and tests/test_gpu_scan_context.py's."""
import ctypes as C

import numpy as np
import pytest

from funny_lidar_slam_b200 import _abi, _lib, synth
from funny_lidar_slam_b200._lib import FlsError
from funny_lidar_slam_b200.keyframes import place_pose
from funny_lidar_slam_b200.registration import PointcloudCluster, Registration, reloc_cfg
from tests import reloc_ref
from tests.test_gpu_relocalize import METHODS, RECOVERY, _cluster, _handle, _off, scene  # noqa: F401  (scene: the shared fixture)
from tests.test_gpu_relocalize_wide import EXHAUSTIVE_COUNTS, GRID_175, GRIDS, WIDE, _same

pytestmark = pytest.mark.gpu

SMALL = dict(xy_radius=2.0, xy_step=1.0, yaw_range=np.deg2rad(30.0), yaw_step=np.deg2rad(10.0), n_refine=16)  # 175 per guess


def _union(per_guess, n):
    """The n first of every guess's coarse scores merged on (score bits, g * P + p): the multi search's selection by definition."""
    s = np.concatenate(per_guess)
    return list(np.lexsort((np.arange(len(s)), s.view(np.uint64)))[:n]), s


def _guess_sets(scene):
    g0 = scene["guess"]
    far = _off(g0, 30.0, -12.0, 70.0)
    spread = [g0, far]
    overlap = [_off(g0, dx, dy, a) for dx, dy, a in ((0, 0, 0), (1.0, 0, 0), (0.5, 0.5, 10.0), (-1.0, 1.0, -10.0), (2.0, -2.0, 20.0))]
    dup = [g0, far, g0, _off(g0, 1.0, 0, 0), g0, _off(far, 0, 0, 10.0), far, _off(g0, -3.0, 2.0, -30.0)]
    return {"spread2": spread, "overlap5": overlap, "duplicates8": dup}


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("grid", ["1m10deg", "wide"])
def test_one_guess_is_the_wide_entry(scene, method, grid):
    g = _handle(scene, method)
    kw, guess = (dict(n_refine=16, **GRIDS[grid]), scene["guess"]) if grid != "wide" else (WIDE, _off(scene["T_true"], 20.0, -15.0, 150.0))
    g.relocalize_wide(scene["scan"], guess, **kw)  # builds the fit grid and the lattice, which count waits and launches once
    mu, em = g.relocalize_multi(scene["scan"], [guess], **kw)
    lm = g.relocalize_wide_levels()
    wi, ew = g.relocalize_wide(scene["scan"], guess, **kw)
    lw = g.relocalize_wide_levels()
    print(f"{grid}: {wi.n_hypotheses} hypotheses, evaluations {ew} / {em}, levels {lw} / {lm}, "
          f"(launches, waits) {(wi.gpu_launches, wi.host_waits)} / {(mu.gpu_launches, mu.host_waits)}")
    _same(wi, mu)
    assert (ew, lw) == (em, lm)
    assert (wi.gpu_launches, wi.host_waits) == (mu.gpu_launches, mu.host_waits)
    assert len(lw) == (1 if grid != "wide" else 2)


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("which", ["spread2", "overlap5", "duplicates8"])
def test_exact_union_on_small_grids(scene, method, which):
    g = _handle(scene, method)
    guesses = _guess_sets(scene)[which]
    per, H = [], []
    for T in guesses:
        r = g.relocalize(scene["scan"], T, coarse_scores=175, **SMALL)
        assert r.n_hypotheses == 175
        per.append(r.coarse_scores)
        H.append(reloc_ref.hypotheses(T, SMALL["xy_radius"], SMALL["xy_step"], SMALL["yaw_range"], SMALL["yaw_step"]))
    H = np.concatenate(H)
    mu, ev = g.relocalize_multi(scene["scan"], guesses, **SMALL)
    iters = [len(g.iter_log(k)) for k in range(mu.n_refined)]
    ref, scores = _union(per, SMALL["n_refine"])
    print(f"{which}: {mu.n_hypotheses} hypotheses, {ev} evaluations, picks from guesses {sorted(set(int(i) // 175 for i in mu.refined_index))}")
    assert mu.n_hypotheses == 175 * len(guesses) and ev == mu.n_hypotheses
    assert list(mu.refined_index) == ref
    assert np.float32(scores[mu.best_hypothesis]).tobytes() == np.float32(mu.coarse_score).tobytes()
    # each refined pose is a Match from its start pose, and its fitness the GetFitnessScore after it
    for k in range(mu.n_refined):
        T = H[mu.refined_index[k]].copy()
        ok = g.Match(_cluster(method, scene["scan"]), T)
        assert np.max(np.abs(T - mu.refined_T[k])) <= 1e-9, k
        assert ok == mu.refined_converged[k] and g.last_stats.iterations == iters[k], k
        assert g.GetFitnessScore(2.0) == mu.refined_fitness[k], k
    conv = np.flatnonzero(mu.refined_converged)
    pool = conv if len(conv) else np.arange(mu.n_refined)
    best = pool[np.lexsort((pool, mu.refined_fitness[pool]))[0]]
    assert mu.best_rank == best and mu.fitness == mu.refined_fitness[best] and np.array_equal(mu.T, mu.refined_T[best])
    assert mu.best_hypothesis == mu.refined_index[best]


PAST = dict(xy_radius=10.0, xy_step=0.5, yaw_range=np.pi, yaw_step=np.deg2rad(5.0), n_refine=64)  # 41 * 41 * 72 = 121 032 per guess


@pytest.mark.parametrize("method", METHODS)
def test_exact_union_past_2_20(scene, method):
    """Nine guesses of 121 032 hypotheses (1.09 M in all): the descent runs.  Every hypothesis is scored by fls_relocalize on its own
    guess; the picks are the n best of all of them wherever the score gaps exceed 1e-6 relative."""
    g = _handle(scene, method)
    T0 = _off(scene["T_true"], 14.0, -9.0, 120.0)
    guesses = [_off(T0, dx, dy, 0.0) for dx in (-15.0, 0.0, 15.0) for dy in (-15.0, 0.0, 15.0)]
    per, wide_evals = [], 0
    for T in guesses:
        per.append(g.relocalize(scene["scan"], T, coarse_scores=1 << 20, **PAST).coarse_scores)
        wide_evals += g.relocalize_wide(scene["scan"], T, **PAST)[1]
    mu, ev = g.relocalize_multi(scene["scan"], guesses, **PAST)
    levels = g.relocalize_wide_levels()
    P = 41 * 41 * 72
    assert mu.n_hypotheses == 9 * P
    score = np.concatenate(per)
    n = mu.n_refined
    order = np.lexsort((np.arange(len(score)), score))
    ref, gaps = order[:n], np.diff(score[order[:n + 1]])
    picks = np.array(mu.refined_index)
    print(f"method {method}: {mu.n_hypotheses} hypotheses, multi {ev} evaluations (levels {levels}), nine wide calls {wide_evals}; "
          f"picks from guesses {sorted(set(int(i) // P for i in picks))}")
    assert len(levels) == 2
    worst = score[picks].max()
    assert worst <= score[order[n - 1]] * (1 + 1e-6)
    below = np.flatnonzero(score < worst * (1 - 1e-6))
    assert np.isin(below, picks).all(), np.setdiff1d(below, picks)[:10]
    for k in range(n):
        tol = 1e-6 * score[ref[k]]
        if gaps[k] > tol and (k == 0 or gaps[k - 1] > tol):
            assert picks[k] == ref[k], k


@pytest.mark.parametrize("method,offset,step,yaw_step", RECOVERY)
def test_recovery_when_the_first_guess_is_a_wrong_place(scene, method, offset, step, yaw_step):
    """tests/test_gpu_relocalize.py's recovery, with two wrong places ahead of the guess it recovers from"""
    g = _handle(scene, method)
    cfg = dict(xy_radius=8.0, xy_step=step, yaw_range=np.pi, yaw_step=np.deg2rad(yaw_step), n_refine=64)
    wrong = [_off(scene["T_true"], -24.0, 19.0, 40.0), _off(scene["T_true"], 25.0, 22.0, -90.0)]
    right = _off(scene["T_true"], *offset)
    top1 = g.relocalize(scene["scan"], wrong[0], **cfg)
    dt1, _ = synth.pose_error(top1.T, scene["T_true"])
    mu, ev = g.relocalize_multi(scene["scan"], wrong + [right], **cfg)
    dt, dr = synth.pose_error(mu.T, scene["T_true"])
    P = mu.n_hypotheses // 3
    print(f"method {method}: from guess 0 alone: accepted={top1.accepted} error {dt1:.2f} m | multi: guess {mu.best_hypothesis // P}, "
          f"error {dt:.4f} m {np.rad2deg(dr):.3f} deg, fitness {mu.fitness:.4f}, {ev} evaluations")
    assert dt1 > 1.0 or not top1.accepted
    assert mu.accepted and mu.converged and mu.best_hypothesis // P == 2
    assert dt < 0.05 and np.rad2deg(dr) < 0.5
    assert g.GetFitnessScore(2.0) == mu.fitness


def test_relocalization_from_the_top_5_of_place_query():
    """tests/test_gpu_scan_context.py's relocalization from place_query, with the five best candidates as the guesses."""
    from tests.test_gpu_scan_context import _rz, _store
    world = synth.make_world(seed=1234)
    traj = synth.trajectory(40)
    T_true = traj[10]
    mp = synth.make_surface_map(world, spacing=0.5, seed=11)
    mp = np.ascontiguousarray(mp[np.all(np.abs(mp[:, :2] - T_true[:2, 3].astype(np.float32)) <= 40.0, axis=1)])
    first_pass = [i for i in range(25) if i != 10]
    s = _store([synth.make_scan(world, traj[i], "vlp16", seed=700 + i)["points"] for i in first_pass])
    T_scan = T_true @ _rz(np.deg2rad(63.0))
    scan = synth.make_scan(world, T_scan, "vlp16", seed=21)["points"]
    cands = s.place_query(scan, 5)
    guesses = [place_pose(traj[first_pass[c.id]], c.yaw) for c in cands]
    g = Registration(_abi.default_config(_abi.FLS_P2PLANE_IVOX))
    g.AddCloudToLocalMap([mp])
    r, ev = g.relocalize_multi(scan, guesses, xy_radius=3.0, xy_step=1.0, yaw_range=np.deg2rad(20.0), yaw_step=np.deg2rad(10.0), n_refine=16)
    dt, dr = synth.pose_error(r.T, T_scan)
    print(f"place_query top 5: keyframes {[first_pass[c.id] for c in cands]}, chosen guess {r.best_hypothesis // (r.n_hypotheses // 5)}, "
          f"error {dt:.4f} m {np.rad2deg(dr):.3f} deg, fitness {r.fitness:.3f}, {ev} evaluations")
    assert len(guesses) == 5
    assert r.accepted
    assert dt < 0.05 and np.rad2deg(dr) < 0.5


@pytest.mark.parametrize("method", METHODS)
def test_deterministic_and_device_entry_equals_host(scene, method):
    import torch
    g = _handle(scene, method)
    guesses = _guess_sets(scene)["overlap5"]
    a, ea = g.relocalize_multi(scene["scan"], guesses, **SMALL)
    b, eb = g.relocalize_multi(scene["scan"], guesses, **SMALL)
    d = torch.from_numpy(scene["scan"]).cuda()
    torch.cuda.synchronize()
    c, ec = g.relocalize_multi_device(d.data_ptr(), d.shape[0], guesses, **SMALL)
    for o, eo in ((b, eb), (c, ec)):
        _same(a, o)
        assert eo == ea


@pytest.mark.parametrize("method", METHODS)
def test_launches_and_waits_do_not_grow_with_the_guesses(scene, method):
    """On 175 hypotheses per guess (11 200 at G = 64) the search scores every hypothesis in one chunk: the counts are those of
    fls_relocalize on GRID_175 (tests/test_gpu_relocalize_wide.py) at every G."""
    g = _handle(scene, method)
    g.relocalize(scene["scan"], scene["guess"], **GRID_175)  # builds the fit grid
    got = {}
    for G in (1, 8, 64):
        guesses = [_off(scene["guess"], 0.25 * (k % 8), 0.25 * (k // 8), 0.0) for k in range(G)]
        r, ev = g.relocalize_multi(scene["scan"], guesses, **GRID_175)
        assert r.n_hypotheses == 175 * G and ev == 175 * G
        got[G] = (r.gpu_launches, r.host_waits)
    print(f"method {method}: (launches, waits) by G: {got}")
    assert got == {G: EXHAUSTIVE_COUNTS[method][2] for G in (1, 8, 64)}


def _raw_multi(g, scan, cfg, guesses, n_guesses):
    """fls_relocalize_multi through ctypes, so that a NULL table or a count that disagrees with it can be passed"""
    a = np.ascontiguousarray(scan, np.float32)
    T = (C.c_double * 16)(*np.full(16, 7.0))
    r = _abi.FlsRelocResult()
    ev = C.c_int64(0)
    gp = guesses.ctypes.data_as(C.c_void_p) if guesses is not None else None
    rc = _lib.lib().fls_relocalize_multi(g._h, a.ctypes.data_as(C.c_void_p), len(a), a.shape[1] * 4, C.byref(cfg), gp, n_guesses, T, C.byref(r),
                                         None, None, None, None, C.byref(ev))
    return rc, np.array(T[:])


def _match_after(scene, method, g, **kw):
    """the Match after a refused call equals the Match of a fresh handle"""
    ref = _handle(scene, method, **kw)
    g0 = synth.perturb_pose(scene["T_true"], seed=6, dpos=0.2, drot_deg=1.0)
    Ta, Tb = g0.copy(), g0.copy()
    cl = _cluster(method, scene["scan"]) if method in METHODS else (
        PointcloudCluster(ordered_cloud=scene["scan"]) if method == _abi.FLS_ICP_P2P else PointcloudCluster(planar_cloud=scene["scan"]))
    oka, okb = g.Match(cl, Ta), ref.Match(cl, Tb)
    assert oka == okb and np.array_equal(Ta, Tb)
    assert g.GetFitnessScore(2.0) == ref.GetFitnessScore(2.0)


def test_refusals_leave_the_handle_untouched(scene):
    method = _abi.FLS_P2PLANE_IVOX
    G = np.stack([np.asarray(scene["guess"], np.float64).T] * 3).copy()  # column-major
    bad_nan, bad_inf = G.copy(), G.copy()
    bad_nan[1, 0, 3] = np.nan
    bad_inf[2, 3, 1] = np.inf
    g = _handle(scene, method)
    for guesses, count in ((None, 3), (G, 0), (G, 65), (G, -1), (bad_nan, 3), (bad_inf, 3)):
        rc, T = _raw_multi(g, scene["scan"], reloc_cfg(xy_radius=2.0), guesses, count)
        assert rc == _abi.FLS_ERR_INVALID_ARG, count
        assert np.all(T == 7.0)
    # G * P past 2^31: two guesses of 2^31 hypotheses each
    rc, T = _raw_multi(g, scene["scan"], reloc_cfg(xy_radius=0.0, yaw_range=np.pi, yaw_step=np.pi / 2 ** 30), G, 2)
    assert rc == _abi.FLS_ERR_INVALID_ARG and np.all(T == 7.0)
    _match_after(scene, method, g)
    # FLS_ERR_CAPACITY: eight guesses off the map tie everywhere at max_range, so every block survives; level 0 would hold 9.4 M
    g = _handle(scene, method)
    off = [_off(scene["guess"], 1000.0 + 100.0 * k, 0.0, 0.0) for k in range(8)]
    with pytest.raises(FlsError) as ei:
        g.relocalize_multi(scene["scan"], off, xy_radius=20.0, xy_step=0.5, yaw_range=np.pi, yaw_step=np.deg2rad(2.0), n_refine=8)
    assert ei.value.status == _abi.FLS_ERR_CAPACITY
    print(f"capacity: levels reached {g.relocalize_wide_levels()}")
    _match_after(scene, method, g)
    # plug-ins without relocalization, and mapping mode
    for m in (_abi.FLS_ICP_P2P, _abi.FLS_P2PLANE_KNN, _abi.FLS_LOAM_FULL):
        g = _handle(scene, m) if m != _abi.FLS_LOAM_FULL else Registration(_abi.default_config(m))  # refused before the map check
        with pytest.raises(FlsError) as ei:
            g.relocalize_multi(scene["scan"], [scene["guess"]])
        assert ei.value.status == _abi.FLS_ERR_UNSUPPORTED
        if m != _abi.FLS_LOAM_FULL:
            _match_after(scene, m, g)
    for m in METHODS:
        g = _handle(scene, m, localization_mode=0)
        with pytest.raises(FlsError) as ei:
            g.relocalize_multi(scene["scan"], [scene["guess"]] * 2)
        assert ei.value.status == _abi.FLS_ERR_UNSUPPORTED
        _match_after(scene, m, g, localization_mode=0)
    # no map
    g = Registration(_abi.default_config(_abi.FLS_NDT))
    with pytest.raises(FlsError) as ei:
        g.relocalize_multi(scene["scan"], [scene["guess"]] * 2)
    assert ei.value.status == _abi.FLS_ERR_NO_MAP
    # a batch in flight
    g = _handle(scene, method)
    g.match_batch_begin([scene["scan"]] * 2, [scene["guess"]] * 2)
    with pytest.raises(FlsError) as ei:
        g.relocalize_multi(scene["scan"], [scene["guess"]] * 2)
    assert ei.value.status == _abi.FLS_ERR_INVALID_ARG
    conv, T = g.match_batch_end()
    ref = _handle(scene, method)
    conv2, T2 = ref.match_batch([scene["scan"]] * 2, [scene["guess"]] * 2)
    assert np.array_equal(conv, conv2) and np.array_equal(T, T2)
    _match_after(scene, method, g)
