"""fls_relocalize_wide on the device, for LOAM-iVox and NDT in localization mode: on every grid fls_relocalize accepts it returns what
fls_relocalize returns; on a grid past that cap it recovers a pose 25 m and 150 degrees off, with fewer evaluations than hypotheses,
and no leaf it skipped scores below the ones it picked; it is deterministic and leaves the handle as fls_relocalize does.  The scene is
tests/test_gpu_relocalize.py's."""
import numpy as np
import pytest

from funny_lidar_slam_b200 import _abi, synth
from funny_lidar_slam_b200._lib import FlsError
from funny_lidar_slam_b200.registration import PointcloudCluster, Registration
from tests import reloc_wide_ref
from tests.test_gpu_relocalize import FLT_MAX, METHODS, _cluster, _handle, _off, scene  # noqa: F401  (scene: the shared fixture)

pytestmark = pytest.mark.gpu

GRIDS = {  # fls_relocalize's grids: 7 x 7 x 24, and DESIGN.md's 1 m x 10 degrees and 0.5 m x 5 degrees over +-10 m
    "7x7x24": dict(xy_radius=3.0, xy_step=1.0, yaw_range=np.pi, yaw_step=np.deg2rad(15.0)),
    "1m10deg": dict(xy_radius=10.0, xy_step=1.0, yaw_range=np.pi, yaw_step=np.deg2rad(10.0)),
    "0.5m5deg": dict(xy_radius=10.0, xy_step=0.5, yaw_range=np.pi, yaw_step=np.deg2rad(5.0)),
}
WIDE = dict(xy_radius=40.0, xy_step=0.5, yaw_range=np.pi, yaw_step=np.deg2rad(2.0), n_refine=64)  # 161 * 161 * 180 = 4 665 780


def _same(a, b):
    """The results of two calls: the selection bit for bit; the refinement (the batch Match, whose sums may run in another order from
    call to call) to test_gpu_relocalize.py's bar between two calls, with how many of its values are bit-identical printed."""
    assert a.n_hypotheses == b.n_hypotheses and a.n_refined == b.n_refined
    assert list(a.refined_index) == list(b.refined_index)
    assert np.float32(a.coarse_score).tobytes() == np.float32(b.coarse_score).tobytes()
    assert np.array_equal(a.refined_converged, b.refined_converged)
    assert (a.best_rank, a.best_hypothesis, a.converged, a.accepted) == (b.best_rank, b.best_hypothesis, b.converged, b.accepted)
    if a.n_refined:
        assert np.max(np.abs(a.refined_T - b.refined_T)) <= 1e-9 and np.max(np.abs(a.T - b.T)) <= 1e-9
        assert np.all(np.abs(a.refined_fitness - b.refined_fitness) <= 1e-5 * np.abs(a.refined_fitness))
        assert abs(a.fitness - b.fitness) <= 1e-5 * a.fitness
    bits = int(a.refined_T.tobytes() == b.refined_T.tobytes()) + int(a.refined_fitness.tobytes() == b.refined_fitness.tobytes())
    print(f"refinement bit-identical: {bits} of 2 (refined_T, refined_fitness); T {a.T.tobytes() == b.T.tobytes()}")


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("grid", list(GRIDS))
@pytest.mark.parametrize("n_refine", [1, 8, 64])
def test_equals_the_exhaustive_search(scene, method, grid, n_refine):
    g = _handle(scene, method)
    ex = g.relocalize(scene["scan"], scene["guess"], n_refine=n_refine, **GRIDS[grid])
    wi, ev = g.relocalize_wide(scene["scan"], scene["guess"], n_refine=n_refine, **GRIDS[grid])
    print(f"{grid} n_refine={n_refine}: {ex.n_hypotheses} hypotheses, {ev} evaluations, waits {ex.host_waits} / {wi.host_waits}")
    _same(ex, wi)
    assert ev >= ex.n_hypotheses  # grids of at most 2^20 hypotheses start at the leaves and score every one


@pytest.mark.parametrize("method", METHODS)
def test_equals_the_exhaustive_search_at_the_edges(scene, method):
    g = _handle(scene, method)
    far = scene["guess"].copy()
    far[:3, 3] += [1000.0, 0.0, 0.0]  # every score ties at max_range: the picks are the lowest indices
    ex = g.relocalize(scene["scan"], far, n_refine=8, **GRIDS["1m10deg"])
    wi, ev = g.relocalize_wide(scene["scan"], far, n_refine=8, **GRIDS["1m10deg"])
    _same(ex, wi)
    assert list(wi.refined_index) == list(range(8))
    empty = np.zeros((0, 4), np.float32)
    ex = g.relocalize(empty, scene["guess"], n_refine=4)
    wi, ev = g.relocalize_wide(empty, scene["guess"], n_refine=4)
    _same(ex, wi)
    assert ev == 0 and wi.n_refined == 0 and np.array_equal(wi.T, scene["guess"])
    assert g.GetFitnessScore(2.0) == FLT_MAX


@pytest.fixture(scope="module")
def wide_runs(scene):
    """Per plug-in: the handle, the guess 25 m and 150 degrees off, and the wide search from it (run twice)."""
    out = {}
    for method in METHODS:
        g = _handle(scene, method)
        guess = _off(scene["T_true"], 20.0, -15.0, 150.0)
        a = g.relocalize_wide(scene["scan"], guess, **WIDE)
        fit_after = g.GetFitnessScore(2.0)
        levels = g.relocalize_wide_levels()
        b = g.relocalize_wide(scene["scan"], guess, **WIDE)
        out[method] = dict(g=g, guess=guess, a=a, b=b, fit_after=fit_after, levels=levels)
    return out


@pytest.mark.parametrize("method", METHODS)
def test_recovers_a_pose_25_m_and_150_degrees_off(scene, wide_runs, method):
    run = wide_runs[method]
    with pytest.raises(FlsError) as ei:  # past fls_relocalize's 2^20 cap
        run["g"].relocalize(scene["scan"], run["guess"], **WIDE)
    assert ei.value.status == _abi.FLS_ERR_INVALID_ARG
    r, ev = run["a"]
    levels = run["levels"]
    dt, dr = synth.pose_error(r.T, scene["T_true"])
    print(f"method {method}: nodes per level from the start level down: {levels}")
    assert len(levels) == 2 and levels[0] == 81 * 81 * 90 and ev == 2 * levels[0] + levels[1]
    print(f"method {method}: {r.n_hypotheses} hypotheses, {ev} evaluations ({ev / r.n_hypotheses:.3f} of them), rank {r.best_rank}, "
          f"fitness {r.fitness:.4f}, error {dt:.4f} m {np.rad2deg(dr):.3f} deg, {r.host_waits} waits, {r.gpu_launches} launches")
    assert r.n_hypotheses == 161 * 161 * 180
    assert ev < r.n_hypotheses
    assert r.accepted and r.converged
    assert dt < 0.05 and np.rad2deg(dr) < 0.5


@pytest.mark.parametrize("method", METHODS)
def test_no_skipped_leaf_scores_below_the_picks(scene, wide_runs, method):
    """2000 random leaves of the wide grid and every pick, each scored alone by the degenerate fls_relocalize from its own pose.  The
    host's cos / sin may differ from the device's by an ulp, so scores are compared with a relative tolerance of 1e-6."""
    run = wide_runs[method]
    r, _ = run["a"]
    g = _handle(scene, method)
    grid = reloc_wide_ref.grid(WIDE["xy_radius"], WIDE["xy_step"], WIDE["yaw_range"], WIDE["yaw_step"])
    nx, nk = 2 * grid.I + 1, grid.n_yaw

    def score(index):
        k, i, j = index % nk, (index // nk) % nx, index // (nk * nx)
        T = reloc_wide_ref.leaf_pose(run["guess"], grid, WIDE["xy_step"], WIDE["yaw_step"], i, j, k)
        return g.relocalize(scene["scan"], T, xy_radius=0.0, yaw_range=0.0, n_refine=1, coarse_scores=1).coarse_scores[0]

    picks = [int(i) for i in r.refined_index]
    pick_scores = np.array([score(i) for i in picks])
    assert np.isclose(pick_scores[r.best_rank], r.coarse_score, rtol=1e-6, atol=0)  # the reported score is the float of the pick's
    assert np.all(np.diff(pick_scores) >= -1e-6 * pick_scores[1:])  # in rank order
    worst = pick_scores.max()
    rng = np.random.default_rng(method)
    sample = [int(i) for i in rng.integers(0, r.n_hypotheses, 2000) if int(i) not in picks]
    s = np.array([score(i) for i in sample])
    print(f"method {method}: n_refine-th pick scores {worst:.5f}; sampled leaves score {s.min():.5f} .. {s.max():.5f}")
    assert np.all(s >= worst * (1 - 1e-6)), (s.min(), worst)


def _tiles(n, side):
    """(centre, radius) of odd-sided tiles of at most `side` indices that cover 0 .. n-1 exactly"""
    out, lo = [], 0
    while lo < n:
        w = min(side, n - lo)
        w -= 1 - w % 2  # odd, so that the tile is a grid centred on one index
        w = max(w, 1)
        out.append((lo + w // 2, w // 2))
        lo += w
    return out


@pytest.mark.parametrize("method", METHODS)
def test_picks_are_the_exhaustive_best_of_the_wide_grid(scene, wide_runs, method):
    """Every hypothesis of the 4.67 M wide grid scored by fls_relocalize, tile by tile (each tile a grid around a shifted
    guess, with the wide grid's rotations and steps): the wide search's picks are the n_refine best of all of them.  A tile's
    translations are t_guess + c step + i step in two fp64 roundings instead of one, so a score may differ in the last bits: ranks
    are compared where the score gaps exceed 1e-6 relative, and no unpicked hypothesis may score below a pick by more than that."""
    run = wide_runs[method]
    r, _ = run["a"]
    g = _handle(scene, method)
    grid = reloc_wide_ref.grid(WIDE["xy_radius"], WIDE["xy_step"], WIDE["yaw_range"], WIDE["yaw_step"])
    nx, nk, step = 2 * grid.I + 1, grid.n_yaw, WIDE["xy_step"]
    score = np.full(grid.P, np.nan)
    tiles = _tiles(nx, 23)  # 161 = 7 * 23: square tiles (fls_relocalize's grid is square) of 23 * 23 * 180 hypotheses
    assert {r_ for _, r_ in tiles} == {11}
    for cj, rj in tiles:
        for ci, ri in tiles:
            T = run["guess"].copy()
            T[0, 3] += (ci - grid.I) * step
            T[1, 3] += (cj - grid.I) * step
            w = 2 * ri + 1
            t = g.relocalize(scene["scan"], T, xy_radius=ri * step, xy_step=step, yaw_range=WIDE["yaw_range"], yaw_step=WIDE["yaw_step"],
                             n_refine=1, coarse_scores=w * w * nk)
            assert t.n_hypotheses == w * w * nk
            sub = t.coarse_scores.reshape(w, w, nk)
            for jj in range(w):
                j = cj - rj + jj
                base = (j * nx + (ci - ri)) * nk
                score[base:base + w * nk] = sub[jj].ravel()
    assert not np.isnan(score).any()
    n = r.n_refined
    order = np.lexsort((np.arange(grid.P), score))
    ref, gaps = order[:n], np.diff(score[order[:n + 1]])
    picks = np.array(r.refined_index)
    worst = score[picks].max()
    print(f"method {method}: exhaustive best {score[order[0]]:.6f}, n-th {score[order[n - 1]]:.6f}; wide picks' worst {worst:.6f}")
    assert worst <= score[order[n - 1]] * (1 + 1e-6)
    below = np.flatnonzero(score < worst * (1 - 1e-6))
    assert np.isin(below, picks).all(), np.setdiff1d(below, picks)[:10]
    for k in range(n):
        tol = 1e-6 * score[ref[k]]
        if gaps[k] > tol and (k == 0 or gaps[k - 1] > tol):
            assert picks[k] == ref[k], k


@pytest.mark.parametrize("method", METHODS)
def test_launches_and_waits_equal_the_exhaustive_search(scene, method):
    """fls_relocalize's counts on this scene (the same as before the wide entry was added); the wide entry on a grid of at most 2^20
    hypotheses runs the same search, so it makes the same launches and waits.  fls_relocalize leaves the wide entry's level record."""
    g = _handle(scene, method)
    got = []
    for kw in (dict(xy_radius=0.0, yaw_range=0.0, n_refine=1), GRID_175, GRID_175):
        r = g.relocalize(scene["scan"], scene["guess"], **kw)
        got.append((r.gpu_launches, r.host_waits))
    assert got == EXHAUSTIVE_COUNTS[method], got
    ex = g.relocalize(scene["scan"], scene["guess"], **GRID_175)
    wi, _ = g.relocalize_wide(scene["scan"], scene["guess"], **GRID_175)
    assert (wi.gpu_launches, wi.host_waits) == (ex.gpu_launches, ex.host_waits)
    assert g.relocalize_wide_levels() == [175]
    g.relocalize(scene["scan"], scene["guess"], **GRID_175)
    assert g.relocalize_wide_levels() == [175]


GRID_175 = dict(xy_radius=2.0, xy_step=1.0, yaw_range=np.deg2rad(30.0), yaw_step=np.deg2rad(10.0), n_refine=8)
# (gpu_launches, host_waits) of fls_relocalize on this scene: the degenerate search on a fresh handle (the fit grid is built: one more
# wait), then the 175-hypothesis search twice.  The library made and reported the same counts before fls_relocalize_wide existed.
EXHAUSTIVE_COUNTS = {_abi.FLS_P2PLANE_IVOX: [(25, 6), (17, 5), (17, 5)], _abi.FLS_NDT: [(33, 8), (32, 7), (32, 7)]}


@pytest.mark.parametrize("method", METHODS)
def test_deterministic_and_the_handle_afterwards(scene, wide_runs, method):
    run = wide_runs[method]
    (a, ea), (b, eb) = run["a"], run["b"]
    _same(a, b)
    assert ea == eb
    assert run["fit_after"] == a.fitness  # fls_fitness after the call scores the chosen pose
    # a following Match behaves as after a plain Match: the same Match on a handle that only ran a plain Match
    start = synth.perturb_pose(scene["T_true"], seed=9, dpos=0.3, drot_deg=2.0)
    g, ref = run["g"], _handle(scene, method)
    T0 = scene["guess"].copy()
    ref.Match(_cluster(method, scene["scan"]), T0)
    Ta, Tb = start.copy(), start.copy()
    oka, okb = g.Match(_cluster(method, scene["scan"]), Ta), ref.Match(_cluster(method, scene["scan"]), Tb)
    assert oka == okb and np.array_equal(Ta, Tb)
    assert g.GetFitnessScore(2.0) == ref.GetFitnessScore(2.0)


def test_unsupported_plugins_and_modes_leave_the_handle_untouched(scene):
    for method in (_abi.FLS_ICP_P2P, _abi.FLS_P2PLANE_KNN):
        g = _handle(scene, method)
        cl = PointcloudCluster(ordered_cloud=scene["scan"]) if method == _abi.FLS_ICP_P2P else PointcloudCluster(planar_cloud=scene["scan"])
        g0 = synth.perturb_pose(scene["T_true"], seed=5, dpos=0.2, drot_deg=1.0)
        Ta = g0.copy()
        g.Match(cl, Ta)
        with pytest.raises(FlsError) as ei:
            g.relocalize_wide(scene["scan"], g0)
        assert ei.value.status == _abi.FLS_ERR_UNSUPPORTED
        Tb = g0.copy()
        g.Match(cl, Tb)
        assert np.array_equal(Ta, Tb)
    for method in METHODS:  # mapping mode: a Match after the refused call is the Match of a handle that never saw it
        a, b = (_handle(scene, method, localization_mode=0) for _ in range(2))
        with pytest.raises(FlsError) as ei:
            a.relocalize_wide(scene["scan"], scene["guess"])
        assert ei.value.status == _abi.FLS_ERR_UNSUPPORTED
        g0 = synth.perturb_pose(scene["T_true"], seed=6, dpos=0.2, drot_deg=1.0)
        Ta, Tb = g0.copy(), g0.copy()
        oka, okb = a.Match(_cluster(method, scene["scan"]), Ta), b.Match(_cluster(method, scene["scan"]), Tb)
        assert oka == okb and np.array_equal(Ta, Tb)
        assert a.map_info().n_voxels == b.map_info().n_voxels
    g = Registration(_abi.default_config(_abi.FLS_NDT))
    with pytest.raises(FlsError) as ei:
        g.relocalize_wide(scene["scan"], scene["guess"])
    assert ei.value.status == _abi.FLS_ERR_NO_MAP
    g = _handle(scene, _abi.FLS_P2PLANE_IVOX)
    for bad in (dict(n_refine=0), dict(n_refine=65), dict(xy_step=0.0), dict(coarse_leaf=float("nan")), dict(max_range=-1.0),
                dict(xy_radius=0.0, yaw_range=np.pi, yaw_step=np.pi / (2 ** 30 + 1)),  # 2^31 + 2 hypotheses
                dict(xy_radius=23170.0, xy_step=1.0, yaw_range=0.0)):  # 46341^2 > 2^31
        with pytest.raises(FlsError) as ei:
            g.relocalize_wide(scene["scan"], scene["guess"], **bad)
        assert ei.value.status == _abi.FLS_ERR_INVALID_ARG, bad
