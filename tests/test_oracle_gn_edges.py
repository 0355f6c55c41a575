"""The reference of one Gauss-Newton step (tests/gn_ref.py) against the oracle, on the constructed cases of tests/gn_cases.py and on
whole Matches of all five plug-ins.  These tests prove the reference on the CPU before the GPU tests hold the device to it:

  * the oracle's solve6_fullpiv, solve6_lu and so3_exp against the Eigen QR restatement, the exact inverse / determinant and SO3Exp,
    wherever the reference says the decisions are decided;
  * every constructed case reaches the branch it was built for, from the reference;
  * the oracle's own iter_log() of whole Matches replays through the reference: every dx within its bound, the returned pose equal
    to the pose composed from the logged dx, and the iteration count and converged flag equal to the reference's decisions;
  * the rank-deficient comparison: no non-axis rank-deficient H of the cases has a decided rank (the evidence DESIGN.md cites)."""
import functools

import numpy as np
import pytest

from oracle import pyoracle as orc
from tests import gn_cases, gn_ref

CASES = {c.name: c for c in gn_cases.all_cases()}
KINDS = sorted({c.kind for c in CASES.values()})


@functools.lru_cache(maxsize=None)
def reference(name, solver="device"):
    c = CASES[name]
    return gn_ref.step(c.method, c.state(), c.tot, c.params(), solver)


def _f(x):
    return np.array([float(a) for a in x])


@pytest.mark.parametrize("kind", KINDS)
def test_cases_reach_their_branch(kind):
    for c in (c for c in CASES.values() if c.kind == kind):
        s = reference(c.name)
        for key, want in c.expect.items():
            got = {"applied": lambda: s.exp.applied, "exp_decided": lambda: s.exp.decided}.get(key, lambda: getattr(s, key))()
            assert got == want, (c.name, key, got, want)
        if kind in ("thres", "second", "cap", "gate", "so3", "well_posed", "guard", "ill"):
            assert s.stop_decided, c.name
        if kind in ("well_posed", "guard", "ill", "thres", "second", "so3"):
            assert np.all(np.isfinite(s.dx_bound)), (c.name, s.dx_bound)
        if kind == "axis" and c.method in gn_ref.LOAM:  # the basic solution: zeros in the unobserved coordinates
            zero = [i for i in range(6) if np.all(gn_ref.unpack(c.tot)[0][i] == 0)]
            assert all(s.dx[i] == 0 for i in zero) and all(s.dx[i] != 0 for i in range(6) if i not in zero), (c.name, _f(s.dx))
        if kind == "ill":
            k = gn_ref.cond2(gn_ref.unpack(c.tot)[0])
            assert 1e5 < k < 1e8, (c.name, k)


@pytest.mark.parametrize("kind", [k for k in KINDS if k != "nan"])
def test_oracle_solvers_equal_reference(kind):
    """The oracle's pivoting solvers (what the device falls back to) against the reference, where the reference decides."""
    for c in (c for c in CASES.values() if c.kind == kind):
        H, g, _ = gn_ref.unpack(c.tot)
        diag = bool(np.all(H[~np.eye(6, dtype=bool)] == 0))
        # full pivoting vs Eigen's FullPivHouseholderQR
        x = orc.solve6_fullpiv(H, g)
        q = gn_ref.fullpiv_qr_solve(H, g)
        if q.decided and not q.tied:
            kept = sorted(q.cols[:q.rank])
            assert all(x[i] == 0 for i in range(6) if i not in kept), (c.name, x)
            if diag:
                assert all(x[i] == g[i] / H[i, i] for i in kept), (c.name, x)
            else:
                b = gn_ref._solve_bound(H, q.x, gn_ref.C_PIV, kept)
                assert np.all(np.abs(x - _f(q.x)) <= b), (c.name, x - _f(q.x), b)
        # partial-pivot LU vs the exact inverse and determinant
        xl, det = orc.solve6_lu(H, g)
        dz, dec = gn_ref.det_zero(H)
        if dec:
            assert (det == 0) == dz, (c.name, det)
        if dec and not dz:
            xr = gn_ref.inverse_solve(H, g)
            b = np.zeros(6) if diag else gn_ref._solve_bound(H, xr, gn_ref.C_PIV)
            assert np.all(np.abs(xl - _f(xr)) <= b), (c.name, xl - _f(xr), b)
        if dz and dec:
            assert np.all(xl == 0), c.name  # x untouched
        # SO3Exp of the rotation part
        s = reference(c.name)
        if s.path == "update" and s.exp is not None and s.exp.decided and s.dx_exact is not None:
            rv = (s.dx_exact[3:6] if c.method == gn_ref.ICP else s.dx_exact[0:3])
            Ro = orc.so3_exp(rv)
            if not s.exp.applied:
                assert np.array_equal(Ro, np.eye(3)), c.name
            else:
                assert np.max(np.abs(Ro - np.array(s.exp.R.tolist(), dtype=float))) < 16 * gn_ref.EPS, c.name


def test_rank_deficient_decisions():
    """Non-axis rank deficiency: the exact trailing corner is zero and Eigen's cut `6 eps max` sits inside the band rounding may
    move it by, so no such rank is decided and the full-pivot LU and Householder QR basic solutions cannot be told apart by a
    decided case.  Axis-aligned deficiency is decided (exact zeros stay exact) and there both give the same basic solution."""
    for c in (c for c in CASES.values() if c.kind == "nonaxis"):
        H, g, _ = gn_ref.unpack(c.tot)
        q = gn_ref.fullpiv_qr_solve(H, g)
        exact_rank = int(c.name.split("rank")[1][0])
        assert q.nonzero_pivots >= exact_rank and not q.decided, (c.name, [(k, i, float(m), float(b)) for k, i, m, b in q.decisions])
        cut = [(m, b) for k, i, m, b in q.decisions if k == "stop" and i == exact_rank]
        assert cut and abs(cut[0][0]) < cut[0][1], c.name
    for c in (c for c in CASES.values() if c.kind == "axis" and c.method == gn_ref.IVOX):
        H, g, _ = gn_ref.unpack(c.tot)
        q = gn_ref.fullpiv_qr_solve(H, g)
        assert q.decided and np.max(np.abs(orc.solve6_fullpiv(H, g) - _f(q.x))) <= 1e-12 * np.max(np.abs(_f(q.x))), c.name


def test_nan_systems_on_the_oracle():
    """NaN in H: the full-pivot search skips NaN (`fabs(NaN) > best` is false), so an all-NaN H gives rank 0 and dx = 0 in the
    oracle's full-pivot solve, where Eigen's QR (whose maxCoeff starts from the first entry) would carry NaN into dx; the
    partial-pivot LU starts from the diagonal entry, so its determinant is NaN (not 0: ICP does not skip) and so is x.  NaN norms
    never satisfy a `<` threshold."""
    H = np.full((6, 6), np.nan)
    g = np.full(6, np.nan)
    assert np.array_equal(orc.solve6_fullpiv(H, g), np.zeros(6))
    x, det = orc.solve6_lu(H, g)
    assert np.isnan(det) and np.all(np.isnan(x))
    for c in (c for c in CASES.values() if c.kind == "nan"):
        s = reference(c.name)
        assert not s.stop_decided and s.path == "update", c.name


# ---- whole Matches ----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def match_scenes(world, traj, scene16):
    scenes = gn_cases.synth_scenes(world, traj, scene16) + gn_cases.edge_scenes() + [gn_cases.floor_scene(gn_cases.IVOX),
                                                                                     gn_cases.floor_scene(gn_cases.KNN)]
    return {s.name: s for s in scenes}


def oracle_match(s):
    cfg = s.config()
    o = orc.Registration(cfg)
    if s.method == gn_cases.FULL:
        o.add_cloud(*s.maps)
        ok, T, st = o.match(s.scan, s.T, corner=s.corner)
    else:
        for m in s.maps:
            o.add_cloud(m)
        ok, T, st = o.match(s.scan, s.T)
    return ok, T, st, o.iter_log(max(1, cfg.max_iterations)), cfg


def assert_reaches(s, rep, logs):
    if s.reaches == "fallback":  # the device's fast path declines every logged system, decidedly
        dec = [gn_ref.spd_decision(lg["H"])[:2] for lg in logs]
        assert all(not spd and decided for spd, decided in dec), dec
    elif s.reaches in ("second", "cap"):
        assert rep.stop_decided and rep.by == s.reaches, (rep.by, rep.stop_at)
    elif s.reaches == "gate":
        assert rep.steps[-1].path == "gate_fail" and len(rep.steps) > 1, [st.path for st in rep.steps]


SCENE_NAMES = ["synth_icp", "synth_ndt", "synth_ivox", "synth_kd", "synth_full", "synth_ivox_second", "synth_ivox_cap", "synth_ndt_gate",
               "edge_ivox_s1", "edge_ndt_axes", "edge_icp_gate", "edge_kd_shells", "edge_full_corners", "floor_2", "floor_3"]


@pytest.mark.parametrize("name", SCENE_NAMES)
def test_oracle_match_replays(match_scenes, name):
    s = match_scenes[name]
    ok, T, st, logs, cfg = oracle_match(s)
    assert len(logs) == st.iterations
    rep = gn_ref.replay(s.method, s.T, logs, gn_ref.params_of(cfg), solver="oracle")
    gn_ref.assert_replay(rep, logs, T, st.iterations, ok, name)
    assert_reaches(s, rep, logs)


def test_step_probe_rejects_bad_arguments():
    """fls_gn_step_probe's argument checks run before any device work."""
    import ctypes as C

    from funny_lidar_slam_b200 import _abi
    from funny_lidar_slam_b200._lib import lib
    L = lib()
    one = (_abi.FlsGnStepCase * 1)()
    out = (_abi.FlsGnStepOut * 1)()
    assert L.fls_gn_step_probe(None, one, 1, out) == _abi.FLS_ERR_INVALID_ARG
    assert C.sizeof(_abi.FlsGnStepCase) == 16 + 8 * (2 + 9 + 3 + 2 + 31)
    assert C.sizeof(_abi.FlsGnStepOut) == 8 * (9 + 3 + 6 + 36 + 6 + 2 + 13 + 18 + 1 + 1) + 4 * 6
