"""Constructed inputs of one Gauss-Newton step (tests/gn_ref.py) for fls_gn_step_probe: each case is a pre-step state, the step's
parameters and the reduced totals of one iteration, built to sit on one branch of the solve, the update or the stop rule.  `expect`
names what the reference must say for the branch the case is built for (tests/test_oracle_gn_edges.py checks it); the GPU tests then
hold the device to the reference on every case.

  well_posed   random SPD H = J^T J (40x6) at H scales 1e-6 .. 1e12, random pose and last norms, every method
  guard        the LDL^T fast path's `pivot > 1e-8 dmax` with the smallest pivot at fl(1e-8 dmax) and 1, 2 ulps either side, on
               each of the six columns (that column uncoupled, so its pivot is exact; the others a coupled SPD block)
  ill          SPD H with cond 1e6 .. 3e7 that the fast path still takes: the bound, not a fixed tolerance, decides
  axis         exact zero rows / columns: a floor (rank 3: rot_z, t_x, t_y unobserved) and a corridor (rank 5: t_y unobserved)
  nonaxis      H = J^T J with small-integer J of rank 4 and 5, exactly representable
  zero         H = 0, g = 0, n_valid = 0
  nan          NaN in one off-diagonal pair of H, in every entry of H and g (a query on its corner line), in g alone
  so3          H = I so dx = g exactly: |dtheta| = 0, eps, one ulp either side of eps, pi, 7 (> 2 pi)
  thres        H = I, dx along one axis: the norm equal to its threshold, and one ulp below
  second       LOAM's second clause at iteration 0 (last norms 0, thresholds below the dx norms): |dtheta| = fl(1e-4) and one ulp
               below; and |dtheta| < 1e-4 with |dt| > 1e-4 (the clause needs both)
  cut          the full-pivot rank cut `pivot <= 6 eps max`: a diagonal H whose smallest pivot is exactly 6 eps (dropped), one ulp
               above it and 20 eps (kept), each on its own column (the fast path declines all three)
  cap          max_iterations = 1 at iteration 0; iteration max - 1 and max - 2
  gate         LOAM n_valid 49 / 50 / 51; NDT n_valid min - 1 / min / min + 1 at iteration 3
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np

from tests.gn_ref import FULL, ICP, IVOX, KNN, LOAM, NDT, pack

EPS = float(np.finfo(np.float64).eps)
FAMILIES = (IVOX, NDT, ICP)       # one of each solver / update side / stop rule
ALL = (ICP, NDT, IVOX, KNN, FULL)


@dataclass
class Case:
    name: str
    kind: str
    method: int
    tot: np.ndarray
    R: np.ndarray = field(default_factory=lambda: np.eye(3))
    t: np.ndarray = field(default_factory=lambda: np.zeros(3))
    last_rot: float = 0.0
    last_pos: float = 0.0
    iter: int = 0
    max_iterations: int = 10
    min_effective: int = 50
    rot_thres: float = 0.01
    pos_thres: float = 0.01
    expect: dict = field(default_factory=dict)

    def probe(self):
        return dict(method=self.method, max_iterations=self.max_iterations, min_effective=self.min_effective, iter=self.iter,
                    rot_thres=self.rot_thres, pos_thres=self.pos_thres, R=self.R, t=self.t, last_rot=self.last_rot,
                    last_pos=self.last_pos, tot=self.tot)

    def state(self):
        return dict(R=self.R, t=self.t, last_rot=self.last_rot, last_pos=self.last_pos, iter=self.iter)

    def params(self):
        return dict(max_iterations=self.max_iterations, min_effective=self.min_effective, rot_thres=self.rot_thres,
                    pos_thres=self.pos_thres)


def rot(rpy):
    r, p, y = rpy
    Rx = np.array([[1, 0, 0], [0, math.cos(r), -math.sin(r)], [0, math.sin(r), math.cos(r)]])
    Ry = np.array([[math.cos(p), 0, math.sin(p)], [0, 1, 0], [-math.sin(p), 0, math.cos(p)]])
    Rz = np.array([[math.cos(y), -math.sin(y), 0], [math.sin(y), math.cos(y), 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def _pose(rng):
    return rot(rng.uniform(-0.6, 0.6, 3)), rng.uniform(-20, 20, 3)


def _ulps(x, k):
    for _ in range(abs(k)):
        x = np.nextafter(x, np.inf if k > 0 else -np.inf)
    return float(x)


def _rot_pos(method, rotv, posv):
    """dx in the method's layout from its rotation and translation parts."""
    return np.r_[posv, rotv] if method == ICP else np.r_[rotv, posv]


def well_posed():
    out = []
    rng = np.random.default_rng(11)
    for method in ALL:
        for scale in (1e-6, 1e-3, 1.0, 1e3, 1e6, 1e9, 1e12):
            J = rng.normal(size=(40, 6))
            H = J.T @ J * scale
            x = rng.normal(size=6) * 0.05
            g = H @ x
            R, t = _pose(rng)
            out.append(Case(f"well_posed_{method}_{scale:g}", "well_posed", method, pack(H, g, 100), R, t, float(rng.uniform(0, 0.1)),
                            float(rng.uniform(0, 0.1)), iter=2, expect=dict(spd=True, spd_decided=True, path="update")))
    return out


def _coupled_block(rng, n=5):
    J = rng.normal(size=(3 * n, n))
    B = J.T @ J
    return B / np.max(np.diag(B))


def guard():
    out = []
    rng = np.random.default_rng(12)
    for method in FAMILIES:
        for k in range(6):
            others = [i for i in range(6) if i != k]
            B = _coupled_block(rng)
            H = np.zeros((6, 6))
            H[np.ix_(others, others)] = B
            dmax = float(np.max(np.diag(H)))
            tiny = 1e-8 * dmax
            for d in (-2, -1, 0, 1, 2):
                Hk = H.copy()
                Hk[k, k] = _ulps(tiny, d)
                x = rng.normal(size=6) * 0.01
                g = Hk @ x
                R, t = _pose(rng)
                out.append(Case(f"guard_{method}_col{k}_{d:+d}ulp", "guard", method, pack(Hk, g, 100), R, t, 1.0, 1.0, iter=1,
                                expect=dict(spd=d > 0, spd_decided=True, path="update")))
    return out


def ill():
    out = []
    rng = np.random.default_rng(13)
    for method in FAMILIES:
        for cond in (1e6, 1e7, 3e7):
            Q, _ = np.linalg.qr(rng.normal(size=(6, 6)))
            lam = np.geomspace(1.0, 1.0 / cond, 6)
            H = (Q * lam) @ Q.T
            H = 0.5 * (H + H.T)
            x = rng.normal(size=6) * 0.01
            g = H @ x
            R, t = _pose(rng)
            out.append(Case(f"ill_{method}_{cond:g}", "ill", method, pack(H, g, 100), R, t, 1.0, 1.0, iter=1,
                            expect=dict(spd=True, spd_decided=True, path="update")))
    return out


def _plane_rows(rng, n, normal, offset, box=8.0):
    """Point-to-plane Jacobian rows [p x n, n] of n points on the plane n.p = offset, coordinates multiples of 1/8."""
    rows = []
    normal = np.asarray(normal, float)
    for _ in range(n):
        p = np.round(rng.uniform(-box, box, 3) * 8) / 8
        p -= normal * (normal @ p - offset)
        rows.append(np.r_[np.cross(p, normal), normal])
    return np.array(rows)


def axis():
    out = []
    rng = np.random.default_rng(14)
    floor = _plane_rows(rng, 40, (0, 0, 1), -1.75)
    corridor = np.vstack([floor, _plane_rows(rng, 20, (1, 0, 0), 2.0), _plane_rows(rng, 20, (-1, 0, 0), 2.0)])
    for label, J, zero in (("floor", floor, [2, 3, 4]), ("corridor", corridor, [4])):
        H = J.T @ J
        r = np.round(rng.uniform(-1, 1, len(J)) * 64) / 1024
        g = -(J.T @ r)
        assert np.all(H[zero] == 0) and np.all(g[zero] == 0)
        for method in ALL:
            exp = dict(path="update")
            if method in LOAM:
                exp.update(spd=False, solver="fullpiv", rank=6 - len(zero), rank_decided=True)
            elif method == ICP:
                exp.update(path="skip", det_zero=(True, True))
            else:
                exp.update(spd=False, solver="lu")
            R, t = _pose(rng)
            out.append(Case(f"axis_{label}_{method}", "axis", method, pack(H, g, 100), R, t, 1.0, 1.0, iter=1, expect=exp))
    return out


def nonaxis():
    out = []
    rng = np.random.default_rng(15)
    for rank in (4, 5, 4, 5):
        A = rng.integers(-3, 4, size=(40, rank)).astype(float)
        B = rng.integers(-2, 3, size=(rank, 6)).astype(float)
        while np.linalg.matrix_rank(B) < rank:
            B = rng.integers(-2, 3, size=(rank, 6)).astype(float)
        J = A @ B
        H = J.T @ J
        g = -(J.T @ rng.integers(-3, 4, size=40).astype(float))
        assert np.max(np.abs(H)) < 2 ** 40  # every entry an exact integer
        for method in (IVOX, NDT, ICP):
            out.append(Case(f"nonaxis_rank{rank}_{len(out)}_{method}", "nonaxis", method, pack(H, g, 100), iter=1,
                            rot_thres=1e-300, pos_thres=1e-300, expect=dict(spd=False, spd_decided=True)))
    return out


def zero():
    out = []
    for method in ALL:
        exp = {IVOX: dict(path="update", stop=True, stop_by="thresholds", converged=0, rank=0),
               KNN: dict(path="update", stop=True, stop_by="thresholds", converged=0, rank=0),
               FULL: dict(path="update", stop=True, stop_by="thresholds", converged=0, rank=0),
               ICP: dict(path="skip", stop=False, det_zero=(True, True)),
               NDT: dict(path="gate_fail", stop=True, failed=1, converged=0)}[method]
        out.append(Case(f"zero_{method}", "zero", method, pack(np.zeros((6, 6)), np.zeros(6), 0), expect=exp))
    return out


def nan():
    out = []
    rng = np.random.default_rng(16)
    J = rng.normal(size=(40, 6))
    H0 = J.T @ J
    g0 = H0 @ (rng.normal(size=6) * 0.01)
    for method in FAMILIES:
        Ha = H0.copy()
        Ha[1, 4] = Ha[4, 1] = np.nan
        out.append(Case(f"nan_offdiag_{method}", "nan", method, pack(Ha, g0, 100), expect=dict(spd=False)))
        out.append(Case(f"nan_all_{method}", "nan", method, pack(np.full((6, 6), np.nan), np.full(6, np.nan), 100), expect=dict(spd=False)))
        gb = g0.copy()
        gb[2] = np.nan
        out.append(Case(f"nan_g_{method}", "nan", method, pack(H0, gb, 100), expect=dict(spd=True)))
    return out


def so3():
    out = []
    rng = np.random.default_rng(17)
    thetas = {"0": 0.0, "eps": EPS, "eps-1ulp": _ulps(EPS, -1), "eps+1ulp": _ulps(EPS, 1), "pi": math.pi, "7": 7.0}
    for method in FAMILIES:
        for label, th in thetas.items():
            axis_ = rng.integers(0, 3)
            rv = np.zeros(3)
            rv[axis_] = th
            g = _rot_pos(method, rv, np.zeros(3))
            R, t = _pose(rng)
            out.append(Case(f"so3_{method}_{label}", "so3", method, pack(np.eye(6), g, 100), R, t, 1.0, 1.0, iter=1,
                            rot_thres=1e-300, pos_thres=1e-300, expect=dict(applied=th > EPS, exp_decided=True)))
    return out


def thres():
    out = []
    rng = np.random.default_rng(18)
    for method in FAMILIES:
        for which in ("rot", "pos"):
            thr = 0.005 if method != IVOX else 0.01
            for d, stop in ((0, False), (-1, True)):
                v = np.zeros(3)
                v[rng.integers(0, 3)] = _ulps(thr, d) * (1 if rng.uniform() < 0.5 else -1)
                rv, pv = (v, np.zeros(3)) if which == "rot" else (np.zeros(3), v)
                R, t = _pose(rng)
                exp = dict(stop=stop, stop_decided=True, stop_by="thresholds" if stop else "")
                if method == ICP:
                    exp["converged"] = 1 if stop else -1
                out.append(Case(f"thres_{method}_{which}_{d:+d}ulp", "thres", method, pack(np.eye(6), _rot_pos(method, rv, pv), 100), R, t,
                                1.0, 1.0, iter=1, rot_thres=thr, pos_thres=thr, expect=exp))
    return out


def second():
    out = []
    rng = np.random.default_rng(19)
    for method in LOAM:
        for label, rv, pv, stop in (("at", [1e-4, 0, 0], [0, 0, 0], False), ("below", [_ulps(1e-4, -1), 0, 0], [0, 0, 0], True),
                                    ("pos_open", [5e-5, 0, 0], [0, 1e-3, 0], False)):
            R, t = _pose(rng)
            out.append(Case(f"second_{method}_{label}", "second", method, pack(np.eye(6), _rot_pos(method, np.array(rv), np.array(pv)), 100),
                            R, t, 0.0, 0.0, iter=0, rot_thres=1e-5, pos_thres=1e-5,
                            expect=dict(stop=stop, stop_decided=True, stop_by="second" if stop else "")))
    return out


def cut():
    out = []
    rng = np.random.default_rng(22)
    for method in FAMILIES:
        for k, (label, piv) in enumerate((("6eps", 6 * EPS), ("6eps+1ulp", _ulps(6 * EPS, 1)), ("20eps", 20 * EPS))):
            col = (2 * k + 1) % 6
            d = np.array([1.0, 0.5, 2.0, 1.0, 0.25, 1.5]) * (2.0 ** -1)
            d[np.argmax(d)] = 1.0
            d[col] = piv
            g = np.round(rng.uniform(-1, 1, 6) * 64) / 4096
            g[col] = piv * 3.0  # dx = 3 on the small pivot's column where it is kept
            exp = dict(spd=False, spd_decided=True, path="update")
            if method in LOAM:
                exp.update(solver="fullpiv", rank=5 if label == "6eps" else 6, rank_decided=True)
            R, t = _pose(rng)
            out.append(Case(f"cut_{method}_{label}", "cut", method, pack(np.diag(d), g, 100), R, t, 1.0, 1.0, iter=1, expect=exp))
    return out


def cap():
    out = []
    rng = np.random.default_rng(20)
    for method in FAMILIES:
        for mx, it, stop in ((1, 0, True), (10, 9, True), (10, 8, False)):
            R, t = _pose(rng)
            g = _rot_pos(method, np.array([0.05, -0.02, 0.01]), np.array([0.2, 0.1, -0.1]))
            out.append(Case(f"cap_{method}_max{mx}_it{it}", "cap", method, pack(np.eye(6), g, 100), R, t, 1.0, 1.0, iter=it,
                            max_iterations=mx, expect=dict(stop=stop, stop_by="cap" if stop else "")))
    return out


def gate():
    out = []
    rng = np.random.default_rng(21)
    J = rng.normal(size=(40, 6))
    H = J.T @ J
    g = H @ (rng.normal(size=6) * 0.02)
    for method in LOAM:
        for n in (49, 50, 51):
            R, t = _pose(rng)
            out.append(Case(f"gate_{method}_{n}", "gate", method, pack(H, g, n), R, t, 1.0, 1.0, iter=2,
                            expect=dict(converged=1 if n >= 50 else 0, path="update")))
    for d in (-1, 0, 1):
        R, t = _pose(rng)
        m = 50
        exp = dict(failed=1, converged=0, stop=True, path="gate_fail") if d < 0 else dict(failed=0, converged=1, path="update")
        out.append(Case(f"gate_ndt_min{d:+d}", "gate", NDT, pack(H, g, m + d), R, t, iter=3, min_effective=m, expect=exp))
    return out


def all_cases():
    return well_posed() + guard() + ill() + axis() + nonaxis() + zero() + nan() + so3() + thres() + second() + cut() + cap() + gate()


# ---- whole Matches for the replays -----------------------------------------------------------------------------------------------
@dataclass
class MatchScene:
    """One Match to replay: the plug-in, its configuration overrides, the map clouds, the scan (ordered cloud for ICP / NDT, planar
    cloud for the LOAM plug-ins, plus LoamFull's corner cloud) and the initial pose.  `reaches` names the branch the Match is built
    to end on (checked from the reference): "fallback" (the pivoting solver on every iteration), "second" (LOAM's second clause),
    "cap" (max_iterations), "gate" (NDT's effective-point gate after iteration 0)."""
    name: str
    method: int
    cfg: dict
    maps: list
    scan: np.ndarray
    T: np.ndarray
    corner: np.ndarray | None = None
    reaches: str = ""

    def config(self):
        from funny_lidar_slam_b200 import default_config
        from funny_lidar_slam_b200._abi import FLS_FLAG_ITER_LOG
        return default_config(self.method, flags=FLS_FLAG_ITER_LOG, **self.cfg)


def floor_scene(method=IVOX):
    """A flat floor seen from 1.75 m: only z, roll and pitch are observed, H has three near-zero directions and the fast path
    declines it on every iteration."""
    rng = np.random.default_rng(31)
    g = np.arange(-24.0, 24.0, 0.25)
    xx, yy = np.meshgrid(g, g)
    mp = np.stack([xx.ravel() + rng.uniform(-0.05, 0.05, xx.size), yy.ravel() + rng.uniform(-0.05, 0.05, xx.size),
                   np.full(xx.size, -1.75), np.zeros(xx.size)], 1).astype(np.float32)
    r = rng.uniform(3.0, 20.0, 3000)
    a = rng.uniform(-math.pi, math.pi, 3000)
    scan = np.stack([r * np.cos(a), r * np.sin(a), np.full(3000, -1.75), np.zeros(3000)], 1).astype(np.float32)
    T = np.eye(4)
    T[:3, :3] = rot((0.01, -0.008, 0.0))
    T[:3, 3] = (0.0, 0.0, 0.04)
    cfg = dict(max_iterations=10)
    if method == KNN:
        cfg.update(map_cloud_filter_size=0.2)
    return MatchScene(f"floor_{method}", method, cfg, [mp], scan, T, reaches="fallback")


def synth_scenes(world, traj, scene16):
    from funny_lidar_slam_b200 import synth
    m, s, guess = scene16["map"], scene16["scan"], scene16["guess"]
    out = [MatchScene("synth_icp", ICP, {}, [m], s, guess), MatchScene("synth_ndt", NDT, {}, [m], s, guess),
           MatchScene("synth_ivox", IVOX, {}, [m], s, guess), MatchScene("synth_kd", KNN, {}, [m], s, scene16["guess_small"]),
           MatchScene("synth_ivox_second", IVOX, dict(max_iterations=30, rotation_converge_thres=0.0, position_converge_thres=0.0),
                      [m], s, guess, reaches="second"),
           MatchScene("synth_ivox_cap", IVOX, dict(max_iterations=3, rotation_converge_thres=0.0, position_converge_thres=0.0), [m], s,
                      guess, reaches="cap"),
           # from this guess the effective count goes 204, 198, ...: a gate of 200 passes iteration 0 and fails iteration 1
           MatchScene("synth_ndt_gate", NDT, dict(ndt_min_effective_pts=200), [m], s, synth.perturb_pose(traj[5], seed=11, dpos=0.6, drot_deg=5.0),
                      reaches="gate")]
    # LoamFull: feature clouds of a projected scan, maps from neighbouring poses (loam_full_kdtree.h runs in mapping mode here)
    maps_p, maps_c = [], []
    for k in (3, 4, 6, 7):
        p, c = _features(world, traj[k], k)
        maps_p.append(_to_world(p, traj[k]))
        maps_c.append(_to_world(c, traj[k]))
    p5, c5 = _features(world, traj[5], 55)
    out.append(MatchScene("synth_full", FULL, dict(localization_mode=1), [np.concatenate(maps_p), np.concatenate(maps_c)], p5,
                          synth.perturb_pose(traj[5], dpos=0.1, drot_deg=1.0), corner=c5))
    return out


def _features(world, pose, seed):
    from funny_lidar_slam_b200 import synth
    from oracle import pyoracle as orc
    proj = synth.make_projected_scan(world, pose, kind="spin", sensor="vlp16", seed=seed)
    ci, pi, _ = orc.extract_features(proj["depth"], proj["col"], len(proj["ordered"]), proj["row_start"], proj["row_end"], 1.0, 0.1)
    return proj["ordered"][pi].copy(), proj["ordered"][ci].copy()


def _to_world(pts, T):
    out = pts.copy()
    out[:, :3] = (pts[:, :3].astype(np.float64) @ T[:3, :3].T + T[:3, 3]).astype(np.float32)
    return out


def edge_scenes():
    """The earlier edge tests' scenes, run for several iterations."""
    from tests import ivox_scenes, loam_kd_scenes, ndt_icp_scenes
    out = []
    s = ivox_scenes.s1_dense_staged()
    out.append(MatchScene("edge_ivox_s1", IVOX, dict(max_iterations=5), [s.map], s.scan, np.eye(4)))
    n = ndt_icp_scenes.ndt_axes()
    out.append(MatchScene("edge_ndt_axes", NDT, dict(max_iterations=5, ndt_voxel_size=n.voxel, ndt_min_points_in_voxel=n.min_pts,
                                                     ndt_max_points_in_voxel=n.max_pts, source_cloud_filter_size=n.leaf,
                                                     ndt_outlier_thres=n.thres, ndt_min_effective_pts=1), n.calls, n.scan, n.T))
    c = ndt_icp_scenes.icp_gate(1.0)
    out.append(MatchScene("edge_icp_gate", ICP, dict(max_iterations=5, icp_max_correspond_distance=c.max_corr, source_cloud_filter_size=0.01,
                                                     map_cloud_filter_size=0.01), [c.map], c.scan, c.T))
    k = loam_kd_scenes.kd_shells()
    out.append(MatchScene("edge_kd_shells", KNN, dict(max_iterations=5, map_cloud_filter_size=k.leaf), [k.planar_map], k.planar, k.T))
    f = loam_kd_scenes.full_corners()
    out.append(MatchScene("edge_full_corners", FULL, dict(max_iterations=5, localization_mode=0, map_cloud_filter_size=f.leaf,
                                                          corner_map_filter_size=f.leaf, point_search_thres=f.thres,
                                                          line_ratio_thres=f.line_ratio, point_to_planar_thres=f.plane_thres),
                          [f.planar_map, f.corner_map], f.planar, f.T, corner=f.corner))
    return out
