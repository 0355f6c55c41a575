"""fls_relocalize_multi (one search over the grids of G guesses) against G separate fls_relocalize_wide calls on the same guesses.

Scene: tools/bench_relocalize_wide.py's (the default synthetic world, its 0.3 m surface map as the global map, one 64-line scan at
trajectory(16)[5]), plus a keyframe store of 48 64-line scans taken every 2 m along the figure-8 trajectory.  The guesses are
place_pose of the first G candidates of place_query(scan, 20), G = 1, 5 and 20; the local map is cut at the first candidate.
Grids, coarse_leaf 1.0, max_range 2.0, n_refine 64:
  - near: +-4 m at 0.5 m x +-30 degrees at 5 degrees (3 757 hypotheses per guess): every hypothesis scored;
  - mid: +-10 m at 0.5 m x +-45 degrees at 2 degrees (75 645 per guess): the branch and bound descends at G = 20 (1.51 M).
Per (plug-in, grid, G), one JSON line: wall ms (a host clock around calls that end in a synchronise; the lattice is built in the
warm-up), evaluations, Matches run (refined poses), host waits and launches, and the chosen pose's error, for the multi call and for
the G wide calls together (their result: the accepted pose of lowest fitness, else the lowest fitness, as a caller would pick).
The card's name, power limit and max SM clock are read in the same run.

    python tools/bench_relocalize_multi.py [--reps 3] [--warmup 1] [--out FILE.jsonl]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

GRIDS = {"near": dict(xy_radius=4.0, xy_step=0.5, yaw_range=np.deg2rad(30.0), yaw_step=np.deg2rad(5.0)),
         "mid": dict(xy_radius=10.0, xy_step=0.5, yaw_range=np.deg2rad(45.0), yaw_step=np.deg2rad(2.0))}


def _time(call, reps, warmup):
    for _ in range(warmup):
        out = call()
    wall = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = call()
        wall.append((time.perf_counter() - t0) * 1e3)
    return out, wall


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from bench_relocalize import _card
    from funny_lidar_slam_b200 import _abi, synth
    from funny_lidar_slam_b200._lib import FlsError, lib
    from funny_lidar_slam_b200.keyframes import KeyFrameStore, place_pose
    from funny_lidar_slam_b200.registration import Registration
    if lib().fls_device_count() < 1:
        raise SystemExit("bench_relocalize_multi needs a CUDA device")
    card = _card()
    world = synth.make_world()
    mp = synth.make_surface_map(world, spacing=0.3, seed=4321)
    T_true = synth.trajectory(16)[5]
    scan = synth.make_scan(world, T_true, "hdl64", seed=55)["points"]
    d_scan = torch.from_numpy(scan).cuda()
    torch.cuda.synchronize()
    traj = synth.trajectory(48, step=2.0)
    kf = [synth.make_scan(world, T, "hdl64", seed=900 + i)["points"] for i, T in enumerate(traj)]
    store = KeyFrameStore(sum(len(c) for c in kf))
    for c in kf:
        store.add(c)
    cands = store.place_query(scan, 20)
    guesses = [place_pose(traj[c.id], c.yaw) for c in cands]
    errs = [synth.pose_error(T, T_true) for T in guesses]
    print(json.dumps(dict(bench="relocalize_multi", card=card, candidates=[int(c.id) for c in cands],
                          guess_error_m=[round(e[0], 2) for e in errs], guess_error_deg=[round(float(np.rad2deg(e[1])), 1) for e in errs])), flush=True)
    lines = []
    for name, method in (("p2plane_ivox", _abi.FLS_P2PLANE_IVOX), ("ndt", _abi.FLS_NDT)):
        g = Registration(_abi.default_config(method, ndt_capacity=2000000))
        g.set_global_map(mp)
        _, n_local = g.update_local_map(guesses[0])
        for grid, kw in GRIDS.items():
            search = dict(coarse_leaf=1.0, max_range=2.0, accept_fitness=1.0, n_refine=64, **kw)
            for G in (1, 5, 20):
                gs = guesses[:G]
                try:
                    (m, ev), wm = _time(lambda: g.relocalize_multi_device(d_scan.data_ptr(), d_scan.shape[0], gs, **search), args.reps, args.warmup)
                except FlsError as e:  # FLS_ERR_CAPACITY: too many blocks survive a level
                    print(json.dumps(dict(bench="relocalize_multi", plugin=name, grid=grid, guesses=G, card=card, status=e.status)), flush=True)
                    continue
                levels = g.relocalize_wide_levels()
                sep, ws = _time(lambda: [g.relocalize_wide_device(d_scan.data_ptr(), d_scan.shape[0], T, **search) for T in gs], args.reps, args.warmup)
                pool = [r for r, _ in sep if r.accepted] or [r for r, _ in sep]
                best = min(pool, key=lambda r: r.fitness)
                dt, dr = synth.pose_error(m.T, T_true)
                dts, drs = synth.pose_error(best.T, T_true)
                line = dict(bench="relocalize_multi", plugin=name, grid=grid, guesses=G, card=card, scan_points=int(len(scan)),
                            local_map_points=int(n_local), n_hypotheses=m.n_hypotheses,
                            multi_ms_median=float(np.median(wm)), multi_ms_min=float(np.min(wm)), multi_evaluations=int(ev),
                            multi_nodes_per_level=levels, multi_matches=m.n_refined, multi_host_waits=m.host_waits,
                            multi_gpu_launches=m.gpu_launches, multi_accepted=m.accepted, multi_guess=int(m.best_hypothesis // (m.n_hypotheses // G)),
                            multi_error_m=dt, multi_error_deg=float(np.rad2deg(dr)),
                            separate_ms_median=float(np.median(ws)), separate_ms_min=float(np.min(ws)),
                            separate_evaluations=int(sum(e for _, e in sep)), separate_matches=int(sum(r.n_refined for r, _ in sep)),
                            separate_host_waits=int(sum(r.host_waits for r, _ in sep)), separate_gpu_launches=int(sum(r.gpu_launches for r, _ in sep)),
                            separate_accepted=best.accepted, separate_error_m=dts, separate_error_deg=float(np.rad2deg(drs)))
                print(json.dumps(line), flush=True)
                lines.append(line)
        g.close()
    if args.out:
        with open(args.out, "w") as f:
            for l in lines:
                f.write(json.dumps(l) + "\n")


if __name__ == "__main__":
    main()
