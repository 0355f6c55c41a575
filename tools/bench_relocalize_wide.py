"""fls_relocalize_wide (exact branch and bound) against fls_relocalize (every hypothesis scored) on the same grids.

Scene: tools/bench_relocalize.py's (the default synthetic world, its 0.3 m surface map as the global map, the +-100 m local map cut at
the guess, one 64-line scan).  Grids, coarse_leaf 1.0, max_range 2.0, n_refine 64:
  - +-10 m at 1 m x the full circle at 10 degrees (15 876 hypotheses), guess 3.3 m, 2.6 m and 33 degrees off: both entries;
  - +-10 m at 0.5 m x 5 degrees (121 032), the same guess: both entries;
  - +-40 m at 0.5 m x 2 degrees (4 665 780), a guess 20 m, 15 m and 150 degrees off: the wide entry only (fls_relocalize's cap is
    2^20 hypotheses).
Wall time is a host clock around calls that end in a synchronise (the lattice is built in the warm-up, as the map is loaded once).
wide_nodes_per_level lists the nodes the search reached at each level, from its start level down to single hypotheses.
Prints one JSON line per (plug-in, grid) with the card's name, power limit and max SM clock.

    python tools/bench_relocalize_wide.py [--reps 5] [--warmup 1] [--out FILE.jsonl]
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


def _off(T, dx, dy, yaw_deg):
    a = np.deg2rad(yaw_deg)
    out = T.copy()
    out[:3, :3] = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]]) @ T[:3, :3]
    out[:3, 3] += [dx, dy, 0.0]
    return out


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
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from bench_relocalize import _card
    from funny_lidar_slam_b200 import _abi, synth
    from funny_lidar_slam_b200._lib import lib
    from funny_lidar_slam_b200.registration import Registration
    if lib().fls_device_count() < 1:
        raise SystemExit("bench_relocalize_wide needs a CUDA device")
    card = _card()
    world = synth.make_world()
    mp = synth.make_surface_map(world, spacing=0.3, seed=4321)
    T_true = synth.trajectory(16)[5]
    scan = synth.make_scan(world, T_true, "hdl64", seed=55)["points"]
    d_scan = torch.from_numpy(scan).cuda()
    torch.cuda.synchronize()
    near, far = _off(T_true, 3.3, -2.6, 33.0), _off(T_true, 20.0, -15.0, 150.0)
    grids = [("1m10deg", near, dict(xy_radius=10.0, xy_step=1.0, yaw_step=np.deg2rad(10.0)), True),
             ("0.5m5deg", near, dict(xy_radius=10.0, xy_step=0.5, yaw_step=np.deg2rad(5.0)), True),
             ("wide_40m_0.5m2deg", far, dict(xy_radius=40.0, xy_step=0.5, yaw_step=np.deg2rad(2.0)), False)]
    lines = []
    for name, method in (("p2plane_ivox", _abi.FLS_P2PLANE_IVOX), ("ndt", _abi.FLS_NDT)):
        for grid, guess, kw, both in grids:
            search = dict(yaw_range=np.pi, coarse_leaf=1.0, max_range=2.0, accept_fitness=1.0, n_refine=64, **kw)
            g = Registration(_abi.default_config(method, ndt_capacity=2000000))
            g.set_global_map(mp)
            _, n_local = g.update_local_map(guess)
            (w, ev), ww = _time(lambda: g.relocalize_wide_device(d_scan.data_ptr(), d_scan.shape[0], guess, **search), args.reps, args.warmup)
            levels = g.relocalize_wide_levels()
            dt, dr = synth.pose_error(w.T, T_true)
            line = dict(bench="relocalize_wide", plugin=name, grid=grid, card=card, scan_points=int(len(scan)), local_map_points=int(n_local),
                        n_hypotheses=w.n_hypotheses, wide_evaluations=int(ev), wide_nodes_per_level=levels, wide_ms_median=float(np.median(ww)), wide_ms_min=float(np.min(ww)),
                        wide_host_waits=w.host_waits, wide_gpu_launches=w.gpu_launches, accepted=w.accepted, error_m=dt, error_deg=float(np.rad2deg(dr)))
            if both:
                e, we = _time(lambda: g.relocalize_device(d_scan.data_ptr(), d_scan.shape[0], guess, **search), args.reps, args.warmup)
                line.update(exhaustive_evaluations=e.n_hypotheses, exhaustive_ms_median=float(np.median(we)), exhaustive_ms_min=float(np.min(we)),
                            same_picks=list(e.refined_index) == list(w.refined_index), same_best=e.best_hypothesis == w.best_hypothesis)
            print(json.dumps(line), flush=True)
            lines.append(line)
            g.close()
    if args.out:
        with open(args.out, "w") as f:
            for l in lines:
                f.write(json.dumps(l) + "\n")


if __name__ == "__main__":
    main()
