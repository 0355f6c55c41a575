"""Relocalization from a coarse pose (fls_relocalize) against what a caller can do without it.

  (a) reloc : one fls_relocalize_device call — voxel filter, every x-y-yaw hypothesis scored on the device, the n_refine best refined by
              one batch Match, GetFitnessScore of each refined pose, the choice
  (b) loop  : n_refine sequential fls_match_device + fls_fitness from the same start poses (the hypotheses (a) refined)

Scene: the default synthetic world (synth.make_world), its surface map at 0.3 m as the global map, the +-100 m local map cut on the
device at the guess (fls_update_local_map), one 64-line scan (hdl64) at a trajectory pose, and a guess 3.3 m, 2.6 m and 33 degrees
off.  Searches: +-10 m at 1 m x the full circle at 10 degrees (15 876 hypotheses) and +-10 m at 0.5 m x 5 degrees (121 032),
coarse_leaf 1.0, max_range 2.0, n_refine 64.
Wall time is a host clock around calls that end in a synchronise; the coarse stage's device time is the sum of its kernels
(hypotheses, 8-pose scoring, score reduction, radix sort, pick) in a separate torch.profiler run.  Prints one JSON line per plug-in
with the card's name, power limit and max SM clock.

    python tools/bench_relocalize.py [--reps 10] [--warmup 2] [--n-refine 64] [--out FILE.jsonl]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"
    except Exception:
        return "unknown"


def _start_pose(guess, index, xy_radius, xy_step, yaw_step):
    """Start pose of grid index `index` (fls_b200.h: yaw fastest, then x, then y; full circle)."""
    I = int(np.floor(xy_radius / xy_step + 1e-9))
    K = int(np.floor(np.pi / yaw_step + 1e-9))
    k0 = -K + 1 if 2.0 * K * yaw_step >= 2.0 * np.pi - 1e-9 else -K
    n_yaw, nx = K - k0 + 1, 2 * I + 1
    k, i, j = index % n_yaw, (index // n_yaw) % nx, index // (n_yaw * nx)
    psi = (k0 + k) * yaw_step
    c, s = np.cos(psi), np.sin(psi)
    T = guess.copy()
    g0, g1 = guess[0, :3].copy(), guess[1, :3].copy()
    T[0, :3], T[1, :3] = c * g0 - s * g1, s * g0 + c * g1
    T[:3, 3] = guess[:3, 3] + np.array([(i - I) * xy_step, (j - I) * xy_step, 0.0])
    return T


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--n-refine", type=int, default=64)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from funny_lidar_slam_b200 import _abi, synth
    from funny_lidar_slam_b200._lib import lib
    from funny_lidar_slam_b200.registration import Registration
    if lib().fls_device_count() < 1:
        raise SystemExit("bench_relocalize needs a CUDA device")
    card = _card()
    world = synth.make_world()
    mp = synth.make_surface_map(world, spacing=0.3, seed=4321)
    T_true = synth.trajectory(16)[5]
    scan = synth.make_scan(world, T_true, "hdl64", seed=55)["points"]
    a = np.deg2rad(33.0)
    guess = T_true.copy()
    guess[:3, :3] = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]]) @ T_true[:3, :3]
    guess[:3, 3] += [3.3, -2.6, 0.0]
    d_scan = torch.from_numpy(scan).cuda()
    torch.cuda.synchronize()
    lines = []
    for name, method, step, yaw_step in (("p2plane_ivox", _abi.FLS_P2PLANE_IVOX, 1.0, 10.0), ("p2plane_ivox", _abi.FLS_P2PLANE_IVOX, 0.5, 5.0),
                                         ("ndt", _abi.FLS_NDT, 1.0, 10.0), ("ndt", _abi.FLS_NDT, 0.5, 5.0)):
        search = dict(xy_radius=10.0, xy_step=step, yaw_range=np.pi, yaw_step=np.deg2rad(yaw_step), coarse_leaf=1.0, max_range=2.0,
                      accept_fitness=1.0, n_refine=args.n_refine)
        g = Registration(_abi.default_config(method, ndt_capacity=2000000))
        g.set_global_map(mp)
        _, n_local = g.update_local_map(guess)
        call = lambda: g.relocalize_device(d_scan.data_ptr(), d_scan.shape[0], guess, **search)
        for _ in range(args.warmup):
            r = call()
        wall = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            r = call()
            wall.append((time.perf_counter() - t0) * 1e3)
        dt, dr = synth.pose_error(r.T, T_true)
        # coarse-stage kernels, in a run of their own
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        coarse_us, n_k = 0.0, 0
        for e in prof.events():
            k = e.name
            if "reloc_rep_poses_kernel" in k or "pose_score_kernel<8" in k or "RadixSort" in k or "reloc_pick_kernel" in k or "pose_score_reduce" in k:
                coarse_us += e.device_time
                n_k += 1
        # (b) the loop a caller can write today: n_refine Matches + GetFitnessScore from the same start poses
        starts = [_start_pose(guess, int(i), search["xy_radius"], search["xy_step"], search["yaw_step"]) for i in r.refined_index]
        loop_fit = []

        def loop():
            loop_fit.clear()
            out = []
            for T0 in starts:
                T = T0.copy()
                ok = g.match_device(d_scan.data_ptr(), d_scan.shape[0], T)
                loop_fit.append(g.GetFitnessScore(2.0))
                out.append((ok, T))
            return out
        for _ in range(args.warmup):
            res = loop()
        lw = []
        for _ in range(max(1, args.reps // 2)):
            t0 = time.perf_counter()
            res = loop()
            lw.append((time.perf_counter() - t0) * 1e3)
        same = all(abs(f - rf) == 0.0 for f, rf in zip(loop_fit, r.refined_fitness))
        maxdT = max(float(np.max(np.abs(T - rT))) for (_, T), rT in zip(res, r.refined_T))
        line = dict(bench="relocalize", plugin=name, xy_step=step, yaw_step_deg=yaw_step, card=card, scan_points=int(len(scan)), local_map_points=int(n_local),
                    n_hypotheses=r.n_hypotheses, n_refine=r.n_refined, reloc_ms_median=float(np.median(wall)), reloc_ms_min=float(np.min(wall)),
                    coarse_stage_kernels_ms=coarse_us / 1e3, coarse_stage_kernel_count=n_k, loop_ms_median=float(np.median(lw)),
                    loop_ms_min=float(np.min(lw)), accepted=r.accepted, fitness=r.fitness, best_rank=r.best_rank, error_m=dt,
                    error_deg=float(np.rad2deg(dr)), host_waits=r.host_waits, gpu_launches=r.gpu_launches, loop_fitness_equal=same,
                    loop_pose_max_abs_diff=maxdT)
        print(json.dumps(line), flush=True)
        lines.append(line)
        g.close()
    if args.out:
        with open(args.out, "w") as f:
            for l in lines:
                f.write(json.dumps(l) + "\n")


if __name__ == "__main__":
    main()
