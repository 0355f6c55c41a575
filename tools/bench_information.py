"""Cost of FLS_FLAG_INFORMATION: median device ms (the call's CUDA events, fls_match_stats.gpu_ms) and wall ms of fls_match_device and
of a 64-scan fls_match_batch_device, with and without the flag, for every plug-in on the bench scene (a 64-line scan against a map
built from neighbouring scans, localization mode).  Prints one JSON line; writes nothing."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch

    from funny_lidar_slam_b200 import FLS_ICP_P2P, FLS_NDT, FLS_P2PLANE_IVOX, FLS_P2PLANE_KNN, default_config, synth
    from funny_lidar_slam_b200._abi import FLS_FLAG_INFORMATION, FLS_LOAM_FULL
    from funny_lidar_slam_b200.registration import Registration

    world, traj = synth.make_world(), synth.trajectory(16)
    scan = synth.make_scan(world, traj[6], "hdl64", seed=6)["points"]
    mp = synth.make_map_from_scans(world, traj[2:12:3], "hdl64", leaf=0.3)
    guess = synth.perturb_pose(traj[6], dpos=0.05, drot_deg=0.5)
    d_scan = torch.from_numpy(np.ascontiguousarray(scan)).cuda()
    methods = {"ivox": FLS_P2PLANE_IVOX, "ndt": FLS_NDT, "icp": FLS_ICP_P2P, "kd": FLS_P2PLANE_KNN, "full": FLS_LOAM_FULL}
    out = {"gpu": subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                                 text=True).stdout.strip(), "reps": args.reps, "scan_points": len(scan), "map_points": len(mp), "results": {}}
    for name, method in methods.items():
        res = {}
        for flag in (0, FLS_FLAG_INFORMATION):
            g = Registration(default_config(method, localization_mode=1, flags=flag))
            g.AddCloudToLocalMap([mp, mp[::3].copy()] if method == FLS_LOAM_FULL else [mp])
            key = "flag" if flag else "plain"

            def single():
                T = guess.copy()
                if method == FLS_LOAM_FULL:
                    g.match_cluster_device(0, 0, d_scan.data_ptr(), len(scan), d_scan.data_ptr(), len(scan) // 7, T)
                else:
                    g.match_device(d_scan.data_ptr(), len(scan), T)
                return g.last_stats.gpu_ms

            def batch():
                B = 64
                g.match_batch_device([d_scan.data_ptr()] * B, [len(scan)] * B, np.stack([guess] * B))
                return g.last_batch_stats[0].gpu_ms

            for what, fn in (("single", single), ("batch64", batch)):
                if what == "batch64" and method == FLS_LOAM_FULL:
                    continue
                dev, wall = [], []
                for i in range(args.warmup + args.reps):
                    t0 = time.perf_counter()
                    ms = fn()
                    t1 = time.perf_counter()
                    if i >= args.warmup:
                        dev.append(ms)
                        wall.append((t1 - t0) * 1e3)
                res[f"{what}_{key}"] = {"device_ms_median": float(np.median(dev)), "wall_ms_median": float(np.median(wall))}
            g.close()
        out["results"][name] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
