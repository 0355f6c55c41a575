"""Batch Match for IcpOptimized and LoamPointToPlaneKdtree against B sequential single Matches, with device-resident scans.

  (a) seq   : B sequential fls_match_device calls
  (b) batch : one fls_match_batch_device call (one cooperative launch, a sub-grid and a Gauss-Newton loop per scan)

Shapes of bench.py's side entries icp_16line and loam_kdtree_16line: the default synthetic world, its surface map at 0.3 m, 16-line
scans (vlp16, the raw scan standing in for the kd-tree plug-in's planar cloud) at bench.py's three trajectory poses, cycled to fill
a batch, guesses perturbed by 0.3 m / 3 deg (ICP) and 0.1 m / 1 deg (kd-tree).  Every slot of a batch has its own device buffer:
the ICP batch voxel-filters a repeated (pointer, count) once, and a fleet or an offline run has distinct scans, so sharing buffers
between slots would time less work than B single Matches do.  Wall time per scan is a host clock around calls that end in a
synchronise; the fused kernel's time comes from FLS_FLAG_PROFILE (CUDA events around the one Gauss-Newton launch of a call).  Parity: the largest entry of the
difference of the 4x4 poses of (b) and (a), and whether converged / iterations / n_valid are equal.  Prints the card's name and
power limit and one JSON line per (plug-in, B).

    python tools/bench_icp_kd_batch.py [--scans 200] [--warmup 20] [--sizes 1,8,32,64] [--out FILE.jsonl]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=200, help="timed scans per leg (rounded up to whole batches)")
    ap.add_argument("--warmup", type=int, default=20, help="warm-up scans per leg (rounded up to whole batches)")
    ap.add_argument("--sizes", default="1,8,32,64")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    from funny_lidar_slam_b200 import _abi, synth
    from funny_lidar_slam_b200.registration import Registration
    if not torch.cuda.is_available():
        raise SystemExit("bench_icp_kd_batch needs a CUDA device")
    card = _card()
    print(f"card: {card}", flush=True)
    world = synth.make_world()
    traj = synth.trajectory(16)
    mp = synth.make_surface_map(world, spacing=0.3, seed=4321)
    n_pool = 3  # bench.py's three scans, cycled
    sizes = [int(b) for b in args.sizes.split(",")]
    out = open(args.out, "a") if args.out else None
    for name, method, dpos, drot in (("icp_16line", _abi.FLS_ICP_P2P, 0.3, 3.0), ("loam_kdtree_16line", _abi.FLS_P2PLANE_KNN, 0.1, 1.0)):
        scans = [synth.make_scan(world, traj[3 + 2 * i], "vlp16", seed=300 + i)["points"] for i in range(n_pool)]
        d_pool = [torch.from_numpy(s).cuda() for s in scans]
        reg = Registration(_abi.default_config(method, flags=_abi.FLS_FLAG_PROFILE))
        reg.AddCloudToLocalMap([mp])
        for B in sizes:
            idx = [k % n_pool for k in range(B)]
            guesses = np.stack([synth.perturb_pose(traj[3 + 2 * i], seed=900 + k, dpos=dpos, drot_deg=drot) for k, i in enumerate(idx)])
            d_slots = [d_pool[i].clone() for i in idx]  # one buffer per slot (see above)
            ptrs, ns = [t.data_ptr() for t in d_slots], [len(scans[i]) for i in idx]
            n_calls = -(-args.scans // B)
            n_warm = -(-args.warmup // B)

            def seq():
                res, k_ms = [], 0.0
                for k in range(B):
                    T = guesses[k].copy()
                    ok = reg.match_device(ptrs[k], ns[k], T)
                    st = reg.last_stats
                    res.append((ok, T, st.iterations, st.n_valid))
                    k_ms += st.kernel_ms
                return res, k_ms

            def batch():
                oks, Ts = reg.match_batch_device(ptrs, ns, guesses)
                sts = reg.last_batch_stats
                return [(bool(oks[k]), Ts[k], sts[k].iterations, sts[k].n_valid) for k in range(B)], sts[0].kernel_ms

            row = {"plugin": name, "B": B, "card": card, "timed_scans": n_calls * B}
            results = {}
            for leg, fn in (("seq", seq), ("batch", batch)):
                for _ in range(n_warm):
                    fn()
                torch.cuda.synchronize()
                k_ms = 0.0
                its = 0
                t0 = time.perf_counter()
                for _ in range(n_calls):
                    res, km = fn()  # every call ends in the handle's stream synchronise
                    k_ms += km
                    its += sum(r[2] for r in res)
                wall = time.perf_counter() - t0
                results[leg] = res
                row[leg] = {"wall_us_per_scan": 1e6 * wall / (n_calls * B), "scans_per_s": n_calls * B / wall,
                            "kernel_us_per_scan": 1e3 * k_ms / (n_calls * B), "mean_iterations": its / (n_calls * B)}
            a, b = results["seq"], results["batch"]
            dT = max(float(np.max(np.abs(x[1] - y[1]))) for x, y in zip(a, b))  # largest entry of T_batch - T_seq
            row["parity"] = {"max_abs_dT": dT, "discrete_equal": all(x[0] == y[0] and x[2] == y[2] and x[3] == y[3] for x, y in zip(a, b))}
            line = json.dumps(row)
            print(line, flush=True)
            if out:
                out.write(line + "\n")
        reg.close()
    if out:
        out.close()


if __name__ == "__main__":
    main()
