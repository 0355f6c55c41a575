"""Device cost of the translation term of the de-skew: each pre-processing entry against its _motion sibling on the same scan.

A 64-line sweep (tests/deskew_motion_scene.py: HDL-64-shaped, 1800 columns, about 110 k points, the sensor moving at 15 m/s) is put
in device memory once; then, alternating call by call so both see the same machine state:
  a  fls_preprocess_device  vs  fls_preprocess_device_motion        (range gate, de-skew, jump span, voxel filter; device outputs)
  b  fls_preprocess_loam_device  vs  fls_preprocess_loam_device_motion  (projection with de-skew, features, two voxel filters)
Two measurements, in separate phases after a warm-up:
  device  the device time per call: the durations of the call's kernels, copies and memsets as torch.profiler (CUDA activities)
          records them, summed over --prof-calls calls and divided by the count; parent and sibling are profiled in alternating
          windows, --prof-rounds of each.  The library launches on its own streams; the CUDA activity trace sees them all.
  wall    host clocks around calls that return with their work complete (each entry ends in a device synchronise), so IMU upload,
          argument checks and waits are included; medians and the 10th / 90th percentiles in ms over --reps alternating calls.
The counts of every timed _motion call, and its planar cloud at the end, are compared with those of the first _motion call.
Prints the GPU name and power limit read in the same run, then one JSON line.  Needs a GPU: there is no fallback.

    python tools/bench_deskew_motion.py --reps 300 --warmup 30 --prof-calls 100 --prof-rounds 3
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--prof-calls", type=int, default=100)
    ap.add_argument("--prof-rounds", type=int, default=3)
    args = ap.parse_args()
    import torch

    from funny_lidar_slam_b200 import synth
    from funny_lidar_slam_b200._lib import lib
    from funny_lidar_slam_b200.features import LoamFrontEnd, preprocess_device
    from tests import deskew_motion_scene as ms
    if lib().fls_device_count() < 1:
        raise SystemExit("bench_deskew_motion needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "-i", str(args.device), "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(f"GPU: {gpu}")
    world, traj = synth.make_world(), synth.trajectory(16)
    s = ms.moving_sweep(world, traj[3])
    raw, n = s["raw"], len(s["raw"])
    dev = f"cuda:{args.device}"
    d_xyzi = torch.from_numpy(np.ascontiguousarray(raw[:, :4])).to(dev)
    d_time = torch.from_numpy(np.ascontiguousarray(raw[:, 4])).to(dev)
    d_ring = torch.from_numpy(s["ring"]).to(dev)
    d_ord = torch.empty((n, 4), dtype=torch.float32, device=dev)
    d_pl = torch.empty((n, 4), dtype=torch.float32, device=dev)
    sn = synth.SENSORS["hdl64"]
    V, H, h_res = sn.lines, sn.cols, float(np.float32(2 * np.pi / sn.cols))
    d_c = torch.empty((120 * V, 4), dtype=torch.float32, device=dev)
    d_p = torch.empty((V * H, 4), dtype=torch.float32, device=dev)
    torch.cuda.synchronize()
    fe = LoamFrontEnd(H, V, h_res, ms.MIN_D, 80.0, 1.0, 0.1, 0.2, 0.4, device=args.device)
    imu, vel = s["imu"], s["velocity"]

    def pp(v):
        preprocess_device(d_xyzi.data_ptr(), d_time.data_ptr(), n, imu, ms.MIN_D, ms.MAX_D, ms.JUMP, ms.LEAF, device=args.device,
                          device_out=(d_ord.data_ptr(), d_pl.data_ptr()), host_out=False, velocity=v)
        return preprocess_device.last_counts

    def loam(v):
        fe.run_device(d_xyzi.data_ptr(), d_ring.data_ptr(), d_time.data_ptr(), n, imu, device_out=(d_c.data_ptr(), d_p.data_ptr()), host_out=False,
                      velocity=v)
        return fe.last_counts

    out = dict(gpu=gpu, n_points=n, reps=args.reps)
    for name, fn in (("preprocess_device", pp), ("preprocess_loam_device", loam)):
        for _ in range(args.warmup):
            fn(None)
            fn(vel)
        ref_counts = fn(vel)
        ref_pl = d_pl.clone() if fn is pp else d_p.clone()
        t = {"parent": [], "motion": []}
        for k in range(args.reps):
            for which, v in (("parent", None), ("motion", vel)) if k % 2 == 0 else (("motion", vel), ("parent", None)):
                t0 = time.perf_counter()
                c = fn(v)
                t[which].append((time.perf_counter() - t0) * 1e3)
                if which == "motion":
                    assert c == ref_counts
        assert fn(vel) == ref_counts  # the loop may end on a parent call
        now = d_pl if fn is pp else d_p
        assert torch.equal(now[:ref_counts[1]], ref_pl[:ref_counts[1]])
        for which, ts in t.items():
            p10, p50, p90 = np.percentile(ts, [10, 50, 90])
            out[f"{name}_{which}_ms"] = dict(median=round(float(p50), 4), p10=round(float(p10), 4), p90=round(float(p90), 4))
            print(f"{name:24s} {which:7s} median {p50:.4f} ms  (p10 {p10:.4f}, p90 {p90:.4f})")
        out[f"{name}_motion_over_parent"] = round(float(np.median(t["motion"]) / np.median(t["parent"])), 4)
        dev_ms = {"parent": [], "motion": []}
        for _ in range(args.prof_rounds):
            for which, v in (("parent", None), ("motion", vel)):
                dev_ms[which].append(device_ms_per_call(torch, lambda: fn(v), args.prof_calls))
        for which, ms_ in dev_ms.items():
            out[f"{name}_{which}_device_ms"] = [round(x, 4) for x in ms_]
            print(f"{name:24s} {which:7s} device {', '.join(f'{x:.4f}' for x in ms_)} ms per call ({args.prof_rounds} windows)")
    print(json.dumps(out))


def device_ms_per_call(torch, call, n):
    """Summed duration of the CUDA activities (kernels, copies, memsets) recorded over n calls, per call, in ms."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            call()
        torch.cuda.synchronize()
    us = sum(e.time_range.elapsed_us() for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
    if us <= 0:
        raise SystemExit("torch.profiler recorded no CUDA activity")
    return us / n / 1e3


if __name__ == "__main__":
    main()
