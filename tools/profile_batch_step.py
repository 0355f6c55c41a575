#!/usr/bin/env python
"""Device-time profile of the headline step: one batched LOAM-iVox Match of B scans per step on two handles in flight
(`match_batch_begin_device` / `match_batch_end`), a 256 MiB L2 flush before every step — the shape of bench.py's `value` leg.

    python tools/profile_batch_step.py [--steps 6] [--warmup 3] [--batch 8] [--workload p2plane_ivox_64] [--out DIR]

Runs the steps under torch.profiler (CUDA activities) and writes the Chrome trace to DIR/trace.json.  Prints, for every
profiled step, each kernel / memcpy / memset of that stream in start order with its device time and the idle gap before it,
the time between two batch-kernel starts, and the device time of the query preparation (what the batch kernel's stream ran
since its previous batch kernel, the read-back of the previous results aside: table copy, ordering kernels, memsets).
Card name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import WORKLOADS, build_scene, make_cfg  # noqa: E402

BATCH_KERNEL = "p2plane_v9_kernel"


def card_info() -> str:
    import torch
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit not readable"
    return f"{name}, power limit / max SM clock: {q}"


def short(name: str) -> str:
    if name.startswith("void "):
        name = name[5:]
    name = name.replace("(anonymous namespace)::", "")
    base = name.split("(")[0].split("<")[0]
    if "Fill" in name or "fill" in base:
        return "l2_flush (fill)"
    return base.split("::")[-1] or name[:40]


def device_events(trace_path: str):
    with open(trace_path) as f:
        tr = json.load(f)
    ev = []
    for e in tr.get("traceEvents", []):
        if e.get("ph") != "X":
            continue
        cat = e.get("cat", "")
        if cat not in ("kernel", "gpu_memcpy", "gpu_memset"):
            continue
        ev.append((float(e["ts"]), float(e["dur"]), cat, e["name"], e.get("args", {}).get("stream")))
    ev.sort()
    return ev


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--workload", default="p2plane_ivox_64", choices=sorted(WORKLOADS))
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "fls_profile_batch_step"))
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    from funny_lidar_slam_b200.registration import Registration

    if not torch.cuda.is_available():
        raise SystemExit("profile_batch_step.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    wl = WORKLOADS[args.workload]
    B = max(2, min(args.batch, 64))
    n_pool = max(16, 2 * B)
    mp, scans, _, guesses = build_scene(wl, n_pool, lambda m: None)
    cfg = make_cfg(wl, 0, len(mp))
    regs = [Registration(cfg), Registration(cfg)]
    for r in regs:
        r.AddCloudToLocalMap([mp])
    d_scans = [torch.from_numpy(s).to(dev) for s in scans]
    flush_buf = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def ids(i):
        return [(i * B + j) % n_pool for j in range(B)]

    def begin(i):
        k = ids(i)
        regs[i % 2].match_batch_begin_device([d_scans[j].data_ptr() for j in k], [d_scans[j].shape[0] for j in k],
                                             np.stack([guesses[j] for j in k]))

    def end(i):
        return regs[i % 2].match_batch_end()

    def run(first, n):
        for i in range(first, first + n):
            flush_buf.zero_()
            begin(i)
            if i > first:
                end(i - 1)
        end(first + n - 1)
        torch.cuda.synchronize()

    run(0, args.warmup)
    os.makedirs(args.out, exist_ok=True)
    trace = os.path.join(args.out, "trace.json")
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        run(args.warmup, args.steps)
    prof.export_chrome_trace(trace)

    print(f"# {card_info()}")
    print(f"# workload {args.workload}, batch {B}, two handles in flight, trace {trace}")
    report(trace)


def report(trace: str):
    ev = device_events(trace)
    # a step = one launch of the batch kernel; its query preparation = what ran on the same stream since that stream's previous
    # batch kernel, except the read-back of the previous results
    batch = [e for e in ev if short(e[3]).startswith(BATCH_KERNEL)]
    chain_us, chain_n, step_us = [], [], []
    for s in range(1, len(batch)):
        ts, dur, _, _, stream = batch[s]
        prev_same = max((b for b in batch[:s] if b[4] == stream), default=None, key=lambda b: b[0])
        t0 = prev_same[0] + prev_same[1] if prev_same else batch[s - 1][0]
        rows = [e for e in ev if e[4] == stream and t0 <= e[0] < ts and "DtoH" not in e[3] and not short(e[3]).startswith(BATCH_KERNEL)]
        t_step = ts - batch[s - 1][0]
        print(f"\n## step {s}: {t_step:.1f} us between the starts of two batch kernels; stream {stream}")
        print(f"{'gap_us':>8} {'dev_us':>8}  name")
        prev_end = t0
        for r in rows + [batch[s]]:
            nm = short(r[3]) if r[2] == "kernel" else r[3]
            print(f"{r[0] - prev_end:8.1f} {r[1]:8.1f}  {nm}")
            prev_end = r[0] + r[1]
        chain = sum(r[1] for r in rows)
        print(f"   query preparation: {len(rows)} device ops, {chain:.1f} us device time; batch kernel {dur:.1f} us")
        chain_us.append(chain)
        chain_n.append(len(rows))
        step_us.append(t_step)
    if chain_us:
        print(f"\n# summary over {len(chain_us)} steps: step {np.median(step_us):.1f} us median; query preparation "
              f"{np.median(chain_us):.1f} us median device time in {int(np.median(chain_n))} device ops")


if __name__ == "__main__":
    main()
