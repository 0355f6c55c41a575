"""Keyframe-map assembly: the device-resident store (fls_keyframes_assemble) against the two routes that exist without it.

  (a) store   : keyframes resident in a KeyFrameStore, one fls_keyframes_assemble per map
  (b) loop    : what a caller can do with fls_voxel_grid alone — per keyframe fls_voxel_grid (upload, two host waits, copy back) and a
                host TransformPointCloud (the oracle's float transform), concatenation, and one more fls_voxel_grid for the final pass
  (c) oracle  : the CPU oracle composition (orc.voxel_grid, orc.transform_f, concatenation), with its OpenMP thread count

Shapes: System::SaveMap (every keyframe, leaf 0.3, final 0.3) at K = 50, 500, 2000 and LoopClosure::GetSubMap (21 keyframes, leaf
0.2, no final pass).  Keyframes are synthetic 64-line scans (synth.make_scan) placed along synth.trajectory; a pool of --pool distinct
scans is reused cyclically so that K = 2000 does not need 2000 ray casts.  Device time is the store's CUDA-event time (stats.gpu_ms),
wall time a host clock around calls that end in a synchronise.  Every output of (a) is compared bit for bit with (b), and with (c)
where (c) runs.  Prints one JSON line per shape and route, plus the card's name and power limit; --out writes them to a file.

    python tools/bench_keyframe_map.py [--ks 50,500,2000] [--reps 3] [--pool 24] [--cpu-max-k 2000] [--out FILE.jsonl]
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


def _same(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def route_store(store, ids, poses, leaf, final_leaf):
    t0 = time.perf_counter()
    out = store.assemble(ids, poses, leaf, final_leaf)
    wall = (time.perf_counter() - t0) * 1e3
    st = store.last_stats
    return out, dict(wall_ms=wall, gpu_ms=st.gpu_ms, launches=st.gpu_launches, host_waits=st.iterations)


def route_loop(clouds, ids, poses, leaf, final_leaf):
    """fls_voxel_grid per keyframe + host transform; device time is not observable per call, so only wall time is reported."""
    from funny_lidar_slam_b200.registration import voxel_grid
    from oracle import pyoracle as orc
    t0 = time.perf_counter()
    parts = [orc.transform_f(voxel_grid(clouds[i], leaf), T) for i, T in zip(ids, poses)]
    m = np.concatenate(parts) if parts else np.zeros((0, 4), np.float32)
    if final_leaf:
        m = voxel_grid(m, final_leaf)
    wall = (time.perf_counter() - t0) * 1e3
    calls = len(ids) + (1 if final_leaf else 0)
    # voxel_grid_device: 8 library launches and 2 host waits per call, plus the call's own final wait
    return m, dict(wall_ms=wall, gpu_ms=None, launches=8 * calls, host_waits=3 * calls)


def route_oracle(clouds, ids, poses, leaf, final_leaf):
    from oracle import pyoracle as orc
    t0 = time.perf_counter()
    parts = [orc.transform_f(orc.voxel_grid(clouds[i], leaf), T) for i, T in zip(ids, poses)]
    m = np.concatenate(parts) if parts else np.zeros((0, 4), np.float32)
    if final_leaf:
        m = orc.voxel_grid(m, final_leaf)
    return m, dict(wall_ms=(time.perf_counter() - t0) * 1e3, gpu_ms=None, launches=0, host_waits=0, threads=orc.num_threads())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="50,500,2000")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--pool", type=int, default=24)
    ap.add_argument("--cpu-max-k", type=int, default=2000)
    ap.add_argument("--loop-max-k", type=int, default=2000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    from funny_lidar_slam_b200 import synth
    from funny_lidar_slam_b200._lib import lib
    from funny_lidar_slam_b200.keyframes import KeyFrameStore

    if lib().fls_device_count() < 1:
        raise SystemExit("bench_keyframe_map needs a CUDA device (the library has no CPU fallback)")
    ks = [int(k) for k in a.ks.split(",") if k]
    K = max(ks + [21])
    world = synth.make_world()
    traj = synth.trajectory(K, step=1.0)
    pool = [synth.make_scan(world, traj[(i * K) // a.pool], "hdl64", seed=900 + i)["points"] for i in range(a.pool)]
    clouds = [pool[k % a.pool] for k in range(K)]
    store = KeyFrameStore(sum(len(c) for c in clouds))
    t0 = time.perf_counter()
    for c in clouds:
        store.add(c)
    add_ms = (time.perf_counter() - t0) * 1e3
    card = _card()
    lines = [dict(what="setup", card=card, keyframes=K, points=store.n_points, mean_points=store.n_points / K, add_ms_total=add_ms)]
    print(json.dumps(lines[-1]), flush=True)

    shapes = [(f"save_map_K{k}", list(range(k)), 0.3, 0.3) for k in ks] + [("get_submap_K21", list(range(K // 2 - 10, K // 2 + 11)), 0.2, None)]
    for name, ids, leaf, final_leaf in shapes:
        P = np.asarray(traj)[ids]
        route_store(store, ids, P, leaf, final_leaf)  # warm-up: allocations, CUB's tuning, module load
        runs = [route_store(store, ids, P, leaf, final_leaf) for _ in range(a.reps)]
        out = runs[-1][0]
        rec = dict(what=name, route="store", n_in=int(sum(len(clouds[i]) for i in ids)), n_out=len(out), card=card,
                   wall_ms=sorted(r[1]["wall_ms"] for r in runs), gpu_ms=sorted(r[1]["gpu_ms"] for r in runs),
                   launches=runs[-1][1]["launches"], host_waits=runs[-1][1]["host_waits"],
                   identical_across_reps=all(_same(r[0], out) for r in runs))
        print(json.dumps(rec), flush=True)
        lines.append(rec)
        if len(ids) <= a.loop_max_k:
            route_loop(clouds, ids[:2], P[:2], leaf, final_leaf)
            lr = [route_loop(clouds, ids, P, leaf, final_leaf) for _ in range(max(1, a.reps if len(ids) <= 500 else 1))]
            rec = dict(what=name, route="loop", n_out=len(lr[-1][0]), wall_ms=sorted(r[1]["wall_ms"] for r in lr), launches=lr[-1][1]["launches"],
                       host_waits=lr[-1][1]["host_waits"], bit_exact_vs_store=_same(lr[-1][0], out), card=card)
            print(json.dumps(rec), flush=True)
            lines.append(rec)
        if len(ids) <= a.cpu_max_k:
            o, info = route_oracle(clouds, ids, P, leaf, final_leaf)
            rec = dict(what=name, route="oracle", n_out=len(o), wall_ms=[info["wall_ms"]], threads=info["threads"],
                       bit_exact_vs_store=_same(o, out))
            print(json.dumps(rec), flush=True)
            lines.append(rec)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            for r in lines:
                fh.write(json.dumps(r) + "\n")
    store.close()


if __name__ == "__main__":
    main()
