"""Scan Context place recognition on the keyframe store (fls_keyframes_detect_loop / _place_query) at K = 1 000, 10 000 and 50 000
keyframes, against the numpy restatement of the same definitions (tests/scan_context_ref.py) at K = 1 000.

Keyframes are ray-cast 64-line scans (synth.make_scan) thinned to every --thin-th point so that 50 000 of them fit the arena; a pool of
--pool distinct scans is reused cyclically, as tools/bench_keyframe_map.py does, and added from device memory.  Per K:
  describe_all  the first detect_loop after a cfg change: every keyframe described, then one search
  detect_loop   the same call again: the search alone (query = the last keyframe, min_span 30)
  place_query   a host scan as the query: the scan described, then one search over every keyframe
Device time is the store's CUDA-event time (stats.gpu_ms), wall time a host clock around the call (each call ends in a synchronise);
both are medians over --reps calls, with launches and host waits.  Prints one JSON line per measurement and the card's name and power
limit; --out writes them to a file.

    python tools/bench_place_recognition.py [--ks 1000,10000,50000] [--reps 5] [--pool 16] [--thin 4] [--out FILE.jsonl]
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


def _timed(store, call, reps):
    walls, gpus, res = [], [], None
    for _ in range(reps):
        t0 = time.perf_counter()
        res = call()
        walls.append((time.perf_counter() - t0) * 1e3)
        gpus.append(store.last_stats.gpu_ms)
    st = store.last_stats
    return res, dict(wall_ms_median=float(np.median(walls)), gpu_ms_median=float(np.median(gpus)), wall_ms=sorted(walls), gpu_ms=sorted(gpus),
                     launches=st.gpu_launches, host_waits=st.iterations)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1000,10000,50000")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--pool", type=int, default=16)
    ap.add_argument("--thin", type=int, default=4)
    ap.add_argument("--ref-k", type=int, default=1000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import torch

    from funny_lidar_slam_b200 import synth
    from funny_lidar_slam_b200._lib import lib
    from funny_lidar_slam_b200.keyframes import KeyFrameStore, sc_cfg
    from tests import scan_context_ref as ref

    if lib().fls_device_count() < 1:
        raise SystemExit("bench_place_recognition needs a CUDA device (the library has no CPU fallback)")
    ks = sorted(int(k) for k in a.ks.split(",") if k)
    K = ks[-1]
    world = synth.make_world()
    traj = synth.trajectory(a.pool + 1, step=7.0)
    pool = [np.ascontiguousarray(synth.make_scan(world, traj[i], "hdl64", seed=900 + i)["points"][::a.thin]) for i in range(a.pool)]
    d_pool = [torch.from_numpy(c).cuda() for c in pool]
    torch.cuda.synchronize()
    query = synth.make_scan(world, traj[a.pool], "hdl64", seed=999)["points"]
    store = KeyFrameStore(sum(len(pool[k % a.pool]) for k in range(K)))
    card = _card()
    cfg_a, cfg_b = sc_cfg(), sc_cfg(z_offset=2.5)
    lines = [dict(what="setup", card=card, pool=a.pool, points_per_keyframe=float(np.mean([len(c) for c in pool])), query_points=len(query))]
    print(json.dumps(lines[-1]), flush=True)

    def emit(rec):
        rec["card"] = card
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    for k in ks:
        while len(store) < k:
            i = len(store) % a.pool
            store.add_device(d_pool[i].data_ptr(), len(pool[i]))
        store.detect_loop(k - 1, 30, 5, cfg_a)  # warm-up: allocations, CUB's tuning, module load
        walls, gpus = [], []
        for r in range(a.reps):  # describe every keyframe: alternate two cfgs, so each call re-describes all
            c = cfg_b if r % 2 == 0 else cfg_a
            t0 = time.perf_counter()
            store.detect_loop(k - 1, 30, 5, c)
            walls.append((time.perf_counter() - t0) * 1e3)
            gpus.append(store.last_stats.gpu_ms)
        st = store.last_stats
        emit(dict(what="describe_all_plus_search", keyframes=k, points=store.n_points, wall_ms_median=float(np.median(walls)),
                  gpu_ms_median=float(np.median(gpus)), launches=st.gpu_launches, host_waits=st.iterations, n_source=st.n_source))
        res, info = _timed(store, lambda: store.detect_loop(k - 1, 30, 5, c), a.reps)
        emit(dict(what="detect_loop", keyframes=k, candidates=store.last_stats.n_valid, best=[(m.id, m.distance) for m in res[:3]], **info))
        res, info = _timed(store, lambda: store.place_query(query, 5, c), a.reps)
        emit(dict(what="place_query", keyframes=k, best=[(m.id, m.distance) for m in res[:3]], **info))
        if k == a.ref_k:
            desc = store.scan_context(range(k), c)
            t0 = time.perf_counter()
            q = ref.descriptor(query, c.n_rings, c.n_sectors, c.max_radius, c.z_offset)
            D, s, _ = ref.distances(q, desc)
            order = ref.rank(D)
            wall = (time.perf_counter() - t0) * 1e3
            got = store.place_query(query, 5, c)
            emit(dict(what="numpy_reference_place_query", keyframes=k, wall_ms=wall, same_top5=[m.id for m in got] == order[:5].tolist(),
                      max_abs_distance_diff_top5=float(max(abs(m.distance - D[m.id]) for m in got))))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            for r in lines:
                fh.write(json.dumps(r) + "\n")
    store.close()


if __name__ == "__main__":
    main()
