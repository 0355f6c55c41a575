"""Per-scan cost of taking a LiDAR PointCloud2 message to a LoamFull pose, with the conversion on the device or on the CPU.

For HDL-64-shaped (64 x 1800) and VLP-16-shaped (16 x 1800) Velodyne messages in a Velodyne's firing order (the yaw falls from point
to point), with a `time` field and without one (the latter runs ComputePointOffsetTime), per scan:
  a  message -> fls_convert_cloud (device outputs) -> fls_preprocess_loam_device (device outputs) -> fls_match_cluster_device
  b  the CPU oracle's ConvertMessageToCloud -> fls_preprocess_loam (host input and outputs) -> host fls_match
Wall times are host clocks around calls that end in a device synchronise (every entry returns with its work complete), after a
warm-up.  Bytes per scan come from the calls' stats.  The poses of (a) and (b) are compared on every timed scan.  Prints the GPU name
and power limit, then one JSON line.  Needs a GPU: there is no fallback.

    python tools/bench_convert.py --scans 200 --warmup 20
    python tools/bench_convert.py --profile   # per-kernel device time of fls_convert_cloud (torch.profiler), a run of its own
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

CORNER_THR, PLANAR_THR, CORNER_LEAF, PLANAR_LEAF = 1.0, 0.1, 0.2, 0.4  # config_nclt_loam_full.yaml
MIN_D, MAX_D = 2.0, 80.0
POOL = 12  # distinct scans per sensor, cycled through
# velodyne_pointcloud's PointXYZIRT (x, y, z, pad, intensity, ring, time) and the same record without `time`
LAYOUT_T = (["x", "y", "z", "intensity", "ring", "time"], ["<f4", "<f4", "<f4", "<f4", "<u2", "<f4"], [0, 4, 8, 16, 20, 24], 32)
LAYOUT_NT = (["x", "y", "z", "intensity", "ring"], ["<f4", "<f4", "<f4", "<f4", "<u2"], [0, 4, 8, 16, 20], 24)


def messages(world, traj, sensor, with_time):
    from funny_lidar_slam_b200 import synth
    from funny_lidar_slam_b200.features import PointCloud2
    names, formats, offsets, itemsize = LAYOUT_T if with_time else LAYOUT_NT
    dt = np.dtype({"names": names, "formats": formats, "offsets": offsets, "itemsize": itemsize})
    out = []
    for k in range(POOL):
        sc = synth.make_scan(world, traj[k], sensor, seed=700 + k)
        # firing order with a Velodyne's sense of rotation: the yaw falls from point to point, so ComputePointOffsetTime carries
        # time_last through the ring (the synthetic scanner's columns run the other way)
        order = np.lexsort((sc["ring"], -sc["col"]))
        pts, ring, col = sc["points"][order], sc["ring"][order], sc["col"][order]
        col = sc["col"].max() - col
        rec = np.zeros(len(pts), dt)
        for j, f in enumerate(("x", "y", "z", "intensity")):
            rec[f] = pts[:, j]
        rec["ring"] = ring
        if with_time:
            rec["time"] = (col / synth.SENSORS[sensor].cols * 0.1).astype(np.float32)
        out.append(PointCloud2.from_records(rec, stamp_us=1_700_000_000_000_000 + 100_000 * k))
    return out


def to_world(pts, T):
    out = pts.copy()
    out[:, :3] = (pts[:, :3].astype(np.float64) @ T[:3, :3].T + T[:3, 3]).astype(np.float32)
    return out


def run_case(sensor, with_time, world, traj, args, log):
    import torch

    from funny_lidar_slam_b200 import FLS_LOAM_FULL, default_config, synth
    from funny_lidar_slam_b200._abi import FLS_LIDAR_VELODYNE
    from funny_lidar_slam_b200.features import LoamFrontEnd, convert_message
    from funny_lidar_slam_b200.registration import PointcloudCluster, Registration
    from oracle_convert import pyoracle_convert as orcc
    sn = synth.SENSORS[sensor]
    V, H, h_res = sn.lines, sn.cols, float(np.float32(2 * np.pi / sn.cols))
    msgs = messages(world, traj, sensor, with_time)
    conv_kw = dict(lidar_type=FLS_LIDAR_VELODYNE, n_rows=V, time_scale=1.0)
    guesses = [synth.perturb_pose(traj[k], dpos=0.05, drot_deg=0.5, seed=k) for k in range(POOL)]
    fe = LoamFrontEnd(H, V, h_res, MIN_D, MAX_D, CORNER_THR, PLANAR_THR, CORNER_LEAF, PLANAR_LEAF, device=args.device)
    cfg = default_config(FLS_LOAM_FULL, device=args.device, localization_mode=0, local_map_size=6, corner_local_map_size=4)
    reg_a, reg_b = Registration(cfg), Registration(cfg)
    for k in (0, 3, 6, 9):
        cv = orcc.convert_message(msgs[k], **conv_kw)
        c, p = fe.run(cv["xyzi"], cv["ring"], cv["time"])
        for reg in (reg_a, reg_b):
            reg.AddCloudToLocalMap([to_world(p, traj[k]), to_world(c, traj[k])])
    dev = f"cuda:{args.device}"
    cap = max(m.width * m.height for m in msgs)
    dx = torch.empty((cap, 4), dtype=torch.float32, device=dev)
    dr = torch.empty(cap, dtype=torch.int32, device=dev)
    dtm = torch.empty(cap, dtype=torch.float32, device=dev)
    d_c = torch.empty((120 * V, 4), dtype=torch.float32, device=dev)
    d_p = torch.empty((V * H, 4), dtype=torch.float32, device=dev)
    torch.cuda.synchronize(dev)
    bytes_a, bytes_b = [0, 0], [0, 0]

    def leg_a(i):
        r = convert_message(msgs[i % POOL], device=args.device, device_out=(dx.data_ptr(), dr.data_ptr(), dtm.data_ptr()), host_out=False, **conv_kw)
        fe.run_device(dx.data_ptr(), dr.data_ptr(), dtm.data_ptr(), r["n"], device_out=(d_c.data_ptr(), d_p.data_ptr()), host_out=False)
        nc, npl = fe.last_counts
        T = guesses[i % POOL].copy()
        reg_a.match_cluster_device(0, 0, d_p.data_ptr(), npl, d_c.data_ptr(), nc, T)
        for s in (r["stats"], fe.last_stats, reg_a.last_stats):
            bytes_a[0] += s.h2d_bytes
            bytes_a[1] += s.d2h_bytes
        return T, r["recomputed"]

    def leg_b(i):
        cv = orcc.convert_message(msgs[i % POOL], **conv_kw)
        c, p = fe.run(cv["xyzi"], cv["ring"], cv["time"])
        st = fe.last_stats
        T = guesses[i % POOL].copy()
        reg_b.Match(PointcloudCluster(planar_cloud=p, corner_cloud=c), T)
        for s in (st, reg_b.last_stats):
            bytes_b[0] += s.h2d_bytes
            bytes_b[1] += s.d2h_bytes
        return T

    for i in range(args.warmup):
        leg_a(i)
        leg_b(i)
    bytes_a[:], bytes_b[:] = [0, 0], [0, 0]
    ta = tb = 0.0
    pa, pb, rec = [], [], []
    for i in range(args.scans):
        t0 = time.perf_counter()
        T, r = leg_a(i)
        ta += time.perf_counter() - t0
        pa.append(T)
        rec.append(r)
        t0 = time.perf_counter()
        pb.append(leg_b(i))
        tb += time.perf_counter() - t0
    S = args.scans
    res = {"points_per_scan": int(np.mean([m.width * m.height for m in msgs])), "message_bytes": int(np.mean([m.row_step * m.height for m in msgs])),
           "offsets_recomputed": bool(all(rec)), "a_device_convert_frontend_match_ms": ta * 1e3 / S, "b_cpu_convert_host_frontend_match_ms": tb * 1e3 / S,
           "a_h2d_bytes": bytes_a[0] // S, "a_d2h_bytes": bytes_a[1] // S, "b_h2d_bytes": bytes_b[0] // S, "b_d2h_bytes": bytes_b[1] // S,
           "poses_a_equal_b": bool(all(np.array_equal(a, b) for a, b in zip(pa, pb)))}
    log(f"{sensor} time={with_time}: {res}")
    return res


def profile_kernels(args, log):
    """Mean device time per call of every kernel fls_convert_cloud launches, from torch.profiler over --scans conversions per case."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    from funny_lidar_slam_b200 import synth
    from funny_lidar_slam_b200._abi import FLS_LIDAR_VELODYNE
    from funny_lidar_slam_b200.features import convert_message
    world, traj = synth.make_world(), synth.trajectory(POOL)
    out = {}
    for sensor in ("hdl64", "vlp16"):
        for with_time in (True, False):
            msgs = messages(world, traj, sensor, with_time)
            kw = dict(lidar_type=FLS_LIDAR_VELODYNE, n_rows=synth.SENSORS[sensor].lines, time_scale=1.0, device=args.device)
            cap = max(m.width * m.height for m in msgs)
            bufs = [torch.empty((cap, 4), device=f"cuda:{args.device}"), torch.empty(cap, dtype=torch.int32, device=f"cuda:{args.device}"),
                    torch.empty(cap, device=f"cuda:{args.device}")]
            d_out = tuple(b.data_ptr() for b in bufs)
            for i in range(args.warmup):
                convert_message(msgs[i % POOL], device_out=d_out, host_out=False, **kw)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for i in range(args.scans):
                    convert_message(msgs[i % POOL], device_out=d_out, host_out=False, **kw)
            ker = {}
            for e in prof.key_averages():
                if str(getattr(e, "device_type", "")).endswith("CUDA") and "emcpy" not in e.key and "emset" not in e.key:
                    k = e.key[:100]  # template instantiations that share a long prefix are summed
                    ker[k] = round(ker.get(k, 0.0) + e.device_time_total / args.scans, 2)
            out[f"{sensor}_{'time' if with_time else 'no_time'}_us_per_call"] = ker
            log(f"{sensor} time={with_time}: {ker}")
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--scans", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--profile", action="store_true", help="per-kernel device times of the conversion instead of the wall-time comparison")
    args = ap.parse_args()
    log = lambda m: print(m, file=sys.stderr, flush=True)
    if args.profile:
        out = profile_kernels(args, log)
        gpu = subprocess.run(["nvidia-smi", "-i", str(args.device), "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True).stdout.strip()
        out["gpu"] = gpu
        print(f"gpu: {gpu}")
        print(json.dumps(out))
        return
    from funny_lidar_slam_b200 import synth
    world = synth.make_world()
    traj = synth.trajectory(POOL)
    out = {"scans": args.scans, "warmup": args.warmup}
    for sensor in ("hdl64", "vlp16"):
        for with_time in (True, False):
            out[f"{sensor}_{'time' if with_time else 'no_time'}"] = run_case(sensor, with_time, world, traj, args, log)
    gpu = subprocess.run(["nvidia-smi", "-i", str(args.device), "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    out["gpu"] = gpu
    print(f"gpu: {gpu}")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
