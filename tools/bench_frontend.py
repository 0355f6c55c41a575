"""Per-scan cost of the LoamFull front end: fls_preprocess_loam against the chain of per-stage calls it replaces.

For HDL-64-shaped (64 x 1800) and VLP-16-shaped (16 x 1800) raw scans with IMU de-skew, per scan:
  a  fls_preprocess_loam, host outputs
  b  fls_preprocess_loam into device buffers + fls_match_cluster_device against a LoamFull map
  c  fls_project_imu -> fls_extract_features -> host gather -> fls_voxel_grid x 2, then host fls_match
  d  the CPU oracle's front-end chain (projection, features, two voxel filters; no Match)
Wall times are host clocks around calls that end in a device synchronise (each entry returns with its work complete), after a
warm-up.  Bytes per scan: (a) and (b) from the calls' stats; (c) from its features and Match stats plus the copies of the projector
and voxel-filter entries counted from their shapes (those entries report no stats).  The outputs of (a) and (c) are compared on
every timed scan.  Prints the GPU name and power limit, then one JSON line.  Needs a GPU: there is no fallback.

    python tools/bench_frontend.py --scans 200 --warmup 20
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


def raw_scans(world, traj, sensor):
    from funny_lidar_slam_b200 import synth
    out = []
    for k in range(POOL):
        sc = synth.make_scan(world, traj[k], sensor, seed=500 + k)
        order = np.lexsort((sc["ring"], sc["col"]))
        col = sc["col"][order]
        out.append((sc["points"][order], sc["ring"][order].astype(np.int32), (col / synth.SENSORS[sensor].cols * 0.1).astype(np.float32)))
    return out


def imu_buffer():
    ref = 1_700_000_000_000_000
    t = (ref - 20_000 + np.arange(0, 125_000, 5000)).astype(np.uint64)  # 200 Hz, covers the whole 0.1 s sweep
    ang = 0.05 * np.sin(np.linspace(0, 2.0, len(t)))
    q = np.stack([np.zeros_like(ang), np.zeros_like(ang), np.sin(ang / 2), np.cos(ang / 2)], 1)
    return dict(t_us=t, q_xyzw=q, ref_time_us=ref, T_lidar_to_imu=np.eye(4))


def oracle_chain(raw, ring, tm, imu, V, H, h_res):
    from oracle import pyoracle as orc
    pr = orc.project_imu(raw, ring, tm, imu, V, H, h_res, MIN_D, MAX_D)
    ci, pi, _ = orc.extract_features(pr["depth"], pr["col"], pr["n"], pr["row_start"], pr["row_end"], CORNER_THR, PLANAR_THR)
    return orc.voxel_grid(pr["ordered"][ci], CORNER_LEAF), orc.voxel_grid(pr["ordered"][pi], PLANAR_LEAF)


def to_world(pts, T):
    out = pts.copy()
    out[:, :3] = (pts[:, :3].astype(np.float64) @ T[:3, :3].T + T[:3, 3]).astype(np.float32)
    return out


def run_sensor(sensor, world, traj, imu, args, log):
    from funny_lidar_slam_b200 import FLS_LOAM_FULL, default_config, synth
    from funny_lidar_slam_b200.features import FeatureExtractor, LoamFrontEnd, PointcloudProjector, project_imu
    from funny_lidar_slam_b200.registration import PointcloudCluster, Registration, voxel_grid
    sn = synth.SENSORS[sensor]
    V, H, h_res = sn.lines, sn.cols, float(np.float32(2 * np.pi / sn.cols))
    scans = raw_scans(world, traj, sensor)
    guesses = [synth.perturb_pose(traj[k], dpos=0.05, drot_deg=0.5, seed=k) for k in range(POOL)]
    # (d) first: the CPU part runs before any device call
    n_cpu = min(args.cpu_scans, args.scans)
    t0 = time.perf_counter()
    for i in range(n_cpu):
        oracle_chain(*scans[i % POOL], imu, V, H, h_res)
    cpu_ms = (time.perf_counter() - t0) * 1e3 / n_cpu
    map_clouds = [oracle_chain(*scans[k], imu, V, H, h_res) for k in (0, 3, 6, 9)]

    import torch
    fe = LoamFrontEnd(H, V, h_res, MIN_D, MAX_D, CORNER_THR, PLANAR_THR, CORNER_LEAF, PLANAR_LEAF, device=args.device)
    proj = PointcloudProjector(H, V, h_res, MIN_D, MAX_D, device=args.device)
    fx = FeatureExtractor(CORNER_THR, PLANAR_THR, device=args.device)
    cfg = default_config(FLS_LOAM_FULL, device=args.device, localization_mode=0, local_map_size=6, corner_local_map_size=4)
    reg_b, reg_c = Registration(cfg), Registration(cfg)
    for (c, p), k in zip(map_clouds, (0, 3, 6, 9)):
        for reg in (reg_b, reg_c):
            reg.AddCloudToLocalMap([to_world(p, traj[k]), to_world(c, traj[k])])
    dev = f"cuda:{args.device}"
    d_c = torch.empty((120 * V, 4), dtype=torch.float32, device=dev)
    d_p = torch.empty((V * H, 4), dtype=torch.float32, device=dev)
    torch.cuda.synchronize(dev)

    bytes_c = [0, 0]  # (c): h2d, d2h over the timed scans

    def leg_a(i):
        return fe.run(*scans[i % POOL], imu)

    def leg_b(i):
        fe.run(*scans[i % POOL], imu, device_out=(d_c.data_ptr(), d_p.data_ptr()), host_out=False)
        nc, npl = fe.last_counts
        T = guesses[i % POOL].copy()
        reg_b.match_cluster_device(0, 0, d_p.data_ptr(), npl, d_c.data_ptr(), nc, T)
        return T

    def leg_c(i):
        raw, ring, tm = scans[i % POOL]
        pr = project_imu(proj, raw, ring, tm, imu)
        ci, pi = fx.extract_indices(pr["depth"], pr["col"], pr["n"], pr["row_start"], pr["row_end"])
        c = voxel_grid(pr["ordered"][ci], CORNER_LEAF, device=args.device)
        p = voxel_grid(pr["ordered"][pi], PLANAR_LEAF, device=args.device)
        T = guesses[i % POOL].copy()
        reg_c.Match(PointcloudCluster(planar_cloud=p, corner_cloud=c), T)
        bytes_c[0] += len(raw) * (16 + 4 + 4) + (len(imu["t_us"]) * 40) + len(ci) * 16 + len(pi) * 16 + fx.last_stats.h2d_bytes
        bytes_c[1] += V * H * 8 + (2 * V + 1) * 4 + pr["n"] * 16 + (len(c) + len(p)) * 16 + fx.last_stats.d2h_bytes
        bytes_c[0] += reg_c.last_stats.h2d_bytes
        bytes_c[1] += reg_c.last_stats.d2h_bytes
        return c, p, T

    for i in range(args.warmup):
        leg_a(i)
        leg_b(i)
        leg_c(i)
    bytes_c[:] = [0, 0]
    out_a, out_c, poses_b, poses_c = [], [], [], []
    ta = tb = tc = 0.0
    ba, bb = [0, 0], [0, 0]
    for i in range(args.scans):
        t0 = time.perf_counter()
        out_a.append(leg_a(i))
        ta += time.perf_counter() - t0
        ba[0] += fe.last_stats.h2d_bytes
        ba[1] += fe.last_stats.d2h_bytes
        t0 = time.perf_counter()
        poses_b.append(leg_b(i))
        tb += time.perf_counter() - t0
        bb[0] += fe.last_stats.h2d_bytes + reg_b.last_stats.h2d_bytes
        bb[1] += fe.last_stats.d2h_bytes + reg_b.last_stats.d2h_bytes
        t0 = time.perf_counter()
        c, p, T = leg_c(i)
        tc += time.perf_counter() - t0
        out_c.append((c, p))
        poses_c.append(T)
    same = all(np.array_equal(a[0], c[0]) and np.array_equal(a[1], c[1]) for a, c in zip(out_a, out_c))
    same_pose = all(np.array_equal(a, b) for a, b in zip(poses_b, poses_c))
    S = args.scans
    res = {"raw_points_per_scan": int(np.mean([len(s[0]) for s in scans])), "rows": V, "cols": H,
           "corner_per_scan": float(np.mean([len(a[0]) for a in out_a])), "planar_per_scan": float(np.mean([len(a[1]) for a in out_a])),
           "a_fused_host_ms": ta * 1e3 / S, "b_fused_device_plus_match_ms": tb * 1e3 / S, "c_five_calls_plus_match_ms": tc * 1e3 / S,
           "d_cpu_oracle_frontend_ms": cpu_ms, "d_cpu_scans": n_cpu,
           "a_h2d_bytes": ba[0] // S, "a_d2h_bytes": ba[1] // S, "b_h2d_bytes": bb[0] // S, "b_d2h_bytes": bb[1] // S,
           "c_h2d_bytes": bytes_c[0] // S, "c_d2h_bytes": bytes_c[1] // S,
           "a_equals_c_bitwise": bool(same), "b_poses_equal_c": bool(same_pose)}
    log(f"{sensor}: {res}")
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--scans", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--cpu-scans", type=int, default=24, help="scans timed on the CPU oracle (d)")
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()
    log = lambda m: print(m, file=sys.stderr, flush=True)
    from funny_lidar_slam_b200 import synth
    world = synth.make_world()
    traj = synth.trajectory(POOL)
    imu = imu_buffer()
    out = {"scans": args.scans, "warmup": args.warmup}
    for sensor in ("hdl64", "vlp16"):
        out[sensor] = run_sensor(sensor, world, traj, imu, args, log)
    gpu = subprocess.run(["nvidia-smi", "-i", str(args.device), "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    out["gpu"] = gpu
    print(f"gpu: {gpu}")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
