#!/usr/bin/env python
"""bench.py — scans/sec of the H100 scan-matching hot path, with the live roofline of its residual kernel, a parity block
against the CPU oracle on the very scans that were timed, and the CPU oracle timed beside it.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--workload NAME] [--impl ours|reference] [--batch B] [--dump-outputs DIR]

One "step" = one batched Match of B synthetic scans per GPU against a static (replicated) map (SURVEY.md §8d/§8e).
For N > 1 launch under torchrun (one rank per GPU): every rank matches its own B scans per step; the per-scan results
{pose, converged, iterations} are written by the GN kernel into a device buffer and all-gathered over NCCL asynchronously —
the gathered batch is consumed two steps later (funny_lidar_slam_b200/parallel.py), so no rank waits for another inside a step.
Rank 0 prints ONE JSON line.

Timed legs (all inside this process, nothing under a profiler):
  value     device-resident scans (float4 in HBM) -> fls_match_batch_device; per-step CUDA events, L2 flushed between steps
  e2e       pinned HOST scans -> fls_match_batch (H2D copy + Match + D2H of the state blocks inside the timed region)
  roofline  same steps on a handle created with FLS_FLAG_PROFILE: CUDA events around every residual-kernel launch
  cpu_baseline / --impl reference: the CPU oracle (port of the reference algorithm, OpenMP; thread count chosen by a sweep)
  parity    GPU results of the scan pool vs the oracle's results for the same scans and guesses (N = 1, rank 0)

--dump-outputs DIR writes what the `value` leg returned in its last timed step (rank 0): the B poses, converged flags,
iterations and n_valid, and the indices of the scans in the seeded pool, as DIR/<name>.npy (float64).  The scene, the scans
and the guesses are generated from fixed seeds, so two builds run with the same arguments can be compared output for output.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from funny_lidar_slam_b200 import _abi, synth  # noqa: E402
from funny_lidar_slam_b200._mem import tune_malloc  # noqa: E402

tune_malloc()

_BIG = dict(world_half=350.0, n_boxes=500, n_cyls=400, map_spacing=0.3)
_SMALL = dict(world_half=100.0, n_boxes=40, n_cyls=30, map_spacing=0.3)
WORKLOADS = {
    # BASELINE.json configs[3] shape on one GPU: LoamPointToPlaneIVOX semantics, 64-line ~100k-pt scans, multi-million-point iVox map
    "p2plane_ivox_64": dict(method=_abi.FLS_P2PLANE_IVOX, sensor="hdl64", dpos=0.3, drot=3.0, cfg={}, **_BIG,
                            desc="LoamPointToPlaneIVOX (point-to-plane GN on iVox 5-NN), 64-line ~100k-pt scans vs static ~5M-pt iVox map"),
    # reduced variant for quick checks on small boxes
    "p2plane_ivox_64_small": dict(method=_abi.FLS_P2PLANE_IVOX, sensor="hdl64", dpos=0.3, drot=3.0, cfg={}, **_SMALL,
                                  desc="LoamPointToPlaneIVOX, 64-line scans vs ~0.5M-pt iVox map (reduced)"),
    # BASELINE.json configs[4]: dense 128-line scan, IncrementalNDT, exactly 10 GN iterations (thresholds 0), no down-sampling
    # (a 1 cm leaf makes pcl::VoxelGrid return its input: dx*dy*dz > INT_MAX), static NDT map (localization semantics)
    "ndt_128_10it": dict(method=_abi.FLS_NDT, sensor="os128", dpos=0.05, drot=0.5, **_SMALL,
                         cfg=dict(ndt_capacity=2000000, source_cloud_filter_size=0.01, max_iterations=10, position_converge_thres=0.0,
                                  rotation_converge_thres=0.0),
                         desc="IncrementalNDT::Match, dense 128-line scans (~140k pts, unfiltered), exactly 10 GN iterations, static NDT map"),
    # BASELINE.json configs[1] shape as a static-map batch: 64-line scans, shipped NDT parameters (leaf 0.2, <= 30 iterations)
    "ndt_64": dict(method=_abi.FLS_NDT, sensor="hdl64", dpos=0.05, drot=0.5, cfg=dict(ndt_capacity=2000000), **_SMALL,
                   desc="IncrementalNDT::Match, 64-line ~100k-pt scans (VoxelGrid 0.2 inside Match), static NDT map"),
}
DEFAULT_WORKLOAD = "p2plane_ivox_64"
POS_TOL, ROT_TOL = 1e-4, 1e-4  # BASELINE.json north_star: final SE(3) within 1e-4 m / 1e-4 rad of the reference CPU path


def load_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        try:
            return float(json.load(open(p))["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
        except Exception:
            pass
    return 3350.0, "fallback (H100 SXM data sheet: 3.35 TB/s HBM3, not a measurement)"


# ---- host CPU: how many cores may this process really use ---------------------------------------------------------------
def effective_cores():
    """min(affinity mask, cgroup CPU quota).  A 1-GPU lease of a big host often carries a quota far below the affinity
    mask; forcing one OpenMP thread per visible CPU then oversubscribes the quota (round 1: 2.6 vs 21 scans/s)."""
    aff = len(os.sched_getaffinity(0))
    quota = None
    try:
        q, per = open("/sys/fs/cgroup/cpu.max").read().split()[:2]  # cgroup v2
        if q != "max":
            quota = float(q) / float(per)
    except Exception:
        pass
    if quota is None:
        try:  # cgroup v1
            q = int(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())
            per = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            if q > 0 and per > 0:
                quota = q / per
        except Exception:
            pass
    phys = None
    try:
        ids = set()
        pid = cid = None
        for ln in open("/proc/cpuinfo"):
            if ln.startswith("physical id"):
                pid = ln.split(":")[1].strip()
            elif ln.startswith("core id"):
                cid = ln.split(":")[1].strip()
            elif not ln.strip():
                if pid is not None and cid is not None:
                    ids.add((pid, cid))
                pid = cid = None
        phys = len(ids) or None
    except Exception:
        pass
    eff = aff if quota is None else max(1, min(aff, int(math.ceil(quota))))
    return {"affinity": aff, "cgroup_quota": quota, "physical_cores_visible": phys, "effective": eff}


def tune_oracle_threads(orc, reg, scans, guesses, log, budget_s=25.0):
    """Sweep OpenMP thread counts {1, eff/2, eff, 2*eff, physical} on a few Match calls and keep the fastest.
    Returns (best_threads, {threads: scans/s}, cores_info)."""
    cores = effective_cores()
    eff = cores["effective"]
    cand = {1, max(1, eff // 2), eff, min(2 * eff, max(cores["affinity"], eff))}
    if cores["physical_cores_visible"]:
        cand.add(max(1, min(cores["physical_cores_visible"], cores["affinity"])))
    sweep = {}
    t_start = time.time()
    for th in sorted(cand, reverse=True):  # 1 thread last: it is the slowest probe
        orc.set_num_threads(th)
        reps = 1 if th == 1 else 3
        if th > 1:
            reg.match(scans[0], guesses[0])  # warm the thread pool at this size
        t = 0.0
        done = 0
        for i in range(reps):
            reg.match(scans[(i + 1) % len(scans)], guesses[(i + 1) % len(scans)])
            t += reg.last_seconds
            done += 1
            if time.time() - t_start > budget_s and done >= 1:
                break
        sweep[th] = done / max(t, 1e-9)
        log(f"oracle threads {th}: {sweep[th]:.2f} scans/s")
    best = max(sweep, key=sweep.get)
    orc.set_num_threads(best)
    return best, sweep, cores


class ClockSampler:
    """SM clock / throttle reasons sampled DURING the timed regions, in-process through NVML (a Python thread, 10 ms period).
    Round 1 spawned `nvidia-smi -lms` per rank right before the 20 ms timed leg: its start-up (it attaches to every GPU of
    the box) both missed the region (0 samples) and stalled the first leg of the 8-rank run."""

    def __init__(self, index: int):
        self.index = index
        self.samples = []  # (sm_mhz, reasons bitmask, power_w)
        self.active = False
        self._stop = False
        self._thread = None
        self.max_mhz = None
        self.err = None
        try:
            import pynvml
            self.nv = pynvml
            pynvml.nvmlInit()
            self.h = pynvml.nvmlDeviceGetHandleByIndex(self._physical_index(index))
            self.max_mhz = float(pynvml.nvmlDeviceGetMaxClockInfo(self.h, pynvml.NVML_CLOCK_SM))
        except Exception as e:  # noqa: BLE001
            self.nv = None
            self.err = repr(e)

    @staticmethod
    def _physical_index(local: int) -> int:
        vis = os.environ.get("CUDA_VISIBLE_DEVICES")
        if vis:
            try:
                return int(vis.split(",")[local])
            except Exception:
                return local
        return local

    def start(self):
        if self.nv is None:
            return
        self._thread = threading.Thread(target=self._run, daemon=True)
        self._thread.start()

    def _run(self):
        nv = self.nv
        while not self._stop:
            if self.active:
                try:
                    mhz = nv.nvmlDeviceGetClockInfo(self.h, nv.NVML_CLOCK_SM)
                    try:
                        rs = nv.nvmlDeviceGetCurrentClocksEventReasons(self.h)
                    except Exception:
                        rs = nv.nvmlDeviceGetCurrentClocksThrottleReasons(self.h)
                    try:
                        pw = nv.nvmlDeviceGetPowerUsage(self.h) / 1000.0
                    except Exception:
                        pw = None
                    self.samples.append((float(mhz), int(rs), pw))
                except Exception as e:  # noqa: BLE001
                    self.err = repr(e)
            time.sleep(0.01)

    def stop(self):
        self._stop = True
        if self.nv is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "samples": 0, "reasons": ["nvml unavailable: " + str(self.err)]}
        if self._thread:
            self._thread.join(timeout=1.0)
        nv = self.nv
        names = {"hw_slowdown": getattr(nv, "nvmlClocksThrottleReasonHwSlowdown", 0x8),
                 "hw_thermal_slowdown": getattr(nv, "nvmlClocksThrottleReasonHwThermalSlowdown", 0x40),
                 "sw_thermal_slowdown": getattr(nv, "nvmlClocksThrottleReasonSwThermalSlowdown", 0x20),
                 "sw_power_cap": getattr(nv, "nvmlClocksThrottleReasonSwPowerCap", 0x4)}
        reasons = sorted(n for n, bit in names.items() if any(s[1] & bit for s in self.samples))
        sm = [s[0] for s in self.samples]
        pw = [s[2] for s in self.samples if s[2] is not None]
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": self.max_mhz, "samples": len(sm), "reasons": reasons,
                "power_w_max": max(pw) if pw else None, "how": "NVML in-process, 10 ms period, only while a timed leg is running"}


def build_scene(wl: dict, n_pool: int, log):
    """Map + a pool of scans shared by every rank (same seeds everywhere): rank r takes scans (step*B + j + r*B) mod pool, so
    over a run whose scans-per-rank is a multiple of the pool every GPU does the same total work (weak scaling by definition)."""
    t0 = time.time()
    world = synth.make_world(seed=1234, half=wl["world_half"], n_boxes=wl["n_boxes"], n_cyls=wl["n_cyls"], keepout=8.0)
    mp = synth.make_surface_map(world, spacing=wl["map_spacing"], seed=4321)
    log(f"map: {len(mp)} points ({time.time() - t0:.1f}s)")
    traj = synth.trajectory(4096, step=1.0, scale=min(120.0, wl["world_half"] * 0.4))
    scans, truths, guesses = [], [], []
    for i in range(n_pool):
        k = i * 7 % len(traj)
        sc = synth.make_scan(world, traj[k], wl["sensor"], seed=100 + i)
        scans.append(sc["points"])
        truths.append(traj[k])
        guesses.append(synth.perturb_pose(traj[k], seed=77 + i, dpos=wl["dpos"], drot_deg=wl["drot"]))
    log(f"scans: {n_pool} x ~{int(np.mean([len(s) for s in scans]))} points ({time.time() - t0:.1f}s)")
    return mp, scans, truths, guesses


def make_cfg(wl: dict, device: int, n_map: int, flags: int = 0):
    extra = dict(wl["cfg"])
    if wl["method"] == _abi.FLS_P2PLANE_IVOX:
        extra.setdefault("ivox_capacity", max(1000000, 2 * n_map))
    return _abi.default_config(wl["method"], device=device, flags=flags, **extra)


def parity_block(gpu_res, orc_res):
    """GPU vs oracle on the same scans and guesses: (ok, T, iterations, n_valid) per scan."""
    from funny_lidar_slam_b200 import synth as sy
    n = min(len(gpu_res), len(orc_res))
    dpos = drot = 0.0
    it_eq = conv_eq = True
    nv_diff = 0
    for g, o in zip(gpu_res[:n], orc_res[:n]):
        dt, dr = sy.pose_error(g[1], o[1])
        dpos, drot = max(dpos, dt), max(drot, dr)
        it_eq = it_eq and (g[2] == o[2])
        conv_eq = conv_eq and (bool(g[0]) == bool(o[0]))
        nv_diff = max(nv_diff, abs(int(g[3]) - int(o[3])))
    ok = bool(n > 0 and dpos < POS_TOL and drot < ROT_TOL and it_eq and conv_eq)
    return {"n_scans": n, "max_dpos_m": dpos, "max_drot_rad": drot, "iters_equal": bool(it_eq), "converged_equal": bool(conv_eq),
            "max_n_valid_diff": int(nv_diff), "tol_m": POS_TOL, "tol_rad": ROT_TOL, "ok": ok,
            "against": "CPU oracle (port of the reference algorithm) on the same scans, guesses and map"}


def secondary_kernels(device: int, peak: float, log, steps: int = 6):
    """Short measurements of the other §8 kernels (K2 NDT, K3 ICP, K4 features, K5 kd-tree LOAM) beside the headline: scans/s
    with the scan resident in HBM, live roofline of the residual kernel (CUDA events per launch), the CPU oracle on the same
    inputs and the pose difference between the two.  Reduced scene (100 m world) so the default run stays within minutes."""
    import torch

    from funny_lidar_slam_b200.features import FeatureExtractor
    from funny_lidar_slam_b200.registration import Registration
    from oracle import pyoracle as orc
    out = {}
    world = synth.make_world()
    traj = synth.trajectory(16)
    mp = synth.make_surface_map(world, spacing=0.3, seed=4321)
    dev = torch.device("cuda", device)
    for name, method, sensor, dpos, drot, extra in (
            ("ndt_64line", _abi.FLS_NDT, "hdl64", 0.05, 0.5, dict(ndt_capacity=2000000)),
            ("ndt_128line_10iters", _abi.FLS_NDT, "os128", 0.05, 0.5, WORKLOADS["ndt_128_10it"]["cfg"]),
            ("icp_16line", _abi.FLS_ICP_P2P, "vlp16", 0.3, 3.0, {}),
            # K5: kd-tree point-to-plane (exact unbounded 5-NN on the grid); the raw 16-line scan stands in for the planar cloud
            ("loam_kdtree_16line", _abi.FLS_P2PLANE_KNN, "vlp16", 0.1, 1.0, {})):
        scans = [synth.make_scan(world, traj[3 + 2 * i], sensor, seed=300 + i)["points"] for i in range(3)]
        guesses = [synth.perturb_pose(traj[3 + 2 * i], seed=900 + i, dpos=dpos, drot_deg=drot) for i in range(3)]
        cfg = _abi.default_config(method, device=device, flags=_abi.FLS_FLAG_PROFILE, **extra)
        reg = Registration(cfg)
        reg.AddCloudToLocalMap([mp])
        d_scans = [torch.from_numpy(s).to(dev) for s in scans]
        g_T = []
        for i in range(3):
            T = guesses[i].copy()
            ok = reg.match_device(d_scans[i].data_ptr(), len(scans[i]), T)
            g_T.append((ok, T, reg.last_stats.iterations, reg.last_stats.n_valid))
        ms = k_ms = 0.0
        k_n = k_b = its = nsrc = 0
        for i in range(steps):
            reg.match_device(d_scans[i % 3].data_ptr(), len(scans[i % 3]), guesses[i % 3].copy())
            st = reg.last_stats
            ms += st.gpu_ms
            k_ms += st.kernel_ms
            k_n += st.kernel_launches
            k_b += st.algo_bytes
            its += st.iterations
            nsrc += st.n_source
        oreg = orc.Registration(_abi.default_config(method, **extra))
        oreg.add_cloud(mp)
        t_cpu = 0.0
        o_T = []
        for i in range(3):
            ok, T, st = oreg.match(scans[i], guesses[i])
            o_T.append((ok, T, st.iterations, st.n_valid))
            t_cpu += oreg.last_seconds
        par = parity_block(g_T, o_T)
        ach = (k_b / max(k_ms, 1e-9)) / 1e6  # bytes/ms -> GB/s
        out[name] = {"scans_per_s_gpu_span": steps / (ms * 1e-3), "mean_gn_iters": its / steps, "points_in_gn_loop": nsrc // steps,
                     "kernel_avg_us": 1e3 * k_ms / max(k_n, 1), "roofline_achieved_gbs": ach, "roofline_frac": ach / peak,
                     "cpu_oracle_scans_per_s": 3 / t_cpu, "cpu_threads": orc.num_threads(), "map_points": int(len(mp)), "l2": "warm",
                     "parity": {k: par[k] for k in ("max_dpos_m", "max_drot_rad", "iters_equal", "converged_equal", "ok")}}
        log(f"secondary {name}: {out[name]}")
    # mapping mode — the reference frontend's default (frontend.cpp:30-88): one scan per call, the map grows with every Match
    # (LOAM-iVox: cached-5-NN insertion rule + incremental iVox insert; NDT: UpdateVoxel), GPU and oracle each on their own stream
    from funny_lidar_slam_b200.registration import PointcloudCluster
    stream_traj = synth.trajectory(64)
    for name, method, sensor, extra in (("p2plane_ivox_64_stream", _abi.FLS_P2PLANE_IVOX, "hdl64", {}),
                                        ("ndt_64_stream", _abi.FLS_NDT, "hdl64", {})):
        n_stream = 12
        cfg = _abi.default_config(method, device=device, localization_mode=0, **extra)
        reg, oreg = Registration(cfg), orc.Registration(_abi.default_config(method, localization_mode=0, **extra))
        first = synth.transform_points(synth.make_scan(world, stream_traj[0], sensor, seed=500)["points"], stream_traj[0])
        reg.AddCloudToLocalMap([first])
        oreg.add_cloud(first)
        g_ms, o_ms, dpos, its = [], [], 0.0, 0
        for k in range(1, n_stream + 1):
            scan = synth.make_scan(world, stream_traj[k], sensor, seed=500 + k)["points"]
            guess = synth.perturb_pose(stream_traj[k], seed=1500 + k, dpos=0.05, drot_deg=0.5)
            T = guess.copy()
            cl = PointcloudCluster(planar_cloud=scan) if method == _abi.FLS_P2PLANE_IVOX else PointcloudCluster(ordered_cloud=scan)
            t0 = time.perf_counter()
            reg.Match(cl, T)
            g_ms.append((time.perf_counter() - t0) * 1e3)
            its += reg.last_stats.iterations
            ok, To, st = oreg.match(scan, guess)
            o_ms.append(oreg.last_seconds * 1e3)
            dpos = max(dpos, synth.pose_error(T, To)[0])
        mi = reg.map_info()
        out[name] = {"scans": n_stream, "ms_per_match_wall_incl_h2d_and_map_update": float(np.mean(g_ms[2:])), "mean_gn_iters": its / n_stream,
                     "cpu_oracle_ms_per_match": float(np.mean(o_ms[2:])), "cpu_threads": orc.num_threads(), "map_points_end": int(mi.n_points),
                     "map_voxels_end": int(mi.n_voxels), "incremental_inserts": int(mi.incremental_inserts), "full_builds": int(mi.full_builds),
                     "max_dpos_vs_oracle_m": float(dpos), "voxels_equal_at_end": bool(mi.n_voxels == oreg.map_voxels)}
        log(f"secondary {name}: {out[name]}")
        del reg, oreg
    fx = FeatureExtractor(1.0, 0.1, device=device)
    shapes = {"features_livox_shaped": dict(kind="livox", seed=13, samples=65000),
              "features_hdl64_shaped": dict(kind="spinning", seed=13, sensor="hdl64")}
    for name, kw in shapes.items():
        proj = synth.make_projected_scan(world, traj[2], **kw)
        n = len(proj["ordered"])
        for _ in range(2):
            gc, gp = fx.extract_indices(proj["depth"], proj["col"], n, proj["row_start"], proj["row_end"])
        g_ms = k_ms = 0.0
        k_b = 0
        for _ in range(steps):
            fx.extract_indices(proj["depth"], proj["col"], n, proj["row_start"], proj["row_end"])
            g_ms += fx.last_stats.gpu_ms
            k_ms += fx.last_stats.kernel_ms
            k_b = fx.last_stats.algo_bytes
        oc, op, sec = orc.extract_features(proj["depth"], proj["col"], n, proj["row_start"], proj["row_end"], 1.0, 0.1)
        ach = k_b / max(k_ms / steps, 1e-9) / 1e6
        out[name] = {"points": n, "rows": int(proj["rows"]), "gpu_ms_incl_h2d_d2h": g_ms / steps, "kernels_ms": k_ms / steps,
                     "cpu_oracle_ms_1thread": sec * 1e3, "roofline_achieved_gbs": ach, "roofline_frac": ach / peak,
                     "index_lists_identical_to_oracle": bool(np.array_equal(gc, oc) and np.array_equal(gp, op))}
        log(f"secondary {name}: {out[name]}")
    return out


def run_reference(args, wl, log):
    """--impl reference: the CPU oracle (the reference cannot be built here: no Eigen/PCL/TBB), thread count chosen by a sweep
    over the host's effective cores, same config/metric; rank 0 only."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    from oracle import pyoracle as orc
    B = max(1, min(int(args.batch), 64))
    n_pool = max(16, 2 * B)
    mp, scans, truths, guesses = build_scene(wl, n_pool, log)
    cfg = make_cfg(wl, 0, len(mp))
    reg = orc.Registration(cfg)
    reg.add_cloud(mp)
    best, sweep, cores = tune_oracle_threads(orc, reg, scans, guesses, log)
    # a step = the same batch of B scans our arm matches per step, one Match call after the other (the reference's API);
    # bounded: at most ~60 s of Match time; `value` is scans actually matched / time actually spent (never extrapolated)
    for i in range(min(args.warmup, 2)):
        reg.match(scans[i % n_pool], guesses[i % n_pool])
    t, done, steps_done = 0.0, 0, 0
    for i in range(args.steps):
        for j in range(B):
            k = (i * B + j) % n_pool
            reg.match(scans[k], guesses[k])
            t += reg.last_seconds
            done += 1
        steps_done += 1
        if t > 60.0:
            break
    val = done / t
    out = {
        "impl": "reference", "metric": "scans/sec", "value": val, "unit": "scans/s", "n_gpus": args.gpus, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": 1e3 * t / steps_done, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f64", "data": "synthetic",
        "config": {"workload": args.workload, "desc": wl["desc"], "map_points": int(len(mp)), "scan_points": int(np.mean([len(s) for s in scans])),
                   "scans_per_gpu_per_step": B, "steps_timed": steps_done},
        "cpu_baseline": {"value": val, "unit": "scans/s", "cores": best, "kind": "port",
                         "threads": best, "effective_cores": cores, "thread_sweep_scans_per_s": {str(k): v for k, v in sorted(sweep.items())},
                         "one_thread_value": sweep.get(1),
                         "sample": f"{done} Match calls ({steps_done} steps of {B}) over {n_pool} distinct scans, oracle (OpenMP, {best} threads = "
                                   "fastest of the sweep) timed with steady_clock inside Match; reference unbuildable here (no Eigen/PCL/TBB)"},
        "e2e": {"value": val, "unit": "scans/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workload", default=DEFAULT_WORKLOAD, choices=sorted(WORKLOADS))
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--cpu-seconds", type=float, default=15.0, help="budget of the cpu_baseline sample")
    ap.add_argument("--verbose", action="store_true")
    ap.add_argument("--no-secondary", action="store_true", help="skip the short K2/K3/K4/K5 side measurements")
    ap.add_argument("--no-cpu", action="store_true", help="skip the cpu_baseline + parity leg (profiling runs)")
    ap.add_argument("--batch", type=int, default=8, help="scans per GPU per step (one fls_match_batch call; BASELINE config 4 uses batches of 8)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the results of the last timed step of the value leg as DIR/<name>.npy (float64)")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    wl = WORKLOADS[args.workload]
    rank = int(os.environ.get("RANK", "0"))
    world_size = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))

    def log(msg):
        if args.verbose or os.environ.get("FLS_BENCH_VERBOSE"):
            print(f"[bench r{rank}] {msg}", file=sys.stderr, flush=True)

    if args.impl == "reference":
        run_reference(args, wl, log)
        return

    import torch
    import torch.distributed as dist

    from funny_lidar_slam_b200 import parallel
    from funny_lidar_slam_b200._lib import lib
    from funny_lidar_slam_b200.registration import Registration

    if not torch.cuda.is_available() or lib().fls_device_count() < 1:
        raise SystemExit("bench.py needs a CUDA device: the product has no CPU fallback")
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    sampler = ClockSampler(local_rank)
    sampler.start()  # NVML attached long before the first timed leg; samples are only taken while `active`
    if world_size > 1:
        dist.init_process_group("nccl", device_id=dev)

    B = max(1, min(int(args.batch), 64))
    n_pool = max(16, 2 * B)
    mp, scans, truths, guesses = build_scene(wl, n_pool, log)
    cfg = make_cfg(wl, local_rank, len(mp))
    batched = wl["method"] in (_abi.FLS_P2PLANE_IVOX, _abi.FLS_NDT)  # plug-ins with a batch entry (fls_match_batch)
    reg = Registration(cfg)
    reg.AddCloudToLocalMap([mp])
    mi = reg.map_info()
    log(f"map on device: {mi.n_points} pts, {mi.n_voxels} voxels, {mi.bytes / 1e6:.0f} MB")

    d_scans = [torch.from_numpy(s).to(dev) for s in scans]
    h_scans = [torch.from_numpy(s).pin_memory() for s in scans]
    flush_buf = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    # the one collective of a step: {4x4 pose, converged, iterations} of this rank's B scans, written by the GN kernel into a
    # device buffer and all-gathered over NCCL asynchronously; consumed two steps later (never inside the step)
    gather = parallel.AsyncResultGather(B, device=dev, depth=3)
    gathered_steps = [0]
    last_value_step = {}  # results of the last timed step of the value leg (--dump-outputs)

    def keep_last(i, oks, Ts, st):
        last_value_step.update(scan_index=np.array(ids(i), np.float64), pose=np.asarray(Ts, np.float64).reshape(-1, 4, 4),
                               converged=np.asarray(oks, np.float64), iterations=np.array([x.iterations for x in st], np.float64),
                               n_valid=np.array([x.n_valid for x in st], np.float64))

    def flush_l2():
        flush_buf.zero_()
        torch.cuda.synchronize()

    def ids(i):
        return [((i + rank) * B + j) % n_pool for j in range(B)]

    def run_batch(r, k, host):
        if batched:
            if host:
                return r.match_batch([h_scans[j].numpy() for j in k], np.stack([guesses[j] for j in k]))
            return r.match_batch_device([d_scans[j].data_ptr() for j in k], [d_scans[j].shape[0] for j in k], np.stack([guesses[j] for j in k]))
        oks, Ts, sts = [], [], []
        for j in k:  # plug-ins without a batch entry: B separate Match calls
            T = guesses[j].copy()
            if host:
                from funny_lidar_slam_b200.registration import PointcloudCluster
                ok = r.Match(PointcloudCluster(ordered_cloud=h_scans[j].numpy(), planar_cloud=h_scans[j].numpy()), T)
            else:
                ok = r.match_device(d_scans[j].data_ptr(), d_scans[j].shape[0], T)
            oks.append(ok)
            Ts.append(T)
            sts.append(r.last_stats)
        r.last_batch_stats = sts
        return np.array(oks, bool), np.stack(Ts)

    def step(i, r, host):
        k = ids(i)
        if batched:
            r.set_result_buffer_device(gather.begin_step().data_ptr(), B)
        else:
            gather.begin_step()
        oks, Ts = run_batch(r, k, host)
        if not batched:  # single-scan entries: stage the results (small) — only the batch entry writes them on the device
            loc = np.stack([parallel.pack_result(T, ok, st.iterations) for T, ok, st in zip(Ts, oks, r.last_batch_stats)])
            gather.local[gather.cur].copy_(torch.from_numpy(loc.reshape(-1)))
        gather.launch()
        if len(gather.pending) > 2 and gather._collect(gather.pending.pop(0)) is not None:
            gathered_steps[0] += 1
        return oks, Ts

    def barrier():
        if world_size > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(host, r, steps, warmup):
        for i in range(warmup):
            step(i, r, host)
        gather.drain()
        barrier()
        tot_ms, launches, iters, h2d, d2h, errs = 0.0, 0, 0, 0, 0, []
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        sampler.active = True
        for i in range(steps):
            flush_l2()
            e0.record()
            oks, Ts = step(warmup + i, r, host)
            e1.record()
            torch.cuda.synchronize()
            tot_ms += e0.elapsed_time(e1)
            st = r.last_batch_stats
            launches += sum(x.gpu_launches for x in st)
            iters += sum(x.iterations for x in st)
            h2d += sum(x.h2d_bytes for x in st)
            d2h += sum(x.d2h_bytes for x in st)
            for j, T in zip(ids(warmup + i), Ts):
                errs.append(synth.pose_error(T, truths[j]))
            if not host and i == steps - 1:
                keep_last(warmup + i, oks, Ts, st)
        # the collectives still in flight belong to the K timed steps: drain them inside the timed region
        e0.record()
        gather.drain()
        e1.record()
        torch.cuda.synchronize()
        drain_ms = e0.elapsed_time(e1)
        tot_ms += drain_ms
        sampler.active = False
        barrier()
        mine = torch.tensor([tot_ms, float(iters)], dtype=torch.float64, device=dev)
        if world_size > 1:
            allr = torch.zeros(2 * world_size, dtype=torch.float64, device=dev)
            dist.all_gather_into_tensor(allr, mine)
            allr = allr.cpu().numpy().reshape(world_size, 2)
        else:
            allr = mine.cpu().numpy().reshape(1, 2)
        return float(allr[:, 0].max()), launches, iters, h2d, d2h, errs, allr, drain_ms

    def timed_pipelined(steps, warmup, host):
        """host=True: e2e through fls_match_batch_begin / _end on TWO handles (each with its own copy of the map): the host->device copy of
        step i+1 runs while the kernels of step i do — every step still copies its scans from pinned host memory and reads its
        results back.  Timed as one region (the steps overlap, so there is no per-step interval): CUDA events on the idle torch
        stream right after a device-wide synchronize on both sides; L2 is flushed before every step is enqueued.
        host=False: the same with the scans resident in HBM (the `value` leg): what overlaps is the per-call host work (tables,
        launches, the wait for the results) of one batch with the kernels of the other."""
        reg2 = Registration(cfg)
        reg2.AddCloudToLocalMap([mp])
        regs = [reg, reg2]
        gs = [gather, parallel.AsyncResultGather(B, device=dev, depth=3)]

        def begin(i):
            h = i % 2
            regs[h].set_result_buffer_device(gs[h].begin_step().data_ptr(), B)
            k = ids(i)
            if host:
                regs[h].match_batch_begin([h_scans[j].numpy() for j in k], np.stack([guesses[j] for j in k]))
            else:
                regs[h].match_batch_begin_device([d_scans[j].data_ptr() for j in k], [d_scans[j].shape[0] for j in k], np.stack([guesses[j] for j in k]))

        def end(i, acc):
            h = i % 2
            oks, Ts = regs[h].match_batch_end()
            if not host and i == warmup + steps - 1:
                keep_last(i, oks, Ts, regs[h].last_batch_stats)
            gs[h].launch()
            if len(gs[h].pending) > 2:
                gs[h]._collect(gs[h].pending.pop(0))
            if acc is not None:
                st = regs[h].last_batch_stats
                acc[0] += sum(x.h2d_bytes for x in st)
                acc[1] += sum(x.d2h_bytes for x in st)
                acc[2] += sum(x.gpu_launches for x in st)
                acc[3] += sum(x.iterations for x in st)
                for j, T in zip(ids(i), Ts):
                    acc[4].append(synth.pose_error(T, truths[j]))

        for i in range(warmup):
            begin(i)
            end(i, None)
        for g in gs:
            g.drain()
        barrier()
        acc = [0, 0, 0, 0, []]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        sampler.active = True
        torch.cuda.synchronize()
        e0.record()
        for i in range(steps):
            flush_buf.zero_()  # L2 flush, asynchronous: ordered before this step's kernels only by time, which is what a flush needs
            begin(warmup + i)
            if i > 0:
                end(warmup + i - 1, acc)
        end(warmup + steps - 1, acc)
        for g in gs:
            g.drain()
        torch.cuda.synchronize()
        e1.record()
        torch.cuda.synchronize()
        tot_ms = e0.elapsed_time(e1)
        sampler.active = False
        barrier()
        for r_ in regs:
            r_.set_result_buffer_device(0, 0)
        del reg2
        mine = torch.tensor([tot_ms, float(acc[3])], dtype=torch.float64, device=dev)
        if world_size > 1:
            allr = torch.zeros(2 * world_size, dtype=torch.float64, device=dev)
            dist.all_gather_into_tensor(allr, mine)
            allr = allr.cpu().numpy().reshape(world_size, 2)
        else:
            allr = mine.cpu().numpy().reshape(1, 2)
        return float(allr[:, 0].max()), acc[2], acc[3], acc[0], acc[1], acc[4], allr, 0.0

    pipelined = wl["method"] == _abi.FLS_P2PLANE_IVOX and B > 1 and not os.environ.get("FLS_BENCH_SERIAL")
    if pipelined:
        ms_dev, launches, iters, _, _, errs, ranks_dev, drain_dev = timed_pipelined(args.steps, args.warmup, False)
        ms_e2e, _, _, h2d, d2h, _, ranks_e2e, _ = timed_pipelined(args.steps, args.warmup, True)
    else:
        ms_dev, launches, iters, _, _, errs, ranks_dev, drain_dev = timed(False, reg, args.steps, args.warmup)
        ms_e2e, _, _, h2d, d2h, _, ranks_e2e, _ = timed(True, reg, args.steps, args.warmup)
    reg.set_result_buffer_device(0, 0)
    if args.dump_outputs and rank == 0:
        os.makedirs(args.dump_outputs, exist_ok=True)
        for name, arr in last_value_step.items():
            np.save(os.path.join(args.dump_outputs, f"{name}.npy"), arr)

    # roofline leg: same steps with CUDA events around every residual-kernel launch
    reg_p = Registration(make_cfg(wl, local_rank, len(mp), flags=_abi.FLS_FLAG_PROFILE))
    reg_p.AddCloudToLocalMap([mp])
    for i in range(args.warmup):
        run_batch(reg_p, ids(i), False)
    k_ms, k_launch, k_bytes = 0.0, 0, 0
    sampler.active = True
    for i in range(args.steps):
        flush_l2()
        run_batch(reg_p, ids(args.warmup + i), False)
        st = reg_p.last_batch_stats
        k_ms += sum(x.kernel_ms for x in st)
        k_launch += sum(x.kernel_launches for x in st)
        k_bytes += sum(x.algo_bytes for x in st)
    sampler.active = False
    del reg_p
    peak, peak_src = load_peaks()
    achieved = (k_bytes / max(k_launch, 1)) / ((k_ms / max(k_launch, 1)) * 1e-3) / 1e9 if k_ms > 0 else 0.0

    total_scans = args.steps * world_size * B
    value = total_scans / (ms_dev * 1e-3)
    e2e = total_scans / (ms_e2e * 1e-3)

    # latency figure beside the throughput: one scan per call (the reference's Match signature), L2 flushed, device-resident scan
    lat_ms = 0.0
    n_lat = min(args.steps, 10)
    for i in range(n_lat + 2):
        flush_l2()
        T = guesses[i % n_pool].copy()
        ds = d_scans[i % n_pool]
        reg.match_device(ds.data_ptr(), ds.shape[0], T)
        if i >= 2:
            lat_ms += reg.last_stats.gpu_ms
    single = {"ms_per_match_gpu_span": lat_ms / max(n_lat, 1), "scans_per_s": 1e3 * n_lat / max(lat_ms, 1e-9)}

    cpu = parity = None
    if rank == 0 and world_size == 1 and not args.no_cpu:
        from oracle import pyoracle as orc
        # GPU results of the whole scan pool (same entry the timed legs use), then the oracle on the same scans and guesses
        gpu_res = []
        for b0 in range(0, n_pool, B):
            k = [(b0 + j) % n_pool for j in range(B)]
            oks, Ts = run_batch(reg, k, False)
            for j, ok, T, st in zip(k, oks, Ts, reg.last_batch_stats):
                if len(gpu_res) < n_pool:
                    gpu_res.append((bool(ok), T, st.iterations, st.n_valid))
        oreg = orc.Registration(cfg)
        oreg.add_cloud(mp)
        best, sweep, cores = tune_oracle_threads(orc, oreg, scans, guesses, log)
        t_cpu, n_cpu, orc_res = 0.0, 0, []
        while (t_cpu < args.cpu_seconds or n_cpu < n_pool) and n_cpu < 4 * n_pool and t_cpu < 4 * args.cpu_seconds + 30:
            j = n_cpu % n_pool
            ok, T, st = oreg.match(scans[j], guesses[j])
            if n_cpu < n_pool:
                orc_res.append((ok, T, st.iterations, st.n_valid))
            t_cpu += oreg.last_seconds
            n_cpu += 1
        parity = parity_block(gpu_res, orc_res)
        cpu = {"value": n_cpu / t_cpu, "unit": "scans/s", "cores": best, "kind": "port", "threads": best, "effective_cores": cores,
               "thread_sweep_scans_per_s": {str(k): v for k, v in sorted(sweep.items())}, "one_thread_value": sweep.get(1),
               "sample": f"{n_cpu} Match calls ({t_cpu:.1f}s) of the CPU oracle on the same scans/map, OpenMP with {best} threads (fastest of "
                         "the sweep), reference unbuildable here (no Eigen/PCL/TBB)"}
        del oreg
    other = None
    if rank == 0 and world_size == 1 and not args.no_secondary:
        try:
            sampler.active = True
            other = secondary_kernels(local_rank, peak, log)
        except Exception as e:  # the headline line must not depend on the side measurements
            other = {"error": repr(e)}
        sampler.active = False
    clocks = sampler.stop()

    if rank == 0:
        pos = float(np.median([e[0] for e in errs]))
        launch_us = 1e3 * k_ms / max(k_launch, 1)
        roof = {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                "peak_source": peak_src, "launches": int(k_launch), "avg_launch_us": launch_us, "algo_bytes_per_launch": k_bytes / max(k_launch, 1)}
        if wl["method"] == _abi.FLS_P2PLANE_IVOX:
            roof["kernel"] = ("p2plane_v9_kernel (whole GN loop fused: TMA-staged iVox 5-NN + plane fit + J/r + DMMA 6x6 reduction + solve; one "
                              "launch = every iteration of every scan of the batch)")
        else:
            roof["kernel"] = ("ndt_gn_batch_kernel (one cooperative launch per batch: a sub-grid and a fused GN loop per scan — 7-probe NDT "
                              "residual + 6x6 reduction + solve)")
        out = {
            "metric": "scans/sec", "value": value, "unit": "scans/s", "n_gpus": world_size, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": ms_dev / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f64",
            "data": "synthetic",
            "config": {"workload": args.workload, "desc": wl["desc"], "map_points": int(mi.n_points), "map_voxels": int(mi.n_voxels),
                       "scan_points": int(np.mean([len(s) for s in scans])), "scans_per_gpu_per_step": B, "gn_iter_cap": int(cfg.max_iterations),
                       "mean_gn_iters": iters / max(args.steps * B, 1), "parallelism": f"scan-sharded x{world_size}, map replicated",
                       "scan_pool": f"{n_pool} distinct scans shared by all ranks; rank r, step i matches scans ((i + r) * {B} + j) mod {n_pool}",
                       "l2": "flushed before every timed step (256 MiB write)",
                       "timing": ("two handles, one batch in flight on each (fls_match_batch_begin[_device] / _end): K steps in one region between two "
                                  "device-wide synchronizes, CUDA events on the idle torch stream") if pipelined else "per-step CUDA events summed",
                       "median_pos_err_vs_truth_m": pos},
            "e2e": {"value": e2e, "unit": "scans/s", "h2d_bytes_per_step": h2d // max(args.steps, 1), "d2h_bytes_per_step": d2h // max(args.steps, 1),
                    "ms_per_step": ms_e2e / args.steps,
                    "how": ("fls_match_batch_begin/_end on two handles: the pinned host->device copy of step i+1 overlaps the kernels of step i; "
                            "every step copies its scans in and its results out; one timed region over all steps") if pipelined else
                           "fls_match_batch per step: copy in, match, copy out, strictly one after the other"},
            "gpu_launches": int(launches),
            "roofline": roof,
            "parity": parity,
            "multi_gpu": {"collective": "ncclAllGather (torch.distributed all_gather_into_tensor, async_op) of 18 doubles per scan, input written by "
                                        "the GN kernel on the device, consumed two steps later",
                          "bytes_per_rank_per_step": 18 * 8 * B, "drain_ms_after_last_step": drain_dev,
                          "per_rank_ms_value_leg": [float(x) for x in ranks_dev[:, 0]], "per_rank_mean_iters": [float(x) / max(args.steps * B, 1) for x in ranks_dev[:, 1]],
                          "per_rank_ms_e2e_leg": [float(x) for x in ranks_e2e[:, 0]]},
            "single_scan_latency": single,
            "cpu_baseline": cpu,
            "clocks": clocks,
            "other_kernels": other,
        }
        print(json.dumps(out), flush=True)
    if world_size > 1:
        dist.destroy_process_group()
    if rank == 0 and parity is not None and not parity["ok"]:
        print(f"[bench] PARITY FAILURE vs the CPU oracle: {parity}", file=sys.stderr, flush=True)
        sys.exit(3)


if __name__ == "__main__":
    main()
