#!/usr/bin/env python
"""Regenerates the golden vectors under tests/golden/ from the CPU oracle on seeded synthetic scenes.

The reference cannot be built or imported here (SURVEY.md §8c) and ships no fixture for this path, so these
goldens pin the ORACLE (regression anchor for the restatement), not the reference: parity stays "unpinned".
Run from the repo root:  python tests/golden/make_golden.py
(`--reference-tree DIR` instead rewrites reference_line_counts.json from a checkout of the reference.)
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from funny_lidar_slam_b200 import FLS_ICP_P2P, FLS_NDT, FLS_P2PLANE_IVOX, default_config, synth  # noqa: E402
from funny_lidar_slam_b200._abi import FLS_FLAG_ITER_LOG, FLS_LOAM_FULL, FLS_P2PLANE_KNN  # noqa: E402
from oracle import pyoracle as orc  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def scene16():
    world = synth.make_world()
    traj = synth.trajectory(16)
    scan = synth.make_scan(world, traj[5], "vlp16", seed=5)["points"]
    mp = synth.make_map_from_scans(world, traj[0:12:2], "vlp16", leaf=0.3)
    return dict(world=world, traj=traj, scan=scan, map=mp, truth=traj[5], guess=synth.perturb_pose(traj[5]),
                guess_small=synth.perturb_pose(traj[5], dpos=0.05, drot_deg=0.5))


def run(method, sc, scan, guess, **kw):
    cfg = default_config(method, flags=FLS_FLAG_ITER_LOG, **kw)
    r = orc.Registration(cfg)
    r.add_cloud(sc["map"])
    ok, T, st = r.match(scan, guess)
    log = r.iter_log()
    return dict(T=T, ok=ok, iters=st.iterations, n_valid=st.n_valid, H0=log[0]["H"], g0=log[0]["g"], n_valid0=log[0]["n_valid"],
                scan_checksum=float(np.sum(scan.astype(np.float64))), map_checksum=float(np.sum(sc["map"].astype(np.float64))))


def main():
    sc = scene16()
    np.savez(os.path.join(OUT, "p2plane_scene16_4000.npz"), **run(FLS_P2PLANE_IVOX, sc, sc["scan"][:4000], sc["guess"]))
    np.savez(os.path.join(OUT, "p2plane_scene16.npz"), **run(FLS_P2PLANE_IVOX, sc, sc["scan"], sc["guess"]))
    np.savez(os.path.join(OUT, "ndt_scene16.npz"), **run(FLS_NDT, sc, sc["scan"], sc["guess_small"]))
    np.savez(os.path.join(OUT, "icp_scene16.npz"), **run(FLS_ICP_P2P, sc, sc["scan"], sc["guess"]))
    proj = synth.make_projected_scan(sc["world"], sc["traj"][7], kind="spin", sensor="vlp16", seed=12)
    ci, pi, _ = orc.extract_features(proj["depth"], proj["col"], len(proj["ordered"]), proj["row_start"], proj["row_end"], 1.0, 0.1)
    np.savez(os.path.join(OUT, "features_vlp16.npz"), corner_idx=ci, planar_idx=pi, n=len(proj["ordered"]),
             depth_checksum=float(np.sum(proj["depth"].astype(np.float64))))
    vg = orc.voxel_grid(sc["scan"], 0.4)
    np.savez(os.path.join(OUT, "voxelgrid_scene16_0p4.npz"), n=len(vg), checksum=float(np.sum(vg.astype(np.float64))), first=vg[:8], last=vg[-8:])
    # kd-tree LOAM plug-ins on feature clouds (same scene as tests/test_oracle_loam_kd.py::feature_scene)
    def feats(pose, seed):
        pr = synth.make_projected_scan(sc["world"], pose, kind="spin", sensor="vlp16", seed=seed)
        c_i, p_i, _ = orc.extract_features(pr["depth"], pr["col"], len(pr["ordered"]), pr["row_start"], pr["row_end"], 1.0, 0.1)
        return pr["ordered"][p_i].copy(), pr["ordered"][c_i].copy()

    def to_world(pts, T):
        o = pts.copy()
        o[:, :3] = (pts[:, :3].astype(np.float64) @ T[:3, :3].T + T[:3, 3]).astype(np.float32)
        return o

    traj = sc["traj"]
    maps = [feats(traj[k], k) for k in (3, 4, 6, 7)]
    maps_p = [to_world(m[0], traj[k]) for m, k in zip(maps, (3, 4, 6, 7))]
    maps_c = [to_world(m[1], traj[k]) for m, k in zip(maps, (3, 4, 6, 7))]
    p5, c5 = feats(traj[5], 55)
    guess = synth.perturb_pose(traj[5], dpos=0.1, drot_deg=1.0)

    def pack(r, ok, T, st):
        lg = r.iter_log()
        return dict(T=T, ok=ok, iters=st.iterations, n_valid=st.n_valid, H0=lg[0]["H"], g0=lg[0]["g"],
                    planar_checksum=float(np.sum(p5.astype(np.float64))))

    r = orc.Registration(default_config(FLS_P2PLANE_KNN, flags=FLS_FLAG_ITER_LOG))
    r.add_cloud(np.concatenate(maps_p))
    np.savez(os.path.join(OUT, "kdtree_features.npz"), **pack(r, *r.match(p5, guess)))
    r = orc.Registration(default_config(FLS_LOAM_FULL, localization_mode=0, flags=FLS_FLAG_ITER_LOG))
    for mp_, mc_ in zip(maps_p, maps_c):
        r.add_cloud(mp_, mc_)
    np.savez(os.path.join(OUT, "loamfull_features.npz"), **pack(r, *r.match(p5, guess, corner=c5)))
    print("golden vectors written to", OUT)


def round2():
    """Goldens of the round-2 oracle parts: de-skew / pre-processing / projector with de-skew (oracle/orc_deskew.h) and the LRU of the
    iVox map (oracle/orc_ivox.h) on the seeded case of tests/test_oracle_deskew.py."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_oracle_deskew import make_case
    raw, imu = make_case(n=6000, seed=0)
    o_ord, o_pl = orc.preprocess(raw, imu, 2.0, 60.0, 4, 0.5)
    rng = np.random.default_rng(1)
    ring = rng.integers(0, 16, len(raw)).astype(np.int32)
    pr = orc.project_imu(raw[:, :4], ring, raw[:, 4], imu, 16, 900, np.float32(2 * np.pi / 900), 2.0, 60.0)
    np.savez(os.path.join(OUT, "deskew_case0.npz"), n_ordered=len(o_ord), n_planar=len(o_pl), ordered_first=o_ord[:16], ordered_last=o_ord[-16:],
             ordered_checksum=float(np.sum(o_ord.astype(np.float64))), planar_checksum=float(np.sum(o_pl.astype(np.float64))),
             proj_n=pr["n"], proj_checksum=float(np.sum(pr["ordered"].astype(np.float64))), proj_depth_checksum=float(np.sum(pr["depth"].astype(np.float64))),
             proj_col_checksum=int(np.sum(pr["col"].astype(np.int64))), proj_row_start=pr["row_start"], proj_row_end=pr["row_end"])
    # LRU: three clouds through an IVoxMap of 5000 voxels (the second and third cloud evict)
    world = synth.make_world()
    traj = synth.trajectory(16)
    iv = orc.IVox(0.5, 2, 5000)
    counts = []
    for k in range(3):
        c = synth.transform_points(synth.make_scan(world, traj[k], "vlp16", seed=60 + k)["points"], traj[k])
        iv.add(c)
        counts.append((iv.num_voxels, iv.num_points))
    np.savez(os.path.join(OUT, "ivox_lru_cap5000.npz"), counts=np.array(counts, np.int64))


def reference_line_counts(ref: str):
    """Line counts of the reference's citable files (path relative to `ref`), which tests/test_citations.py checks the
    `file:line` citations of this repository against."""
    import json
    counts = {}
    for d, _, fs in os.walk(ref):
        if "/.git" in d:
            continue
        for f in fs:
            if f.endswith((".h", ".cpp", ".yaml", ".md", ".txt")):
                with open(os.path.join(d, f), errors="ignore") as fh:
                    counts[os.path.relpath(os.path.join(d, f), ref)] = sum(1 for _ in fh)
    with open(os.path.join(OUT, "reference_line_counts.json"), "w") as fh:
        json.dump(dict(sorted(counts.items())), fh, indent=0)


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "--reference-tree":
        reference_line_counts(sys.argv[2])
    else:
        main()
        round2()
