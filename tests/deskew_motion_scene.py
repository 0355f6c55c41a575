"""A 64-line sweep taken by a sensor moving at constant velocity through synth.World, with the known answer of its de-skew.

Every column fires at its own time t_c = c / n_cols * 0.1 s and is ray-cast from the sensor's position at that time, o_c = o_0 + v t_c;
the orientation stays R_0, so the IMU buffer is the identity quaternion throughout and the lidar -> imu extrinsic is the identity.  The
reference time is the start of the sweep.  In the body frame at the reference time a return then sits at p_body + v_body t_c, which is
what the velocity-aware de-skew computes; the rotation-only de-skew leaves it at p_body, v t_c away from the surface it hit."""
from __future__ import annotations

import numpy as np

from funny_lidar_slam_b200 import synth

REF = 1_700_000_000_000_000
SWEEP = 0.1
MIN_D, MAX_D, JUMP, LEAF = 2.0, 100.0, 3, 0.5


def moving_sweep(world, pose, speed=15.0, sensor="hdl64", seed=7, noise=0.02):
    """dict: raw (n,5) x, y, z, intensity, time [s] in firing order, ring, imu, velocity (body frame, m/s), pose, hit (n,3) the measured
    world points (noise included), surface (n,3) the noise-free surface points and dt (n,) each point's firing time."""
    sn = synth.SENSORS[sensor]
    d, ring, col = synth.sensor_dirs(sn)  # column-major firing order
    R0, o0 = pose[:3, :3], pose[:3, 3]
    v_body = np.array([speed, 0.0, 0.0])  # along the heading
    v_world = R0 @ v_body
    dw = d @ R0.T
    t_col = (np.arange(sn.cols) / sn.cols * SWEEP).astype(np.float32)
    rng = np.random.default_rng(seed)
    rng_t = np.full(len(d), np.inf)
    for c in range(sn.cols):  # one ray cast per column, from where the sensor is when that column fires
        sel = slice(c * sn.lines, (c + 1) * sn.lines)
        rng_t[sel] = synth.raycast(world, o0 + v_world * float(t_col[c]), dw[sel], MAX_D)[0]
    eps = rng.normal(0.0, noise, len(d))
    meas = rng_t + eps
    keep = np.isfinite(rng_t) & (meas >= MIN_D) & (meas <= MAX_D)
    tc = t_col[col[keep]]
    raw = np.zeros((int(keep.sum()), 5), np.float32)
    raw[:, :3] = d[keep] * meas[keep, None]
    raw[:, 3] = (ring[keep] % 7) * 10.0 + 5.0
    raw[:, 4] = tc
    origin = o0[None, :] + v_world[None, :] * tc[:, None].astype(np.float64)
    t_us = (REF + np.arange(-20_000, 125_001, 5_000)).astype(np.uint64)  # 200 Hz, covering the sweep
    q = np.tile([0.0, 0.0, 0.0, 1.0], (len(t_us), 1))
    imu = dict(t_us=t_us, q_xyzw=q, ref_time_us=REF, T_lidar_to_imu=np.eye(4))
    return dict(raw=raw, ring=ring[keep].astype(np.int32), imu=imu, velocity=v_body, pose=pose, dt=tc.astype(np.float64),
                hit=origin + dw[keep] * meas[keep, None], surface=origin + dw[keep] * rng_t[keep, None])


def world_error(cloud, s):
    """|R_0 p + o_0 - hit| per point of an ordered cloud (all raw points kept: same order as s["raw"])."""
    T = s["pose"]
    w = cloud[:, :3].astype(np.float64) @ T[:3, :3].T + T[:3, 3]
    return np.linalg.norm(w - s["hit"], axis=1), np.linalg.norm(w - s["surface"], axis=1)


def surface_map(world, pose, radius=90.0):
    """The static surfaces of the world around the pose, sampled every 0.3 m."""
    m = synth.make_surface_map(world, spacing=0.3, seed=11)
    near = np.hypot(m[:, 0] - pose[0, 3], m[:, 1] - pose[1, 3]) < radius
    return np.ascontiguousarray(m[near])


def negative_zero_scenes():
    """Scenes whose rotation-only de-skew yields -0.0 coordinates, so that skipping the translation term for a zero velocity (the
    pinned rule) and adding +0.0 (which turns -0.0 into +0.0) give different bits.  Both orientations are the identity rotation, as
    q_ref = (0, 0, 0, -1) and q(t) = (0, 0, -0.0, 1); the extrinsic translation is (-0.0, 0, 0); every point has coordinates in
    {+-0, +-3} and fires 3 or 4.5 ms after the reference time (the rotation then sends (-0, -0, -3) to (-0, ...)).  Returns a de-skew
    scene (the keys of tests/frontend_scenes.deskew_scenes) and a projector scene (those of project_scenes)."""
    import itertools
    pts = [list(c) for c in itertools.product([-0.0, 0.0, -3.0, 3.0], repeat=3) if any(x != 0 for x in c)]
    n = len(pts)
    raw = np.zeros((2 * n, 5), np.float32)
    raw[:, :3] = pts + pts
    raw[:, 3] = np.arange(2 * n) % 7
    raw[:n, 4], raw[n:, 4] = np.float32(0.003), np.float32(0.0045)
    T = np.eye(4)
    T[0, 3] = -0.0
    q_ref, q_pt = (0.0, 0.0, 0.0, -1.0), (0.0, 0.0, -0.0, 1.0)
    imu = dict(t_us=(REF + np.array([-1000, 0, 1000, 5000])).astype(np.uint64), q_xyzw=np.array([q_ref, q_ref, q_pt, q_pt]), ref_time_us=REF,
               T_lidar_to_imu=T)
    deskew = dict(name="negative_zero", raw=raw, imu=imu, min_d=0.5, max_d=100.0, jump=1, leaf=0.5, reaches=("negative_zero",))
    V = 2 * n
    project = dict(name="negative_zero", raw=np.ascontiguousarray(raw[:, :4]), ring=np.arange(V, dtype=np.int32),
                   time=np.ascontiguousarray(raw[:, 4]), imu=imu, V=V, H=16, h_res=np.float32(2 * np.pi / 16), min_d=0.5, max_d=100.0)
    return deskew, project
