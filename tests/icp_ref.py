"""Brute-force reference of IcpOptimized's exact 1-NN, its first Gauss-Newton pass and GetFitnessScore (CPU only, independent of the
oracle and of the CUDA library; the PCL voxel filter is taken from orc.voxel_grid, which the GPU filter matches bit for bit).

`nn1` finds the nearest map point of every query without any grid: candidates come from a kd-tree, distances are recomputed in fp32
in the order of pointcloud_utility.h:13-17 upstream, (dx^2 + dy^2) + dz^2, and every point at the smallest distance is kept — a tie
is reported, not resolved.  `icp_pass` applies the gate of icp_optimized.h:87 (double(d2) > max_corr rejects, [quirk 4]) and sums
iteration 0's H, g and n_valid (:70-127); `fitness` is GetFitnessScore (:191-215).  Margins are in fp32 ulps of d2 to the gates."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
from scipy.spatial import cKDTree

from oracle import pyoracle as orc
from tests.ivox_ref import dist2, ulp_gap

F32 = np.float32
EPS = float(np.finfo(np.float64).eps)


def transform_f(pts, T):
    """TransformPointCloud with R, t cast to float (pointcloud_utility.h:141-158): ((r0 x + r1 y) + r2 z) + t in fp32.  For a pose
    whose rotation is the identity every product is exact and only `+ t` rounds, so any contraction gives the same point."""
    T = np.asarray(T, np.float64)
    Rf, tf = T[:3, :3].astype(F32), T[:3, 3].astype(F32)
    p = np.asarray(pts, F32)[:, :3]
    return np.stack([((Rf[a, 0] * p[:, 0] + Rf[a, 1] * p[:, 1]) + Rf[a, 2] * p[:, 2]) + tf[a] for a in range(3)], axis=1).astype(F32)


@dataclass
class Nn1:
    d2: np.ndarray     # (n,) fp32 smallest squared distance (inf: empty map)
    ties: list         # (n,) map indices at that distance
    gap12: np.ndarray  # (n,) ulps between ranks 1 and 2 (0: a tie)


def nn1(map_pts, q, k=16):
    m = np.asarray(map_pts, F32)[:, :3]
    q = np.asarray(q, F32)[:, :3]
    tree = cKDTree(m.astype(np.float64))
    n = len(q)
    out = Nn1(np.full(n, np.inf, F32), [[] for _ in range(n)], np.full(n, -1, np.int64))
    kk = min(k, len(m))
    _, idx = tree.query(q.astype(np.float64), k=kk)
    idx = np.asarray(idx).reshape(n, kk)
    for i in range(n):
        cand = idx[i]
        d = dist2(m[cand], q[i])
        # the fp64 kd-tree ranks by the exact distance; fp32 rounding can only reorder points whose exact distances are within a
        # few ulps, so every fp32 minimum is among the candidates as long as the k-th candidate is clearly farther
        assert kk == len(m) or float(np.max(d)) > float(np.min(d)) * (1 + 1e-5), i
        order = np.argsort(d, kind="stable")
        best = d[order[0]]
        out.d2[i] = best
        out.ties[i] = sorted(int(cand[j]) for j in order if d[j] == best)
        if len(order) > 1:
            out.gap12[i] = ulp_gap(best, d[order[1]])
    return out


@dataclass
class IcpPass:
    H: np.ndarray
    g: np.ndarray
    n_valid: int
    valid: np.ndarray
    nn: Nn1
    q: np.ndarray           # transformed source (fp32)
    src: np.ndarray         # filtered source
    gate_ulps: np.ndarray   # (n,) ulps from d2 to max_corr rounded to fp32 (negative: inside)
    tol_H: np.ndarray
    tol_g: np.ndarray
    J: list


def icp_pass(map_pts, scan, T, max_corr, src_leaf, map_leaf):
    """Iteration 0 of IcpOptimized::Match in localization mode (map = VoxelGridCloud(cloud, map_leaf), :165-189)."""
    mp = orc.voxel_grid(np.asarray(map_pts, F32), map_leaf)
    src = orc.voxel_grid(np.asarray(scan, F32), src_leaf)  # :57
    T = np.asarray(T, np.float64)
    q = transform_f(src, T)
    nn = nn1(mp, q)
    R = T[:3, :3]
    H, g, aH, ag = np.zeros((6, 6)), np.zeros(6), np.zeros((6, 6)), np.zeros(6)
    valid = np.zeros(len(q), bool)
    Js = []
    gate = np.array([ulp_gap(F32(max_corr), d) if np.isfinite(d) else 1 << 30 for d in nn.d2])
    for i in range(len(q)):
        if not np.isfinite(nn.d2[i]) or float(nn.d2[i]) > max_corr:  # :87
            continue
        valid[i] = True
        m = mp[nn.ties[i][0], :3].astype(np.float64)
        e = q[i].astype(np.float64) - m
        p = src[i, :3].astype(np.float64)
        hat = np.array([[0, -p[2], p[1]], [p[2], 0, -p[0]], [-p[1], p[0], 0]])
        J = np.hstack([np.eye(3), -R @ hat])  # :100
        Js.append((i, J, e))
        H += J.T @ J
        g += -J.T @ e
        aH += np.abs(J).T @ np.abs(J)
        ag += np.abs(J).T @ np.abs(e)
    n = int(valid.sum())
    return IcpPass(H, g, n, valid, nn, q, src, gate, 16 * (n + 4) * EPS * aH, 16 * (n + 4) * EPS * ag, Js)


def fitness(map_pts, src_f, T, max_range):
    """GetFitnessScore(max_range): mean fp32 squared 1-NN distance over points with d2 <= max_range (:191-215), accumulated in
    fp32 as upstream; FLT_MAX without inliers.  src_f: the filtered source of the last Match.  Returns (score, d2 of the inliers,
    ulps of every d2 to max_range)."""
    q = transform_f(src_f, T)
    nn = nn1(map_pts, q)
    keep = nn.d2 <= F32(max_range)
    gate = np.array([ulp_gap(F32(max_range), d) for d in nn.d2])
    if not np.any(keep):
        return float(np.finfo(F32).max), nn.d2[keep], gate
    return float(np.sum(nn.d2[keep].astype(np.float64)) / np.sum(keep)), nn.d2[keep], gate


def assert_matches(H, g, n_valid, ref: IcpPass):
    assert int(n_valid) == ref.n_valid, (n_valid, ref.n_valid)
    H, g = np.asarray(H), np.asarray(g)
    assert np.all(np.abs(H - ref.H) <= ref.tol_H), np.max(np.abs(H - ref.H) / np.maximum(ref.tol_H, 1e-300))
    assert np.all(np.abs(g - ref.g) <= ref.tol_g), np.max(np.abs(g - ref.g) / np.maximum(ref.tol_g, 1e-300))


def assert_gates_clear(ref: IcpPass, tie_ok=True):
    """The gate is decided exactly (d2 is an fp32 number compared in fp64: no rounding between the sides); what must be clear is
    the choice of neighbour: a rank-1/rank-2 gap of zero is a tie, reported in nn.ties, and only allowed where the caller checks
    membership instead of identity."""
    if not tie_ok:
        assert all(len(t) <= 1 for t in ref.nn.ties)


def assert_sensitive(ref: IcpPass, factor=100.0):
    """Dropping any one accepted point moves H (its identity block counts n_valid) or g by at least `factor` x the tolerance."""
    tH, tg = np.maximum(ref.tol_H, 1e-300), np.maximum(ref.tol_g, 1e-300)
    for i, J, e in ref.J:
        move = max(np.max(np.abs(J.T @ J) / tH), np.max(np.abs(J.T @ e) / tg))
        assert move >= factor, (i, move)
