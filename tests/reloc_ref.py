"""Independent reference of fls_relocalize's coarse stage (include/fls_b200.h): the hypothesis grid in fp64, the coarse score of every
hypothesis with an exact 1-NN (scipy cKDTree) on the float-transformed coarse cloud, the margin of every inlier gate in ulps, and the
selection of the n best with the gaps that decide it."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
from scipy.spatial import cKDTree

from tests.icp_ref import transform_f

F32 = np.float32
MAX_HYPOTHESES = 1 << 20


@dataclass
class Grid:
    I: int
    K: int
    k0: int
    n_yaw: int
    P: int


def grid(xy_radius, xy_step, yaw_range, yaw_step) -> Grid:
    """Offsets -I..I in x and y, yaw offsets k0..K; ValueError above 2^20 hypotheses."""
    I = int(np.floor(xy_radius / xy_step + 1e-9)) if xy_radius > 0 else 0
    K = int(np.floor(min(yaw_range, np.pi) / yaw_step + 1e-9)) if yaw_range > 0 else 0
    k0 = -K
    if yaw_range >= np.pi and K > 0 and 2.0 * K * yaw_step >= 2.0 * np.pi - 1e-9:
        k0 = -K + 1  # -K would repeat +K
    n_yaw = K - k0 + 1
    P = (2 * I + 1) ** 2 * n_yaw
    if P > MAX_HYPOTHESES:
        raise ValueError(f"{P} hypotheses")
    return Grid(I, K, k0, n_yaw, P)


def yaw_offsets(g: Grid, yaw_step) -> np.ndarray:
    return np.arange(g.k0, g.K + 1, dtype=np.float64) * (yaw_step if g.K else 0.0)


def hypotheses(T_guess, xy_radius, xy_step, yaw_range, yaw_step) -> np.ndarray:
    """(P, 4, 4) fp64 poses in index order (yaw fastest, then x, then y): R = Rz(psi) R_guess, t = t_guess + (dx, dy, 0)."""
    g = grid(xy_radius, xy_step, yaw_range, yaw_step)
    step = xy_step if g.I else 0.0
    psi = yaw_offsets(g, yaw_step)
    c, s = np.cos(psi), np.sin(psi)
    Rg = np.asarray(T_guess, np.float64)[:3, :3]
    R = np.empty((g.n_yaw, 3, 3))
    R[:, 0, :] = c[:, None] * Rg[0][None, :] - s[:, None] * Rg[1][None, :]
    R[:, 1, :] = s[:, None] * Rg[0][None, :] + c[:, None] * Rg[1][None, :]
    R[:, 2, :] = Rg[2][None, :]
    off = np.arange(-g.I, g.I + 1, dtype=np.float64) * step
    out = np.zeros((g.P, 4, 4))
    p = 0
    for dy in off:
        for dx in off:
            for k in range(g.n_yaw):
                out[p, :3, :3] = R[k]
                out[p, :3, 3] = T_guess[:3, 3] + np.array([dx, dy, 0.0])
                out[p, 3, 3] = 1.0
                p += 1
    return out


def d2_nn(tree: cKDTree, fit: np.ndarray, q: np.ndarray, k: int = 4) -> np.ndarray:
    """fp32 squared distance to the nearest fit point in the reference's operation order ((dx*dx + dy*dy) + dz*dz), the minimum over
    the k nearest in fp64 so that a near tie cannot pick a different fp32 value."""
    kk = min(k, len(fit))
    _, idx = tree.query(q.astype(np.float64), k=kk)
    idx = idx.reshape(len(q), kk)
    d = (fit[idx] - q[:, None, :]).astype(F32)
    return np.min((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2], axis=1).astype(F32)


@dataclass
class Coarse:
    score: np.ndarray         # (P,) fp64
    inliers: np.ndarray       # (P,) int
    gate_ulps: np.ndarray     # (P,) smallest |d2 - max_range| of the hypothesis, in ulps of max_range


def coarse_scores(fit_cloud, coarse_cloud, poses, max_range) -> Coarse:
    fit = np.ascontiguousarray(fit_cloud[:, :3], F32)
    tree = cKDTree(fit.astype(np.float64))
    m = len(coarse_cloud)
    mr = F32(max_range)
    ulp = float(np.spacing(mr))
    P = len(poses)
    score, inl, margin = np.zeros(P), np.zeros(P, np.int64), np.zeros(P)
    for p in range(P):
        q = transform_f(coarse_cloud, poses[p])
        d2 = d2_nn(tree, fit, q)
        keep = d2 <= mr
        inl[p] = int(keep.sum())
        score[p] = (float(np.sum(d2[keep].astype(np.float64))) + (m - inl[p]) * float(mr)) / m
        margin[p] = float(np.min(np.abs(d2.astype(np.float64) - float(mr)))) / ulp
    return Coarse(score, inl, margin)


def select(score: np.ndarray, n: int):
    """The n smallest scores, ties to the lower index; and for each rank r the gap to the next score in that order (how decided r is)."""
    order = np.lexsort((np.arange(len(score)), score))
    s = score[order]
    gaps = np.append(np.diff(s), np.inf)
    return order[:n], gaps[:n]
