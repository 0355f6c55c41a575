"""Independent restatement of fls_relocalize_wide's search geometry and of the slack of its lower bound (include/fls_b200.h,
fls_reloc.cu): the caps of the grid, the blocks of a level and their representatives, and delta_i, the distance by which any
hypothesis of a block can move scan point i away from where the representative puts it, including the fp32 rounding of both
transforms and of the squared distance."""
from __future__ import annotations

import numpy as np

from tests import reloc_ref
from tests.icp_ref import transform_f

F32 = np.float32
U = 2.0 ** -24  # unit roundoff of fp32
MAX_HYPOTHESES = 1 << 31
MAX_I = 32767
START_NODES = 1 << 20


def grid(xy_radius, xy_step, yaw_range, yaw_step) -> reloc_ref.Grid:
    """reloc_ref.grid with the wide caps: ValueError above 2^31 hypotheses or 32767 x-y steps."""
    I = int(np.floor(xy_radius / xy_step + 1e-9)) if xy_radius > 0 else 0
    K = int(np.floor(min(yaw_range, np.pi) / yaw_step + 1e-9)) if yaw_range > 0 else 0
    if I > MAX_I or K > MAX_HYPOTHESES:
        raise ValueError(f"I={I} K={K}")
    k0 = -K + 1 if (yaw_range >= np.pi and K > 0 and 2.0 * K * yaw_step >= 2.0 * np.pi - 1e-9) else -K
    n_yaw = K - k0 + 1
    P = (2 * I + 1) ** 2 * n_yaw
    if P > MAX_HYPOTHESES:
        raise ValueError(f"{P} hypotheses")
    return reloc_ref.Grid(I, K, k0, n_yaw, P)


def blocks(n: int, level: int) -> int:
    return (n + (1 << level) - 1) >> level


def start_level(g: reloc_ref.Grid) -> int:
    """The lowest level with at most 2^20 blocks."""
    nx, l = 2 * g.I + 1, 0
    while blocks(nx, l) ** 2 * blocks(g.n_yaw, l) > START_NODES:
        l += 1
    return l


def block_rep(b: int, level: int, n: int):
    """(representative index, largest offset to any index) of block b of an axis of n leaves."""
    lo = b << level
    hi = min(lo + (1 << level), n) - 1
    r = min(lo + (1 << (level - 1)), hi) if level else lo
    return r, max(r - lo, hi - r)


def leaf_pose(T_guess, g: reloc_ref.Grid, xy_step, yaw_step, ix, jy, ky) -> np.ndarray:
    """Hypothesis (x index ix, y index jy, yaw index ky), all from 0, in fp64 as the grid defines it."""
    psi = (g.k0 + ky) * (yaw_step if g.K else 0.0)
    c, s = np.cos(psi), np.sin(psi)
    T = np.array(T_guess, np.float64)
    g0, g1 = T[0, :3].copy(), T[1, :3].copy()
    T[0, :3], T[1, :3] = c * g0 - s * g1, s * g0 + c * g1
    step = xy_step if g.I else 0.0
    T[0, 3] = T_guess[0, 3] + (ix - g.I) * step
    T[1, 3] = T_guess[1, 3] + (jy - g.I) * step
    return T


def slack(p, R_guess, hx, hy, hk, xy_step, yaw_step, tau, max_range) -> np.ndarray:
    """delta_i for the points p (n, 3): sqrt(hx^2 + hy^2) xy_step + hk yaw_step |(R_guess p)_xy| + eps_i, with
    eps_i = 32u (tau + |p_i|_1) + 8u sqrt(max_range) (tau: the largest translation coordinate of any hypothesis)."""
    p = np.asarray(p, np.float64)
    v = p @ np.asarray(R_guess, np.float64)[:2, :3].T
    eps = 32.0 * U * (tau + np.abs(p).sum(axis=1)) + 8.0 * U * np.sqrt(max_range)
    return np.hypot(hx, hy) * xy_step + hk * yaw_step * np.hypot(v[:, 0], v[:, 1]) + eps


def dist2_f(a, b) -> np.ndarray:
    """dist2_ref: ((dx*dx + dy*dy) + dz*dz) in fp32."""
    d = (np.asarray(a, F32) - np.asarray(b, F32)).astype(F32)
    return ((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).astype(F32)


def bound_terms(q_rep, fit, p, R_guess, hx, hy, hk, xy_step, yaw_step, tau, max_range) -> np.ndarray:
    """min(max(0, b_i - delta_i)^2, max_range) with the tightest b_i there is: the exact distance from the representative's fp32
    point to its fit point."""
    b = np.linalg.norm(np.asarray(q_rep, np.float64) - np.asarray(fit, np.float64), axis=1)
    e = np.maximum(0.0, b - slack(p, R_guess, hx, hy, hk, xy_step, yaw_step, tau, max_range))
    return np.minimum(e * e, float(F32(max_range)))


def leaf_terms(q_leaf, fit, max_range) -> np.ndarray:
    """GetFitnessScore's gated term of each point at a leaf: min(fp32 squared distance, max_range)."""
    return np.minimum(dist2_f(q_leaf, fit).astype(np.float64), float(F32(max_range)))


def moved(p, T) -> np.ndarray:
    return transform_f(np.asarray(p, F32), T)
