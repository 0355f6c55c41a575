"""Restatement of the Scan Context definitions of include/fls_b200.h (fls_sc_cfg) in numpy: the descriptor, the column norms, the
distance at every shift, the ranking and the yaw.  Angles come from the pinned atan2f's CPU twin (oracle_convert); everything else is
float64, one rounded operation at a time (numpy never contracts to FMA), summed in the stated order: columns ascending, rings
ascending.  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import numpy as np

from oracle_convert.pyoracle_convert import atan2f

TWO_PI = 6.283185307179586  # the fp64 constant 2*pi
PI = 3.141592653589793


def f2ord(v: np.ndarray) -> np.ndarray:
    """order-preserving float32 -> uint32 (-0.0 below +0.0); no finite value maps to 0, the empty cell"""
    u = np.asarray(v, np.float32).view(np.uint32)
    return np.where(u & 0x80000000, ~u, u | 0x80000000).astype(np.uint32)


def ord2f(o: np.ndarray) -> np.ndarray:
    o = np.asarray(o, np.uint32)
    return np.where(o & 0x80000000, o & 0x7fffffff, ~o).astype(np.uint32).view(np.float32)


def descriptor(cloud, n_rings: int = 20, n_sectors: int = 60, max_radius: float = 80.0, z_offset: float = 2.0) -> np.ndarray:
    """(n_rings, n_sectors) float32 descriptor of a packed (n,4) or pcl (n,8) float32 cloud."""
    p = np.asarray(cloud, np.float32)[:, :3]
    p = p[np.isfinite(p).all(axis=1)]
    x, y = p[:, 0].astype(np.float64), p[:, 1].astype(np.float64)
    r = np.sqrt(x * x + y * y)
    R = np.float64(np.float32(max_radius))
    keep = r < R
    p, r = p[keep], r[keep]
    ring = np.minimum(n_rings - 1, np.floor((r * n_rings) / R)).astype(np.int64)
    th = atan2f(p[:, 1], p[:, 0]).astype(np.float64)
    th = np.where(th < 0.0, th + TWO_PI, th)
    sector = np.minimum(n_sectors - 1, np.floor((th * n_sectors) / TWO_PI)).astype(np.int64)
    val = (p[:, 2] + np.float32(z_offset)).astype(np.float32)
    cells = np.zeros(n_rings * n_sectors, np.uint32)
    np.maximum.at(cells, ring * n_sectors + sector, f2ord(val))
    out = np.where(cells == 0, np.float32(0.0), ord2f(cells)).astype(np.float32)
    return out.reshape(n_rings, n_sectors)


def column_norms(desc: np.ndarray) -> np.ndarray:
    """fp64 column norms of (..., n_rings, n_sectors) descriptors: rings summed in order, then sqrt"""
    d = np.asarray(desc, np.float64)
    s = np.zeros(d.shape[:-2] + d.shape[-1:])
    for r in range(d.shape[-2]):
        v = d[..., r, :]
        s = s + v * v
    return np.sqrt(s)


def shift_distances(Q: np.ndarray, Cs: np.ndarray) -> np.ndarray:
    """d_s of query Q (n_rings, n_sectors) against each candidate of Cs (n, n_rings, n_sectors): (n, n_sectors) float64"""
    Q = np.asarray(Q, np.float64)
    Cs = np.asarray(Cs, np.float64).reshape((-1,) + Q.shape)
    n_rings, S = Q.shape
    n = len(Cs)
    qn, cn = column_norms(Q), column_norms(Cs)
    shifts = np.arange(S)
    sums = np.zeros((n, S))
    E = np.zeros((n, S), np.int64)
    with np.errstate(divide="ignore", invalid="ignore"):
        for j in range(S):
            col = (j + shifts) % S
            b = cn[:, col]
            valid = (qn[j] != 0.0) & (b != 0.0)
            Cc = Cs[:, :, col]
            dot = np.zeros((n, S))
            for r in range(n_rings):
                dot = dot + Q[r, j] * Cc[:, r, :]
            sums = np.where(valid, sums + dot / (qn[j] * b), sums)
            E += valid
        return np.where(E > 0, 1.0 - sums / np.maximum(E, 1), 1.0)


def distances(Q, Cs):
    """(D, best shift, every d_s) of each candidate: D = min_s d_s, ties to the smallest s"""
    d = shift_distances(Q, Cs)
    s = np.argmin(d, axis=1)
    return d[np.arange(len(d)), s], s, d


def yaw(shift, n_sectors: int):
    """s * (2*pi / n_sectors), wrapped to (-pi, pi]"""
    psi = np.asarray(shift, np.float64) * (TWO_PI / n_sectors)
    return np.where(psi > PI, psi - TWO_PI, psi)


def rank(D, ids=None):
    """indices ordered by (D, id)"""
    D = np.asarray(D)
    ids = np.arange(len(D)) if ids is None else np.asarray(ids)
    return np.lexsort((ids, D))
