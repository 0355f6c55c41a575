"""Reference of the FLS_FLAG_INFORMATION record (CPU only, independent of the CUDA library): H = sum J^T W J, g = sum J^T W r,
n_valid and sum_residual at a pose, with the correspondences, gates, residuals and weights of the brute-force first-pass references
(tests/ivox_ref.py, ndt_ref.py, icp_ref.py, loam_kd_ref.py) and the Jacobians written analytically in the fusion parameterization:
order [dθ; dp], T perturbed as R <- R·Exp(dθ), p <- p + dp.

A point p (body frame) lands at q = R p + t; under the perturbation q(dθ, dp) = R Exp(dθ) p + t + dp, so dq/d[dθ; dp] = [-R hat(p), I]
(`j_point`).  A scalar residual r(q) has J = (dr/dq) j_point; a vector residual e(q) has J = j_point.  The references give dr/dq of the
LOAM terms as the position half of their J (the coefficient of dt in dx = [dθ, dt]): the signed plane normal, or n x u for a corner
line.  Nothing here reads the plug-ins' own dx or the map A the library applies."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np


def hat(p):
    return np.array([[0.0, -p[2], p[1]], [p[2], 0.0, -p[0]], [-p[1], p[0], 0.0]])


def j_point(R, p):
    """dq / d[dθ; dp] of q = R Exp(dθ) p + t + dp at 0 (3x6)."""
    return np.hstack([-np.asarray(R, np.float64) @ hat(np.asarray(p, np.float64)), np.eye(3)])


def exp_so3(v):
    th = float(np.linalg.norm(v))
    if th < 1e-300:
        return np.eye(3)
    k = hat(np.asarray(v, np.float64) / th)
    return np.eye(3) + np.sin(th) * k + (1 - np.cos(th)) * (k @ k)


@dataclass
class Record:
    H: np.ndarray
    g: np.ndarray
    n_valid: int
    sum_residual: float

    def add_scalar(self, R, p, grad_q, r):
        J = np.asarray(grad_q, np.float64) @ j_point(R, p)
        self.H += np.outer(J, J)
        self.g += J * r
        self.n_valid += 1
        self.sum_residual += r

    def add_vector(self, R, p, e, W, res):
        J = j_point(R, p)
        self.H += J.T @ W @ J
        self.g += J.T @ W @ e
        self.n_valid += 1
        self.sum_residual += res


def empty():
    return Record(np.zeros((6, 6)), np.zeros(6), 0, 0.0)


def ivox_record(ref, scan, T):
    """from ivox_ref.planar_pass(map, scan, T, ...)"""
    out, R = empty(), np.asarray(T, np.float64)[:3, :3]
    for i in np.nonzero(ref.valid)[0]:
        out.add_scalar(R, scan[i, :3].astype(np.float64), ref.J[i, 3:], float(ref.ad[i]))
    return out


def kd_record(ref, planar, corner, T):
    """from loam_kd_ref.kd_pass(...): both classes count (LoamFull's corner terms included)"""
    assert not ref.nan and not any(t.in_band for t in ref.terms), "a decision within rounding: pick another scene"
    out, R = empty(), np.asarray(T, np.float64)[:3, :3]
    for t in ref.terms:
        if not t.valid:
            continue
        src = corner if t.cls == "corner" else planar
        out.add_scalar(R, src[t.i, :3].astype(np.float64), t.J[3:], float(t.r))
    return out


def icp_record(ref, T):
    """from icp_ref.icp_pass(...): e = q - m, W = I, residual |e|"""
    out, R = empty(), np.asarray(T, np.float64)[:3, :3]
    for i, _, e in ref.J:
        out.add_vector(R, ref.src[i, :3].astype(np.float64), e, np.eye(3), float(np.linalg.norm(e)))
    return out


def ndt_record(ref, src, T):
    """from ndt_ref.ndt_pass(...) over the filtered source `src`: one term per accepted point-voxel pair, e = q - mu, W = the voxel's
    information, residual e^T W e"""
    out, R = empty(), np.asarray(T, np.float64)[:3, :3]
    for term in ref.terms:
        i, I, e = term[0], term[3], term[4]
        out.add_vector(R, src[i, :3].astype(np.float64), e, I, float(e @ I @ e))
    return out


def assert_record(rec, ref: Record, what=""):
    """The issue's tolerances: n_valid equal, H within 1e-9 |H|, g within 1e-9 |g| + 1e-12, sum_residual 1e-9 relative."""
    assert rec is not None, what
    assert rec["n_valid"] == ref.n_valid, (what, rec["n_valid"], ref.n_valid)
    nH, ng = np.abs(ref.H).max(), np.abs(ref.g).max()
    assert np.abs(rec["H"] - ref.H).max() <= 1e-9 * nH, (what, np.abs(rec["H"] - ref.H).max() / nH)
    assert np.abs(rec["g"] - ref.g).max() <= 1e-9 * ng + 1e-12, (what, np.abs(rec["g"] - ref.g).max(), ng)
    assert abs(rec["sum_residual"] - ref.sum_residual) <= 1e-9 * abs(ref.sum_residual) + 1e-300, what
