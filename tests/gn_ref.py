"""High-precision reference of one Gauss-Newton step of every plug-in: the 6x6 solve, the pose update and the stop rule (CPU only,
independent of the oracle and of the CUDA library; mpmath at 50 digits).

What is restated, from the published behaviour of Eigen 3.3.7 and the upstream lines:

* `fullpiv_qr_solve` is Eigen's FullPivHouseholderQR<Matrix6d>::compute + solve (loam_point_to_plane_ivox.h:167,
  loam_point_to_plane_kdtree.h:108, loam_full_kdtree.h:141): at step k the pivot is the entry of largest magnitude of the remaining
  corner, found in Eigen's column-major visiting order (first strictly larger wins); the factorisation stops early once that entry is
  `<= 6 eps * biggest` (isMuchSmallerThan with precision eps * 6, biggest = the largest entry of H); a Householder reflector
  (beta = -sign(c0) |column|, tau = (beta - c0) / beta; tau = 0 and beta = c0 when the tail is zero) is applied to the corner; rank
  is the count of |R_kk| > 6 eps * max|R_kk|; solve applies the reflectors to g, back-substitutes the leading rank x rank triangle
  and writes zeros to the columns the permutation dropped.
* `inverse_solve` and `determinant` are H.inverse() * g and H.determinant() (icp_optimized.h:129-133, incremental_ndt.h:311),
  exact.  `det_zero` says whether the device's `det == 0` is decided: yes for a structurally singular H (a zero row), no (det != 0)
  when H is numerically regular and |det| sits far above the double underflow, otherwise undecided.
* `so3_exp` is SO3Exp with its epsilon guard, identity unless |v| > eps (math_function.h:74-89).
* `step` is one iteration as upstream runs it, per plug-in (SURVEY.md section 8a):
    LOAM (ivox, kd-tree, LoamFull)  dx = [dtheta, dt], R <- Exp(dtheta) R, full-pivot QR, stop when (rn < rot && pn < pos) or
                                    (|rn - last_rot| < 1e-4 && |pn - last_pos| < 1e-4), last_* starting at 0
                                    (loam_point_to_plane_ivox.h:158-189), converged = n_valid >= 50 of the last iteration (:201-203);
    NDT                             n_valid < min_effective -> T = current iterate, return false (incremental_ndt.h:306-309); else
                                    dx = H^-1 g = [dtheta, dt], R <- R Exp(dtheta), stop when rn < rot && pn < pos; converged forced
                                    true after the loop (:325);
    ICP                             det(H) == 0 -> `continue` (pose unchanged, no stop); else dx = H^-1 g = [dt, dtheta],
                                    R <- R Exp(dtheta), stop and converged when rn < rot && pn < pos (icp_optimized.h:129-149);
  and every loop stops once it + 1 >= max_iterations.

Which solver the device runs is part of the reference: the register LDL^T fast path (solve6_spd) when every pivot exceeds
1e-8 * max diag(H), otherwise the pivoting solver of the plug-in.  The fast-path decision is predicted from the exact pivots.

Bounds.  A solve that is backward stable, (H + dH) x^ = g with ||dH||_2 <= c u ||H||_2 (u = 2^-53), has
||x^ - x||_2 <= (c u k) / (1 - c u k) ||x||_2 with k = cond_2(H); every dx entry gets that normwise bound.  The constants:
  * LDL^T without pivoting of a symmetric positive definite H: |dH| <= gamma_{3n+1} |L||D||L^T| (Higham, Accuracy and Stability,
    Thm 10.4, stated there for Cholesky; LDL^T performs the same products) and || |L||D||L^T| ||_2 <= n ||H||_2, so c = n (3n + 1)
    = 114 for n = 6; C_SPD doubles it for the divisions LDL^T adds (228).
  * LU with partial or complete pivoting: |dH| <= gamma_{3n} |L||U| (Thm 9.4) and || |L||U| ||_inf <= (1 + 2 (n^2 - n) rho) ||H||_inf
    with growth rho <= 2^(n-1) (Lemma 9.6), and a factor n between the inf- and 2-norms: C_PIV = 3n (1 + 60 * 32) n = 207468.
  A bound that would exceed half of ||x|| is reported as infinite (no claim).  A diagonal H is solved exactly up to one rounding per
  entry on every path (no elimination touches it): its dx is fl(g_i / H_ii) with bound 0.

Decisions.  Every decision carries its margin in ulps of its threshold and the band, in the same ulps, that rounding of what it
compares can cover: `rn` vs rot_thres, `pn` vs pos_thres, |rn - last_rot| and |pn - last_pos| vs 1e-4 (band: the dx bound plus 3
ulps of a rounded norm, 0 when the norm is of a single exactly known entry), the fast-path pivots vs 1e-8 * dmax (band:
gamma_{3n+1} (|L||D||L^T|)_kk, 0 for a column no other column couples to), the full-pivot rank decisions vs 6 eps * max (band:
C_QR u ||H||_F (1 + ||R11^-1 R12||_F), 0 when every row and column left in the corner is uncoupled, where Householder steps copy
exact zeros), n_valid vs the gates (exact).  A decision inside its band is `decided = False`: reported, never asserted.
`replay` feeds a Match's logged H, g and n_valid through `step`."""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import mpmath
import numpy as np

mpmath.mp.dps = 50
mpf = mpmath.mpf

EPS = float(np.finfo(np.float64).eps)  # 2^-52
U = EPS / 2
N = 6
C_SPD = 2 * N * (3 * N + 1)
C_PIV = 3 * N * (1 + 2 * (N * N - N) * 2 ** (N - 1)) * N
C_QR = 2 * N * N
ICP, NDT, IVOX, KNN, FULL = 0, 1, 2, 3, 4
LOAM = (IVOX, KNN, FULL)
NAMES = {ICP: "icp", NDT: "ndt", IVOX: "ivox", KNN: "kd", FULL: "full"}


def ulp(x):
    x = abs(float(x))
    return math.ulp(x) if x > 0 else math.ulp(0.0)


# ---- H / g from the reduced totals ---------------------------------------------------------------------------------------------------
def tri6(r, c):
    return r * 6 - (r * (r - 1)) // 2 + (c - r)


def unpack(tot):
    tot = np.asarray(tot, np.float64)
    H = np.zeros((6, 6))
    for r in range(6):
        for c in range(r, 6):
            H[r, c] = H[c, r] = tot[tri6(r, c)]
    return H, tot[21:27].copy(), int(math.floor(tot[27] + 0.5))


def pack(H, g, n_valid, sum_res=0.0, cand=0.0, hits=0.0):
    t = np.zeros(31)
    for r in range(6):
        for c in range(r, 6):
            t[tri6(r, c)] = H[r, c]
    t[21:27] = g
    t[27], t[28], t[29], t[30] = float(n_valid), sum_res, cand, hits
    return t


def uncoupled(H, idx):
    """No other row or column of H has a non-zero (or NaN) entry coupling it to an index of idx."""
    return all(all(H[i, j] == 0 and H[j, i] == 0 for j in range(6) if j != i) for i in idx)


def _mat(H):
    return mpmath.matrix([[mpf(float(v)) for v in row] for row in np.asarray(H)])


def cond2(H):
    """2-norm condition number of a symmetric H (inf when singular)."""
    ev = mpmath.eigsy(_mat(H), eigvals_only=True)
    a = sorted(abs(e) for e in ev)
    return mpmath.inf if a[0] == 0 else a[-1] / a[0]


# ---- Eigen FullPivHouseholderQR, restated --------------------------------------------------------------------------------------------
@dataclass
class QR:
    x: list                 # basic solution (mpf)
    rank: int
    cols: list              # column permutation: cols[i] is the H column of factor column i
    nonzero_pivots: int     # where the factorisation stopped
    decisions: list         # (kind, k, margin, band): margin = value - threshold (stop: thr - corner), band its rounding band
    decided: bool
    tied: bool              # a pivot choice had an exact tie (Eigen and the device may resolve it differently)


def fullpiv_qr_solve(H, g):
    Hf = np.asarray(H, np.float64)
    A = _mat(Hf)
    b = mpmath.matrix([mpf(float(v)) for v in g])
    n = 6
    biggest0 = mpf(float(np.max(np.abs(Hf))))
    thr = mpf(float(np.max(np.abs(Hf))) * (6 * EPS))
    hnorm = mpmath.sqrt(sum(mpf(float(v)) ** 2 for v in Hf.ravel()))
    cols = list(range(n))
    rows_t, hc, ess = [], [], []
    nz = n
    decisions, tied = [], False
    for k in range(n):
        best, br, bc, tie = mpf(-1), k, k, False
        for j in range(k, n):       # column-major: the first strictly larger entry wins
            for i in range(k, n):
                v = abs(A[i, j])
                if v > best:
                    best, br, bc, tie = v, i, j, False
                elif v == best and v != 0:
                    tie = True
        tied = tied or tie
        exact_corner = uncoupled(Hf, [cols[j] for j in range(k, n)])
        band = mpf(0) if exact_corner else C_QR * U * hnorm * (1 + _r11inv_r12(A, k))
        decisions.append(("stop", k, thr - best, band))
        if best <= thr:
            nz = k
            break
        rows_t.append(br)
        if br != k:
            for j in range(n):
                A[k, j], A[br, j] = A[br, j], A[k, j]
        if bc != k:
            for i in range(n):
                A[i, k], A[i, bc] = A[i, bc], A[i, k]
            cols[k], cols[bc] = cols[bc], cols[k]
        c0 = A[k, k]
        tail = sum(A[i, k] ** 2 for i in range(k + 1, n))
        if tail <= mpf(2.2250738585072014e-308):
            tau, beta, v = mpf(0), c0, [mpf(0)] * (n - k - 1)
        else:
            beta = mpmath.sqrt(c0 ** 2 + tail)
            if c0 >= 0:
                beta = -beta
            v = [A[i, k] / (c0 - beta) for i in range(k + 1, n)]
            tau = (beta - c0) / beta
        A[k, k] = beta
        for i in range(k + 1, n):
            A[i, k] = mpf(0)
        if tau != 0:
            for j in range(k + 1, n):
                s = A[k, j] + sum(v[i - k - 1] * A[i, j] for i in range(k + 1, n))
                A[k, j] -= tau * s
                for i in range(k + 1, n):
                    A[i, j] -= tau * v[i - k - 1] * s
        hc.append(tau)
        ess.append(v)
    maxpiv = max([abs(A[i, i]) for i in range(nz)], default=mpf(0))
    rthr = maxpiv * 6 * EPS
    rank = 0
    for i in range(nz):
        exact = uncoupled(Hf, [cols[i]])
        band = mpf(0) if exact else C_QR * U * hnorm * (1 + _r11inv_r12(A, i))
        decisions.append(("rank", i, abs(A[i, i]) - rthr, band))
        rank += 1 if abs(A[i, i]) > rthr else 0
    x = [mpf(0)] * n
    if rank > 0:
        c = b.copy()
        for k in range(rank):
            c[k], c[rows_t[k]] = c[rows_t[k]], c[k]
            if hc[k] != 0:
                s = c[k] + sum(ess[k][i - k - 1] * c[i] for i in range(k + 1, n))
                c[k] -= hc[k] * s
                for i in range(k + 1, n):
                    c[i] -= hc[k] * ess[k][i - k - 1] * s
        y = [mpf(0)] * rank
        for i in range(rank - 1, -1, -1):
            s = c[i] - sum(A[i, j] * y[j] for j in range(i + 1, rank))
            y[i] = s / A[i, i]
        for i in range(rank):
            x[cols[i]] = y[i]
    decided = all(_decided(m, bd) for _, _, m, bd in decisions)
    return QR(x, rank, cols, nz, decisions, decided, tied)


def _r11inv_r12(A, k):
    """||R11^-1 R12||_F of the factor after k steps (how far a perturbation of H moves the remaining corner)."""
    if k == 0:
        return mpf(0)
    R11 = mpmath.matrix([[A[i, j] for j in range(k)] for i in range(k)])
    R12 = mpmath.matrix([[A[i, j] for j in range(k, 6)] for i in range(k)])
    try:
        M = mpmath.inverse(R11) * R12
    except ZeroDivisionError:
        return mpmath.inf
    return mpmath.mnorm(M, "f")


def _decided(margin, band):
    return band == 0 or abs(margin) > band


# ---- exact inverse / determinant -------------------------------------------------------------------------------------------------
def _fractions(H):
    from fractions import Fraction
    return [[Fraction(float(v)) for v in row] for row in np.asarray(H, np.float64)]


def _frac_eliminate(H, g=None):
    """Gaussian elimination in exact rational arithmetic (every double is a rational): (det, solution or None)."""
    from fractions import Fraction
    A = _fractions(H)
    b = [Fraction(float(v)) for v in g] if g is not None else [Fraction(0)] * 6
    det = Fraction(1)
    for k in range(6):
        p = next((i for i in range(k, 6) if A[i][k] != 0), None)
        if p is None:
            return Fraction(0), None
        if p != k:
            A[k], A[p] = A[p], A[k]
            b[k], b[p] = b[p], b[k]
            det = -det
        det *= A[k][k]
        for i in range(k + 1, 6):
            f = A[i][k] / A[k][k]
            if f:
                for j in range(k, 6):
                    A[i][j] -= f * A[k][j]
                b[i] -= f * b[k]
    x = [Fraction(0)] * 6
    for i in range(5, -1, -1):
        x[i] = (b[i] - sum(A[i][j] * x[j] for j in range(i + 1, 6))) / A[i][i]
    return det, x


def determinant(H):
    """det(H), exact (rational arithmetic), as an mpf."""
    d, _ = _frac_eliminate(H)
    return mpf(d.numerator) / d.denominator


def inverse_solve(H, g):
    """H^-1 g exactly; None when H is singular (Eigen's inverse() then holds inf / NaN)."""
    d, x = _frac_eliminate(H, g)
    if d == 0:
        return None
    return [mpf(v.numerator) / v.denominator for v in x]


def det_zero(H):
    """(is det(H) == 0 on the device, decided?) for the `det == 0` test: True decided for a structurally singular H (a zero row);
    False decided when H is numerically regular for the pivoting solver and |det| is far above the double underflow."""
    Hf = np.asarray(H, np.float64)
    if any(np.all(Hf[i] == 0) for i in range(6)):
        return True, True
    d = determinant(Hf)
    if d == 0:
        return True, False
    k = cond2(Hf)
    return False, bool(C_PIV * U * k < 0.5 and abs(d) > mpf(1e-290))


# ---- SO3Exp -----------------------------------------------------------------------------------------------------------------------
@dataclass
class Exp:
    R: mpmath.matrix
    applied: bool     # |v| > eps: Rodrigues, else identity
    margin_ulps: float
    band_ulps: float
    decided: bool


def _norm3_band(v):
    """Rounding band of the device's norm3 of exactly known doubles: 0 for at most one non-zero entry, else 3 ulps."""
    return 0.0 if sum(1 for a in v if a != 0) <= 1 else 3 * ulp(math.sqrt(sum(float(a) ** 2 for a in v)))


def so3_exp(v, v_err=0.0):
    """SO3Exp(v) exactly (v: floats or mpf); the guard decision is taken on the exact norm of v, with band v_err plus the rounding
    of the device's norm."""
    vm = [a if isinstance(a, mpmath.mpf) else mpf(float(a)) for a in v]
    th = mpmath.sqrt(sum(a * a for a in vm))
    band = float(v_err) + _norm3_band([float(a) for a in v])
    applied = th > EPS
    R = mpmath.eye(3)
    if applied:
        n = [a / th for a in vm]
        c, s = mpmath.cos(th), mpmath.sin(th)
        S = [[0, -n[2], n[1]], [n[2], 0, -n[0]], [-n[1], n[0], 0]]
        for i in range(3):
            for j in range(3):
                R[i, j] = c * (1 if i == j else 0) + (1 - c) * n[i] * n[j] + s * S[i][j]
    m = float((th - EPS) / ulp(EPS))
    b = band / ulp(EPS)
    return Exp(R, bool(applied), m, b, b == 0 or abs(m) > b)


# ---- one step ---------------------------------------------------------------------------------------------------------------------
@dataclass
class Decision:
    holds: bool
    margin_ulps: float   # (threshold - value) in ulps of the threshold: > 0 when `value < threshold` holds (gates: n_valid - min)
    band_ulps: float
    decided: bool


def less(value, thr, band):
    """`value < thr` with value known up to `band` (absolute)."""
    v, t = mpf(value) if not isinstance(value, mpmath.mpf) else value, mpf(float(thr))
    m = float((t - v) / ulp(thr)) if thr != 0 else float(t - v)
    b = float(band) / ulp(thr) if thr != 0 else float(band)
    return Decision(bool(v < t), m, b, b == 0 or abs(m) > b)


@dataclass
class Step:
    method: int
    path: str                 # "gate_fail" (NDT), "skip" (ICP det == 0), "update"
    spd: bool                 # the LDL^T fast path takes the system
    spd_decided: bool
    spd_margins: list         # per pivot: (pivot - tiny) / band
    solver: str               # "spd", "fullpiv", "lu"
    dx: list | None           # exact dx in the device's layout (mpf); None where upstream's inverse is singular
    dx_bound: np.ndarray      # per entry; inf: no claim
    dx_exact: np.ndarray | None  # the exact double the device computes (diagonal H), else None
    rank: int
    rank_decided: bool
    qr: QR | None
    R: mpmath.matrix | None = None
    t: list | None = None
    exp: Exp | None = None
    clauses: dict = field(default_factory=dict)   # name -> Decision
    stop: bool = False
    stop_decided: bool = True
    stop_by: str = ""         # "thresholds", "second", "cap", "gate", ""
    converged: int = -1       # -1: the step leaves the state's flag alone (ICP without a stop)
    failed: int = 0
    iter: int = 0
    n_valid: int = 0
    new_last: tuple = (0.0, 0.0)
    det_zero: tuple = (False, True)
    path_decided: bool = True  # False: whether ICP skips (det == 0) or NDT's LU meets an exact zero pivot is inside rounding

    def result_record(self, converged_state):
        """The 18 doubles the step writes when it stops: column-major pose, converged, iterations."""
        r = np.zeros(18)
        for c in range(3):
            for rr in range(3):
                r[c * 4 + rr] = float(self.R[rr, c])
        r[12:15] = [float(a) for a in self.t]
        r[15] = 1.0
        r[16] = 1.0 if converged_state > 0 else 0.0
        r[17] = float(self.iter)
        return r


def ldlt_pivots(H):
    """Exact LDL^T pivots in natural order and each one's rounding band gamma_{3n+1} (|L||D||L^T|)_kk (0 for an uncoupled column)."""
    Hf = np.asarray(H, np.float64)
    A = _mat(Hf)
    d, L = [], mpmath.zeros(6, 6)
    for k in range(6):
        s = A[k, k] - sum(L[k, j] ** 2 * d[j] for j in range(k))
        d.append(s)
        L[k, k] = 1
        for i in range(k + 1, 6):
            L[i, k] = (A[i, k] - sum(L[i, j] * L[k, j] * d[j] for j in range(k))) / s if s != 0 else mpf(0)
    gam = (3 * N + 1) * U / (1 - (3 * N + 1) * U)
    bands = []
    for k in range(6):
        if uncoupled(Hf, [k]):
            bands.append(mpf(0))
        else:
            bands.append(gam * sum(abs(L[k, j]) ** 2 * abs(d[j]) for j in range(k + 1)))
    return d, bands


def spd_decision(H):
    """(takes the fast path, decided, margins) for solve6_spd: dmax = max diag(H) > 0 and every pivot > fl(1e-8 * dmax)."""
    Hf = np.asarray(H, np.float64)
    if np.isnan(Hf).any():
        return False, True, []
    dmax = float(np.max(np.diag(Hf)))
    if not dmax > 0:
        return False, True, []
    tiny = 1e-8 * dmax
    d, bands = ldlt_pivots(Hf)
    margins, decided, ok = [], True, True
    for k in range(6):
        m = d[k] - tiny
        margins.append(float(m / bands[k]) if bands[k] != 0 else (math.inf if m > 0 else -math.inf if m < 0 else 0.0))
        if not _decided(m, bands[k]):
            decided = False
        if not d[k] > tiny:
            ok = False
            break  # the device returns at the first failing pivot: later ones are never looked at
    return ok, decided, margins


def _solve_bound(H, x, c, idx=None):
    """Normwise forward-error bound of a backward-stable solve with constant c, on the index set idx (default: all)."""
    idx = list(range(6)) if idx is None else idx
    if not idx:
        return np.zeros(6)
    sub = np.asarray(H)[np.ix_(idx, idx)]
    ev = mpmath.eigsy(_mat(sub), eigvals_only=True)
    a = sorted(abs(e) for e in ev)
    out = np.zeros(6)
    if a[0] == 0:
        out[idx] = math.inf
        return out
    k = a[-1] / a[0]
    r = c * U * k
    if r >= 0.5:
        out[idx] = math.inf
        return out
    xn = mpmath.sqrt(sum(x[i] ** 2 for i in idx))
    out[idx] = float(r / (1 - r) * xn) * (1 + 4 * EPS)
    return out


def _norm_and_band(v, bound):
    vm = [mpf(float(a)) if not isinstance(a, mpmath.mpf) else a for a in v]
    n = mpmath.sqrt(sum(a * a for a in vm))
    b = float(np.sqrt(np.sum(np.square(bound)))) if np.all(np.isfinite(bound)) else math.inf
    if b == 0:
        b = _norm3_band([float(a) for a in vm])
    else:
        b += 3 * ulp(float(n))
    return n, b


def _compose(method, R, t, dxv, dx_err):
    """Exact pose after the update with dx (mpf or float), per plug-in; returns (R, t, Exp)."""
    Rm = mpmath.matrix([[mpf(float(R[i][j])) for j in range(3)] for i in range(3)])
    tm = [mpf(float(a)) for a in t]
    if method == ICP:
        rot, pos, rot_err = dxv[3:6], dxv[0:3], dx_err[3:6]
    else:
        rot, pos, rot_err = dxv[0:3], dxv[3:6], dx_err[0:3]
    ex = so3_exp(rot, float(np.linalg.norm(rot_err)) if np.all(np.isfinite(rot_err)) else math.inf)
    Rn = ex.R * Rm if method in LOAM else Rm * ex.R
    tn = [tm[a] + (mpf(pos[a]) if isinstance(pos[a], float) else pos[a]) for a in range(3)]
    return Rn, tn, ex


def so3_exp_mp(v):
    th = mpmath.sqrt(sum(a * a for a in v))
    R = mpmath.eye(3)
    if th == 0:
        return R
    n = [a / th for a in v]
    c, s = mpmath.cos(th), mpmath.sin(th)
    S = [[0, -n[2], n[1]], [n[2], 0, -n[0]], [-n[1], n[0], 0]]
    for i in range(3):
        for j in range(3):
            R[i, j] = c * (1 if i == j else 0) + (1 - c) * n[i] * n[j] + s * S[i][j]
    return R


def step(method, state, tot, params, solver="device"):
    """One step.  state: R (3x3), t (3), last_rot, last_pos, iter; params: max_iterations, min_effective, rot_thres, pos_thres.
    solver="device": the fast path where solve6_spd takes the system; "oracle": always the pivoting solver (the CPU oracle)."""
    H, g, n_valid = unpack(tot)
    it = int(state["iter"])
    s = Step(method, "update", False, True, [], "", None, np.full(6, math.inf), None, 6, True, None, iter=it + 1, n_valid=n_valid)
    s.new_last = (float(state.get("last_rot", 0.0)), float(state.get("last_pos", 0.0)))
    if solver == "device":  # a property of H: the probe reports it on every path, the step consults it past the NDT gate
        s.spd, s.spd_decided, s.spd_margins = spd_decision(H)
    if method == NDT or method in LOAM:  # NDT's early-out, LOAM's `< 50` failure: exact integer comparisons
        mn = int(params["min_effective"])
        s.clauses["gate"] = Decision(n_valid >= mn, float(n_valid - mn), 0.0, True)
    if method == NDT and n_valid < int(params["min_effective"]):
        s.path, s.failed, s.converged, s.stop, s.stop_by = "gate_fail", 1, 0, True, "gate"
        s.dx, s.dx_bound, s.dx_exact = [mpf(0)] * 6, np.zeros(6), np.zeros(6)
        s.R = mpmath.matrix([[mpf(float(state["R"][i][j])) for j in range(3)] for i in range(3)])
        s.t = [mpf(float(a)) for a in state["t"]]
        return s
    nan = bool(np.isnan(H).any() or np.isnan(g).any())
    s.solver = "spd" if s.spd else ("fullpiv" if method in LOAM else "lu")
    diag = bool(np.all(H[~np.eye(6, dtype=bool)] == 0))
    if nan:
        s.stop_decided = False
        s.rank_decided = False
        return s
    if method in LOAM:
        if s.spd:
            x = inverse_solve(H, g)
            s.dx = x
            s.dx_bound = _solve_bound(H, x, C_SPD)
        else:
            q = fullpiv_qr_solve(H, g)
            s.qr, s.rank, s.rank_decided, s.dx = q, q.rank, q.decided, q.x
            kept = sorted(q.cols[:q.rank])
            s.dx_bound = _solve_bound(H, q.x, C_PIV, kept) if q.decided else np.full(6, math.inf)
    else:
        dz, dz_decided = det_zero(H) if not s.spd else (False, True)
        s.det_zero = (dz, dz_decided)
        x = inverse_solve(H, g)
        s.dx = x
        if x is None:
            s.rank, s.rank_decided = 5, dz_decided
        else:
            s.dx_bound = _solve_bound(H, x, C_SPD if s.spd else C_PIV)
        if method == ICP and dz:
            s.path, s.dx, s.dx_bound, s.dx_exact = "skip", [mpf(0)] * 6, np.zeros(6), np.zeros(6)
            if not dz_decided:  # the device's LU may or may not meet its exact zero pivot
                s.path_decided = s.stop_decided = False
        elif method == NDT and x is None:
            # upstream's inverse() of a singular H is inf / NaN; the device's LU leaves dx = 0 where it meets an exact zero pivot
            # (DESIGN.md section 8); a singular H without a zero row leaves that to rounding
            s.dx, s.dx_exact, s.dx_bound = [mpf(0)] * 6, np.zeros(6), np.zeros(6)
            if not dz_decided:
                s.dx_exact, s.dx_bound, s.path_decided = None, np.full(6, math.inf), False
    if diag and s.path == "update":
        ex = np.zeros(6)
        for i in range(6):
            keep = True
            if s.qr is not None:
                keep = i in s.qr.cols[:s.qr.rank]
            ex[i] = g[i] / H[i, i] if (keep and H[i, i] != 0) else 0.0
        if method not in LOAM and any(H[i, i] == 0 for i in range(6)):
            ex[:] = 0.0  # singular LU: dx untouched
        s.dx_exact = ex
        s.dx = [mpf(float(a)) for a in ex]
        s.dx_bound = np.zeros(6)
    if s.path == "skip":
        s.R = mpmath.matrix([[mpf(float(state["R"][i][j])) for j in range(3)] for i in range(3)])
        s.t = [mpf(float(a)) for a in state["t"]]
    else:
        dxv = [float(a) for a in s.dx] if s.dx_exact is not None else s.dx
        s.R, s.t, s.exp = _compose(method, state["R"], state["t"], dxv, s.dx_bound)
    rot, pos = (slice(3, 6), slice(0, 3)) if method == ICP else (slice(0, 3), slice(3, 6))
    if s.path == "update":
        rn, rb = _norm_and_band(s.dx[rot], s.dx_bound[rot])
        pn, pb = _norm_and_band(s.dx[pos], s.dx_bound[pos])
        c = s.clauses
        c["rot"] = less(rn, params["rot_thres"], rb)
        c["pos"] = less(pn, params["pos_thres"], pb)
        thr_stop = c["rot"].holds and c["pos"].holds
        thr_decided = (c["rot"].decided and c["pos"].decided) or (c["rot"].decided and not c["rot"].holds) or \
                      (c["pos"].decided and not c["pos"].holds)
        second, second_decided = False, True
        if method in LOAM:
            lr, lp = float(state.get("last_rot", 0.0)), float(state.get("last_pos", 0.0))
            if rb == 0 and pb == 0:  # norms known as the exact doubles the device computes: so are the differences
                rnd, pnd = float(rn), float(pn)
                c["drot"] = less(mpf(abs(rnd - lr)), 1e-4, 0.0)
                c["dpos"] = less(mpf(abs(pnd - lp)), 1e-4, 0.0)
                s.new_last = (rnd, pnd)
            else:
                c["drot"] = less(abs(rn - lr), 1e-4, rb + ulp(float(abs(rn - lr))))
                c["dpos"] = less(abs(pn - lp), 1e-4, pb + ulp(float(abs(pn - lp))))
                s.new_last = (float(rn), float(pn))
            second = c["drot"].holds and c["dpos"].holds
            second_decided = (c["drot"].decided and c["dpos"].decided) or (c["drot"].decided and not c["drot"].holds) or \
                             (c["dpos"].decided and not c["dpos"].holds)
        s.stop = thr_stop or second
        s.stop_decided = (thr_decided and second_decided) or (thr_decided and thr_stop) or (second_decided and second)
        s.stop_by = "thresholds" if thr_stop else ("second" if second else "")
        if method == ICP:
            s.converged = 1 if thr_stop else -1
        elif method == NDT:
            s.converged = 1
        else:
            s.converged = 1 if n_valid >= int(params["min_effective"]) else 0
    else:  # ICP skip
        s.converged = -1
    if it + 1 >= int(params["max_iterations"]):
        if not s.stop:
            s.stop_by = "cap"
        s.stop = True
        s.stop_decided = True
    return s


# ---- whole Matches ----------------------------------------------------------------------------------------------------------------
@dataclass
class Replay:
    steps: list          # Step per logged iteration, each at the pose composed from the logged dx before it
    dx: list             # reference dx per iteration
    T: np.ndarray        # pose composed from the logged dx (4x4 float64, from the exact composition)
    stop_at: int | None  # 1-based iteration at which the reference stops (None: it does not stop within the log)
    stop_decided: bool
    converged: bool | None
    by: str


def replay(method, T0, logs, params, solver="device"):
    """Feed a Match's logged H, g and n_valid through `step`; the pose advances by each iteration's LOGGED dx (what the device or
    the oracle applied), so the composition is checked on its own and the solve is checked iteration by iteration."""
    R = [[float(T0[i][j]) for j in range(3)] for i in range(3)]
    t = [float(T0[i][3]) for i in range(3)]
    Rm = mpmath.matrix(R)
    tm = [mpf(a) for a in t]
    last = (0.0, 0.0)
    steps, stop_at, decided, conv, by = [], None, True, 0, ""
    for i, lg in enumerate(logs):
        H = np.asarray(lg["H"], np.float64).reshape(6, 6)
        tot = pack(H, lg["g"], lg["n_valid"])
        st = dict(R=[[float(Rm[a, b]) for b in range(3)] for a in range(3)], t=[float(a) for a in tm], last_rot=last[0],
                  last_pos=last[1], iter=i)
        s = step(method, st, tot, params, solver)
        # the decisions of the loop are taken on the logged dx: re-evaluate the stop rule with it exactly
        logged = [float(a) for a in lg["dx"]]
        if s.path == "update":
            s2 = _decide_logged(method, s, logged, last, params, i)
            last = s2
        steps.append(s)
        if s.path != "gate_fail" and s.path != "skip":
            Rm, tm, _ = _compose_exact(method, Rm, tm, logged)
        if s.converged >= 0:
            conv = s.converged
        decided = decided and s.stop_decided
        if s.stop and stop_at is None:
            stop_at, by = i + 1, s.stop_by
            break
    T = np.eye(4)
    for a in range(3):
        for b in range(3):
            T[a, b] = float(Rm[a, b])
        T[a, 3] = float(tm[a])
    return Replay(steps, [s.dx for s in steps], T, stop_at, decided, bool(conv) if stop_at else None, by)


def _compose_exact(method, Rm, tm, dx):
    if method == ICP:
        rot, pos = dx[3:6], dx[0:3]
    else:
        rot, pos = dx[0:3], dx[3:6]
    th = math.sqrt(sum(a * a for a in rot))
    E = so3_exp_mp([mpf(a) for a in rot]) if th > EPS else mpmath.eye(3)
    Rn = E * Rm if method in LOAM else Rm * E
    return Rn, [tm[a] + mpf(pos[a]) for a in range(3)], E


def _decide_logged(method, s, dx, last, params, it):
    """Overwrite the stop decisions of s with the ones taken on the logged (exact double) dx; returns the new last norms."""
    rot, pos = (dx[3:6], dx[0:3]) if method == ICP else (dx[0:3], dx[3:6])
    rn, pn = mpmath.sqrt(sum(mpf(a) ** 2 for a in rot)), mpmath.sqrt(sum(mpf(a) ** 2 for a in pos))
    rb, pb = _norm3_band(rot), _norm3_band(pos)
    c = s.clauses
    c["rot"] = less(rn, params["rot_thres"], rb)
    c["pos"] = less(pn, params["pos_thres"], pb)
    thr_stop = c["rot"].holds and c["pos"].holds
    thr_dec = (c["rot"].decided and c["pos"].decided) or (c["rot"].decided and not c["rot"].holds) or (c["pos"].decided and not c["pos"].holds)
    second, second_dec = False, True
    rnd, pnd = float(rn), float(pn)
    if method in LOAM:
        c["drot"] = less(abs(rn - last[0]), 1e-4, rb + ulp(abs(rnd - last[0])))
        c["dpos"] = less(abs(pn - last[1]), 1e-4, pb + ulp(abs(pnd - last[1])))
        second = c["drot"].holds and c["dpos"].holds
        second_dec = (c["drot"].decided and c["dpos"].decided) or (c["drot"].decided and not c["drot"].holds) or \
                     (c["dpos"].decided and not c["dpos"].holds)
    s.stop = thr_stop or second
    s.stop_decided = (thr_dec and second_dec) or (thr_dec and thr_stop) or (second_dec and second)
    s.stop_by = "thresholds" if thr_stop else ("second" if second else "")
    if method == ICP:
        s.converged = 1 if thr_stop else -1
    if it + 1 >= int(params["max_iterations"]):
        if not s.stop:
            s.stop_by = "cap"
        s.stop, s.stop_decided = True, True
    return (rnd, pnd)


def params_of(cfg, method=None):
    """The step parameters of an fls_config (LOAM plug-ins: 50 valid planar points)."""
    m = cfg.method if method is None else method
    return dict(max_iterations=cfg.max_iterations, min_effective=cfg.ndt_min_effective_pts if m == NDT else 50,
                rot_thres=cfg.rotation_converge_thres, pos_thres=cfg.position_converge_thres)


def pose_tol(s: Step, t):
    """Tolerance of a device pose against the exact one of step s: the dx bound carried through Exp and the update, plus the
    rounding of so3_exp (cos, sin, the normalisation) and of the 3x3 product, taken as 32 eps."""
    b = s.dx_bound
    rot = b[3:6] if s.method == ICP else b[0:3]
    pos = b[0:3] if s.method == ICP else b[3:6]
    if not (np.all(np.isfinite(rot)) and np.all(np.isfinite(pos))):
        return math.inf, math.inf
    rt = float(np.linalg.norm(rot)) + 32 * EPS
    tt = float(np.linalg.norm(pos)) + 4 * EPS * (1 + float(np.max(np.abs(t))))
    return rt, tt


def dx_errors(steps, logs):
    """Per iteration: (|logged dx - reference dx| per entry, the bound), for the iterations whose reference dx exists."""
    out = []
    for s, lg in zip(steps, logs):
        if s.dx is None or s.path == "gate_fail":
            continue
        err = np.array([abs(float(mpf(float(a)) - b)) for a, b in zip(lg["dx"], s.dx)])
        out.append((err, s.dx_bound))
    return out


def assert_replay(rep: Replay, logs, T, iterations, converged, tag=""):
    """A whole Match against its replay: every logged dx within its bound of the reference solve of the logged H and g, the returned
    pose equal to the pose composed from the logged dx to 1e-12, and the iteration count and converged flag equal to the
    reference's decisions where those are decided."""
    for i, (err, bound) in enumerate(dx_errors(rep.steps, logs)):
        assert np.all(err <= bound), (tag, i, err, bound)
    assert np.max(np.abs(np.asarray(T) - rep.T)) < 1e-12, (tag, np.asarray(T) - rep.T)
    if rep.stop_decided:
        assert rep.stop_at == iterations == len(logs), (tag, rep.stop_at, iterations, len(logs))
        assert rep.converged == bool(converged), (tag, rep.converged, converged)
