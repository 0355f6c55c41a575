"""Brute-force references of the LOAM-iVox k-NN and of one PlanerMatch + SumCoefficient pass (CPU only, independent of the
oracle and of the CUDA library).

`knn5` restates IVoxMap::GetClosestPoint (ivox_map.cpp:6-37, :43-66, :145-147 upstream) without any map structure: every
map point is keyed, the query's stencil is walked in the reference order and the candidates are ranked by
(fp32 squared distance, visit order).  `planar_pass` restates loam_point_to_plane_ivox.h:256-340 at a fixed pose with the
plane fit solved in 50-digit arithmetic, and reports how far each point is from the gates and how much fp64 rounding may
move its normal, so that a test can tell a wrong neighbour or a wrong normal from rounding."""
from __future__ import annotations

import math
from dataclasses import dataclass

import mpmath
import numpy as np

F32 = np.float32
EPS = float(np.finfo(np.float64).eps)

# ivox_map.cpp:43-66 upstream: CENTER, NEARBY6, NEARBY18, NEARBY26 are the first 1, 7, 19, 27 of this list
STENCIL = np.array([(0, 0, 0), (-1, 0, 0), (1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, -1), (0, 0, 1), (1, 1, 0), (-1, 1, 0), (1, -1, 0),
                    (-1, -1, 0), (1, 0, 1), (-1, 0, 1), (1, 0, -1), (-1, 0, -1), (0, 1, 1), (0, -1, 1), (0, 1, -1), (0, -1, -1),
                    (1, 1, 1), (-1, 1, 1), (1, -1, 1), (1, 1, -1), (-1, -1, 1), (-1, 1, -1), (1, -1, -1), (-1, -1, -1)], np.int64)
STENCIL_LEN = (1, 7, 19, 27)


def voxel_key(xyz, res):
    """Pos2Grid: the fp32 product p * (1 / res) rounded half away from zero (std::round), per axis."""
    inv = F32(1.0) / F32(res)
    v = (np.asarray(xyz, F32) * inv).astype(np.float64)  # the product is rounded to fp32 first; the rounding below is exact
    return (np.sign(v) * np.floor(np.abs(v) + 0.5)).astype(np.int64)


def dist2(p, q):
    """fp32 squared distance in the order of pointcloud_utility.h:13-17 upstream: (dx^2 + dy^2) + dz^2, no contraction."""
    d = np.asarray(p, F32)[..., :3] - np.asarray(q, F32)[..., :3]
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def ulp_gap(a, b):
    """Distance in fp32 ulps between two non-negative floats."""
    return int(np.asarray(b, F32).view(np.int32)) - int(np.asarray(a, F32).view(np.int32))


@dataclass
class Knn:
    idx: np.ndarray    # (n, 5) map indices, nearest first, ascending (d2, visit order); -1 pads
    found: np.ndarray  # (n,) neighbours in range (<= 5)
    run: np.ndarray    # (n,) candidates in the query's stencil before the range test (the stencil run length)
    d2: np.ndarray     # (n, 6) fp32 squared distances of ranks 1..6; inf pads
    gap01: np.ndarray  # (n,) ulps between ranks 1 and 2 (-1: fewer than 2 in range)
    gap45: np.ndarray  # (n,) ulps between ranks 5 and 6 (-1: fewer than 6 in range)


def knn5(map_pts, q, res, nearby, max_range):
    """IVoxMap::GetClosestPoint(q, 5, max_range) for every query row of q, by brute force over map_pts (insertion order)."""
    map_pts = np.asarray(map_pts, F32)
    q = np.atleast_2d(np.asarray(q, F32))
    keys = voxel_key(map_pts[:, :3], res)
    buckets: dict = {}
    for i, k in enumerate(map(tuple, keys)):
        buckets.setdefault(k, []).append(i)
    r2 = F32(max_range) * F32(max_range)
    n = len(q)
    out = Knn(np.full((n, 5), -1, np.int64), np.zeros(n, np.int64), np.zeros(n, np.int64), np.full((n, 6), np.inf, F32),
              np.full(n, -1, np.int64), np.full(n, -1, np.int64))
    qkeys = voxel_key(q[:, :3], res)
    for r in range(n):
        cand = []
        for o in STENCIL[:STENCIL_LEN[nearby]]:
            cand.extend(buckets.get(tuple(qkeys[r] + o), ()))
        out.run[r] = len(cand)
        if not cand:
            continue
        cand = np.asarray(cand, np.int64)
        d = dist2(map_pts[cand], q[r])
        keep = np.nonzero(d < r2)[0]  # strict, voxel_grid_node.cpp:27 upstream
        order = keep[np.argsort(d[keep], kind="stable")]  # stable: equal distances keep visit order
        m = min(len(order), 5)
        out.found[r] = m
        out.idx[r, :m] = cand[order[:m]]
        ds = d[order[:6]]
        out.d2[r, :len(ds)] = ds
        if len(ds) >= 2:
            out.gap01[r] = ulp_gap(ds[0], ds[1])
        if len(ds) >= 6:
            out.gap45[r] = ulp_gap(ds[4], ds[5])
    return out


def transform(scan, T):
    """transform_point_d / xform_row_d: fp64 rows ((r0 x + r1 y) + r2 z) + t, rounded to fp32."""
    p = np.asarray(scan, F32)[:, :3].astype(np.float64)
    q = np.empty((len(p), 3), F32)
    for a in range(3):
        q[:, a] = (((T[a, 0] * p[:, 0] + T[a, 1] * p[:, 1]) + T[a, 2] * p[:, 2]) + T[a, 3]).astype(F32)
    return q


def _plane_mp(A):
    """min ||A c + 1|| in 50-digit arithmetic.  An exactly zero column gets c = 0 (the rank rule of colPivHouseholderQr, the
    same in orc_math.h and fls_plane.cuh: a zero remaining column is never pivoted and its unknown stays 0); the remaining
    columns are solved through the exact normal equations.  Returns (c as mpf list, rank, condition number of the
    column-normalised kept columns)."""
    keep = [j for j in range(3) if np.any(A[:, j] != 0.0)]
    c = [mpmath.mpf(0)] * 3
    if not keep:
        return c, 0, np.inf
    with mpmath.workdps(50):
        M = mpmath.matrix(len(keep), len(keep))
        rhs = mpmath.matrix(len(keep), 1)
        for a, ja in enumerate(keep):
            rhs[a] = -mpmath.fsum(mpmath.mpf(float(x)) for x in A[:, ja])
            for b, jb in enumerate(keep):
                M[a, b] = mpmath.fsum(mpmath.mpf(float(x)) * mpmath.mpf(float(y)) for x, y in zip(A[:, ja], A[:, jb]))
        sol = mpmath.lu_solve(M, rhs)
        for a, ja in enumerate(keep):
            c[ja] = sol[a]
    Ak = A[:, keep] / np.linalg.norm(A[:, keep], axis=0)
    s = np.linalg.svd(Ak, compute_uv=False)
    return c, len(keep), (s[0] / s[-1]) if s[-1] > 0 else np.inf


def colpiv_qr(A):
    """The 5x3 least-squares plane min ||A c + 1|| in the arithmetic the GPU's QR fallback (fls_plane.cuh plane_lstsq) and the
    oracle (orc_math.h lstsq_colpiv_qr) share, operation for operation in IEEE fp64 without contraction: column pivoting on
    norms recomputed per step, Eigen's reflector form, the rank cut (eps sqrt(max column norm^2) / 5)^2.  Where a remaining
    column is rounding noise the rank is decided by that noise, so this restatement is the only reference for it.
    Returns (c, rank)."""
    A = [[float(A[i][j]) for j in range(3)] for i in range(5)]
    b = [-1.0] * 5
    perm = [0, 1, 2]
    maxcn = 0.0
    for j in range(3):
        s = 0.0
        for i in range(5):
            s += A[i][j] * A[i][j]
        maxcn = max(maxcn, s)
    h = EPS * math.sqrt(maxcn) / 5.0
    thr = h * h
    rank = 3
    for k in range(3):
        piv, best = k, -1.0
        for j in range(k, 3):
            s = 0.0
            for i in range(k, 5):
                s += A[i][j] * A[i][j]
            if s > best:
                best, piv = s, j
        if best < thr or best == 0.0:
            rank = k
            break
        if piv != k:
            for i in range(5):
                A[i][k], A[i][piv] = A[i][piv], A[i][k]
            perm[k], perm[piv] = perm[piv], perm[k]
        alpha = A[k][k]
        tail = 0.0
        for i in range(k + 1, 5):
            tail += A[i][k] * A[i][k]
        beta, tau, v = alpha, 0.0, [0.0] * 5
        if tail != 0.0:
            beta = math.sqrt(alpha * alpha + tail)
            if alpha >= 0:
                beta = -beta
            for i in range(k + 1, 5):
                v[i] = A[i][k] / (alpha - beta)
            tau = (beta - alpha) / beta
        v[k] = 1.0
        A[k][k] = beta
        for i in range(k + 1, 5):
            A[i][k] = 0.0
        if tau != 0.0:
            for j in range(k + 1, 3):
                s = 0.0
                for i in range(k, 5):
                    s += v[i] * A[i][j]
                s *= tau
                for i in range(k, 5):
                    A[i][j] -= s * v[i]
            s = 0.0
            for i in range(k, 5):
                s += v[i] * b[i]
            s *= tau
            for i in range(k, 5):
                b[i] -= s * v[i]
    y = [0.0] * 3
    for i in range(rank - 1, -1, -1):
        s = b[i]
        for j in range(i + 1, rank):
            s -= A[i][j] * y[j]
        y[i] = s / A[i][i]
    c = [0.0] * 3
    for i in range(rank):
        c[perm[i]] = y[i]
    return np.array(c), rank


LDLT_GUARD = 1e-7  # fls_plane.cuh: the normal equations are solved by LDL^T while both Schur complements keep this share


def ldlt_share(A):
    """The smaller of the two Schur-complement shares the GPU's LDL^T fast path measures (fls_plane.cuh, same fp64 operations;
    the device may contract them to FMAs, so only a share well away from LDLT_GUARD predicts the path).  0: sxx == 0."""
    x, y, z = (A[:, k].astype(np.float64) for k in range(3))
    sxx, sxy, sxz, syy, syz, szz = (float(np.sum(u * v)) for u, v in ((x, x), (x, y), (x, z), (y, y), (y, z), (z, z)))
    if not sxx > 0.0:
        return 0.0
    l10, l20 = sxy / sxx, sxz / sxx
    d1 = syy - l10 * sxy
    e = syz - l10 * sxz
    t2 = szz - l20 * sxz
    if not d1 > 0.0:
        return 0.0
    l21 = e / d1
    den = max(szz, abs(l21 * e))
    return min(d1 / syy, (t2 - l21 * e) / den) if den > 0.0 else 0.0


def normal_error_bound(cond, rho, share):
    """Relative error the fp64 plane fit may carry on a neighbourhood of column-normalised condition number `cond` and relative
    least-squares residual `rho`.  Householder QR (the oracle; the GPU's fallback) is backward stable: cond * eps +
    cond^2 * eps * rho.  The normal equations (the GPU's LDL^T path, taken while the Schur share exceeds LDLT_GUARD) lose
    cond^2 * eps.  Only a share below the guard by more than 10x is certain to take QR; any other may take LDL^T."""
    qr = 64.0 * EPS * (cond + cond * cond * rho)
    if share < 0.1 * LDLT_GUARD:
        return qr
    return max(qr, 64.0 * EPS * cond * cond)


@dataclass
class PlaneTerm:
    """One point's PlanerMatch term (J, |d|), its gate margins and the bounds dJ, dad on how far fp64 may move J and |d|."""
    valid: bool
    J: np.ndarray          # (6,) 0 unless valid
    ad: float
    plane_margin: float    # thres - max_j |A_j c + 1| / |c|   (> 0: the plane gate passes; nan: |c| = 0)
    near_margin: float     # (|p| - 81 d^2) / |p|             (>= 0: the near-point gate passes; nan: not reached)
    normal_err: float      # bound on the relative error of the fp64 normal (normal_error_bound)
    rank: int
    scale: float           # largest coordinate magnitude of the neighbourhood
    dJ: np.ndarray         # (6,)
    dad: float


def plane_term(A, q, ps, R, plane_thres, qr_rule=False):
    """The plane term shared by every LOAM plug-in (loam_point_to_plane_ivox.h:275-321 == loam_point_to_plane_kdtree.h:226-269 ==
    loam_full_kdtree.h:295-342 upstream) for the five fp32 neighbours A (nearest first), the transformed fp32 query q, the body-frame
    point ps and the rotation R, with the plane solved in 50-digit arithmetic.  qr_rule: take the plane from colpiv_qr (the only
    reference for neighbourhoods whose rank is decided by rounding)."""
    A = np.asarray(A, np.float64)
    q = np.asarray(q, F32)
    if qr_rule:
        cq, rank = colpiv_qr(A)
        c, cond = [mpmath.mpf(float(x)) for x in cq], 0.0
    else:
        c, rank, cond = _plane_mp(A)
    t = PlaneTerm(False, np.zeros(6), 0.0, np.nan, np.nan, 0.0, rank, float(np.abs(A).max()), np.zeros(6), 0.0)
    with mpmath.workdps(50):
        cn = mpmath.sqrt(c[0] ** 2 + c[1] ** 2 + c[2] ** 2)
        if cn == 0:
            return t
        resid = mpmath.sqrt(mpmath.fsum((sum(mpmath.mpf(float(A[j, a])) * c[a] for a in range(3)) + 1) ** 2 for j in range(5)))
        rho = float(resid / (mpmath.mpf(float(np.linalg.norm(A))) * cn))
    t.normal_err = ne = normal_error_bound(cond, rho, ldlt_share(A))
    with mpmath.workdps(50):
        worst = max(abs(sum(mpmath.mpf(float(A[j, a])) * c[a] for a in range(3)) + 1) / cn for j in range(5))
        t.plane_margin = float(plane_thres - worst)
        if worst > plane_thres:
            return t
        nrm = [x / cn for x in c]
        d = sum((mpmath.mpf(float(q[a])) - mpmath.mpf(float(A[0, a]))) * nrm[a] for a in range(3))  # from the nearest [quirk 2]
        ps = np.asarray(ps, F32)[:3].astype(np.float64)
        pn = float(np.linalg.norm(ps))
        t.near_margin = float((mpmath.mpf(pn) - 81 * d * d) / pn) if pn > 0 else -np.inf
        if pn < 81 * float(d) ** 2:  # body-frame norm [quirk 3]
            return t
    nf = np.array([float(x) for x in nrm])
    s = 1.0 if d > 0 else -1.0
    Rp = np.asarray(R, np.float64) @ ps
    t.valid = True
    t.J = np.concatenate([np.cross(Rp, nf) * s, nf * s])
    t.ad = abs(float(d))
    t.dJ[:3] = (np.linalg.norm(Rp) + 1.0) * (ne + 4 * EPS)
    t.dJ[3:] = ne + 4 * EPS
    t.dad = float(np.linalg.norm(q.astype(np.float64) - A[0])) * ne + 4 * EPS * float(np.abs(q).max())
    return t


def sum_bounds(J, dJ, r, dr):
    """Per-entry bounds on H = sum J J^T and g = -sum J r of terms whose J and r are known to within dJ and dr (rows: terms),
    plus 1e-9 of sum |J_a J_b| for the summation itself.  Returns (tol_H, tol_g)."""
    aJ, ar = np.abs(np.asarray(J, np.float64)), np.abs(np.asarray(r, np.float64))
    dJ, dr = np.asarray(dJ, np.float64), np.asarray(dr, np.float64)
    tol_H = aJ.T @ dJ + dJ.T @ aJ + dJ.T @ dJ + 1e-9 * (aJ.T @ aJ)
    tol_g = dJ.T @ ar + aJ.T @ dr + dJ.T @ dr + 1e-9 * (aJ.T @ ar)
    return tol_H, tol_g


@dataclass
class PlanarPass:
    H: np.ndarray          # (6, 6) sum of J J^T over valid points
    g: np.ndarray          # (6,) sum of -J |d|
    n_valid: int
    valid: np.ndarray      # (n,) bool
    J: np.ndarray          # (n, 6) Jacobian rows (0 where not valid)
    ad: np.ndarray         # (n,) |d|
    plane_margin: np.ndarray  # (n,) thres - max_j |A_j c + 1| / |c|   (> 0: the plane gate passes; nan: < 5 neighbours)
    near_margin: np.ndarray   # (n,) (|p| - 81 d^2) / |p|             (>= 0: the near-point gate passes; nan: not reached)
    normal_err: np.ndarray    # (n,) bound on the relative error of the fp64 normal (normal_error_bound)
    rank: np.ndarray          # (n,) rank of the neighbourhood (-1: < 5 neighbours)
    scale: np.ndarray         # (n,) largest coordinate magnitude of the neighbourhood
    knn: Knn
    tol_H: np.ndarray      # (6, 6) bound on |H - H_fp64| per entry: the normal_err of every point + 1e-9 of sum |J_a J_b|
    tol_g: np.ndarray      # (6,) the same for g


def planar_pass(map_pts, scan, T, plane_thres=0.1, res=0.5, nearby=2, max_range=5.0, qr_rule=False):
    """One PlanerMatch + SumCoefficient pass of LoamPointToPlaneIVOX at pose T (4x4) with every valid flag cleared, i.e.
    iteration 0 of a Match (loam_point_to_plane_ivox.h:256-340 upstream).  qr_rule: take every plane from colpiv_qr (the
    only reference for neighbourhoods whose rank is decided by rounding; their QR takes no LDL^T fast path on the GPU)."""
    map_pts = np.asarray(map_pts, F32)
    scan = np.asarray(scan, F32)
    T = np.asarray(T, np.float64)
    n = len(scan)
    q = transform(scan, T)
    kn = knn5(map_pts, q, res, nearby, max_range)
    R = T[:3, :3]
    J = np.zeros((n, 6))
    ad = np.zeros(n)
    valid = np.zeros(n, bool)
    pm = np.full(n, np.nan)
    nm = np.full(n, np.nan)
    ne = np.zeros(n)
    rank = np.full(n, -1)
    scale = np.zeros(n)
    dJ = np.zeros((n, 6))
    dad = np.zeros(n)
    for i in range(n):
        if kn.found[i] < 5:  # :271-273
            continue
        t = plane_term(map_pts[kn.idx[i], :3], q[i], scan[i, :3], R, plane_thres, qr_rule)  # :274-321
        valid[i], J[i], ad[i], pm[i], nm[i], ne[i], rank[i], scale[i], dJ[i], dad[i] = (
            t.valid, t.J, t.ad, t.plane_margin, t.near_margin, t.normal_err, t.rank, t.scale, t.dJ, t.dad)
    H = np.einsum("ni,nj->ij", J[valid], J[valid])
    g = -(J[valid] * ad[valid, None]).sum(0)
    tol_H, tol_g = sum_bounds(J, dJ, ad, dad)
    return PlanarPass(H, g, int(valid.sum()), valid, J, ad, pm, nm, ne, rank, scale, kn, tol_H, tol_g)


def assert_sensitive(ref: PlanarPass, factor=100.0):
    """Removing any single valid point from the reference moves H by at least `factor` x the tolerance the comparison uses:
    a test with this tolerance tells one wrong neighbourhood from rounding."""
    if ref.n_valid == 0:
        return
    tol = np.maximum(ref.tol_H, 1e-300)
    for i in np.nonzero(ref.valid)[0]:
        move = np.max(np.abs(np.outer(ref.J[i], ref.J[i])) / tol)  # the entry of H that point i moves most, in tolerances
        assert move >= factor, (i, move)


def assert_matches(H, g, ref: PlanarPass):
    """H and g of a first pass within the per-entry bounds of the reference."""
    H, g = np.asarray(H), np.asarray(g)
    assert np.all(np.abs(H - ref.H) <= ref.tol_H), np.max(np.abs(H - ref.H) / np.maximum(ref.tol_H, 1e-300))
    assert np.all(np.abs(g - ref.g) <= ref.tol_g), np.max(np.abs(g - ref.g) / np.maximum(ref.tol_g, 1e-300))


def assert_gates_clear(ref: PlanarPass, factor=10.0):
    """Every point reaching a gate is clear of it by more than `factor` x what the fp64 rounding of its normal may move it."""
    for i in np.nonzero(~np.isnan(ref.plane_margin))[0]:
        slack = factor * (ref.normal_err[i] + 4 * EPS) * (ref.scale[i] + 1.0)
        assert abs(ref.plane_margin[i]) > slack, (i, ref.plane_margin[i], slack)
        if not np.isnan(ref.near_margin[i]):
            assert abs(ref.near_margin[i]) > slack, (i, ref.near_margin[i], slack)
