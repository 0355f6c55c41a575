"""Brute-force reference of the kd-tree LOAM plug-ins' first Gauss-Newton pass (LoamPointToPlaneKdtree, loam_point_to_plane_kdtree.h
:204-288, and LoamFull, loam_full_kdtree.h:211-372 upstream), CPU only and independent of the oracle and of the CUDA library.

`knn5` is the exact fp32 5-NN by brute force: every map point's squared distance in the order of pointcloud_utility.h:13-17, (dx^2 +
dy^2) + dz^2, ranked without any index.  Ties are reported, never resolved: the points strictly inside the 5th distance, the points at
it, and the points at the nearest distance (FLANN's order among equal distances is unspecified too).  A map of fewer than five points
answers nothing (upstream reads five indices the tree does not have; only the library's behaviour, no contribution, is pinned).

`search_gate` is LoamFull's `dist.back() > point_search_thres` (:227, :291): the fp32 5th distance widened to double against the
double threshold.  The decision is exact, so its margin is reported in fp32 ulps of the 5th distance from fp32(thres).  The library's
search also stops early once every unseen map point provably lies beyond the gate; with LoamFull's cell of 1.001 sqrt(thres) that
bound is passed at the first ring, where every point inside sqrt(thres) has been seen, so the early stop only saves work and no
scene can see it.

`corner_term` is CornerMatch's line (:231-270) in 50-digit arithmetic: the covariance of the five fp32 neighbours, its eigenvalues
and principal axis (mpmath.eigsy; the fp64 JacobiSVD of a PSD matrix has the same singular values and vectors), the margin of the
gate `lam0 <= line_ratio lam1` against the band fp64 rounding may move it (a decision inside the band is reported, not asserted),
the point-to-line distance d, J and per-entry bounds on both.  A query exactly on the line has d = 0 and upstream divides by it:
J is NaN.  `plane_term` is the planar term K1 shares (tests/ivox_ref.py).

`kd_pass` sums iteration 0 (or, given the terms of the iteration before, iteration 1 with the stale-record rule of [quirk 1] for both
classes): H, g, sum_residual and n_valid (planar points only: the `< 50` failure test counts nothing else), with per-entry bounds.

Geometry of the library's search grid (used to prove that a scene reaches a branch, never to compute a result): keys are
floor(fl(p * fl(1 / cell))) in fp32, `face` is the distance in cells from the query's key coordinate u = fl(q / cell) to the nearest
face of its cell, and after the rings of Chebyshev radius <= R have been scanned the search settles once the 5th distance is within
((R + face) cell 0.9995)^2.  Why the 0.9995 covers key rounding: a map point p outside those rings has a key coordinate at least
R + 1 from the query's, so fl(p_a / cell) - u_a >= R + 1 - frac(u_a) >= R + face along that axis.  Each of the two fp32 products
is off its exact value by at most half an ulp of a number below 2^13 when |p|, |q| < 2^13 cells (7.3 km at a 0.9 m cell), i.e.
by 2^-11 cells together, and fl(1 / cell) is off by 2^-24 relative.  So |p_a - q_a| >= (R + face - 2^-11)(1 - 2^-23) cell, which
exceeds 0.9995 (R + face) cell for every R >= 1 because 0.0005 (R + face) >= 0.0005 > 2^-11 = 0.000488.  The far scenes sit 5 km out,
where that slack is smallest; a point whose coordinates reach 2^14 cells would need a wider margin."""
from __future__ import annotations

import itertools
from dataclasses import dataclass, field

import mpmath
import numpy as np

from tests.ivox_ref import STENCIL, dist2, plane_term, sum_bounds, transform, ulp_gap

F32 = np.float32
EPS = float(np.finfo(np.float64).eps)
KMAX_SHELL = 6
SETTLE = 0.9995


# ---- exact 5-NN ------------------------------------------------------------------------------------------------------
@dataclass
class Knn5:
    found: np.ndarray   # (n,) bool: the map holds at least five points
    d2: np.ndarray      # (n, 6) fp32 squared distances of ranks 1..6 (inf pads)
    sure: list          # per query: map indices strictly inside the 5th distance, nearest first
    tied: list          # per query: map indices at the 5th distance
    first: list         # per query: map indices at the smallest distance
    gap45: np.ndarray   # (n,) ulps between ranks 5 and 6 (-1: no 6th point)

    def choices(self, i, cap=256):
        """Every (neighbours nearest first, ...) the exact search may return for query i: the sure points, then each choice among
        the tied ones; the nearest may be any point at the smallest distance."""
        need = 5 - len(self.sure[i])
        out = []
        for combo in itertools.combinations(self.tied[i], need):
            pts = list(self.sure[i]) + list(combo)
            for f in self.first[i]:
                if f in pts:
                    out.append([f] + [j for j in pts if j != f])
            if len(out) > cap:
                raise ValueError("too many tie resolutions")
        return out


def knn5(map_pts, q):
    m = np.asarray(map_pts, F32)[:, :3]
    q = np.atleast_2d(np.asarray(q, F32))[:, :3]
    n = len(q)
    out = Knn5(np.zeros(n, bool), np.full((n, 6), np.inf, F32), [[] for _ in range(n)], [[] for _ in range(n)], [[] for _ in range(n)],
               np.full(n, -1, np.int64))
    for i in range(n):
        d = dist2(m, q[i])
        order = np.argsort(d, kind="stable")
        out.d2[i, :min(6, len(m))] = d[order[:6]]
        if len(m) < 5:
            continue
        out.found[i] = True
        d5 = d[order[4]]
        out.sure[i] = [int(j) for j in order if d[j] < d5]
        out.tied[i] = [int(j) for j in order if d[j] == d5]
        out.first[i] = [int(j) for j in order if d[j] == d[order[0]]]
        if len(m) > 5:
            out.gap45[i] = ulp_gap(d5, d[order[5]])
    return out


def search_gate(d4, thres):
    """(passes, ulps of d4 from fp32(thres)): LoamFull rejects when double(d4) > thres (:227, :291)."""
    return not (float(d4) > float(thres)), ulp_gap(F32(thres), F32(d4))


# ---- search-grid geometry (classification only) ---------------------------------------------------------------------
def kd_cell(method_full, leaf=0.45, thres=1.0):
    """The library's cell: 1.001 sqrt(point_search_thres) for LoamFull, max(0.8, 2 map_cloud_filter_size) for the kd-tree
    point-to-plane plug-in (fls_api.cu, documented in DESIGN.md)."""
    if method_full:
        return F32(np.sqrt(thres) * 1.001)
    return max(F32(0.8), F32(2.0) * F32(leaf))


def grid_coords(p, cell):
    """(fp32 key coordinate u = fl(p * fl(1 / cell)), integer key, face distance in cells) per row."""
    inv = F32(1.0) / F32(cell)
    u = np.atleast_2d(np.asarray(p, F32))[:, :3] * inv
    k = np.floor(u)
    fr = u - k
    face = np.minimum(fr, F32(1.0) - fr).min(axis=1)
    return u, k.astype(np.int64), face


def shells(map_pts, q, idx, cell):
    """Chebyshev key distance from query q to each map point of idx."""
    _, kq, _ = grid_coords(q, cell)
    _, km, _ = grid_coords(np.asarray(map_pts, F32)[idx], cell)
    return np.abs(km - kq[0]).max(axis=1)


def stencil_lane(offset, lanes=8):
    """Lane of the 27-cell first pass that scans the cell at `offset` (cells go round-robin to the lanes in stencil order)."""
    s = int(np.nonzero((STENCIL == np.asarray(offset)).all(axis=1))[0][0])
    return s % lanes


@dataclass
class Reach:
    shell5: int        # Chebyshev ring of the farthest of the 5 nearest
    face: float        # query's distance to its cell's nearest face, in cells
    settle_ring: int   # smallest R >= 1 with sqrt(d5) <= (R + face) cell (exact); > KMAX_SHELL: only the full scan settles it
    r1_ratio: float    # 5th distance among the first 27 cells / ((1 + face) cell); inf: fewer than 5 there
    lanes: list        # first-pass lanes of the 5 nearest (-1: outside the 27 cells)


def reach(map_pts, q, idx, d5, cell):
    m = np.asarray(map_pts, F32)
    _, kq, face = grid_coords(q, cell)
    sh = shells(m, q, idx, cell)
    dist = np.sqrt(float(d5))
    R = max(1, int(np.ceil(dist / float(cell) - float(face[0]))))
    _, km, _ = grid_coords(m, cell)
    in27 = np.abs(km - kq[0]).max(axis=1) <= 1
    d27 = np.sort(dist2(m[in27], np.asarray(q, F32)))
    r1 = np.sqrt(float(d27[4])) / ((1.0 + float(face[0])) * float(cell)) if len(d27) >= 5 else np.inf
    lanes = [stencil_lane(km[j] - kq[0]) if sh[k] <= 1 else -1 for k, j in enumerate(idx)]
    return Reach(int(sh.max()), float(face[0]), R, r1, lanes)


# ---- corner term ----------------------------------------------------------------------------------------------------
@dataclass
class CornerTerm:
    valid: bool
    in_band: bool          # the line_ratio gate lies within fp64 rounding: decision reported, not asserted
    lam: tuple             # exact eigenvalues of the covariance, descending
    ratio_margin: float    # lam0 - line_ratio lam1 (exact); <= 0 rejects
    band: float            # how far fp64 rounding may move lam0 - line_ratio lam1
    J: np.ndarray
    d: float
    dJ: np.ndarray
    dd: float
    on_line: bool = False  # d == 0 exactly: upstream's J is 0 / 0


def _mp(x):
    return mpmath.mpf(float(x))


def corner_term(X, q, ps, R, line_ratio, q_ulps=0):
    """X: the five fp32 neighbours; q: the transformed fp32 query; ps: the body-frame point; R: the rotation of the pose.
    q_ulps: fp32 ulps by which q itself is uncertain (iteration 1 at a pose known to rounding)."""
    X = np.asarray(X, F32)[:, :3].astype(np.float64)
    q = np.asarray(q, F32)[:3]
    with mpmath.workdps(50):
        Xm = [[_mp(X[j, a]) for a in range(3)] for j in range(5)]
        c = [mpmath.fsum(Xm[j][a] for j in range(5)) / 5 for a in range(3)]
        dev = [[Xm[j][a] - c[a] for a in range(3)] for j in range(5)]
        S = mpmath.matrix(3, 3)
        for a in range(3):
            for b in range(3):
                S[a, b] = mpmath.fsum(dev[j][a] * dev[j][b] for j in range(5)) / 5
        E, Q = mpmath.eigsy(S)
        order = sorted(range(3), key=lambda k: -E[k])
        lam = tuple(E[k] for k in order)
        n = [Q[a, order[0]] for a in range(3)]
        margin = lam[0] - line_ratio * lam[1]
        # fp64: the centre is off by <= 4 eps max|X| per axis, each deviation by that plus eps |dev|; S_ab then by the bound below,
        # and the Jacobi sweeps add a backward error of a few eps |S|
        ec = 4 * EPS * float(np.abs(X).max())
        ad = np.abs(np.array([[float(v) for v in row] for row in dev]))
        dS = np.zeros((3, 3))
        for a in range(3):
            for b in range(3):
                e = (ec + EPS * ad[:, a]) * ad[:, b] + (ec + EPS * ad[:, b]) * ad[:, a] + (ec + EPS * ad[:, a]) * (ec + EPS * ad[:, b])
                dS[a, b] = 4 * (float(np.sum(e)) / 5 + 4 * EPS * float(np.sum(ad[:, a] * ad[:, b])) / 5)
        dlam = float(np.linalg.norm(dS)) + 64 * EPS * float(lam[0])
        band = (1 + line_ratio) * dlam
        t = CornerTerm(False, abs(float(margin)) <= band, tuple(float(x) for x in lam), float(margin), band, np.zeros(6), 0.0, np.zeros(6), 0.0)
        if margin <= 0 and not t.in_band:  # :249
            return t
        qm = [_mp(q[a]) for a in range(3)]
        v = [qm[a] - c[a] for a in range(3)]
        w = [v[1] * n[2] - v[2] * n[1], v[2] * n[0] - v[0] * n[2], v[0] * n[1] - v[1] * n[0]]  # (q - c) x n
        d = mpmath.sqrt(w[0] ** 2 + w[1] ** 2 + w[2] ** 2)  # :260
        t.valid = bool(margin > 0)  # in the band the term is computed for both decisions
        Rp = np.asarray(R, np.float64) @ np.asarray(ps, F32)[:3].astype(np.float64)
        if d == 0:  # (q - c) x n / 0 (:263)
            t.on_line = True
            t.J = np.full(6, np.nan)
            return t
        u = [x / d for x in w]
        nxu = [n[1] * u[2] - n[2] * u[1], n[2] * u[0] - n[0] * u[2], n[0] * u[1] - n[1] * u[0]]
        Rpm = [_mp(x) for x in Rp]
        head = [Rpm[1] * nxu[2] - Rpm[2] * nxu[1], Rpm[2] * nxu[0] - Rpm[0] * nxu[2], Rpm[0] * nxu[1] - Rpm[1] * nxu[0]]
        t.J = np.array([float(x) for x in head + nxu])
        t.d = float(d)
        gap = float(lam[0] - lam[1])
        en = 2 * dlam / gap + 16 * EPS  # the principal axis moves by at most ~|dS| / (lam0 - lam1)
        vq = float(mpmath.sqrt(v[0] ** 2 + v[1] ** 2 + v[2] ** 2))
        eq = q_ulps * float(np.sqrt(3.0)) * float(np.spacing(np.abs(q).max()))
        dw = np.sqrt(3.0) * ec + vq * en + 8 * EPS * vq + eq
        du = 2 * dw / float(d) + 8 * EPS
        t.dd = dw + 4 * EPS * float(d)
        t.dJ[3:] = en + du + 4 * EPS
        t.dJ[:3] = (float(np.linalg.norm(Rp)) + 1.0) * (en + du + 8 * EPS)
        return t


# ---- one pass --------------------------------------------------------------------------------------------------------
@dataclass
class Term:
    cls: str               # "corner" | "planar"
    i: int                 # index in its class
    valid: bool
    J: np.ndarray
    r: float
    dJ: np.ndarray
    dr: float
    stale: bool = False
    in_band: bool = False  # corner gate within rounding: both decisions allowed
    alt: object = None     # the term the other decision gives (None: no contribution)


@dataclass
class KdPass:
    H: np.ndarray
    g: np.ndarray
    sum_res: float
    n_valid: int           # planar points only
    n_corner: int
    tol_H: np.ndarray
    tol_g: np.ndarray
    tol_res: float
    terms: list            # every Term that contributes (and every in-band one)
    knn: dict              # class -> Knn5
    q: dict                # class -> transformed fp32 queries
    gate: dict             # class -> (n,) [passes, ulps]; LoamFull only
    corner: list = field(default_factory=list)  # CornerTerm per corner query (None: not reached)
    planar: list = field(default_factory=list)  # PlaneTerm per planar query (None: not reached)
    nan: bool = False      # a corner query on its line: H and g are NaN

    def alternatives(self):
        """(H, g, sum_res, n_valid) for every resolution of the in-band decisions."""
        band = [t for t in self.terms if t.in_band]
        for flips in itertools.product((False, True), repeat=len(band)):
            H, g, s = self.H.copy(), self.g.copy(), self.sum_res
            nv = self.n_valid
            for t, f in zip(band, flips):
                if not f:
                    continue
                for sign, tt in zip((-1.0, 1.0), t.alt):  # drop the summed decision, add the other
                    if tt is None:
                        continue
                    H += sign * np.outer(tt.J, tt.J)
                    g -= sign * tt.J * tt.r
                    s += sign * tt.r
            yield H, g, s, nv


def kd_pass(planar_map, corner_map, planar, corner, T, full, thres=1.0, line_ratio=3.0, plane_thres=0.1, prev=None, q_ulps=0):
    """Iteration 0 of Match at pose T (prev=None), or the iteration after `prev` at pose T: a point rejected now that was accepted
    in an earlier iteration of the same Match contributes its stored term again [quirk 1], in its own class."""
    T = np.asarray(T, np.float64)
    R = T[:3, :3]
    out = KdPass(np.zeros((6, 6)), np.zeros(6), 0.0, 0, 0, None, None, 0.0, [], {}, {}, {})
    classes = (("corner", corner_map, corner), ("planar", planar_map, planar)) if full else (("planar", planar_map, planar),)
    for cls, mp, src in classes:  # corners first (:347-372)
        src = np.zeros((0, 4), F32) if src is None else np.asarray(src, F32)
        q = transform(src, T) if len(src) else np.zeros((0, 3), F32)
        kn = knn5(mp, q) if len(src) else knn5(np.zeros((0, 4), F32), q)
        out.knn[cls], out.q[cls] = kn, q
        gates = []
        terms_cls = []
        for i in range(len(src)):
            term = None
            if kn.found[i]:
                ok, ulps = search_gate(kn.d2[i, 4], thres) if full else (True, 0)
                gates.append((ok, ulps))
                if ok:
                    alts = []
                    for nb in kn.choices(i):
                        A = np.asarray(mp, F32)[nb, :3]
                        if cls == "corner":
                            ct = corner_term(A, q[i], src[i, :3], R, line_ratio, q_ulps)
                            alts.append(ct)
                        else:
                            pt = plane_term(A.astype(np.float64), q[i], src[i, :3], R, plane_thres)
                            if q_ulps and pt.valid:
                                pt.dad += q_ulps * 3 * float(np.spacing(np.abs(q[i]).max()))
                            alts.append(pt)
                    term = alts[0]
                    for a in alts[1:]:  # a tie must not matter: every resolution gives the same term within its bounds
                        assert a.valid == term.valid, (cls, i)
                        if a.valid and not getattr(a, "on_line", False):
                            r0, r1 = (term.d, a.d) if cls == "corner" else (term.ad, a.ad)
                            dr0 = term.dd if cls == "corner" else term.dad
                            assert np.all(np.abs(a.J - term.J) <= 2 * term.dJ + 1e-12) and abs(r1 - r0) <= 2 * dr0 + 1e-12, (cls, i)
            else:
                gates.append((False, 0))
            (out.corner if cls == "corner" else out.planar).append(term)
            terms_cls.append(term)
        out.gate[cls] = gates
        for i, term in enumerate(terms_cls):
            now = None
            if term is not None and term.valid:
                r, dr = (term.d, term.dd) if cls == "corner" else (term.ad, term.dad)
                now = Term(cls, i, True, term.J, r, term.dJ, dr)
            band = cls == "corner" and term is not None and term.in_band
            old = None
            if prev is not None:
                old = next((t for t in prev.terms if t.cls == cls and t.i == i and t.valid), None)
            if band:  # both decisions possible: sum the exact one, keep the other as the alternative
                acc = Term(cls, i, True, term.J, term.d, term.dJ, term.dd)
                rej = Term(cls, i, True, old.J, old.r, old.dJ, old.dr, stale=True) if old is not None else None
                base, other = (acc, rej) if term.valid else (rej, acc)
                if base is not None:
                    out.terms.append(base)
                    _add(out, base)
                out.terms.append(Term(cls, i, False, np.zeros(6), 0.0, np.zeros(6), 0.0, in_band=True, alt=(base, other)))
                continue
            if now is not None:
                out.terms.append(now)
                _add(out, now)
            elif old is not None:  # stale record [quirk 1]
                st = Term(cls, i, True, old.J, old.r, old.dJ, old.dr, stale=True)
                out.terms.append(st)
                _add(out, st)
    rows = [t for t in out.terms if t.valid] + [t.alt[1] for t in out.terms if t.in_band and t.alt[1] is not None]
    J = np.array([t.J for t in rows]).reshape(-1, 6)
    out.nan = bool(np.any(np.isnan(J)))
    if out.nan:
        J = np.nan_to_num(J)
    out.tol_H, out.tol_g = sum_bounds(J, np.array([t.dJ for t in rows]).reshape(-1, 6), [t.r for t in rows], [t.dr for t in rows])
    out.tol_res = sum(t.dr for t in rows) + 1e-12 * sum(abs(t.r) for t in rows)
    return out


def next_pose(T, dx):
    """The LOAM update after an iteration (loam_full_kdtree.h:141-145): R <- Exp(dx[:3]) R, t <- t + dx[3:]."""
    T, dx = np.asarray(T, np.float64), np.asarray(dx, np.float64)
    th = float(np.linalg.norm(dx[:3]))
    K = np.zeros((3, 3))
    if th > 0:
        a = dx[:3] / th
        K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    E = np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K
    out = T.copy()
    out[:3, :3] = E @ T[:3, :3]
    out[:3, 3] = T[:3, 3] + dx[3:]
    return out


def _add(out, t):
    out.H += np.outer(t.J, t.J)
    out.g -= t.J * t.r
    out.sum_res += t.r
    if t.cls == "planar":
        out.n_valid += 1
    else:
        out.n_corner += 1


def assert_matches(lg, ref: KdPass):
    """H, g, sum_residual and n_valid of one logged iteration within the reference's bounds, for some resolution of the in-band
    corner decisions."""
    H, g, s, nv = np.asarray(lg["H"]), np.asarray(lg["g"]), float(lg["sum_residual"]), int(lg["n_valid"])
    assert nv == ref.n_valid, (nv, ref.n_valid)
    if ref.nan:
        assert np.all(np.isnan(H)) and np.all(np.isnan(g)), (H, g)
        assert abs(s - ref.sum_res) <= ref.tol_res, (s, ref.sum_res)
        return
    worst = []
    for aH, ag, ares, _ in ref.alternatives():
        eH = np.max(np.abs(H - aH) / np.maximum(ref.tol_H, 1e-300))
        eg = np.max(np.abs(g - ag) / np.maximum(ref.tol_g, 1e-300))
        er = abs(s - ares) / max(ref.tol_res, 1e-300)
        if eH <= 1 and eg <= 1 and er <= 1:
            return
        worst.append((eH, eg, er))
    raise AssertionError(f"no resolution within bounds (H, g, res in tolerances): {worst}")


def assert_sensitive(ref: KdPass, factor=100.0):
    """Dropping any one contributing term moves H or g by at least `factor` x the tolerance: one wrong neighbourhood, one wrong
    decision or one missing stale record is told apart from rounding."""
    if ref.nan:
        return
    tH, tg = np.maximum(ref.tol_H, 1e-300), np.maximum(ref.tol_g, 1e-300)
    for t in ref.terms:
        if not t.valid or t.in_band:
            continue
        move = max(np.max(np.abs(np.outer(t.J, t.J)) / tH), np.max(np.abs(t.J * t.r) / tg))
        assert move >= factor, (t.cls, t.i, move)


def assert_gates_clear(ref: KdPass, factor=10.0):
    """Every planar point reaching a plane gate is clear of it by more than `factor` x its rounding (tests/ivox_ref.py)."""
    for t in ref.planar:
        if t is None or np.isnan(t.plane_margin):
            continue
        slack = factor * (t.normal_err + 4 * EPS) * (t.scale + 1.0)
        assert abs(t.plane_margin) > slack, (t.plane_margin, slack)
        if not np.isnan(t.near_margin):
            assert abs(t.near_margin) > slack, (t.near_margin, slack)
