"""Plain-Python reference of IncrementalNDT (include/registration/incremental_ndt.h upstream), CPU only and independent of the
oracle and of the CUDA library (the PCL voxel filter is taken from orc.voxel_grid, which the GPU filter matches bit for bit).

`NdtRef` keeps the map exactly as upstream does, sequentially: an LRU list of VoxelData (emplace_front on creation, splice to the
front on a touch, pop_back once the list reaches `capacity`, :193-214), AddPoint counting points only before the first estimate
(:71-76) and UpdateVoxel with its first-scan, carry, first-estimate, running-merge, eigenvalue-clamp and freeze branches
(:130-179).  The merge's information matrix restates JacobiSVD as V diag(1/sigma) U^T (:166-177): for a PSD matrix U = V, except
where Eigen meets a negative diagonal and negates U's column — which only a smallest eigenvalue within rounding of zero can give.
Such voxels are flagged `undecidable` (the scenes must avoid them); an exactly zero variance (all points on z = const) is exact.

`ndt_pass` is iteration 0 of Match (:246-304): H, g and n_valid, with every gate's margin — how far q / voxel is from an integer,
chi from outlier_thres — and per-entry bounds on how far another correct fp64 evaluation may land."""
from __future__ import annotations

from collections import OrderedDict
from dataclasses import dataclass, field
from fractions import Fraction

import numpy as np

from oracle import pyoracle as orc

F32 = np.float32
EPS = float(np.finfo(np.float64).eps)
STENCIL7 = ((0, 0, 0), (-1, 0, 0), (1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, -1), (0, 0, 1))  # :122-127


def ndt_key(p, inv):
    """(p.cast<double>() * inv_voxel_size_).cast<int>() (:195, :256): the fp64 product, truncated toward zero [quirk 5]."""
    return tuple(int(float(x) * inv) for x in p)


@dataclass
class Voxel:
    pts: list = field(default_factory=list)  # points_ (fp64 triples)
    mu: np.ndarray = field(default_factory=lambda: np.zeros(3))
    sigma: np.ndarray = field(default_factory=lambda: np.zeros((3, 3)))
    info: np.ndarray = field(default_factory=lambda: np.zeros((3, 3)))
    estimated: bool = False
    num_points: int = 0
    n_total: int = 0          # every point that ever entered the voxel's estimates (drives the rounding bounds)
    scale: float = 0.0        # largest coordinate magnitude seen
    tol_mu: float = 0.0       # bound on |mu - mu_fp64 of any evaluation order|
    tol_info: float = 0.0     # the same for every entry of info
    undecidable: bool = False
    branch: str = ""          # last UpdateVoxel branch taken


def _mean_cov(pts):
    """ComputeMeanAndCov (:92-110): sequential sums, mean, covariance / (n - 1)."""
    n = len(pts)
    s = [0.0, 0.0, 0.0]
    for p in pts:
        for a in range(3):
            s[a] += p[a]
    mean = [s[a] / n for a in range(3)]
    c = [[0.0] * 3 for _ in range(3)]
    for p in pts:
        v = [p[a] - mean[a] for a in range(3)]
        for a in range(3):
            for b in range(3):
                c[a][b] += v[a] * v[b]
    return np.array(mean), np.array(c) / (n - 1)


def _eig_info(sigma):
    """V diag(1 / lambda') V^T with lambda' clamped to 1e-3 lambda_max (:166-177).  Returns (info, lam_sorted_desc, exact_zero_axes)."""
    zero_axes = [a for a in range(3) if np.all(sigma[a, :] == 0.0) and np.all(sigma[:, a] == 0.0)]
    lam, V = np.linalg.eigh(sigma)
    lam, V = lam[::-1].copy(), V[:, ::-1].copy()
    for a in zero_axes:  # an exactly zero row / column: eigenvalue exactly 0 along that axis
        k = int(np.argmax(np.abs(V[a, :])))
        lam[k] = 0.0
    lp = lam.copy()
    for k in (1, 2):
        if lp[k] < lp[0] * 1e-3:
            lp[k] = lp[0] * 1e-3
    return (V / lp) @ V.T, lam, zero_axes


class NdtRef:
    """IncrementalNDT's map: AddCloudToLocalMap and UpdateVoxel, sequential and in upstream's order."""

    def __init__(self, voxel_size=1.0, min_pts=5, max_pts=50, capacity=100000, leaf=0.2, localization=True):
        self.voxel, self.inv = float(voxel_size), 1.0 / float(voxel_size)
        self.min_pts, self.max_pts, self.capacity = min_pts, max_pts, capacity
        self.leaf, self.loc = float(leaf), localization
        self.first_scan = True
        self.data: OrderedDict = OrderedDict()  # last = front of upstream's list
        self.events: list = []                  # per call: dict of what happened (evictions, re-creations, branches)

    def add_cloud(self, cloud):
        cloud = orc.voxel_grid(np.asarray(cloud, F32), self.leaf)  # :186
        ev = dict(evicted=[], recreated=[], branches={}, created=0)
        evicted_now = set()
        active = []
        for p in cloud[:, :3].astype(np.float64):
            pe = (float(p[0]), float(p[1]), float(p[2]))
            key = ndt_key(pe, self.inv)
            v = self.data.get(key)
            if v is None:
                if key in evicted_now:
                    ev["recreated"].append(key)
                self.data[key] = Voxel(pts=[pe], num_points=1)
                ev["created"] += 1
                if len(self.data) >= self.capacity:  # :202-205
                    old, _ = self.data.popitem(last=False)
                    ev["evicted"].append(old)
                    evicted_now.add(old)
            else:
                v.pts.append(pe)
                if not v.estimated:
                    v.num_points += 1
                self.data.move_to_end(key)
            if key not in active:
                active.append(key)
        for key in active:
            v = self.data.get(key)
            if v is None:  # evicted later in the same call and not created again
                continue
            b = self._update(v)
            ev["branches"][b] = ev["branches"].get(b, 0) + 1
        self.first_scan = self.loc  # :222-226
        self.events.append(ev)
        return ev

    def _first_estimate(self, v):
        mean, cov = _mean_cov(v.pts)
        v.scale = max(v.scale, max(abs(x) for p in v.pts for x in p))
        v.n_total = len(v.pts)
        v.mu, v.sigma = mean, cov
        v.info = np.linalg.inv(cov + np.eye(3) * 1e-3)
        spread = max(abs(p[a] - mean[a]) for p in v.pts for a in range(3))
        n = len(v.pts)
        v.tol_mu = 4 * n * EPS * v.scale
        tol_sig = 8 * n * EPS * (spread * spread + spread * v.scale)
        lam_min = 1.0 / float(np.max(np.linalg.eigvalsh(v.info)))
        v.tol_info = 16 * tol_sig / lam_min ** 2 + 64 * EPS * float(np.max(np.abs(v.info))) * float(np.linalg.cond(cov + np.eye(3) * 1e-3))

    def _update(self, v: Voxel) -> str:
        if self.first_scan:  # :131-143
            if len(v.pts) > 1:
                self._first_estimate(v)
                v.branch = "first_scan"
            else:
                v.mu = np.array(v.pts[0])
                v.info = np.eye(3) * 1e2
                v.scale, v.n_total, v.tol_mu, v.tol_info = max(abs(x) for x in v.pts[0]), 1, 0.0, 0.0
                v.branch = "first_scan_single"
            v.estimated = True
            v.pts = []
            return v.branch
        if v.estimated and v.num_points > self.max_pts:  # :145-147
            v.branch = "frozen"
            return v.branch
        npts = len(v.pts)
        if not v.estimated and npts > self.min_pts:  # :149-153
            self._first_estimate(v)
            v.estimated = True
            v.pts = []
            v.branch = "estimate"
        elif v.estimated and npts > self.min_pts:  # :154-178
            cm, cv = _mean_cov(v.pts)
            m, n = v.num_points, npts  # UpdateMeanAndCov (:112-120)
            nm = (m * v.mu + n * cm) / (m + n)
            d0, d1 = v.mu - nm, cm - nm
            nv = (m * (v.sigma + np.outer(d0, d0)) + n * (cv + np.outer(d1, d1))) / (m + n)
            scale = max(v.scale, max(abs(x) for p in v.pts for x in p))
            spread = max(max(abs(p[a] - nm[a]) for p in v.pts for a in range(3)), float(np.max(np.abs(d0))), float(np.sqrt(np.max(np.abs(v.sigma)))))
            v.n_total += npts
            v.tol_mu = v.tol_mu + 4 * (npts + 4) * EPS * scale
            tol_sig = 8 * v.n_total * EPS * (spread * spread + spread * scale) + 4 * spread * v.tol_mu
            v.mu, v.sigma, v.scale = nm, nv, scale
            v.num_points += npts
            v.pts = []
            v.info, lam, zero_axes = _eig_info(nv)
            lp_min = max(lam[2], lam[0] * 1e-3)
            # the smallest eigenvalue is not provably of one sign unless it is exactly zero or clear of the rounding of sigma
            v.undecidable = len(zero_axes) == 0 and abs(lam[2]) <= 1e3 * (tol_sig + EPS * lam[0])
            v.tol_info = 16 * (tol_sig + 8 * EPS * lam[0]) / lp_min ** 2
            v.branch = "merge"
        else:
            v.branch = "carry"
        return v.branch

    # -- views ------------------------------------------------------------------------------------------------
    def frozen(self, v):
        return v.estimated and v.num_points > self.max_pts

    def dump(self):
        """Every voxel sorted by key, in the layout of fls_get_ndt_voxels (carry_count 0 for a frozen voxel: the GPU drops the points
        upstream keeps in points_ but never reads again)."""
        keys = sorted(self.data)
        out = dict(key=np.array(keys, np.int64).reshape(-1, 3), mu=np.zeros((len(keys), 3)), info=np.zeros((len(keys), 6)),
                   estimated=np.zeros(len(keys), np.int64), num_points=np.zeros(len(keys), np.int64), carry_count=np.zeros(len(keys), np.int64),
                   pending=np.zeros(len(keys), np.int64), tol_mu=np.zeros(len(keys)), tol_info=np.zeros(len(keys)),
                   undecidable=np.zeros(len(keys), bool))
        for i, k in enumerate(keys):
            v = self.data[k]
            out["estimated"][i] = v.estimated
            out["num_points"][i] = v.num_points
            out["pending"][i] = len(v.pts)
            out["carry_count"][i] = 0 if self.frozen(v) else len(v.pts)
            if v.estimated:
                I = v.info
                out["mu"][i] = v.mu
                out["info"][i] = [I[0, 0], 0.5 * (I[0, 1] + I[1, 0]), 0.5 * (I[0, 2] + I[2, 0]), I[1, 1], 0.5 * (I[1, 2] + I[2, 1]), I[2, 2]]
            out["tol_mu"][i], out["tol_info"][i], out["undecidable"][i] = v.tol_mu, v.tol_info, v.undecidable
        return out


def sym6_to_3x3(s):
    s = np.asarray(s)
    return np.array([[s[0], s[1], s[2]], [s[1], s[3], s[4]], [s[2], s[4], s[5]]])


def assert_dump_matches(got, ref, mu_factor=1.0):
    """A map dump (fls_get_ndt_voxels or the oracle's, both sorted by key) against NdtRef.dump(): keys and counters exact, mu and
    information within the reference's bounds."""
    assert not np.any(ref["undecidable"]), "scene holds a voxel whose smallest eigenvalue is within rounding of zero"
    assert np.array_equal(np.asarray(got["key"], np.int64), ref["key"])
    for f in ("estimated", "num_points", "carry_count"):
        assert np.array_equal(np.asarray(got[f], np.int64), ref[f]), (f, np.nonzero(np.asarray(got[f]) != ref[f])[0][:5])
    dmu = np.abs(np.asarray(got["mu"]) - ref["mu"])
    assert np.all(dmu <= ref["tol_mu"][:, None] * mu_factor), np.max(dmu / np.maximum(ref["tol_mu"][:, None], 1e-300))
    dinf = np.abs(np.asarray(got["info"]) - ref["info"])
    assert np.all(dinf <= ref["tol_info"][:, None]), np.max(dinf / np.maximum(ref["tol_info"][:, None], 1e-300))


def _exact(x):
    return Fraction(float(x))


def _chi_exact(e, I):
    """chi = e^T I e in exact arithmetic, and whether every partial product and sum of any evaluation order is an fp64 number
    (then every order, with or without FMA contraction, returns chi exactly)."""
    ok = True
    u = []
    for a in range(3):
        terms = [_exact(I[a, b]) * _exact(e[b]) for b in range(3)]
        s = sum(terms)
        ok &= all(Fraction(float(t)) == t for t in terms) and Fraction(float(s)) == s and Fraction(float(terms[0] + terms[1])) == terms[0] + terms[1]
        u.append(s)
    terms = [_exact(e[a]) * u[a] for a in range(3)]
    chi = sum(terms)
    ok &= all(Fraction(float(t)) == t for t in terms) and Fraction(float(chi)) == chi and Fraction(float(terms[0] + terms[1])) == terms[0] + terms[1]
    return chi, ok


@dataclass
class NdtPass:
    H: np.ndarray
    g: np.ndarray
    n_valid: int
    n_hits: int
    terms: list            # (point, stencil slot, J (3x6), info (3x3), e (3,)) of every accepted pair
    key_margin: np.ndarray  # (n,) smallest distance of q * inv to an integer over the axes (0: on a face)
    chi_margin: list        # (point, slot, chi - thres, bound on |chi - chi_fp64|) for every estimated voxel reached
    unestimated_hits: int   # hits on voxels that exist but carry no estimate
    tol_H: np.ndarray
    tol_g: np.ndarray


def ndt_pass(ref: NdtRef, scan, T, outlier_thres, leaf=None):
    """Iteration 0 of IncrementalNDT::Match (:246-304) at pose T (4x4) against the map of `ref`."""
    src = orc.voxel_grid(np.asarray(scan, F32), ref.leaf if leaf is None else leaf)  # :232
    T = np.asarray(T, np.float64)
    R, t = T[:3, :3], T[:3, 3]
    H, g = np.zeros((6, 6)), np.zeros(6)
    aH, ag = np.zeros((6, 6)), np.zeros(6)  # sums of |terms| and of the propagated map bounds
    terms, chi_m = [], []
    km = np.zeros(len(src))
    hits = unest = 0
    for i, sp in enumerate(src[:, :3].astype(np.float64)):
        q = np.array([((R[a, 0] * sp[0] + R[a, 1] * sp[1]) + R[a, 2] * sp[2]) + t[a] for a in range(3)])  # :255
        u = q * ref.inv
        km[i] = float(np.min(np.abs(u - np.round(u))))
        key = tuple(int(x) for x in u)  # :256 truncation
        hat = np.array([[0, -sp[2], sp[1]], [sp[2], 0, -sp[0]], [-sp[1], sp[0], 0]])
        J = np.hstack([-R @ hat, np.eye(3)])  # :273-275
        for s, o in enumerate(STENCIL7):
            v = ref.data.get((key[0] + o[0], key[1] + o[1], key[2] + o[2]))
            if v is None:
                continue
            hits += 1
            if not v.estimated:  # :263
                unest += 1
                continue
            e = q - v.mu
            I = v.info
            chi_x, exact = _chi_exact(e, I)
            ae = np.abs(e)
            tol_chi = 0.0 if (exact and v.tol_mu == 0 and v.tol_info == 0) else (
                16 * EPS * float(ae @ np.abs(I) @ ae) + 2 * float(np.abs(I @ e).sum()) * v.tol_mu + float(ae.sum()) ** 2 * v.tol_info
                + 8 * EPS * float(np.abs(q).max()) * float(np.abs(I @ e).sum()))
            chi = float(chi_x)
            chi_m.append((i, s, float(chi_x - Fraction(float(outlier_thres))), tol_chi))
            if np.isnan(chi) or chi > outlier_thres:  # :267-271
                continue
            H += J.T @ I @ J
            g += -J.T @ I @ e
            aJ, aI = np.abs(J), np.abs(I)
            aH += aJ.T @ aI @ aJ
            ag += aJ.T @ (aI @ ae)
            # the map's own bounds: info off by tol_info per entry, mu (hence e) off by tol_mu per axis
            H_map = aJ.T @ np.full((3, 3), v.tol_info) @ aJ
            g_map = aJ.T @ (np.full((3, 3), v.tol_info) @ ae + aI @ np.full(3, v.tol_mu + 4 * EPS * float(np.abs(q).max())))
            terms.append((i, s, J, I, e, H_map, g_map))
    n = len(terms)
    tol_H = 64 * (n + 8) * EPS * aH + sum((tt[5] for tt in terms), np.zeros((6, 6)))
    tol_g = 64 * (n + 8) * EPS * ag + sum((tt[6] for tt in terms), np.zeros(6))
    return NdtPass(H, g, n, hits, terms, km, chi_m, unest, tol_H, tol_g)


def assert_matches(H, g, n_valid, ref: NdtPass):
    assert int(n_valid) == ref.n_valid, (n_valid, ref.n_valid)
    H, g = np.asarray(H), np.asarray(g)
    assert np.all(np.abs(H - ref.H) <= ref.tol_H), np.max(np.abs(H - ref.H) / np.maximum(ref.tol_H, 1e-300))
    assert np.all(np.abs(g - ref.g) <= ref.tol_g), np.max(np.abs(g - ref.g) / np.maximum(ref.tol_g, 1e-300))


def assert_gates_clear(ref: NdtPass, factor=10.0):
    """Every chi gate is decided: chi is clear of outlier_thres by more than `factor` x its rounding bound, or it is computed
    exactly by every evaluation order (bound 0)."""
    for i, s, m, tol in ref.chi_margin:
        assert tol == 0.0 or abs(m) > factor * tol, (i, s, m, tol)


def assert_sensitive(ref: NdtPass, factor=100.0):
    """Dropping any single accepted (point, voxel) pair moves H or g by at least `factor` x the tolerance of that entry."""
    tH, tg = np.maximum(ref.tol_H, 1e-300), np.maximum(ref.tol_g, 1e-300)
    for tt in ref.terms:
        J, I, e = tt[2], tt[3], tt[4]
        move = max(np.max(np.abs(J.T @ I @ J) / tH), np.max(np.abs(J.T @ I @ e) / tg))
        assert move >= factor, (tt[0], tt[1], move)
