"""Adversarial LOAM-iVox scenes: small deterministic maps and scans that put the k-NN selection and the plane fit on their
edges.  Map point i carries intensity i, so a test can tell duplicate map points apart; the scans are given in the map
frame and matched at the identity pose, so every query is exactly the scan point.

Every scene lists the (ivox_resolution, ivox_max_range) pairs it runs with: (0.5, 5) takes the fast selection (every stencil
candidate is provably in range), (0.5, 1) and (1.5, 5) take the range-gated one."""
from __future__ import annotations

from dataclasses import dataclass, field
from fractions import Fraction

import numpy as np

from tests.ivox_ref import F32, dist2

FAST = (0.5, 5.0)
GATED = (0.5, 1.0)
GATED_COARSE = (1.5, 5.0)


@dataclass
class Scene:
    name: str
    map: np.ndarray   # (n, 4) float32 x, y, z, intensity = index
    scan: np.ndarray  # (m, 4) float32
    configs: list = field(default_factory=lambda: [FAST, GATED])


def _cloud(xyz):
    xyz = np.asarray(xyz, F32).reshape(-1, 3)
    out = np.zeros((len(xyz), 4), F32)
    out[:, :3] = xyz
    out[:, 3] = np.arange(len(xyz), dtype=F32)
    return out


def _scan(xyz):
    xyz = np.asarray(xyz, F32).reshape(-1, 3)
    out = np.zeros((len(xyz), 4), F32)
    out[:, :3] = xyz
    return out


def _patch(rng, centre, n, half, slope=(0.2, 0.1)):
    """n points of the plane z = cz + sx (x - cx) + sy (y - cy), x, y uniform within +-half of the centre."""
    c = np.asarray(centre, np.float64)
    xy = rng.uniform(-half, half, (n, 2))
    z = slope[0] * xy[:, 0] + slope[1] * xy[:, 1]
    return np.column_stack([c[0] + xy[:, 0], c[1] + xy[:, 1], c[2] + z])


def _above(rng, centre, n, half, lift, slope=(0.2, 0.1)):
    p = _patch(rng, centre, n, half, slope)
    p[:, 2] += lift * np.where(rng.random(n) < 0.5, -1.0, 1.0) * rng.uniform(0.3, 1.0, n)
    return p


def s1_dense_staged():
    """Runs of 65..352 candidates: past the 6-bit position of the quantised keys (exact comparator), still staged by v9."""
    rng = np.random.default_rng(11)
    mp = np.concatenate([_patch(rng, (5.0, 2.0, 1.0), 150, 0.2), _patch(rng, (5.0, 3.0, 1.0), 90, 0.2)])
    q = np.concatenate([_above(rng, (5.0, 2.0, 1.0), 40, 0.2, 0.05), _above(rng, (5.0, 3.0, 1.0), 20, 0.2, 0.05),
                        _above(rng, (5.0, 2.5, 1.0), 10, 0.2, 0.05)])
    return Scene("s1_dense_staged", _cloud(mp), _scan(q))


def s1_dense_global():
    """Runs longer than v9's stage buffer (352 records): read from global memory."""
    rng = np.random.default_rng(12)
    mp = _patch(rng, (-6.0, 3.0, 1.5), 420, 0.22)
    q = _above(rng, (-6.0, 3.0, 1.5), 40, 0.22, 0.05)
    return Scene("s1_dense_global", _cloud(mp), _scan(q))


def s1_mixed_warps():
    """80 separate patches of 40 points, one query each: every run fits the stage buffer alone, the 32 distinct runs of a
    chunk do not, so some lanes of a warp read staged runs and some read global memory."""
    rng = np.random.default_rng(13)
    mp, q = [], []
    for i in range(10):
        for j in range(8):
            c = (-9.0 + 2.0 * i, -7.0 + 2.0 * j, 0.5)
            p = _patch(rng, c, 40, 0.2)
            mp.append(p)
            q.append(p[-1:] + (0.01, -0.01, 0.04))  # the last candidate of the run is the nearest
    return Scene("s1_mixed_warps", _cloud(np.concatenate(mp)), _scan(np.concatenate(q)))


def s2_exact_ties():
    """A 0.125 m lattice on the plane z = 1 in shuffled insertion order, with duplicate points: queries at cell centres, edge
    centres and on lattice points have ranks 1/2 and 5/6 at exactly equal distances (every coordinate is a multiple of
    1/16, so every fp32 distance is exact)."""
    rng = np.random.default_rng(21)
    g = 2.0 + 0.125 * np.arange(16)
    X, Y = np.meshgrid(g, g, indexing="ij")
    lat = np.column_stack([X.ravel(), Y.ravel(), np.ones(X.size)])
    lat = lat[rng.permutation(len(lat))]
    dup = lat[rng.choice(len(lat), 24, replace=False)]
    mp = np.concatenate([lat, dup])
    q = []
    for i in range(1, 14, 3):
        for j in range(1, 14, 2):
            q.append((g[i] + 0.0625, g[j] + 0.0625, 1.03))  # cell centre: 4 at one distance
            q.append((g[i], g[j] + 0.0625, 1.0625))         # edge centre: 2, then 2 + 2
            q.append((g[i], g[j], 1.03125))                 # lattice point: 1 (2 with a duplicate), then 4
    return Scene("s2_exact_ties", _cloud(mp), _scan(q))


def s3_near_ties():
    """Near ties the 26-bit keys cannot order.  Around each of 20 queries, ranks 1/2 and ranks 5/6 are pairs whose fp32
    squared distances share their 26-bit prefix and differ by 1..8 ulps, the nearer one of each pair inserted (visited)
    later.  Around 8 more, ranks 1/2 are one ulp apart across a prefix boundary and the contracted (FMA) distance of the fast
    selection swaps them.  The 28 runs of 8..12 candidates fit v9's stage buffer together, so a batch takes the LDS hot path."""
    mp, q = [], []
    dz = 0.03
    for k in range(20):
        c = np.array([-8.0 + 2.0 * (k % 10), 4.0 + 2.0 * (k // 10), 0.6])
        qq = (c + (0.0, 0.0, dz)).astype(F32)
        m = 1 + k % 8

        def at(t, ang, lift=0.0):
            r = np.sqrt(float(t) - (dz - lift) ** 2)
            for a in ang + 0.05 * np.arange(20):  # the first direction along which a point at exactly `t` exists
                p = _on_sphere(qq, (c + (r * np.cos(a), r * np.sin(a), lift)).astype(F32), t)
                if p is not None:
                    return p
            raise AssertionError((qq, t))

        def plain(rr, ang):
            return c + (rr * np.cos(ang), rr * np.sin(ang), 0.0)

        def pair(nominal):
            bits = (np.float32(nominal).view(np.int32) & ~np.int32(63)) | np.int32(40)
            return bits.view(F32), (bits - np.int32(m)).view(F32)

        a_far, a_near = pair(0.0045)   # ranks 2 (visited first) and 1 (visited later)
        d_far, d_near = pair(0.0125)   # ranks 6 (visited first) and 5 (visited later)
        # the members of each pair sit 4 mm on either side of the plane of the others: which one is the nearest neighbour
        # (the anchor of the point-to-plane distance) and which one is in the 5-set (the fitted plane) shows in H and g
        pts = [at(a_far, 0.3), at(d_far, 1.9, -0.004), plain(0.085, 3.1), plain(0.095, 4.2)]
        pts += [c + (0.15 * np.cos(t), 0.15 * np.sin(t), 0.0) for t in np.linspace(0.5, 5.5, 6)]
        pts += [at(a_near, 2.5, 0.004), at(d_near, 5.0, 0.004)]
        mp.append(np.asarray(pts, np.float64))
        q.append(qq)
    rng = np.random.default_rng(32)
    for k in range(8):  # adjacent prefixes that the contracted distance swaps
        c = np.array([-8.0 + 2.0 * k, 8.0, 0.6])
        qq = (c + (0.0, 0.0, dz)).astype(F32)
        near, far = _fma_swapped_pair(rng, c, qq)
        # ranks 1/2 one ulp apart across a prefix boundary (reference: near first); the contracted distances are swapped
        # across the same boundary, so only the adjacent-prefix test of the fast selection sends the query to the exact path
        pts = [far, near] + [c + (0.09 * np.cos(t), 0.09 * np.sin(t), 0.0) for t in np.linspace(0.5, 5.5, 6)]
        mp.append(np.asarray(pts, np.float64))
        q.append(qq)
    return Scene("s3_near_ties", _cloud(np.concatenate(mp)), _scan(q))


def _on_sphere(q, p0, target, all_hits=False):
    """p0 moved by a few fp32 ulps per axis so that the reference's fp32 squared distance to q is exactly `target`."""
    q = np.asarray(q, F32)
    p0 = np.asarray(p0, F32)
    steps = np.arange(-48, 49)
    bx = p0[0] + steps.astype(F32) * np.spacing(p0[0])
    by = p0[1] + steps.astype(F32) * np.spacing(p0[1])
    X, Y = np.meshgrid(bx.astype(F32), by.astype(F32), indexing="ij")
    P = np.stack([X.ravel(), Y.ravel(), np.full(X.size, p0[2], F32)], 1)
    hit = np.nonzero(dist2(P, q) == F32(target))[0]
    if all_hits:
        return P[hit]
    return P[hit[len(hit) // 2]] if len(hit) else None


def _fma_swapped_pair(rng, c, q):
    """Two points around q on either side of the plane z = c_z (+-4 mm): `near` one fp32 ulp of squared distance below a
    26-bit prefix boundary, `far` just above it, whose contracted (FMA) distances fall on the other side of the boundary
    from each other's: the reference orders near first, the 26-bit keys of the contracted distances far first."""
    n = 200000
    ang = rng.uniform(0, 2 * np.pi, n)
    lift = np.where(np.arange(n) % 2 == 0, 0.004, -0.004)
    r = np.sqrt(0.0045 - (float(q[2]) - c[2] - lift) ** 2) + rng.uniform(-2e-6, 2e-6, n)  # squared distance ~0.0045
    P = np.stack([c[0] + r * np.cos(ang), c[1] + r * np.sin(ang), c[2] + lift], 1).astype(F32)
    bits = dist2(P, q).view(np.int32).astype(np.int64)
    ups, downs = {}, {}
    for i in np.nonzero((bits % 64 == 63) & (lift > 0))[0]:  # last ulp of prefix P, contracted into P + 1
        if int(np.asarray(fma_dist2(P[i], q)).view(np.int32)) == bits[i] + 1:
            ups.setdefault(bits[i] >> 6, i)
    for i in np.nonzero((bits % 64 == 0) & (lift < 0))[0]:  # first ulp of prefix P + 1, contracted into P
        if int(np.asarray(fma_dist2(P[i], q)).view(np.int32)) == bits[i] - 1:
            downs.setdefault((bits[i] >> 6) - 1, i)
    common = sorted(set(ups) & set(downs))
    assert common, (len(ups), len(downs))
    return P[ups[common[0]]], P[downs[common[0]]]


def _round32(x):
    """An exact rational rounded to the nearest fp32 (ties to even)."""
    f = np.float32(float(x))
    best = min((f, np.nextafter(f, F32(-np.inf)), np.nextafter(f, F32(np.inf))),
               key=lambda c: (abs(Fraction(float(c)) - x), int(np.asarray(c, F32).view(np.int32)) & 1))
    return F32(best)


def fma_dist2(p, q):
    """The fast selection's contracted squared distance fmaf(dz, dz, fmaf(dy, dy, dx * dx)) (fls_knn.cuh dist2_fast)."""
    d = np.asarray(p, F32)[:3] - np.asarray(q, F32)[:3]
    xx = d[0] * d[0]
    t = _round32(Fraction(float(d[1])) ** 2 + Fraction(float(xx)))
    return _round32(Fraction(float(d[2])) ** 2 + Fraction(float(t)))


def _range_cluster(q, direction, r, inner):
    """Candidates of query q: `inner` close ones, then three at fp32 squared distance r^2 - 1 ulp, r^2 and r^2 + 1 ulp along
    `direction` (the last two are out of range: the range test is strict)."""
    q = np.asarray(q, np.float64)
    u = np.asarray(direction, np.float64) / np.linalg.norm(direction)
    r2 = F32(r) * F32(r)
    pts = [q + np.array([0.05 + 0.03 * k, 0.02 * k, -0.01]) for k in range(inner)]
    for t in (np.nextafter(r2, F32(0)), r2, np.nextafter(r2, F32(np.inf))):
        p = _on_sphere(q, (q + r * u).astype(F32), t)
        assert p is not None, (q, t)
        pts.append(p)
    return pts


def s4_range_gate():
    """max_range = 1 at 0.5 m voxels: candidates one ulp below, exactly at and one ulp above max_range^2, reachable through
    the diagonal offsets of NEARBY18 / NEARBY26, behind 2, 4 or 5 closer candidates."""
    mp, q = [], []
    for k, inner in enumerate((2, 4, 5)):
        qq = (-0.24 + 3.0 * k, -0.24, 0.0)
        mp += _range_cluster(qq, (1.0, 1.0, 0.0), 1.0, inner)
        q.append(qq)
    return Scene("s4_range_gate", _cloud(np.array(mp)), _scan(q), configs=[GATED])


def s4_range_gate_exact():
    """max_range = 1 with a run of more than 64 candidates, so that both kernels settle it with their exact comparator
    (v9: knn5_exact_any): three close candidates and the boundary pair r^2 - 1 ulp (in range) and r^2 (out of range), all on
    the plane z = 0, then 70 candidates just beyond the range in the same voxel.  With a correct strict range test the
    query has 4 neighbours and no plane; counting the r^2 candidate in would give it 5 and a valid plane."""
    q = np.array([-0.24, -0.24, 0.03])
    qf = q.astype(F32)
    pts = [q + (0.05 + 0.03 * k, 0.02 * k, -0.03) for k in range(3)]
    r2 = F32(1.0)
    for t in (np.nextafter(r2, F32(0)), r2):
        for a in np.pi / 4 + 0.01 * np.arange(-10, 11):  # the first direction near the diagonal with a point at exactly t
            base = q + np.sqrt(1.0 - 0.03 ** 2) * np.array([np.cos(a), np.sin(a), 0.0])
            p = _on_sphere(qf, np.array([base[0], base[1], 0.0], F32), t)
            if p is not None:
                break
        assert p is not None
        pts.append(p)
    pts += [q + (0.74 + 0.002 * k, 0.73 - 0.001 * k, -0.03) for k in range(70)]
    return Scene("s4_range_gate_exact", _cloud(np.array(pts)), _scan([q]), configs=[GATED])


def s4_range_gate_coarse():
    """ivox_resolution = 1.5 with max_range = 5: the same boundary candidates, reachable only through NEARBY26's corners."""
    mp, q = [], []
    for k, inner in enumerate((2, 4, 5)):
        qq = (-0.7 + 9.0 * k, -0.7, -0.7)
        mp += _range_cluster(qq, (1.0, 1.0, 1.0), 5.0, inner)
        q.append(qq)
    return Scene("s4_range_gate_coarse", _cloud(np.array(mp)), _scan(q), configs=[GATED_COARSE])


def s5_voxel_edges():
    """Map points and queries exactly at (k + 0.5) * res, on both sides of the origin: Pos2Grid rounds half away from zero."""
    h = 0.25 * np.arange(-7, 8, 2)  # +-0.25, +-0.75, ... +-1.75
    X, Y = np.meshgrid(h, h, indexing="ij")
    top = np.column_stack([X.ravel(), Y.ravel(), np.full(X.size, 1.25)])
    bot = np.column_stack([X.ravel() + 5.0, Y.ravel(), np.full(X.size, -1.25)])
    q = []
    for x in (-1.25, -0.25, 0.75):
        for y in (-0.75, 0.25, 1.25):
            q += [(x, y, 1.25), (x, y, 1.27), (x + 5.0, y, -1.25), (x + 5.0, y, -1.23)]
    return Scene("s5_voxel_edges", _cloud(np.concatenate([top, bot])), _scan(q))


def s6_thin():
    """Groups of 1..4 points (fewer than 5 neighbours) and queries with an empty stencil."""
    mp, q = [], []
    for k in range(1, 5):
        c = np.array([3.0 * k, -3.0, 0.5])
        mp += [c + np.array([0.03 * m, -0.02 * m, 0.01 * m]) for m in range(k)]
        q.append(c + (0.02, 0.02, 0.0))
    q += [(40.0, 40.0, 1.0), (-3.0, 9.0, -2.0)]
    return Scene("s6_thin", _cloud(np.array(mp)), _scan(q))


def _plane_basis(nrm):
    n = np.asarray(nrm, np.float64) / np.linalg.norm(nrm)
    a = np.array([1.0, 0, 0]) if abs(n[0]) < 0.9 else np.array([0, 1.0, 0])
    u = np.cross(n, a)
    u /= np.linalg.norm(u)
    return n, u, np.cross(n, u)


def _worst_gate(P):
    A = np.asarray(P, np.float64)
    c = np.linalg.lstsq(A, -np.ones(len(A)), rcond=None)[0]
    return np.max(np.abs(A @ c + 1.0)) / np.linalg.norm(c)


def s7_plane_fit():
    """Isolated 5-point neighbourhoods, 2 m apart, one query each, for every branch of the plane fit: well conditioned;
    near-collinear (fails the 1e-7 LDL^T guard, takes QR); 2..8 km from the origin; an exactly zero column (the plane
    x = 0, points on an axis: the QR rank rule); the plane gate at 0.09 and 0.11; the near-point gate on both sides."""
    rng = np.random.default_rng(71)
    mp, q = [], []

    def add(P, qq):
        mp.extend(np.asarray(P, np.float64))
        q.append(qq)

    slot = iter(range(100))

    def centre():
        k = next(slot)
        return np.array([-9.0 + 2.0 * (k % 10), 8.0 + 2.0 * (k // 10), 1.0])

    for k in range(4):  # well conditioned
        c = centre()
        n, u, w = _plane_basis(rng.normal(size=3))
        P = [c + a * u + b * w for a, b in rng.uniform(-0.15, 0.15, (5, 2))]
        add(P, c + 0.04 * n)
    for k, off in enumerate((2e-5, 6e-5, 2e-4)):  # near-collinear
        c = centre()
        n, u, w = _plane_basis((0.1 * k, 0.3, 1.0))
        P = [c + t * u + off * s * w for t, s in zip((-0.15, -0.07, 0.0, 0.08, 0.15), (1, -1, 0.5, -0.5, 1))]
        add(P, c + 0.03 * n + 0.01 * u)
    for k, far in enumerate(((2000.0, 300.0, 40.0), (-3500.0, 4100.0, 12.0), (7900.0, -600.0, -30.0))):  # km from the origin
        for j in range(2):
            c = np.array(far) + (2.0 * j, 0.0, 0.0)
            n, u, w = _plane_basis(rng.normal(size=3))
            P = [c + a * u + b * w for a, b in rng.uniform(-0.2, 0.2, (5, 2))]
            add(P, c + 0.05 * n)
    c = centre()  # the plane x = 0: column 0 exactly zero
    P = [(0.0, c[1] + a, c[2] + b) for a, b in rng.uniform(-0.15, 0.15, (5, 2))]
    add(P, (0.03, c[1], c[2]))
    add([(7.0 + t, 0.0, 0.0) for t in (-0.04, -0.02, 0.0, 0.01, 0.03)], (7.01, 0.02, -0.01))  # the x axis: two zero columns
    add([(0.0, -7.0 + t, 0.0) for t in (-0.04, -0.02, 0.0, 0.01, 0.03)], (0.01, -6.99, 0.02))  # the y axis
    for target in (0.09, 0.11):  # the plane gate (thres 0.1): one point lifted until the worst |A c + 1| / |c| is the target
        c = centre()
        n, u, w = _plane_basis((0.2, -0.1, 1.0))
        base = [c + a * u + b * w for a, b in ((-0.15, -0.15), (0.15, -0.15), (-0.15, 0.15), (0.15, 0.15), (0.0, 0.0))]
        lo, hi = 0.0, 0.25
        for _ in range(60):
            h = 0.5 * (lo + hi)
            P = [p + (h * n if i == 4 else 0) for i, p in enumerate(base)]
            lo, hi = (h, hi) if _worst_gate(np.asarray(P, F32)) < target else (lo, h)
        add(P, c + 0.02 * n + 0.05 * u)
    for f in (0.9, 1.1):  # the near-point gate |p| >= 81 d^2 on both sides
        c = centre()
        n, u, w = _plane_basis((0.0, 0.0, 1.0))
        P = [c + a * u + b * w for a, b in rng.uniform(-0.15, 0.15, (5, 2))]
        qq = c + 0.0
        for _ in range(40):  # fixed point of 81 h^2 = f |q|
            h = np.sqrt(f * np.linalg.norm(qq) / 81.0)
            qq = c + h * n
        add(P, qq)
    return Scene("s7_plane_fit", _cloud(np.array(mp)), _scan(q))


def s7_rounding_rank():
    """Neighbourhoods of rank 1 or 2 in exact arithmetic, where the QR's remaining column after the reflections is fp64
    rounding noise of the order of the rank cut: five copies of one general point (40 of them, scattered over +-20 m), three
    copies of one point and two of another, dyadic off-axis lines (exactly collinear in fp32) and poles (x and y fixed).
    Which rank the QR settles on depends on that noise; the GPU and the oracle share the arithmetic that decides it.
    Scanned at the identity pose, one query 3..5 cm off each neighbourhood."""
    rng = np.random.default_rng(77)
    mp, q = [], []
    slots = [(x, y) for x in np.arange(-19.0, 20.0, 2.0) for y in (-17.0, -11.0, -5.0, 1.0, 7.0, 13.0)]
    slot = iter(slots)

    def off(p, k):
        d = rng.normal(size=3)
        return p + (0.03 + 0.02 * k / 40.0) * d / np.linalg.norm(d)

    for k in range(40):  # five copies of one general point
        x, y = next(slot)
        p = np.array([x, y, rng.uniform(-3, 3)]) + rng.uniform(-0.2, 0.2, 3)
        mp += [p] * 5
        q.append(off(p, k))
    for k in range(6):  # three copies of P, two of Q
        x, y = next(slot)
        P = np.array([x, y, rng.uniform(-3, 3)]) + rng.uniform(-0.2, 0.2, 3)
        Q = P + rng.uniform(-0.1, 0.1, 3)
        mp += [P, Q, P, Q, P]
        q.append(off(0.5 * (P + Q), k))
    for k in range(6):  # off-axis lines with dyadic points: exactly collinear
        x, y = next(slot)
        p0 = np.array([x + 0.125 * k, y - 0.0625, 1.25 - 0.375 * k])
        u = np.array([0.0625, -0.03125 * (k % 3 - 1), 0.015625 * (k + 1)])
        mp += [p0 + t * u for t in (-2, -1, 0, 1, 2)]
        q.append(off(p0, k))
    for k in range(6):  # poles
        x, y = next(slot)
        p0 = np.array([x + 0.0625 * k, y + 0.125, -1.0 + 0.5 * k])
        mp += [p0 + (0.0, 0.0, 0.046875 * t) for t in (-2, -1, 0, 1, 2)]
        q.append(p0 + (0.03, 0.02, 0.01))
    return Scene("s7_rounding_rank", _cloud(np.array(mp)), _scan(q))


def all_scenes():
    return [s1_dense_staged(), s1_dense_global(), s1_mixed_warps(), s2_exact_ties(), s3_near_ties(), s4_range_gate(),
            s4_range_gate_exact(), s4_range_gate_coarse(), s5_voxel_edges(), s6_thin(), s7_plane_fit()]
