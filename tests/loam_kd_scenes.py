"""Small seeded scenes at the edges of the kd-tree LOAM kernel (K5, fls_loam.cu): its exact grid 5-NN, LoamFull's search gate and
the corner term.  Each scene says which branch it targets; tests/test_oracle_loam_kd_edges.py proves from tests/loam_kd_ref.py that
it reaches it.  Planar neighbourhoods lie on noisy planes (+-0.03 m), so that any other choice of five neighbours moves the plane.

The kd-tree point-to-plane plug-in filters its map with map_cloud_filter_size before the search; every scene keeps each of its map
points alone in its leaf, so the filtered map is the scene's map."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from tests.ivox_ref import STENCIL, dist2
from tests.loam_kd_ref import kd_cell
from tests.ndt_icp_scenes import _cloud, _ulps, point_at_d2

F32 = np.float32
FAR = np.array([4999.0, -5003.0, 701.0])  # about 5 km from the origin


@dataclass
class KdScene:
    name: str
    full: bool                       # LoamFull (else LoamPointToPlaneKdtree)
    planar_map: np.ndarray
    planar: np.ndarray
    corner_map: np.ndarray | None = None
    corner: np.ndarray | None = None
    targets: str = ""
    T: np.ndarray = field(default_factory=lambda: np.eye(4))
    leaf: float = 0.45               # map_cloud_filter_size
    thres: float = 1.0               # point_search_thres (LoamFull)
    line_ratio: float = 3.0
    plane_thres: float = 0.1

    @property
    def cell(self):
        return kd_cell(self.full, self.leaf, self.thres)

    def config(self, max_iterations=1, **kw):
        from funny_lidar_slam_b200 import default_config
        from funny_lidar_slam_b200._abi import FLS_FLAG_ITER_LOG, FLS_LOAM_FULL, FLS_P2PLANE_KNN
        return default_config(FLS_LOAM_FULL if self.full else FLS_P2PLANE_KNN, flags=FLS_FLAG_ITER_LOG, max_iterations=max_iterations,
                              localization_mode=0 if self.full else 1, map_cloud_filter_size=self.leaf, corner_map_filter_size=self.leaf,
                              point_search_thres=self.thres, line_ratio_thres=self.line_ratio, point_to_planar_thres=self.plane_thres, **kw)

    def maps(self):
        return (self.planar_map, self.corner_map) if self.full else (self.planar_map, None)


def _centre(k, cell):
    """fp32 centre of key k (3 ints) of a grid of `cell`."""
    return ((np.asarray(k, np.float64) + 0.5) * float(cell)).astype(F32)


def _face(k, cell, ulps):
    """The fp32 coordinate `ulps` ulps above the first one whose key fl(x * fl(1 / cell)) reaches k: a few ulps inside the face."""
    inv = F32(1.0) / F32(cell)
    x = F32(k * float(cell))
    while np.floor(x * inv) >= k:
        x = _ulps(x, -1)
    while np.floor(x * inv) < k:
        x = _ulps(x, 1)
    return _ulps(x, ulps)


def _patch(rng, q, offsets, cell, dz=-0.1, noise=0.03):
    """Map points at q + offsets (in cells, in the xy plane), on the plane z = q_z + dz with +-noise."""
    off = np.asarray(offsets, np.float64) * float(cell)
    p = np.zeros((len(off), 3))
    p[:, :2] = q[:2].astype(np.float64) + off
    p[:, 2] = float(q[2]) + dz + rng.uniform(-noise, noise, len(off))
    return p


# ---- the ring search (kd-tree point-to-plane, 0.9 m cell) -----------------------------------------------------------
def kd_shells(offset=(0.0, 0.0, 0.0), name="kd_shells"):
    """One query per region, 30 m apart, at the centre of its cell, 0.1 m above a noisy patch.  Region S (1..6) holds seven points
    in Chebyshev ring S (nearest along +y and -y, which only the edge rows of a ring reach; three more along x, which every row
    reaches); region 7 holds them in rings 7-8 (only
    the full scan finds them).  Then queries a few ulps inside a cell face (x), an edge (x, y) and a corner (x, y, z), each with a
    27-cell 5th just outside the settle bound at 1.0015 cells and a ring-2 point at 1.001 cells that must replace it."""
    rng = np.random.default_rng(41)
    cell = kd_cell(False, 0.45)
    o = np.asarray(offset, np.float64)
    mp, sc = [], []
    for S in range(1, 8):
        k = np.floor((o + np.array([40.0 + 30.0 * S, 20.0, 3.0])) / float(cell)).astype(np.int64)
        q = _centre(k, cell)
        r = S - 0.3 if S < 7 else 7.2
        offs = [(0.0, r), (0.0, -(r + 0.02)), (r + 0.04, 0.0), (-(r + 0.06), 0.0), (0.55, r + 0.08), (-0.55, -(r + 0.1)), (0.55, r + 0.6),
                (r + 0.6, 0.0), (-(r + 0.6), 0.0), (r + 0.3, -0.6)]  # ranks 8-10 in the rows' end cells: a search that
        # skipped the edge rows would settle on them
        mp.append(_patch(rng, q, offs, cell))
        sc.append(q)
    for j, axes in enumerate(((0,), (0, 1), (0, 1, 2))):
        k = np.floor((o + np.array([300.0 + 30.0 * j, 20.0, 3.0])) / float(cell)).astype(np.int64)
        q = _centre(k, cell)
        for a in axes:
            q[a] = _face(int(k[a]), cell, 1)
        # four 27-cell points within 0.5 cells; x_a: the last fp32 x in key k - 2 (ring 2, about 1 + face cells away); x_b: the
        # 27-cell 5th one ulp farther on the +x side, just outside the settle bound, which x_a must replace
        p = _patch(rng, q, [(0.3, 0.3), (0.35, -0.35), (-0.3, 0.35), (-0.35, -0.3)], cell, dz=-0.02, noise=0.015)
        inv = F32(1.0) / F32(cell)
        xa = F32((int(k[0]) - 1) * float(cell))
        while np.floor(xa * inv) > k[0] - 2:
            xa = _ulps(xa, -1)
        xb = _ulps(F32(q[0] + (q[0] - xa)), 1)
        p = np.vstack([p, [[float(xa), float(q[1]), float(q[2])], [float(xb), float(q[1]), float(q[2])]]])
        mp.append(p)
        sc.append(q)
    return KdScene(name, False, _cloud(np.vstack(mp)), _cloud(np.array(sc)), targets="rings 1-6, the full scan, settle bound at faces",
                   plane_thres=0.3 if np.any(o) else 0.1)


def kd_shells_far():
    """The ring scene about 5 km out (the plane gate widened to 0.3 m: 5 km from the origin the fp64 plane fit is only known to
    ~1e-6 relative, which puts the default gate within rounding of the noisy patches)."""
    return kd_shells(offset=FAR, name="kd_shells_far_5km")


# ---- lanes and ties (0.8 m cell: leaf 0.1) --------------------------------------------------------------------------
def kd_lanes():
    """Query A: all five nearest in cell (0, -1, 0), which one lane of the 27-cell pass owns, and five farther points in cells of
    other lanes.  Query B: one point in each of the 26 neighbour cells (every lane has candidates), the five nearest in face
    cells 1-5 of the stencil, i.e. in five lanes."""
    rng = np.random.default_rng(42)
    cell = kd_cell(False, 0.1)
    mp, sc = [], []
    k = np.array([40, 25, 4])
    q = _centre(k, cell)
    own = [(-0.3, -0.6), (0.1, -0.62), (0.35, -0.7), (-0.1, -0.8), (0.2, -0.9), (-0.35, -0.95)]
    far = [(1.3, 0.2), (-1.35, 0.1), (0.2, 1.4), (1.2, 1.1), (-1.25, 1.2)]
    mp.append(_patch(rng, q, own + far, cell))
    sc.append(q)
    k = np.array([70, 25, 4])
    q = _centre(k, cell)
    pts = []
    for s, off in enumerate(STENCIL[1:], start=1):
        radius = 0.6 + 0.01 * s if s <= 6 else 0.95 + 0.01 * (s % 5)  # the six face cells nearest; inside their cells
        v = off / np.linalg.norm(off)
        pts.append(q.astype(np.float64) + v * radius * float(cell) + rng.uniform(-0.02, 0.02, 3))
    mp.append(np.array(pts))
    sc.append(q)
    return KdScene("kd_lanes", False, _cloud(np.vstack(mp)), _cloud(np.array(sc)), leaf=0.1, plane_thres=1e3,
                   targets="five nearest in one lane's cell; five nearest over five lanes")


def kd_ties():
    """A dyadic lattice (0.75 m) on the exact plane z = 3.5 and a query 0.25 m above the point (32, 48), which is a corner of the
    0.8 m search grid: four points tie at rank 1 in four cells, eight at rank 5, all on the plane (every choice gives the same
    term); off-plane points 2 % farther than the rank-5 tie."""
    h = np.arange(-3, 3) * 0.75 + 0.375
    lat = np.array([[32.0 + x, 48.0 + y, 3.5] for x in h for y in h], F32)
    q = np.array([32.0, 48.0, 3.75], F32)
    d5 = np.sort(np.sqrt(dist2(lat, q).astype(np.float64)))[4]
    off = np.array([[32.0 + 1.02 * d5, 48.0, 3.8], [32.0, 48.0 - 1.02 * d5, 3.2]])
    return KdScene("kd_ties", False, _cloud(np.vstack([lat, off])), _cloud(q[None]), leaf=0.1, targets="ties of 4 and 8 across lanes")


def kd_map_size(n):
    """A map of exactly n points (4, 5 or 6) on a noisy plane and three queries over it."""
    rng = np.random.default_rng(43 + n)
    base = np.array([30.0, 12.0, 2.0])
    offs = [(0.0, 0.0), (0.6, 0.1), (-0.1, 0.7), (-0.7, -0.2), (0.2, -0.8), (1.0, 1.0)][:n]
    mp = _patch(rng, base.astype(F32) + F32(0.1) * np.array([0, 0, 1], F32), offs, 1.0)
    sc = base + np.array([[0.1, 0.1, 0.05], [-0.2, 0.3, 0.08], [0.3, -0.3, 0.02]])
    return KdScene(f"kd_map{n}", False, _cloud(mp), _cloud(sc), targets=f"a map of {n} points")


# ---- LoamFull: the search gate --------------------------------------------------------------------------------------
def full_gate(thres, offset=(0.0, 0.0, 0.0), name=None):
    """Planar queries whose 5th neighbour lies at d2 = fp32(thres) exactly and one fp32 ulp either side (four nearer neighbours on a
    noisy patch; at the origin only), and queries a few ulps above the face x = k cell whose 5th lies 0.9999 sqrt(thres) away
    across that face (0.999 at 5 km)."""
    rng = np.random.default_rng(44)
    cell = kd_cell(True, thres=thres)
    r = float(np.sqrt(thres))
    o = np.asarray(offset, np.float64)
    mp, sc = [], []
    for j, k in enumerate((0, 1, -1, 0, 1, -1) if not np.any(o) else ()):  # near the origin, where fp32 can hit d2 exactly
        q = np.array([4.0 * j + 0.37, 0.41, 0.29], F32)
        near = _patch(rng, q, [(0.1, 0.1), (-0.15, 0.2), (0.2, -0.2), (-0.25, -0.1)], r, dz=-0.02, noise=0.01)
        fifth = point_at_d2(q, _ulps(F32(thres), k), axis=j % 2, sign=1.0 if j < 3 else -1.0)
        mp += [near, fifth[None].astype(np.float64)]
        sc.append(q)
    for j in range(3):
        kx = int(np.floor((o[0] + 100.0 + 8.0 * j) / float(cell)))
        q = (o + np.array([0.0, 12.0, 2.0])).astype(F32)
        q[0] = _face(kx, cell, 2 + j)
        near = _patch(rng, q, [(0.1, 0.1), (0.15, -0.2), (0.3, 0.05), (0.2, 0.25)], r, dz=-0.02, noise=0.01)
        nb = q.astype(np.float64).copy()
        nb[0] = float(F32(q[0] - F32(0.999 if np.any(o) else 0.9999) * F32(r)))  # 0.999 at 5 km, where an ulp is 5e-4 m
        mp += [near, nb[None]]
        sc.append(q)
    sc = np.array(sc)
    return KdScene(name or f"full_gate_{thres}", True, _cloud(np.vstack(mp)), _cloud(sc), corner_map=_cloud(np.vstack(mp)),
                   corner=_cloud(np.zeros((0, 3))), thres=thres, targets="d4 at thres and one ulp either side; 5th across a face")


# ---- LoamFull: the corner term --------------------------------------------------------------------------------------
def _corner_region(centre, pts):
    return np.asarray(centre, np.float64) + np.asarray(pts, np.float64)


def full_corners(offset=(0.0, 0.0, 0.0), name="full_corners"):
    """Corner neighbourhoods 6 m apart, each with its query: exactly collinear along (1, 2, 0) (lam1 = lam2 = 0); an isotropic
    tetrahedron with its centre; a square with its centre (lam0 = lam1 > lam2 = 0: the gate rejects, a gate on lam2 would not); the
    integer set with lam0 / lam1 = 3 exactly (in the fp64 rounding band) and copies with one coordinate 2 fp32 ulps either side
    (ratio 3 +- 1e-7: clear); a noisy general line.  Planar: two queries on a noisy patch."""
    rng = np.random.default_rng(45)
    o = np.asarray(offset, np.float64)
    ratio3 = np.array([(-3, -2), (-3, 2), (2, -1), (2, 0), (2, 1)], np.float64) * 0.125
    sets = [
        ("collinear", np.outer(np.arange(-2, 3), [0.125, 0.25, 0.0]), [0.05, -0.12, 0.2]),
        ("isotropic", np.array([[0, 0, 0], [1, 1, 1], [1, -1, -1], [-1, 1, -1], [-1, -1, 1]]) * 0.25, [0.1, 0.05, 0.02]),
        ("square", np.array([[0, 0, 0], [1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0]]) * 0.25, [0.05, 0.02, 0.2]),
        ("ratio3", np.column_stack([ratio3, np.zeros(5)]), [0.1, 0.1, 0.15]),
        ("ratio3_up", np.column_stack([ratio3, np.zeros(5)]), [0.1, 0.1, 0.15]),
        ("ratio3_down", np.column_stack([ratio3, np.zeros(5)]), [0.1, 0.1, 0.15]),
        ("line", np.outer(np.linspace(-0.4, 0.4, 5), [0.3, -0.5, 0.81]) + rng.normal(0, 0.01, (5, 3)), [0.12, 0.1, -0.05]),
    ]
    mp, sc = [], []
    for j, (nm, pts, dq) in enumerate(sets):
        c = (o + np.array([30.0 + 6.0 * j, -10.0, 2.0])).astype(F32).astype(np.float64)
        p = (c + pts).astype(F32)
        if nm in ("ratio3_up", "ratio3_down"):  # x of the point (-3, -2) * 0.125 moved 2 fp32 ulps outwards / inwards
            p[0, 0] = _ulps(p[0, 0], -2 if nm == "ratio3_up" else 2)
        mp.append(p.astype(np.float64))
        sc.append((c + np.asarray(dq)).astype(F32))
    pq = (o + np.array([30.0, 10.0, 2.0])).astype(F32)
    pm = _patch(rng, pq, [(0.1, 0.1), (-0.15, 0.2), (0.2, -0.2), (-0.25, -0.1), (0.3, 0.3), (-0.3, 0.25)], 1.0)
    planar = np.array([pq, pq + np.array([0.1, -0.05, 0.01], F32)])
    return KdScene(name, True, _cloud(pm), _cloud(planar), corner_map=_cloud(np.vstack(mp)), corner=_cloud(np.array(sc)),
                   targets="collinear, isotropic, lam0 = lam1 > lam2, ratio 3 in and out of the band, a general line")


def full_corners_far():
    """The corner scene about 5 km out: the covariance comes from deviations of 0.1-0.5 m around 5000 m."""
    return full_corners(offset=FAR, name="full_corners_far_5km")


def full_on_line():
    """A query exactly on an axis-aligned line through its five neighbours: d = 0 and upstream divides by it."""
    c = np.array([30.0, -10.0, 2.0])
    pts = c + np.outer(np.arange(-2, 3) * 0.125, [1.0, 0.0, 0.0])
    q = (c + np.array([0.3, 0.0, 0.0])).astype(F32)
    pq = np.array([30.0, 10.0, 2.0], F32)
    pm = _patch(np.random.default_rng(46), pq, [(0.1, 0.1), (-0.15, 0.2), (0.2, -0.2), (-0.25, -0.1), (0.3, 0.3)], 1.0)
    return KdScene("full_on_line", True, _cloud(pm), _cloud(pq[None]), corner_map=_cloud(pts), corner=_cloud(q[None]),
                   targets="d = 0 on the fitted line")


# ---- LoamFull: the stale records (iteration 1) ----------------------------------------------------------------------
def full_stale():
    """Iteration 0 moves the pose about 0.25 m along +x: plane pairs 8 m from the origin facing x want +0.24 and +0.26 m, pairs
    facing y and z want +-0.01 m, so every driver stays valid at iteration 1 with |d| ~ 0.01.  A corner point 0.5 m beyond the end
    of a line along x and a planar point 0.75 m beside a patch facing z, both on the +x side, are about 0.9 m from their fifth
    neighbour: valid at iteration 0, beyond sqrt(thres) once moved, so at iteration 1 both contribute their stored terms
    [quirk 1]."""
    rng = np.random.default_rng(47)
    mp, sc = [], []
    u = np.linspace(-1.2, 1.2, 9)
    gu, gv = (a.ravel() for a in np.meshgrid(u, u, indexing="ij"))
    for axis in range(3):
        for side, want in ((-1.0, 0.24 if axis == 0 else 0.01), (1.0, 0.26 if axis == 0 else -0.01)):
            a1, a2 = [b for b in range(3) if b != axis]
            P = np.zeros((len(gu), 3))
            P[:, axis], P[:, a1], P[:, a2] = side * 8.0, gu, gv
            mp.append(P)
            Q = np.zeros((6, 3))
            Q[:, axis], Q[:, a1], Q[:, a2] = side * 8.0 - want, rng.uniform(-0.8, 0.8, 6), rng.uniform(-0.8, 0.8, 6)
            sc.append(Q)
    # planar victim: a small noisy patch facing z; the query 0.75 m on its +x side, 0.01 m above it
    vp = np.array([3.0, 4.0, 3.0])
    patch = vp + np.array([[0.0, 0.0, 0.0], [0.1, 0.15, 0.0], [-0.12, 0.1, 0.0], [0.05, -0.15, 0.0], [0.12, -0.05, 0.0]])
    patch[:, 2] += rng.uniform(-0.01, 0.01, 5)
    mp.append(patch)
    sc.append((vp + np.array([0.75, 0.0, 0.01]))[None])
    # corner victim: a line along x from -0.2 to 0.2; the query 0.5 m beyond its +x end and 0.1 m off it
    vc = np.array([-3.0, -4.0, 3.0])
    line = vc + np.outer(np.linspace(-0.2, 0.2, 5), [1.0, 0.0, 0.0]) + rng.normal(0, 0.003, (5, 3))
    cq = (vc + np.array([0.7, 0.0, 0.1]))[None]
    return KdScene("full_stale", True, _cloud(np.vstack(mp)), _cloud(np.vstack(sc)), corner_map=_cloud(line), corner=_cloud(cq),
                   targets="a corner and a planar record reused at iteration 1")


def kd_scenes():
    return [kd_shells(), kd_shells_far(), kd_lanes(), kd_ties(), kd_map_size(4), kd_map_size(5), kd_map_size(6)]


def full_scenes():
    return [full_gate(1.0), full_gate(0.1), full_gate(1.0, offset=FAR, name="full_gate_far_5km"), full_corners(), full_corners_far(),
            full_on_line()]
