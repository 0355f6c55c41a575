"""Small deterministic scenes at the edges of the IncrementalNDT and IcpOptimized kernels (fls_ndt.cu, fls_icp.cu).  Map point i
carries intensity i, so a neighbour the GPU picks can be told apart from its duplicates.

NDT: clouds straddling the axis planes (truncated keys make key 0 twice as wide, [quirk 5]), queries a few ulps either side of voxel
faces at v = 1.0 and v = 0.3 (keys come from q * (1 / v); for fp32 coordinates no face query found makes that differ from
q / v, so the v = 0.3 scene checks the product's keys rather than a disagreement), single-point voxels (information 100 I), voxels that exist
without an estimate, chi exactly at outlier_thres and a few ulps either side, a copy about 5 km from the origin, and an open-loop
mapping stream in which every voxel goes carry -> estimate -> merge -> freeze, planar and linear voxels make the 1e-3 eigenvalue
clamp bite, and the map crosses ndt_capacity with a voxel evicted and created again in the same call.

ICP: nearest distances at max_corr and one fp32 ulp either side for max_corr in {0.25, 1, 2}, queries on faces and corners of the
search grid with the nearest point just inside sqrt(max_corr), exact ties on a lattice, a far guess without any correspondence, a
map of fewer than 27 occupied cells, and a fitness scene whose nearest point hides behind the 0.998-scaled cell bound."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from tests.ivox_ref import dist2

F32 = np.float32


def _cloud(xyz):
    xyz = np.asarray(xyz, F32).reshape(-1, 3)
    out = np.zeros((len(xyz), 4), F32)
    out[:, :3] = xyz
    out[:, 3] = np.arange(len(xyz), dtype=F32)
    return out


def _ulps(x, k):
    """x moved by k fp32 ulps (k may be negative)."""
    x = F32(x)
    for _ in range(abs(k)):
        x = np.nextafter(x, F32(np.inf) if k > 0 else F32(-np.inf))
    return x


# ---- NDT ------------------------------------------------------------------------------------------------------------
@dataclass
class NdtScene:
    name: str
    calls: list                 # AddCloudToLocalMap clouds, in order
    scan: np.ndarray
    T: np.ndarray = field(default_factory=lambda: np.eye(4))
    voxel: float = 1.0
    min_pts: int = 5
    max_pts: int = 50
    capacity: int = 100000
    leaf: float = 0.01
    thres: float = 5.0
    localization: bool = True

    def config(self, **kw):
        from funny_lidar_slam_b200 import FLS_NDT, default_config
        from funny_lidar_slam_b200._abi import FLS_FLAG_ITER_LOG
        return default_config(FLS_NDT, flags=FLS_FLAG_ITER_LOG, max_iterations=1, localization_mode=int(self.localization),
                              ndt_voxel_size=self.voxel, ndt_min_points_in_voxel=self.min_pts, ndt_max_points_in_voxel=self.max_pts,
                              ndt_capacity=self.capacity, source_cloud_filter_size=self.leaf, ndt_outlier_thres=self.thres,
                              ndt_min_effective_pts=1, **kw)


def _cluster(rng, centre, half, n):
    return np.asarray(centre, np.float64) + rng.uniform(-half, half, (n, 3))


def _face_queries(faces, v, ks=(-3, -1, 1, 3), others=(0.3, 0.4)):
    """Points k fp32 ulps either side of the planes x = f, y = f, z = f (f in `faces`); the other coordinates from `others`."""
    q = []
    for f in faces:
        for k in ks:
            c = _ulps(f, k) if f != 0 else F32(np.sign(k) * np.float32(1.4e-45) * abs(k))
            for axis in range(3):
                p = [F32(others[0]), F32(others[1]), F32(others[0] * 0.5)]
                p[axis] = c
                q.append(p)
    return np.array(q, F32)


def ndt_axes(offset=(0.0, 0.0, 0.0), name="ndt_axes"):
    """Clusters straddling x = 0, y = 0 and z = 0 (key 0 spans (-1, 1)), neighbours at +-1, single points; queries on faces."""
    rng = np.random.default_rng(11)
    o = np.asarray(offset)
    pts = [_cluster(rng, o + c, 0.45, 12) for c in ((0.0, 0.0, 0.0), (1.5, 0.3, 0.2), (-1.5, 0.3, 0.2), (0.3, 1.5, 0.2), (0.3, -1.5, 0.2),
                                                     (0.3, 0.3, 1.5), (0.3, 0.3, -1.5))]
    pts += [o + np.array([[-0.6, -0.6, 0.1]])]  # (-0.6, -0.6, 0.1) -> key (0, 0, 0) with truncation, (-1, -1, 0) with floor
    scan = _face_queries([0.0, 1.0, -1.0], 1.0).astype(np.float64)
    if np.any(o):  # far copy: the faces next to the offset, a few ulps either side
        scan = np.vstack([_face_queries([F32(o[0] + 1.0), F32(o[0] + 2.0)], 1.0, others=(F32(o[1] + 0.3), F32(o[2] + 0.4))),
                          rng.uniform(-0.4, 0.4, (30, 3)) + o]).astype(np.float64)
    return NdtScene(name, [_cloud(np.vstack(pts))], _cloud(scan))


def ndt_far():
    return ndt_axes(offset=(4999.0, -5001.0, 5000.0), name="ndt_far_5km")


def ndt_v03():
    """v = 0.3: keys are trunc(q * (1 / 0.3)); queries a few ulps either side of k * 0.3 for k = 1, 2, -1."""
    rng = np.random.default_rng(12)
    pts = [_cluster(rng, c, 0.12, 10) for c in ((0.15, 0.15, 0.15), (0.45, 0.15, 0.15), (0.75, 0.15, 0.15), (-0.15, 0.15, 0.15), (0.15, 0.45, 0.15),
                                                (0.15, 0.15, 0.45), (0.45, 0.45, 0.15))]
    faces = [F32(0.3), F32(0.6), F32(-0.3)]
    scan = _face_queries(faces, 0.3, others=(0.12, 0.2))
    return NdtScene("ndt_v03", [_cloud(np.vstack(pts))], _cloud(scan), voxel=0.3, thres=20.0)


def ndt_chi():
    """Single-point voxels (information 100 I): a query at e = (0.25, 0, 0) has chi = 6.25 exactly = outlier_thres; queries one to three
    fp32 ulps either side.  Cells 4 apart so that no stencil sees two of them."""
    singles, scan = [], []
    for j, k in enumerate((0, 1, -1, 2, -2, 3, -3)):
        base = np.array([4.0 * j + 0.5, 0.5, 0.5], F32)
        singles.append(base)
        scan.append([_ulps(F32(base[0] + F32(0.25)), k), base[1], base[2]])
    # a cluster voxel so that the first-estimate branch is also reached
    rng = np.random.default_rng(13)
    clus = _cluster(rng, (40.5, 0.5, 0.5), 0.4, 10)
    scan.append([40.3, 0.6, 0.4])
    return NdtScene("ndt_chi_single", [_cloud(np.vstack([np.array(singles, np.float64), clus]))], _cloud(np.array(scan, F32)), thres=6.25)


def ndt_unestimated():
    """Mapping mode: a first (estimated) cloud, then a second call that creates voxels with 2 points each (< min_points_in_voxel):
    they exist, count as hits and are skipped.  Queries whose 7-stencil holds both kinds."""
    rng = np.random.default_rng(14)
    first = np.vstack([_cluster(rng, (0.5 + 3 * j, 0.5, 0.5), 0.4, 10) for j in range(4)])
    second = np.vstack([_cluster(rng, (1.5 + 3 * j, 0.5, 0.5), 0.4, 2) for j in range(4)] + [_cluster(rng, (0.5 + 3 * j, 1.5, 0.5), 0.4, 2)
                                                                                             for j in range(4)])
    scan = np.array([[0.5 + 3 * j + dx, 0.5 + dy, 0.5] for j in range(4) for dx in (-0.3, 0.0, 0.3) for dy in (-0.2, 0.2)], F32)
    return NdtScene("ndt_unestimated", [_cloud(first), _cloud(second)], _cloud(scan), localization=False, thres=50.0)


def ndt_stream(capacity=40):
    """Open-loop mapping stream of AddCloudToLocalMap calls (min 3, max 12 points per voxel).  Group A voxels get 2 points per call:
    carry (2) -> estimate (4) -> carry -> merge (8) -> carry -> merge (12) -> carry -> merge (16 > 12) -> frozen.  Their points lie on
    z = const (planar: the clamp bites), on y = z = const (linear) or are generic.  From call 5 on, new voxels at low z push the map over
    `capacity`; the least recently touched voxel sits at high z, so PCL's filter order (z-major) touches it again after its eviction."""
    rng = np.random.default_rng(15)
    calls = []
    groupA = [(x, y) for x in range(3) for y in range(3)]
    first = []
    for j in range(4):  # call 0 (first scan): voxels estimated at once, one of them a single point, one at high z to be evicted later
        first.append(_cluster(rng, (0.5 + 2 * j, 20.5, 9.5), 0.4, 1 if j == 0 else 4))
    calls.append(_cloud(np.vstack(first)))
    for c in range(1, 11):
        pts = []
        for n_a, (x, y) in enumerate(groupA):
            base = np.array([2.0 * x + 0.5, 2.0 * y + 0.5, 3.5])
            p = base + rng.uniform(-0.4, 0.4, (2, 3))
            if n_a % 3 == 0:
                p[:, 2] = 3.5  # planar: zero variance in z exactly
            elif n_a % 3 == 1:
                p[:, 1], p[:, 2] = base[1] + 0.25, 3.5  # linear: only x varies
            pts.append(p)
        if c >= 5:  # new voxels at low z (created first in PCL order), then a touch of the old high-z voxels
            for k in range(6):
                pts.append(np.array([[0.5 + 2 * k + 0.1 * c, -10.5 - 2 * c, -9.5]]))
            if c == 9:
                pts.append(np.array([[2.5, 20.5, 9.5], [4.5, 20.3, 9.2]]))
        calls.append(_cloud(np.vstack(pts)))
    scan = np.array([[2.0 * x + 0.5 + dx, 2.0 * y + 0.5, 3.5 + dz] for x, y in groupA for dx in (-0.2, 0.2) for dz in (0.0, 0.05)], F32)
    return NdtScene("ndt_stream", calls, _cloud(scan), min_pts=3, max_pts=12, capacity=capacity, localization=False, thres=1e6)


def ndt_scenes():
    return [ndt_axes(), ndt_far(), ndt_v03(), ndt_chi(), ndt_unestimated()]


# ---- ICP ------------------------------------------------------------------------------------------------------------
@dataclass
class IcpScene:
    name: str
    map: np.ndarray
    scan: np.ndarray
    max_corr: float
    T: np.ndarray = field(default_factory=lambda: np.eye(4))
    ties: bool = False

    def config(self, **kw):
        from funny_lidar_slam_b200 import FLS_ICP_P2P, default_config
        from funny_lidar_slam_b200._abi import FLS_FLAG_ITER_LOG
        return default_config(FLS_ICP_P2P, flags=FLS_FLAG_ITER_LOG, max_iterations=1, icp_max_correspond_distance=self.max_corr,
                              source_cloud_filter_size=0.01, map_cloud_filter_size=0.01, **kw)


def point_at_d2(q, target, axis=0, sign=1.0):
    """An fp32 map point whose fp32 squared distance to q is exactly `target` (an fp32 number), found among the fp32 neighbours of
    q + sign sqrt(target) along `axis` (or, failing that, another axis), with a small offset on the next axis when one axis alone
    cannot hit it."""
    q = np.asarray(q, F32)
    target = F32(target)
    r = F32(np.sqrt(np.float64(target)))
    for ax in (axis, (axis + 1) % 3, (axis + 2) % 3):  # the requested axis first
        for off in [F32(0)] + [F32(m * 2.0 ** -e) for e in range(6, 14) for m in (1.0, 1.25, 1.5, 1.75)]:
            c = q.copy()
            c[(ax + 1) % 3] = q[(ax + 1) % 3] + off
            x0 = F32(q[ax] + F32(sign) * r)
            for k in range(-64, 65):
                c[ax] = _ulps(x0, k)
                if dist2(c, q) == target:
                    return c.copy()
    raise ValueError("no fp32 point at that distance")


def icp_gate(max_corr):
    """Per query: one map point with d2 = max_corr exactly, or one fp32 ulp either side; and queries on a face / corner of the search
    grid (cell = sqrt(max_corr) * 1.001) whose only neighbour sits 0.9999 sqrt(max_corr) away across the face."""
    mc = F32(max_corr)
    mp, sc = [], []
    for j, k in enumerate((0, 1, -1, 0, 1, -1)):
        q = np.array([10.0 * j + 0.37, 0.41, 0.29], F32)
        mp.append(point_at_d2(q, _ulps(mc, k), axis=j % 3, sign=1.0 if j < 3 else -1.0))
        sc.append(q)
    # queries just above the face x = 0 of the search grid (cell 0 starts at 0 for every cell size), alone or also just above z = 0
    # (a corner); the only neighbour lies 0.9999 sqrt(max_corr) away towards -x, one cell down with cell >= sqrt(max_corr) and two
    # cells down with a cell any smaller than that
    r = F32(np.sqrt(max_corr))
    for j, (x, z) in enumerate(((1e-6, 0.3), (1e-4, 0.3), (1e-6, 1e-6), (3e-4, 1e-6))):
        q = np.array([x, 100.0 + 10 * j, z], F32)
        nb = q.copy()
        nb[0] = F32(q[0] - F32(0.9999) * r)
        mp.append(nb)
        sc.append(q)
    # every query twice: Match refuses ten points or fewer before filtering, and the filter folds each pair back into one
    return IcpScene(f"icp_gate_{max_corr}", _cloud(np.array(mp)), _cloud(np.vstack([sc, sc])), max_corr)


def icp_ties():
    """A unit lattice: queries at cell centres and edge midpoints are equidistant to 8 / 4 / 2 lattice points.  Eleven copies of one
    query (Match refuses ten points or fewer; the filter folds them into one)."""
    g = np.stack(np.meshgrid(np.arange(4.0), np.arange(4.0), np.arange(3.0), indexing="ij"), -1).reshape(-1, 3)
    return IcpScene("icp_ties", _cloud(g), _cloud(np.tile([[1.5, 1.5, 0.5]], (11, 1))), 1.0, ties=True)


def icp_ties_edge():
    g = np.stack(np.meshgrid(np.arange(4.0), np.arange(4.0), np.arange(3.0), indexing="ij"), -1).reshape(-1, 3)
    return IcpScene("icp_ties_edge", _cloud(g), _cloud(np.tile([[2.0, 1.5, 1.5]], (11, 1))), 1.0, ties=True)


def icp_far():
    """A far guess: every query is more than 100 m from the map, nothing corresponds."""
    rng = np.random.default_rng(21)
    mp = rng.uniform(-5, 5, (200, 3))
    T = np.eye(4)
    T[:3, 3] = (1024.0, 0.0, 0.0)
    return IcpScene("icp_far", _cloud(mp), _cloud(mp[:40] + 0.05), 1.0, T=T)


def icp_sparse():
    """Five map points in five cells (fewer than the 27 of one stencil) and queries all around them."""
    mp = np.array([[0.3, 0.2, 0.1], [1.7, 0.4, 0.3], [0.2, 1.9, 0.2], [5.0, 5.0, 5.0], [-0.7, -0.4, 0.5]])
    rng = np.random.default_rng(22)
    sc = np.vstack([mp[j] + rng.uniform(-0.9, 0.9, (6, 3)) for j in range(5)])
    return IcpScene("icp_sparse", _cloud(mp), _cloud(sc), 1.0)


def icp_scenes():
    return [icp_gate(0.25), icp_gate(1.0), icp_gate(2.0), icp_ties(), icp_ties_edge(), icp_far(), icp_sparse()]


def fitness_scene(max_range=1.0):
    """GetFitnessScore edges at the identity pose: d2 = max_range and one ulp either side, and queries at the centre of a search cell
    (cell = sqrt(max_range) * 1.001) whose nearest point lies just across the face of the next cell while a point 0.1 % farther sits in
    the query's own cell (visited first): only the 0.998-scaled box bound lets the search reach the nearest one."""
    mr = F32(max_range)
    mp, sc = [], []
    for j, k in enumerate((0, 1, -1)):
        q = np.array([10.0 * j + 0.37, 0.41, 0.29], F32)
        mp.append(point_at_d2(q, _ulps(mr, k)))
        sc.append(q)
    cell = F32(np.sqrt(np.float32(max_range)) * np.float32(1.001))
    for j in range(3):
        cu = np.array([50 + 10 * j, 2, 2], np.float64)
        q = ((cu + 0.5) * np.float64(cell)).astype(F32)
        a = q.copy()
        a[0] = F32((cu[0] + 1) * np.float64(cell) + 1e-4)  # just inside the next cell
        da = float(dist2(a, q))
        rb = np.sqrt(da * 1.001)  # 0.1 % farther in d2, on the diagonal of the query's own cell
        b = (q.astype(np.float64) - rb / np.sqrt(2) * np.array([1.0, 1.0, 0.0])).astype(F32)
        mp += [b, a]
        sc.append(q)
    return _cloud(np.array(mp)), _cloud(np.array(sc))
