"""Sequential references of the LOAM-iVox mapping-mode map (CPU only, independent of the oracle and of the CUDA library).

`IVoxMapRef` is IVoxMap::AddPoints (ivox_map.cpp:122-143 upstream) done literally, point by point: an LRU list of voxels with
their point lists, a voxel created at the front, a touched voxel moved to the front, the tail dropped whenever a creation
brings the size to the capacity.  Its neighbour answers are `ivox_ref.knn5` over the surviving points in insertion order.

`insert_rule` is the Match-internal AddCloudToLocalMap (loam_point_to_plane_ivox.h:79-128 upstream, [quirk 8]): each body-frame
point is moved to the map with the final pose and classified by the 5 neighbours its last PlanerMatch cached at the pose
before the last update, and by the centre of its `filter` cell."""
from __future__ import annotations

from collections import OrderedDict
from dataclasses import dataclass

import numpy as np

from tests import ivox_ref

F32 = np.float32
EPS = float(np.finfo(np.float64).eps)


class IVoxMapRef:
    def __init__(self, res, capacity):
        self.res = float(res)
        self.capacity = int(capacity)
        self._lru = OrderedDict()  # key -> [(seq, point)], least recently used first
        self._seq = 0

    def add(self, pts):
        pts = np.asarray(pts, F32).reshape(-1, 4)
        keys = ivox_ref.voxel_key(pts[:, :3], self.res)
        for p, k in zip(pts, map(tuple, keys.tolist())):
            rec = (self._seq, p.copy())
            self._seq += 1
            if k not in self._lru:
                self._lru[k] = [rec]
                if len(self._lru) >= self.capacity:
                    self._lru.popitem(last=False)
            else:
                self._lru[k].append(rec)
                self._lru.move_to_end(k)

    @property
    def points(self):
        """(n, 4) surviving points in global insertion order."""
        recs = sorted((r for v in self._lru.values() for r in v), key=lambda r: r[0])
        return np.array([p for _, p in recs], F32).reshape(-1, 4)

    @property
    def voxels(self):
        """{key: (m, 4) points in insertion order}."""
        return {k: np.array([p for _, p in v], F32) for k, v in self._lru.items()}

    @property
    def lru_dump(self):
        """(n, 4) the points voxel by voxel, most recently used voxel first (IVoxMap's grids_cache_ order)."""
        return np.array([p for v in reversed(self._lru.values()) for _, p in v], F32).reshape(-1, 4)

    @property
    def num_voxels(self):
        return len(self._lru)


@dataclass
class InsertRule:
    cls: np.ndarray       # (n,) 0 dropped, 1 added, 2 added without down-sampling
    world: np.ndarray     # (n, 4) the points at the final pose (fp64 rows rounded to fp32), intensity kept
    appended: np.ndarray  # (m, 4) what enters the map: class 1 in input order, then class 2
    gap01: np.ndarray     # (n,) knn5's ulps between the cached ranks 0 and 1 (-1: fewer than 2)
    gap45: np.ndarray     # (n,) knn5's ulps between ranks 4 and 5 (-1: fewer than 6 in range)
    axis_margin: np.ndarray  # (n,) min over axes of |nearest - centre| - filter/2 (> 0 on every axis: class 2; nan: no neighbour)
    near_margin: np.ndarray  # (n,) min over the 5 neighbours of |neighbour - centre|^2 - (dist + 1e-6) (< 0: dropped; nan: not tested)
    near_tol: np.ndarray     # (n,) how far fp64 rounding of the squared norms (contracted or not) may move near_margin

    def ties(self):
        """Points whose class-1 decision lies within fp64 rounding: the test is not told apart from rounding there."""
        return np.nonzero(np.abs(self.near_margin) <= self.near_tol)[0]


def insert_rule(map_pts, scan, T_prev, T_fin, res, nearby, max_range, filter=0.5):
    map_pts = np.asarray(map_pts, F32).reshape(-1, 4)
    scan = np.asarray(scan, F32).reshape(-1, 4)
    n = len(scan)
    kn = ivox_ref.knn5(map_pts, ivox_ref.transform(scan, np.asarray(T_prev, np.float64)), res, nearby, max_range)
    world = np.empty((n, 4), F32)
    world[:, :3] = ivox_ref.transform(scan, np.asarray(T_fin, np.float64))
    world[:, 3] = scan[:, 3]
    cls = np.ones(n, np.int8)
    axis = np.full(n, np.nan)
    near = np.full(n, np.nan)
    tol = np.zeros(n)
    half = 0.5 * filter
    for i in range(n):
        if kn.found[i] == 0:  # no cached neighbour (:93-96, :125-127)
            continue
        pv = world[i, :3].astype(np.float64)
        c = (np.floor(pv / filter) + 0.5) * filter  # :97-99
        d0 = map_pts[kn.idx[i, 0], :3].astype(np.float64) - c
        axis[i] = float(np.min(np.abs(d0) - half))
        if axis[i] > 0.0:  # :103-108
            cls[i] = 2
            continue
        e = pv - c
        dist = (e[0] * e[0] + e[1] * e[1]) + e[2] * e[2]
        if kn.found[i] < 5:  # :112
            continue
        lim = dist + 1.0e-6
        m = np.inf
        for r in range(5):
            f = map_pts[kn.idx[i, r], :3].astype(np.float64) - c
            m = min(m, (f[0] * f[0] + f[1] * f[1]) + f[2] * f[2] - lim)
        near[i] = m
        tol[i] = 8.0 * EPS * (abs(lim) + abs(m + lim))
        if m < 0.0:  # :113-120
            cls[i] = 0
    appended = np.concatenate([world[cls == 1], world[cls == 2]])
    return InsertRule(cls, world, appended, kn.gap01, kn.gap45, axis, near, tol)


def _pts(xyz, first=0):
    xyz = np.asarray(xyz, np.float64).reshape(-1, 3)
    out = np.zeros((len(xyz), 4), F32)
    out[:, :3] = xyz
    out[:, 3] = np.arange(first, first + len(xyz), dtype=F32)
    return out


@dataclass
class RuleScene:
    map: np.ndarray     # (n, 4) the map of the first AddCloudToLocalMap
    scan: np.ndarray    # (m, 4) corner points (on the map's planes) interleaved with the probes
    probes: dict        # name -> scan rows
    on_map: np.ndarray  # (k, 4) corner points that coincide with map points: every one is dropped


def rule_scene():
    """Insertion-rule edges around a three-plane corner.  Every coordinate is a multiple of 2^-8 (one neighbour sits 2e-6 past a
    tie and is fp32-rounded), so at the identity every cell centre, squared norm and comparison of the rule is exact.  The
    corner's planes (z = -1, x = -2, y = 1.5, 0.125 m lattice) give 108 scan points with a zero residual, enough for a
    converged Match whose one Gauss-Newton step stays at rounding level; every probe has fewer than 5 neighbours or a
    non-planar five, so it adds no residual.  Probes (res 0.5, ivox_max_range 1.0):
      none      no candidate in its stencil                  beyond  candidates in the stencil, all beyond max_range
      few1..4   1..4 cached neighbours (5-neighbour test skipped)
      axis_eq   nearest exactly filter/2 from the centre on x: not class 2      axis_gt  2^-8 further: class 2
      eq        a neighbour exactly as far from the centre as the point: dropped
      eps2      the nearest neighbour 2e-6 further than the point, the rest far: kept
      face      on voxel and cell faces, negative coordinates
      tie_a     rank 0 tied, the class-2 neighbour inserted first: class 2      tie_b  the other first: class 1"""
    lat = np.arange(17) * 0.125
    floor = [(-2.0 + a, 1.5 + b, -1.0) for a in lat[1:] for b in lat[1:]]
    wall_x = [(-2.0, 1.5 + a, -1.0 + b) for a in lat[1:] for b in lat[1:]]
    wall_y = [(-2.0 + a, 1.5, -1.0 + b) for a in lat[1:] for b in lat[1:]]
    mp = [np.array(floor + wall_x + wall_y)]
    g = 0.25 * np.arange(6) + 0.0625
    corner = ([(-1.625 + a, 1.875 + b, -1.0) for a in g for b in g] + [(-2.0, 1.875 + a, -0.625 + b) for a in g for b in g]
              + [(-1.625 + a, 1.5, -0.625 + b) for a in g for b in g])
    on_map = [(-1.5 + a, 2.0 + b, -1.0) for a in lat[:8] for b in lat[:8]]
    probes, rows = {}, []

    def probe(name, p, neighbours=()):
        probes[name] = len(rows)
        rows.append(tuple(float(v) for v in p))
        if len(neighbours):
            mp.append(np.asarray(neighbours, np.float64).reshape(-1, 3))

    probe("none", (20.0, 20.0, 5.0))
    probe("beyond", (3.75, 5.25, 5.25), [(4.7421875, 5.7421875, 5.7421875), (4.7421875, 5.5, 5.5)])
    for k in range(1, 5):
        b = np.array([12.0, 3.0 * k, 0.0])
        offs = [(0.3125, 0.3125, 0.3125), (-0.1875, 0.125, 0.0625), (0.0625, -0.25, 0.1875), (-0.3125, -0.0625, -0.3125)][:k]
        probe(f"few{k}", b + (0.0625, 0.0625, 0.0625), [b + o for o in offs])
    c = np.array([-6.25, -4.75, -2.25])
    probe("axis_eq", c + 0.0625, [c + (0.25, 0.375, 0.375)])
    c = np.array([-9.25, -4.75, -2.25])
    probe("axis_gt", c + 0.0625, [c + (0.25 + 2.0 ** -8, 0.375, 0.375)])
    tet = [(0.375, 0.375, 0.375), (-0.375, 0.375, -0.375), (0.375, -0.375, -0.375), (-0.375, -0.375, 0.375)]
    c = np.array([-6.25, 4.25, 3.25])
    probe("eq", c + (0.125, 0.0, 0.0), [c + (0.0, 0.125, 0.0)] + [c + t for t in tet])
    c = np.array([-9.25, 4.25, 3.25])
    s = float(F32(c[2] + np.sqrt(0.125 ** 2 + 2e-6))) - c[2]
    probe("eps2", c + (0.125, 0.0, 0.0), [c + (0.0, 0.0, s)] + [c + t for t in tet])
    probe("face", (-10.25, -7.75, -3.5), [(-10.5, -7.5, -3.25), (-10.0, -7.75, -3.75), (-10.25, -8.0, -3.5)])
    probe("face2", (-10.5, -10.0, -3.25), [(-10.75, -10.25, -3.0), (-10.25, -9.75, -3.5)])
    a, b, p = (8.625, -4.875, 3.0625), (8.625, -4.875, 2.8125), (8.25, -5.25, 2.9375)
    probe("tie_a", p, [a, b])
    sh = np.array([3.0, 0.0, 0.0])
    probe("tie_b", p + sh, [b + sh, a + sh])
    # probes interleaved with the corner points: the appended slice has to be re-ordered, class 1 first
    scan = [tuple(map(float, p)) for p in corner]
    step = len(corner) // (len(rows) + 1)
    for j, r in enumerate(rows):
        scan.insert((j + 1) * step + j, r)
    probes = {k: scan.index(rows[v]) for k, v in probes.items()}
    return RuleScene(_pts(np.concatenate(mp)), _pts(scan, 10000), probes, _pts(on_map, 20000))
