"""Host-side mirror of the reference's registration plug-in interface, over the C ABI.

`Registration` mirrors RegistrationInterface (include/registration/registration_interface.h:11-20 upstream):
`Match(cluster, T) -> bool` (T in-out), `AddCloudToLocalMap([cloud, ...])`, `GetFitnessScore(max_range)`.
`create_matcher(mode_string, ...)` mirrors the factory branches of FrontEnd::InitMatcher
(src/slam/frontend.cpp:30-88 upstream) keyed by the same mode strings (constant_variable.h:21-25).
Clouds are numpy float32 arrays: (n,4) packed x,y,z,intensity or (n,8) pcl::PointXYZI records.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from . import _abi
from ._abi import FlsConfig, FlsInformation, FlsIterLog, FlsMapInfo, FlsMatchStats
from ._lib import check, lib


@dataclass
class PointcloudCluster:
    """The members of PointcloudCluster (include/lidar/pointcloud_cluster.h:13-26 upstream) a matcher reads."""
    ordered_cloud: np.ndarray | None = None
    planar_cloud: np.ndarray | None = None
    corner_cloud: np.ndarray | None = None
    point_depth_vec: np.ndarray | None = None
    point_col_index_vec: np.ndarray | None = None
    row_start_index_vec: np.ndarray | None = None
    row_end_index_vec: np.ndarray | None = None
    timestamp: int = 0
    extra: dict = field(default_factory=dict)


def _cloud(a):
    if a is None:
        return None, 0, 16, None
    a = np.ascontiguousarray(a, dtype=np.float32)
    if a.ndim != 2 or a.shape[1] not in (4, 8):
        raise ValueError("cloud must be (n,4) packed xyzi or (n,8) pcl::PointXYZI records")
    return a.ctypes.data_as(C.c_void_p), a.shape[0], a.shape[1] * 4, a


@dataclass
class RelocResult:
    """What Registration.relocalize returns: the chosen pose T (4,4) and fls_reloc_result's fields; the per-refined arrays are in
    refinement rank order (rank 0 = best coarse score) and coarse_scores in hypothesis index order (None unless asked for)."""
    T: np.ndarray
    accepted: bool
    converged: bool
    fitness: float
    coarse_score: float
    n_hypotheses: int
    best_hypothesis: int
    best_rank: int
    n_refined: int
    host_waits: int
    gpu_launches: int
    refined_T: np.ndarray
    refined_converged: np.ndarray
    refined_fitness: np.ndarray
    refined_index: np.ndarray
    coarse_scores: np.ndarray | None = None


def reloc_cfg(xy_radius=10.0, xy_step=1.0, yaw_range=np.pi, yaw_step=np.deg2rad(10.0), coarse_leaf=1.0, max_range=2.0, accept_fitness=1.0,
              n_refine=64) -> _abi.FlsRelocCfg:
    """fls_reloc_cfg; the defaults search +-10 m at 1 m and the full circle at 10 deg around the guess, with Localization::Init's
    GetFitnessScore(2.0) < 1.0 as the acceptance rule (src/slam/localization.cpp:135-140 upstream)."""
    c = _abi.FlsRelocCfg()
    c.xy_radius, c.xy_step, c.yaw_range, c.yaw_step = float(xy_radius), float(xy_step), float(yaw_range), float(yaw_step)
    c.coarse_leaf, c.max_range, c.accept_fitness, c.n_refine = float(coarse_leaf), float(max_range), float(accept_fitness), int(n_refine)
    return c


def _guesses(Ts):
    """The guesses of a multi-guess call, column-major per pose, and the start value of its output pose (guess 0, which the call
    overwrites; the identity when there is none)."""
    Ts = np.asarray(Ts, np.float64).reshape(-1, 4, 4)
    return _batch_poses(Ts), (Ts[0] if len(Ts) else np.eye(4))


def _batch_poses(Ts):
    return np.ascontiguousarray(np.transpose(np.asarray(Ts, np.float64), (0, 2, 1))).copy()  # Eigen column-major per pose


def _host_batch(scans, Ts):
    """Host scans of a batch call: (keep-alive arrays, pointer array, count array, stride, column-major poses)."""
    ptrs, ns, keep, stride = [], [], [], None
    for c in scans:
        p, n, s, a = _cloud(c)
        if stride is not None and s != stride:
            raise ValueError("all scans of one batch must share a layout")
        stride = s
        ptrs.append(p)
        ns.append(n)
        keep.append(a)
    B = len(scans)
    return keep, (C.c_void_p * B)(*ptrs), (C.c_size_t * B)(*ns), stride, _batch_poses(Ts)


def _device_batch(d_ptrs, ns, Ts):
    """Device-resident scans of a batch call: (pointer array, count array, column-major poses)."""
    B = len(d_ptrs)
    return (C.c_void_p * B)(*[int(p) for p in d_ptrs]), (C.c_size_t * B)(*[int(n) for n in ns]), _batch_poses(Ts)


class Registration:
    def __init__(self, cfg: FlsConfig):
        self.cfg = cfg
        self._h = C.c_void_p()
        check(lib().fls_create(C.byref(cfg), C.byref(self._h)), "fls_create")
        self.last_stats = FlsMatchStats()

    # -- RegistrationInterface ----------------------------------------------------------------------------
    def AddCloudToLocalMap(self, cloud_list) -> None:
        if isinstance(cloud_list, np.ndarray):
            cloud_list = [cloud_list]
        ptrs, ns, keep, stride = [], [], [], None
        for c in cloud_list:
            p, n, s, a = _cloud(c)
            if stride is not None and s != stride:
                raise ValueError("all clouds of one call must share a layout")
            stride = s
            ptrs.append(p)
            ns.append(n)
            keep.append(a)
        arr_p = (C.c_void_p * len(ptrs))(*ptrs)
        arr_n = (C.c_size_t * len(ns))(*ns)
        check(lib().fls_add_cloud(self._h, len(ptrs), arr_p, arr_n, stride), "fls_add_cloud")

    def Match(self, cluster: PointcloudCluster, T: np.ndarray) -> bool:
        """T: (4,4) float64, updated in place (also on failure, as upstream)."""
        po, no, so, ko = _cloud(cluster.ordered_cloud)
        pp, npl, sp, kp = _cloud(cluster.planar_cloud)
        pc, nc, scn, kc = _cloud(cluster.corner_cloud)
        strides = {s for s, k in ((so, ko), (sp, kp), (scn, kc)) if k is not None}
        if len(strides) > 1:
            raise ValueError("all clouds of one cluster must share a layout")
        stride = strides.pop() if strides else 16
        Tc = np.ascontiguousarray(np.asarray(T, np.float64).T).copy()  # Eigen column-major memory
        conv = C.c_int(0)
        st = FlsMatchStats()
        rc = lib().fls_match(self._h, po, no, pp, npl, pc, nc, stride, Tc.ctypes.data_as(C.c_void_p), C.byref(conv), C.byref(st))
        check(rc, "fls_match")
        T[...] = Tc.T
        self.last_stats = st
        return bool(conv.value)

    def GetFitnessScore(self, max_range: float) -> float:
        out = C.c_float(0)
        rc = lib().fls_fitness(self._h, float(max_range), C.byref(out))
        if rc == _abi.FLS_ERR_UNSUPPORTED:
            return float(np.finfo(np.float32).max)
        check(rc, "fls_fitness")
        return float(out.value)

    # -- batched Match (throughput entry; LOAM-iVox, NDT, ICP and kd-tree point-to-plane in localization mode) -----
    def _batch_results(self, conv, st, Tc):
        self.last_batch_stats = list(st)
        self.last_stats = st[0]
        return np.array(conv[:], bool), np.transpose(Tc, (0, 2, 1)).copy()

    def match_batch(self, scans, Ts):
        """scans: list of (n,4)/(n,8) host clouds — the planar clouds for the LOAM plug-ins, the ordered clouds for NDT and ICP (LoamFull
        has no batch); Ts: (B,4,4) float64 initial poses.  Returns (converged[B], T[B,4,4]); self.last_batch_stats holds the per-scan
        fls_match_stats (call-level timings on element 0)."""
        B = len(scans)
        keep, arr_p, arr_n, stride, Tc = _host_batch(scans, Ts)
        conv = (C.c_int * B)()
        st = (FlsMatchStats * B)()
        check(lib().fls_match_batch(self._h, B, arr_p, arr_n, stride, Tc.ctypes.data_as(C.c_void_p), conv, st), "fls_match_batch")
        return self._batch_results(conv, st, Tc)

    def match_batch_begin(self, scans, Ts) -> None:
        """First half of match_batch: enqueue copies + matching + read-back on the handle's stream, do not wait (the scans should sit
        in pinned host memory).  With two handles the copy of one batch overlaps the kernels of the other."""
        B = len(scans)
        keep, arr_p, arr_n, stride, Tc = _host_batch(scans, Ts)
        self._pending = (keep, arr_p, arr_n, Tc, B)
        check(lib().fls_match_batch_begin(self._h, B, arr_p, arr_n, stride, Tc.ctypes.data_as(C.c_void_p)), "fls_match_batch_begin")

    def match_batch_begin_device(self, d_ptrs, ns, Ts) -> None:
        """match_batch_begin with device-resident packed float4 scans."""
        B = len(d_ptrs)
        arr_p, arr_n, Tc = _device_batch(d_ptrs, ns, Ts)
        self._pending = ((), arr_p, arr_n, Tc, B)
        check(lib().fls_match_batch_begin_device(self._h, B, arr_p, arr_n, Tc.ctypes.data_as(C.c_void_p)), "fls_match_batch_begin_device")

    def match_batch_end(self):
        keep, arr_p, arr_n, Tc, B = self._pending
        conv = (C.c_int * B)()
        st = (FlsMatchStats * B)()
        check(lib().fls_match_batch_end(self._h, Tc.ctypes.data_as(C.c_void_p), conv, st), "fls_match_batch_end")
        self._pending = None
        return self._batch_results(conv, st, Tc)

    def match_batch_device(self, d_ptrs, ns, Ts):
        """Same with device-resident packed float4 scans: d_ptrs = list of device addresses, ns = point counts."""
        B = len(d_ptrs)
        arr_p, arr_n, Tc = _device_batch(d_ptrs, ns, Ts)
        conv = (C.c_int * B)()
        st = (FlsMatchStats * B)()
        check(lib().fls_match_batch_device(self._h, B, arr_p, arr_n, Tc.ctypes.data_as(C.c_void_p), conv, st), "fls_match_batch_device")
        return self._batch_results(conv, st, Tc)

    def set_result_buffer_device(self, d_ptr: int, capacity_scans: int) -> None:
        """Every later Match also writes {column-major pose, converged, iterations} (18 doubles per scan) to this device
        buffer from inside the GN kernel — the input of the per-batch pose all-gather (parallel.py)."""
        check(lib().fls_set_result_buffer_device(self._h, C.c_void_p(d_ptr) if d_ptr else None, int(capacity_scans)), "fls_set_result_buffer_device")

    # -- device-resident scan (bench `value` leg) ---------------------------------------------------------
    def match_device(self, d_ptr: int, n: int, T: np.ndarray) -> bool:
        Tc = np.ascontiguousarray(np.asarray(T, np.float64).T).copy()
        conv = C.c_int(0)
        st = FlsMatchStats()
        check(lib().fls_match_device(self._h, C.c_void_p(d_ptr), n, Tc.ctypes.data_as(C.c_void_p), C.byref(conv), C.byref(st)), "fls_match_device")
        T[...] = Tc.T
        self.last_stats = st
        return bool(conv.value)

    def match_cluster_device(self, d_ordered: int, n_ordered: int, d_planar: int, n_planar: int, d_corner: int, n_corner: int, T: np.ndarray) -> bool:
        """Match with the cluster's clouds already in device memory (packed float4 device addresses, 0 for an unused cloud); the
        plug-in reads the same clouds as Match.  The device-resident Match of LoamFull (planar + corner)."""
        Tc = np.ascontiguousarray(np.asarray(T, np.float64).T).copy()
        conv = C.c_int(0)
        st = FlsMatchStats()
        vp = lambda a: C.c_void_p(int(a)) if a else None
        check(lib().fls_match_cluster_device(self._h, vp(d_ordered), int(n_ordered), vp(d_planar), int(n_planar), vp(d_corner), int(n_corner),
                                             Tc.ctypes.data_as(C.c_void_p), C.byref(conv), C.byref(st)), "fls_match_cluster_device")
        T[...] = Tc.T
        self.last_stats = st
        return bool(conv.value)

    # -- relocalization from a coarse pose (Localization::Init upstream) -----------------------------------
    def _relocalize(self, call, T_guess, coarse_scores, cfg, wide=False, name=None):
        c = cfg if isinstance(cfg, _abi.FlsRelocCfg) else reloc_cfg(**cfg)
        k = max(1, int(c.n_refine))
        Tc = np.ascontiguousarray(np.asarray(T_guess, np.float64).T).copy()
        res = _abi.FlsRelocResult()
        rT = np.zeros((k, 4, 4), np.float64)
        rconv = np.zeros(k, np.int32)
        rfit = np.zeros(k, np.float32)
        ridx = np.zeros(k, np.int64)
        cs = np.zeros(max(int(coarse_scores), 1), np.float64)
        vp = lambda a: a.ctypes.data_as(C.c_void_p)
        evals = C.c_int64(-1)
        if wide:
            check(call(C.byref(c), vp(Tc), C.byref(res), vp(rT), vp(rconv), vp(rfit), vp(ridx), C.byref(evals)),
                  name or "fls_relocalize_wide")
        else:
            check(call(C.byref(c), vp(Tc), C.byref(res), vp(rT), vp(rconv), vp(rfit), vp(ridx), vp(cs) if coarse_scores else None, int(coarse_scores)),
                  "fls_relocalize")
        n = res.n_refined
        ncs = min(int(coarse_scores), int(res.n_hypotheses)) if res.n_refined else 0
        r = RelocResult(T=Tc.T.copy(), accepted=bool(res.accepted), converged=bool(res.converged), fitness=float(res.fitness),
                           coarse_score=float(res.coarse_score), n_hypotheses=int(res.n_hypotheses), best_hypothesis=int(res.best_hypothesis),
                           best_rank=int(res.best_rank), n_refined=int(n), host_waits=int(res.host_waits), gpu_launches=int(res.gpu_launches),
                           refined_T=np.transpose(rT[:n], (0, 2, 1)).copy(), refined_converged=rconv[:n].astype(bool), refined_fitness=rfit[:n].copy(),
                           refined_index=ridx[:n].copy(), coarse_scores=cs[:ncs].copy() if coarse_scores else None)
        return (r, int(evals.value)) if wide else r

    def relocalize(self, cloud_or_cluster, T_guess, coarse_scores: int = 0, cfg=None, **kw) -> RelocResult:
        """fls_relocalize: score an x-y-yaw grid of hypotheses around T_guess (4,4), refine the best n_refine in one batch Match and
        return the pose Localization::Init's rule would pick.  cloud_or_cluster: the cloud Match reads ((n,4)/(n,8) float32; the
        planar cloud for LOAM-iVox, the ordered cloud for NDT) or a PointcloudCluster.  cfg: an FlsRelocCfg, else reloc_cfg(**kw).
        coarse_scores: how many coarse scores (index order) to return."""
        c = cloud_or_cluster
        if isinstance(c, PointcloudCluster):
            c = c.ordered_cloud if self.cfg.method == _abi.FLS_NDT else c.planar_cloud
        p, n, s, keep = _cloud(c)
        return self._relocalize(lambda *a: lib().fls_relocalize(self._h, p, n, s, *a), T_guess, coarse_scores, cfg if cfg is not None else kw)

    def relocalize_device(self, d_ptr: int, n: int, T_guess, coarse_scores: int = 0, cfg=None, **kw) -> RelocResult:
        """relocalize with a device-resident packed float4 scan (it must stay valid until the next Match, as in match_device)."""
        return self._relocalize(lambda *a: lib().fls_relocalize_device(self._h, C.c_void_p(int(d_ptr)) if d_ptr else None, int(n), *a), T_guess,
                                coarse_scores, cfg if cfg is not None else kw)

    def relocalize_wide(self, cloud_or_cluster, T_guess, cfg=None, **kw):
        """fls_relocalize_wide: relocalize's results on the same grid without its 2^20 cap (up to 2^31 hypotheses), searched by exact
        branch and bound.  Returns (RelocResult without coarse_scores, the number of pose evaluations the search ran)."""
        c = cloud_or_cluster
        if isinstance(c, PointcloudCluster):
            c = c.ordered_cloud if self.cfg.method == _abi.FLS_NDT else c.planar_cloud
        p, n, s, keep = _cloud(c)
        return self._relocalize(lambda *a: lib().fls_relocalize_wide(self._h, p, n, s, *a), T_guess, 0, cfg if cfg is not None else kw, wide=True)

    def relocalize_wide_device(self, d_ptr: int, n: int, T_guess, cfg=None, **kw):
        """relocalize_wide with a device-resident packed float4 scan (it must stay valid until the next Match)."""
        return self._relocalize(lambda *a: lib().fls_relocalize_wide_device(self._h, C.c_void_p(int(d_ptr)) if d_ptr else None, int(n), *a), T_guess, 0,
                                cfg if cfg is not None else kw, wide=True)

    def relocalize_multi(self, cloud_or_cluster, guesses, cfg=None, **kw):
        """fls_relocalize_multi: relocalize_wide over the grids of every guess in `guesses` ((G,4,4), 1..64 poses, e.g. place_pose of
        each place_query candidate) as one search; hypothesis g * P + p is hypothesis p of guess g's grid.  Returns (RelocResult
        without coarse_scores, the number of pose evaluations the search ran)."""
        c = cloud_or_cluster
        if isinstance(c, PointcloudCluster):
            c = c.ordered_cloud if self.cfg.method == _abi.FLS_NDT else c.planar_cloud
        p, n, s, keep = _cloud(c)
        G, T0 = _guesses(guesses)
        return self._relocalize(lambda cp, *a: lib().fls_relocalize_multi(self._h, p, n, s, cp, G.ctypes.data_as(C.c_void_p), len(G), *a), T0, 0,
                                cfg if cfg is not None else kw, wide=True, name="fls_relocalize_multi")

    def relocalize_multi_device(self, d_ptr: int, n: int, guesses, cfg=None, **kw):
        """relocalize_multi with a device-resident packed float4 scan (it must stay valid until the next Match)."""
        G, T0 = _guesses(guesses)
        d = C.c_void_p(int(d_ptr)) if d_ptr else None
        return self._relocalize(lambda cp, *a: lib().fls_relocalize_multi_device(self._h, d, int(n), cp, G.ctypes.data_as(C.c_void_p), len(G), *a), T0,
                                0, cfg if cfg is not None else kw, wide=True, name="fls_relocalize_multi_device")

    def relocalize_wide_levels(self) -> list:
        """fls_relocalize_wide_levels: the nodes the last relocalize_wide reached per level, from its start level down to 0."""
        buf = (C.c_int64 * 64)()
        n = lib().fls_relocalize_wide_levels(self._h, buf, 64)
        if n < 0:
            check(n, "fls_relocalize_wide_levels")
        return [int(v) for v in buf[:n]]

    # -- localization-mode map path (Localization::LoadLocalMap upstream) ---------------------------------
    def set_global_map(self, cloud: np.ndarray) -> None:
        p, n, s, keep = _cloud(cloud)
        check(lib().fls_set_global_map(self._h, p, n, s), "fls_set_global_map")

    def update_local_map(self, T: np.ndarray):
        """Re-cut the +-100 m local map around T when needed and hand it to the plug-in; returns (updated, n_local_points)."""
        Tc = np.ascontiguousarray(np.asarray(T, np.float64).T).copy()
        upd, nl = C.c_int(0), C.c_size_t(0)
        check(lib().fls_update_local_map(self._h, Tc.ctypes.data_as(C.c_void_p), C.byref(upd), C.byref(nl)), "fls_update_local_map")
        return bool(upd.value), int(nl.value)

    # -- introspection ---------------------------------------------------------------------------------
    def map_points(self) -> np.ndarray:
        """(n, 4) float32 points of the LOAM-iVox map, insertion order."""
        cap = max(int(self.map_info().n_points), 1)
        out = np.zeros((cap, 4), np.float32)
        n = C.c_size_t(0)
        check(lib().fls_get_map_points(self._h, out.ctypes.data_as(C.c_void_p), cap, C.byref(n)), "fls_get_map_points")
        return out[:min(cap, n.value)]

    def voxel_keys(self) -> np.ndarray:
        """(n, 3) int32 voxel keys the map currently holds (NDT / LOAM-iVox), unordered."""
        cap = max(int(self.map_info().n_voxels), 1)
        out = np.zeros((cap, 3), np.int32)
        n = C.c_size_t(0)
        check(lib().fls_get_voxel_keys(self._h, out.ctypes.data_as(C.c_void_p), cap, C.byref(n)), "fls_get_voxel_keys")
        return out[:min(cap, n.value)]

    def ndt_voxels(self) -> dict:
        """Every live voxel of the NDT map sorted by key: key (n,3) int32, mu (n,3), info (n,6) as stored (xx, xy, xz, yy, yz, zz),
        estimated, num_points, carry_count (n,) int32."""
        cap = max(int(self.map_info().n_voxels), 1)
        buf = (_abi.FlsNdtVoxel * cap)()
        n = C.c_size_t(0)
        check(lib().fls_get_ndt_voxels(self._h, buf, cap, C.byref(n)), "fls_get_ndt_voxels")
        a = np.frombuffer(buf, dtype=np.dtype([("key", "<i4", 3), ("estimated", "<i4"), ("num_points", "<i4"), ("carry_count", "<i4"),
                                               ("mu", "<f8", 3), ("info", "<f8", 6)]))[:min(cap, n.value)]
        return {f: a[f].copy() for f in a.dtype.names}

    def iter_log(self, scan: int = 0):
        """Per-iteration H, g, dx, sum_residual, n_valid of scan `scan` of the last Match (needs FLS_FLAG_ITER_LOG)."""
        cap = max(1, self.cfg.max_iterations)
        buf = (FlsIterLog * cap)()
        n = lib().fls_get_iter_log_scan(self._h, int(scan), buf, cap)
        if n < 0:
            check(n, "fls_get_iter_log_scan")
        return [dict(H=np.array(b.H).reshape(6, 6), g=np.array(b.g), dx=np.array(b.dx), sum_residual=b.sum_residual, n_valid=b.n_valid)
                for b in buf[:n]]

    def information(self, scan: int = 0):
        """The information record of scan `scan` of the last Match (needs FLS_FLAG_INFORMATION): dict of H (6x6), g (6), n_valid and
        sum_residual at the returned pose, in the order [dθ; dp] with R <- R·Exp(dθ), p <- p + dp; None when there is no record."""
        rec = FlsInformation()
        check(lib().fls_get_information_scan(self._h, int(scan), C.byref(rec)), "fls_get_information_scan")
        if not rec.valid:
            return None
        return dict(H=np.array(rec.H).reshape(6, 6), g=np.array(rec.g), n_valid=int(rec.n_valid), sum_residual=float(rec.sum_residual))

    def gn_step_probe(self, cases):
        """One Gauss-Newton step (solve, pose update, stop rule) per case on the handle's device: fls_gn_step_probe.  A case is a dict
        with method, max_iterations, min_effective, iter, rot_thres, pos_thres, R (3x3), t (3), last_rot, last_pos and tot (31 totals:
        upper-triangular H row by row, g, n_valid, sum of residuals, candidates, hits).  Returns one dict per case: the post-step
        R, t, dx, H, g, last_rot, last_pos, n_valid, iter, converged, failed, done, the published R / t / stop word, the result record
        (NaN where none was written), spd (the LDL^T fast path accepted the system), det_spd and published_ok."""
        n = len(cases)
        cin = (_abi.FlsGnStepCase * max(n, 1))()
        for c, d in zip(cin, cases):
            c.method, c.max_iterations, c.min_effective, c.iter = int(d["method"]), int(d["max_iterations"]), int(d["min_effective"]), int(d["iter"])
            c.rot_thres, c.pos_thres = float(d["rot_thres"]), float(d["pos_thres"])
            c.R[:] = [float(v) for v in np.asarray(d["R"], np.float64).reshape(9)]
            c.t[:] = [float(v) for v in np.asarray(d["t"], np.float64).reshape(3)]
            c.last_rot, c.last_pos = float(d["last_rot"]), float(d["last_pos"])
            c.tot[:] = [float(v) for v in np.asarray(d["tot"], np.float64).reshape(31)]
        cout = (_abi.FlsGnStepOut * max(n, 1))()
        check(lib().fls_gn_step_probe(self._h, cin, n, cout), "fls_gn_step_probe")
        out = []
        for o in cout[:n]:
            pub = np.array(o.published)
            out.append(dict(R=np.array(o.R).reshape(3, 3), t=np.array(o.t), dx=np.array(o.dx), H=np.array(o.H).reshape(6, 6), g=np.array(o.g),
                            last_rot=o.last_rot, last_pos=o.last_pos, n_valid=o.n_valid, iter=o.iter, converged=o.converged, failed=o.failed,
                            done=o.done, published_R=pub[:9].reshape(3, 3), published_t=pub[9:12], published_stop=pub[12],
                            result=np.array(o.result), spd=bool(o.spd), det_spd=o.det_spd, published_ok=bool(o.published_ok)))
        return out

    def map_info(self) -> FlsMapInfo:
        mi = FlsMapInfo()
        check(lib().fls_get_map_info(self._h, C.byref(mi)), "fls_get_map_info")
        return mi

    def ivox_add_points(self, pts: np.ndarray) -> None:
        """IVoxMap::AddPoints: append map-frame points (LRU at ivox_capacity), no insertion rule."""
        p, n, s, keep = _cloud(pts)
        check(lib().fls_ivox_add_points(self._h, p, n, s), "fls_ivox_add_points")

    def ivox_knn(self, queries: np.ndarray, k: int = 5):
        p, n, s, keep = _cloud(queries)
        out = np.zeros((n, k, 4), np.float32)
        cnt = np.zeros(n, np.int32)
        check(lib().fls_ivox_knn(self._h, p, n, s, k, out.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p)), "fls_ivox_knn")
        return out, cnt

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            lib().fls_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def create_matcher(mode: str, **params) -> Registration:
    """Factory keyed by the reference's mode strings ("PointToPlane_IVOX", "IncrementalNDT", "IcpOptimized", ...)."""
    if mode not in _abi.METHOD_BY_MODE_STRING:
        raise ValueError(f"unknown registration_and_searcher_mode {mode!r}")
    return Registration(_abi.default_config(_abi.METHOD_BY_MODE_STRING[mode], **params))


def gn_step_probe(cases, device: int = 0):
    """Registration.gn_step_probe on a scratch handle of `device` (the step reads nothing of a handle but its device and stream)."""
    cfg = _abi.default_config(_abi.FLS_P2PLANE_IVOX)
    cfg.device = device
    r = Registration(cfg)
    try:
        return r.gn_step_probe(cases)
    finally:
        r.close()


def voxel_grid(points: np.ndarray, leaf: float, device: int = 0) -> np.ndarray:
    """VoxelGridCloud (include/common/pointcloud_utility.h:216-224 upstream) on the device."""
    p, n, s, keep = _cloud(points)
    out = np.empty((max(n, 1), 4), np.float32)
    n_out = C.c_size_t(0)
    check(lib().fls_voxel_grid(device, p, n, s, float(leaf), out.ctypes.data_as(C.c_void_p), C.byref(n_out)), "fls_voxel_grid")
    return out[:n_out.value].copy()


def pcd_write(path: str, cloud: np.ndarray) -> None:
    """pcl::io::savePCDFileBinary of an x y z intensity cloud."""
    c = np.ascontiguousarray(cloud, np.float32)
    assert c.ndim == 2 and c.shape[1] == 4
    check(lib().fls_pcd_write(str(path).encode(), c.ctypes.data_as(C.c_void_p), len(c)), "fls_pcd_write")


def pcd_read(path: str) -> np.ndarray:
    """pcl::io::loadPCDFile into packed x y z intensity records."""
    n = C.c_size_t(0)
    check(lib().fls_pcd_read(str(path).encode(), None, 0, C.byref(n)), "fls_pcd_read")
    out = np.zeros((max(n.value, 1), 4), np.float32)
    check(lib().fls_pcd_read(str(path).encode(), out.ctypes.data_as(C.c_void_p), n.value, C.byref(n)), "fls_pcd_read")
    return out[:n.value]
