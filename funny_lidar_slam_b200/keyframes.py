"""Keyframe maps on the device (fls_keyframes_*, include/fls_b200.h).

`KeyFrameStore` keeps the ordered cloud of every keyframe in device memory, indexed by keyframe id as System::keyframes_ is
(include/slam/system.h:187 upstream), and `assemble` rebuilds a point map from a selection of them in one device call:

    map = [base] ++ concat_k TransformPointCloud(VoxelGridCloud(cloud[ids[k]], leaf), T[k])
    if final_leaf: map = VoxelGridCloud(map, final_leaf)

The three helpers below restate the upstream sites that run this primitive: `save_map_cloud` (System::SaveMap,
src/slam/system.cpp:299-341), `global_map_round` (one round of System::VisualizeGlobalMap, src/slam/system.cpp:847-896) and
`loopclosure_submap` (LoopClosure::GetSubMap, src/slam/loop_closure.cpp:179-231).  Poses are (4, 4) float64 matrices, one per
keyframe id; clouds are (n,4) packed x,y,z,intensity or (n,8) pcl::PointXYZI float32 records.

Place recognition by Scan Context (include/fls_b200.h, DESIGN.md §3.12): `detect_loop` is LoopClosure::DetectByFeature
(src/slam/loop_closure.cpp:62-64, a stub upstream) and `place_query` finds the keyframe a scan was taken near.  Each returns
PlaceMatch records ordered by (distance, id); `place_pose` turns one into the coarse pose T_kf @ Rz(yaw) that fls_relocalize refines.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._abi import FlsMatchStats, FlsPlaceMatch, FlsScCfg
from ._lib import check, lib
from .registration import _batch_poses, _cloud


def sc_cfg(n_rings: int = 20, n_sectors: int = 60, max_radius: float = 80.0, z_offset: float = 2.0) -> FlsScCfg:
    """fls_sc_cfg; the defaults are the paper's 20 rings x 60 sectors out to 80 m, with z lifted by the sensor height."""
    c = FlsScCfg()
    c.n_rings, c.n_sectors, c.max_radius, c.z_offset = int(n_rings), int(n_sectors), float(max_radius), float(z_offset)
    return c


def place_pose(T_keyframe, yaw: float) -> np.ndarray:
    """The coarse world pose of a query matched to a keyframe at pose T_keyframe with relative yaw `yaw`: T_keyframe @ Rz(yaw)."""
    Rz = np.eye(4)
    Rz[:2, :2] = [[np.cos(yaw), -np.sin(yaw)], [np.sin(yaw), np.cos(yaw)]]
    return np.asarray(T_keyframe, np.float64) @ Rz


class KeyFrameStore:
    """Device-resident keyframe clouds: an arena of `capacity_points` records on `device`, fixed at creation."""

    def __init__(self, capacity_points: int, device: int = 0):
        self.device = int(device)
        self._s = C.c_void_p()
        check(lib().fls_keyframes_create(self.device, int(capacity_points), C.byref(self._s)), "fls_keyframes_create")
        self._sizes: list[int] = []
        self.last_stats = FlsMatchStats()
        self.last_count = 0

    def close(self) -> None:
        if self._s:
            lib().fls_keyframes_destroy(self._s)
            self._s = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __len__(self) -> int:
        n = C.c_size_t(0)
        check(lib().fls_keyframes_count(self._s, C.byref(n), None), "fls_keyframes_count")
        return n.value

    @property
    def n_points(self) -> int:
        n = C.c_size_t(0)
        check(lib().fls_keyframes_count(self._s, None, C.byref(n)), "fls_keyframes_count")
        return n.value

    def add(self, cloud, id: int | None = None) -> int:
        """Append a keyframe's ordered cloud from host memory; `id` defaults to the next one.  Returns the id."""
        kf = len(self._sizes) if id is None else int(id)
        p, n, s, keep = _cloud(cloud)
        check(lib().fls_keyframes_add(self._s, kf, p, n, s), "fls_keyframes_add")
        self._sizes.append(n)
        return kf

    def add_device(self, d_points: int, n: int, id: int | None = None) -> int:
        """Append a keyframe's ordered cloud from device memory (n packed float4 records at address d_points, on the store's device)."""
        kf = len(self._sizes) if id is None else int(id)
        check(lib().fls_keyframes_add_device(self._s, kf, C.c_void_p(int(d_points)) if d_points else None, int(n)), "fls_keyframes_add_device")
        self._sizes.append(int(n))
        return kf

    def assemble(self, ids, poses, leaf: float, final_leaf: float | None = None, base=None, device_out=None, host_out: bool = True):
        """The map of keyframes `ids` at `poses` (one (4, 4) pose per id).  base=(d_ptr, n): device records placed first.
        device_out=(d_ptr, capacity): device buffer that receives the map.  Returns the map as (n,4) float32 (None with
        host_out=False); self.last_count is its size, self.last_stats the call's fls_match_stats."""
        ids = np.ascontiguousarray(np.asarray(ids, np.int64).reshape(-1))
        Tc = _batch_poses(np.asarray(poses, np.float64).reshape(-1, 4, 4))
        if len(Tc) != len(ids):
            raise ValueError("one pose per selected keyframe")
        if len(ids) and (ids.min() < 0 or ids.max() >= len(self._sizes)):
            raise IndexError("keyframe id out of range")
        d_base, n_base = (int(base[0]), int(base[1])) if base is not None else (0, 0)
        if device_out is not None:
            d_out, cap = int(device_out[0]), int(device_out[1])
        else:
            d_out, cap = 0, n_base + sum(self._sizes[i] for i in ids.tolist())  # the map never has more records than its inputs
        out = np.empty((max(cap, 1), 4), np.float32) if host_out else None
        if out is None and not d_out:
            cap = 0
        n_out = C.c_size_t(0)
        st = FlsMatchStats()
        vp = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
        dp = lambda a: C.c_void_p(a) if a else None
        rc = lib().fls_keyframes_assemble(self._s, vp(ids), len(ids), vp(Tc), float(leaf), float(final_leaf or 0.0), dp(d_base), n_base, vp(out),
                                          dp(d_out), cap, C.byref(n_out), C.byref(st))
        self.last_count = n_out.value
        check(rc, "fls_keyframes_assemble")
        self.last_stats = st
        return out[:n_out.value].copy() if host_out else None

    # -- place recognition (Scan Context) ---------------------------------------------------------------------------------------
    def scan_context(self, ids, cfg: FlsScCfg | None = None) -> np.ndarray:
        """The descriptors of keyframes `ids` as (len(ids), n_rings, n_sectors) float32."""
        c = cfg or sc_cfg()
        ids = np.ascontiguousarray(np.asarray(ids, np.int64).reshape(-1))
        out = np.empty((len(ids), c.n_rings, c.n_sectors), np.float32)
        check(lib().fls_keyframes_scan_context(self._s, C.byref(c), ids.ctypes.data_as(C.c_void_p), len(ids), out.ctypes.data_as(C.c_void_p)),
              "fls_keyframes_scan_context")
        return out

    def _matches(self, call, k: int, where: str):
        buf = (FlsPlaceMatch * max(int(k), 1))()
        n = C.c_size_t(0)
        st = FlsMatchStats()
        check(call(int(k), buf, C.byref(n), C.byref(st)), where)
        self.last_stats = st
        return buf[:n.value]

    def detect_loop(self, query_id: int, min_span: int, k: int = 1, cfg: FlsScCfg | None = None):
        """LoopClosure::DetectByFeature: the k stored keyframes with query_id - id > min_span nearest to keyframe query_id, as
        FlsPlaceMatch records ordered by (distance, id).  No distance threshold is applied."""
        c = cfg or sc_cfg()
        return self._matches(lambda k_, b, n, st: lib().fls_keyframes_detect_loop(self._s, C.byref(c), int(query_id), int(min_span), k_, b, n, st), k,
                             "fls_keyframes_detect_loop")

    def place_query(self, cloud, k: int = 1, cfg: FlsScCfg | None = None, return_desc: bool = False):
        """The k stored keyframes nearest to the scan `cloud` ((n,4) or (n,8) float32, sensor frame).  With return_desc, also the
        scan's descriptor: (matches, (n_rings, n_sectors) float32)."""
        c = cfg or sc_cfg()
        p, n, s, keep = _cloud(cloud)
        desc = np.empty((c.n_rings, c.n_sectors), np.float32)
        dp = desc.ctypes.data_as(C.c_void_p) if return_desc else None
        m = self._matches(lambda k_, b, n_, st: lib().fls_keyframes_place_query(self._s, C.byref(c), p, n, s, k_, b, n_, dp, st), k,
                          "fls_keyframes_place_query")
        return (m, desc) if return_desc else m

    def place_query_device(self, d_points: int, n: int, k: int = 1, cfg: FlsScCfg | None = None, return_desc: bool = False):
        """place_query with a scan of n packed float4 records in device memory on the store's device."""
        c = cfg or sc_cfg()
        desc = np.empty((c.n_rings, c.n_sectors), np.float32)
        dp = desc.ctypes.data_as(C.c_void_p) if return_desc else None
        d = C.c_void_p(int(d_points)) if d_points else None
        m = self._matches(lambda k_, b, n_, st: lib().fls_keyframes_place_query_device(self._s, C.byref(c), d, int(n), k_, b, n_, dp, st), k,
                          "fls_keyframes_place_query_device")
        return (m, desc) if return_desc else m


def save_map_cloud(store: KeyFrameStore, poses, leaf: float = 0.3, final_leaf: float = 0.3):
    """System::SaveMap (src/slam/system.cpp:299-341 upstream) up to savePCDFileBinary: every keyframe VoxelGridCloud(ordered, 0.3),
    TransformPointCloud by its pose, concatenated, then VoxelGridCloud(map, 0.3).  None when there is no keyframe (upstream returns
    false, :306-308)."""
    n = len(store)
    if n == 0:
        return None
    return store.assemble(np.arange(n), np.asarray(poses)[:n], leaf, final_leaf)


class GlobalMapState:
    """What System::VisualizeGlobalMap keeps between its rounds (src/slam/system.cpp:851-852): the running global_map, held on the
    device in two buffers used in turn (one is the base of a round, the other receives its result), and last_frame_id."""

    def __init__(self, device: int = 0):
        self.device = int(device)
        self.last_frame_id = -1
        self.n = 0
        self._bufs = [None, None]
        self._cur = 0

    def reset(self) -> None:
        self.n = 0
        self.last_frame_id = -1

    def _buffer(self, i: int, records: int):
        import torch
        b = self._bufs[i]
        if b is None or b.shape[0] < records:
            b = torch.empty((max(records, 1), 4), dtype=torch.float32, device=f"cuda:{self.device}")
            self._bufs[i] = b
        return b


def global_map_round(store: KeyFrameStore, state: GlobalMapState, poses, resolution: float, need_update: bool = False):
    """One round of System::VisualizeGlobalMap (src/slam/system.cpp:864-893 upstream), after its subscriber check: a pending pose
    update (need_update_global_map_visualization_, set after every loop-closure optimisation, :720) clears the map and restarts
    from keyframe 0; the keyframes since last_frame_id are filtered at `resolution`, transformed, appended to global_map and the
    whole map is filtered again.  Returns the published global_map as (n,4) float32, or None when the round publishes nothing
    (upstream's `continue` at :874-876 — note it waits for two new keyframes)."""
    if need_update:
        state.reset()
    count = len(store)
    if count == 0 or state.last_frame_id + 1 >= count - 1:
        return None
    ids = np.arange(state.last_frame_id + 1, count)
    state.last_frame_id = count - 1
    cap = state.n + sum(store._sizes[i] for i in ids.tolist())
    base = state._bufs[state._cur] if state.n else None
    nxt = state._buffer(1 - state._cur, cap)
    out = store.assemble(ids, np.asarray(poses)[ids], resolution, resolution, base=(base.data_ptr(), state.n) if base is not None else None,
                         device_out=(nxt.data_ptr(), nxt.shape[0]))
    state._cur = 1 - state._cur
    state.n = store.last_count
    return out


def loopclosure_submap(store: KeyFrameStore, poses, keyframe_id: int, left: int, right: int, use_local_pose: bool, leaf: float = 0.2):
    """LoopClosure::GetSubMap (src/slam/loop_closure.cpp:179-231 upstream): keyframes keyframe_id-left .. keyframe_id+right, clipped
    to the keyframe range (:194-200), each VoxelGridCloud(., 0.2) and transformed by its pose — relative to the reference keyframe
    with use_local_pose (:210-215; numpy's inverse stands in for Eigen's here) — and concatenated, with no final filter."""
    poses = np.asarray(poses, np.float64)
    n = len(store)
    ids = [keyframe_id + i for i in range(-left, right + 1) if 0 <= keyframe_id + i < n]
    P = [poses[k] for k in ids]
    if use_local_pose:
        ref_pose_inv = np.linalg.inv(poses[keyframe_id])
        P = [ref_pose_inv @ p for p in P]
    return store.assemble(ids, np.asarray(P, np.float64).reshape(-1, 4, 4), leaf)
