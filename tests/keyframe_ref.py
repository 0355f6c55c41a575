"""References for the keyframe-map assembly (fls_keyframes_assemble).

* `assemble_ref`: the oracle composition — orc.voxel_grid per keyframe, orc.transform_f by its pose, concatenation after an optional
  base, an optional final orc.voxel_grid.  No new CPU algorithm: only primitives the oracle already pins.
* `np_voxel_grid` / `np_transform_f`: independent numpy restatements of VoxelGridCloud (PCL 1.10, pointcloud_utility.h:216-224,263-271
  upstream) and TransformPointCloud with R, t cast to float (pointcloud_utility.h:141-158), fp32 throughout, no FMA.
* `save_map_literal`, `GlobalMapLiteral`, `get_submap_literal`: the loops of System::SaveMap (src/slam/system.cpp:299-341),
  System::VisualizeGlobalMap (src/slam/system.cpp:847-896) and LoopClosure::GetSubMap (src/slam/loop_closure.cpp:179-231), line for
  line, over any VoxelGridCloud / TransformPointCloud pair.
"""
from __future__ import annotations

import numpy as np

EMPTY = np.zeros((0, 4), np.float32)


def _orc():
    from oracle import pyoracle as orc
    return orc


def orc_voxel(c, leaf):
    return _orc().voxel_grid(c, leaf) if len(c) else EMPTY.copy()


def orc_transform(c, T):
    return _orc().transform_f(c, T) if len(c) else EMPTY.copy()


def _cat(parts):
    parts = [np.asarray(p, np.float32).reshape(-1, 4) for p in parts]
    return np.ascontiguousarray(np.concatenate(parts, 0)) if parts else EMPTY.copy()


def assemble_ref(clouds, ids, poses, leaf, final_leaf=None, base=None):
    """[base] ++ concat_k transform_f(voxel_grid(clouds[ids[k]], leaf), poses[k]); then voxel_grid(., final_leaf) if final_leaf."""
    parts = [base] if base is not None else []
    for i, T in zip(ids, poses):
        parts.append(orc_transform(orc_voxel(clouds[i], leaf), T))
    m = _cat(parts)
    if final_leaf:
        m = orc_voxel(m, final_leaf)
    return m


def np_voxel_grid(pts, leaf):
    pts = np.ascontiguousarray(pts, np.float32)
    if len(pts) == 0:
        return EMPTY.copy()
    inv = np.float32(1.0) / np.float32(leaf)
    xyz = pts[:, :3]
    mn, mx = xyz.min(0), xyz.max(0)
    d = [int(np.float32(mx[a] - mn[a]) * inv) + 1 for a in range(3)]
    if d[0] * d[1] * d[2] > 2147483647:
        return pts.copy()
    minb = np.floor(mn * inv).astype(np.int64)
    divb = np.floor(mx * inv).astype(np.int64) - minb + 1
    cell = (np.floor(xyz * inv) - minb.astype(np.float32)).astype(np.int64)
    lin = (cell[:, 0] + cell[:, 1] * divb[0] + cell[:, 2] * divb[0] * divb[1]) & 0xffffffff
    order = np.argsort(lin, kind="stable")
    sl = lin[order]
    starts = np.flatnonzero(np.r_[True, sl[1:] != sl[:-1]])
    counts = np.diff(np.r_[starts, len(sl)])
    acc = np.zeros((len(starts), 4), np.float32)
    for k in range(int(counts.max())):  # sequential fp32 sums in input order, all cells at once
        live = counts > k
        acc[live] += pts[order[starts[live] + k]]
    return acc / counts.astype(np.float32)[:, None]


def np_transform_f(pts, T):
    pts = np.asarray(pts, np.float32).reshape(-1, 4)
    R = np.asarray(T, np.float64)[:3, :3].astype(np.float32)
    t = np.asarray(T, np.float64)[:3, 3].astype(np.float32)
    out = pts.copy()
    for r in range(3):
        out[:, r] = ((R[r, 0] * pts[:, 0] + R[r, 1] * pts[:, 1]) + R[r, 2] * pts[:, 2]) + t[r]
    return out


def save_map_literal(clouds, poses, voxel=orc_voxel, transform=orc_transform):
    """System::SaveMap, system.cpp:306-316: None for no keyframe, else the map it writes with savePCDFileBinary."""
    if len(clouds) == 0:
        return None
    map_cloud = EMPTY.copy()
    for cloud, pose in zip(clouds, poses):
        cloud = voxel(cloud, 0.3)
        map_cloud = _cat([map_cloud, transform(cloud, pose)])
    return voxel(map_cloud, 0.3)


class GlobalMapLiteral:
    """System::VisualizeGlobalMap, system.cpp:847-896: `round(clouds, poses, need_update)` is one pass of the while loop after the
    subscriber check; it returns the published global_map or None."""

    def __init__(self, resolution, voxel=orc_voxel, transform=orc_transform):
        self.global_map = EMPTY.copy()
        self.last_frame_id = -1
        self.res = resolution
        self.voxel, self.transform = voxel, transform

    def round(self, clouds, poses, need_update=False):
        if need_update:
            self.global_map = EMPTY.copy()
            self.last_frame_id = -1
        if len(clouds) == 0 or self.last_frame_id + 1 >= len(clouds) - 1:  # keyframes_.back()->id_ == size - 1
            return None
        keyframes = list(range(self.last_frame_id + 1, len(clouds)))
        self.last_frame_id = len(clouds) - 1
        temp_local_cloud = EMPTY.copy()
        for i in keyframes:
            temp_local_cloud = _cat([temp_local_cloud, self.transform(self.voxel(clouds[i], self.res), poses[i])])
        self.global_map = _cat([self.global_map, temp_local_cloud])
        self.global_map = self.voxel(self.global_map, self.res)
        return self.global_map


def get_submap_literal(clouds, poses, keyframe_id, left_range, right_range, use_local_pose, voxel=orc_voxel, transform=orc_transform):
    """LoopClosure::GetSubMap, loop_closure.cpp:179-231 (numpy's inverse for Eigen's)."""
    local_map, ps = [], []
    ref_pose = np.asarray(poses[keyframe_id], np.float64)
    for i in range(-left_range, right_range + 1):
        k = keyframe_id + i
        if k < 0 or k >= len(clouds):
            continue
        local_map.append(clouds[k])
        ps.append(np.asarray(poses[k], np.float64))
    if use_local_pose:
        ref_pose_inv = np.linalg.inv(ref_pose)
        ps = [ref_pose_inv @ p for p in ps]
    local_map = [voxel(c, 0.2) for c in local_map]
    out = EMPTY.copy()
    for c, p in zip(local_map, ps):
        out = _cat([out, transform(c, p)])
    return out
