"""CPU checks of the keyframe store (fls_keyframes_*): argument checks that fail before any device is touched, the header-only adapter
(funny_lidar_slam_b200/shim/b200_keyframe_map.h) compiled against stand-ins of the reference headers it includes, its citations, and
the literal restatements of the three upstream loops in tests/keyframe_ref.py against the oracle composition they all reduce to."""
import ctypes as C
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

from funny_lidar_slam_b200 import _abi, _lib
from funny_lidar_slam_b200._abi import FlsMatchStats
from tests import keyframe_ref as ref
from tests.test_citations import GOLDEN, PAT, ROOT

SHIM = os.path.join(ROOT, "funny_lidar_slam_b200", "shim", "b200_keyframe_map.h")


# ---- argument checks ----------------------------------------------------------------------------------------------------------
def test_create_checks_arguments_then_needs_a_device():
    L = _lib.lib()
    s = C.c_void_p()
    assert L.fls_keyframes_create(0, 1000, None) == _abi.FLS_ERR_INVALID_ARG
    assert L.fls_keyframes_create(0, 0, C.byref(s)) == _abi.FLS_ERR_INVALID_ARG
    assert L.fls_keyframes_create(0, 1 << 32, C.byref(s)) == _abi.FLS_ERR_INVALID_ARG
    assert L.fls_keyframes_create(-1, 1000, C.byref(s)) == _abi.FLS_ERR_NO_DEVICE
    if L.fls_device_count() == 0:
        assert L.fls_keyframes_create(0, 1000, C.byref(s)) == _abi.FLS_ERR_NO_DEVICE
        assert not s.value


def test_entries_reject_a_null_store():
    L = _lib.lib()
    pts = np.zeros((4, 4), np.float32)
    p = pts.ctypes.data_as(C.c_void_p)
    assert L.fls_keyframes_add(None, 0, p, 4, 16) == _abi.FLS_ERR_INVALID_ARG
    assert L.fls_keyframes_add_device(None, 0, p, 4) == _abi.FLS_ERR_INVALID_ARG
    n = C.c_size_t(7)
    assert L.fls_keyframes_count(None, C.byref(n), None) == _abi.FLS_ERR_INVALID_ARG
    ids = np.zeros(1, np.int64)
    T = np.eye(4).ravel()
    st = FlsMatchStats()
    assert L.fls_keyframes_assemble(None, ids.ctypes.data_as(C.c_void_p), 1, T.ctypes.data_as(C.c_void_p), 0.3, 0.3, None, 0, p, None, 4,
                                    C.byref(n), C.byref(st)) == _abi.FLS_ERR_INVALID_ARG
    assert n.value == 0
    assert L.fls_keyframes_assemble(None, None, 0, None, 0.3, 0.0, None, 0, None, None, 0, None, None) == _abi.FLS_ERR_INVALID_ARG
    L.fls_keyframes_destroy(None)


# ---- the adapter ----------------------------------------------------------------------------------------------------------------
MOCKS = {
    "glog/logging.h": """
#pragma once
struct NullStream { template <class T> NullStream& operator<<(const T&) { return *this; } };
#define CHECK_EQ(a, b) ((a) == (b) ? NullStream() : NullStream())
#define LOG(x) NullStream()
""",
    "cuda_runtime_api.h": """
#pragma once
#include <cstddef>
typedef int cudaError_t;
static const cudaError_t cudaSuccess = 0;
cudaError_t cudaMalloc(void** p, size_t bytes);
cudaError_t cudaFree(void* p);
""",
    "common/data_type.h": """
#pragma once
#include <cstdint>
#include <memory>
#include <vector>
struct alignas(16) PCLPointXYZI { float x, y, z, pad; float intensity, p1, p2, p3; };
struct PCLPointCloudXYZI {
    using Ptr = std::shared_ptr<PCLPointCloudXYZI>;
    std::vector<PCLPointXYZI> points;
    uint32_t width = 0, height = 0;
    size_t size() const { return points.size(); }
};
struct Mat4d {
    double m[16];
    double* data() { return m; }
    const double* data() const { return m; }
    Mat4d inverse() const { return *this; }
    Mat4d operator*(const Mat4d& o) const { return o; }
};
""",
    "common/keyframe.h": """
#pragma once
#include "common/data_type.h"
struct KeyFrame {
    using Ptr = std::shared_ptr<KeyFrame>;
    using ID = int;
    ID id_ = -1;
    Mat4d pose_{};
};
""",
}

USER = """
#include "b200_keyframe_map.h"
size_t use(const std::vector<KeyFrame::Ptr>& keyframes, const PCLPointCloudXYZI& ordered, const float* d_ordered) {
    B200KeyFrameMap store(0, 1000000);
    bool ok = store.AddKeyFrame(0, ordered);
    ok = ok && store.AddKeyFrameDevice(1, d_ordered, 10);
    const size_t n = store.SaveMap(keyframes, "/tmp/map.pcd");
    PCLPointCloudXYZI::Ptr sub = store.GetSubMap(keyframes, 1, 10, 10, true);
    B200KeyFrameMap::GlobalMap global_map(store, 0.5f);
    PCLPointCloudXYZI::Ptr g = global_map.Round(keyframes, false);
    return n + (ok ? 1 : 0) + (sub ? sub->size() : 0) + (g ? g->size() : 0);
}
"""


def test_adapter_compiles_against_the_reference_types(tmp_path):
    gxx = shutil.which("g++") or "/usr/bin/g++"
    if not os.path.exists(gxx):
        pytest.skip("no C++ compiler")
    for rel, body in MOCKS.items():
        p = tmp_path / "mock" / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(body)
    (tmp_path / "user.cpp").write_text(USER)
    cmd = [gxx, "-std=c++17", "-Wall", "-Wextra", "-Werror", "-Wno-unused-parameter", "-fsyntax-only", "-I", str(tmp_path / "mock"),
           "-I", os.path.join(ROOT, "include"), "-I", os.path.dirname(SHIM), str(tmp_path / "user.cpp")]
    env = dict(os.environ)
    env.pop("CXX", None)
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr


def test_adapter_citations_resolve():
    with open(GOLDEN) as fh:
        counts = json.load(fh)
    files = {}
    for rel in counts:
        files.setdefault(os.path.basename(rel), []).append(rel)
    srcs = [SHIM, os.path.join(ROOT, "funny_lidar_slam_b200", "keyframes.py"), os.path.join(ROOT, "tests", "keyframe_ref.py")]
    checked, bad = 0, []
    for src in srcs:
        for m in PAT.finditer(open(src).read()):
            path, last = m.group(1), int(m.group(3) or m.group(2))
            if os.path.basename(path).startswith(("fls_", "orc_", "b200_")):
                continue
            checked += 1
            cands = files.get(os.path.basename(path), [])
            if "/" in path:
                cands = [c for c in cands if ("/" + c).endswith("/" + path.lstrip("./"))] or cands
            if not cands or max(counts[c] for c in cands) < last:
                bad.append((os.path.basename(src), m.group(0)))
    assert checked > 10
    assert not bad, bad


# ---- literal restatements of the upstream loops vs the oracle composition -------------------------------------------------------
def _keyframes(rng, k=7, n=3000):
    clouds, poses = [], []
    for i in range(k):
        m = 0 if i == 3 else int(rng.integers(1, n))
        c = np.concatenate([rng.uniform(-20, 20, (m, 3)), rng.uniform(0, 255, (m, 1))], 1).astype(np.float32)
        clouds.append(c)
        a = rng.uniform(-np.pi, np.pi)
        T = np.eye(4)
        T[:3, :3] = [[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]]
        T[:3, 3] = rng.uniform(-50, 50, 3)
        poses.append(T)
    return clouds, np.array(poses)


def _same(a, b):
    return a.shape == b.shape and np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


def test_numpy_restatements_agree_with_the_oracle_primitives():
    rng = np.random.default_rng(11)
    clouds, poses = _keyframes(rng)
    for c, T in zip(clouds, poses):
        for leaf in (0.2, 0.3, 1.0):
            assert _same(ref.np_voxel_grid(c, leaf), ref.orc_voxel(c, leaf))
        assert _same(ref.np_transform_f(c, T), ref.orc_transform(c, T))
    wide = np.concatenate([rng.uniform(-400, 400, (500, 3)), np.ones((500, 1))], 1).astype(np.float32)
    assert _same(ref.np_voxel_grid(wide, 0.01), wide) and _same(ref.orc_voxel(wide, 0.01), wide)


@pytest.mark.parametrize("voxel,transform", [(ref.orc_voxel, ref.orc_transform), (ref.np_voxel_grid, ref.np_transform_f)])
def test_save_map_loop_is_the_composition(voxel, transform):
    rng = np.random.default_rng(5)
    clouds, poses = _keyframes(rng)
    got = ref.save_map_literal(clouds, poses, voxel, transform)
    assert _same(got, ref.assemble_ref(clouds, range(len(clouds)), poses, 0.3, 0.3))
    assert ref.save_map_literal([], []) is None


@pytest.mark.parametrize("voxel,transform", [(ref.orc_voxel, ref.orc_transform), (ref.np_voxel_grid, ref.np_transform_f)])
def test_global_map_rounds_are_the_composition(voxel, transform):
    rng = np.random.default_rng(6)
    clouds, poses = _keyframes(rng, k=9)
    vis = ref.GlobalMapLiteral(0.5, voxel, transform)
    base, last = None, -1
    for k, upd in ((1, False), (2, False), (3, False), (6, False), (7, False), (9, False), (9, True)):
        if upd:
            poses = poses.copy()
            poses[:, :3, 3] += 0.37
            base, last = None, -1
        got = vis.round(clouds[:k], poses[:k], upd)
        if k == 0 or last + 1 >= k - 1:
            assert got is None
            continue
        ids = list(range(last + 1, k))
        base = ref.assemble_ref(clouds, ids, poses[ids], 0.5, 0.5, base)
        last = k - 1
        assert _same(got, base)


@pytest.mark.parametrize("use_local_pose", [False, True])
def test_submap_loop_is_the_composition(use_local_pose):
    rng = np.random.default_rng(8)
    clouds, poses = _keyframes(rng, k=9)
    for kf, left, right in ((4, 2, 2), (0, 3, 1), (8, 1, 5), (2, 10, 10)):
        got = ref.get_submap_literal(clouds, poses, kf, left, right, use_local_pose)
        ids = [i for i in range(kf - left, kf + right + 1) if 0 <= i < len(clouds)]
        P = [np.linalg.inv(poses[kf]) @ poses[i] if use_local_pose else poses[i] for i in ids]
        assert _same(got, ref.assemble_ref(clouds, ids, P, 0.2))
        got_np = ref.get_submap_literal(clouds, poses, kf, left, right, use_local_pose, ref.np_voxel_grid, ref.np_transform_f)
        assert _same(got_np, got)
