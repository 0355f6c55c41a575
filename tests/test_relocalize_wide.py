"""fls_relocalize_wide without a device: argument checks, the caps of its grid, the blocks of its levels, the shim's RelocalizeWide, and
the slack of its lower bound against fp32-emulated transforms and distances (tests/reloc_wide_ref.py)."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from funny_lidar_slam_b200 import _abi, _lib
from funny_lidar_slam_b200.registration import reloc_cfg
from tests import reloc_ref, reloc_wide_ref, test_shim_compiles

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _call(cfg, h=None, n=0, stride=16, device=False):
    L = _lib.lib()
    T = (C.c_double * 16)(*np.eye(4).T.ravel())
    r = _abi.FlsRelocResult()
    ev = C.c_int64(0)
    if device:
        return L.fls_relocalize_wide_device(h, None, n, C.byref(cfg) if cfg else None, T, C.byref(r), None, None, None, None, C.byref(ev))
    return L.fls_relocalize_wide(h, None, n, stride, C.byref(cfg) if cfg else None, T, C.byref(r), None, None, None, None, C.byref(ev))


@pytest.mark.parametrize("device", [False, True])
def test_argument_checks(device):
    assert _call(reloc_cfg(), device=device) == _abi.FLS_ERR_INVALID_ARG  # no handle
    assert _call(None, device=device) == _abi.FLS_ERR_INVALID_ARG
    assert _call(reloc_cfg(), n=5, device=device) == _abi.FLS_ERR_INVALID_ARG  # NULL scan with points
    if not device:
        assert _call(reloc_cfg(), stride=12) == _abi.FLS_ERR_INVALID_ARG


def test_grid_caps():
    # the 0.5 m x 2 degree search over +-40 m and the full circle: past fls_relocalize's cap, inside this one
    g = reloc_wide_ref.grid(40.0, 0.5, np.pi, np.deg2rad(2.0))
    assert (g.I, g.n_yaw, g.P) == (80, 180, 161 * 161 * 180) and g.P == 4665780
    with pytest.raises(ValueError):
        reloc_ref.grid(40.0, 0.5, np.pi, np.deg2rad(2.0))
    # 2^31 hypotheses exactly (the full circle in 2^31 steps) and one step more
    assert reloc_wide_ref.grid(0.0, 1.0, np.pi, np.pi / 2 ** 30).P == 1 << 31
    with pytest.raises(ValueError):
        reloc_wide_ref.grid(0.0, 1.0, np.pi, np.pi / (2 ** 30 + 1))
    # x-y: 46339^2 fits 2^31, 46341^2 does not; the 32767-step cap is reached before the hypothesis cap only with more yaws than 0
    assert reloc_wide_ref.grid(23169.0, 1.0, 0.0, 1.0).P == 46339 ** 2
    with pytest.raises(ValueError):
        reloc_wide_ref.grid(23170.0, 1.0, 0.0, 1.0)
    with pytest.raises(ValueError):
        reloc_wide_ref.grid(32768.0, 1.0, 0.0, 1.0)
    # and the grid itself is fls_relocalize's wherever both accept it
    for args in [(10.0, 1.0, np.pi, np.deg2rad(10.0)), (0.3, 0.1, 0.5, 0.2), (0.0, 1.0, 0.0, 1.0)]:
        assert reloc_wide_ref.grid(*args) == reloc_ref.grid(*args)


def test_start_level():
    assert reloc_wide_ref.start_level(reloc_wide_ref.grid(10.0, 0.5, np.pi, np.deg2rad(5.0))) == 0  # 121 032: every leaf scored
    assert reloc_wide_ref.start_level(reloc_wide_ref.grid(40.0, 0.5, np.pi, np.deg2rad(2.0))) == 1  # 81 * 81 * 90 blocks
    assert reloc_wide_ref.start_level(reloc_wide_ref.grid(0.0, 1.0, np.pi, np.pi / 2 ** 30)) == 11


@pytest.mark.parametrize("n,level", [(1, 0), (7, 1), (8, 2), (9, 2), (161, 1), (161, 3), (180, 4), (5, 5)])
def test_blocks_partition_an_axis_around_their_representatives(n, level):
    seen = []
    for b in range(reloc_wide_ref.blocks(n, level)):
        r, h = reloc_wide_ref.block_rep(b, level, n)
        members = [i for i in range(n) if i >> level == b]
        assert r in members and max(abs(i - r) for i in members) == h
        assert h <= max(1 << (level - 1), 0) if level else h == 0
        seen += members
    assert seen == list(range(n))


USER = """
#include "b200_registration.h"
bool init(const fls_config& cfg, const PointcloudClusterPtr& cluster, Mat4d& T) {
    B200Registration m(cfg);
    fls_reloc_cfg rc{40.0, 0.5, 3.14159265358979, 0.0349066, 1.0f, 2.0f, 1.0f, 64};
    float fitness = 0.f;
    return m.RelocalizeWide(cluster, T, rc, &fitness) && fitness < 1.0f;
}
"""


def test_shim_relocalize_wide_compiles(tmp_path):
    gxx = shutil.which("g++") or "/usr/bin/g++"
    if not os.path.exists(gxx):
        pytest.skip("no g++")
    for rel, body in test_shim_compiles.MOCKS.items():
        p = tmp_path / "mock" / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(body)
    (tmp_path / "user.cpp").write_text(USER)
    cmd = [gxx, "-std=c++17", "-Wall", "-Wextra", "-Werror", "-Wno-unused-parameter", "-fsyntax-only", "-I", str(tmp_path / "mock"),
           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "funny_lidar_slam_b200", "shim"), str(tmp_path / "user.cpp")]
    env = dict(os.environ)
    env.pop("CXX", None)
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr


def _rot(yaw, roll, pitch):
    cz, sz, cx, sx, cy, sy = np.cos(yaw), np.sin(yaw), np.cos(roll), np.sin(roll), np.cos(pitch), np.sin(pitch)
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    return Rz @ Ry @ Rx


@pytest.mark.parametrize("offset", [0.0, 100.0, 1000.0, 10000.0])
def test_slack_bounds_every_leaf_of_a_block(offset):
    """For random guesses up to `offset` metres from the origin, random grids, blocks, representatives and leaves of the block, and
    fit points placed within sqrt(max_range) of the leaf's fp32 point (where the gate does not hide an error): the leaf's gated fp32
    term is never below the bound's term computed from the representative's fp32 point."""
    rng = np.random.default_rng(int(offset) + 7)
    worst, n_checked = np.inf, 0
    for trial in range(300):
        T = np.eye(4)
        T[:3, :3] = _rot(rng.uniform(-np.pi, np.pi), rng.normal(0, 0.05), rng.normal(0, 0.05))
        T[:3, 3] = rng.uniform(-1, 1, 3) * offset + rng.normal(0, 3, 3)
        xy_step, yaw_step = rng.choice([0.1, 0.25, 0.5, 1.0]), np.deg2rad(rng.choice([0.5, 1.0, 2.0, 5.0, 10.0]))
        g = reloc_wide_ref.grid(rng.uniform(0.0, 40.0), xy_step, np.pi, yaw_step)
        nx, max_range = 2 * g.I + 1, float(rng.choice([0.5, 2.0, 4.0]))
        level = int(rng.integers(1, 6))
        b = [int(rng.integers(0, reloc_wide_ref.blocks(n, level))) for n in (nx, nx, g.n_yaw)]
        (rx, hx), (ry, hy), (rk, hk) = (reloc_wide_ref.block_rep(bb, level, n) for bb, n in zip(b, (nx, nx, g.n_yaw)))
        lx, ly, lk = (int(rng.integers(bb << level, min((bb + 1) << level, n))) for bb, n in zip(b, (nx, nx, g.n_yaw)))
        T_rep = reloc_wide_ref.leaf_pose(T, g, xy_step, yaw_step, rx, ry, rk)
        T_leaf = reloc_wide_ref.leaf_pose(T, g, xy_step, yaw_step, lx, ly, lk)
        p = (rng.normal(0, 1, (64, 3)) * rng.choice([1.0, 10.0, 60.0], (64, 1))).astype(np.float32)
        q_rep, q_leaf = reloc_wide_ref.moved(p, T_rep), reloc_wide_ref.moved(p, T_leaf)
        fit = (q_leaf.astype(np.float64) + rng.normal(0, 1, (64, 3)) * rng.uniform(0, np.sqrt(max_range), (64, 1))).astype(np.float32)
        tau = max(max(abs(T[0, 3]), abs(T[1, 3])) + g.I * xy_step, abs(T[2, 3]))
        lb = reloc_wide_ref.bound_terms(q_rep, fit, p, T[:3, :3], hx, hy, hk, xy_step, yaw_step, tau, max_range)
        leaf = reloc_wide_ref.leaf_terms(q_leaf, fit, max_range)
        assert np.all(leaf >= lb), (trial, np.min(leaf - lb))
        # the tightest the bound gets: a leaf that is its block's representative moves no point, so only eps_i separates the terms
        lb0 = reloc_wide_ref.bound_terms(q_leaf, fit, p, T[:3, :3], 0, 0, 0, xy_step, yaw_step, tau, max_range)
        assert np.all(leaf >= lb0), (trial, np.min(leaf - lb0))
        inside = leaf < float(np.float32(max_range))
        if inside.any():
            worst = min(worst, float(np.min((leaf - lb0)[inside])))
        n_checked += 2 * len(p)
    print(f"offset {offset:g} m: {n_checked} point terms, smallest leaf - bound margin at a representative, inside the gate, {worst:.3e}")


@pytest.mark.parametrize("offset", [0.0, 100.0, 1000.0, 10000.0])
def test_rounding_terms_of_the_slack(offset):
    """The two float parts of eps_i on their own.  (1) A hypothesis moves a point to within 16u (|p|_1 + tau) of the exact R p + t
    (half of eps_i's 32u term: one pose each for the representative and the leaf), against a 64-bit-mantissa evaluation of the fp64
    pose.  (2) dist2_ref's fp32 squared distance is at least d^2 (1 - 6u), which the 8u sqrt(max_range) term covers near the gate."""
    rng = np.random.default_rng(int(offset) + 11)
    ratio = 0.0
    for trial in range(400):
        T = np.eye(4)
        T[:3, :3] = _rot(rng.uniform(-np.pi, np.pi), rng.normal(0, 0.05), rng.normal(0, 0.05))
        T[:3, 3] = rng.uniform(-1, 1, 3) * offset + rng.normal(0, 3, 3)
        g = reloc_wide_ref.grid(rng.uniform(0.0, 40.0), 0.5, np.pi, np.deg2rad(2.0))
        i, j, k = (int(v) for v in rng.integers(0, [2 * g.I + 1, 2 * g.I + 1, g.n_yaw]))
        L = reloc_wide_ref.leaf_pose(T, g, 0.5, np.deg2rad(2.0), i, j, k)
        p = (rng.normal(0, 1, (256, 3)) * rng.choice([1.0, 10.0, 100.0], (256, 1))).astype(np.float32)
        q = reloc_wide_ref.moved(p, L).astype(np.longdouble)
        exact = p.astype(np.longdouble) @ L[:3, :3].astype(np.longdouble).T + L[:3, 3].astype(np.longdouble)
        err = np.sqrt(((q - exact) ** 2).sum(axis=1)).astype(np.float64)
        tau = float(np.max(np.abs(L[:3, 3])))
        allow = 16.0 * reloc_wide_ref.U * (np.abs(p.astype(np.float64)).sum(axis=1) + tau)
        assert np.all(err <= allow), (trial, np.max(err / allow))
        ratio = max(ratio, float(np.max(err / allow)))
        # (2): pairs of fp32 points at these coordinates, within a few metres
        a = q.astype(np.float32)
        b = (a.astype(np.float64) + rng.normal(0, 1, a.shape) * rng.uniform(0, 3, (len(a), 1))).astype(np.float32)
        d2 = np.sum((a.astype(np.longdouble) - b.astype(np.longdouble)) ** 2, axis=1)
        assert np.all(reloc_wide_ref.dist2_f(a, b).astype(np.longdouble) >= d2 * (1 - 6 * reloc_wide_ref.U)), trial
    print(f"offset {offset:g} m: largest transform error {ratio:.3f} of its allowance")
