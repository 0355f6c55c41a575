"""fls_relocalize_multi without a device: argument checks, the shim's RelocalizeMulti, the hypothesis index and node layouts over G
guesses restated in numpy, and the worst-case slack of the lower bound over guesses of different roll and pitch against
fp32-emulated transforms and distances (tests/reloc_wide_ref.py)."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from funny_lidar_slam_b200 import _abi, _lib
from funny_lidar_slam_b200.registration import reloc_cfg
from tests import reloc_wide_ref, test_shim_compiles
from tests.test_relocalize_wide import _rot

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _call(cfg, guesses, n_guesses, h=None, n=0, stride=16, device=False):
    L = _lib.lib()
    T = (C.c_double * 16)(*np.eye(4).T.ravel())
    r = _abi.FlsRelocResult()
    ev = C.c_int64(0)
    g = guesses.ctypes.data_as(C.c_void_p) if guesses is not None else None
    c = C.byref(cfg) if cfg else None
    if device:
        return L.fls_relocalize_multi_device(h, None, n, c, g, n_guesses, T, C.byref(r), None, None, None, None, C.byref(ev))
    return L.fls_relocalize_multi(h, None, n, stride, c, g, n_guesses, T, C.byref(r), None, None, None, None, C.byref(ev))


@pytest.mark.parametrize("device", [False, True])
def test_argument_checks(device):
    G = np.stack([np.eye(4)] * 3)
    assert _call(reloc_cfg(), G, 3, device=device) == _abi.FLS_ERR_INVALID_ARG  # no handle
    assert _call(None, G, 3, device=device) == _abi.FLS_ERR_INVALID_ARG
    assert _call(reloc_cfg(), None, 3, device=device) == _abi.FLS_ERR_INVALID_ARG
    for count in (0, -1, 65):
        assert _call(reloc_cfg(), G, count, device=device) == _abi.FLS_ERR_INVALID_ARG
    for bad in (np.nan, np.inf, -np.inf):
        B = G.copy()
        B[2, 3, 3] = bad
        assert _call(reloc_cfg(), B, 3, device=device) == _abi.FLS_ERR_INVALID_ARG
    assert _call(reloc_cfg(), G, 3, n=5, device=device) == _abi.FLS_ERR_INVALID_ARG  # NULL scan with points
    if not device:
        assert _call(reloc_cfg(), G, 3, stride=12) == _abi.FLS_ERR_INVALID_ARG


USER = """
#include "b200_registration.h"
bool init(const fls_config& cfg, const PointcloudClusterPtr& cluster, const std::vector<Mat4d>& candidates, Mat4d& T) {
    B200Registration m(cfg);
    fls_reloc_cfg rc{3.0, 1.0, 0.349066, 0.174533, 1.0f, 2.0f, 1.0f, 16};
    float fitness = 0.f;
    return m.RelocalizeMulti(cluster, candidates, T, rc, &fitness) && fitness < 1.0f;
}
"""


def test_shim_relocalize_multi_compiles(tmp_path):
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


# ---- the layouts (fls_reloc.cu): leaf g * P + p, node g * N_l + b, b ordered as the leaves (yaw fastest, then x, then y) ----------
def _per_guess_nodes(nx, nk, l):
    return reloc_wide_ref.blocks(nx, l) ** 2 * reloc_wide_ref.blocks(nk, l)


def _node_idx(node, l, nx, nk):
    nbk, nbx = reloc_wide_ref.blocks(nk, l), reloc_wide_ref.blocks(nx, l)
    g, b = divmod(node, nbk * nbx * nbx)
    return g, b % nbk, (b // nbk) % nbx, b // (nbk * nbx)


def _leaves(node, l, nx, nk):
    """the leaves (global indices) of a node"""
    g, bk, bx, by = _node_idx(node, l, nx, nk)
    P = nx * nx * nk
    return {g * P + (y * nx + x) * nk + k for y in range(by << l, min((by + 1) << l, nx)) for x in range(bx << l, min((bx + 1) << l, nx))
            for k in range(bk << l, min((bk + 1) << l, nk))}


def _rep(node, l, nx, nk):
    g, bk, bx, by = _node_idx(node, l, nx, nk)
    (rk, _), (rx, _), (ry, _) = (reloc_wide_ref.block_rep(b, l, n) for b, n in ((bk, nk), (bx, nx), (by, nx)))
    return g * nx * nx * nk + (ry * nx + rx) * nk + rk


def _children(node, l, nx, nk):
    g, bk, bx, by = _node_idx(node, l, nx, nk)
    ck, cx = reloc_wide_ref.blocks(nk, l - 1), reloc_wide_ref.blocks(nx, l - 1)
    return [((g * cx + y) * cx + x) * ck + k for y in range(2 * by, min(2 * by + 2, cx)) for x in range(2 * bx, min(2 * bx + 2, cx))
            for k in range(2 * bk, min(2 * bk + 2, ck))]


@pytest.mark.parametrize("G,I,nk", [(1, 2, 7), (3, 1, 5), (5, 3, 12), (8, 0, 9), (2, 4, 1)])
def test_index_and_node_layouts(G, I, nk):
    nx = 2 * I + 1
    P = nx * nx * nk
    for l in range(0, 5):
        N = G * _per_guess_nodes(nx, nk, l)
        seen = []
        for node in range(N):
            leaves = _leaves(node, l, nx, nk)
            g = node // _per_guess_nodes(nx, nk, l)
            assert leaves and {i // P for i in leaves} == {g}  # a node never spans two guesses
            assert _rep(node, l, nx, nk) in leaves
            seen += sorted(leaves)
            if l:
                kids = _children(node, l, nx, nk)
                assert set().union(*(_leaves(c, l - 1, nx, nk) for c in kids)) == leaves
        assert sorted(seen) == list(range(G * P))  # the nodes of a level partition every guess's leaves
        if l == 0:
            assert seen == list(range(G * P))  # a level-0 node is its leaf
    # the start level: the lowest at which G * N_l <= 2^20
    g = reloc_wide_ref.grid(40.0, 0.5, np.pi, np.deg2rad(2.0))
    for G_, ls in ((1, 1), (2, 2), (8, 2), (64, 3)):
        l = 0
        while G_ * _per_guess_nodes(2 * g.I + 1, g.n_yaw, l) > reloc_wide_ref.START_NODES:
            l += 1
        assert l == ls, G_


def _slack_multi(p, Rs, hx, hy, hk, xy_step, yaw_step, tau, max_range):
    """delta_i with the worst case over the guesses: w_i = max_g |(R_g p_i)_xy| (rounded up to fp32, as the slack cloud stores it)"""
    p = np.asarray(p, np.float64)
    w = np.max([np.hypot(*(p @ np.asarray(R, np.float64)[:2, :3].T).T) for R in Rs], axis=0)
    w = np.nextafter(w.astype(np.float32), np.float32(np.inf)).astype(np.float64)
    eps = 32.0 * reloc_wide_ref.U * (tau + np.abs(p).sum(axis=1)) + 8.0 * reloc_wide_ref.U * np.sqrt(max_range)
    return np.hypot(hx, hy) * xy_step + hk * yaw_step * w + eps


@pytest.mark.parametrize("offset", [0.0, 100.0, 1000.0])
def test_worst_case_slack_bounds_every_guess(offset):
    """G guesses of different yaw, roll and pitch up to `offset` metres apart; a block of one of them, its representative and a leaf:
    with w and tau taken over all guesses, the leaf's gated fp32 term is never below the bound's term from the representative."""
    rng = np.random.default_rng(int(offset) + 29)
    for trial in range(200):
        G = int(rng.integers(2, 9))
        Ts = []
        for _ in range(G):
            T = np.eye(4)
            T[:3, :3] = _rot(rng.uniform(-np.pi, np.pi), rng.normal(0, 0.1), rng.normal(0, 0.1))
            T[:3, 3] = rng.uniform(-1, 1, 3) * offset + rng.normal(0, 3, 3)
            Ts.append(T)
        xy_step, yaw_step = rng.choice([0.25, 0.5, 1.0]), np.deg2rad(rng.choice([1.0, 2.0, 5.0, 10.0]))
        g = reloc_wide_ref.grid(rng.uniform(0.0, 30.0), xy_step, np.pi, yaw_step)
        nx, max_range = 2 * g.I + 1, float(rng.choice([0.5, 2.0, 4.0]))
        tau = max(max(max(abs(T[0, 3]), abs(T[1, 3])) + g.I * xy_step, abs(T[2, 3])) for T in Ts)
        gi = int(rng.integers(0, G))
        level = int(rng.integers(1, 6))
        b = [int(rng.integers(0, reloc_wide_ref.blocks(n, level))) for n in (nx, nx, g.n_yaw)]
        (rx, hx), (ry, hy), (rk, hk) = (reloc_wide_ref.block_rep(bb, level, n) for bb, n in zip(b, (nx, nx, g.n_yaw)))
        lx, ly, lk = (int(rng.integers(bb << level, min((bb + 1) << level, n))) for bb, n in zip(b, (nx, nx, g.n_yaw)))
        T_rep = reloc_wide_ref.leaf_pose(Ts[gi], g, xy_step, yaw_step, rx, ry, rk)
        T_leaf = reloc_wide_ref.leaf_pose(Ts[gi], g, xy_step, yaw_step, lx, ly, lk)
        p = (rng.normal(0, 1, (64, 3)) * rng.choice([1.0, 10.0, 60.0], (64, 1))).astype(np.float32)
        q_rep, q_leaf = reloc_wide_ref.moved(p, T_rep), reloc_wide_ref.moved(p, T_leaf)
        fit = (q_leaf.astype(np.float64) + rng.normal(0, 1, (64, 3)) * rng.uniform(0, np.sqrt(max_range), (64, 1))).astype(np.float32)
        bnd = np.linalg.norm(q_rep.astype(np.float64) - fit.astype(np.float64), axis=1)
        e = np.maximum(0.0, bnd - _slack_multi(p, [T[:3, :3] for T in Ts], hx, hy, hk, xy_step, yaw_step, tau, max_range))
        lb = np.minimum(e * e, float(np.float32(max_range)))
        leaf = reloc_wide_ref.leaf_terms(q_leaf, fit, max_range)
        assert np.all(leaf >= lb), (trial, np.min(leaf - lb))
        # for G = 1 the worst case is the single guess's own slack
        one = _slack_multi(p, [Ts[gi][:3, :3]], hx, hy, hk, xy_step, yaw_step, tau, max_range)
        own = reloc_wide_ref.slack(p, Ts[gi][:3, :3], hx, hy, hk, xy_step, yaw_step, tau, max_range)
        assert np.all(one >= own) and np.all(one - own <= hk * yaw_step * 1e-6 * (1 + np.abs(p).sum(axis=1)))
