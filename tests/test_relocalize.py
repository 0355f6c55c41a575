"""fls_relocalize without a device: argument checks, the layout of fls_reloc_cfg / fls_reloc_result against gcc, the shim's Relocalize
in the stand-in setting of test_shim_compiles.py, and the reference grid's edge cases."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from funny_lidar_slam_b200 import _abi, _lib
from funny_lidar_slam_b200.registration import reloc_cfg
from tests import reloc_ref, test_shim_compiles

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _call(cfg, h=None, n=0, stride=16, device=False):
    L = _lib.lib()
    T = (C.c_double * 16)(*np.eye(4).T.ravel())
    r = _abi.FlsRelocResult()
    if device:
        return L.fls_relocalize_device(h, None, n, C.byref(cfg) if cfg else None, T, C.byref(r), None, None, None, None, None, 0)
    return L.fls_relocalize(h, None, n, stride, C.byref(cfg) if cfg else None, T, C.byref(r), None, None, None, None, None, 0)


@pytest.mark.parametrize("device", [False, True])
def test_argument_checks(device):
    assert _call(reloc_cfg(), device=device) == _abi.FLS_ERR_INVALID_ARG  # no handle
    assert _call(None, device=device) == _abi.FLS_ERR_INVALID_ARG
    assert _call(reloc_cfg(), n=5, device=device) == _abi.FLS_ERR_INVALID_ARG  # NULL scan with points
    if not device:
        assert _call(reloc_cfg(), stride=12) == _abi.FLS_ERR_INVALID_ARG


def test_handles_need_a_device():
    L = _lib.lib()
    if L.fls_device_count() > 0:
        pytest.skip("a device is visible")
    for m in (_abi.FLS_P2PLANE_IVOX, _abi.FLS_NDT):
        cfg = _abi.default_config(m)
        h = C.c_void_p()
        assert L.fls_create(C.byref(cfg), C.byref(h)) == _abi.FLS_ERR_NO_DEVICE


def test_struct_layouts_match_gcc(tmp_path):
    gcc = shutil.which("gcc") or "/usr/bin/gcc"
    if not os.path.exists(gcc):
        pytest.skip("no gcc")
    src = tmp_path / "l.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "fls_b200.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(fls_reloc_cfg), offsetof(fls_reloc_cfg, coarse_leaf),'
                   ' offsetof(fls_reloc_cfg, accept_fitness), offsetof(fls_reloc_cfg, n_refine), sizeof(fls_reloc_result),'
                   ' offsetof(fls_reloc_result, n_refined), offsetof(fls_reloc_result, fitness), offsetof(fls_reloc_result, host_waits),'
                   ' offsetof(fls_reloc_result, gpu_launches));\n  return 0;\n}\n')
    exe = tmp_path / "l"
    subprocess.check_call([gcc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    Cf, Rr = _abi.FlsRelocCfg, _abi.FlsRelocResult
    assert got == [C.sizeof(Cf), Cf.coarse_leaf.offset, Cf.accept_fitness.offset, Cf.n_refine.offset, C.sizeof(Rr), Rr.n_refined.offset,
                   Rr.fitness.offset, Rr.host_waits.offset, Rr.gpu_launches.offset]


USER = """
#include "b200_registration.h"
bool init(const fls_config& cfg, const PointcloudClusterPtr& cluster, Mat4d& T) {
    B200Registration m(cfg);
    fls_reloc_cfg rc{10.0, 1.0, 3.14159265358979, 0.1745329, 1.0f, 2.0f, 1.0f, 64};
    float fitness = 0.f;
    return m.Relocalize(cluster, T, rc, &fitness) && fitness < 1.0f;
}
"""


def test_shim_relocalize_compiles(tmp_path):
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


def test_grid_zero_radius_and_zero_yaw_is_the_guess():
    g = reloc_ref.grid(0.0, float("nan"), 0.0, float("nan"))
    assert (g.I, g.n_yaw, g.P) == (0, 1, 1)
    T = np.eye(4)
    T[:3, 3] = [1.0, -2.0, 0.5]
    H = reloc_ref.hypotheses(T, 0.0, float("nan"), 0.0, float("nan"))
    assert np.array_equal(H[0], T)


def test_grid_radius_not_a_step_multiple():
    assert reloc_ref.grid(2.5, 1.0, 0.0, 1.0).I == 2
    assert reloc_ref.grid(0.3, 0.1, 0.0, 1.0).I == 3  # 0.3 / 0.1 = 2.9999999999999996 in fp64
    assert reloc_ref.grid(0.99, 1.0, 0.0, 1.0).P == 1


@pytest.mark.parametrize("yaw_range", [np.pi, np.pi + 0.5, 10.0])
def test_full_circle_has_no_duplicate(yaw_range):
    step = np.deg2rad(10.0)
    g = reloc_ref.grid(10.0, 1.0, yaw_range, step)
    assert g.n_yaw == 36 and g.P == 21 * 21 * 36 == 15876
    psi = reloc_ref.yaw_offsets(g, step)
    wrapped = np.mod(np.round(np.rad2deg(psi), 6), 360.0)
    assert len(np.unique(wrapped)) == len(psi)
    # a step that does not divide the circle keeps both ends, which are different angles
    g7 = reloc_ref.grid(0.0, 1.0, np.pi, np.deg2rad(7.0))
    assert g7.n_yaw == 51


def test_partial_yaw_range_is_symmetric():
    g = reloc_ref.grid(0.0, 1.0, np.deg2rad(30.0), np.deg2rad(10.0))
    assert (g.k0, g.K, g.n_yaw) == (-3, 3, 7)


def test_hypothesis_index_order_is_yaw_then_x_then_y():
    T = np.eye(4)
    H = reloc_ref.hypotheses(T, 1.0, 1.0, np.deg2rad(10.0), np.deg2rad(10.0))
    assert len(H) == 27
    assert np.allclose(H[0, :3, 3], [-1, -1, 0]) and np.allclose(H[3, :3, 3], [0, -1, 0]) and np.allclose(H[9, :3, 3], [-1, 0, 0])
    yaw = np.arctan2(H[:3, 1, 0], H[:3, 0, 0])
    assert np.allclose(np.rad2deg(yaw), [-10, 0, 10])


def test_hypothesis_cap():
    assert reloc_ref.grid(255.0, 1.0, 0.0, 1.0).P == 511 * 511 <= 1 << 20
    with pytest.raises(ValueError):
        reloc_ref.grid(512.0, 1.0, 0.0, 1.0)
    with pytest.raises(ValueError):
        reloc_ref.grid(10.0, 1.0, np.pi, np.deg2rad(0.1))


def test_selection_breaks_ties_by_index():
    s = np.array([3.0, 1.0, 2.0, 1.0, 0.5])
    idx, gaps = reloc_ref.select(s, 3)
    assert list(idx) == [4, 1, 3]
    assert gaps[1] == 0.0 and gaps[2] == 1.0
