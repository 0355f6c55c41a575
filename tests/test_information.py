"""FLS_FLAG_INFORMATION on the CPU: the record's layout against gcc, the argument checks of fls_get_information(_scan), and the map A
from each plug-in's Gauss-Newton update to the fusion parameterization ([dθ; dp], R <- R·Exp(dθ), p <- p + dp) that the fold
kernel applies (fls_info.cu), checked against a numpy composition of the two updates."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from funny_lidar_slam_b200 import _abi
from tests import info_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_record_layout_matches_gcc(tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    src = tmp_path / "info.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "fls_b200.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %zu %zu %u\\n", sizeof(fls_information), offsetof(fls_information, g), offsetof(fls_information, sum_residual),'
                   ' offsetof(fls_information, n_valid), offsetof(fls_information, valid), (unsigned)FLS_FLAG_INFORMATION);\n  return 0;\n}\n')
    exe = tmp_path / "info"
    subprocess.check_call([gcc, "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    F = _abi.FlsInformation
    assert got == [C.sizeof(F), F.g.offset, F.sum_residual.offset, F.n_valid.offset, F.valid.offset, _abi.FLS_FLAG_INFORMATION]
    assert C.sizeof(F) == 8 * (36 + 6 + 1 + 1) + 8


def test_argument_checks():
    from funny_lidar_slam_b200._lib import lib
    L = lib()
    rec = _abi.FlsInformation()
    assert L.fls_get_information(None, C.byref(rec)) == _abi.FLS_ERR_INVALID_ARG
    assert L.fls_get_information_scan(None, 0, C.byref(rec)) == _abi.FLS_ERR_INVALID_ARG
    assert L.fls_get_information_scan(None, -1, None) == _abi.FLS_ERR_INVALID_ARG


def _A(method, R):
    A = np.eye(6)
    if method == "icp":
        A = np.zeros((6, 6))
        A[0:3, 3:6] = np.eye(3)
        A[3:6, 0:3] = np.eye(3)
    elif method == "loam":
        A[0:3, 0:3] = R
    return A


def _plugin_update(method, R, t, dx):
    """gn_step_pre (fls_gn.cuh): LOAM dx = [dθ, dt], R <- Exp(dθ) R; NDT dx = [dθ, dt], R <- R Exp(dθ); ICP dx = [dt, dθ], R <- R Exp(dθ);
    every one t <- t + dt."""
    if method == "icp":
        dt, dth = dx[:3], dx[3:]
    else:
        dth, dt = dx[:3], dx[3:]
    E = Rotation.from_rotvec(dth).as_matrix()
    return (E @ R if method == "loam" else R @ E), t + dt


@pytest.mark.parametrize("method", ["loam", "ndt", "icp"])
def test_A_maps_the_plugin_update_to_the_fusion_update(method):
    rng = np.random.default_rng(3)
    for _ in range(20):
        R = Rotation.from_rotvec(rng.normal(size=3)).as_matrix()
        t = rng.normal(size=3) * 10
        delta = rng.normal(size=6) * 1e-6
        R_f, t_f = R @ Rotation.from_rotvec(delta[:3]).as_matrix(), t + delta[3:]  # EdgeRotation's R * Exp(dθ), p + dp
        R_p, t_p = _plugin_update(method, R, t, _A(method, R) @ delta)
        assert np.abs(R_p - R_f).max() < 1e-11 and np.abs(t_p - t_f).max() < 1e-12


def test_adapter_reports_the_record(tmp_path):
    """GetPoseInformation of the adapter compiles and copies a record: built against stand-ins of the reference headers and of the
    two library calls it makes."""
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("no g++")
    shim = os.path.join(ROOT, "funny_lidar_slam_b200", "shim", "b200_registration.h")
    src = tmp_path / "info.cpp"
    src.write_text(
        '#include <cstdint>\n#include <cstring>\n#include "fls_b200.h"\n'
        "struct Mat6d { double v[36]; double& operator()(int r, int c) { return v[r * 6 + c]; } };\n"
        "struct Vec6d { double v[6]; double& operator()(int r) { return v[r]; } };\n"
        "static fls_information g_rec;\n"
        'extern "C" int fls_get_information(const fls_handle*, fls_information* out) { *out = g_rec; return FLS_OK; }\n'
        "struct Probe { fls_handle* handle_ = nullptr;\n"
        + open(shim).read().split("    // The information matrix of the last Match")[1].split("\n    }\n")[0].join(["    // ", "\n    }\n"])
        + "};\n"
        "int main() {\n"
        "  for (int i = 0; i < 36; ++i) g_rec.H[i] = i;\n"
        "  for (int i = 0; i < 6; ++i) g_rec.g[i] = -i;\n"
        "  g_rec.n_valid = 7;\n  g_rec.sum_residual = 2.5;\n"
        "  Probe p; Mat6d H; Vec6d g; int64_t n = 0; double s = 0;\n"
        "  if (p.GetPoseInformation(H, &g, &n, &s)) return 1;\n"
        "  g_rec.valid = 1;\n"
        "  if (!p.GetPoseInformation(H, &g, &n, &s) || H(2, 3) != 15 || g(4) != -4 || n != 7 || s != 2.5) return 2;\n"
        "  return 0;\n}\n")
    exe = tmp_path / "info"
    subprocess.check_call([gxx, "-std=c++17", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    assert subprocess.call([str(exe)]) == 0


def _perturbed(R, t, p, delta):
    """q of body point p under upstream's perturbation: R·Exp(dθ) p + t + dp"""
    return R @ info_ref.exp_so3(delta[:3]) @ p + t + delta[3:]


@pytest.mark.parametrize("kind", ["plane", "corner", "point", "ndt"])
def test_reference_jacobians_against_finite_differences(kind):
    """The reference's analytic J (tests/info_ref.py) against central differences of each residual under R·Exp(dθ), p + dp with the
    correspondence held fixed: the reference uses upstream's fusion parameterization."""
    rng = np.random.default_rng({"plane": 1, "corner": 2, "point": 3, "ndt": 4}[kind])
    for _ in range(10):
        R = info_ref.exp_so3(rng.normal(size=3))
        t = rng.normal(size=3) * 5
        p = rng.normal(size=3) * 8
        q0 = R @ p + t
        n = rng.normal(size=3)
        n /= np.linalg.norm(n)
        a0 = q0 + rng.normal(size=3) * 0.3
        if kind == "plane":
            f = lambda q: np.array([abs(n @ (q - a0))])
            grad = np.sign(n @ (q0 - a0)) * n
            J = (grad @ info_ref.j_point(R, p))[None, :]
        elif kind == "corner":
            f = lambda q: np.array([np.linalg.norm(np.cross(q - a0, n))])
            w = np.cross(q0 - a0, n)
            J = (np.cross(n, w / np.linalg.norm(w)) @ info_ref.j_point(R, p))[None, :]
        else:  # ICP point-to-point, NDT e = q - mu (its weight does not enter J)
            f = lambda q: q - a0
            J = info_ref.j_point(R, p)
        h = 1e-6
        Jfd = np.stack([(f(_perturbed(R, t, p, h * e)) - f(_perturbed(R, t, p, -h * e))) / (2 * h) for e in np.eye(6)], 1)
        assert np.abs(Jfd - J).max() < 1e-6 * max(1.0, np.abs(J).max()), (kind, Jfd, J)
