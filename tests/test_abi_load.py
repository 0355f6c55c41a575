"""CPU-side checks of the drop-in boundary: the C-ABI library loads and exports every symbol of include/fls_b200.h."""
import ctypes as C
import os
import re

from funny_lidar_slam_b200 import _abi, _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_functions():
    src = open(os.path.join(ROOT, "include", "fls_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(fls_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    L = _lib.lib()
    names = _header_functions()
    assert len(names) >= 14
    for n in names:
        assert hasattr(L, n), f"libfls_b200.so does not export {n}"
    assert set(names) == set(_lib.EXPORTS)
    assert L.fls_abi_version() == _abi.FLS_ABI_VERSION


def test_config_default_matches_python_twin():
    L = _lib.lib()
    for m in range(5):
        c = _abi.FlsConfig()
        assert L.fls_config_default(C.byref(c), m) == 0
        p = _abi.default_config(m)
        for name, _ in _abi.FlsConfig._fields_:
            if name == "reserved":
                continue
            assert getattr(c, name) == getattr(p, name), (m, name)


def test_struct_sizes_match_header_layout():
    # layouts are fixed by the C header; these sizes are what gcc produces for it (checked by the build)
    assert C.sizeof(_abi.FlsMatchStats) == 72
    assert C.sizeof(_abi.FlsIterLog) == 8 * (36 + 6 + 6 + 1 + 1)
    assert C.sizeof(_abi.FlsMapInfo) == 48


def test_error_strings_and_invalid_args():
    L = _lib.lib()
    assert b"no CPU fallback" in L.fls_strerror(_abi.FLS_ERR_NO_DEVICE)
    assert L.fls_create(None, None) == _abi.FLS_ERR_INVALID_ARG
    bad = _abi.default_config(_abi.FLS_P2PLANE_IVOX, max_iterations=2147483647)  # IntNaN sentinel upstream
    h = C.c_void_p()
    assert L.fls_create(C.byref(bad), C.byref(h)) == _abi.FLS_ERR_INVALID_ARG


def test_all_five_plugins_validate_and_fail_loudly_without_a_device():
    """Every method of the reference's factory is accepted by the validator; on a box without a GPU creation stops at
    FLS_ERR_NO_DEVICE (there is no CPU fallback), never at FLS_ERR_UNSUPPORTED."""
    L = _lib.lib()
    if L.fls_device_count() > 0:
        return  # covered by the -m gpu tests on a GPU box
    for m in range(5):
        h = C.c_void_p()
        cfg = _abi.default_config(m)
        assert L.fls_create(C.byref(cfg), C.byref(h)) == _abi.FLS_ERR_NO_DEVICE, m
    # constructor-argument checks of the kd-tree plug-ins (the reference CHECK_NE()s them against its NaN sentinels)
    h = C.c_void_p()
    bad = _abi.default_config(_abi.FLS_LOAM_FULL, corner_local_map_size=0)
    assert L.fls_create(C.byref(bad), C.byref(h)) == _abi.FLS_ERR_INVALID_ARG
    bad = _abi.default_config(_abi.FLS_P2PLANE_KNN, map_cloud_filter_size=0.0)
    assert L.fls_create(C.byref(bad), C.byref(h)) == _abi.FLS_ERR_INVALID_ARG
    bad = _abi.default_config(_abi.FLS_NDT, max_iterations=300)  # iteration field of the hand-over tags is 8 bits
    assert L.fls_create(C.byref(bad), C.byref(h)) == _abi.FLS_ERR_UNSUPPORTED


def test_batch_and_projector_argument_checks():
    L = _lib.lib()
    assert L.fls_match_batch(None, 1, None, None, 16, None, None, None) == _abi.FLS_ERR_INVALID_ARG
    assert L.fls_match_batch_device(None, 1, None, None, None, None, None) == _abi.FLS_ERR_INVALID_ARG
    import numpy as np
    raw = np.zeros((4, 4), np.float32)
    ring = np.zeros(4, np.int32)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    n_out = C.c_size_t(0)
    # null outputs are rejected before any device work
    rc = L.fls_project(0, vp(raw), vp(ring), C.c_size_t(4), C.c_size_t(16), 2, 8, C.c_float(0.78), C.c_float(1.0), C.c_float(50.0), None, None,
                       None, None, None, C.byref(n_out))
    assert rc == _abi.FLS_ERR_INVALID_ARG
    rc = L.fls_project(0, vp(raw), vp(ring), C.c_size_t(4), C.c_size_t(12), 2, 8, C.c_float(0.78), C.c_float(1.0), C.c_float(50.0), vp(raw), vp(raw),
                       vp(ring), vp(ring), vp(ring), C.byref(n_out))
    assert rc == _abi.FLS_ERR_INVALID_ARG  # stride 12 is neither layout


def test_round2_entries_argument_checks():
    """The entries added in round 2 reject bad arguments before any device work (and a missing device is reported, not hidden)."""
    import numpy as np
    L = _lib.lib()
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    no, npl = C.c_size_t(0), C.c_size_t(0)
    raw = np.zeros((4, 5), np.float32)
    out = np.zeros((4, 4), np.float32)
    # fls_preprocess: jump_span >= 1, leaf > 0, outputs required
    assert L.fls_preprocess(0, vp(raw), C.c_size_t(4), None, C.c_float(1.0), C.c_float(50.0), 0, C.c_float(0.5), vp(out), C.byref(no), vp(out),
                            C.byref(npl)) == _abi.FLS_ERR_INVALID_ARG
    assert L.fls_preprocess(0, vp(raw), C.c_size_t(4), None, C.c_float(1.0), C.c_float(50.0), 4, C.c_float(0.0), vp(out), C.byref(no), vp(out),
                            C.byref(npl)) == _abi.FLS_ERR_INVALID_ARG
    assert L.fls_preprocess(0, vp(raw), C.c_size_t(4), None, C.c_float(1.0), C.c_float(50.0), 4, C.c_float(0.5), None, C.byref(no), vp(out),
                            C.byref(npl)) == _abi.FLS_ERR_INVALID_ARG
    if L.fls_device_count() < 1:
        assert L.fls_preprocess(0, vp(raw), C.c_size_t(4), None, C.c_float(1.0), C.c_float(50.0), 4, C.c_float(0.5), vp(out), C.byref(no), vp(out),
                                C.byref(npl)) == _abi.FLS_ERR_NO_DEVICE
    # handle entries with a null handle / null outputs
    assert L.fls_match_batch_begin(None, 1, None, None, 16, None) == _abi.FLS_ERR_INVALID_ARG
    assert L.fls_match_batch_begin_device(None, 1, None, None, None) == _abi.FLS_ERR_INVALID_ARG
    assert L.fls_match_batch_end(None, None, None, None) == _abi.FLS_ERR_INVALID_ARG
    assert L.fls_ivox_add_points(None, None, 0, 16) == _abi.FLS_ERR_INVALID_ARG
    assert L.fls_set_global_map(None, None, 0, 16) == _abi.FLS_ERR_INVALID_ARG
    assert L.fls_update_local_map(None, None, None, None) == _abi.FLS_ERR_INVALID_ARG
    assert L.fls_get_voxel_keys(None, None, 0, None) == _abi.FLS_ERR_INVALID_ARG
    assert L.fls_get_map_points(None, None, 0, None) == _abi.FLS_ERR_INVALID_ARG
    assert L.fls_get_ndt_voxels(None, None, 0, None) == _abi.FLS_ERR_INVALID_ARG
    assert L.fls_pcd_read(None, None, 0, None) == _abi.FLS_ERR_INVALID_ARG
    assert L.fls_pcd_write(None, None, 0) == _abi.FLS_ERR_INVALID_ARG


def test_header_is_plain_c_and_struct_layouts_match_ctypes(tmp_path):
    """include/fls_b200.h must compile as C99 (the boundary is a C ABI) and gcc's struct layouts must be the ones the ctypes
    mirror (and therefore the tests and the bench) assume."""
    import shutil
    import subprocess
    gcc = shutil.which("gcc")
    if gcc is None:
        return
    src = tmp_path / "abi.c"
    src.write_text(
        '#include <stdio.h>\n#include <stddef.h>\n#include "fls_b200.h"\n'
        "int main(void) {\n"
        '  printf("%zu %zu %zu %zu %zu ", sizeof(fls_config), sizeof(fls_match_stats), sizeof(fls_iter_log), sizeof(fls_map_info), sizeof(fls_feature_cfg));\n'
        '  printf("%zu %zu %zu %zu ", offsetof(fls_config, point_to_planar_thres), offsetof(fls_config, ndt_voxel_size), offsetof(fls_config, point_search_thres), offsetof(fls_match_stats, algo_bytes));\n'
        '  printf("%zu %zu %zu\\n", sizeof(fls_ndt_voxel), offsetof(fls_ndt_voxel, carry_count), offsetof(fls_ndt_voxel, mu));\n'
        "  return 0;\n}\n")
    exe = tmp_path / "abi"
    subprocess.check_call([gcc, "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    want = [C.sizeof(_abi.FlsConfig), C.sizeof(_abi.FlsMatchStats), C.sizeof(_abi.FlsIterLog), C.sizeof(_abi.FlsMapInfo), C.sizeof(_abi.FlsFeatureCfg),
            _abi.FlsConfig.point_to_planar_thres.offset, _abi.FlsConfig.ndt_voxel_size.offset, _abi.FlsConfig.point_search_thres.offset,
            _abi.FlsMatchStats.algo_bytes.offset, C.sizeof(_abi.FlsNdtVoxel), _abi.FlsNdtVoxel.carry_count.offset, _abi.FlsNdtVoxel.mu.offset]
    assert got == want, (got, want)
