"""CPU checks of Scan Context place recognition (fls_keyframes_scan_context / _detect_loop / _place_query): the argument checks that
return before any device work, the two structs' layouts against gcc, the properties of the numpy reference (tests/scan_context_ref.py)
and the extended keyframe adapter compiled against stand-ins of the reference headers."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from funny_lidar_slam_b200 import _abi, _lib
from funny_lidar_slam_b200._abi import FlsMatchStats, FlsPlaceMatch, FlsScCfg
from funny_lidar_slam_b200.keyframes import place_pose, sc_cfg
from tests import scan_context_ref as ref
from tests.test_keyframe_map import MOCKS, SHIM, USER

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID = _abi.FLS_ERR_INVALID_ARG

BAD_CFGS = [dict(n_rings=0), dict(n_rings=65), dict(n_sectors=0), dict(n_sectors=361), dict(n_rings=64, n_sectors=65), dict(max_radius=0.0),
            dict(max_radius=-1.0), dict(max_radius=float("nan")), dict(max_radius=float("inf")), dict(z_offset=float("nan")),
            dict(z_offset=float("-inf"))]


# ---- argument checks ----------------------------------------------------------------------------------------------------------
def test_entries_check_arguments_before_touching_the_store():
    """Every refusal here returns before the store is dereferenced, so a dangling store pointer is safe to pass: only a bad argument
    is given with it."""
    L = _lib.lib()
    fake = C.c_void_p(0x10)  # never dereferenced: each call below has one bad argument
    good = sc_cfg()
    out = (FlsPlaceMatch * 4)()
    n = C.c_size_t(7)
    st = FlsMatchStats()
    pts = np.zeros((4, 4), np.float32)
    p = pts.ctypes.data_as(C.c_void_p)
    desc = np.zeros(20 * 60, np.float32)
    ids = np.zeros(1, np.int64)
    dp, ip = desc.ctypes.data_as(C.c_void_p), ids.ctypes.data_as(C.c_void_p)

    def refusals(store, cfg, k=4, o=out, nf=C.byref(n)):
        return [L.fls_keyframes_detect_loop(store, cfg, 3, 1, k, o, nf, C.byref(st)),
                L.fls_keyframes_place_query(store, cfg, p, 4, 16, k, o, nf, dp, C.byref(st)),
                L.fls_keyframes_place_query_device(store, cfg, p, 4, k, o, nf, dp, C.byref(st))]

    assert refusals(None, C.byref(good)) == [INVALID] * 3
    assert L.fls_keyframes_scan_context(None, C.byref(good), ip, 1, dp) == INVALID
    assert refusals(fake, None) == [INVALID] * 3
    assert L.fls_keyframes_scan_context(fake, None, ip, 1, dp) == INVALID
    for bad in BAD_CFGS:
        n.value = 7
        assert refusals(fake, C.byref(sc_cfg(**bad))) == [INVALID] * 3, bad
        assert n.value == 0  # cleared on refusal
        assert L.fls_keyframes_scan_context(fake, C.byref(sc_cfg(**bad)), ip, 1, dp) == INVALID, bad
    assert refusals(fake, C.byref(good), k=0) == [INVALID] * 3
    assert refusals(fake, C.byref(good), o=None) == [INVALID] * 3
    assert refusals(fake, C.byref(good), nf=None) == [INVALID] * 3
    # detect_loop: negative query id or span
    assert L.fls_keyframes_detect_loop(fake, C.byref(good), -1, 1, 4, out, C.byref(n), None) == INVALID
    assert L.fls_keyframes_detect_loop(fake, C.byref(good), 3, -1, 4, out, C.byref(n), None) == INVALID
    # place_query: null points with n > 0, a stride that is neither layout
    assert L.fls_keyframes_place_query(fake, C.byref(good), None, 4, 16, 4, out, C.byref(n), None, None) == INVALID
    assert L.fls_keyframes_place_query(fake, C.byref(good), p, 4, 12, 4, out, C.byref(n), None, None) == INVALID
    assert L.fls_keyframes_place_query_device(fake, C.byref(good), None, 4, 4, out, C.byref(n), None, None) == INVALID
    # scan_context: null ids or output with n_ids > 0
    assert L.fls_keyframes_scan_context(fake, C.byref(good), None, 1, dp) == INVALID
    assert L.fls_keyframes_scan_context(fake, C.byref(good), ip, 1, None) == INVALID


@pytest.mark.gpu
def test_cfg_limits_are_inclusive():
    """The shapes at the limits of fls_sc_cfg are accepted by a real store and the ones just past them refused.  Without a device
    every entry stops at its store argument first, so this needs one."""
    from funny_lidar_slam_b200.keyframes import KeyFrameStore
    cloud = np.array([[3.0, 4.0, 1.0, 1.0], [-20.0, 5.0, -2.5, 1.0], [0.5, -60.0, 4.0, 1.0]], np.float32)
    s = KeyFrameStore(16)
    s.add(cloud)
    s.add(cloud)
    for ok in (dict(n_rings=64, n_sectors=64), dict(n_rings=1, n_sectors=360), dict(n_rings=11, n_sectors=360), dict(n_rings=64, n_sectors=1),
               dict(max_radius=1e-30, z_offset=-5.0)):
        c = sc_cfg(**ok)
        got = s.detect_loop(1, 0, 1, c)
        assert len(got) == 1 and got[0].id == 0
        want = ref.descriptor(cloud, c.n_rings, c.n_sectors, c.max_radius, c.z_offset)
        assert np.array_equal(s.scan_context([1], c)[0].view(np.uint32), want.view(np.uint32)), ok
    for bad in BAD_CFGS:
        with pytest.raises(_lib.FlsError) as e:
            s.detect_loop(1, 0, 1, sc_cfg(**bad))
        assert e.value.status == INVALID, bad


# ---- struct layouts -----------------------------------------------------------------------------------------------------------
def test_struct_layouts_match_gcc(tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "abi.c"
    src.write_text(
        '#include <stdio.h>\n#include <stddef.h>\n#include "fls_b200.h"\n'
        "int main(void) {\n"
        '  printf("%zu %zu %zu %zu ", sizeof(fls_sc_cfg), offsetof(fls_sc_cfg, n_sectors), offsetof(fls_sc_cfg, max_radius), offsetof(fls_sc_cfg, z_offset));\n'
        '  printf("%zu %zu %zu %zu %zu\\n", sizeof(fls_place_match), offsetof(fls_place_match, distance), offsetof(fls_place_match, yaw),'
        " offsetof(fls_place_match, shift), offsetof(fls_place_match, reserved));\n"
        "  return 0;\n}\n")
    exe = tmp_path / "abi"
    subprocess.check_call([gcc, "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    want = [C.sizeof(FlsScCfg), FlsScCfg.n_sectors.offset, FlsScCfg.max_radius.offset, FlsScCfg.z_offset.offset, C.sizeof(FlsPlaceMatch),
            FlsPlaceMatch.distance.offset, FlsPlaceMatch.yaw.offset, FlsPlaceMatch.shift.offset, FlsPlaceMatch.reserved.offset]
    assert got == want, (got, want)
    assert got[0] == 16 and got[4] == 32


# ---- properties of the reference ----------------------------------------------------------------------------------------------
def _sector_centre_cloud(rng, n_rings=20, n_sectors=60, R=80.0, per_cell=0.4):
    """points at sector centres (one angle per sector), random rings and heights"""
    pts = []
    for s in range(n_sectors):
        for r in range(n_rings):
            if rng.random() < per_cell:
                rad = (r + rng.uniform(0.2, 0.8)) * R / n_rings
                z = rng.uniform(-1.5, 6.0)
                pts.append((s, rad, z))
    return pts


def _cloud_from(pts, n_sectors, turn):
    out = []
    for s, rad, z in pts:
        a = (s + 0.5 - turn) * 2 * np.pi / n_sectors
        out.append((rad * np.cos(a), rad * np.sin(a), z, 1.0))
    return np.array(out, np.float32)


@pytest.mark.parametrize("m", [0, 1, 7, 30, 59])
def test_turned_cloud_rolls_the_descriptor(m):
    """A cloud turned by -m sectors about z (the sensor turned by +m sectors) is the descriptor rolled by -m columns, and the
    distance to the original is 0 at shift m."""
    rng = np.random.default_rng(10 + m)
    pts = _sector_centre_cloud(rng)
    a = ref.descriptor(_cloud_from(pts, 60, 0))
    b = ref.descriptor(_cloud_from(pts, 60, m))
    assert np.array_equal(b, np.roll(a, -m, axis=1))
    D, s, d = ref.distances(b, a[None])
    assert s[0] == m and abs(D[0]) < 1e-12 and abs(d[0, m]) < 1e-12
    yaw = ref.yaw(s[0], 60)
    assert abs(np.angle(np.exp(1j * (yaw - m * 2 * np.pi / 60)))) < 1e-12


def test_identical_disjoint_and_empty():
    rng = np.random.default_rng(3)
    a = ref.descriptor(_cloud_from(_sector_centre_cloud(rng), 60, 0))
    D, s, _ = ref.distances(a, a[None])
    assert abs(D[0]) < 1e-12 and s[0] == 0
    left, right = np.zeros((20, 60), np.float32), np.zeros((20, 60), np.float32)
    left[:, :30] = rng.uniform(0.5, 3.0, (20, 30))
    right[:, 30:] = rng.uniform(0.5, 3.0, (20, 30))
    right[:, 0] = 0.0
    # at shift 0 no column is non-zero in both: d_0 = 1 exactly
    assert ref.shift_distances(left, right[None])[0, 0] == 1.0
    one = np.zeros((20, 60), np.float32)
    one[:, 5] = 1.0
    two = np.zeros((20, 60), np.float32)
    two[:, 6] = 1.0
    d = ref.shift_distances(one, two[None])[0]
    assert abs(d[1]) < 1e-12 and np.all(d[np.arange(60) != 1] == 1.0)
    empty = np.zeros((20, 60), np.float32)
    assert np.all(ref.shift_distances(empty, a[None]) == 1.0) and np.all(ref.shift_distances(a, empty[None]) == 1.0)
    assert np.all(ref.descriptor(np.zeros((0, 4), np.float32)) == 0)


def test_descriptor_edges_of_the_definition():
    """non-finite points are skipped, r == R is out, a negative cell stays negative, -0.0 loses to +0.0"""
    pts = np.array([[np.nan, 1, 1, 0], [1, np.inf, 1, 0], [1, 1, -np.inf, 0], [80.0, 0, 5, 0], [0, -80.0, 5, 0], [10, 0, -7.5, 0],
                    [10, 0.0001, -9.0, 0]], np.float32)
    d = ref.descriptor(pts, z_offset=2.0)
    assert np.count_nonzero(d) == 1
    assert d[2, 0] == np.float32(-5.5)
    z = ref.descriptor(np.array([[0, 20, -2.0, 0]], np.float32))
    assert z[5, 15] == 0 and not np.signbit(z[5, 15])
    nz = ref.descriptor(np.array([[0, 20, -0.0, 0]], np.float32), z_offset=-0.0)
    assert np.signbit(nz[5, 15])
    both = ref.descriptor(np.array([[0, 20, -0.0, 0], [0, 20, 0.0, 0]], np.float32), z_offset=-0.0)
    assert not np.signbit(both[5, 15])


def test_place_pose_is_T_times_Rz():
    T = np.eye(4)
    T[:3, 3] = [1.0, 2.0, 3.0]
    P = place_pose(T, np.pi / 2)
    assert np.allclose(P[:3, :3] @ [1, 0, 0], [0, 1, 0]) and np.allclose(P[:3, 3], [1, 2, 3])


# ---- the adapter --------------------------------------------------------------------------------------------------------------
PLACE_USER = USER + """
double place(const PCLPointCloudXYZI& scan) {
    B200KeyFrameMap store(0, 1000000);
    const B200KeyFrameMap::PlaceMatch loop = store.DetectLoopByFeature(42, 10);
    const B200KeyFrameMap::PlaceMatch where = store.PlaceQuery(scan);
    const KeyFrame::ID id = loop.candidate_id;
    return loop.distance + loop.yaw + where.distance + where.yaw + id + where.candidate_id;
}
"""


def test_extended_adapter_compiles_against_the_reference_types(tmp_path):
    gxx = shutil.which("g++") or "/usr/bin/g++"
    if not os.path.exists(gxx):
        pytest.skip("no C++ compiler")
    for rel, body in MOCKS.items():
        p = tmp_path / "mock" / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(body)
    (tmp_path / "user.cpp").write_text(PLACE_USER)
    cmd = [gxx, "-std=c++17", "-Wall", "-Wextra", "-Werror", "-Wno-unused-parameter", "-fsyntax-only", "-I", str(tmp_path / "mock"),
           "-I", os.path.join(ROOT, "include"), "-I", os.path.dirname(SHIM), str(tmp_path / "user.cpp")]
    env = dict(os.environ)
    env.pop("CXX", None)
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr
