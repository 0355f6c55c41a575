"""GPU parity of the keyframe store (fls_keyframes_assemble) with the oracle composition — orc.voxel_grid per keyframe, orc.transform_f
by its pose, concatenation, an optional final orc.voxel_grid — compared bit for bit (uint32 views of x, y, z and intensity, same
order, same count), for the three upstream call sites and the edge cases of the segmented pass."""
import ctypes as C
import threading

import numpy as np
import pytest

from funny_lidar_slam_b200 import _abi, synth
from tests import keyframe_ref as ref
from tests.conftest import to_pcl

pytestmark = pytest.mark.gpu


def _same(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _store(clouds, capacity=None):
    from funny_lidar_slam_b200.keyframes import KeyFrameStore
    s = KeyFrameStore(capacity or max(sum(len(c) for c in clouds), 1))
    for c in clouds:
        s.add(c)
    return s


def _pose(rng, scale=30.0):
    a, b = rng.uniform(-np.pi, np.pi), rng.uniform(-0.2, 0.2)
    Rz = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    Rx = np.array([[1, 0, 0], [0, np.cos(b), -np.sin(b)], [0, np.sin(b), np.cos(b)]])
    T = np.eye(4)
    T[:3, :3] = Rz @ Rx
    T[:3, 3] = rng.uniform(-scale, scale, 3)
    return T


def _cloud(rng, n, half=15.0):
    return np.concatenate([rng.uniform(-half, half, (n, 3)), rng.uniform(0, 255, (n, 1))], 1).astype(np.float32)


@pytest.fixture(scope="module")
def keyframes(world):
    """Twelve 64-line keyframes along the trajectory (body frame) with their poses."""
    traj = synth.trajectory(12)
    clouds = [synth.make_scan(world, traj[i], "hdl64", seed=100 + i)["points"] for i in range(12)]
    return clouds, np.array(traj)


# ---- the three call sites ------------------------------------------------------------------------------------------------------
def test_save_map_bit_exact(keyframes):
    from funny_lidar_slam_b200.keyframes import save_map_cloud
    clouds, poses = keyframes
    s = _store(clouds)
    got = save_map_cloud(s, poses)
    want = ref.save_map_literal(clouds, poses)
    assert len(want) > 10000 and _same(got, want)
    assert _same(got, ref.assemble_ref(clouds, range(len(clouds)), poses, 0.3, 0.3))


@pytest.mark.parametrize("use_local_pose", [False, True])
def test_loopclosure_submap_bit_exact(keyframes, use_local_pose):
    from funny_lidar_slam_b200.keyframes import loopclosure_submap
    clouds, poses = keyframes
    s = _store(clouds)
    for kf, left, right in ((5, 3, 3), (0, 4, 2), (11, 2, 6), (6, 20, 20)):
        got = loopclosure_submap(s, poses, kf, left, right, use_local_pose)
        want = ref.get_submap_literal(clouds, poses, kf, left, right, use_local_pose)
        assert len(want) > 1000 and _same(got, want), (kf, left, right)


def test_global_map_rounds_and_reset(keyframes):
    from funny_lidar_slam_b200.keyframes import GlobalMapState, KeyFrameStore, global_map_round
    clouds, poses = keyframes
    s = KeyFrameStore(sum(len(c) for c in clouds))
    state = GlobalMapState()
    lit = ref.GlobalMapLiteral(0.5)
    published = 0
    for k, upd in ((1, False), (3, False), (4, False), (7, False), (10, False), (12, True)):
        while len(s) < k:
            s.add(clouds[len(s)])
        if upd:  # a loop closure re-optimised every pose
            poses = poses.copy()
            poses[:, :3, 3] += np.array([0.11, -0.07, 0.02])
        got = global_map_round(s, state, poses[:k], 0.5, upd)
        want = lit.round(clouds[:k], poses[:k], upd)
        assert (got is None) == (want is None), k
        if want is not None:
            published += 1
            assert _same(got, want), k
    assert published >= 4


# ---- edge cases of the segmented pass ------------------------------------------------------------------------------------------
def test_edge_keyframes():
    rng = np.random.default_rng(3)
    wide = _cloud(rng, 3000, half=400.0)  # overflows at 0.05 m (dx*dy*dz > INT_MAX): points pass unchanged, input order
    wide[5, 0] = -0.0
    wide[6, :3] = -0.0
    one = np.array([[1.5, -2.25, 3.0, 9.0]], np.float32)
    grid = np.stack(np.meshgrid(np.arange(-3, 3, 0.25), np.arange(-3, 3, 0.25), [0.0, 0.5, -0.5], indexing="ij"), -1).reshape(-1, 3)
    border = np.concatenate([grid, np.arange(len(grid))[:, None]], 1).astype(np.float32)  # exactly on cell borders, negative too
    clouds = [wide, np.zeros((0, 4), np.float32), one, np.repeat(one, 1000, axis=0), border, _cloud(rng, 5000) - 40.0]
    s = _store(clouds)
    poses = np.array([_pose(rng) for _ in clouds])
    for leaf in (0.05, 0.25, 0.5):
        ids = list(range(len(clouds)))
        got = s.assemble(ids, poses, leaf)
        assert _same(got, ref.assemble_ref(clouds, ids, poses, leaf)), leaf
    got = s.assemble([0], np.eye(4)[None], 0.05)
    assert _same(got, ref.orc_transform(wide, np.eye(4))) and _same(got, ref.np_transform_f(wide, np.eye(4)))
    # an empty selection and an empty keyframe contribute nothing
    assert s.assemble([], np.zeros((0, 4, 4)), 0.3).shape == (0, 4)
    assert s.assemble([1], np.eye(4)[None], 0.3).shape == (0, 4)
    assert s.assemble([1, 1], np.stack([np.eye(4)] * 2), 0.3, 0.3).shape == (0, 4)


def test_overflowing_segment_keeps_negative_zero_bits():
    """PCL copies an overflowing cloud: a -0.0 survives the filter (0.f + -0.f would give +0.f) and the transform adds +0.0 to it."""
    rng = np.random.default_rng(4)
    wide = _cloud(rng, 2000, half=400.0)
    wide[7, :3] = -0.0
    s = _store([wide])
    T = np.eye(4)
    T[:3, 3] = -0.0  # t = -0.0 keeps (-0.0 * 1 + ...) + -0.0 = -0.0
    got = s.assemble([0], T[None], 0.05)
    want = ref.assemble_ref([wide], [0], T[None], 0.05)
    assert _same(got, want)
    assert np.signbit(got[7, :3]).all()


def test_whole_map_overflows_at_final_leaf():
    rng = np.random.default_rng(5)
    clouds = [_cloud(rng, 2000, half=5.0) for _ in range(4)]
    poses = np.array([_pose(rng, scale=600.0) for _ in clouds])
    s = _store(clouds)
    got = s.assemble(range(4), poses, 0.3, 0.01)
    cat = ref.assemble_ref(clouds, range(4), poses, 0.3)
    assert _same(got, cat)  # returned as the unfiltered concatenation, as PCL does
    assert _same(got, ref.assemble_ref(clouds, range(4), poses, 0.3, 0.01))


def test_many_segments_of_mixed_sizes():
    """Sizes around the 8192-point tile of the bbox / key kernels and a 256-thread block, more than 256 keyframes, repeated ids."""
    rng = np.random.default_rng(6)
    sizes = [1, 2, 255, 256, 257, 8191, 8192, 8193, 16385, 0, 31, 4096] + list(rng.integers(0, 400, 300))
    clouds = [_cloud(rng, int(n), half=rng.uniform(2, 20)) for n in sizes]
    s = _store(clouds)
    ids = list(range(len(clouds))) + [6, 6, 0, 8]
    poses = np.array([_pose(rng) for _ in ids])
    assert len(ids) > 300
    got = s.assemble(ids, poses, 0.3)
    assert _same(got, ref.assemble_ref(clouds, ids, poses, 0.3))
    got = s.assemble(ids, poses, 0.4, 0.7)
    assert _same(got, ref.assemble_ref(clouds, ids, poses, 0.4, 0.7))
    rev = ids[::-1]
    got = s.assemble(rev, poses[::-1], 0.3, 0.3)
    assert _same(got, ref.assemble_ref(clouds, rev, poses[::-1], 0.3, 0.3))


def test_segments_equal_fls_voxel_grid_then_transform(keyframes):
    from funny_lidar_slam_b200.registration import voxel_grid
    clouds, poses = keyframes
    s = _store(clouds[:6])
    got = s.assemble(range(6), poses[:6], 0.2)
    parts = [ref.orc_transform(voxel_grid(c, 0.2), T) for c, T in zip(clouds[:6], poses[:6])]
    assert _same(got, np.concatenate(parts))


def test_pcl_layout_store_equals_packed(keyframes):
    clouds, poses = keyframes
    a, b = _store(clouds[:3]), _store([to_pcl(c) for c in clouds[:3]])
    assert _same(a.assemble(range(3), poses[:3], 0.3, 0.3), b.assemble(range(3), poses[:3], 0.3, 0.3))


# ---- base, device output --------------------------------------------------------------------------------------------------------
def test_base_present_absent_empty(keyframes):
    import torch
    clouds, poses = keyframes
    s = _store(clouds[:4])
    rng = np.random.default_rng(8)
    base = _cloud(rng, 7000, half=40.0)
    d_base = torch.from_numpy(base).cuda()
    torch.cuda.synchronize()
    for final in (None, 0.3):
        got = s.assemble(range(4), poses[:4], 0.3, final, base=(d_base.data_ptr(), len(base)))
        assert _same(got, ref.assemble_ref(clouds, range(4), poses[:4], 0.3, final, base)), final
        got = s.assemble(range(4), poses[:4], 0.3, final, base=(d_base.data_ptr(), 0))
        assert _same(got, ref.assemble_ref(clouds, range(4), poses[:4], 0.3, final)), final
        got = s.assemble(range(4), poses[:4], 0.3, final)
        assert _same(got, ref.assemble_ref(clouds, range(4), poses[:4], 0.3, final)), final
        got = s.assemble([], np.zeros((0, 4, 4)), 0.3, final, base=(d_base.data_ptr(), len(base)))
        assert _same(got, ref.assemble_ref(clouds, [], [], 0.3, final, base)), final


def test_device_output_and_aliasing(keyframes):
    import torch
    clouds, poses = keyframes
    s = _store(clouds[:3])
    want = ref.assemble_ref(clouds, range(3), poses[:3], 0.3, 0.3)
    for final in (None, 0.3):
        w = ref.assemble_ref(clouds, range(3), poses[:3], 0.3, final)
        d = torch.full((len(w) + 10, 4), float("nan"), dtype=torch.float32, device="cuda:0")
        torch.cuda.synchronize()
        assert s.assemble(range(3), poses[:3], 0.3, final, device_out=(d.data_ptr(), d.shape[0]), host_out=False) is None
        assert s.last_count == len(w)
        assert _same(d[:len(w)].cpu().numpy(), w)
        assert torch.isnan(d[len(w):]).all()
    d = torch.zeros((len(want) * 2, 4), dtype=torch.float32, device="cuda:0")
    torch.cuda.synchronize()
    from funny_lidar_slam_b200._lib import FlsError
    with pytest.raises(FlsError) as e:  # a base inside the output buffer
        s.assemble(range(3), poses[:3], 0.3, 0.3, base=(d.data_ptr() + 16, 5), device_out=(d.data_ptr(), d.shape[0]))
    assert e.value.status == _abi.FLS_ERR_INVALID_ARG


# ---- errors -------------------------------------------------------------------------------------------------------------------
def test_capacity_and_id_errors(keyframes):
    from funny_lidar_slam_b200._lib import lib
    from funny_lidar_slam_b200.keyframes import KeyFrameStore
    clouds, poses = keyframes
    L = lib()
    s = KeyFrameStore(len(clouds[0]) + len(clouds[1]))
    s.add(clouds[0])
    p = clouds[1].ctypes.data_as(C.c_void_p)
    assert L.fls_keyframes_add(s._s, 0, p, len(clouds[1]), 16) == _abi.FLS_ERR_INVALID_ARG  # id already taken
    assert L.fls_keyframes_add(s._s, 2, p, len(clouds[1]), 16) == _abi.FLS_ERR_INVALID_ARG  # id skips one
    big = np.concatenate([clouds[1], clouds[1][:1]])
    assert L.fls_keyframes_add(s._s, 1, big.ctypes.data_as(C.c_void_p), len(big), 16) == _abi.FLS_ERR_CAPACITY
    assert len(s) == 1 and s.n_points == len(clouds[0])
    s.add(clouds[1])
    assert s.n_points == len(clouds[0]) + len(clouds[1])
    assert L.fls_keyframes_add(s._s, 2, p, 1, 16) == _abi.FLS_ERR_CAPACITY
    assert L.fls_keyframes_add(s._s, 2, None, 0, 16) == _abi.FLS_OK  # an empty keyframe always fits
    # output capacity: *n_out gets the size the map needs, nothing is written
    want = ref.assemble_ref(clouds, [0, 1], poses[:2], 0.3, 0.3)
    ids = np.array([0, 1], np.int64)
    Tc = np.ascontiguousarray(np.transpose(poses[:2], (0, 2, 1)))
    for final in (0.3, 0.0):
        w = want if final else ref.assemble_ref(clouds, [0, 1], poses[:2], 0.3)
        out = np.full((len(w), 4), np.nan, np.float32)
        n = C.c_size_t(0)
        rc = L.fls_keyframes_assemble(s._s, ids.ctypes.data_as(C.c_void_p), 2, Tc.ctypes.data_as(C.c_void_p), 0.3, final, None, 0,
                                      out.ctypes.data_as(C.c_void_p), None, len(w) - 1, C.byref(n), None)
        assert rc == _abi.FLS_ERR_CAPACITY and n.value == len(w)
        assert np.isnan(out).all()
        rc = L.fls_keyframes_assemble(s._s, ids.ctypes.data_as(C.c_void_p), 2, Tc.ctypes.data_as(C.c_void_p), 0.3, final, None, 0, None, None, 0,
                                      C.byref(n), None)
        assert rc == _abi.FLS_ERR_CAPACITY and n.value == len(w)  # size query
        rc = L.fls_keyframes_assemble(s._s, ids.ctypes.data_as(C.c_void_p), 2, Tc.ctypes.data_as(C.c_void_p), 0.3, final, None, 0,
                                      out.ctypes.data_as(C.c_void_p), None, len(w), C.byref(n), None)
        assert rc == _abi.FLS_OK and n.value == len(w) and _same(out, w)
    bad = np.array([0, 3], np.int64)
    n = C.c_size_t(0)
    assert L.fls_keyframes_assemble(s._s, bad.ctypes.data_as(C.c_void_p), 2, Tc.ctypes.data_as(C.c_void_p), 0.3, 0.3, None, 0, None, None, 0,
                                    C.byref(n), None) == _abi.FLS_ERR_INVALID_ARG


# ---- device-added keyframes ----------------------------------------------------------------------------------------------------
def test_device_added_store_equals_host_added(world):
    import torch
    from funny_lidar_slam_b200.features import LoamFrontEnd, preprocess_device
    from funny_lidar_slam_b200.keyframes import KeyFrameStore
    from tests.test_gpu_preprocess_loam import _raw_scan, _shape
    traj = synth.trajectory(6)
    V, H, h_res = _shape("hdl64")
    fe = LoamFrontEnd(H, V, h_res, 1.0, 100.0, 1.0, 0.1, 0.2, 0.4)
    host, dev = KeyFrameStore(4_000_000), KeyFrameStore(4_000_000)
    poses, clouds = [], []
    for i in range(3):
        raw, ring, time = _raw_scan(world, traj[i], "hdl64", 40 + i)
        d_xyzi = torch.from_numpy(np.ascontiguousarray(raw)).cuda()
        d_ring = torch.from_numpy(ring).cuda()
        d_time = torch.from_numpy(time).cuda()
        d_ord = torch.empty((len(raw), 4), dtype=torch.float32, device="cuda:0")
        d_pl = torch.empty((V * H, 4), dtype=torch.float32, device="cuda:0")
        torch.cuda.synchronize()
        ordered, _ = preprocess_device(d_xyzi.data_ptr(), d_time.data_ptr(), len(raw), None, 1.0, 100.0, 1, 0.5,
                                       device_out=(d_ord.data_ptr(), 0))
        _, planar = fe.run_device(d_xyzi.data_ptr(), d_ring.data_ptr(), d_time.data_ptr(), len(raw), device_out=(0, d_pl.data_ptr()))
        host.add(ordered)
        dev.add_device(d_ord.data_ptr(), len(ordered))
        host.add(planar)
        dev.add_device(d_pl.data_ptr(), fe.last_counts[1])
        poses += [traj[i], traj[i]]
        clouds += [ordered, planar]
    ids = list(range(6))
    g_host = host.assemble(ids, poses, 0.3, 0.3)
    g_dev = dev.assemble(ids, poses, 0.3, 0.3)
    assert len(g_host) > 1000 and _same(g_host, g_dev)
    assert _same(g_dev, ref.assemble_ref(clouds, ids, poses, 0.3, 0.3))


# ---- host waits and launches, threads -------------------------------------------------------------------------------------------
def test_waits_and_launches_do_not_depend_on_the_keyframe_count():
    rng = np.random.default_rng(9)
    clouds = [_cloud(rng, int(n)) for n in rng.integers(500, 3000, 300)]
    s = _store(clouds)
    poses = np.array([_pose(rng) for _ in clouds])
    for final in (None, 0.3):
        s.assemble([0], poses[:1], 0.3, final)
        a = (s.last_stats.gpu_launches, s.last_stats.iterations)
        s.assemble(range(300), poses, 0.3, final)
        b = (s.last_stats.gpu_launches, s.last_stats.iterations)
        assert a == b, (final, a, b)
        assert b[1] == (4 if final else 2)
        assert s.last_stats.n_source == sum(len(c) for c in clouds) and s.last_stats.gpu_ms > 0


def test_two_threads_share_one_store(keyframes):
    clouds, poses = keyframes
    s = _store(clouds)
    jobs = [(list(range(12)), 0.3, 0.3), (list(range(3, 9)), 0.2, None)] * 3
    serial = [s.assemble(ids, poses[ids], leaf, fin) for ids, leaf, fin in jobs]
    results = [None] * len(jobs)

    def work(j):
        ids, leaf, fin = jobs[j]
        results[j] = s.assemble(ids, poses[ids], leaf, fin)

    threads = [threading.Thread(target=work, args=(j,)) for j in range(len(jobs))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for a, b in zip(results, serial):
        assert _same(a, b)
