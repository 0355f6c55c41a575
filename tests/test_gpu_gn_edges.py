"""GPU: the Gauss-Newton step every persistent Match kernel runs after its sums (gn_step_pre: the 6x6 solve, the pose update and the
stop rule) against the high-precision reference of tests/gn_ref.py, proven against the oracle by tests/test_oracle_gn_edges.py.

  * every constructed case of tests/gn_cases.py through fls_gn_step_probe: the fast-path decision, dx (bit for bit where the reference
    knows the exact double, else within its bound), the pose, the stop word the step publishes, converged / failed / done, the last
    norms and the result record;
  * whole Matches replayed from their FLS_FLAG_ITER_LOG logs: ICP, NDT single and batch, LOAM-iVox single (v8) and batches of 1, 9
    and 64 scans (v9), kd-tree LOAM, LoamFull on the host route and through fls_match_cluster_device: every logged dx within its
    bound of the reference solve of the logged H and g, the returned pose equal to the pose composed from the logged dx, the
    iteration count and converged flag equal to the reference's decisions, and the result record the kernel writes equal to the
    returned pose bit for bit.  Among them a floor that puts the LOAM kernels on the pivoting solver, a Match that ends through
    LOAM's second clause, one that hits max_iterations and an NDT Match that fails its gate at iteration 1."""
import numpy as np
import pytest

from oracle import pyoracle as orc
from tests import gn_cases, gn_ref
from tests.test_oracle_gn_edges import CASES, KINDS, SCENE_NAMES, assert_reaches, reference

pytestmark = pytest.mark.gpu
EPS = gn_ref.EPS


def _probe(cases):
    from funny_lidar_slam_b200.registration import gn_step_probe
    return gn_step_probe([c.probe() for c in cases])


def _bits(a):
    return np.asarray(a, np.float64).view(np.int64)


def _check_record(c, o):
    """The published records and the result record against the state the step left."""
    assert o["published_ok"], c.name
    assert np.array_equal(o["published_R"], o["R"], equal_nan=True) and np.array_equal(o["published_t"], o["t"], equal_nan=True), c.name
    assert o["published_stop"] == (1.0 if o["done"] else 0.0), c.name
    r = o["result"]
    if not o["done"]:
        assert np.all(np.isnan(r)), c.name
        return
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = o["R"], o["t"]
    assert np.array_equal(r[:16], T.T.reshape(16), equal_nan=True), (c.name, r[:16])  # column-major Mat4d, [15] = 1
    assert r[16] == (1.0 if o["converged"] > 0 else 0.0) and r[17] == c.iter + 1, (c.name, r[16:])


def _check_case(c, o):
    s = reference(c.name)
    H, g, n_valid = gn_ref.unpack(c.tot)
    assert np.array_equal(o["H"], H, equal_nan=True) and np.array_equal(o["g"], g, equal_nan=True), c.name
    assert o["n_valid"] == n_valid and o["iter"] == c.iter + 1, c.name
    _check_record(c, o)
    if "spd" in c.expect:
        assert o["spd"] == c.expect["spd"], (c.name, o["spd"])
    if s.spd_decided and c.kind != "nan":
        assert o["spd"] == s.spd, (c.name, o["spd"], s.spd_margins)
    if o["spd"] and c.kind != "nan":
        assert o["det_spd"] > 0, c.name
    if c.kind == "nan":
        return _check_nan(c, o, s)
    if not s.path_decided:
        return
    if s.path in ("gate_fail", "skip"):
        assert np.array_equal(o["R"], c.R) and np.array_equal(o["t"], c.t) and np.all(o["dx"] == 0), (c.name, s.path)
        assert o["failed"] == (1 if s.path == "gate_fail" else 0), c.name
    if s.path == "gate_fail":
        assert o["converged"] == 0 and o["done"] == 1, c.name
    if s.stop_decided:
        assert o["done"] == int(s.stop), (c.name, o["done"], s.stop_by, {k: v for k, v in s.clauses.items()})
    assert o["converged"] == (s.converged if s.converged >= 0 else 0), (c.name, o["converged"], s.converged)
    if s.path != "update":
        return
    # dx
    if s.dx_exact is not None:
        assert np.array_equal(o["dx"], s.dx_exact), (c.name, o["dx"], s.dx_exact)
    else:
        err = np.abs(o["dx"] - np.array([float(a) for a in s.dx]))
        assert np.all(err <= s.dx_bound), (c.name, err, s.dx_bound)
        if s.qr is not None and s.rank_decided:
            assert all(o["dx"][i] == 0 for i in range(6) if i not in s.qr.cols[:s.rank]), (c.name, o["dx"])
    # pose
    Rr = np.array(s.R.tolist(), dtype=float)
    tr = np.array([float(a) for a in s.t])
    if s.exp is not None and s.exp.decided and not s.exp.applied and s.dx_exact is not None:
        assert np.array_equal(o["R"], c.R), c.name  # Exp = I: the product with the identity is exact
    rt, tt = gn_ref.pose_tol(s, c.t)
    assert np.max(np.abs(o["R"] - Rr)) <= rt, (c.name, np.max(np.abs(o["R"] - Rr)), rt)
    assert np.max(np.abs(o["t"] - tr)) <= tt, (c.name, np.max(np.abs(o["t"] - tr)), tt)
    # the norms LOAM carries to the next iteration
    if c.method in gn_ref.LOAM:
        rn, pn = np.linalg.norm(o["dx"][0:3]), np.linalg.norm(o["dx"][3:6])
        assert abs(o["last_rot"] - rn) <= 4 * EPS * rn and abs(o["last_pos"] - pn) <= 4 * EPS * pn, c.name
        if s.dx_exact is not None and sum(1 for a in s.dx_exact[0:3] if a) <= 1 and sum(1 for a in s.dx_exact[3:6] if a) <= 1:
            assert (o["last_rot"], o["last_pos"]) == s.new_last, c.name
    else:
        assert o["last_rot"] == c.last_rot and o["last_pos"] == c.last_pos, c.name


def _check_nan(c, o, s):
    """NaN systems: the device equals the oracle's solver of the path it took, NaN for NaN; NaN norms never stop the loop."""
    H, g, _ = gn_ref.unpack(c.tot)
    if not o["spd"]:
        ref = orc.solve6_fullpiv(H, g) if c.method in gn_ref.LOAM else orc.solve6_lu(H, g)[0]
        if c.method == gn_ref.ICP and orc.solve6_lu(H, g)[1] == 0:
            ref = np.zeros(6)
        assert np.array_equal(np.isnan(o["dx"]), np.isnan(ref)), (c.name, o["dx"], ref)
        fin = ~np.isnan(ref)
        assert np.allclose(o["dx"][fin], ref[fin], rtol=1e-9, atol=1e-12), (c.name, o["dx"], ref)
    if np.isnan(o["dx"]).any():
        assert not o["done"], c.name
        assert np.isnan(o["R"]).any() or np.isnan(o["t"]).any(), c.name


@pytest.mark.parametrize("kind", KINDS)
def test_step_probe_cases(kind):
    cases = [c for c in CASES.values() if c.kind == kind]
    for c, o in zip(cases, _probe(cases)):
        _check_case(c, o)


def test_step_probe_is_one_launch_over_all_cases():
    """All cases in one call give what they give one at a time (one thread per case, nothing shared)."""
    cases = list(CASES.values())
    together = _probe(cases)
    for i in (0, 57, len(cases) - 1):
        alone = _probe([cases[i]])[0]
        for k in ("R", "t", "dx", "result"):
            assert np.array_equal(_bits(alone[k]), _bits(together[i][k])), (cases[i].name, k)


# ---- whole Matches ----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def match_scenes(world, traj, scene16):
    scenes = gn_cases.synth_scenes(world, traj, scene16) + gn_cases.edge_scenes() + [gn_cases.floor_scene(gn_cases.IVOX),
                                                                                     gn_cases.floor_scene(gn_cases.KNN)]
    return {s.name: s for s in scenes}


def _registration(s):
    from funny_lidar_slam_b200.registration import Registration
    g = Registration(s.config())
    g.AddCloudToLocalMap(s.maps)
    return g


def _result_buffer(g, n):
    import torch

    from funny_lidar_slam_b200 import parallel
    buf = torch.full((n * parallel.RESULT_LEN,), -7.0, dtype=torch.float64, device="cuda:0")
    g.set_result_buffer_device(buf.data_ptr(), n)
    return buf


def _check_result(buf, s_idx, T, ok, iterations, tag):
    from funny_lidar_slam_b200 import parallel
    r = buf.cpu().numpy().reshape(-1, parallel.RESULT_LEN)[s_idx]
    assert np.array_equal(_bits(r[:16]), _bits(np.asarray(T).T.reshape(16))), (tag, r[:16], T)
    assert r[16] == (1.0 if ok else 0.0) and r[17] == iterations, (tag, r[16:])


def _replay_check(s, g, T, ok, st, scan=0, T0=None, tag=""):
    logs = g.iter_log(scan)
    assert len(logs) == st.iterations, tag
    rep = gn_ref.replay(s.method, s.T if T0 is None else T0, logs, gn_ref.params_of(g.cfg))
    gn_ref.assert_replay(rep, logs, T, st.iterations, ok, tag or s.name)
    assert_reaches(s, rep, logs)
    return rep


@pytest.mark.parametrize("name", SCENE_NAMES)
def test_match_replays(match_scenes, name):
    from funny_lidar_slam_b200.registration import PointcloudCluster
    s = match_scenes[name]
    g = _registration(s)
    buf = _result_buffer(g, 1)
    T = s.T.copy()
    if s.method in (gn_cases.ICP, gn_cases.NDT):
        cl = PointcloudCluster(ordered_cloud=s.scan)
    else:
        cl = PointcloudCluster(planar_cloud=s.scan, corner_cloud=s.corner)
    ok = g.Match(cl, T)
    st = g.last_stats
    _replay_check(s, g, T, ok, st)
    _check_result(buf, 0, T, ok, st.iterations, name)
    g.set_result_buffer_device(0, 0)


def test_loam_full_cluster_device_replay(match_scenes):
    import torch
    s = match_scenes["synth_full"]
    g = _registration(s)
    buf = _result_buffer(g, 1)
    d_p = torch.from_numpy(np.ascontiguousarray(s.scan, np.float32)).cuda()
    d_c = torch.from_numpy(np.ascontiguousarray(s.corner, np.float32)).cuda()
    T = s.T.copy()
    ok = g.match_cluster_device(0, 0, d_p.data_ptr(), len(s.scan), d_c.data_ptr(), len(s.corner), T)
    st = g.last_stats
    _replay_check(s, g, T, ok, st, tag="full_cluster_device")
    _check_result(buf, 0, T, ok, st.iterations, "full_cluster_device")
    g.set_result_buffer_device(0, 0)


def _batch_guesses(traj, B):
    from funny_lidar_slam_b200 import synth
    return np.stack([synth.perturb_pose(traj[5], seed=300 + i, dpos=0.05 + 0.3 * (i % 5) / 4, drot_deg=0.5 + 2.5 * (i % 7) / 6)
                     for i in range(B)])


@pytest.mark.parametrize("B", [1, 9, 64])
def test_ivox_batch_replays(match_scenes, traj, B):
    """The v9 batch kernel runs gn_step_pre at its own call site: every scan of the batch replays."""
    s = match_scenes["synth_ivox"]
    g = _registration(s)
    buf = _result_buffer(g, B)
    Ts0 = _batch_guesses(traj, B)
    scans = [s.scan[: len(s.scan) - 97 * (i % 11)] for i in range(B)]
    conv, Ts = g.match_batch(scans, Ts0)
    its = []
    for i in range(B):
        st = g.last_batch_stats[i]
        _replay_check(s, g, Ts[i], bool(conv[i]), st, scan=i, T0=Ts0[i], tag=f"ivox_batch{B}_{i}")
        _check_result(buf, i, Ts[i], bool(conv[i]), st.iterations, f"ivox_batch{B}_{i}")
        its.append(st.iterations)
    if B > 1:
        assert len(set(its)) > 1, its  # the scans stop at different iterations
    g.set_result_buffer_device(0, 0)


def test_ndt_batch_replays(match_scenes, traj):
    s = match_scenes["synth_ndt"]
    g = _registration(s)
    buf = _result_buffer(g, 3)
    Ts0 = _batch_guesses(traj, 3)
    conv, Ts = g.match_batch([s.scan, s.scan[:-500], s.scan[::2]], Ts0)
    for i in range(3):
        st = g.last_batch_stats[i]
        _replay_check(s, g, Ts[i], bool(conv[i]), st, scan=i, T0=Ts0[i], tag=f"ndt_batch_{i}")
        _check_result(buf, i, Ts[i], bool(conv[i]), st.iterations, f"ndt_batch_{i}")
    g.set_result_buffer_device(0, 0)
