"""The velocity-aware de-skew oracle (oracle_motion/orc_motion.h) against the 50-digit reference (tests/deskew_motion_ref.py) on the
de-skew and projector edge scenes of tests/frontend_scenes.py; bit-identical to the rotation-only oracle without a velocity; and the
moving-sensor scene (tests/deskew_motion_scene.py) whose thresholds the GPU test uses, rehearsed here through the oracle."""
import numpy as np
import pytest

from oracle import pyoracle as orc
from oracle_motion import pyoracle_motion as orcm
from tests import deskew_motion_ref as mref
from tests import deskew_motion_scene as ms
from tests import frontend_scenes as fs
from tests.test_oracle_frontend_edges import check_ordered, same_bits

NZ_DESKEW, NZ_PROJECT = ms.negative_zero_scenes()
DESKEW = fs.deskew_scenes() + [NZ_DESKEW]
PROJECT = fs.project_scenes() + [NZ_PROJECT]
# 0, +-1e-300 (the term is below every float spacing), 1, 30 and 1e6 m/s, components of both signs
VELOCITIES = {"tiny": (1e-300, -1e-300, 1e-300), "1": (0.6, -0.8, 0.0), "30": (-18.0, 24.0, 0.5), "1e6": (1e6, -6e5, 2.5e5)}
ZEROS = {"null": None, "zero": (0.0, 0.0, 0.0), "signed_zero": (-0.0, 0.0, -0.0)}


def _report(name, decided):
    n_und = int((~decided).sum())
    if n_und:
        print(f"{name}: {n_und} undecided coordinates (not asserted)")


@pytest.mark.parametrize("v", VELOCITIES.values(), ids=list(VELOCITIES))
@pytest.mark.parametrize("s", DESKEW, ids=[s["name"] for s in DESKEW])
def test_preprocess_matches_reference(s, v):
    args = (s["min_d"], s["max_d"], s["jump"], s["leaf"])
    o_ord, o_pl = orcm.preprocess(s["raw"], s["imu"], v, *args)
    r = mref.preprocess(s["raw"], s["imu"], v, *args)
    check_ordered(o_ord, r["ordered"], r["decided"])
    _report(s["name"], r["decided"])
    if r["decided"].all():  # the planar candidates are the reference's; the voxel filter itself is tested on its own edges
        assert same_bits(o_pl, orc.voxel_grid(r["planar_in"], s["leaf"]))


@pytest.mark.parametrize("v", ZEROS.values(), ids=list(ZEROS))
@pytest.mark.parametrize("s", DESKEW, ids=[s["name"] for s in DESKEW])
def test_zero_velocity_is_the_rotation_only_oracle(s, v):
    args = (s["min_d"], s["max_d"], s["jump"], s["leaf"])
    m_ord, m_pl = orcm.preprocess(s["raw"], s["imu"], v, *args)
    o_ord, o_pl = orc.preprocess(s["raw"], s["imu"], *args)
    assert same_bits(m_ord, o_ord) and same_bits(m_pl, o_pl)
    assert np.array_equal(np.signbit(m_ord), np.signbit(o_ord))  # a -0.0 stays -0.0: the term is skipped, not added as +0.0


def _negative_zeros(a):
    a = np.asarray(a)[:, :3]
    return (a == 0) & np.signbit(a)


def test_negative_zero_scenes_tell_skipping_from_adding_zero():
    """The rotation-only outputs of the negative-zero scenes hold -0.0 coordinates, which a term added as +0.0 would turn into +0.0:
    the zero-velocity tests above and in test_gpu_deskew_motion.py would see that."""
    d, p = NZ_DESKEW, NZ_PROJECT
    o_ord, _ = orc.preprocess(d["raw"], d["imu"], d["min_d"], d["max_d"], d["jump"], d["leaf"])
    pr = orc.project_imu(p["raw"], p["ring"], p["time"], p["imu"], p["V"], p["H"], p["h_res"], p["min_d"], p["max_d"])
    for out in (o_ord, pr["ordered"]):
        nz = _negative_zeros(out)
        assert nz.any()
        assert not _negative_zeros(out[:, :3] + np.float32(0.0)).any()  # what adding +0.0 would give


def test_term_moves_every_point_off_the_reference_time():
    """On the main scene, 30 m/s changes exactly the points whose stamp differs from ref_time, by about |v| |dt|."""
    s = DESKEW[0]
    args = (s["min_d"], s["max_d"], s["jump"], s["leaf"])
    v = np.array(VELOCITIES["30"])
    rot = mref.preprocess(s["raw"], s["imu"], None, *args)
    mot = mref.preprocess(s["raw"], s["imu"], tuple(v), *args)
    assert np.array_equal(rot["raw_index"], mot["raw_index"])
    dt = np.array([(fs.ref.point_time(s["imu"]["ref_time_us"], s["raw"][i, 4]) - s["imu"]["ref_time_us"]) * 1e-6 for i in rot["raw_index"]])
    assert (dt < 0).any() and (dt > 0).any() and (dt == 0).any()
    fin = np.isfinite(rot["ordered"][:, 0])
    shift = np.linalg.norm(mot["ordered"][fin, :3].astype(np.float64) - rot["ordered"][fin, :3], axis=1)
    assert np.all(np.abs(shift - np.linalg.norm(v) * np.abs(dt[fin])) < 1e-5)


@pytest.mark.parametrize("v", [VELOCITIES["30"], VELOCITIES["1e6"]], ids=["30", "1e6"])
@pytest.mark.parametrize("s", PROJECT, ids=[s["name"] for s in PROJECT])
def test_project_matches_reference(s, v):
    a = (s["V"], s["H"], s["h_res"], s["min_d"], s["max_d"])
    o = orcm.project_imu(s["raw"], s["ring"], s["time"], s["imu"], v, *a)
    r = mref.project(s["raw"], s["ring"], s["time"], s["imu"], v, *a)
    assert o["n"] == r["n"]
    for k in ("depth", "col", "row_start", "row_end"):
        assert np.array_equal(o[k], r[k]), k
    check_ordered(o["ordered"], r["ordered"], r["decided"])
    _report(s["name"], r["decided"])
    plain = orc.project_imu(s["raw"], s["ring"], s["time"], s["imu"], *a)  # cells, depth and columns are the raw points'
    assert o["n"] == plain["n"] and np.array_equal(o["depth"], plain["depth"]) and np.array_equal(o["col"], plain["col"])


@pytest.mark.parametrize("v", ZEROS.values(), ids=list(ZEROS))
@pytest.mark.parametrize("s", PROJECT, ids=[s["name"] for s in PROJECT])
def test_project_zero_velocity_is_the_rotation_only_oracle(s, v):
    a = (s["V"], s["H"], s["h_res"], s["min_d"], s["max_d"])
    o = orcm.project_imu(s["raw"], s["ring"], s["time"], s["imu"], v, *a)
    p = orc.project_imu(s["raw"], s["ring"], s["time"], s["imu"], *a)
    for k in ("depth", "col", "row_start", "row_end"):
        assert np.array_equal(o[k], p[k]), k
    assert o["n"] == p["n"] and same_bits(o["ordered"], p["ordered"])


# ---- the moving sensor: thresholds of tests/test_gpu_deskew_motion.py, rehearsed on the oracle -------------------------------------
SPEED = 15.0


def check_sweep(s, ordered_motion, ordered_rot):
    """The de-skewed cloud lies on the surfaces the sensor hit, within the scan noise; the rotation-only one is v * dt off."""
    assert len(ordered_motion) == len(ordered_rot) == len(s["raw"])
    e_hit, e_surf = ms.world_error(ordered_motion, s)
    noise = np.linalg.norm(s["hit"] - s["surface"], axis=1)
    assert e_hit.max() < 1e-3, e_hit.max()
    assert np.all(e_surf <= noise + 1e-3)
    r_hit, _ = ms.world_error(ordered_rot, s)
    assert np.all(np.abs(r_hit - SPEED * s["dt"]) < 1e-3)
    print(f"world error: with the term max {e_hit.max():.2e} m (max {e_surf.max():.3f} m to the noise-free surface); rotation only max "
          f"{r_hit.max():.3f} m (v * max dt = {SPEED * s['dt'].max():.3f} m)")
    return r_hit.max()


def check_match(err_motion, err_rot):
    print(f"LOAM-iVox Match vs the true pose: with the term {err_motion[0]:.4f} m / {err_motion[1]:.5f} rad, rotation only "
          f"{err_rot[0]:.4f} m / {err_rot[1]:.5f} rad")
    assert err_motion[0] < 0.05 and err_rot[0] > 0.3 and err_motion[0] < err_rot[0]


def test_moving_sensor_rehearsal(world, traj):
    from funny_lidar_slam_b200 import FLS_P2PLANE_IVOX, default_config, synth
    s = ms.moving_sweep(world, traj[3], speed=SPEED)
    assert 100_000 < len(s["raw"]) < 120_000
    a = (ms.MIN_D, ms.MAX_D, ms.JUMP, ms.LEAF)
    o_mot, p_mot = orcm.preprocess(s["raw"], s["imu"], s["velocity"], *a)
    o_rot, p_rot = orc.preprocess(s["raw"], s["imu"], *a)
    check_sweep(s, o_mot, o_rot)
    mp = ms.surface_map(world, traj[3])
    cfg = default_config(FLS_P2PLANE_IVOX)
    guess = synth.perturb_pose(traj[3], dpos=0.2, drot_deg=1.0, seed=5)
    errs = []
    for pl in (p_mot, p_rot):
        r = orc.Registration(cfg)
        r.add_cloud(mp)
        ok, T, _ = r.match(pl, guess)
        assert ok
        errs.append(synth.pose_error(T, traj[3]))
    check_match(*errs)
