"""The front-end kernels on the edge scenes of tests/frontend_scenes.py, through every route that reaches each stage: equal to the
reference (tests/frontend_ref.py) wherever it is decided, and to the oracle bit for bit everywhere (NaN-aware)."""
import numpy as np
import pytest

from oracle import pyoracle as orc
from tests import frontend_ref as ref
from tests import frontend_scenes as fs
from tests.test_oracle_frontend_edges import check_ordered, same_bits

pytestmark = pytest.mark.gpu

DESKEW = fs.deskew_scenes()
PROJECT = fs.project_scenes()
FEATURES = fs.feature_scenes()
VOXEL = fs.voxel_scenes()


def _device_preprocess(s):
    import torch
    from funny_lidar_slam_b200.features import preprocess_device
    raw = s["raw"]
    dx = torch.from_numpy(np.ascontiguousarray(raw[:, :4])).to("cuda:0")
    dt = torch.from_numpy(np.ascontiguousarray(raw[:, 4])).to("cuda:0")
    torch.cuda.synchronize()
    return preprocess_device(dx.data_ptr(), dt.data_ptr(), len(raw), s["imu"], s["min_d"], s["max_d"], s["jump"], s["leaf"])


@pytest.mark.parametrize("route", ["host", "device"])
@pytest.mark.parametrize("s", DESKEW, ids=[s["name"] for s in DESKEW])
def test_preprocess_edges(s, route):
    from funny_lidar_slam_b200.features import preprocess
    if route == "device" and len(s["raw"]) == 0:
        pytest.skip("no device array of zero points")
    args = (s["raw"], s["imu"], s["min_d"], s["max_d"], s["jump"], s["leaf"])
    g_ord, g_pl = preprocess(*args) if route == "host" else _device_preprocess(s)
    o_ord, o_pl = orc.preprocess(*args)
    r = ref.preprocess(*args)
    assert same_bits(g_ord, o_ord) and same_bits(g_pl, o_pl)
    check_ordered(g_ord, r["ordered"], r["decided"])
    if r["decided"].all():
        assert same_bits(g_pl, r["planar"])


def test_nan_point_time_is_outside_the_buffer():
    """A point time of NaN converts to INT64_MIN (x86-64's rule, which the oracle pins): the point is dropped by the pre-processing
    and does not claim its projector cell, so the next point of that cell wins."""
    from funny_lidar_slam_b200.features import PointcloudProjector, preprocess, project_imu
    s = DESKEW[0]
    i = int(np.nonzero(np.isnan(s["raw"][:, 4]))[0][0])
    one = s["raw"][i:i + 1]
    assert len(preprocess(one, s["imu"], 0.0, 1e9, 1, 0.5)[0]) == 0
    p = PROJECT[0]
    pr = PointcloudProjector(p["H"], p["V"], p["h_res"], p["min_d"], p["max_d"])
    cell = p["probes"][14:19]
    sel = [cell[2], cell[3]]  # the NaN-time point first, then an in-window point of the same cell
    g = project_imu(pr, p["raw"][sel], p["ring"][sel], p["time"][sel], p["imu"])
    assert g["n"] == 1 and np.array_equal(g["depth"][:1], [ref.depth_f32(*p["raw"][cell[3], :3])])


def test_descending_stamps_are_rejected():
    from funny_lidar_slam_b200._lib import FlsError
    from funny_lidar_slam_b200.features import PointcloudProjector, preprocess, project_imu
    imu = fs._imu([-2000, 1000, -500, 3000], fs._QUATS[:4])
    raw = fs._raw([fs.rel_for(k) for k in (-1500, 0, 900)], np.random.default_rng(4))
    with pytest.raises(FlsError):
        preprocess(raw, imu, 0.5, 100.0, 1, 0.5)
    pr = PointcloudProjector(16, 4, 0.01, 0.5, 100.0)
    with pytest.raises(FlsError):
        project_imu(pr, raw[:, :4], np.zeros(3, np.int32), raw[:, 4], imu)
    equal = fs._imu([-2000, 1000, 1000, 3000], fs._QUATS[:4])  # equal neighbours stay allowed
    assert same_bits(preprocess(raw, equal, 0.5, 100.0, 1, 0.5)[0], orc.preprocess(raw, equal, 0.5, 100.0, 1, 0.5)[0])


@pytest.mark.parametrize("s", PROJECT, ids=[s["name"] for s in PROJECT])
def test_project_edges(s):
    from funny_lidar_slam_b200.features import PointcloudProjector, project_imu
    pr = PointcloudProjector(s["H"], s["V"], s["h_res"], s["min_d"], s["max_d"])
    g = project_imu(pr, s["raw"], s["ring"], s["time"], s["imu"])
    o = orc.project_imu(s["raw"], s["ring"], s["time"], s["imu"], s["V"], s["H"], s["h_res"], s["min_d"], s["max_d"])
    r = ref.project(s["raw"], s["ring"], s["time"], s["imu"], s["V"], s["H"], s["h_res"], s["min_d"], s["max_d"])
    assert g["n"] == o["n"] == r["n"]
    for k in ("depth", "col", "row_start", "row_end"):
        assert np.array_equal(g[k], o[k]) and np.array_equal(g[k], r[k]), k
    assert same_bits(g["ordered"], o["ordered"])
    check_ordered(g["ordered"], r["ordered"], r["decided"])


@pytest.mark.parametrize("s", FEATURES, ids=[s["name"] for s in FEATURES])
def test_features_edges(s):
    from funny_lidar_slam_b200.features import FeatureExtractor
    for ct, pt in s["cfgs"]:
        gc, gp = FeatureExtractor(ct, pt).extract_indices(s["depth"], s["col"], s["n"], s["row_start"], s["row_end"])
        oc, op, _ = orc.extract_features(s["depth"], s["col"], s["n"], s["row_start"], s["row_end"], ct, pt)
        rc, rp, _ = ref.features(s["depth"], s["col"], s["n"], s["row_start"], s["row_end"], ct, pt)
        assert np.array_equal(gc, rc) and np.array_equal(gp, rp), (ct, pt)
        assert np.array_equal(gc, oc) and np.array_equal(gp, op), (ct, pt)


@pytest.mark.parametrize("s", VOXEL, ids=[s["name"] for s in VOXEL])
def test_voxel_edges(s):
    from funny_lidar_slam_b200.registration import voxel_grid
    g = voxel_grid(s["pts"], s["leaf"])
    assert same_bits(g, ref.voxel_grid(s["pts"], s["leaf"])[0])
    assert same_bits(g, orc.voxel_grid(s["pts"], s["leaf"]))


@pytest.mark.parametrize("s", PROJECT, ids=[s["name"] for s in PROJECT])
def test_preprocess_loam_edges(s):
    """The composed chain (fls_preprocess_loam): projection with de-skew, features, and both voxel filters, against the oracle's
    chain and the reference's."""
    from funny_lidar_slam_b200.features import preprocess_loam
    ct, pt, cl, pl = 0.5, 0.05, 0.3, 0.5
    gc, gp = preprocess_loam(s["raw"], s["ring"], s["time"], s["imu"], s["H"], s["V"], s["h_res"], s["min_d"], s["max_d"], ct, pt, cl, pl)
    o = orc.project_imu(s["raw"], s["ring"], s["time"], s["imu"], s["V"], s["H"], s["h_res"], s["min_d"], s["max_d"])
    oc, op, _ = orc.extract_features(o["depth"], o["col"], o["n"], o["row_start"], o["row_end"], ct, pt)
    assert same_bits(gc, orc.voxel_grid(o["ordered"][oc], cl)) and same_bits(gp, orc.voxel_grid(o["ordered"][op], pl))
    r = ref.project(s["raw"], s["ring"], s["time"], s["imu"], s["V"], s["H"], s["h_res"], s["min_d"], s["max_d"])
    rc, rp, _ = ref.features(r["depth"], r["col"], r["n"], r["row_start"], r["row_end"], ct, pt)
    assert np.array_equal(rc, oc) and np.array_equal(rp, op)
    if r["decided"].all():
        assert same_bits(gc, ref.voxel_grid(r["ordered"][rc], cl)[0]) and same_bits(gp, ref.voxel_grid(r["ordered"][rp], pl)[0])
