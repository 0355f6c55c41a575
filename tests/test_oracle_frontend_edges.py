"""The front-end references (tests/frontend_ref.py) against the oracle on the edge scenes of tests/frontend_scenes.py (CPU): bit for
bit wherever the reference says the result is decided, and each scene shown to reach the branch it was built for."""
import numpy as np
import pytest

from oracle import pyoracle as orc
from tests import frontend_ref as ref
from tests import frontend_scenes as fs

DESKEW = fs.deskew_scenes()
PROJECT = fs.project_scenes()
FEATURES = fs.feature_scenes()
VOXEL = fs.voxel_scenes()


def same_bits(a, b):
    """Equal shapes, NaN in the same places, every other value bit for bit (NaN payloads differ between x86 and the GPU)."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return bool(np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32)))


def check_ordered(got, want, decided):
    """got == the reference's floats on every decided coordinate, intensities exact."""
    assert got.shape == want.shape
    for c in range(3):
        m = decided[:, c]
        assert same_bits(got[m, c], want[m, c]), c
    assert same_bits(got[:, 3], want[:, 3])


def _reaches(s, r):
    imu, raw = s["imu"], s["raw"]
    times = [ref.point_time(imu["ref_time_us"], t) for t in raw[:, 4]] if imu is not None else []
    kept = set(int(i) for i in r["raw_index"])
    ts = [int(t) for t in imu["t_us"]] if imu is not None else []
    for tag in s["reaches"]:
        if tag == "t0":
            assert any(times[i] == ts[0] for i in kept) and any(times[i] == ts[0] - 1 for i in r["dropped_by_time"])
        elif tag == "tlast":
            assert any(times[i] == ts[-1] for i in kept) and any(times[i] == ts[-1] + 1 for i in r["dropped_by_time"])
        elif tag == "interior":
            assert any(times[i] == ts[3] for i in kept)  # the first of the two equal interior stamps
        elif tag == "trunc":  # -3000.5 us truncates to t[0] (kept), -3001.5 us to t[0] - 1 (dropped)
            k0 = [i for i in range(len(raw)) if raw[i, 4] == np.float32(-0.0030005)][0]
            k1 = [i for i in range(len(raw)) if raw[i, 4] == np.float32(-0.0030015)][0]
            assert times[k0] == ts[0] and k0 in kept and k1 in r["dropped_by_time"]
        elif tag == "trap":  # truncates to the last stamp; a float product would step past it
            k, f = fs.rel_float_trap(9000, 30000)
            i = [j for j in range(len(raw)) if raw[j, 4] == f][0]
            assert times[i] == ts[-1] and i in kept and float(np.float32(f * np.float32(1e6))) >= k + 1
        elif tag == "nan_time":
            for bad in (np.nan, np.inf, -np.inf, 9.3e12, -9.3e12):
                i = [j for j in range(len(raw)) if (np.isnan(raw[j, 4]) if np.isnan(bad) else raw[j, 4] == np.float32(bad))][0]
                assert i in r["dropped_by_time"], bad
            assert ref.point_time(imu["ref_time_us"], np.nan) == (imu["ref_time_us"] - 2 ** 63) % 2 ** 64
        elif tag == "gate":
            g = [i for i in range(len(raw)) if raw[i, 1] == 0 and raw[i, 2] == 0]
            assert [i in kept or i in r["dropped_by_time"] for i in g] == [False, True, True, True, True, False]
        elif tag in ("ref_t0", "ref_tlast"):
            assert imu["ref_time_us"] == (ts[0] if tag == "ref_t0" else ts[-1]) and len(kept) > 0
        elif tag == "scan_dropped":
            assert r["scan_dropped"]
        elif tag == "lerp_zero":  # q(t) = 0 stays unnormalised: the point is float(T p), finite and decided
            assert len(r["lerp_zero"]) == 1
            j = list(r["raw_index"]).index(r["lerp_zero"][0])
            T, p = np.asarray(imu["T_lidar_to_imu"], np.float64), raw[r["lerp_zero"][0]]
            Tp = [ref.round_f32(sum(ref.mpf(float(T[a, b])) * ref.mpf(float(p[b])) for b in range(3)) + ref.mpf(float(T[a, 3])))[0] for a in range(3)]
            assert r["decided"][j].all() and same_bits(r["ordered"][j, :3], Tp)
        elif tag == "qri_zero":
            qri, dec = ref.ref_inverse(imu)
            assert dec and all(c.v == 0 and c.e == 0 for c in qri) and len(kept) > 0 and np.isfinite(r["ordered"]).all()
        elif tag == "nan_coords":
            assert np.isnan(r["ordered"][:, :3]).any() and not np.isnan(r["planar_in"]).any()


@pytest.mark.parametrize("s", DESKEW, ids=[s["name"] for s in DESKEW])
def test_preprocess_reference_equals_oracle(s):
    r = ref.preprocess(s["raw"], s["imu"], s["min_d"], s["max_d"], s["jump"], s["leaf"])
    o_ord, o_pl = orc.preprocess(s["raw"], s["imu"], s["min_d"], s["max_d"], s["jump"], s["leaf"])
    check_ordered(o_ord, r["ordered"], r["decided"])
    if "undecided" in s["reaches"]:  # the LERP near zero norm: its fp64 error bound covers float midpoints (reported, not asserted)
        assert not r["decided"].all()
    elif len(r["decided"]):
        assert r["decided"].mean() > 0.9
    # the planar stage of the oracle is its voxel filter of its own candidates; the reference filter agrees on them
    cand = np.array([i % s["jump"] == 0 for i in r["raw_index"]], bool)
    assert same_bits(o_pl, ref.voxel_grid(o_ord[cand], s["leaf"])[0])
    if r["decided"].all():
        assert same_bits(o_pl, r["planar"])
    _reaches(s, r)


def test_nan_and_huge_point_times_follow_the_x86_conversion():
    """int64_t(rel_time * 1e6) of NaN, +-inf and |t| >= 9.3e12 s is INT64_MIN on x86-64: the point is outside any buffer."""
    for v in (np.nan, np.inf, -np.inf, 9.3e12, -9.3e12):
        assert ref.x86_i64(float(np.float64(np.float32(v)) * 1e6)) == ref.INT64_MIN
    assert ref.x86_i64(-1.5) == -1 and ref.x86_i64(2.9) == 2  # toward zero
    s = DESKEW[0]
    raw = s["raw"][np.isnan(s["raw"][:, 4])]
    assert len(raw) == 1 and len(orc.preprocess(raw, s["imu"], 0.0, 1e9, 1, 0.5)[0]) == 0


def test_descending_stamps_oracle_keeps_the_downward_scan():
    """Upstream (and the oracle) scan down from the end: on a buffer that is not ascending it picks the last sample not later than
    t found from the end.  The reference restates that scan; the device rejects such a buffer."""
    imu = fs._imu([-2000, 1000, -500, 3000], fs._QUATS[:4])
    raw = fs._raw([fs.rel_for(k) for k in (-1500, -600, 0, 900, 1200, 2500)], np.random.default_rng(4))
    r = ref.preprocess(raw, imu, 0.5, 100.0, 1, 0.5)
    o_ord, _ = orc.preprocess(raw, imu, 0.5, 100.0, 1, 0.5)
    check_ordered(o_ord, r["ordered"], r["decided"])
    assert ref.search_two(imu["t_us"], int(imu["ref_time_us"]) + 500) == (2, 3)  # bisection would take (0, 1)


@pytest.mark.parametrize("s", PROJECT, ids=[s["name"] for s in PROJECT])
def test_project_reference_equals_oracle(s):
    r = ref.project(s["raw"], s["ring"], s["time"], s["imu"], s["V"], s["H"], s["h_res"], s["min_d"], s["max_d"])
    o = orc.project_imu(s["raw"], s["ring"], s["time"], s["imu"], s["V"], s["H"], s["h_res"], s["min_d"], s["max_d"])
    assert o["n"] == r["n"] > 1000
    for k in ("depth", "col", "row_start", "row_end"):
        assert np.array_equal(o[k], r[k]), k
    check_ordered(o["ordered"], r["ordered"], r["decided"])
    # the half-column probes: exactly k + 0.5 (margin 0) and one float either side, with k even and odd
    pr = s["probes"]
    qs = [float(ref.column(s["raw"][k, 0], s["raw"][k, 1], s["H"], s["h_res"])[1]) for k in pr[:12]]
    at = qs[1::3]
    assert all(q % 1 == 0.5 for q in at) and {int(q) % 2 for q in at} == {0, 1}
    assert all(r["margin"][k] == 0 for k in pr[1:12:3])
    # +-pi: col = H before the wrap for an even H
    k_pi = pr[12]
    col_before = ref.round_half_away(ref.fast_atan2(s["raw"][k_pi, 1], s["raw"][k_pi, 0]) / np.float32(s["h_res"])) + s["H"] // 2
    assert col_before == s["H"] or s["H"] % 2 == 1
    # the cell hit five times: out of range, past the buffer, NaN time, then the first in-window point wins
    cell = pr[14:19]
    assert len({ref.column(s["raw"][k, 0], s["raw"][k, 1], s["H"], s["h_res"])[0] for k in cell}) == 1 and len(set(s["ring"][cell])) == 1
    assert cell[3] in r["winner"] and not set(cell[:3]) & set(r["winner"]) and cell[4] not in r["winner"]
    assert pr[21] in r["winner"] and pr[19] not in r["winner"]
    assert not set(np.nonzero((s["ring"] < 0) | (s["ring"] >= s["V"]))[0]) & set(r["winner"])


@pytest.mark.parametrize("s", FEATURES, ids=[s["name"] for s in FEATURES])
def test_features_reference_equals_oracle(s):
    for ct, pt in s["cfgs"]:
        oc, op, _ = orc.extract_features(s["depth"], s["col"], s["n"], s["row_start"], s["row_end"], ct, pt)
        rc, rp, mg = ref.features(s["depth"], s["col"], s["n"], s["row_start"], s["row_end"], ct, pt)
        assert np.array_equal(oc, rc) and np.array_equal(op, rp), (ct, pt)
    rough = mg["rough"]
    name = s["name"]
    if name == "ties":
        assert np.sum(rough == 0) > 40 and np.sum(rough == fs.PARABOLA_ROUGH) > 40
        _, _, m2 = ref.features(s["depth"], s["col"], s["n"], s["row_start"], s["row_end"], float(fs.PARABOLA_ROUGH), float(fs.PARABOLA_ROUGH))
        assert (m2["corner"] == 0).any() and (m2["planar"] == 0).any()
    elif name == "occlusion":
        below = float(np.nextafter(np.float32(0.3), np.float32(0), dtype=np.float32))
        assert (mg["occlusion"] == float(np.float32(0.3)) - 0.3).any() and (mg["occlusion"] == below - 0.3).any()
        assert {-1, 0, 1} <= set(mg["col_occ"].astype(int).tolist())
        assert {0, 1} <= set(mg["col_sup"].astype(int).tolist())
    elif name == "parallel":
        assert np.sort(np.abs(mg["parallel"]))[0] < 1e-6
    elif name == "short":
        lens = s["row_end"] - s["row_start"]
        assert {-11, 0, 7} <= set(lens.tolist()) and (lens % 6 != 0).any()
    elif name == "corners21":  # blocks with more than 20 candidates: block_end picked on its first visit, the 21st ends the pass
        _, _, m = ref.features(s["depth"], s["col"], s["n"], s["row_start"], s["row_end"], 0.0005, 0.05)
        assert len(m["be_picked"]) > 0 and len(m["brk"]) > 0
    elif name.startswith("block"):
        assert max((s["row_end"] - s["row_start"]) // 6) == int(name[5:])
    elif name == "ramp":
        assert (s["row_end"][0] - s["row_start"][0]) // 6 > 96 and np.mean(np.diff(rough[6:690]) >= 0) > 0.95


@pytest.mark.parametrize("s", VOXEL, ids=[s["name"] for s in VOXEL])
def test_voxel_reference_equals_oracle(s):
    want, info = ref.voxel_grid(s["pts"], s["leaf"])
    assert same_bits(orc.voxel_grid(s["pts"], s["leaf"]), want)
    if s["reaches"] == "overflow":
        assert info["overflow"] and np.prod(info["d"]) == 2 ** 31
    elif s["reaches"] == "wrapped":
        assert not info["overflow"] and np.prod(info["d"]) <= 2 ** 31 - 1 < np.prod(info["divb"]) and info["wrapped"]
        assert len(want) == 6  # two pairs of the eight points share a cell
    elif s["reaches"] == "faces":
        assert (s["pts"][:, :3] == 0).any() and np.signbit(s["pts"][:, :3][s["pts"][:, :3] == 0]).any()
    elif s["reaches"] == "on_integer":
        inv = np.float32(np.float32(1) / np.float32(s["leaf"]))
        assert np.any((s["pts"][:, 0] * inv) % 1 == 0)
    elif s["reaches"] == "order":
        assert len(want) == 2
