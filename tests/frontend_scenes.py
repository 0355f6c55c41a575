"""Small seeded scenes that sit on the edges of the front end (tests/frontend_ref.py restates what they exercise):

* `deskew_scenes`: IMU buffers and point times on every branch of the de-skew and the pre-processing branch — times at t[0],
  t[m-1], an interior stamp and 1 us either side of each; negative times whose product truncates toward zero, not down; a time
  whose product truncates to the last stamp while a float product would round it past; m = 1 and m = 2; ref_time at t[0], at
  t[m-1] (the l = m-2 branch of SetRefTime) and 1 us outside; equal stamps in the middle and at either end (0 / 0 there: NaN
  coordinates, kept out of the planar stage by the jump span); antipodal neighbours (q, -q) with a point and a ref_time at their
  midpoint (a LERP of exactly zero, which Eigen's normalized() leaves as it is) and a point 1 us from the midpoint of samples
  2^39 us apart (near zero norm: undecided); non-unit samples, a rotation of pi,
  an identity extrinsic beside a general one; times of NaN, +-inf and +-9.3e12 s; depths exactly min_d / max_d and one ulp either
  side; jump spans 1, 7 and more than n with the first raw point gated out; n = 0 and n = 1.
* `project_scenes`: a / h_res exactly at k + 0.5 and one ulp either side for even and odd k (y > 0, see `half_column_y`); x < 0 with y = +-0
  (+-pi: the wrap at col >= H); an odd H; rings -1 and V; cells hit many times whose lowest in-range point is outside the IMU
  window (a time past the buffer, or NaN).
* `feature_scenes`: rows on the feature extractor's thresholds (see `_feature_rows`).
* `voxel_scenes`: cell faces at negative coordinates and at +-0; leaves with an inexact inverse where p * inv lands on an integer in
  fp32; a d-product of 2^31 (INT_MAX itself is prime, so d = (INT_MAX, 1, 1) would need (max - min) * inv to truncate to
  2^31 - 2, and every float in [2^30, 2^31) is a multiple of 128: a d-product can never equal INT_MAX); a d-product that fits while
  the divb-product leaves the int range; one cell of 10^5 points with intensity.
"""
from __future__ import annotations

import numpy as np

from tests import frontend_ref as ref

F32 = np.float32
REF = 1_700_000_000_000_000


def _ulps(x, k):
    x = F32(x)
    d = F32(np.inf) if k > 0 else F32(-np.inf)
    for _ in range(abs(int(k))):
        x = np.nextafter(x, d, dtype=F32)
    return x


def rel_for(k: int):
    """A float32 relative time whose product with 1e6 truncates (toward zero) to exactly k microseconds."""
    f = F32(k * 1e-6)
    for _ in range(256):
        tk = ref.x86_i64(float(np.float64(f) * 1.0e6))
        if tk == k:
            return f
        f = np.nextafter(f, F32(np.inf) if tk < k else F32(-np.inf), dtype=F32)
    raise ValueError(k)


def rel_float_trap(lo: int, hi: int):
    """(k, f): f's exact product with 1e6 truncates to k, while the float product F32(f) * 1e6f rounds up to k + 1 or more."""
    for k in range(lo, hi):
        f = rel_for(k + 1)
        while ref.x86_i64(float(np.float64(f) * 1.0e6)) > k:
            f = np.nextafter(f, F32(-np.inf), dtype=F32)
        if ref.x86_i64(float(np.float64(f) * 1.0e6)) == k and float(F32(f * F32(1.0e6))) >= k + 1:
            return k, f
    raise ValueError("no float-product trap in range")


def _quat(axis, ang, scale=1.0):
    a = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    return np.concatenate([a * np.sin(ang / 2), [np.cos(ang / 2)]]) * scale


def _T(general=True):
    T = np.eye(4)
    if general:
        c, s = np.cos(0.4), np.sin(0.4)
        T[:3, :3] = np.array([[c, -s, 0.0], [s * 0.8, c * 0.8, 0.6], [-s * 0.6, -c * 0.6, 0.8]])
        T[:3, 3] = [0.05, -0.02, 0.1]
    return T


def _imu(dt_us, quats, ref_off=0, general=True):
    t = (REF + np.asarray(dt_us, np.int64)).astype(np.uint64)
    return dict(t_us=t, q_xyzw=np.asarray(quats, np.float64).reshape(-1, 4), ref_time_us=REF + int(ref_off), T_lidar_to_imu=_T(general))


def _raw(times, rng, r=(4.0, 25.0)):
    n = len(times)
    d = rng.normal(0, 1, (n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    raw = np.zeros((n, 5), F32)
    raw[:, :3] = d * rng.uniform(*r, (n, 1))
    raw[:, 3] = rng.uniform(0, 100, n)
    raw[:, 4] = np.asarray(times, F32)
    return raw


def _gate_points(min_d, max_d):
    """(x, 0, 0) points whose fp32 depth is min_d / max_d exactly and one ulp either side."""
    pts = []
    for b in (min_d, max_d):
        for k in (-1, 0, 1):
            x = _ulps(b, k)
            assert ref.depth_f32(x, 0, 0) == x
            pts.append(x)
    return pts


# main buffer: irregular spacing, an interior pair of equal stamps; ref_time at the stamp 0
_STAMPS = [-3000, -1000, 0, 2500, 2500, 6000]
_QUATS = [_quat([0.2, -0.1, 0.97], 0.0), _quat([0.3, 0.9, -0.2], 0.35), _quat([1, 0.2, 0.1], -0.2, 1.0), _quat([0.1, 0.1, 1], 1.1, 2.5),
          _quat([0.5, -0.5, 0.7], 0.9, 0.4), _quat([0.0, 0.0, 1.0], np.pi)]


def _main_times():
    k_trap, f_trap = rel_float_trap(9000, 30000)
    stamps = _STAMPS + [k_trap]
    times = []
    for s in stamps:
        times += [rel_for(s - 1), rel_for(s), rel_for(s + 1)]
    times += [F32(-0.0010005), F32(-0.0030005), F32(-0.0030015), F32(-0.0000005)]  # -1000.5, -3000.5, -3001.5, -0.5 us: toward zero
    times += [f_trap]
    times += [F32(np.nan), F32(np.inf), F32(-np.inf), F32(9.3e12), F32(-9.3e12)]
    rng = np.random.default_rng(3)
    times += list(rng.uniform(-0.0031, k_trap * 1e-6 + 0.0001, 40).astype(F32))
    return stamps, times


def deskew_scenes():
    """List of dicts: name, raw (n,5), imu (or None), min_d, max_d, jump, leaf, and `reaches` (what the scene was built for)."""
    out = []
    stamps, times = _main_times()
    quats = _QUATS + [_quat([0.3, -0.2, 0.9], 0.7)]
    rng = np.random.default_rng(11)
    raw = _raw(times, rng)
    gate = _gate_points(2.0, 60.0)
    graw = _raw([rel_for(100)] * len(gate), rng)
    graw[:, :3] = 0.0
    graw[:, 0] = gate
    raw = np.concatenate([raw, graw])
    out.append(dict(name="stamps", raw=raw, imu=_imu(stamps, quats), min_d=2.0, max_d=60.0, jump=3, leaf=0.5,
                    reaches=("t0", "tlast", "interior", "trunc", "trap", "nan_time", "gate")))
    out.append(dict(name="stamps_identity_T", raw=raw, imu=_imu(stamps, quats, general=False), min_d=2.0, max_d=60.0, jump=1, leaf=0.5,
                    reaches=("t0", "tlast")))
    near = raw.copy()
    near[0, :3] = [0.5, 0.0, 0.0]  # the first raw point is gated out
    out.append(dict(name="ref_first_jump7", raw=near, imu=_imu(stamps, quats, ref_off=stamps[0]), min_d=2.0, max_d=60.0, jump=7, leaf=0.5,
                    reaches=("ref_t0",)))
    out.append(dict(name="ref_last_jump_gt_n", raw=near, imu=_imu(stamps, quats, ref_off=stamps[-1]), min_d=2.0, max_d=60.0, jump=len(near) + 5,
                    leaf=0.5, reaches=("ref_tlast",)))
    for off in (stamps[0] - 1, stamps[-1] + 1):
        out.append(dict(name=f"ref_outside_{off}", raw=raw, imu=_imu(stamps, quats, ref_off=off), min_d=2.0, max_d=60.0, jump=3, leaf=0.5,
                        reaches=("scan_dropped",)))
    out.append(dict(name="m1", raw=raw[:20], imu=_imu([0], quats[:1]), min_d=2.0, max_d=60.0, jump=2, leaf=0.5, reaches=("scan_dropped",)))
    t2 = [rel_for(s) for s in (-501, -500, -499, 0, 700, 1499, 1500, 1501)]
    out.append(dict(name="m2", raw=_raw(t2, rng), imu=_imu([-500, 1500], quats[1:3]), min_d=2.0, max_d=60.0, jump=2, leaf=0.5, reaches=("t0", "tlast")))
    # equal stamps at both ends: a point exactly there has ratio 0 / 0 (NaN); those points sit at odd raw indices, jump 2
    te = [rel_for(s) for s in (-200, -1000, 300, -999, 800, 2000, 1999, 1999)]
    out.append(dict(name="dup_ends", raw=_raw(te, rng), imu=_imu([-1000, -1000, 0, 2000, 2000], quats[:5]), min_d=2.0, max_d=60.0, jump=2,
                    leaf=0.5, reaches=("nan_coords",)))
    # antipodal neighbours (q, -q): at the midpoint, 500 us, the LERP sums to exactly zero and Eigen's normalized() leaves it so; the
    # rotation by the zero quaternion q_ref^-1 * 0 returns its input, so that point comes out as float(T p)
    qa = _quat([0.3, 0.4, 0.8], 0.6)
    ta = [rel_for(s) for s in (-1000, 500, -10, 499, 501, 999, 1300, 1700, 2000)] + [F32(0.0004999)]
    anti = _imu([-1000, 0, 1000, 2000], [qa, qa, -qa, _quat([1, 0, 0], 0.2)])
    out.append(dict(name="antipodal", raw=_raw(ta, rng), imu=anti, min_d=2.0, max_d=60.0, jump=2, leaf=0.5, reaches=("lerp_zero",)))
    # ref_time at that midpoint: q_ref is zero, its inverse() is zero, and every point comes out as float(T p)
    out.append(dict(name="antipodal_ref", raw=_raw(ta, rng), imu=dict(anti, ref_time_us=REF + 500), min_d=2.0, max_d=60.0, jump=1, leaf=0.5,
                    reaches=("qri_zero",)))
    # near zero norm: between q and -q stamped 2^39 us apart, a point 1 us short of the midpoint has |q(t)| ~ 2e-12, and the fp64
    # cancellation leaves its direction (and the coordinates) inside their rounding band
    D = 2 ** 39
    f = F32(1.5 * D * 1e-6)
    k = ref.x86_i64(float(np.float64(f) * 1.0e6))
    tn = [f, rel_for(1000), F32(0.25 * D * 1e-6), F32(1.0 * D * 1e-6)]
    near0 = _imu([0, D, D + 2 * (k - D) + 1], [_quat([1, 0, 0], 0.3), qa, -qa])
    out.append(dict(name="near_zero_norm", raw=_raw(tn, rng), imu=near0, min_d=2.0, max_d=60.0, jump=1, leaf=0.5, reaches=("undecided",)))
    out.append(dict(name="n0", raw=np.zeros((0, 5), F32), imu=_imu(stamps, quats), min_d=2.0, max_d=60.0, jump=1, leaf=0.5, reaches=()))
    out.append(dict(name="n1", raw=raw[1:2], imu=_imu(stamps, quats), min_d=2.0, max_d=60.0, jump=1, leaf=0.5, reaches=()))
    out.append(dict(name="no_imu", raw=raw, imu=None, min_d=2.0, max_d=60.0, jump=3, leaf=0.5, reaches=("gate",)))
    return out


# ---- projector ----------------------------------------------------------------------------------------------------------------
def _fast_atan2_first_quadrant(y, x):
    """FastAtan2 of x > 0, y >= 0 on arrays (the branch `half_column_y` searches); each operation rounded to float."""
    p1, p3, p5, p7 = F32(0.9997878412794807), F32(-0.3258083974640975), F32(0.1555786518463281), F32(-0.04432655554792128)
    eps = F32(1.1920928955078125e-07)

    def poly(c):
        c2 = (c * c).astype(F32)
        return ((((((p7 * c2 + p5).astype(F32) * c2).astype(F32) + p3).astype(F32) * c2).astype(F32) + p1).astype(F32) * c).astype(F32)

    ax, ay = np.full_like(y, x), y
    lo = poly((ay / (ax + eps).astype(F32)).astype(F32))
    hi = (F32(1.57079632679489661923) - poly((ax / (ay + eps).astype(F32)).astype(F32))).astype(F32)
    return np.where(ax >= ay, lo, hi)


def half_column_y(x, k, h_res, which=0):
    """A float y > 0 whose a / h_res, with a = FastAtan2(y, x), is exactly k + 0.5 (which = 0) or one float below / above it
    (which = -1 / +1), found among the 2000 fp32 neighbours of tan((k + 0.5) h_res) x; None when none hits it (a / h_res can step
    over a quotient).  Only y > 0: for y < 0 FastAtan2 passes through 2 pi - a and a - 2 pi, whose float grid is much coarser
    than the quotient's, so exact negative half-columns are out of reach."""
    target = _ulps(F32(k + 0.5), which)
    y0 = F32(np.tan((k + 0.5) * float(h_res)) * float(x))
    ys = (np.int64(y0.view(np.int32)) + np.arange(-1000, 1001)).astype(np.int32).view(F32)
    q = (_fast_atan2_first_quadrant(ys, F32(x)) / F32(h_res)).astype(F32)
    hit = np.nonzero(q == target)[0]
    if len(hit) == 0:
        return None
    y = ys[hit[0]]
    assert F32(ref.fast_atan2(y, x) / F32(h_res)) == target
    return y


def half_column_probes(h_res, ks, want):
    """[(k, x, (y below, y at, y above))] for the first `want` of ks where all three exist, trying a few x."""
    out = []
    for k in ks:
        for x in (F32(10.0), F32(7.0), F32(13.25)):
            ys = [half_column_y(x, k, h_res, w) for w in (-1, 0, 1)]
            if all(y is not None for y in ys):
                out.append((k, x, ys))
                break
        if len(out) == want:
            break
    return out


def project_scenes():
    """List of dicts: name, raw (n,4), ring, time, imu, V, H, h_res, min_d, max_d, and the raw indices of the probes."""
    out = []
    rng = np.random.default_rng(21)
    stamps = [-3000, -1000, 0, 2500, 6000]
    imu = _imu(stamps, _QUATS[:5])
    for H in (1800, 1799):
        V = 8
        h_res = F32(2 * np.pi / H)
        pts, ring, time, probes = [], [], [], []
        # k + 0.5 with k even (std::round goes up, rint down) and odd, small and large columns
        found = []
        for sub in (range(8, 200, 2), range(9, 201, 2), range(200, 400, 2), range(201, 401, 2)):
            found += half_column_probes(h_res, sub, want=1)
        assert len(found) == 4
        for k, x, ys in found:
            for which, y in zip((-1, 0, 1), ys):
                probes.append(len(pts))
                pts.append([x, y, 0.5, 1.0])
                ring.append(which + 1)
                time.append(rel_for(100))
        for y in (F32(0.0), F32(-0.0)):  # +-pi: col = H before the wrap (even H)
            probes.append(len(pts))
            pts.append([F32(-7.0), y, 0.25, 2.0])
            ring.append(3 if y == 0 and not np.signbit(y) else 4)
            time.append(rel_for(200))
        for r in (-1, V):  # rings outside [0, V)
            pts.append([5.0, 1.0, 0.0, 3.0])
            ring.append(r)
            time.append(rel_for(0))
        # one cell hit many times: out of range, past the IMU buffer, NaN time, then in-window points (the first of them wins)
        cell_pts = [[0.5, 0.00625, 0.0], [8.0, 0.1, 0.0], [8.0, 0.1, 0.1], [8.0, 0.1, 0.2], [8.0, 0.1, 0.3]]
        cell_times = [rel_for(0), rel_for(6001), F32(np.nan), rel_for(-3000), rel_for(6000)]
        for p, t in zip(cell_pts, cell_times):
            probes.append(len(pts))
            pts.append(p + [4.0])
            ring.append(5)
            time.append(t)
        cell_times2 = [F32(np.inf), rel_for(-3001), rel_for(-1000)]  # a second cell: time +inf and 1 us early before the winner
        for j, t in enumerate(cell_times2):
            probes.append(len(pts))
            pts.append([-3.0, 4.0, 0.1 * j, 5.0])
            ring.append(6)
            time.append(t)
        n_bulk = 3000
        d = rng.normal(0, 1, (n_bulk, 3))
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        bulk = d * rng.uniform(1.0, 70.0, (n_bulk, 1))
        for k in range(n_bulk):
            pts.append([bulk[k, 0], bulk[k, 1], bulk[k, 2], float(k % 97)])
            ring.append(int(rng.integers(-1, V + 1)))
            time.append(F32(rng.uniform(-0.0032, 0.0062)))
        out.append(dict(name=f"H{H}", raw=np.array(pts, F32), ring=np.array(ring, np.int32), time=np.array(time, F32), imu=imu, V=V, H=H, h_res=h_res,
                        min_d=2.0, max_d=60.0, probes=probes))
    return out


# ---- feature extractor --------------------------------------------------------------------------------------------------------
PARABOLA_ROUGH = F32(110.0 / 1024) * F32(110.0 / 1024)  # roughness of every interior point of a parabola row (exact)


def _row_parabola(n, gap=1):
    i = np.arange(n) - n // 2
    return (8.0 + i * i / 1024.0).astype(F32), np.cumsum(np.full(n, gap)).astype(np.int32)


def _row_flat(n):
    return np.full(n, 10.0, F32), np.arange(n, dtype=np.int32)


def _row_random(n, rng, gaps=(1, 1, 1, 2, 12)):
    d = 8.0 + 3.0 * np.sin(np.arange(n) / rng.uniform(6, 30)) + rng.normal(0, 0.03, n)
    for _ in range(max(1, n // 80)):
        k = int(rng.integers(0, n))
        d[k:] += rng.choice([-1.0, 1.0]) * rng.uniform(0.35, 1.5)
    return np.abs(d).astype(F32) + F32(2.0), np.cumsum(rng.choice(gaps, n)).astype(np.int32)


def _row_step(n, hi, lo, at, gap_at=1):
    """A depth step hi -> lo between positions at and at + 1, with the column gap gap_at there."""
    d = np.where(np.arange(n) <= at, hi, lo).astype(F32)
    step = np.ones(n, np.int32)
    step[at + 1] = gap_at
    return d, np.cumsum(step).astype(np.int32)


def _row_parallel(n, at, above: bool):
    """Point `at` (depth 10) whose left neighbour differs by the float difference just above (or at / below) 0.02 * 10 in double."""
    d = np.full(n, 10.0, F32)
    d[at + 1:] = 10.5
    lim = 0.02 * 10.0
    best = None
    for k in range(-40, 41):
        c = _ulps(F32(10.0 - lim), k)
        diff = float(abs(F32(c - F32(10.0))))
        if (diff > lim) == above and (best is None or abs(diff - lim) < abs(best[1] - lim)):
            best = (c, diff)
    d[:at] = best[0]
    return d, np.arange(n, dtype=np.int32)


def _row_ramp(n):
    i = np.arange(n, dtype=np.float64)
    return (8.0 + i ** 3 / 2.0 ** 23).astype(F32), np.arange(n, dtype=np.int32)


def _assemble(rows):
    depth, col, rs, re = [], [], [], []
    off = 0
    for d, c in rows:
        rs.append(off + 5)
        re.append(off + len(d) - 6)
        depth.append(d)
        col.append(c)
        off += len(d)
    return (np.concatenate(depth).astype(F32), np.concatenate(col).astype(np.int32), np.array(rs, np.int32), np.array(re, np.int32))


def _feature_rows():
    rng = np.random.default_rng(5)
    hi3 = F32(0.75) + F32(2.0 ** -24)
    d03 = F32(hi3 + F32(0.3))  # hi3 + 0.3f is a float: the difference is exactly 0.3f
    assert F32(d03 - hi3) == F32(0.3)
    below = np.nextafter(F32(0.3), F32(0), dtype=F32)
    lo3 = F32(0.375) + F32(2.0 ** -25)
    d03b = F32(lo3 + below)  # a float too: the difference is exactly the float below 0.3f
    assert F32(d03b - lo3) == below
    return {
        "ties": [_row_flat(40), _row_parabola(60), (np.zeros(0, F32), np.zeros(0, np.int32)), _row_parabola(61, gap=12), _row_flat(17)],
        "occlusion": [_row_step(30, d03, hi3, 12), _row_step(30, hi3, d03, 12), _row_step(30, d03b, lo3, 14), _row_step(30, lo3, d03b, 14),
                      _row_step(30, 9.0, 8.4, 12, 9), _row_step(30, 9.0, 8.4, 12, 10), _row_step(30, 9.0, 8.4, 12, 11),
                      _row_step(30, 8.4, 9.0, 15, 10), _row_random(90, rng, gaps=(1, 9, 10, 11))],
        "parallel": [_row_parallel(24, 12, True), _row_parallel(24, 12, False), _row_random(40, rng)],
        "short": [_row_random(k, rng) for k in range(11, 19)] + [(np.zeros(0, F32), np.zeros(0, np.int32))] + [_row_random(k, rng) for k in (25, 26, 30, 31)],
        "corners21": [_row_parabola(161, gap=12), _row_random(200, rng, gaps=(12,)), _row_random(130, rng, gaps=(11, 12))],
        "ramp": [_row_ramp(700), _row_random(50, rng)],
        "block512": [_row_random(6 * 512 + 11, rng), _row_random(300, rng)],
        "block513": [_row_random(6 * 513 + 11, rng), _row_random(300, rng)],
    }


def feature_scenes():
    """List of dicts: name, depth, col, n, row_start, row_end, and the (corner_thr, planar_thr) pairs to run."""
    out = []
    for name, rows in _feature_rows().items():
        depth, col, rs, re = _assemble(rows)
        cfgs = [(1.0, 0.1), (0.0005, 0.05)]
        if name in ("ties", "corners21"):
            cfgs += [(float(PARABOLA_ROUGH), 0.1), (0.001, float(PARABOLA_ROUGH)), (-1.0, 0.0)]
        if name == "ramp":
            cfgs += [(1e-6, 1.0)]
        if name in ("short", "occlusion", "parallel"):
            # thresholds equal to a roughness that occurs in the scene
            r = ref.features(depth, col, len(depth), rs, re, 1.0, 0.1)[2]["rough"]
            nz = np.unique(r[r > 0])
            cfgs += [(float(nz[len(nz) // 2]), float(nz[len(nz) // 3]))]
        out.append(dict(name=name, depth=depth, col=col, n=len(depth), row_start=rs, row_end=re, cfgs=cfgs))
    return out


# ---- voxel filter -------------------------------------------------------------------------------------------------------------
def _on_integer(leaf, k):
    """A float p with p * inv (fp32) exactly the integer k although p / leaf is not k."""
    inv = F32(F32(1.0) / F32(leaf))
    p0 = F32(k * float(leaf))
    for j in range(-64, 65):
        p = _ulps(p0, j)
        if F32(p * inv) == F32(k) and float(p) / float(F32(leaf)) != k:
            return p
    return None


def voxel_scenes():
    """List of dicts: name, pts (n,4), leaf, and what the scene was built for."""
    rng = np.random.default_rng(31)
    out = []
    faces = [[x, y, z] for x in (-1.5, -1.0, -0.5, -0.0, 0.0, 0.5) for y in (-2.0, 0.0, -0.0) for z in (-0.5, 1.0)]
    pts = np.array([f + [float(i)] for i, f in enumerate(faces)], F32)
    pts = np.concatenate([pts, np.c_[rng.uniform(-2, 1, (60, 3)), rng.uniform(0, 50, 60)].astype(F32)])
    out.append(dict(name="faces", pts=pts, leaf=0.5, reaches="faces"))
    for leaf in (0.1, 0.2, 0.3, 0.4):
        ps = []
        for k in range(-40, 41):
            p = _on_integer(leaf, k)
            if p is not None:
                ps.append([p, F32(-p), F32(0.5 * p), F32(k)])
        ps = np.array(ps, F32)
        assert len(ps) >= 4, leaf
        ps = np.concatenate([ps, np.c_[rng.uniform(-4, 4, (40, 3)), rng.uniform(0, 9, 40)].astype(F32)])
        out.append(dict(name=f"inexact_{leaf}", pts=ps, leaf=leaf, reaches="on_integer"))
    big = np.array([[0.0, 0.0, 0.0, 1.0], [2047.5, 1023.5, 1023.5, 2.0], [3.2, 7.1, 9.9, 3.0], [3.4, 7.2, 9.8, 4.0]], F32)
    out.append(dict(name="d_product_2^31", pts=big, leaf=1.0, reaches="overflow"))
    wrap = np.array([[0.5, 0.5, 0.5, 1.0], [1290.2, 1290.2, 1290.2, 2.0], [1289.9, 1289.7, 1290.1, 3.0], [1290.1, 1289.95, 1290.15, 5.0],
                     [700.3, 1200.6, 1100.2, 7.0], [700.7, 1200.1, 1100.9, 11.0], [3.3, 2.2, 1288.4, 13.0], [0.7, 0.9, 0.6, 17.0]], F32)
    out.append(dict(name="divb_wraps", pts=wrap, leaf=1.0, reaches="wrapped"))
    one = np.c_[rng.uniform(0.01, 0.49, (100000, 3)), rng.uniform(0, 255, 100000)].astype(F32)
    one = np.concatenate([one, np.array([[3.2, 0.1, 0.1, 9.0]], F32)])
    out.append(dict(name="one_cell_1e5", pts=one, leaf=0.5, reaches="order"))
    return out
