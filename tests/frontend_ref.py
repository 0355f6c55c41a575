"""Independent references of the front end — the stages every frame passes before a matcher runs (CPU only; shares nothing with
oracle/ or the CUDA library):

* `deskew_point` / `ref_inverse`: LidarDistortionCorrector::SetRefTime / ProcessPoint (src/lidar/lidar_distortion_corrector.cpp:19-64
  upstream) in 50-digit arithmetic (mpmath): DataSearcher::SearchNearestTwoData with its downward scan (include/common/data_searcher.h:
  100-134), the ratio, MotionInterpolator::InterpolateQuaternionLerp (no hemisphere alignment, then normalise; motion_interpolator.h:
  27-35), SetRefTime's inverse, q_ref^-1 * q(t), the lidar -> imu extrinsic and the rotation.  The point time is
  ref_time + int64_t(rel_time * 1.0e6); the product of a float and 1e6 (= 2^6 * 15625) has at most 24 + 14 significant bits, so
  it is exact in fp64, and the conversion follows x86-64's cvttsd2si: toward zero, INT64_MIN for NaN and out-of-range values.
  A buffer of fewer than two samples finds no pair (upstream would read past its deque).
* `preprocess`: PreProcessing::Run's branch without features (src/slam/preprocessing.cpp:181-225): range gate (inclusive at both
  ends, fp32 depth), de-skew, ordered cloud, planar candidates by the RAW index modulo the jump span, then `voxel_grid`.
* `project`: PointcloudProjector::Project (src/loam/pointcloud_projector.cpp:32-133): FastAtan2 (math_function.h:159-186) op by op
  in np.float32, col = round(a / h_res) + H / 2 with std::round's half-away-from-zero and the wrap, first hit wins, a point whose
  time is outside the IMU buffer does not claim its cell (:100-103), row_start / row_end (:115, :131).  Every column decision
  reports how far a / h_res lies from its half-column boundary, in fp32 ulps.
* `features`: FeatureExtractor::{SelectValidPoints, ComputeRoughness, SelectFeatures} (src/loam/feature_extractor.cpp:46-222),
  loop for loop, with position as the explicit tie-break of the roughness sort, and the margin of every decision.
* `voxel_grid`: pcl::VoxelGrid (PCL 1.10) as VoxelGridCloud wraps it (include/common/pointcloud_utility.h:216-224,263-271).

De-skew rounding.  Each output coordinate comes with its exact value, the float nearest to it, and whether that float is
*decided*: the fp64 evaluation the device and the oracle perform (one rounding per operation, in the order of fls_deskew.cuh)
is within a bound `err` of the exact value, and the rounding to float is decided when the exact value lies farther than `err`
from every float midpoint (or err = 0).  Then the fp64 result rounds to the same float, so "device float == this float" is a
bit-level check that does not depend on the oracle.  `err` is a running bound carried through the same operations: an input
held exactly has err 0, an operation on exact inputs whose exact result is a double does not round (err stays 0), and
otherwise, with u = 2^-53 and |fl(x) - x| <= u |x| for every rounding (no underflow on these magnitudes),
    a +- b : ea + eb                          + u (|a +- b| + ea + eb)
    a * b  : |a| eb + |b| ea + ea eb          + u (|ab| + ...)
    a / b  : (ea + |a / b| eb) / (|b| - eb)   + u (|a / b| + ...)   (none when |b| <= eb)
    sqrt a : min(ea / sqrt(a), sqrt(ea))      + u (sqrt(a) + ...)
— the first term bounds what the inputs' errors do to the exact result, the second the rounding of the computed value, whose
magnitude is at most the exact one plus the propagated error.  For a point at 10 m this comes to about 1e-13 m against a float
spacing of about 1e-6 m, so nearly every coordinate is decided; a LERP that passes near zero norm is where it is not.
Eigen 3.3.7's guards are restated: q.normalized() leaves a quaternion whose squared norm is not > 0 unchanged, and inverse()
of one is zero — so a LERP that sums to exactly zero (q and -q at ratio 0.5) gives q(t) = 0, and the rotation by a zero
quaternion returns its input: the point comes out as float(T p).  Where the fp64 guard itself is within rounding of zero the
point is reported undecided.  A 0 / 0 ratio (equal stamps at the end of the buffer, the point exactly there) makes the
coordinates NaN here and on the device; upstream's CHECK in InterpolateQuaternionLerp ends the process there instead.
"""
from __future__ import annotations

import math

import mpmath
import numpy as np

mpmath.mp.dps = 50
mpf = mpmath.mpf
F32 = np.float32
U = mpf(2) ** -53
INT64_MIN = -(2 ** 63)
FMAX = float(np.finfo(np.float32).max)


# ---- time ---------------------------------------------------------------------------------------------------------------------
def x86_i64(v: float) -> int:
    """static_cast<int64_t>(double) as x86-64 computes it: toward zero; NaN and values outside [-2^63, 2^63) give INT64_MIN."""
    if not (-9.2233720368547758e18 <= v < 9.2233720368547758e18):
        return INT64_MIN
    return int(v)


def point_time(ref_time: int, rel_time) -> int:
    """ProcessPoint's uint64 time stamp of a point (:41): the int64 sum in unsigned arithmetic."""
    prod = float(np.float64(F32(rel_time)) * 1.0e6)  # exact (see the module docstring)
    return (int(ref_time) + x86_i64(prod)) % 2 ** 64


def search_two(ts, t: int):
    """SearchNearestTwoData (data_searcher.h:100-134): (l, r) or None."""
    m = len(ts)
    if m == 0 or int(ts[0]) > t or int(ts[-1]) < t or m < 2:
        return None
    if int(ts[0]) == t:
        return 0, 1
    if int(ts[-1]) == t:
        return m - 2, m - 1
    i = m - 1
    while t < int(ts[i]):
        i -= 1
    return i, i + 1


# ---- exact values with a running bound on the fp64 evaluation -------------------------------------------------------------------
class R:
    """Exact value `v` of an fp64 expression and a bound `e` on |fp64 evaluation - v| (the module docstring)."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=0):
        self.v = mpf(v)
        self.e = mpf(e)

    def _r(self, v, e):
        if e == 0 and mpf(float(v)) == v:  # exact inputs and a result that is a double: the operation does not round
            return R(v, 0)
        return R(v, e + U * (abs(v) + e))

    def __add__(self, o):
        return self._r(self.v + o.v, self.e + o.e)

    def __sub__(self, o):
        return self._r(self.v - o.v, self.e + o.e)

    def __mul__(self, o):
        return self._r(self.v * o.v, abs(self.v) * o.e + abs(o.v) * self.e + self.e * o.e)

    def __truediv__(self, o):
        if abs(o.v) <= o.e:
            return R(mpmath.nan, mpmath.inf)
        q = self.v / o.v
        return self._r(q, (self.e + abs(q) * o.e) / (abs(o.v) - o.e))

    def __neg__(self):
        return R(-self.v, self.e)

    def sqrt(self):
        if self.v < 0:
            return R(mpmath.nan, mpmath.inf)
        s = mpmath.sqrt(self.v)
        prop = mpmath.sqrt(self.e) if s == 0 else min(self.e / s, mpmath.sqrt(self.e))
        return self._r(s, prop)


def _ex(x) -> R:
    return R(mpf(float(x)))


def _f32_next(f, d):
    return np.nextafter(F32(f), F32(d * np.inf), dtype=F32)


def round_f32(v) -> tuple:
    """(nearest float32 to the exact v, ties to even; distance from v to the nearest float midpoint)."""
    if mpmath.isnan(v):
        return F32(np.nan), mpmath.inf
    f = F32(float(v))
    best = min((f, _f32_next(f, -1), _f32_next(f, 1)), key=lambda c: (abs(mpf(float(c)) - v), int(c.view(np.uint32)) & 1))
    lo, hi = _f32_next(best, -1), _f32_next(best, 1)
    mid_lo = (mpf(float(best)) + mpf(float(lo))) / 2
    mid_hi = (mpf(float(best)) + mpf(float(hi))) / 2
    return F32(best), min(abs(v - mid_lo), abs(mid_hi - v))


# ---- de-skew ------------------------------------------------------------------------------------------------------------------
def _positive(x: R):
    """Eigen's `squaredNorm() > 0` guard on an fp64 value within x.e of x.v: True / False when decided, None when the bound straddles
    zero (the fp64 comparison could go either way)."""
    if x.v > x.e:
        return True
    if x.v == 0 and x.e == 0:
        return False
    return None


def _lerp(qa, qb, s: R, one=R(1)):
    """InterpolateQuaternionLerp: (q, decided).  q.normalized() in Eigen 3.3.7 returns the coefficients unchanged unless the
    squared norm is > 0 (between q and -q at ratio 0.5 the sum is exactly zero)."""
    u = one - s
    q = [_ex(qa[k]) * u + _ex(qb[k]) * s for k in range(4)]
    sq = ((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3]
    pos = _positive(sq)
    if pos is False:
        return q, True
    n = sq.sqrt()
    return [c / n for c in q], pos is not None


def _ratio(ts, l, r, t):
    num, den = t - int(ts[l]), int(ts[r]) - int(ts[l])
    if den == 0:
        return None  # 0 / 0: NaN
    return R(num) / R(den)  # both integers are exact in fp64 on these buffers (< 2^53)


def ref_inverse(imu):
    """SetRefTime (:19-34): (q_ref^-1 as four R, decided), or None when ref_time is outside the buffer.  Quaternion::inverse() in
    Eigen 3.3.7 returns zero unless the squared norm is > 0; a 0 / 0 ratio makes the LERP NaN, which fails that test too."""
    ts, q = imu["t_us"], np.asarray(imu["q_xyzw"], np.float64)
    lr = search_two(ts, int(imu["ref_time_us"]))
    if lr is None:
        return None
    l, r = lr
    s = _ratio(ts, l, r, int(imu["ref_time_us"]))
    if s is None:
        return [R(0)] * 4, True
    n, dec = _lerp(q[l], q[r], s)
    n2 = ((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2]) + n[3] * n[3]
    pos = _positive(n2)
    if pos is False:
        return [R(0)] * 4, dec
    return [-n[0] / n2, -n[1] / n2, -n[2] / n2, n[3] / n2], dec and pos is not None


def deskew_point(imu, qri, x, y, z, rel_time):
    """ProcessPoint (:37-64); qri is what `ref_inverse` returned.  None when the point's time is outside the buffer; else a dict:
    exact (3 mpf), f (3 float32, the correctly rounded exact values), err (3 bounds on the fp64 evaluation), decided (3 bools),
    l (the interval's left sample), t, lerp_zero (q(t) is exactly zero and stays unnormalised).
    A 0 / 0 ratio (equal stamps at the end of the buffer, the point exactly there) makes the coordinates NaN; upstream's
    CHECK_GE(t, 0.0) in InterpolateQuaternionLerp fails on that NaN and ends the process, which is not restated."""
    ts, q = imu["t_us"], np.asarray(imu["q_xyzw"], np.float64)
    t = point_time(imu["ref_time_us"], rel_time)
    lr = search_two(ts, t)
    if lr is None:
        return None
    l, r = lr
    s = _ratio(ts, l, r, t)
    if s is None:
        nan = F32(np.nan)
        return dict(exact=[mpmath.nan] * 3, f=[nan] * 3, err=[mpf(0)] * 3, decided=[True] * 3, l=l, t=t, lerp_zero=False)
    qc, dec_c = _lerp(q[l], q[r], s)
    qri, dec_r = qri
    ax, ay, az, aw = qri
    qx, qy, qz, qw = qc
    px = ((aw * qx + ax * qw) + ay * qz) - az * qy
    py = ((aw * qy + ay * qw) + az * qx) - ax * qz
    pz = ((aw * qz + az * qw) + ax * qy) - ay * qx
    pw = ((aw * qw - ax * qx) - ay * qy) - az * qz
    T = np.asarray(imu["T_lidar_to_imu"], np.float64)
    p = [_ex(F32(x)), _ex(F32(y)), _ex(F32(z))]
    v = [((_ex(T[a, 0]) * p[0] + _ex(T[a, 1]) * p[1]) + _ex(T[a, 2]) * p[2]) + _ex(T[a, 3]) for a in range(3)]
    ux, uy, uz = py * v[2] - pz * v[1], pz * v[0] - px * v[2], px * v[1] - py * v[0]
    ux, uy, uz = ux + ux, uy + uy, uz + uz
    o = [(v[0] + pw * ux) + (py * uz - pz * uy), (v[1] + pw * uy) + (pz * ux - px * uz), (v[2] + pw * uz) + (px * uy - py * ux)]
    out = dict(exact=[c.v for c in o], err=[c.e for c in o], f=[], decided=[], l=l, t=t, lerp_zero=all(c.v == 0 and c.e == 0 for c in qc))
    for c in o:
        f, dist = round_f32(c.v)
        out["f"].append(f)
        out["decided"].append(bool(dec_c and dec_r and (c.e == 0 or dist > c.e)))
    return out


# ---- pre-processing -----------------------------------------------------------------------------------------------------------
def depth_f32(x, y, z):
    """sqrt((x*x + y*y) + z*z) in float, each operation rounded (upstream's float expression, no contraction)."""
    x, y, z = F32(x), F32(y), F32(z)
    return F32(np.sqrt(F32(F32(F32(x * x) + F32(y * y)) + F32(z * z))))


def preprocess(raw, imu, min_d, max_d, jump_span, leaf):
    """preprocessing.cpp:181-225.  Returns dict: ordered (n,4) float32, decided (n,3) bool (all True without an IMU buffer),
    raw_index (n,) of every ordered point, planar_in (the jump-span candidates, in order), planar (after voxel_grid),
    dropped_by_time (raw indices inside the range gate whose time is outside the buffer), lerp_zero (raw indices whose q(t) is
    exactly zero), scan_dropped."""
    raw = np.asarray(raw, F32)
    lo, hi = F32(min_d), F32(max_d)
    qri = None
    if imu is not None:
        qri = ref_inverse(imu)
        if qri is None:
            e = np.zeros((0, 4), F32)
            return dict(ordered=e, decided=np.zeros((0, 3), bool), raw_index=np.zeros(0, int), planar_in=e, planar=e, dropped_by_time=[],
                        lerp_zero=[], scan_dropped=True)
    ordered, decided, idx, pl, dropped, zero = [], [], [], [], [], []
    for i, p in enumerate(raw):
        d = depth_f32(p[0], p[1], p[2])
        if d < lo or d > hi:
            continue
        c, dec = [p[0], p[1], p[2]], [True] * 3
        if imu is not None:
            r = deskew_point(imu, qri, p[0], p[1], p[2], p[4])
            if r is None:
                dropped.append(i)
                continue
            c, dec = r["f"], r["decided"]
            if r["lerp_zero"]:
                zero.append(i)
        rec = [c[0], c[1], c[2], p[3]]
        ordered.append(rec)
        decided.append(dec)
        idx.append(i)
        if i % int(jump_span) == 0:
            pl.append(rec)
    ordered = np.array(ordered, F32).reshape(-1, 4)
    planar_in = np.array(pl, F32).reshape(-1, 4)
    planar, _ = voxel_grid(planar_in, leaf)
    return dict(ordered=ordered, decided=np.array(decided, bool).reshape(-1, 3), raw_index=np.array(idx, int), planar_in=planar_in,
                planar=planar, dropped_by_time=dropped, lerp_zero=zero, scan_dropped=False)


# ---- projector ----------------------------------------------------------------------------------------------------------------
def fast_atan2(y, x):
    """FastAtan2<float> (math_function.h:159-186), every operation rounded to float."""
    y, x = F32(y), F32(x)
    p1, p3, p5, p7 = F32(0.9997878412794807), F32(-0.3258083974640975), F32(0.1555786518463281), F32(-0.04432655554792128)
    ax, ay = F32(abs(x)), F32(abs(y))
    eps = F32(1.1920928955078125e-07)

    def poly(c):
        c2 = F32(c * c)
        return F32(F32(F32(F32(F32(F32(F32(p7 * c2) + p5) * c2) + p3) * c2) + p1) * c)

    if ax >= ay:
        a = poly(F32(ay / F32(ax + eps)))
    else:
        a = F32(F32(1.57079632679489661923) - poly(F32(ax / F32(ay + eps))))
    if x < 0:
        a = F32(F32(3.14159265358979323846) - a)
    if y < 0:
        a = F32(F32(6.28318530717958647692) - a)
    if a > F32(3.14159265358979323846):
        a = F32(a - F32(6.28318530717958647692))
    return a


def round_half_away(q) -> int:
    """std::round(float): half away from zero (|q| + 0.5 is exact in fp64 for a float q)."""
    q = float(q)
    return int(math.copysign(math.floor(abs(q) + 0.5), q))


def column(x, y, H, h_res):
    """(col before the wrap check of :81-82, quotient a / h_res, its distance from the nearest half-column boundary in fp32 ulps)."""
    qv = F32(fast_atan2(y, x) / F32(h_res))
    col = round_half_away(qv) + int(H) // 2
    if col >= H:
        col -= H
    b = math.floor(float(qv)) + 0.5
    return col, qv, abs(float(qv) - b) / float(np.spacing(F32(abs(b)) if b != 0 else F32(0.5)))


def project(raw, ring, time, imu, V, H, h_res, min_d, max_d):
    """pointcloud_projector.cpp:32-133 with the de-skew claim rule; the winners de-skewed by `deskew_point`.  Returns the oracle's
    dict layout plus winner (raw index per emitted point), decided (n,3) and margin (raw index -> half-column distance in ulps)."""
    raw = np.asarray(raw, F32)
    lo, hi = F32(min_d), F32(max_d)
    qri = ref_inverse(imu) if imu is not None else None
    owner = {}
    margin = {}
    if imu is None or qri is not None:
        for k, p in enumerate(raw):
            d = depth_f32(p[0], p[1], p[2])
            if d < lo or d > hi:
                continue
            row = int(ring[k])
            col, _, mg = column(p[0], p[1], H, h_res)
            margin[k] = mg
            if row >= V or row < 0 or col < 0 or col >= H:
                continue
            if (row, col) in owner:
                continue
            if imu is not None and search_two(imu["t_us"], point_time(imu["ref_time_us"], time[k])) is None:
                continue  # ProcessPoint fails: the cell stays free for a later point
            owner[(row, col)] = k
    ordered, depth, cols, winner, decided = [], [], [], [], []
    rs, re = np.zeros(V, np.int32), np.zeros(V, np.int32)
    for row in range(V):
        rs[row] = len(ordered) + 5
        for c in range(H):
            k = owner.get((row, c))
            if k is None:
                continue
            p = raw[k]
            rec, dec = [p[0], p[1], p[2], p[3]], [True] * 3
            if imu is not None:
                r = deskew_point(imu, qri, p[0], p[1], p[2], time[k])
                rec[:3], dec = r["f"], r["decided"]
            ordered.append(rec)
            decided.append(dec)
            depth.append(depth_f32(p[0], p[1], p[2]))
            cols.append(c)
            winner.append(k)
        re[row] = len(ordered) - 6
    n = len(ordered)
    dep = np.zeros(V * H, F32)
    col = np.zeros(V * H, np.int32)
    dep[:n], col[:n] = depth, cols
    return dict(ordered=np.array(ordered, F32).reshape(-1, 4), depth=dep, col=col, row_start=rs, row_end=re, n=n, winner=np.array(winner, int),
                decided=np.array(decided, bool).reshape(-1, 3), margin=margin)


# ---- feature extractor --------------------------------------------------------------------------------------------------------
def features(depth, col, n, row_start, row_end, corner_thr, planar_thr):
    """Loop-for-loop restatement of FeatureExtractor::{SelectValidPoints, ComputeRoughness, SelectFeatures}
    (src/loam/feature_extractor.cpp:46-222 upstream): fp32 arithmetic where upstream has float, double comparisons where it
    promotes (`d1 - d2 > 0.3`, `diff > 0.02 * depth`).  Upstream's std::sort is unstable; ties in roughness are broken by position,
    explicitly.  Returns (corner indices, planar indices, margins): margins holds, per decision kind, the signed distance of what
    was compared from its threshold — occlusion (float difference - 0.3 in double, for both directions), parallel (diff - 0.02 *
    depth, both sides), corner / planar (roughness - threshold, in float, for every visit), col_occ (|col gap| - 10 of an occlusion
    test, decision `< 10`), col_sup (|col gap| - 10 of a suppression step, decision `> 10`) — plus be_picked (corners picked on the
    inclusive `block_end` visit), brk (the 21st candidate of a block, where the corner pass stops) and `rough`, the roughness array."""
    f32 = F32
    depth = np.asarray(depth, f32)
    col = np.asarray(col, np.int64)
    mg = dict(occlusion=[], parallel=[], corner=[], planar=[], col_occ=[], col_sup=[], be_picked=[], brk=[])
    valid = np.ones(n + 8, bool)
    corner = np.zeros(n + 8, bool)
    valid[:5] = False
    valid[n - 6:n] = False
    for i in range(5, n - 6):
        d1, d2 = depth[i], depth[i + 1]
        gap = abs(int(col[i + 1]) - int(col[i]))
        mg["col_occ"].append(gap - 10)
        if gap < 10:
            mg["occlusion"] += [float(f32(d1 - d2)) - 0.3, float(f32(d2 - d1)) - 0.3]
            if float(f32(d1 - d2)) > 0.3:
                valid[i - 5:i + 1] = False
            elif float(f32(d2 - d1)) > 0.3:
                valid[i + 1:i + 7] = False
        a, b = abs(f32(depth[i - 1] - depth[i])), abs(f32(depth[i + 1] - depth[i]))
        lim = 0.02 * float(depth[i])
        mg["parallel"] += [float(a) - lim, float(b) - lim]
        if float(a) > lim and float(b) > lim:
            valid[i] = False
    rough = np.zeros(n, f32)
    for i in range(5, n - 5):
        s = f32(0)
        for k in (-5, -4, -3, -2, -1, 1, 2, 3, 4, 5):
            s = f32(s + depth[i + k])
        s = f32(s - f32(f32(10.0) * depth[i]))
        rough[i] = f32(s * s)
    feat_r, feat_i = rough.copy(), np.arange(n)  # point_features_: sorted in place block by block

    def suppress(idx):
        for k in range(1, 6):
            g = abs(int(col[idx + k]) - int(col[idx + k - 1]))
            mg["col_sup"].append(g - 10)
            if g > 10:
                break
            valid[idx + k] = False
        for k in range(-1, -6, -1):
            g = abs(int(col[idx + k]) - int(col[idx + k + 1]))
            mg["col_sup"].append(g - 10)
            if g > 10:
                break
            valid[idx + k] = False

    ct, pt = f32(corner_thr), f32(planar_thr)
    corners, planars = [], []
    for rs, re in zip(row_start, row_end):
        for b in range(6):
            t = int((int(re) - int(rs)) / 6)  # C integer division (truncation)
            bs, be = int(rs) + b * t, int(rs) + (b + 1) * t
            if bs >= be:
                continue
            order = sorted(range(bs, be), key=lambda j: (feat_r[j], feat_i[j]))  # roughness, then position
            feat_r[bs:be], feat_i[bs:be] = feat_r[order].copy(), feat_i[order].copy()
            picked = 0
            for j in range(be, bs - 1, -1):  # inclusive of `be`
                idx = int(feat_i[j])
                mg["corner"].append(float(feat_r[j]) - float(ct))
                if feat_r[j] > ct and valid[idx]:
                    picked += 1
                    if picked <= 20:
                        corner[idx] = True
                        corners.append(idx)
                        if j == be:
                            mg["be_picked"].append(idx)
                    else:
                        mg["brk"].append(idx)  # the 21st candidate: the pass ends without touching it
                        break
                    valid[idx] = False
                    suppress(idx)
            for j in range(bs, be + 1):  # inclusive of `be`
                idx = int(feat_i[j])
                mg["planar"].append(float(feat_r[j]) - float(pt))
                if valid[idx] and feat_r[j] < pt:
                    valid[idx] = False
                    suppress(idx)
                if not corner[idx]:
                    planars.append(idx)
    margins = {k: np.array(v, np.float64) for k, v in mg.items()}
    margins["rough"] = rough
    return np.array(corners, np.int32), np.array(planars, np.int32), margins


# ---- voxel filter -------------------------------------------------------------------------------------------------------------
def _i32(v: int) -> int:
    return (v + 2 ** 31) % 2 ** 32 - 2 ** 31


def voxel_grid(pts, leaf):
    """pcl::VoxelGrid<PointXYZI>::filter (PCL 1.10), downsample_all_data, as VoxelGridCloud wraps it.  fp32 cell maths; the two
    sizes PCL keeps apart: the overflow test uses d = int((max - min) * inv) + 1 per axis (product > INT_MAX: the input comes back
    unchanged), the ids use divb = floor(max * inv) - floor(min * inv) + 1, which can be one larger per axis.  The id
    i + j * divb0 + k * divb0 * divb1 is int arithmetic (it wraps), stored as unsigned; cells sorted by that unsigned id (ties in
    input order), centroids as sequential fp32 sums of x, y, z and intensity divided by float(count).
    Returns (cloud, info): info has d, divb, overflow and wrapped (some id or multiplier left the int range)."""
    pts = np.asarray(pts, F32).reshape(-1, 4)
    info = dict(d=None, divb=None, overflow=False, wrapped=False)
    if len(pts) == 0:
        return pts.copy(), info
    inv = F32(F32(1.0) / F32(leaf))
    mn, mx = pts[:, :3].min(0), pts[:, :3].max(0)
    d = [int(F32(F32(mx[a] - mn[a]) * inv)) + 1 for a in range(3)]
    minb = [int(np.floor(F32(mn[a] * inv))) for a in range(3)]
    maxb = [int(np.floor(F32(mx[a] * inv))) for a in range(3)]
    divb = [maxb[a] - minb[a] + 1 for a in range(3)]
    info.update(d=d, divb=divb)
    if d[0] * d[1] * d[2] > 2 ** 31 - 1:
        info["overflow"] = True
        return pts.copy(), info
    mul1, mul2_true = divb[0], divb[0] * divb[1]
    mul2 = _i32(mul2_true)
    ids = []
    for p in pts:
        ijk = [int(F32(np.floor(F32(p[a] * inv)) - F32(minb[a]))) for a in range(3)]
        true = ijk[0] + ijk[1] * mul1 + ijk[2] * mul2
        if mul2 != mul2_true or true != _i32(true):
            info["wrapped"] = True
        ids.append(true % 2 ** 32)
    order = sorted(range(len(pts)), key=lambda k: (ids[k], k))
    out = []
    s = 0
    while s < len(order):
        e = s
        while e < len(order) and ids[order[e]] == ids[order[s]]:
            e += 1
        acc = np.zeros(4, F32)
        for k in order[s:e]:
            acc = (acc + pts[k]).astype(F32)
        out.append(acc / F32(e - s))
        s = e
    return np.array(out, F32).reshape(-1, 4), info
