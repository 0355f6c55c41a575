"""Independent reference of the velocity-aware de-skew of the *_motion entries (include/fls_b200.h; not upstream, which de-skews
rotation only): p_corr = q_ref^-1 q(t) (R_li p + t_li) + v * dt, in 50-digit arithmetic on tests/frontend_ref.py's machinery.

The rotation part is frontend_ref.deskew_point's exact value and its bound on the fp64 evaluation; the term adds, in the pinned
order, dt = (double)dt_us * 1.0e-6 (dt_us = t - ref_time as a signed count, exact as a double on these buffers), v[k] * dt and the
sum, each one more rounding tracked by frontend_ref.R.  A coordinate is decided when the rotation part's interpolation and inverse
are decided and the exact sum lies farther than the bound from every float midpoint; then "device float == this float" is a
bit-level check that does not depend on the oracle.  NaN coordinates (a 0 / 0 ratio) stay NaN and are decided.  A velocity that is
None or all +-0 skips the term: the outputs are frontend_ref's."""
from __future__ import annotations

import mpmath
import numpy as np

from tests import frontend_ref as ref

F32 = np.float32
ONE_US = ref.R(ref.mpf(float(1.0e-6)))  # the double nearest 1e-6, exactly


def moving(velocity) -> bool:
    return velocity is not None and any(float(c) != 0.0 for c in velocity)


def deskew_point(imu, qri, x, y, z, rel_time, velocity):
    """frontend_ref.deskew_point plus v * dt: None when the point's time is outside the buffer, else the same dict (exact, f, err,
    decided, l, t, lerp_zero) for the corrected coordinates."""
    out = ref.deskew_point(imu, qri, x, y, z, rel_time)
    if out is None or not moving(velocity) or mpmath.isnan(out["exact"][0]):
        return out
    # the interpolation and inverse flags: deskew_point folds them into `decided`, so take them from the same helpers it uses
    ts, q = imu["t_us"], np.asarray(imu["q_xyzw"], np.float64)
    l, t = out["l"], out["t"]
    dec_c = ref._lerp(q[l], q[l + 1], ref._ratio(ts, l, l + 1, t))[1]
    dec = dec_c and qri[1]
    dt_us = (t - int(imu["ref_time_us"]) + 2 ** 63) % 2 ** 64 - 2 ** 63
    dt = ref.R(dt_us) * ONE_US
    res = dict(out, exact=[], f=[], err=[], decided=[])
    for k in range(3):
        c = ref.R(out["exact"][k], out["err"][k]) + ref.R(ref.mpf(float(velocity[k]))) * dt
        f, dist = ref.round_f32(c.v)
        res["exact"].append(c.v)
        res["err"].append(c.e)
        res["f"].append(f)
        res["decided"].append(bool(dec and (c.e == 0 or dist > c.e)))
    return res


def preprocess(raw, imu, velocity, min_d, max_d, jump_span, leaf):
    """frontend_ref.preprocess with the term: the same dict (ordered, decided, raw_index, planar_in, planar, dropped_by_time, ...)."""
    if not moving(velocity) or imu is None:
        return ref.preprocess(raw, imu, min_d, max_d, jump_span, leaf)
    raw = np.asarray(raw, F32)
    lo, hi = F32(min_d), F32(max_d)
    qri = ref.ref_inverse(imu)
    if qri is None:
        return ref.preprocess(raw, imu, min_d, max_d, jump_span, leaf)
    ordered, decided, idx, pl, dropped = [], [], [], [], []
    for i, p in enumerate(raw):
        d = ref.depth_f32(p[0], p[1], p[2])
        if d < lo or d > hi:
            continue
        r = deskew_point(imu, qri, p[0], p[1], p[2], p[4], velocity)
        if r is None:
            dropped.append(i)
            continue
        rec = [r["f"][0], r["f"][1], r["f"][2], p[3]]
        ordered.append(rec)
        decided.append(r["decided"])
        idx.append(i)
        if i % int(jump_span) == 0:
            pl.append(rec)
    ordered = np.array(ordered, F32).reshape(-1, 4)
    planar_in = np.array(pl, F32).reshape(-1, 4)
    planar, _ = ref.voxel_grid(planar_in, leaf)
    return dict(ordered=ordered, decided=np.array(decided, bool).reshape(-1, 3), raw_index=np.array(idx, int), planar_in=planar_in, planar=planar,
                dropped_by_time=dropped, scan_dropped=False)


def project(raw, ring, time, imu, velocity, V, H, h_res, min_d, max_d):
    """frontend_ref.project with the winners' coordinates de-skewed by `deskew_point` above; cells, depth and columns are the raw
    points', so only `ordered` and `decided` change."""
    out = ref.project(raw, ring, time, imu, V, H, h_res, min_d, max_d)
    if imu is None or not moving(velocity) or out["n"] == 0:
        return out
    qri = ref.ref_inverse(imu)
    raw = np.asarray(raw, F32)
    ordered, decided = out["ordered"].copy(), out["decided"].copy()
    for j, k in enumerate(out["winner"]):
        r = deskew_point(imu, qri, raw[k, 0], raw[k, 1], raw[k, 2], time[k], velocity)
        ordered[j, :3] = r["f"]
        decided[j] = r["decided"]
    return dict(out, ordered=ordered, decided=decided)
