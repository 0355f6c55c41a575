// fls_deskew.cuh — LidarDistortionCorrector::ProcessPoint (src/lidar/lidar_distortion_corrector.cpp:37-64 upstream) on the device:
// IMU orientation interpolated at the point's time (DataSearcher::SearchNearestTwoData, include/common/data_searcher.h:100-134;
// MotionInterpolator::InterpolateQuaternionLerp, include/common/motion_interpolator.h:27-35), point moved lidar -> imu and rotated
// by q_ref^-1 * q(t).  fp64 with explicit roundings in the evaluation order the oracle pins (oracle/orc_deskew.h), so the
// corrected coordinates are bit-identical.  With a body velocity (the *_motion entries, not upstream) the constant-velocity
// translation v * dt is added in fp64 before the rounding to float (oracle_motion/orc_motion.h pins that order).
#pragma once
#include "fls_common.cuh"

namespace fls {

struct DeskewView {
    const unsigned long long* __restrict__ t;  // IMU time stamps [us], ascending (device)
    const double* __restrict__ q;              // quaternions x, y, z, w (device)
    int m;                                     // 0: no de-skew (identity)
    int move;                                  // 1: add v * dt (v has a non-zero component); 0: rotation only
    unsigned long long ref_time;
    double qri[4];   // q_ref^-1 (x, y, z, w) — SetRefTime (:19-34), computed on the host
    double T[16];    // lidar -> imu, column-major
    double v[3];     // body velocity [m/s] in the IMU frame at ref_time (read when move)
};

#ifdef __CUDACC__
__device__ __forceinline__ bool deskew_point(const DeskewView& d, float x, float y, float z, float rel_time, float& xo, float& yo, float& zo) {
    const long long dt_us = trunc_i64(__dmul_rn((double)rel_time, 1.0e6));
    const unsigned long long t = (unsigned long long)((long long)d.ref_time + dt_us);
    const int m = d.m;
    if (m < 2 || d.t[0] > t || d.t[m - 1] < t) return false;
    int l;
    if (d.t[0] == t) l = 0;
    else if (d.t[m - 1] == t) l = m - 2;
    else {  // last sample not later than t
        int lo = 0, hi = m - 1;
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (d.t[mid] <= t) lo = mid;
            else hi = mid;
        }
        l = lo;
    }
    const int r = l + 1;
    const double s = __ddiv_rn((double)(t - d.t[l]), (double)(d.t[r] - d.t[l]));
    const double u = __dsub_rn(1.0, s);
    const double* a = d.q + 4 * l;
    const double* b = d.q + 4 * r;
    double qx = __dadd_rn(__dmul_rn(a[0], u), __dmul_rn(b[0], s));
    double qy = __dadd_rn(__dmul_rn(a[1], u), __dmul_rn(b[1], s));
    double qz = __dadd_rn(__dmul_rn(a[2], u), __dmul_rn(b[2], s));
    double qw = __dadd_rn(__dmul_rn(a[3], u), __dmul_rn(b[3], s));
    // q.normalized(): Eigen 3.3.7 leaves the coefficients as they are unless the squared norm is > 0 (q(t) = 0 between q and -q;
    // NaN from a 0 / 0 ratio)
    const double sq = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(qx, qx), __dmul_rn(qy, qy)), __dmul_rn(qz, qz)), __dmul_rn(qw, qw));
    if (sq > 0.0) {
        const double n = __dsqrt_rn(sq);
        qx = __ddiv_rn(qx, n); qy = __ddiv_rn(qy, n); qz = __ddiv_rn(qz, n); qw = __ddiv_rn(qw, n);
    }
    // q = q_ref^-1 * q(t)
    const double ax = d.qri[0], ay = d.qri[1], az = d.qri[2], aw = d.qri[3];
    const double px = __dsub_rn(__dadd_rn(__dadd_rn(__dmul_rn(aw, qx), __dmul_rn(ax, qw)), __dmul_rn(ay, qz)), __dmul_rn(az, qy));
    const double py = __dsub_rn(__dadd_rn(__dadd_rn(__dmul_rn(aw, qy), __dmul_rn(ay, qw)), __dmul_rn(az, qx)), __dmul_rn(ax, qz));
    const double pz = __dsub_rn(__dadd_rn(__dadd_rn(__dmul_rn(aw, qz), __dmul_rn(az, qw)), __dmul_rn(ax, qy)), __dmul_rn(ay, qx));
    const double pw = __dsub_rn(__dsub_rn(__dsub_rn(__dmul_rn(aw, qw), __dmul_rn(ax, qx)), __dmul_rn(ay, qy)), __dmul_rn(az, qz));
    // lidar -> imu
    const double* T = d.T;
    const double vx = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[0], (double)x), __dmul_rn(T[4], (double)y)), __dmul_rn(T[8], (double)z)), T[12]);
    const double vy = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[1], (double)x), __dmul_rn(T[5], (double)y)), __dmul_rn(T[9], (double)z)), T[13]);
    const double vz = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[2], (double)x), __dmul_rn(T[6], (double)y)), __dmul_rn(T[10], (double)z)), T[14]);
    // v + w * (2 q x v) + q x (2 q x v)
    double ux = __dsub_rn(__dmul_rn(py, vz), __dmul_rn(pz, vy));
    double uy = __dsub_rn(__dmul_rn(pz, vx), __dmul_rn(px, vz));
    double uz = __dsub_rn(__dmul_rn(px, vy), __dmul_rn(py, vx));
    ux = __dadd_rn(ux, ux); uy = __dadd_rn(uy, uy); uz = __dadd_rn(uz, uz);
    double ox = __dadd_rn(__dadd_rn(vx, __dmul_rn(pw, ux)), __dsub_rn(__dmul_rn(py, uz), __dmul_rn(pz, uy)));
    double oy = __dadd_rn(__dadd_rn(vy, __dmul_rn(pw, uy)), __dsub_rn(__dmul_rn(pz, ux), __dmul_rn(px, uz)));
    double oz = __dadd_rn(__dadd_rn(vz, __dmul_rn(pw, uz)), __dsub_rn(__dmul_rn(px, uy), __dmul_rn(py, ux)));
    if (d.move) {  // + v * dt; skipped (not + 0.0) without motion, so a -0.0 stays -0.0
        const double dt = __dmul_rn((double)dt_us, 1.0e-6);
        ox = __dadd_rn(ox, __dmul_rn(d.v[0], dt));
        oy = __dadd_rn(oy, __dmul_rn(d.v[1], dt));
        oz = __dadd_rn(oz, __dmul_rn(d.v[2], dt));
    }
    xo = (float)ox;
    yo = (float)oy;
    zo = (float)oz;
    return true;
}
#endif

// Host half of SetRefTime (:19-34): q_ref^-1 from the IMU samples around ref_time; same evaluation order as the oracle.
// Returns false when ref_time is outside the buffer.
bool deskew_ref_inverse(const unsigned long long* t, const double* q_xyzw, size_t m, unsigned long long ref_time, double* qri);

}  // namespace fls
