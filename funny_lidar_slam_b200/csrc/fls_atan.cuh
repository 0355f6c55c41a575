// fls_atan.cuh — the two arc tangents of the pre-processing path, each with one fixed sequence of individually rounded operations so
// that the device and the oracle (oracle_convert/orc_convert.h) agree bit for bit:
//   fast_atan2_ref  FastAtan2<float> (include/common/math_function.h:159-186 upstream): the projector's column and the ring of the
//                   sensor type None (src/slam/preprocessing.cpp:485-489);
//   atan2f_pinned   std::atan2(float, float) = atan2f: the yaw of ComputePointOffsetTime (:531).  fp64 octant reduction and fdlibm's
//                   atan on [0, 1], error below about 2 ulp of fp64 before one rounding to float: correctly rounded except where the
//                   true value lies within a few fp64 ulps of a float rounding boundary, and on every pair tested (DESIGN.md §5).
#pragma once

namespace fls {

__device__ __forceinline__ float fast_atan2_ref(float y, float x) {
    const float p1 = 0.9997878412794807f, p3 = -0.3258083974640975f, p5 = 0.1555786518463281f, p7 = -0.04432655554792128f;
    const float ax = fabsf(x), ay = fabsf(y);
    const float eps = 1.1920928955078125e-07f;
    float a;
    if (ax >= ay) {
        const float c = __fdiv_rn(ay, __fadd_rn(ax, eps));
        const float c2 = __fmul_rn(c, c);
        a = __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c);
    } else {
        const float c = __fdiv_rn(ax, __fadd_rn(ay, eps));
        const float c2 = __fmul_rn(c, c);
        a = __fsub_rn(1.57079632679489661923f,
                      __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c));
    }
    if (x < 0.f) a = __fsub_rn(3.14159265358979323846f, a);
    if (y < 0.f) a = __fsub_rn(6.28318530717958647692f, a);
    if (a > 3.14159265358979323846f) a = __fsub_rn(a, 6.28318530717958647692f);
    return a;
}

// fdlibm s_atan.c coefficients
__device__ __forceinline__ double atan01_pinned(double t) {
    const double atanhi0 = 4.63647609000806093515e-01, atanhi1 = 7.85398163397448278999e-01;
    const double atanlo0 = 2.26987774529616870924e-17, atanlo1 = 3.06161699786838301793e-17;
    const double a0 = 3.33333333333329318027e-01, a1 = -1.99999999998764832476e-01, a2 = 1.42857142725034663711e-01,
                 a3 = -1.11111104054623557880e-01, a4 = 9.09088713343650656196e-02, a5 = -7.69187620504482999495e-02,
                 a6 = 6.66107313738753120669e-02, a7 = -5.83357013379057348645e-02, a8 = 4.97687799461593236017e-02,
                 a9 = -3.65315727442169155270e-02, a10 = 1.62858201153657823623e-02;
    int id;
    if (t < 0.4375) {
        if (t < 7.450580596923828125e-09) return t;  // 2^-27
        id = -1;
    } else if (t < 0.6875) {
        id = 0;
        t = __ddiv_rn(__dsub_rn(__dmul_rn(2.0, t), 1.0), __dadd_rn(2.0, t));
    } else {
        id = 1;
        t = __ddiv_rn(__dsub_rn(t, 1.0), __dadd_rn(t, 1.0));
    }
    const double z = __dmul_rn(t, t), w = __dmul_rn(z, z);
    // s1 = z*(a0+w*(a2+w*(a4+w*(a6+w*(a8+w*a10))))), s2 = w*(a1+w*(a3+w*(a5+w*(a7+w*a9))))
    double e = __dadd_rn(a8, __dmul_rn(w, a10));
    e = __dadd_rn(a6, __dmul_rn(w, e));
    e = __dadd_rn(a4, __dmul_rn(w, e));
    e = __dadd_rn(a2, __dmul_rn(w, e));
    e = __dadd_rn(a0, __dmul_rn(w, e));
    const double s1 = __dmul_rn(z, e);
    double o = __dadd_rn(a7, __dmul_rn(w, a9));
    o = __dadd_rn(a5, __dmul_rn(w, o));
    o = __dadd_rn(a3, __dmul_rn(w, o));
    o = __dadd_rn(a1, __dmul_rn(w, o));
    const double s2 = __dmul_rn(w, o);
    const double ts = __dmul_rn(t, __dadd_rn(s1, s2));
    if (id < 0) return __dsub_rn(t, ts);
    const double hi = id == 0 ? atanhi0 : atanhi1, lo = id == 0 ? atanlo0 : atanlo1;
    return __dsub_rn(hi, __dsub_rn(__dsub_rn(ts, lo), t));
}

__device__ __forceinline__ float atan2f_pinned(float y, float x) {
    const double pio2_hi = 1.57079632679489655800e+00, pio2_lo = 6.12323399573676603587e-17;
    const double pi_hi = 3.14159265358979311600e+00, pi_lo = 1.22464679914735317720e-16;
    if (isnan(x) || isnan(y)) return __fadd_rn(x, y);
    const double ax = fabs((double)x), ay = fabs((double)y);
    const bool neg_x = signbit(x);
    double a;
    if (ax == 0.0 && ay == 0.0) {
        a = neg_x ? pi_hi : 0.0;
    } else if (isinf(ax) && isinf(ay)) {
        a = neg_x ? 2.35619449019234483700e+00 : 7.85398163397448278999e-01;  // 3pi/4, pi/4
    } else {
        const bool swap = ay > ax;
        a = atan01_pinned(swap ? __ddiv_rn(ax, ay) : __ddiv_rn(ay, ax));
        if (swap) a = __dsub_rn(pio2_hi, __dsub_rn(a, pio2_lo));
        if (neg_x) a = __dsub_rn(pi_hi, __dsub_rn(a, pi_lo));
    }
    const float r = __double2float_rn(a);
    return signbit(y) ? -r : r;
}

}  // namespace fls
