// fls_plane.cuh — the per-point geometry shared by the LOAM point-to-plane plug-ins (iVox, kd-tree, LoamFull planar term):
// top-5 selection registers, the 5x3 least-squares plane (normal equations with a measured-cancellation guard, column-
// pivoted Householder QR as the out-of-line fallback) and the residual / Jacobian of
// loam_point_to_plane_ivox.h:275-321 == loam_point_to_plane_kdtree.h:226-283 == loam_full_kdtree.h:295-343 upstream.
#pragma once
#include "fls_common.cuh"

namespace fls {
namespace {

// ---- branch-free top-5 ---------------------------------------------------------------------------------------------
// Each entry is ONE 64-bit key {hi = IEEE bits of the fp32 squared distance, lo = candidate index} held in a double
// register: for non-negative, non-NaN floats the bit pattern orders like the value, and positive doubles order like
// their bit patterns, so fp64 min/max (one DMNMX each) is a compare-exchange on (distance, visit order) — the
// ascending-index tie-break IS the reference's "earlier candidate wins" rule.  Rejected candidates carry the
// sentinel key {+inf, 0xffffffff}, which never displaces anything.
// (measured: holding {distance bits, index} as one fp64 key and using fmin/fmax compiles to DSETP + 2 FSEL per
//  min/max — slower than the separate float / index compare-exchange below.)
struct Top5 {
    float d0, d1, d2, d3, d4;
    unsigned k0, k1, k2, k3, k4;
    __device__ __forceinline__ void init() {
        d0 = d1 = d2 = d3 = d4 = INFINITY;
        k0 = k1 = k2 = k3 = k4 = 0xffffffffu;
    }
#define FLS_CE(da, ja, db, jb)               \
    {                                        \
        const bool c_ = (db) < (da);         \
        const float td_ = (da);              \
        const unsigned tj_ = (ja);           \
        (da) = c_ ? (db) : (da);             \
        (ja) = c_ ? (jb) : (ja);             \
        (db) = c_ ? td_ : (db);              \
        (jb) = c_ ? tj_ : (jb);              \
    }
    // ascending (d, visit order): strict '<' everywhere, so a later candidate never passes an equal earlier one;
    // a rejected candidate arrives as {+inf, 0xffffffff} and never displaces anything
    __device__ __forceinline__ void push(float d, unsigned j) {
        const bool c = d < d4;
        d4 = c ? d : d4;
        k4 = c ? j : k4;
        FLS_CE(d3, k3, d4, k4)
        FLS_CE(d2, k2, d3, k3)
        FLS_CE(d1, k1, d2, k2)
        FLS_CE(d0, k0, d1, k1)
    }
#undef FLS_CE
    __device__ __forceinline__ unsigned idx(unsigned k) const { return k; }
    __device__ __forceinline__ bool full() const { return k4 != 0xffffffffu; }
};

// ---- 5x3 least squares ---------------------------------------------------------------------------------------------
// Column-pivoted Householder QR, operation for operation the one of the oracle (orc_math.h lstsq_colpiv_qr): the Eigen
// reflector form (v = [1, x_tail / (alpha - beta)], tau = (beta - alpha) / beta), pivot norms recomputed per step, the rank
// cut (eps sqrt(max column norm^2) / 5)^2.  Every product, sum, quotient and root is rounded on its own (no FMA contraction),
// as the oracle's -ffp-contract=off build does.  A neighbourhood whose remaining column is rounding noise (repeated points, a
// pole, an off-axis line) is decided by that noise against the cut; with the same arithmetic on both sides the GPU and the
// oracle take the same rank decision bit for bit (DESIGN.md §5).
__device__ __forceinline__ double rn_add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double rn_sub(double a, double b) { return __dadd_rn(a, -b); }
__device__ __forceinline__ double rn_mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double rn_div(double a, double b) { return __ddiv_rn(a, b); }

// min || A c + 1 ||  — Eigen colPivHouseholderQr().solve(b) with b = -1 (loam_point_to_plane_ivox.h:275-283 upstream).
// A is destroyed.
__device__ __forceinline__ void plane_lstsq(double (&A)[5][3], double (&c)[3]) {
    double b[5] = {-1.0, -1.0, -1.0, -1.0, -1.0};
    int perm[3] = {0, 1, 2};
    double maxcn = 0.0;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        double s = 0.0;
#pragma unroll
        for (int i = 0; i < 5; ++i) s = rn_add(s, rn_mul(A[i][j], A[i][j]));
        maxcn = fmax(maxcn, s);
    }
    const double h = rn_div(rn_mul(2.220446049250313e-16, __dsqrt_rn(maxcn)), 5.0);
    const double thr = rn_mul(h, h);
    int rank = 3;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        int piv = k;
        double best = -1.0;
#pragma unroll
        for (int j = k; j < 3; ++j) {
            double s = 0.0;
#pragma unroll
            for (int i = k; i < 5; ++i) s = rn_add(s, rn_mul(A[i][j], A[i][j]));
            if (s > best) {
                best = s;
                piv = j;
            }
        }
        if (best < thr || best == 0.0) {
            rank = k;
            break;
        }
        if (piv != k) {
#pragma unroll
            for (int i = 0; i < 5; ++i) {
                const double t = A[i][k];
                A[i][k] = A[i][piv];
                A[i][piv] = t;
            }
            const int t = perm[k];
            perm[k] = perm[piv];
            perm[piv] = t;
        }
        const double alpha = A[k][k];
        double tail = 0.0;
#pragma unroll
        for (int i = k + 1; i < 5; ++i) tail = rn_add(tail, rn_mul(A[i][k], A[i][k]));
        double beta = alpha, tau = 0.0, v[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
        if (tail != 0.0) {
            beta = __dsqrt_rn(rn_add(rn_mul(alpha, alpha), tail));
            if (alpha >= 0) beta = -beta;
            const double den = rn_sub(alpha, beta);
#pragma unroll
            for (int i = k + 1; i < 5; ++i) v[i] = rn_div(A[i][k], den);
            tau = rn_div(rn_sub(beta, alpha), beta);
        }
        v[k] = 1.0;
        A[k][k] = beta;
#pragma unroll
        for (int i = k + 1; i < 5; ++i) A[i][k] = 0.0;
        if (tau != 0.0) {
#pragma unroll
            for (int j = k + 1; j < 3; ++j) {
                double s = 0.0;
#pragma unroll
                for (int i = k; i < 5; ++i) s = rn_add(s, rn_mul(v[i], A[i][j]));
                s = rn_mul(s, tau);
#pragma unroll
                for (int i = k; i < 5; ++i) A[i][j] = rn_sub(A[i][j], rn_mul(s, v[i]));
            }
            double s = 0.0;
#pragma unroll
            for (int i = k; i < 5; ++i) s = rn_add(s, rn_mul(v[i], b[i]));
            s = rn_mul(s, tau);
#pragma unroll
            for (int i = k; i < 5; ++i) b[i] = rn_sub(b[i], rn_mul(s, v[i]));
        }
    }
    double y[3] = {0.0, 0.0, 0.0};
#pragma unroll
    for (int i = 2; i >= 0; --i) {
        if (i < rank) {
            double s = b[i];
#pragma unroll
            for (int j = i + 1; j < 3; ++j)
                if (j < rank) s = rn_sub(s, rn_mul(A[i][j], y[j]));
            y[i] = rn_div(s, A[i][i]);
        }
    }
    c[0] = c[1] = c[2] = 0.0;
#pragma unroll
    for (int i = 0; i < 3; ++i)
        if (i < rank) c[perm[i]] = y[i];
}

// neighbour fetch: read-only global path (kLdg) or a generic load (the point may sit in shared memory: K1 stages the
// candidate runs of a chunk there with cp.async.bulk, fls_p2plane.cu)
template <bool kLdg>
__device__ __forceinline__ float4 plane_ld(const float4* p) {
    if (kLdg) return __ldg(p);
    return *p;
}

// Out-of-line QR path for ill-conditioned neighbourhoods (kept out of the hot path's register budget).
template <bool kLdg>
__device__ __noinline__ void plane_lstsq_qr(const float4* lists, unsigned j0, unsigned j1, unsigned j2, unsigned j3, unsigned j4,
                                            double (&c)[3]) {
    const unsigned js[5] = {j0, j1, j2, j3, j4};
    double A[5][3];
#pragma unroll
    for (int i = 0; i < 5; ++i) {
        const float4 a = plane_ld<kLdg>(lists + js[i]);
        A[i][0] = a.x; A[i][1] = a.y; A[i][2] = a.z;
    }
    plane_lstsq(A, c);
}

// Plane through the 5 neighbours P[js[0..4]] (js[0] = nearest) -> J (6) and |d| of source point `sp` whose transformed
// position is q.  Returns false when upstream rejects the point (invalid plane, near-point gate).
template <bool kLdg = true>
__device__ __forceinline__ bool plane_term(const float4* P, const unsigned (&js)[5], const float4 sp, float qx, float qy, float qz,
                                           const double* __restrict__ pose /*R[9], t[3]*/, double plane_thres, double (&J)[6], double& ad,
                                           unsigned& n_fallback) {
    double c[3];
    {
        // Fast path: normal equations (A^T A) c = -A^T 1 by a pivot-free LDL^T.  The inputs are fp32, so every product
        // is exact in fp64 and each sum carries ~1e-16 relative error; the only loss is cancellation in the two Schur
        // complements, which is measured — if either keeps fewer than ~9 digits the point takes the QR path below.
        double sxx = 0, sxy = 0, sxz = 0, syy = 0, syz = 0, szz = 0, bx = 0, by = 0, bz = 0;
#pragma unroll
        for (int i = 0; i < 5; ++i) {
            const float4 a = plane_ld<kLdg>(P + js[i]);
            const double x = a.x, y = a.y, z = a.z;
            sxx += x * x; sxy += x * y; sxz += x * z; syy += y * y; syz += y * z; szz += z * z;
            bx -= x; by -= y; bz -= z;
        }
        bool ok = sxx > 0.0;
        const double i0 = 1.0 / sxx;
        const double l10 = sxy * i0, l20 = sxz * i0;
        const double d1 = syy - l10 * sxy;
        const double e = syz - l10 * sxz;
        const double t2 = szz - l20 * sxz;
        ok = ok && (d1 > 1e-7 * syy);
        const double i1 = 1.0 / d1;
        const double l21 = e * i1;
        const double d2 = t2 - l21 * e;
        ok = ok && (d2 > 1e-7 * fmax(szz, fabs(l21 * e)));
        if (ok) {
            const double y1 = by - l10 * bx;
            const double y2 = bz - l20 * bx - l21 * y1;
            const double c2 = y2 / d2;
            const double c1 = y1 * i1 - l21 * c2;
            c[0] = bx * i0 - l10 * c1 - l20 * c2;
            c[1] = c1;
            c[2] = c2;
        } else {
            ++n_fallback;
            double cq[3];  // the out-of-line solve's result goes through memory; `c` stays in registers on the fast path
            plane_lstsq_qr<kLdg>(P, js[0], js[1], js[2], js[3], js[4], cq);
            c[0] = cq[0];
            c[1] = cq[1];
            c[2] = cq[2];
        }
    }
    const double cn = sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]);
    // |A_j c + 1| / ||c|| > thres  (:286-293), evaluated as |A_j c + 1| > thres * ||c||; the 5 rows are re-read
    // (L1 hits) instead of being kept live across the QR
    const double lim = plane_thres * cn;
    bool valid = cn > 0.0;
    float4 a0 = make_float4(0, 0, 0, 0);
#pragma unroll
    for (int i = 0; i < 5; ++i) {
        const float4 a = plane_ld<kLdg>(P + js[i]);
        if (i == 0) a0 = a;
        if (fabs((double)a.x * c[0] + (double)a.y * c[1] + (double)a.z * c[2] + 1.0) > lim) valid = false;
    }
    if (!valid) return false;
    const double icn = 1.0 / cn;
    const double nx = c[0] * icn, ny = c[1] * icn, nz = c[2] * icn;
    const double d = ((double)qx - (double)a0.x) * nx + ((double)qy - (double)a0.y) * ny + ((double)qz - (double)a0.z) * nz;  // :306
    const double px = sp.x, py = sp.y, pz = sp.z;
    if (sqrt(px * px + py * py + pz * pz) < 81.0 * d * d) return false;  // :309 body-frame norm
    const double s = d > 0 ? 1.0 : -1.0;
    const double rx = pose[0] * px + pose[1] * py + pose[2] * pz;
    const double ry = pose[3] * px + pose[4] * py + pose[5] * pz;
    const double rz = pose[6] * px + pose[7] * py + pose[8] * pz;
    J[0] = s * (ry * nz - rz * ny);  // (R p) x n  == -hat(R p)^T n  (:315)
    J[1] = s * (rz * nx - rx * nz);
    J[2] = s * (rx * ny - ry * nx);
    J[3] = s * nx;
    J[4] = s * ny;
    J[5] = s * nz;
    ad = fabs(d);
    return true;
}

}  // namespace
}  // namespace fls
