// ORACLE — TEST INFRASTRUCTURE ONLY.  parity unpinned (the reference ships no test, fixture or
// golden vector for the registration / iVox / LOAM-feature path; see DESIGN.md §oracle).
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may use
// anything under oracle/.  The product (funny_lidar_slam_b200/) never links or calls this code.
//
// Small dense linear algebra + SO(3) helpers restating what the reference gets from Eigen and
// from include/common/math_function.h.  Row-major double arrays, no dependencies.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>

namespace orc {

// ---- 3x3 helpers (row-major) -------------------------------------------------------------------
inline void mat3_mul(const double* A, const double* B, double* C) {
    double t[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) t[i * 3 + j] = A[i * 3 + 0] * B[0 * 3 + j] + A[i * 3 + 1] * B[1 * 3 + j] + A[i * 3 + 2] * B[2 * 3 + j];
    std::memcpy(C, t, sizeof(t));
}
inline void mat3_vec(const double* A, const double* v, double* o) {
    double t0 = A[0] * v[0] + A[1] * v[1] + A[2] * v[2];
    double t1 = A[3] * v[0] + A[4] * v[1] + A[5] * v[2];
    double t2 = A[6] * v[0] + A[7] * v[1] + A[8] * v[2];
    o[0] = t0; o[1] = t1; o[2] = t2;
}
inline void cross3(const double* a, const double* b, double* o) {
    double t0 = a[1] * b[2] - a[2] * b[1];
    double t1 = a[2] * b[0] - a[0] * b[2];
    double t2 = a[0] * b[1] - a[1] * b[0];
    o[0] = t0; o[1] = t1; o[2] = t2;
}
inline double dot3(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
inline double norm3(const double* a) { return std::sqrt(dot3(a, a)); }

// reference: include/common/math_function.h:52-64 (SO3Hat)
inline void so3_hat(const double* v, double* S) {
    S[0] = 0;     S[1] = -v[2]; S[2] = v[1];
    S[3] = v[2];  S[4] = 0;     S[5] = -v[0];
    S[6] = -v[1]; S[7] = v[0];  S[8] = 0;
}

// reference: include/common/math_function.h:74-89 (SO3Exp: Rodrigues, identity when theta <= eps)
inline void so3_exp(const double* v, double* R) {
    const double theta = norm3(v);
    for (int i = 0; i < 9; ++i) R[i] = (i % 4 == 0) ? 1.0 : 0.0;
    if (theta > std::numeric_limits<double>::epsilon()) {
        const double n[3] = {v[0] / theta, v[1] / theta, v[2] / theta};
        const double c = std::cos(theta), s = std::sin(theta);
        double S[9];
        so3_hat(n, S);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j)
                R[i * 3 + j] = c * (i == j ? 1.0 : 0.0) + (1.0 - c) * n[i] * n[j] + s * S[i * 3 + j];
    }
}

// reference: include/common/math_function.h:100-131 (SE3Exp; v = [translation, rotation]).  Only used
// to pin so3_exp/so3_hat against the golden 4x4 in test/math_function_ut.cpp:135-148.
inline void se3_exp(const double* v, double* T /*4x4 row-major*/) {
    const double* w = v + 3;
    const double theta = norm3(w);
    double R[9], W[9], W2[9], J[9];
    so3_exp(w, R);
    so3_hat(w, W);
    mat3_mul(W, W, W2);
    if (theta < std::numeric_limits<double>::epsilon()) {
        std::memcpy(J, R, sizeof(J));
    } else {
        const double t2 = theta * theta;
        for (int i = 0; i < 9; ++i)
            J[i] = (i % 4 == 0 ? 1.0 : 0.0) + (1.0 - std::cos(theta)) / t2 * W[i] + (theta - std::sin(theta)) / (t2 * theta) * W2[i];
    }
    double t[3];
    mat3_vec(J, v, t);
    for (int i = 0; i < 16; ++i) T[i] = 0;
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) T[i * 4 + j] = R[i * 3 + j];
        T[i * 4 + 3] = t[i];
    }
    T[15] = 1;
}

// reference: include/common/math_function.h:139-149 (RotationMatrixToRPY)
inline void rot_to_rpy(const double* R, double* rpy) {
    rpy[0] = std::atan2(R[2 * 3 + 1], R[2 * 3 + 2]);
    rpy[1] = std::asin(-R[2 * 3 + 0]);
    rpy[2] = std::atan2(R[1 * 3 + 0], R[0 * 3 + 0]);
}

// reference: include/common/math_function.h:159-186 (FastAtan2<float>)
inline float fast_atan2f(float y, float x) {
    const float p1 = 0.9997878412794807f, p3 = -0.3258083974640975f, p5 = 0.1555786518463281f, p7 = -0.04432655554792128f;
    float ax = std::fabs(x), ay = std::fabs(y), a, c, c2;
    if (ax >= ay) {
        c = ay / (ax + std::numeric_limits<float>::epsilon());
        c2 = c * c;
        a = (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
    } else {
        c = ax / (ay + std::numeric_limits<float>::epsilon());
        c2 = c * c;
        a = float(M_PI_2) - (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
    }
    if (x < 0) a = float(M_PI) - a;
    if (y < 0) a = float(2 * M_PI) - a;
    if (a > float(M_PI)) a -= float(2 * M_PI);
    return a;
}

// ---- least squares: Householder QR with column pivoting -----------------------------------------
// Restates Eigen::ColPivHouseholderQR<Matrix<double,M,N>>::solve as used at
// loam_point_to_plane_ivox.h:283 (5x3 plane fit).  Solution of a full-rank LS problem is unique; on
// exactly-zero remaining columns the corresponding unknowns are set to 0 (Eigen's nonzeroPivots rule).  The GPU's QR
// (fls_plane.cuh plane_lstsq) performs the same operations in the same order, so rank decisions on rounding-level columns
// agree bit for bit (DESIGN.md §5): change both or neither.
template <int M, int N>
inline void lstsq_colpiv_qr(const double* A_in /*MxN row-major*/, const double* b_in, double* x) {
    double A[M * N], b[M];
    std::memcpy(A, A_in, sizeof(A));
    std::memcpy(b, b_in, sizeof(b));
    int perm[N];
    double cn[N];
    (void)cn;
    double maxcn = 0;
    for (int j = 0; j < N; ++j) {
        perm[j] = j;
        double s = 0;
        for (int i = 0; i < M; ++i) s += A[i * N + j] * A[i * N + j];
        cn[j] = s;
        maxcn = std::max(maxcn, s);
    }
    const double eps = std::numeric_limits<double>::epsilon();
    const double thr = (eps * std::sqrt(maxcn) / double(M)) * (eps * std::sqrt(maxcn) / double(M));
    int rank = N;
    for (int k = 0; k < N; ++k) {
        int piv = k;
        double best = -1;
        for (int j = k; j < N; ++j) {  // recompute exactly (tiny sizes) instead of norm down-dating
            double s = 0;
            for (int i = k; i < M; ++i) s += A[i * N + j] * A[i * N + j];
            cn[j] = s;
            if (s > best) { best = s; piv = j; }
        }
        if (best < thr || best == 0.0) { rank = k; break; }
        if (piv != k) {
            for (int i = 0; i < M; ++i) std::swap(A[i * N + k], A[i * N + piv]);
            std::swap(perm[k], perm[piv]);
        }
        // Householder vector for column k, rows k..M-1
        double alpha = A[k * N + k];
        double tail = 0;
        for (int i = k + 1; i < M; ++i) tail += A[i * N + k] * A[i * N + k];
        double beta, tau, v[M];
        if (tail == 0.0) {
            tau = 0; beta = alpha;
            for (int i = 0; i < M; ++i) v[i] = 0;
        } else {
            beta = std::sqrt(alpha * alpha + tail);
            if (alpha >= 0) beta = -beta;
            for (int i = k + 1; i < M; ++i) v[i] = A[i * N + k] / (alpha - beta);
            tau = (beta - alpha) / beta;
        }
        v[k] = 1.0;
        A[k * N + k] = beta;
        for (int i = k + 1; i < M; ++i) A[i * N + k] = 0;
        if (tau != 0.0) {
            for (int j = k + 1; j < N; ++j) {
                double s = 0;
                for (int i = k; i < M; ++i) s += v[i] * A[i * N + j];
                s *= tau;
                for (int i = k; i < M; ++i) A[i * N + j] -= s * v[i];
            }
            double s = 0;
            for (int i = k; i < M; ++i) s += v[i] * b[i];
            s *= tau;
            for (int i = k; i < M; ++i) b[i] -= s * v[i];
        }
    }
    double y[N];
    for (int i = 0; i < N; ++i) y[i] = 0;
    for (int i = rank - 1; i >= 0; --i) {
        double s = b[i];
        for (int j = i + 1; j < rank; ++j) s -= A[i * N + j] * y[j];
        y[i] = s / A[i * N + i];
    }
    for (int i = 0; i < N; ++i) x[i] = 0;
    for (int i = 0; i < rank; ++i) x[perm[i]] = y[i];
}

// ---- NxN solve with complete pivoting -----------------------------------------------------------
// Stands in for Eigen::FullPivHouseholderQR<Matrix6d>::solve (loam_point_to_plane_ivox.h:167,
// loam_point_to_plane_kdtree.h:108, loam_full_kdtree.h:141).  For a non-singular system every stable
// method returns the same x to ~cond*eps; rank deficiency (pivot <= eps*N*maxpivot) yields the basic
// solution with zeros, as Eigen's rank-revealing solve does.
template <int N>
inline void solve_fullpiv(const double* H_in, const double* g_in, double* x) {
    double A[N * N], b[N];
    std::memcpy(A, H_in, sizeof(A));
    std::memcpy(b, g_in, sizeof(b));
    int cperm[N];
    for (int i = 0; i < N; ++i) cperm[i] = i;
    double maxpiv = 0;
    int rank = N;
    const double eps = std::numeric_limits<double>::epsilon();
    for (int k = 0; k < N; ++k) {
        int pr = k, pc = k;
        double best = -1;
        for (int i = k; i < N; ++i)
            for (int j = k; j < N; ++j)
                if (std::fabs(A[i * N + j]) > best) { best = std::fabs(A[i * N + j]); pr = i; pc = j; }
        if (k == 0) maxpiv = best;
        if (best <= eps * N * maxpiv || best == 0.0) { rank = k; break; }
        if (pr != k) {
            for (int j = 0; j < N; ++j) std::swap(A[k * N + j], A[pr * N + j]);
            std::swap(b[k], b[pr]);
        }
        if (pc != k) {
            for (int i = 0; i < N; ++i) std::swap(A[i * N + k], A[i * N + pc]);
            std::swap(cperm[k], cperm[pc]);
        }
        for (int i = k + 1; i < N; ++i) {
            const double f = A[i * N + k] / A[k * N + k];
            if (f == 0.0) continue;
            for (int j = k; j < N; ++j) A[i * N + j] -= f * A[k * N + j];
            b[i] -= f * b[k];
        }
    }
    double y[N];
    for (int i = 0; i < N; ++i) y[i] = 0;
    for (int i = rank - 1; i >= 0; --i) {
        double s = b[i];
        for (int j = i + 1; j < rank; ++j) s -= A[i * N + j] * y[j];
        y[i] = s / A[i * N + i];
    }
    for (int i = 0; i < N; ++i) x[i] = 0;
    for (int i = 0; i < rank; ++i) x[cperm[i]] = y[i];
}

// ---- NxN partial-pivot LU: solve + determinant ---------------------------------------------------
// Stands in for Eigen's `H.inverse() * b` and `H.determinant()` (icp_optimized.h:129,133;
// incremental_ndt.h:311).  Returns the determinant; x is untouched when det == 0.
template <int N>
inline double solve_lu(const double* H_in, const double* g_in, double* x) {
    double A[N * N], b[N];
    std::memcpy(A, H_in, sizeof(A));
    std::memcpy(b, g_in, sizeof(b));
    double det = 1.0;
    for (int k = 0; k < N; ++k) {
        int pr = k;
        double best = std::fabs(A[k * N + k]);
        for (int i = k + 1; i < N; ++i)
            if (std::fabs(A[i * N + k]) > best) { best = std::fabs(A[i * N + k]); pr = i; }
        if (best == 0.0) return 0.0;
        if (pr != k) {
            for (int j = 0; j < N; ++j) std::swap(A[k * N + j], A[pr * N + j]);
            std::swap(b[k], b[pr]);
            det = -det;
        }
        det *= A[k * N + k];
        for (int i = k + 1; i < N; ++i) {
            const double f = A[i * N + k] / A[k * N + k];
            for (int j = k; j < N; ++j) A[i * N + j] -= f * A[k * N + j];
            b[i] -= f * b[k];
        }
    }
    for (int i = N - 1; i >= 0; --i) {
        double s = b[i];
        for (int j = i + 1; j < N; ++j) s -= A[i * N + j] * x[j];
        x[i] = s / A[i * N + i];
    }
    return det;
}

// 3x3 inverse by cofactors (Eigen's fixed-size 3x3 inverse; incremental_ndt.h:134,151)
inline void inv3(const double* A, double* Ai) {
    const double c00 = A[4] * A[8] - A[5] * A[7], c01 = A[5] * A[6] - A[3] * A[8], c02 = A[3] * A[7] - A[4] * A[6];
    const double det = A[0] * c00 + A[1] * c01 + A[2] * c02;
    const double id = 1.0 / det;
    Ai[0] = c00 * id; Ai[1] = (A[2] * A[7] - A[1] * A[8]) * id; Ai[2] = (A[1] * A[5] - A[2] * A[4]) * id;
    Ai[3] = c01 * id; Ai[4] = (A[0] * A[8] - A[2] * A[6]) * id; Ai[5] = (A[2] * A[3] - A[0] * A[5]) * id;
    Ai[6] = c02 * id; Ai[7] = (A[1] * A[6] - A[0] * A[7]) * id; Ai[8] = (A[0] * A[4] - A[1] * A[3]) * id;
}

// Symmetric 3x3 eigen-decomposition by cyclic Jacobi; eigenvalues sorted descending, V columns.
// Stands in for Eigen::JacobiSVD on a symmetric PSD matrix (incremental_ndt.h:166, loam_full_kdtree.h:244):
// for such a matrix U == V and the singular values are the eigenvalues.
inline void sym_eig3(const double* S, double* lam, double* V) {
    double A[9];
    std::memcpy(A, S, sizeof(A));
    for (int i = 0; i < 9; ++i) V[i] = (i % 4 == 0) ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 60; ++sweep) {
        const double off = std::fabs(A[1]) + std::fabs(A[2]) + std::fabs(A[5]);
        if (off < 1e-300) break;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                const double apq = A[p * 3 + q];
                if (apq == 0.0) continue;
                const double theta = (A[q * 3 + q] - A[p * 3 + p]) / (2.0 * apq);
                const double t = (theta >= 0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
                const double c = 1.0 / std::sqrt(t * t + 1.0), s = t * c;
                for (int k = 0; k < 3; ++k) {
                    const double akp = A[k * 3 + p], akq = A[k * 3 + q];
                    A[k * 3 + p] = c * akp - s * akq;
                    A[k * 3 + q] = s * akp + c * akq;
                }
                for (int k = 0; k < 3; ++k) {
                    const double apk = A[p * 3 + k], aqk = A[q * 3 + k];
                    A[p * 3 + k] = c * apk - s * aqk;
                    A[q * 3 + k] = s * apk + c * aqk;
                }
                for (int k = 0; k < 3; ++k) {
                    const double vkp = V[k * 3 + p], vkq = V[k * 3 + q];
                    V[k * 3 + p] = c * vkp - s * vkq;
                    V[k * 3 + q] = s * vkp + c * vkq;
                }
            }
    }
    int idx[3] = {0, 1, 2};
    double d[3] = {A[0], A[4], A[8]};
    std::sort(idx, idx + 3, [&](int a, int b) { return d[a] > d[b]; });
    double Vs[9];
    for (int j = 0; j < 3; ++j) {
        lam[j] = d[idx[j]];
        for (int i = 0; i < 3; ++i) Vs[i * 3 + j] = V[i * 3 + idx[j]];
    }
    std::memcpy(V, Vs, sizeof(Vs));
}

}  // namespace orc
