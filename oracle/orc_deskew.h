// orc_deskew.h — CPU restatement (test infrastructure, see orc_math.h) of the pre-hot-path point pipeline:
//   LidarDistortionCorrector::SetRefTime / ProcessPoint   src/lidar/lidar_distortion_corrector.cpp:19-64
//   DataSearcher::SearchNearestTwoData                    include/common/data_searcher.h:100-134
//   MotionInterpolator::InterpolateQuaternionLerp         include/common/motion_interpolator.h:27-35
//   PreProcessing::Run, the non-feature branch            src/slam/preprocessing.cpp:181-225
//   PointcloudProjector::Project with its per-point de-skew  src/loam/pointcloud_projector.cpp:32-133 (:100-103)
// Eigen's quaternion algebra is restated with a fixed evaluation order (left to right, no FMA); the GPU path reproduces
// exactly this order, so the two agree bit for bit.
#pragma once
#include <cmath>
#include <cstdint>
#include <limits>
#include <vector>

#include "orc_cloud.h"
#include "orc_features.h"

namespace orc {

struct Quat { double x, y, z, w; };  // Eigen coefficient order

struct ImuBuffer {
    std::vector<uint64_t> t;  // microseconds, ascending
    std::vector<Quat> q;
    uint64_t ref_time = 0;
    double T_li[16];  // lidar -> imu, column-major 4x4
};

// int64_t(rel_time * 1.0e6) of ProcessPoint (:41) as x86-64's cvttsd2si computes it: toward zero, INT64_MIN for NaN and for
// values outside the int64 range (a plain conversion is undefined behaviour there).  The device uses the same rule (trunc_i64).
inline int64_t time_to_i64(double v) {
    return (v >= -9.2233720368547758e18 && v < 9.2233720368547758e18) ? int64_t(v) : std::numeric_limits<int64_t>::min();
}

// data_searcher.h:100-134
inline bool search_two(const ImuBuffer& b, uint64_t t, size_t& l, size_t& r) {
    const size_t m = b.t.size();
    if (m == 0) return false;
    if (b.t.front() > t || b.t.back() < t) return false;
    if (m < 2) return false;  // upstream would read past the deque
    if (b.t.front() == t) { l = 0; r = 1; return true; }
    if (b.t.back() == t) { r = m - 1; l = m - 2; return true; }
    size_t i = m - 1;
    while (t < b.t[i]) --i;
    l = i;
    r = i + 1;
    return true;
}

// motion_interpolator.h:27-35: normalised linear interpolation of the coefficients (no hemisphere alignment).  Eigen 3.3.7's
// normalized() returns the coefficients unchanged when the squared norm is not > 0 (q and -q at ratio 0.5: zero; a NaN ratio).
inline Quat lerp(const Quat& a, const Quat& b, double s) {
    const double u = 1.0 - s;
    Quat q{a.x * u + b.x * s, a.y * u + b.y * s, a.z * u + b.z * s, a.w * u + b.w * s};
    const double sq = ((q.x * q.x + q.y * q.y) + q.z * q.z) + q.w * q.w;
    if (!(sq > 0.0)) return q;
    const double n = std::sqrt(sq);
    return Quat{q.x / n, q.y / n, q.z / n, q.w / n};
}
inline Quat qmul(const Quat& a, const Quat& b) {
    return Quat{((a.w * b.x + a.x * b.w) + a.y * b.z) - a.z * b.y, ((a.w * b.y + a.y * b.w) + a.z * b.x) - a.x * b.z,
                ((a.w * b.z + a.z * b.w) + a.x * b.y) - a.y * b.x, ((a.w * b.w - a.x * b.x) - a.y * b.y) - a.z * b.z};
}
// Eigen 3.3.7 Quaternion::inverse(): zero when the squared norm is not > 0
inline Quat qinv(const Quat& a) {
    const double n2 = ((a.x * a.x + a.y * a.y) + a.z * a.z) + a.w * a.w;
    if (!(n2 > 0.0)) return Quat{0.0, 0.0, 0.0, 0.0};
    return Quat{-a.x / n2, -a.y / n2, -a.z / n2, a.w / n2};
}
// Eigen QuaternionBase::_transformVector: v + w * (2 q x v) + q x (2 q x v)
inline void qrot(const Quat& q, const double* v, double* o) {
    double ux = q.y * v[2] - q.z * v[1], uy = q.z * v[0] - q.x * v[2], uz = q.x * v[1] - q.y * v[0];
    ux += ux; uy += uy; uz += uz;
    o[0] = (v[0] + q.w * ux) + (q.y * uz - q.z * uy);
    o[1] = (v[1] + q.w * uy) + (q.z * ux - q.x * uz);
    o[2] = (v[2] + q.w * uz) + (q.x * uy - q.y * ux);
}

// lidar_distortion_corrector.cpp:19-34
inline bool ref_inverse(const ImuBuffer& b, Quat& q_ref_inv) {
    size_t l, r;
    if (!search_two(b, b.ref_time, l, r)) return false;
    const double ratio = double(b.ref_time - b.t[l]) / double(b.t[r] - b.t[l]);
    q_ref_inv = qinv(lerp(b.q[l], b.q[r], ratio));
    return true;
}
// lidar_distortion_corrector.cpp:37-64
inline bool process_point(const ImuBuffer& b, const Quat& q_ref_inv, float x, float y, float z, float rel_time, float* out) {
    const uint64_t t = b.ref_time + uint64_t(time_to_i64(double(rel_time) * 1.0e6));  // the int64 sum, in unsigned arithmetic
    size_t l, r;
    if (!search_two(b, t, l, r)) return false;
    const double ratio = double(t - b.t[l]) / double(b.t[r] - b.t[l]);
    const Quat qc = lerp(b.q[l], b.q[r], ratio);
    const double* T = b.T_li;  // column-major
    const double p[3] = {double(x), double(y), double(z)};
    const double pi[3] = {((T[0] * p[0] + T[4] * p[1]) + T[8] * p[2]) + T[12], ((T[1] * p[0] + T[5] * p[1]) + T[9] * p[2]) + T[13],
                          ((T[2] * p[0] + T[6] * p[1]) + T[10] * p[2]) + T[14]};
    double o[3];
    qrot(qmul(q_ref_inv, qc), pi, o);
    out[0] = float(o[0]);
    out[1] = float(o[1]);
    out[2] = float(o[2]);
    return true;
}

struct Preprocessed { Cloud ordered, planar; };
// preprocessing.cpp:181-225 (PointToPlane_IVOX / PointToPlane_KdTree / IcpOptimized / IncrementalNDT branch)
inline Preprocessed preprocess(const float* raw_xyzit, size_t n, const ImuBuffer* imu, float min_d, float max_d, int jump_span, float leaf) {
    Preprocessed out;
    Quat qri{0, 0, 0, 1};
    if (imu && !ref_inverse(*imu, qri)) return out;
    Cloud planar;
    for (size_t i = 0; i < n; ++i) {
        const float* p = raw_xyzit + 5 * i;
        float x = p[0], y = p[1], z = p[2];
        const float depth = std::sqrt(x * x + y * y + z * z);
        if (depth < min_d || depth > max_d) continue;
        if (imu) {
            float c[3];
            if (!process_point(*imu, qri, x, y, z, p[4], c)) continue;
            x = c[0]; y = c[1]; z = c[2];
        }
        const P4 q{x, y, z, p[3]};
        if (i % size_t(jump_span) == 0) planar.push_back(q);
        out.ordered.push_back(q);
    }
    out.planar = voxel_grid(planar, leaf);
    return out;
}

// pointcloud_projector.cpp:32-133 including the de-skew of :100-103 (a point whose time is outside the IMU buffer does not
// claim its cell); depth stays the range of the raw point (:57, :105)
inline Projected project_imu(const Cloud& raw, const std::vector<int>& ring, const float* time, const ImuBuffer* imu, int V, int H, float h_res,
                             float min_d, float max_d) {
    Projected out;
    const float FMAX = std::numeric_limits<float>::max();
    std::vector<float> range(size_t(V) * H, FMAX);
    std::vector<P4> tmp(size_t(V) * H);
    Quat qri{0, 0, 0, 1};
    const bool ok_ref = !imu || ref_inverse(*imu, qri);
    for (size_t k = 0; k < raw.size() && ok_ref; ++k) {
        const float x = raw[k].x, y = raw[k].y, z = raw[k].z;
        const float depth = std::sqrt(x * x + y * y + z * z);
        if (depth < min_d || depth > max_d) continue;
        const int row = ring[k];
        int colv = int(std::round(fast_atan2f(y, x) / h_res)) + H / 2;
        if (colv >= H) colv -= H;
        if (row >= V || row < 0 || colv < 0 || colv >= H) continue;
        const size_t index = size_t(row) * H + colv;
        if (range[index] != FMAX) continue;
        P4 q = raw[k];
        if (imu) {
            float c[3];
            if (!process_point(*imu, qri, x, y, z, time[k], c)) continue;
            q.x = c[0]; q.y = c[1]; q.z = c[2];
        }
        range[index] = depth;
        tmp[index] = q;
    }
    out.depth.resize(size_t(V) * H);
    out.col.assign(size_t(V) * H, 0);
    out.row_start.resize(V);
    out.row_end.resize(V);
    int count = 0;
    for (int row = 0; row < V; ++row) {
        out.row_start[row] = count + 5;
        for (int c = 0; c < H; ++c) {
            const size_t index = size_t(row) * H + c;
            if (range[index] == FMAX) continue;
            out.depth[count] = range[index];
            out.ordered.push_back(tmp[index]);
            out.col[count] = c;
            ++count;
        }
        out.row_end[row] = count - 6;
    }
    return out;
}

}  // namespace orc
