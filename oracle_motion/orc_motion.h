// orc_motion.h — CPU restatement (test infrastructure, see oracle/orc_math.h) of the de-skew with the sensor's translation that the
// *_motion entries of include/fls_b200.h add.  NOT UPSTREAM: LidarDistortionCorrector de-skews rotation only
// (src/lidar/lidar_distortion_corrector.cpp:34 ends SetRefTime with "TODO: add translation").  Under a constant body velocity v
// (IMU frame at ref_time) a kept point becomes
//     p_corr = q_ref^-1 q(t) (R_li p + t_li) + v * dt,   dt = double(t - ref_time as signed us) * 1e-6
// evaluated in fp64 in the device's order (fls_deskew.cuh) with -ffp-contract=off, then rounded to float.  The rotation part is
// oracle/orc_deskew.h's process_point, restated here only because that function rounds to float before the term can be added; the
// rotation-only oracle itself is left as it is.  v == nullptr (or all three components +-0) skips the term: the outputs are those of
// orc::preprocess / orc::project_imu bit for bit.
#pragma once
#include "../oracle/orc_deskew.h"

namespace orc {

inline bool moving(const double* v) { return v && (v[0] != 0.0 || v[1] != 0.0 || v[2] != 0.0); }

// process_point (lidar_distortion_corrector.cpp:37-64) + v * dt
inline bool process_point_motion(const ImuBuffer& b, const Quat& q_ref_inv, const double* v, float x, float y, float z, float rel_time, float* out) {
    const int64_t dt_us = time_to_i64(double(rel_time) * 1.0e6);
    const uint64_t t = b.ref_time + uint64_t(dt_us);
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
    if (moving(v)) {
        const double dt = double(dt_us) * 1.0e-6;
        for (int k = 0; k < 3; ++k) o[k] = o[k] + v[k] * dt;
    }
    out[0] = float(o[0]);
    out[1] = float(o[1]);
    out[2] = float(o[2]);
    return true;
}

// preprocess (preprocessing.cpp:181-225) with process_point_motion
inline Preprocessed preprocess_motion(const float* raw_xyzit, size_t n, const ImuBuffer* imu, const double* v, float min_d, float max_d, int jump_span,
                                      float leaf) {
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
            if (!process_point_motion(*imu, qri, v, x, y, z, p[4], c)) continue;
            x = c[0]; y = c[1]; z = c[2];
        }
        const P4 q{x, y, z, p[3]};
        if (i % size_t(jump_span) == 0) planar.push_back(q);
        out.ordered.push_back(q);
    }
    out.planar = voxel_grid(planar, leaf);
    return out;
}

// project_imu (pointcloud_projector.cpp:32-133) with process_point_motion; depth stays the range of the raw point (:57, :105)
inline Projected project_imu_motion(const Cloud& raw, const std::vector<int>& ring, const float* time, const ImuBuffer* imu, const double* v, int V,
                                     int H, float h_res, float min_d, float max_d) {
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
            if (!process_point_motion(*imu, qri, v, x, y, z, time[k], c)) continue;
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
