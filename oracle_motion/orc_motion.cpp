// C entries of the velocity-aware de-skew oracle (orc_motion.h) for oracle_motion/pyoracle_motion.py.  TEST INFRASTRUCTURE ONLY.
// Same argument layout as orc_preprocess / orc_project_imu of oracle/fls_oracle.cpp, plus the velocity (NULL: rotation only).
#include <cstring>

#include "orc_motion.h"

using namespace orc;

namespace {

ImuBuffer make_imu(const uint64_t* t, const double* q_xyzw, size_t m, uint64_t ref_time, const double* T_li) {
    ImuBuffer b;
    b.t.assign(t, t + m);
    b.q.resize(m);
    for (size_t i = 0; i < m; ++i) b.q[i] = Quat{q_xyzw[4 * i], q_xyzw[4 * i + 1], q_xyzw[4 * i + 2], q_xyzw[4 * i + 3]};
    b.ref_time = ref_time;
    std::memcpy(b.T_li, T_li, sizeof(b.T_li));
    return b;
}

}  // namespace

extern "C" {

// returns n_ordered; *n_planar set; outputs sized n (packed xyzi)
size_t orc_preprocess_motion(const float* raw_xyzit, size_t n, const uint64_t* imu_t, const double* imu_q, size_t m, uint64_t ref_time,
                             const double* T_li, const double* v, float min_d, float max_d, int jump_span, float leaf, float* ordered, float* planar,
                             size_t* n_planar) {
    ImuBuffer b;
    if (imu_t) b = make_imu(imu_t, imu_q, m, ref_time, T_li);
    const Preprocessed p = preprocess_motion(raw_xyzit, n, imu_t ? &b : nullptr, v, min_d, max_d, jump_span, leaf);
    std::memcpy(ordered, p.ordered.data(), p.ordered.size() * sizeof(P4));
    std::memcpy(planar, p.planar.data(), p.planar.size() * sizeof(P4));
    *n_planar = p.planar.size();
    return p.ordered.size();
}

// raw: n packed xyzi records; outputs sized V*H (ordered x4, depth, col) and V (row_start / row_end); returns n_ordered
size_t orc_project_imu_motion(const float* raw, const int* ring, const float* time, size_t n, const uint64_t* imu_t, const double* imu_q, size_t m,
                              uint64_t ref_time, const double* T_li, const double* v, int V, int H, float h_res, float min_d, float max_d,
                              float* ordered, float* depth, int* col, int* row_start, int* row_end) {
    Cloud c(n);
    for (size_t k = 0; k < n; ++k) c[k] = P4{raw[4 * k], raw[4 * k + 1], raw[4 * k + 2], raw[4 * k + 3]};
    std::vector<int> rg(ring, ring + n);
    ImuBuffer b;
    if (imu_t) b = make_imu(imu_t, imu_q, m, ref_time, T_li);
    const Projected p = project_imu_motion(c, rg, time, imu_t ? &b : nullptr, v, V, H, h_res, min_d, max_d);
    std::memcpy(ordered, p.ordered.data(), p.ordered.size() * sizeof(P4));
    std::memcpy(depth, p.depth.data(), p.depth.size() * sizeof(float));
    std::memcpy(col, p.col.data(), p.col.size() * sizeof(int));
    std::memcpy(row_start, p.row_start.data(), V * sizeof(int));
    std::memcpy(row_end, p.row_end.data(), V * sizeof(int));
    return p.ordered.size();
}

}  // extern "C"
