// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle/orc_math.h).  The product (funny_lidar_slam_b200/) never links or calls this code.
//
// PreProcessing::ConvertMessageToCloud (src/slam/preprocessing.cpp:262-511), ComputePointOffsetTime (:513-552),
// GetLidarPointMinMaxOffsetTime (:554-571) and the start / end stamps of PreProcessing::Run (:86-104), restated sequentially on plain
// structs: pcl::fromROSMsg into the sensor's point type (include/lidar/lidar_point_type.h:10-119), the per-sensor loop, the offsets.
// Built with -ffp-contract=off so that every fp64 product and sum is rounded on its own, as the device's __dmul_rn / __dadd_rn are.
#pragma once
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <limits>
#include <vector>

#include "../include/fls_b200.h"
#include "../oracle/orc_math.h"

namespace orc {

// Conversions whose C++ result is undefined out of range, pinned: the x86-64 cvtt* result (INT_MIN / INT64_MIN) for the signed ones,
// saturation (NaN -> 0) for the unsigned one, as the device's __double2ull_rz does (DESIGN.md §8).
inline int orc_float_to_int(float v) { return (v >= -2147483648.0f && v < 2147483648.0f) ? (int)v : std::numeric_limits<int>::min(); }
inline int64_t orc_double_to_i64(double v) {
    return (v >= -9.2233720368547758e18 && v < 9.2233720368547758e18) ? (int64_t)v : std::numeric_limits<int64_t>::min();
}
inline uint64_t orc_double_to_u64(double v) {
    if (!(v > 0.0)) return 0;
    return v < 1.8446744073709552e19 ? (uint64_t)v : std::numeric_limits<uint64_t>::max();
}

// ---- std::atan2(float, float), pinned -------------------------------------------------------------------------------------
// atan2f from fp64 octant reduction and fdlibm's atan on [0, 1] (s_atan.c), error below about 2 ulp of fp64 before one rounding to
// float: correctly rounded except within a few fp64 ulps of a float rounding boundary, and on every pair tested.  No libm call:
// glibc's atan2f is not correctly rounded on every version (DESIGN.md §5).  The device's atan2f_pinned (fls_atan.cuh) evaluates the
// same operations, so the two agree bit for bit.
inline double atan01_pinned(double t) {
    static const double atanhi[2] = {4.63647609000806093515e-01, 7.85398163397448278999e-01};
    static const double atanlo[2] = {2.26987774529616870924e-17, 3.06161699786838301793e-17};
    static const double aT[11] = {3.33333333333329318027e-01,  -1.99999999998764832476e-01, 1.42857142725034663711e-01,
                                  -1.11111104054623557880e-01, 9.09088713343650656196e-02,  -7.69187620504482999495e-02,
                                  6.66107313738753120669e-02,  -5.83357013379057348645e-02, 4.97687799461593236017e-02,
                                  -3.65315727442169155270e-02, 1.62858201153657823623e-02};
    int id;
    if (t < 0.4375) {
        if (t < 7.450580596923828125e-09) return t;  // 2^-27
        id = -1;
    } else if (t < 0.6875) {
        id = 0;
        t = (2.0 * t - 1.0) / (2.0 + t);
    } else {
        id = 1;
        t = (t - 1.0) / (t + 1.0);
    }
    const double z = t * t, w = z * z;
    const double s1 = z * (aT[0] + w * (aT[2] + w * (aT[4] + w * (aT[6] + w * (aT[8] + w * aT[10])))));
    const double s2 = w * (aT[1] + w * (aT[3] + w * (aT[5] + w * (aT[7] + w * aT[9]))));
    if (id < 0) return t - t * (s1 + s2);
    return atanhi[id] - ((t * (s1 + s2) - atanlo[id]) - t);
}

inline float atan2f_pinned(float y, float x) {
    const double pio2_hi = 1.57079632679489655800e+00, pio2_lo = 6.12323399573676603587e-17;
    const double pi_hi = 3.14159265358979311600e+00, pi_lo = 1.22464679914735317720e-16;
    if (std::isnan(x) || std::isnan(y)) return x + y;
    const double ax = std::fabs((double)x), ay = std::fabs((double)y);
    const bool neg_x = std::signbit(x);
    double a;
    if (ax == 0.0 && ay == 0.0) {
        a = neg_x ? pi_hi : 0.0;
    } else if (std::isinf(ax) && std::isinf(ay)) {
        a = neg_x ? 2.35619449019234483700e+00 : 7.85398163397448278999e-01;
    } else {
        const bool swap = ay > ax;
        a = atan01_pinned(swap ? ax / ay : ay / ax);
        if (swap) a = pio2_hi - (a - pio2_lo);
        if (neg_x) a = pi_hi - (a - pi_lo);
    }
    const float r = (float)a;
    return std::signbit(y) ? -r : r;
}

// ---- pcl::fromROSMsg ---------------------------------------------------------------------------------------------------------
// The point types' fields (lidar_point_type.h).  A struct field reads the first message field with its name, its datatype and a count
// of 0 or 1 (pcl::FieldMatches); without one it keeps its value-initialised 0.
struct RawPoint {  // the union of the fields the seven types have
    float x = 0, y = 0, z = 0, intensity = 0;
    uint16_t ring16 = 0;
    uint8_t ring8 = 0;
    float time_f = 0;
    uint32_t time_u = 0;
    double timestamp = 0;
    uint8_t line = 0, tag = 0;
};

struct FieldReader {
    const char* name;
    uint32_t datatype;
    size_t member_offset;
    size_t size;
    long src = -1;
};

inline std::vector<FieldReader> point_type_fields(int type) {
    std::vector<FieldReader> f = {{"x", FLS_PF_FLOAT32, offsetof(RawPoint, x), 4},
                                  {"y", FLS_PF_FLOAT32, offsetof(RawPoint, y), 4},
                                  {"z", FLS_PF_FLOAT32, offsetof(RawPoint, z), 4},
                                  {"intensity", FLS_PF_FLOAT32, offsetof(RawPoint, intensity), 4}};
    switch (type) {
        case FLS_LIDAR_VELODYNE:  // VelodynePointXYZIRT :45-61
            f.push_back({"ring", FLS_PF_UINT16, offsetof(RawPoint, ring16), 2});
            f.push_back({"time", FLS_PF_FLOAT32, offsetof(RawPoint, time_f), 4});
            break;
        case FLS_LIDAR_OUSTER:  // OusterPointXYZIRT :63-82 (reflectivity, noise, range are not read)
            f.push_back({"t", FLS_PF_UINT32, offsetof(RawPoint, time_u), 4});
            f.push_back({"ring", FLS_PF_UINT8, offsetof(RawPoint, ring8), 1});
            break;
        case FLS_LIDAR_ROBOSENSE:  // RsPointXYZIRT :10-24
        case FLS_LIDAR_LEISHEN:    // LsPointXYZIRT :26-43
            f.push_back({"ring", FLS_PF_UINT16, offsetof(RawPoint, ring16), 2});
            f.push_back({"timestamp", FLS_PF_FLOAT64, offsetof(RawPoint, timestamp), 8});
            break;
        case FLS_LIDAR_LIVOX_MID_360:  // LivoxMid360PointXYZITLT :84-101
            f.push_back({"tag", FLS_PF_UINT8, offsetof(RawPoint, tag), 1});
            f.push_back({"line", FLS_PF_UINT8, offsetof(RawPoint, line), 1});
            f.push_back({"timestamp", FLS_PF_FLOAT64, offsetof(RawPoint, timestamp), 8});
            break;
        case FLS_LIDAR_LIVOX_AVIA:  // LivoxPointXYZITLT :103-119
            f.push_back({"time", FLS_PF_UINT32, offsetof(RawPoint, time_u), 4});
            f.push_back({"line", FLS_PF_UINT8, offsetof(RawPoint, line), 1});
            f.push_back({"tag", FLS_PF_UINT8, offsetof(RawPoint, tag), 1});
            break;
        default: break;  // None: pcl::PointXYZI
    }
    return f;
}

struct RawCloud {
    std::vector<RawPoint> points;
    uint64_t stamp = 0;
    bool is_dense = true;
};

inline RawCloud from_ros_msg(const fls_pointcloud2& m, const unsigned char* data, int type) {
    std::vector<FieldReader> f = point_type_fields(type);
    for (auto& r : f)
        for (uint32_t j = 0; j < m.n_fields; ++j) {
            const fls_point_field& mf = m.fields[j];
            if (std::strcmp(mf.name, r.name) == 0 && mf.datatype == r.datatype && (mf.count == 1 || mf.count == 0)) {
                r.src = mf.offset;
                break;
            }
        }
    RawCloud c;
    c.stamp = m.stamp_us;
    c.is_dense = m.is_dense == 1;
    c.points.resize((size_t)m.width * m.height);
    for (uint32_t row = 0; row < m.height; ++row)
        for (uint32_t col = 0; col < m.width; ++col) {
            const unsigned char* rec = data + (size_t)row * m.row_step + (size_t)col * m.point_step;
            RawPoint& p = c.points[(size_t)row * m.width + col];
            for (const auto& r : f)
                if (r.src >= 0) std::memcpy(reinterpret_cast<unsigned char*>(&p) + r.member_offset, rec + r.src, r.size);
        }
    return c;
}

// RemoveNaNFromPointCloud (include/common/pointcloud_utility.h:227-260): order-preserving, only when not dense
inline void remove_nan(RawCloud& c) {
    if (c.is_dense) return;
    size_t j = 0;
    for (size_t i = 0; i < c.points.size(); ++i) {
        const RawPoint& p = c.points[i];
        if (!std::isfinite(p.x) || !std::isfinite(p.y) || !std::isfinite(p.z)) continue;
        c.points[j++] = p;
    }
    c.points.resize(j);
    c.is_dense = true;
}

// PointXYZIRT (lidar_point_type.h:121-137)
struct PointXYZIRT {
    float x = 0, y = 0, z = 0, intensity = 0;
    uint8_t ring = 0;
    float time = 0;
};
struct CloudXYZIRT {
    std::vector<PointXYZIRT> points;
    uint64_t stamp = 0;
};

struct ConvertConfig {
    int type;
    int n_rows;          // vertical_scan_num_
    float lower_angle;   // lower_angle_
    float v_res;         // v_res_
    double time_scale;   // lidar_point_time_scale_
};

// ComputePointOffsetTime (:513-552)
inline void compute_point_offset_time(CloudXYZIRT& cloud, const ConvertConfig& cfg, double lidar_rate) {
    const int lidar_scan_num = cfg.n_rows;
    const size_t cloud_size = cloud.points.size();
    const double lidar_omega = 2.0 * M_PI * lidar_rate;
    std::vector<bool> is_first(lidar_scan_num, true);
    std::vector<double> yaw_first_scan(lidar_scan_num, 0.0);
    std::vector<float> time_last(lidar_scan_num, 0.0f);
    for (size_t i = 0; i < cloud_size; i++) {
        const int ring = cloud.points[i].ring;
        if (ring >= lidar_scan_num) continue;
        const double yaw = atan2f_pinned(cloud.points[i].y, cloud.points[i].x);  // std::atan2(float, float) at :531
        if (is_first[ring]) {
            yaw_first_scan[ring] = yaw;
            is_first[ring] = false;
            time_last[ring] = 0.0f;
            continue;
        }
        if (yaw <= yaw_first_scan[ring]) {
            cloud.points[i].time = static_cast<float>((yaw_first_scan[ring] - yaw) / lidar_omega);
        } else {
            cloud.points[i].time = static_cast<float>((yaw_first_scan[ring] - yaw + 2.0 * M_PI) / lidar_omega);
        }
        if (cloud.points[i].time < time_last[ring]) cloud.points[i].time += static_cast<float>(2.0 * M_PI / lidar_omega);
        time_last[ring] = cloud.points[i].time;
    }
}

// ConvertMessageToCloud (:262-511).  Returns false for an empty result (upstream reads points.back() / cloud_rs[0] of it).
inline bool convert_message_to_cloud(const fls_pointcloud2& m, const unsigned char* data, const ConvertConfig& cfg, CloudXYZIRT& out,
                                     bool& recomputed) {
    recomputed = false;
    RawCloud c = from_ros_msg(m, data, cfg.type);
    out.points.clear();
    out.stamp = c.stamp;
    const double scale = cfg.time_scale;
    switch (cfg.type) {
        case FLS_LIDAR_VELODYNE:
        case FLS_LIDAR_OUSTER:
        case FLS_LIDAR_LEISHEN:
        case FLS_LIDAR_ROBOSENSE:
        case FLS_LIDAR_LIVOX_MID_360: {
            remove_nan(c);
            if (c.points.empty()) return false;
            const double ts0 = c.points[0].timestamp;
            if (cfg.type == FLS_LIDAR_ROBOSENSE) out.stamp = orc_double_to_u64(ts0 * 1.0e6);  // :376
            out.points.resize(c.points.size());
            for (size_t i = 0; i < c.points.size(); ++i) {
                const RawPoint& s = c.points[i];
                PointXYZIRT p;
                p.x = s.x, p.y = s.y, p.z = s.z, p.intensity = s.intensity;
                switch (cfg.type) {
                    case FLS_LIDAR_VELODYNE:  // :282-288
                        p.ring = static_cast<uint8_t>(s.ring16);
                        p.time = static_cast<float>(s.time_f * scale);
                        break;
                    case FLS_LIDAR_OUSTER:  // :319-325
                        p.ring = static_cast<uint8_t>(s.ring8);
                        p.time = static_cast<float>(s.time_u * scale);
                        break;
                    case FLS_LIDAR_LEISHEN:  // :351-357
                        p.ring = static_cast<uint8_t>(s.ring16);
                        p.time = static_cast<float>(s.timestamp * scale);
                        break;
                    case FLS_LIDAR_ROBOSENSE:  // :388-394
                        p.ring = static_cast<uint8_t>(s.ring16);
                        p.time = static_cast<float>((s.timestamp - ts0) * scale);
                        break;
                    default:  // Mid-360 :420-427
                        p.ring = 0;
                        p.time = static_cast<float>((s.timestamp - ts0) * scale);
                        break;
                }
                out.points[i] = p;
            }
            if (cfg.type == FLS_LIDAR_VELODYNE && out.points.back().time <= 0.0f) {  // :295-298
                compute_point_offset_time(out, cfg, 10.0);
                recomputed = true;
            }
            return true;
        }
        case FLS_LIDAR_LIVOX_AVIA: {  // :436-464
            const uint8_t num_scans = 6;
            for (const RawPoint& s : c.points) {
                if ((s.line < num_scans) && ((s.tag & 0x30) == 0x10 || (s.tag & 0x30) == 0x00)) {
                    PointXYZIRT p;
                    p.x = s.x, p.y = s.y, p.z = s.z, p.intensity = s.intensity;
                    p.time = static_cast<float>(static_cast<double>(s.time_u) * scale);
                    out.points.push_back(p);
                }
            }
            return !out.points.empty();
        }
        default: {  // None :466-506
            for (const RawPoint& s : c.points) {
                if (!std::isfinite(s.x) || !std::isfinite(s.y) || !std::isfinite(s.z)) continue;
                PointXYZIRT p;
                p.x = s.x, p.y = s.y, p.z = s.z, p.intensity = s.intensity;
                p.time = 0.0;
                const float xy = std::sqrt(s.x * s.x + s.y * s.y);
                const int row = orc_float_to_int(std::round((fast_atan2f(s.z, xy) + cfg.lower_angle) / cfg.v_res));
                if (row >= cfg.n_rows || row < 0) continue;
                p.ring = static_cast<uint8_t>(row);
                out.points.push_back(p);
            }
            if (out.points.empty()) return false;
            if (out.points.back().time <= 0.0f) {
                compute_point_offset_time(out, cfg, 10.0);
                recomputed = true;
            }
            return true;
        }
    }
}

// GetLidarPointMinMaxOffsetTime (:554-571)
inline void min_max_offset_time(const CloudXYZIRT& cloud, float& mn, float& mx) {
    mn = cloud.points[0].time;
    mx = cloud.points[0].time;
    for (const auto& point : cloud.points) {
        if (point.time < mn) mn = point.time;
        if (point.time > mx) mx = point.time;
    }
}

// the start / end stamps of PreProcessing::Run (:90-104); static_cast<int64_t>(float * 1.0e6) with x86-64's cvttsd2si result
// (INT64_MIN) for NaN and out-of-range products
inline void cloud_window(uint64_t stamp, float mn, float mx, uint64_t& start, uint64_t& end) {
    start = stamp + static_cast<uint64_t>(orc_double_to_i64(mn * 1.0e6));  // the int64 sum, in unsigned arithmetic
    end = stamp + static_cast<uint64_t>(orc_double_to_i64(mx * 1.0e6));
    if (stamp < start) {
        start = stamp;
    } else if (stamp > end) {
        end = stamp;
    }
}

}  // namespace orc
