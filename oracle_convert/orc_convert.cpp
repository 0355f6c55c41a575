// C entries of the conversion oracle (orc_convert.h) for oracle_convert/pyoracle_convert.py.  TEST INFRASTRUCTURE ONLY.
#include "orc_convert.h"

extern "C" {

float orc_atan2f_pinned(float y, float x) { return orc::atan2f_pinned(y, x); }

void orc_atan2f_pinned_batch(const float* y, const float* x, size_t n, float* out) {
    for (size_t i = 0; i < n; ++i) out[i] = orc::atan2f_pinned(y[i], x[i]);
}

// ConvertMessageToCloud + GetLidarPointMinMaxOffsetTime + the stamps, as fls_convert_cloud reports them (fls_b200.h).  `data` is the
// message's host bytes; xyzi / ring / time need width * height entries.
int orc_convert_cloud(const fls_convert_cfg* cfg, const fls_pointcloud2* msg, float* xyzi, int32_t* ring, float* time, size_t* n,
                      fls_convert_result* res) {
    orc::ConvertConfig c{cfg->lidar_type, cfg->n_rows, cfg->lower_angle, cfg->v_res, cfg->time_scale};
    orc::CloudXYZIRT cloud;
    bool recomputed = false;
    std::memset(res, 0, sizeof(*res));
    res->stamp_us = msg->stamp_us;
    *n = 0;
    if ((size_t)msg->width * msg->height == 0) return 0;
    if (!orc::convert_message_to_cloud(*msg, static_cast<const unsigned char*>(msg->data), c, cloud, recomputed)) return 0;
    for (size_t i = 0; i < cloud.points.size(); ++i) {
        const orc::PointXYZIRT& p = cloud.points[i];
        xyzi[4 * i] = p.x, xyzi[4 * i + 1] = p.y, xyzi[4 * i + 2] = p.z, xyzi[4 * i + 3] = p.intensity;
        ring[i] = p.ring;
        time[i] = p.time;
    }
    *n = cloud.points.size();
    float mn, mx;
    orc::min_max_offset_time(cloud, mn, mx);
    uint64_t start, end;
    orc::cloud_window(cloud.stamp, mn, mx, start, end);
    res->stamp_us = cloud.stamp;
    res->start_us = start;
    res->end_us = end;
    res->min_time = mn;
    res->max_time = mx;
    res->valid = 1;
    res->recomputed = recomputed ? 1 : 0;
    return 0;
}

}  // extern "C"
