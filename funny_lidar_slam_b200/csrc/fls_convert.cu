// fls_convert.cu — PreProcessing::ConvertMessageToCloud (src/slam/preprocessing.cpp:262-511 upstream) on the device, with
// ComputePointOffsetTime (:513-552), GetLidarPointMinMaxOffsetTime (:554-571) and the scan's start / end stamps (:86-104).
//
// The message's field table is matched on the host (pcl::fromROSMsg's rule: first field with the struct field's name, datatype and a
// count of 0 or 1; no match reads 0) and the kernels get byte offsets.  Kernels, in stream order, one wait at the end:
//   conv_flag     one thread per message point: the sensor's keep rule (NaN removal when not dense, the Avia line / tag filter, the
//                 ring window of None) and the first kept point (RoboSense / Mid-360 times are relative to its timestamp), one
//                 atomicMin per warp
//   (cub scan)    output positions: the compaction keeps the message order
//   conv_emit     xyzi, ring (uint8 casts) and time of every kept point, the count
// ComputePointOffsetTime, Velodyne and None only, gated on the device by the last kept point's time (<= 0):
//   off_prep      pinned atan2f yaw per point, sort key = ring (256 for skipped points)
//   (cub sort)    stable radix sort by ring: every ring's points in cloud order
//   off_heads     the first point of every ring: the head of its run in the sorted keys
//   off_map       per point a map on the 2-element state of time_last (DESIGN.md §3.8)
//   (cub scan)    composition of the maps: the state before every point
//   off_write     the offsets
//   conv_window   min / max time with the sequential loop's rules, the start / end stamps, the result record
#include <cub/cub.cuh>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>

#include "fls_atan.cuh"
#include "fls_frontend.h"

namespace fls {
namespace {

enum { F_X, F_Y, F_Z, F_I, F_RING, F_TIME, F_LINE, F_TAG, F_N };

struct ConvParams {
    const unsigned char* data;
    unsigned width, point_step, row_step;
    int n, type, dense, n_rows;
    float lower_angle, v_res;
    double scale;
    int off[F_N];  // byte offset of each struct field in a record, -1: no matching message field (reads 0)
};

// the struct field every sensor type reads, with its datatype (include/lidar/lidar_point_type.h:10-119; pcl::PointXYZI for None)
struct FieldSpec {
    const char* name;
    unsigned datatype;
};
void sensor_fields(int type, FieldSpec f[F_N]) {
    for (int k = 0; k < F_N; ++k) f[k] = {nullptr, 0};
    f[F_X] = {"x", FLS_PF_FLOAT32};
    f[F_Y] = {"y", FLS_PF_FLOAT32};
    f[F_Z] = {"z", FLS_PF_FLOAT32};
    f[F_I] = {"intensity", FLS_PF_FLOAT32};
    switch (type) {
        case FLS_LIDAR_VELODYNE:  // VelodynePointXYZIRT :45-61
            f[F_RING] = {"ring", FLS_PF_UINT16};
            f[F_TIME] = {"time", FLS_PF_FLOAT32};
            break;
        case FLS_LIDAR_OUSTER:  // OusterPointXYZIRT :63-82
            f[F_RING] = {"ring", FLS_PF_UINT8};
            f[F_TIME] = {"t", FLS_PF_UINT32};
            break;
        case FLS_LIDAR_ROBOSENSE:  // RsPointXYZIRT :10-24
        case FLS_LIDAR_LEISHEN:    // LsPointXYZIRT :26-43
            f[F_RING] = {"ring", FLS_PF_UINT16};
            f[F_TIME] = {"timestamp", FLS_PF_FLOAT64};
            break;
        case FLS_LIDAR_LIVOX_MID_360:  // LivoxMid360PointXYZITLT :84-101
            f[F_TIME] = {"timestamp", FLS_PF_FLOAT64};
            f[F_TAG] = {"tag", FLS_PF_UINT8};
            f[F_LINE] = {"line", FLS_PF_UINT8};
            break;
        case FLS_LIDAR_LIVOX_AVIA:  // LivoxPointXYZITLT :103-119
            f[F_TIME] = {"time", FLS_PF_UINT32};
            f[F_LINE] = {"line", FLS_PF_UINT8};
            f[F_TAG] = {"tag", FLS_PF_UINT8};
            break;
        default: break;  // None: pcl::PointXYZI
    }
}

__device__ __forceinline__ const unsigned char* record(const ConvParams& p, int k) {
    const unsigned r = (unsigned)k / p.width, c = (unsigned)k - r * p.width;
    return p.data + (size_t)r * p.row_step + (size_t)c * p.point_step;
}

// a field of any alignment; 0 when the message has no matching field
template <typename T>
__device__ __forceinline__ T ld(const unsigned char* rec, int off) {
    if (off < 0) return T(0);
    const unsigned char* q = rec + off;
    if (((uintptr_t)q & (sizeof(T) - 1)) == 0) return *reinterpret_cast<const T*>(q);
    T v;
    memcpy(&v, q, sizeof(T));
    return v;
}

__device__ __forceinline__ bool finite3(float x, float y, float z) { return isfinite(x) && isfinite(y) && isfinite(z); }

// the ring of a None point (:485-494): round((FastAtan2(z, xy) + lower_angle) / v_res), all in float; -1 outside [0, n_rows)
__device__ __forceinline__ int none_row(const ConvParams& p, float x, float y, float z) {
    const float xy = __fsqrt_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)));
    const int row = (int)roundf(__fdiv_rn(__fadd_rn(fast_atan2_ref(z, xy), p.lower_angle), p.v_res));
    return (row >= p.n_rows || row < 0) ? -1 : row;
}

// the sensor's keep rule for message point k
__device__ __forceinline__ bool keep_point(const ConvParams& p, int k) {
    const unsigned char* rec = record(p, k);
    const float x = ld<float>(rec, p.off[F_X]), y = ld<float>(rec, p.off[F_Y]), z = ld<float>(rec, p.off[F_Z]);
    if (p.type == FLS_LIDAR_LIVOX_AVIA) {  // :447-449, no NaN removal
        const unsigned line = ld<unsigned char>(rec, p.off[F_LINE]), tag = ld<unsigned char>(rec, p.off[F_TAG]) & 0x30u;
        return line < 6u && (tag == 0x10u || tag == 0x00u);
    }
    if (p.type == FLS_LIDAR_NONE) return finite3(x, y, z) && none_row(p, x, y, z) >= 0;  // :474-476, :491-492
    return p.dense || finite3(x, y, z);  // RemoveNaNFromPointCloud when the cloud is not dense (pointcloud_utility.h:227-260)
}

__global__ void conv_flag_kernel(ConvParams p, unsigned* __restrict__ flag, int* __restrict__ first_kept) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    const bool keep = k < p.n && keep_point(p, k);
    if (k < p.n) flag[k] = keep ? 1u : 0u;
    // the first kept point: one atomic per warp on the smallest kept index of the warp
    const int m = __reduce_min_sync(0xffffffffu, keep ? k : INT_MAX);
    if ((threadIdx.x & 31) == 0 && m != INT_MAX) atomicMin(first_kept, m);
}

__global__ void conv_emit_kernel(ConvParams p, const unsigned* __restrict__ flag, const unsigned* __restrict__ pos, const int* __restrict__ first_kept,
                                 float4* __restrict__ xyzi, int* __restrict__ ring, float* __restrict__ time, int* __restrict__ count) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= p.n) return;
    if (k == p.n - 1) *count = (int)(pos[k] + flag[k]);
    if (!flag[k]) return;
    const unsigned char* rec = record(p, k);
    const float x = ld<float>(rec, p.off[F_X]), y = ld<float>(rec, p.off[F_Y]), z = ld<float>(rec, p.off[F_Z]);
    const float in = ld<float>(rec, p.off[F_I]);
    int r = 0;
    float t = 0.f;
    switch (p.type) {
        case FLS_LIDAR_VELODYNE:  // :286-288
            r = ld<unsigned short>(rec, p.off[F_RING]) & 0xff;
            t = __double2float_rn(__dmul_rn((double)ld<float>(rec, p.off[F_TIME]), p.scale));
            break;
        case FLS_LIDAR_OUSTER:  // :323-325
            r = ld<unsigned char>(rec, p.off[F_RING]);
            t = __double2float_rn(__dmul_rn((double)ld<unsigned>(rec, p.off[F_TIME]), p.scale));
            break;
        case FLS_LIDAR_LEISHEN:  // :355-357
            r = ld<unsigned short>(rec, p.off[F_RING]) & 0xff;
            t = __double2float_rn(__dmul_rn(ld<double>(rec, p.off[F_TIME]), p.scale));
            break;
        case FLS_LIDAR_ROBOSENSE:       // :392-394
        case FLS_LIDAR_LIVOX_MID_360: {  // :424-427, ring 0
            if (p.type == FLS_LIDAR_ROBOSENSE) r = ld<unsigned short>(rec, p.off[F_RING]) & 0xff;
            const double ts0 = ld<double>(record(p, *first_kept), p.off[F_TIME]);
            t = __double2float_rn(__dmul_rn(__dsub_rn(ld<double>(rec, p.off[F_TIME]), ts0), p.scale));
            break;
        }
        case FLS_LIDAR_LIVOX_AVIA:  // :455-456, ring 0
            t = __double2float_rn(__dmul_rn((double)ld<unsigned>(rec, p.off[F_TIME]), p.scale));
            break;
        default:  // None: time 0, ring from elevation (:483-494)
            r = none_row(p, x, y, z) & 0xff;
            break;
    }
    const unsigned j = pos[k];
    xyzi[j] = make_float4(x, y, z, in);
    ring[j] = r;
    time[j] = t;
}

// ---- ComputePointOffsetTime --------------------------------------------------------------------------------------------------
// After point i of a ring, time_last is base_i or base_i + P (P = float(2 pi / omega)), base_i being the wrapped yaw offset of the
// point; the first point of a ring sets it to 0.  Point i's choice depends on the previous value only, so it is a map on a 2-element
// state {0: base_{i-1}, 1: base_{i-1} + P}: bit s of the map is the state after point i when the state before it is s.  The first
// point's map is constant 0, so an inclusive scan of the maps in ring-sorted order gives every point's state with no segment keys.

struct OffsetParams {
    double omega, two_pi;
    float period;
};

__device__ __forceinline__ float offset_base(const OffsetParams& q, double yaw_first, double yaw) {  // :540-544
    const double d = __dsub_rn(yaw_first, yaw);
    return __double2float_rn(__ddiv_rn(yaw <= yaw_first ? d : __dadd_rn(d, q.two_pi), q.omega));
}

__global__ void off_prep_kernel(const float4* __restrict__ xyzi, const int* __restrict__ ring, const float* __restrict__ time, const int* __restrict__ count,
                                int cap, int n_rows, float* __restrict__ yaw, unsigned short* __restrict__ key, int* __restrict__ idx,
                                int* __restrict__ go) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cap) return;
    const int n = *count;
    if (i == 0) go[0] = n > 0 && time[n - 1] <= 0.0f;  // :295, :502
    int r = 256;
    if (i < n && ring[i] < n_rows) {  // :526-529: a ring beyond the model keeps its time
        r = ring[i];
        const float4 p = xyzi[i];
        yaw[i] = atan2f_pinned(p.y, p.x);  // :531
    }
    key[i] = (unsigned short)r;
    idx[i] = i;
}

// the first point of every ring: the first element of its run in the stable ring sort (binary search; -1 for an absent ring)
__global__ void off_heads_kernel(const unsigned short* __restrict__ key, const int* __restrict__ idx, int cap, int* __restrict__ first) {
    const int r = threadIdx.x;
    int lo = 0, hi = cap;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (key[mid] < r) lo = mid + 1;
        else hi = mid;
    }
    first[r] = (lo < cap && key[lo] == r) ? idx[lo] : -1;
}

__global__ void off_map_kernel(OffsetParams q, const unsigned short* __restrict__ key, const int* __restrict__ idx, const float* __restrict__ yaw,
                               const int* __restrict__ first, int cap, unsigned char* __restrict__ map) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= cap) return;
    const int r = key[s];
    unsigned char m = 0;
    if (r < 256) {
        const int i = idx[s], f = first[r];
        if (i != f) {  // the first point of a ring: constant 0 (time_last = 0, :533-537)
            const double yf = yaw[f];
            const float b = offset_base(q, yf, yaw[i]);
            const int pi = idx[s - 1];  // same ring: the sort is stable and i is not the ring's first point
            float v0 = 0.f, v1 = 0.f;
            if (pi != f) {
                v0 = offset_base(q, yf, yaw[pi]);
                v1 = __fadd_rn(v0, q.period);
            }
            m = (unsigned char)((b < v0 ? 1 : 0) | (b < v1 ? 2 : 0));  // :546-548
        }
    }
    map[s] = m;
}

struct ComposeMaps {  // a then b
    __device__ __forceinline__ unsigned char operator()(unsigned char a, unsigned char b) const {
        return (unsigned char)(((b >> (a & 1)) & 1) | (((b >> ((a >> 1) & 1)) & 1) << 1));
    }
};

__global__ void off_write_kernel(OffsetParams q, const unsigned short* __restrict__ key, const int* __restrict__ idx, const float* __restrict__ yaw,
                                 const int* __restrict__ first, const unsigned char* __restrict__ state, const int* __restrict__ go, int cap,
                                 float* __restrict__ time) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= cap || !*go) return;
    const int r = key[s];
    if (r >= 256) return;
    const int i = idx[s], f = first[r];
    if (i == f) return;  // the first point keeps its time
    const float b = offset_base(q, yaw[f], yaw[i]);
    time[i] = (state[s] & 1) ? __fadd_rn(b, q.period) : b;
}

// ---- time window and stamps ------------------------------------------------------------------------------------------------
constexpr int kWinThreads = 1024;

// GetLidarPointMinMaxOffsetTime (:554-571): a NaN first time stays; otherwise the earliest point equal to the extreme (which decides the
// sign of a zero).  Each thread keeps (value, index) with that order, the block reduces; then :86-104.
__global__ void __launch_bounds__(kWinThreads) conv_window_kernel(ConvParams p, unsigned long long stamp, const float* __restrict__ time,
                                                                  const int* __restrict__ count, const int* __restrict__ first_kept,
                                                                  const int* __restrict__ go, fls_convert_result* __restrict__ res) {
    __shared__ float s_v[2][kWinThreads];
    __shared__ int s_i[2][kWinThreads];
    const int n = *count, tid = threadIdx.x;
    float mn = 0.f, mx = 0.f;
    int imn = -1, imx = -1;
    for (int i = tid; i < n; i += kWinThreads) {
        const float t = time[i];
        if (isnan(t)) continue;
        if (imn < 0 || t < mn) mn = t, imn = i;
        if (imx < 0 || t > mx) mx = t, imx = i;
    }
    s_v[0][tid] = mn, s_i[0][tid] = imn, s_v[1][tid] = mx, s_i[1][tid] = imx;
    __syncthreads();
    for (int h = kWinThreads / 2; h > 0; h >>= 1) {
        if (tid < h) {
            for (int w = 0; w < 2; ++w) {
                const int io = s_i[w][tid + h];
                if (io < 0) continue;
                const float vo = s_v[w][tid + h], v = s_v[w][tid];
                const int i = s_i[w][tid];
                const bool better = i < 0 || (w == 0 ? vo < v : vo > v) || (vo == v && io < i);
                if (better) s_v[w][tid] = vo, s_i[w][tid] = io;
            }
        }
        __syncthreads();
    }
    if (tid) return;
    fls_convert_result r;
    memset(&r, 0, sizeof(r));
    r.stamp_us = stamp;
    if (n > 0) {
        if (p.type == FLS_LIDAR_ROBOSENSE)  // :376
            r.stamp_us = __double2ull_rz(__dmul_rn(ld<double>(record(p, *first_kept), p.off[F_TIME]), 1.0e6));
        const float t0 = time[0];
        r.min_time = isnan(t0) ? t0 : s_v[0][0];
        r.max_time = isnan(t0) ? t0 : s_v[1][0];
        unsigned long long start = r.stamp_us + (unsigned long long)trunc_i64(__dmul_rn((double)r.min_time, 1.0e6));  // :90-97
        unsigned long long end = r.stamp_us + (unsigned long long)trunc_i64(__dmul_rn((double)r.max_time, 1.0e6));
        if (r.stamp_us < start) start = r.stamp_us;  // :100-104
        else if (r.stamp_us > end) end = r.stamp_us;
        r.start_us = start;
        r.end_us = end;
        r.valid = 1;
        r.recomputed = go ? *go : 0;
    }
    *res = r;
}

struct ConvWorkspace : Workspace {
    DevBuf<unsigned char> staging, cub_tmp, map, state;
    DevBuf<unsigned> flag, pos;
    DevBuf<int> small;  // [count][first_kept][go][first per ring: 256]
    DevBuf<float4> xyzi;
    DevBuf<int> ring, idx, idx_sorted;
    DevBuf<float> time, yaw;
    DevBuf<unsigned short> key, key_sorted;
    DevBuf<fls_convert_result> res;
    PinnedBuf<fls_convert_result> h_res;
    PinnedBuf<int> h_count;
};

}  // namespace

int convert_cloud_device(const fls_convert_cfg& c, const fls_pointcloud2& m, float* xyzi, int* ring, float* time, float* d_xyzi, int* d_ring,
                         float* d_time, size_t* n_out, fls_convert_result* res, fls_match_stats* stats) {
    // the field mapping of pcl::fromROSMsg, decided on the host from the small table
    ConvParams p;
    std::memset(&p, 0, sizeof(p));
    FieldSpec spec[F_N];
    sensor_fields(c.lidar_type, spec);
    for (int k = 0; k < F_N; ++k) {
        p.off[k] = -1;
        if (!spec[k].name) continue;
        for (uint32_t j = 0; j < m.n_fields; ++j) {
            const fls_point_field& f = m.fields[j];
            if (std::strcmp(f.name, spec[k].name) == 0 && f.datatype == spec[k].datatype && (f.count == 1 || f.count == 0)) {
                p.off[k] = (int)f.offset;
                break;
            }
        }
    }
    const size_t n = (size_t)m.width * m.height;
    p.width = m.width;
    p.point_step = m.point_step;
    p.row_step = m.row_step;
    p.n = (int)n;
    p.type = c.lidar_type;
    p.dense = m.is_dense == 1;  // pcl::fromPCLPointCloud2
    p.n_rows = c.n_rows;
    p.lower_angle = c.lower_angle;
    p.v_res = c.v_res;
    p.scale = c.time_scale;
    const bool offsets = c.lidar_type == FLS_LIDAR_VELODYNE || c.lidar_type == FLS_LIDAR_NONE;
    std::memset(res, 0, sizeof(*res));
    res->stamp_us = m.stamp_us;
    *n_out = 0;
    if (stats) std::memset(stats, 0, sizeof(*stats));
    if (n == 0) return FLS_OK;  // upstream reads points.back() of the empty cloud here (DESIGN.md §8)

    return with_workspace<ConvWorkspace>(c.device, [&](ConvWorkspace& w) -> int {
        Call& call = w.call;
        const cudaStream_t st = call.stream;
        fls_convert_result* const h_res = w.h_res.reserve(1);
        int* const h_count = w.h_count.reserve(1);
        call.begin();
        const size_t bytes = (size_t)m.height * m.row_step;
        if (m.data_on_device) {
            p.data = static_cast<const unsigned char*>(m.data);
        } else {
            w.staging.reserve(bytes + 1);
            FLS_CUDA(cudaMemcpyAsync(w.staging.p, m.data, bytes, cudaMemcpyHostToDevice, st));
            call.h2d += (long long)bytes;
            p.data = w.staging.p;
        }
        float4* ox = d_xyzi ? reinterpret_cast<float4*>(d_xyzi) : w.xyzi.reserve(n);
        int* orr = d_ring ? d_ring : w.ring.reserve(n);
        float* ot = d_time ? d_time : w.time.reserve(n);
        w.flag.reserve(n);
        w.pos.reserve(n);
        w.small.reserve(3 + 256);
        w.res.reserve(1);
        int* d_count = w.small.p;
        int* d_first_kept = w.small.p + 1;
        int* d_go = w.small.p + 2;
        int* d_first = w.small.p + 3;
        FLS_CUDA(cudaMemsetAsync(w.small.p, 0x7f, 3 * sizeof(int), st));  // the first kept point's minimum starts at 0x7f7f7f7f
        FLS_CUDA(cudaMemsetAsync(d_go, 0, sizeof(int), st));
        const unsigned g = (unsigned)((n + 255) / 256);
        conv_flag_kernel<<<g, 256, 0, st>>>(p, w.flag.p, d_first_kept);
        auto positions = [&](void* tmp, size_t& bytes) { return cub::DeviceScan::ExclusiveSum(tmp, bytes, w.flag.p, w.pos.p, (int)n, st); };
        auto sort = [&](void* tmp, size_t& bytes) {
            return cub::DeviceRadixSort::SortPairs(tmp, bytes, w.key.p, w.key_sorted.p, w.idx.p, w.idx_sorted.p, (int)n, 0, 9, st);
        };
        auto compose = [&](void* tmp, size_t& bytes) { return cub::DeviceScan::InclusiveScan(tmp, bytes, w.map.p, w.state.p, ComposeMaps(), (int)n, st); };
        if (offsets) {
            w.key.reserve(n);
            w.key_sorted.reserve(n);
            w.idx.reserve(n);
            w.idx_sorted.reserve(n);
            w.yaw.reserve(n);
            w.map.reserve(n);
            w.state.reserve(n);
            cub_reserve(w.cub_tmp, positions, sort, compose);
        } else {
            cub_reserve(w.cub_tmp, positions);
        }
        cub_run(w.cub_tmp, positions);
        conv_emit_kernel<<<g, 256, 0, st>>>(p, w.flag.p, w.pos.p, d_first_kept, ox, orr, ot, d_count);
        call.launches += 3;
        if (offsets) {  // ComputePointOffsetTime(cloud, 10.0): the kernels run, the last one writes only when the condition holds
            OffsetParams q;
            q.omega = 2.0 * M_PI * 10.0;  // :518
            q.two_pi = 2.0 * M_PI;
            q.period = static_cast<float>(2.0 * M_PI / q.omega);  // :547
            off_prep_kernel<<<g, 256, 0, st>>>(ox, orr, ot, d_count, (int)n, c.n_rows, w.yaw.p, w.key.p, w.idx.p, d_go);
            cub_run(w.cub_tmp, sort);
            off_heads_kernel<<<1, 256, 0, st>>>(w.key_sorted.p, w.idx_sorted.p, (int)n, d_first);
            off_map_kernel<<<g, 256, 0, st>>>(q, w.key_sorted.p, w.idx_sorted.p, w.yaw.p, d_first, (int)n, w.map.p);
            cub_run(w.cub_tmp, compose);
            off_write_kernel<<<g, 256, 0, st>>>(q, w.key_sorted.p, w.idx_sorted.p, w.yaw.p, d_first, w.state.p, d_go, (int)n, ot);
            call.launches += 6;
        }
        conv_window_kernel<<<1, kWinThreads, 0, st>>>(p, m.stamp_us, ot, d_count, d_first_kept, offsets ? d_go : nullptr, w.res.p);
        ++call.launches;
        FLS_CUDA(cudaGetLastError());
        // the host copies cover the capacity, so that the call waits once
        if (xyzi) FLS_CUDA(cudaMemcpyAsync(xyzi, ox, n * sizeof(float4), cudaMemcpyDeviceToHost, st));
        if (ring) FLS_CUDA(cudaMemcpyAsync(ring, orr, n * sizeof(int), cudaMemcpyDeviceToHost, st));
        if (time) FLS_CUDA(cudaMemcpyAsync(time, ot, n * sizeof(float), cudaMemcpyDeviceToHost, st));
        FLS_CUDA(cudaMemcpyAsync(h_count, d_count, sizeof(int), cudaMemcpyDeviceToHost, st));
        FLS_CUDA(cudaMemcpyAsync(h_res, w.res.p, sizeof(fls_convert_result), cudaMemcpyDeviceToHost, st));
        call.d2h += (long long)(n * ((xyzi ? 16 : 0) + (ring ? 4 : 0) + (time ? 4 : 0)) + sizeof(int) + sizeof(fls_convert_result));
        call.end(stats);  // the only wait
        const size_t cnt = (size_t)*h_count;
        *n_out = cnt;
        *res = *h_res;
        if (stats) {
            stats->n_source = (long long)n;
            // the message read once, the outputs written once; the offsets read xyzi + ring and rewrite the times
            stats->algo_bytes = (long long)(n * m.point_step + cnt * 24 + (res->recomputed ? cnt * 24 : 0));
        }
        return FLS_OK;
    });
}

}  // namespace fls
