// b200_keyframe_map.h — header-only adapter that runs funny_lidar_slam's keyframe-map sites on libfls_b200.so's keyframe store.
//
// Drop this file next to b200_registration.h in the reference tree and link the package against libfls_b200.so and the CUDA runtime
// (INTEGRATION.md, "Keyframe maps").  It compiles only inside the reference's build (PCL point types, Eigen typedefs, glog, KeyFrame).
//
// One B200KeyFrameMap holds the ordered cloud of every keyframe on the device (fls_keyframes_*), fed where System creates keyframes
// (src/slam/system.cpp:648-662).  It replaces the CPU loops of
//   System::SaveMap            (src/slam/system.cpp:310-329)  -> SaveMap
//   System::VisualizeGlobalMap (src/slam/system.cpp:864-893)  -> GlobalMap::Round
//   LoopClosure::GetSubMap     (src/slam/loop_closure.cpp:188-230) -> GetSubMap
// and adds place recognition by Scan Context (fls_keyframes_detect_loop / _place_query):
//   LoopClosure::DetectByFeature (src/slam/loop_closure.cpp:120-122, a stub upstream) -> DetectLoopByFeature
//   the keyframe a scan was taken near, for Localization::Init without a clicked pose     -> PlaceQuery
// Each takes the keyframes (for their current pose_) under the caller's mutex_keyframes_, as upstream does.  The store serializes
// calls from the three threads itself.  Poses relative to a reference keyframe are computed here with the caller's Eigen
// (loop_closure.cpp:210-215), so the library receives final poses.
#ifndef FUNNY_LIDAR_SLAM_B200_KEYFRAME_MAP_H
#define FUNNY_LIDAR_SLAM_B200_KEYFRAME_MAP_H

#include <cuda_runtime_api.h>
#include <glog/logging.h>

#include <cstdint>
#include <string>
#include <vector>

#include "common/data_type.h"
#include "common/keyframe.h"
#include "fls_b200.h"

class B200KeyFrameMap {
public:
    // `capacity_points`: arena size in points, fixed (the store returns FLS_ERR_CAPACITY rather than grow on a shared GPU)
    B200KeyFrameMap(int device, size_t capacity_points) {
        const int rc = fls_keyframes_create(device, capacity_points, &store_);
        CHECK_EQ(rc, FLS_OK) << "fls_keyframes_create: " << fls_strerror(rc) << " " << fls_last_error();
    }
    ~B200KeyFrameMap() { fls_keyframes_destroy(store_); }
    B200KeyFrameMap(const B200KeyFrameMap&) = delete;
    B200KeyFrameMap& operator=(const B200KeyFrameMap&) = delete;

    // next to keyframes_.push_back(keyframe) (system.cpp:662): keyframe->cloud_cluster_ptr_->ordered_cloud_, id = keyframe->id_
    bool AddKeyFrame(KeyFrame::ID id, const PCLPointCloudXYZI& ordered_cloud) {
        const size_t n = ordered_cloud.points.size();
        if (!Ok(fls_keyframes_add(store_, id, ordered_cloud.points.data(), n, sizeof(PCLPointXYZI)), "fls_keyframes_add")) return false;
        sizes_.push_back(n);
        return true;
    }
    // the same from device memory, e.g. the ordered output of fls_preprocess_loam_device (packed float4 x, y, z, intensity)
    bool AddKeyFrameDevice(KeyFrame::ID id, const float* d_ordered, size_t n) {
        if (!Ok(fls_keyframes_add_device(store_, id, d_ordered, n), "fls_keyframes_add_device")) return false;
        sizes_.push_back(n);
        return true;
    }

    // System::SaveMap, system.cpp:310-329: every keyframe VoxelGridCloud(., 0.3f) and TransformPointCloud(., pose_), then
    // VoxelGridCloud(map, 0.3), written with savePCDFileBinary's format.  Returns the map size (res.map_size); 0: nothing written.
    size_t SaveMap(const std::vector<KeyFrame::Ptr>& keyframes, const std::string& map_path) {
        std::vector<int64_t> ids;
        std::vector<double> poses;
        for (const auto& keyframe : keyframes) {
            ids.push_back(keyframe->id_);
            poses.insert(poses.end(), keyframe->pose_.data(), keyframe->pose_.data() + 16);
        }
        std::vector<float> map;
        if (!Run(ids, poses, 0.3f, 0.3f, nullptr, 0, &map, nullptr, 0) || map.empty()) return 0;
        const int rc = fls_pcd_write(map_path.c_str(), map.data(), map.size() / 4);
        if (!Ok(rc, "fls_pcd_write")) return 0;
        return map.size() / 4;
    }

    // LoopClosure::GetSubMap, loop_closure.cpp:188-230: keyframes keyframe_id-left .. keyframe_id+right clipped to the range,
    // each VoxelGridCloud(., 0.2) and TransformPointCloud by its pose (relative to keyframe_id's with use_local_pose), concatenated.
    PCLPointCloudXYZI::Ptr GetSubMap(const std::vector<KeyFrame::Ptr>& keyframes, KeyFrame::ID keyframe_id, KeyFrame::ID left_range,
                                     KeyFrame::ID right_range, bool use_local_pose) {
        std::vector<int64_t> ids;
        std::vector<double> poses;
        const Mat4d ref_pose_inv = keyframes[keyframe_id]->pose_.inverse();
        for (int i = -left_range; i <= right_range; ++i) {
            const KeyFrame::ID k = keyframe_id + i;
            if (k < 0 || k >= static_cast<KeyFrame::ID>(keyframes.size())) continue;
            const Mat4d pose = use_local_pose ? Mat4d(ref_pose_inv * keyframes[k]->pose_) : keyframes[k]->pose_;
            ids.push_back(k);
            poses.insert(poses.end(), pose.data(), pose.data() + 16);
        }
        std::vector<float> map;
        Run(ids, poses, 0.2f, 0.f, nullptr, 0, &map, nullptr, 0);
        return ToCloud(map);
    }

    // Scan Context result: the candidate keyframe, its descriptor distance and the yaw that turns the query into its frame
    // (keyframe pose * Rz(yaw) is the query's coarse pose).  candidate_id stays invalid when there is none.
    struct PlaceMatch {
        KeyFrame::ID candidate_id = -1;  // KeyFrame::kInvalidID (include/common/keyframe.h:17)
        double distance = 1.0;
        double yaw = 0.0;
    };

    // LoopClosure::DetectByFeature: the best keyframe with curr_id - id > skip_near_keyframe_threshold (the span rule of
    // CheckCandidateKeyFrames, loop_closure.cpp:171).  The caller compares distance against its threshold and then takes the
    // GetSubMap path with std::make_pair(curr_id, candidate_id).
    PlaceMatch DetectLoopByFeature(KeyFrame::ID curr_id, KeyFrame::ID skip_near_keyframe_threshold) {
        fls_place_match m{};
        size_t n = 0;
        PlaceMatch r;
        if (Ok(fls_keyframes_detect_loop(store_, &sc_cfg_, curr_id, skip_near_keyframe_threshold, 1, &m, &n, nullptr), "fls_keyframes_detect_loop") &&
            n == 1)
            r = PlaceMatch{static_cast<KeyFrame::ID>(m.id), m.distance, m.yaw};
        return r;
    }

    // the stored keyframe nearest to a scan (its ordered cloud, sensor frame)
    PlaceMatch PlaceQuery(const PCLPointCloudXYZI& cloud) {
        fls_place_match m{};
        size_t n = 0;
        PlaceMatch r;
        if (Ok(fls_keyframes_place_query(store_, &sc_cfg_, cloud.points.data(), cloud.points.size(), sizeof(PCLPointXYZI), 1, &m, &n, nullptr,
                                         nullptr),
               "fls_keyframes_place_query") &&
            n == 1)
            r = PlaceMatch{static_cast<KeyFrame::ID>(m.id), m.distance, m.yaw};
        return r;
    }

    // the k stored keyframes nearest to a scan, best first (fewer when the store holds fewer): the guesses of a RelocalizeMulti
    std::vector<PlaceMatch> PlaceQuery(const PCLPointCloudXYZI& cloud, int k) {
        std::vector<fls_place_match> m(k > 0 ? (size_t)k : 0);
        size_t n = 0;
        std::vector<PlaceMatch> r;
        if (k > 0 && Ok(fls_keyframes_place_query(store_, &sc_cfg_, cloud.points.data(), cloud.points.size(), sizeof(PCLPointXYZI), (size_t)k, m.data(), &n,
                                                  nullptr, nullptr),
                        "fls_keyframes_place_query"))
            for (size_t i = 0; i < n; ++i) r.push_back(PlaceMatch{static_cast<KeyFrame::ID>(m[i].id), m[i].distance, m[i].yaw});
        return r;
    }

    // System::VisualizeGlobalMap's state (global_map, last_frame_id; system.cpp:851-852) with global_map kept on the device in two
    // buffers used in turn: one is the base of a round, the other receives its result.
    class GlobalMap {
    public:
        GlobalMap(B200KeyFrameMap& store, float voxel_filter_size) : store_(store), res_(voxel_filter_size) {}
        ~GlobalMap() {
            for (float* b : buf_)
                if (b) cudaFree(b);
        }
        GlobalMap(const GlobalMap&) = delete;
        GlobalMap& operator=(const GlobalMap&) = delete;

        // The loop body after the subscriber check (system.cpp:864-893).  `need_update`: need_update_global_map_visualization_
        // was set (the caller clears it).  Returns the cloud to publish, or nullptr where upstream `continue`s.
        PCLPointCloudXYZI::Ptr Round(const std::vector<KeyFrame::Ptr>& keyframes, bool need_update) {
            if (need_update) {
                n_ = 0;
                last_frame_id_ = -1;
            }
            if (keyframes.empty() || (last_frame_id_ + 1 >= keyframes.back()->id_)) return nullptr;
            std::vector<int64_t> ids;
            std::vector<double> poses;
            for (int i = last_frame_id_ + 1; i <= keyframes.back()->id_; ++i) {
                ids.push_back(i);
                poses.insert(poses.end(), keyframes[i]->pose_.data(), keyframes[i]->pose_.data() + 16);
            }
            const size_t cap = n_ + store_.UpperBound(ids);
            last_frame_id_ = keyframes.back()->id_;
            const int next = 1 - cur_;
            if (cap > cap_[next]) {
                if (buf_[next]) cudaFree(buf_[next]);
                buf_[next] = nullptr;
                cap_[next] = 0;
                void* p = nullptr;
                if (cudaMalloc(&p, cap * 16) != cudaSuccess) return nullptr;
                buf_[next] = static_cast<float*>(p);
                cap_[next] = cap;
            }
            std::vector<float> map;
            size_t n = 0;
            if (!store_.Run(ids, poses, res_, res_, buf_[cur_], n_, &map, buf_[next], cap_[next], &n)) return nullptr;
            cur_ = next;
            n_ = n;
            return ToCloud(map);
        }

    private:
        B200KeyFrameMap& store_;
        float res_;
        float* buf_[2] = {nullptr, nullptr};
        size_t cap_[2] = {0, 0};
        int cur_ = 0;
        size_t n_ = 0;
        KeyFrame::ID last_frame_id_ = -1;
    };

private:
    static bool Ok(int rc, const char* what) {
        if (rc == FLS_OK) return true;
        LOG(WARNING) << what << ": " << fls_strerror(rc) << " " << fls_last_error();
        return false;
    }

    static PCLPointCloudXYZI::Ptr ToCloud(const std::vector<float>& xyzi) {
        PCLPointCloudXYZI::Ptr cloud(new PCLPointCloudXYZI);
        cloud->points.resize(xyzi.size() / 4);
        for (size_t i = 0; i < cloud->points.size(); ++i) {
            cloud->points[i].x = xyzi[4 * i];
            cloud->points[i].y = xyzi[4 * i + 1];
            cloud->points[i].z = xyzi[4 * i + 2];
            cloud->points[i].intensity = xyzi[4 * i + 3];
        }
        cloud->width = static_cast<uint32_t>(cloud->points.size());
        cloud->height = 1;
        return cloud;
    }

    // records the map of `ids` can hold at most: a voxel filter never adds points
    size_t UpperBound(const std::vector<int64_t>& ids) const {
        size_t n = 0;
        for (const int64_t id : ids) n += id >= 0 && id < static_cast<int64_t>(sizes_.size()) ? sizes_[id] : 0;
        return n;
    }

    // the map into *out (host) and, when d_out is given, into d_out (d_cap records); *n_map receives its size
    bool Run(const std::vector<int64_t>& ids, const std::vector<double>& poses, float leaf, float final_leaf, const float* d_base, size_t n_base,
             std::vector<float>* out, float* d_out, size_t d_cap, size_t* n_map = nullptr) {
        const size_t cap = d_out ? d_cap : n_base + UpperBound(ids);
        out->resize(cap * 4);
        size_t n = 0;
        const int rc = fls_keyframes_assemble(store_, ids.data(), ids.size(), poses.data(), leaf, final_leaf, d_base, n_base, out->data(), d_out, cap,
                                              &n, nullptr);
        out->resize(rc == FLS_OK ? n * 4 : 0);
        if (n_map) *n_map = n;
        return Ok(rc, "fls_keyframes_assemble");
    }

    fls_keyframes* store_ = nullptr;
    std::vector<size_t> sizes_;  // records per keyframe id
    fls_sc_cfg sc_cfg_{20, 60, 80.f, 2.f};  // the paper's descriptor
};

#endif  // FUNNY_LIDAR_SLAM_B200_KEYFRAME_MAP_H
