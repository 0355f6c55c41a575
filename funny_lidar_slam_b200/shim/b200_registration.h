// b200_registration.h — header-only adapter that plugs libfls_b200.so into funny_lidar_slam.
//
// Drop this file into the reference tree (e.g. include/registration/b200_registration.h), add
// `include/fls_b200.h` next to it and link the package against libfls_b200.so (INTEGRATION.md shows the three-line
// CMake change and the factory branches).  It compiles only inside the reference's build (it needs the reference's
// own headers: PCL point types, Eigen typedefs, glog); nothing in this repository compiles it.
//
// It derives from the reference's plug-in interface
//     class RegistrationInterface { Match, AddCloudToLocalMap, GetFitnessScore }
//     (include/registration/registration_interface.h:11-20 upstream)
// and forwards each virtual to one C-ABI call.  pcl::PointXYZI is a 32-byte record with x,y,z at byte 0 and
// intensity at byte 16 — exactly FLS_LAYOUT_PCL_XYZI — so clouds are handed over without repacking, and Mat4d is
// Eigen column-major, the pose layout of the ABI.
#ifndef FUNNY_LIDAR_SLAM_B200_REGISTRATION_H
#define FUNNY_LIDAR_SLAM_B200_REGISTRATION_H

#include <glog/logging.h>

#include <algorithm>
#include <limits>
#include <memory>
#include <string>
#include <vector>

#include "common/constant_variable.h"
#include "common/data_type.h"
#include "fls_b200.h"
#include "registration/registration_interface.h"

class B200Registration final : public RegistrationInterface {
public:
    // `cfg` carries the same constructor arguments the five CPU plug-ins take (fls_config_default() fills the shipped
    // YAML defaults); construction failures abort like the reference's CHECK()s do.
    explicit B200Registration(const fls_config& cfg) {
        const int rc = fls_create(&cfg, &handle_);
        CHECK_EQ(rc, FLS_OK) << "fls_create: " << fls_strerror(rc) << " " << fls_last_error();
        method_ = cfg.method;
    }

    ~B200Registration() override { fls_destroy(handle_); }

    B200Registration(const B200Registration&) = delete;
    B200Registration& operator=(const B200Registration&) = delete;

    // registration_interface.h:13 — T is in/out and is written even when false is returned
    bool Match(const PointcloudClusterPtr& source_cloud_cluster, Mat4d& T) override {
        const auto& ordered = source_cloud_cluster->ordered_cloud_.points;
        const auto& planar = source_cloud_cluster->planar_cloud_.points;
        const auto& corner = source_cloud_cluster->corner_cloud_.points;
        int converged = 0;
        fls_match_stats stats;
        const int rc = fls_match(handle_, ordered.data(), ordered.size(), planar.data(), planar.size(), corner.data(), corner.size(),
                                 sizeof(PCLPointXYZI), T.data(), &converged, &stats);
        if (rc != FLS_OK) {
            // the reference's only runtime failure signal is `return false` (frontend.cpp:208-210 drops the scan)
            LOG(WARNING) << "fls_match: " << fls_strerror(rc) << " " << fls_last_error();
            return false;
        }
        DLOG(INFO) << "B200 Match iters=" << stats.iterations << " valid=" << stats.n_valid << " gpu_ms=" << stats.gpu_ms;
        return converged != 0;
    }

    // registration_interface.h:17
    void AddCloudToLocalMap(const std::initializer_list<PCLPointCloudXYZI>& cloud_list) override {
        std::vector<const void*> ptrs;
        std::vector<size_t> sizes;
        for (const auto& c : cloud_list) {
            ptrs.push_back(c.points.data());
            sizes.push_back(c.points.size());
        }
        const int rc = fls_add_cloud(handle_, static_cast<int>(ptrs.size()), ptrs.data(), sizes.data(), sizeof(PCLPointXYZI));
        CHECK_EQ(rc, FLS_OK) << "fls_add_cloud: " << fls_strerror(rc) << " " << fls_last_error();
    }

    // registration_interface.h:19
    [[nodiscard]] float GetFitnessScore(float max_range) const override {
        float score = std::numeric_limits<float>::max();
        const int rc = fls_fitness(handle_, max_range, &score);
        if (rc != FLS_OK) return FloatNaN;
        return score;
    }

    // The information matrix of the last Match at the pose it returned (needs FLS_FLAG_INFORMATION in the config): H (a Mat6d) in the
    // order [rotation; position] of lidar_pose_info_, for EdgeRotation's right perturbation R * Exp(dθ) and p + dp; g (a Vec6d),
    // n_valid and sum_residual optional.  false when the last Match left no record.  Scaling H to a covariance is the integrator's
    // choice.  A template so that the adapter needs no Eigen type until it is used.
    template <class Mat6, class Vec6 = Mat6>
    bool GetPoseInformation(Mat6& H, Vec6* g = nullptr, int64_t* n_valid = nullptr, double* sum_residual = nullptr) const {
        fls_information rec;
        if (fls_get_information(handle_, &rec) != FLS_OK || !rec.valid) return false;
        for (int r = 0; r < 6; ++r)
            for (int c = 0; c < 6; ++c) H(r, c) = rec.H[r * 6 + c];
        if (g)
            for (int r = 0; r < 6; ++r) (*g)(r) = rec.g[r];
        if (n_valid) *n_valid = rec.n_valid;
        if (sum_residual) *sum_residual = rec.sum_residual;
        return true;
    }

    // Localization::Init from the RViz "2D Pose Estimate" (localization.cpp:114-169): searches an x-y-yaw grid around T, refines the
    // best poses and picks one by Init's own rule.  T receives the chosen pose (also when false is returned, as upstream writes it);
    // *fitness its GetFitnessScore(cfg.max_range).  Returns whether it is accepted (converged and fitness < cfg.accept_fitness).
    // PointToPlane_IVOX and IncrementalNDT in localization mode, after fls_update_local_map at the guess.
    bool Relocalize(const PointcloudClusterPtr& source_cloud_cluster, Mat4d& T, const fls_reloc_cfg& cfg, float* fitness) {
        const auto& cloud = method_ == FLS_NDT ? source_cloud_cluster->ordered_cloud_.points : source_cloud_cluster->planar_cloud_.points;
        fls_reloc_result res;
        const int rc = fls_relocalize(handle_, cloud.data(), cloud.size(), sizeof(PCLPointXYZI), &cfg, T.data(), &res, nullptr, nullptr, nullptr,
                                      nullptr, nullptr, 0);
        if (fitness) *fitness = rc == FLS_OK ? res.fitness : FloatNaN;
        if (rc != FLS_OK) {
            LOG(WARNING) << "fls_relocalize: " << fls_strerror(rc) << " " << fls_last_error();
            return false;
        }
        DLOG(INFO) << "B200 Relocalize hypotheses=" << res.n_hypotheses << " rank=" << res.best_rank << " fitness=" << res.fitness;
        return res.accepted != 0;
    }

    // Relocalize over a whole local map (fls_relocalize_wide): the same grid and the same result without the 2^20 hypothesis cap,
    // searched by exact branch and bound; for a click tens of metres or any angle off.
    bool RelocalizeWide(const PointcloudClusterPtr& source_cloud_cluster, Mat4d& T, const fls_reloc_cfg& cfg, float* fitness) {
        const auto& cloud = method_ == FLS_NDT ? source_cloud_cluster->ordered_cloud_.points : source_cloud_cluster->planar_cloud_.points;
        fls_reloc_result res;
        int64_t evaluations = 0;
        const int rc = fls_relocalize_wide(handle_, cloud.data(), cloud.size(), sizeof(PCLPointXYZI), &cfg, T.data(), &res, nullptr, nullptr, nullptr,
                                           nullptr, &evaluations);
        if (fitness) *fitness = rc == FLS_OK ? res.fitness : FloatNaN;
        if (rc != FLS_OK) {
            LOG(WARNING) << "fls_relocalize_wide: " << fls_strerror(rc) << " " << fls_last_error();
            return false;
        }
        DLOG(INFO) << "B200 RelocalizeWide hypotheses=" << res.n_hypotheses << " evaluations=" << evaluations << " fitness=" << res.fitness;
        return res.accepted != 0;
    }

    // Relocalize from several coarse poses in one search (fls_relocalize_multi): the grids of up to 64 guesses, e.g. place_pose of each
    // of KeyFrameMap::PlaceQuery's top-k candidates, ranked together and the best refined by one batch Match.  T receives the chosen
    // pose (also when false is returned); guesses are not modified.
    bool RelocalizeMulti(const PointcloudClusterPtr& source_cloud_cluster, const std::vector<Mat4d>& guesses, Mat4d& T, const fls_reloc_cfg& cfg,
                         float* fitness) {
        const auto& cloud = method_ == FLS_NDT ? source_cloud_cluster->ordered_cloud_.points : source_cloud_cluster->planar_cloud_.points;
        std::vector<double> g(16 * guesses.size());
        for (size_t k = 0; k < guesses.size(); ++k) std::copy(guesses[k].data(), guesses[k].data() + 16, g.data() + 16 * k);
        fls_reloc_result res;
        int64_t evaluations = 0;
        const int rc = fls_relocalize_multi(handle_, cloud.data(), cloud.size(), sizeof(PCLPointXYZI), &cfg, g.data(), (int32_t)guesses.size(), T.data(),
                                            &res, nullptr, nullptr, nullptr, nullptr, &evaluations);
        if (fitness) *fitness = rc == FLS_OK ? res.fitness : FloatNaN;
        if (rc != FLS_OK) {
            LOG(WARNING) << "fls_relocalize_multi: " << fls_strerror(rc) << " " << fls_last_error();
            return false;
        }
        DLOG(INFO) << "B200 RelocalizeMulti guesses=" << guesses.size() << " hypotheses=" << res.n_hypotheses << " evaluations=" << evaluations
                   << " fitness=" << res.fitness;
        return res.accepted != 0;
    }

    // Convenience: the factory branch a maintainer adds to FrontEnd::InitMatcher / Localization::InitMatcher.
    static std::shared_ptr<RegistrationInterface> Create(const std::string& mode, const fls_config& overrides_applied) {
        return std::make_shared<B200Registration>(overrides_applied);
    }

private:
    fls_handle* handle_ = nullptr;
    int method_ = 0;
};

static_assert(sizeof(PCLPointXYZI) == FLS_LAYOUT_PCL_XYZI, "pcl::PointXYZI must be the 32-byte record the ABI expects");

#endif  // FUNNY_LIDAR_SLAM_B200_REGISTRATION_H
