// ORACLE — TEST INFRASTRUCTURE ONLY.  parity unpinned (see orc_math.h header).
//
// CPU restatement of the Gauss-Newton registration plug-ins behind
// include/registration/registration_interface.h:11-20:
//   LoamP2PlaneIvox  <- include/registration/loam_point_to_plane_ivox.h:30-369  (Type=double)
//   IncrementalNdt   <- include/registration/incremental_ndt.h:16-398
//   IcpOptimized     <- include/registration/icp_optimized.h:15-253            (Type=double)
//   LoamP2PlaneKdtree<- include/registration/loam_point_to_plane_kdtree.h:24-322 (Type=double)
//   LoamFull         <- include/registration/loam_full_kdtree.h:24-435          (Type=double)
// Structure kept deliberately close to upstream so that timing it is representative of the CPU
// path: parallel per-point loop (OpenMP here, TBB std::execution::par upstream), SERIAL H/g
// summation, per-iteration allocation of the per-point buffers, fp64 maths on fp32 points.
// Quirks that change results are reproduced and marked [quirk N] (numbering of SURVEY.md §7).
#pragma once
#include <deque>
#include <list>
#include <memory>
#include <set>
#include <unordered_map>
#include <vector>

#include "orc_cloud.h"
#include "orc_ivox.h"
#include "orc_math.h"

namespace orc {

struct IterLog {
    double H[36];
    double g[6];
    double dx[6];
    double sum_res;
    int64_t n_valid;
};

struct MatchResult {
    bool converged = false;
    int iters = 0;           // GN iterations executed
    int64_t n_valid = 0;     // of the last executed iteration
    double sum_res = 0;      // of the last executed iteration
    std::vector<IterLog> log;
};

inline void T_get_Rt(const double* T, double* R, double* t) {
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) R[i * 3 + j] = T[i * 4 + j];
        t[i] = T[i * 4 + 3];
    }
}
inline void T_set_R(double* T, const double* R) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) T[i * 4 + j] = R[i * 3 + j];
}

// mean squared 1-NN distance over points with d2 <= max_range  [quirk 4: squared vs unsquared]
// (icp_optimized.h:191-215, incremental_ndt.h:345-375, loam_point_to_plane_ivox.h:225-254)
inline float fitness_score(const ExactKnn& tree, const Cloud& src, const double* T, float max_range) {
    const Cloud tc = transform_cloud_f(src, T);
    float score = 0.0f;
    int nr = 0;
    for (const P4& q : tc) {
        int idx;
        float d2;
        if (tree.search(q, 1, &idx, &d2) < 1) continue;
        if (d2 <= max_range) { score += d2; nr++; }
    }
    return nr > 0 ? score / float(nr) : std::numeric_limits<float>::max();
}

// =================================================================================================
class LoamP2PlaneIvox {
public:
    LoamP2PlaneIvox(double plane_thres, double pos_thres, double rot_thres, unsigned iters, bool localization,
                    float ivox_res = 0.5f, int nearby = NEARBY18, size_t capacity = 1000000, float max_range = 5.0f)
        : plane_thres_(plane_thres), pos_thres_(pos_thres), rot_thres_(rot_thres), iters_(iters), loc_(localization),
          ivox_res_(ivox_res), nearby_(nearby), capacity_(capacity), max_range_(max_range) {
        init_ivox();
    }

    // loam_point_to_plane_ivox.h:60-139
    void add_cloud(const Cloud& planar) {
        if (loc_) {  // :64-69 — localization mode rebuilds the map on every call
            is_first_ = true;
            init_ivox();
        }
        if (is_first_) {
            ivox_->add_points(planar);
            is_first_ = false;
        } else {
            // :79-128 — body-frame points; inserted or dropped by the cached-5-NN rule  [quirk 8]
            Cloud to_add, no_down;
            for (size_t i = 0; i < n_planar_ && i < planar.size(); ++i) {
                const P4 pw = transform_point_d(planar[i], T_);
                const std::vector<P4>& near = nearest_[i];
                if (near.empty()) { to_add.push_back(pw); continue; }
                double c[3];
                const double pv[3] = {double(pw.x), double(pw.y), double(pw.z)};
                for (int a = 0; a < 3; ++a) c[a] = (std::floor(pv[a] / filter_size_) + 0.5) * filter_size_;  // :97-99 floor+0.5
                const double d0[3] = {double(near[0].x) - c[0], double(near[0].y) - c[1], double(near[0].z) - c[2]};
                if (std::fabs(d0[0]) > 0.5 * filter_size_ && std::fabs(d0[1]) > 0.5 * filter_size_ && std::fabs(d0[2]) > 0.5 * filter_size_) {
                    no_down.push_back(pw);
                    continue;
                }
                bool need = true;
                const double dist = (pv[0] - c[0]) * (pv[0] - c[0]) + (pv[1] - c[1]) * (pv[1] - c[1]) + (pv[2] - c[2]) * (pv[2] - c[2]);
                if (near.size() >= 5u) {
                    for (int r = 0; r < 5; ++r) {
                        const double e[3] = {double(near[r].x) - c[0], double(near[r].y) - c[1], double(near[r].z) - c[2]};
                        if (e[0] * e[0] + e[1] * e[1] + e[2] * e[2] < dist + 1.0e-6) { need = false; break; }
                    }
                }
                if (need) to_add.push_back(pw);
            }
            ivox_->add_points(to_add);
            ivox_->add_points(no_down);
        }
        if (loc_) tree_.build(planar);  // :134-138 — kd-tree only serves GetFitnessScore
    }

    // loam_point_to_plane_ivox.h:141-216
    MatchResult match(const Cloud& planar, double* T /*4x4 row-major, in-out*/) {
        MatchResult res;
        src_ = planar;
        const size_t N = planar.size();
        n_planar_ = N;
        Hc_.resize(N * 36);
        gc_.resize(N * 6);
        flags_.assign(N, 0);  // [quirk 1] reset once per Match, not per iteration (:156)
        resid_.resize(N);
        std::memcpy(T_, T, sizeof(T_));
        double last_rot = 0.0, last_pos = 0.0;
        for (unsigned it = 0; it < iters_; ++it) {
            planar_match(planar);
            IterLog lg{};
            // :326-340 serial sum over ALL flagged points, stale ones included  [quirk 1]
            n_valid_ = 0;
            sum_res_ = 0;
            for (size_t i = 0; i < N; ++i) {
                if (!flags_[i]) continue;
                n_valid_++;
                for (int k = 0; k < 36; ++k) lg.H[k] += Hc_[i * 36 + k];
                for (int k = 0; k < 6; ++k) lg.g[k] += gc_[i * 6 + k];
                sum_res_ += resid_[i];
            }
            lg.n_valid = int64_t(n_valid_);
            lg.sum_res = sum_res_;
            solve_fullpiv<6>(lg.H, lg.g, lg.dx);  // :167
            double Rd[9], R[9], t[3], Rn[9];
            so3_exp(lg.dx, Rd);
            T_get_Rt(T_, R, t);
            mat3_mul(Rd, R, Rn);  // :168-169 left update
            T_set_R(T_, Rn);
            for (int a = 0; a < 3; ++a) T_[a * 4 + 3] += lg.dx[3 + a];  // :170
            res.log.push_back(lg);
            res.iters = int(it) + 1;
            const double rn = norm3(lg.dx), pn = norm3(lg.dx + 3);
            const double drot = std::fabs(rn - last_rot), dpos = std::fabs(pn - last_pos);
            last_rot = rn;
            last_pos = pn;
            if ((rn < rot_thres_ && pn < pos_thres_) || (drot < 1.0e-4 && dpos < 1.0e-4)) break;  // :181-195
        }
        std::memcpy(T, T_, sizeof(T_));  // :198 written even on failure
        std::memcpy(Tfinal_, T_, sizeof(T_));
        bool ok = true;
        if (n_valid_ < 50u) ok = false;  // :201-203
        if (ok && !loc_) add_cloud(planar);  // :205-206
        res.converged = ok;
        res.n_valid = int64_t(n_valid_);
        res.sum_res = sum_res_;
        return res;
    }

    float fitness(float max_range) const {
        if (!loc_) return std::numeric_limits<float>::max();  // FloatNaN, :226-228
        return fitness_score(tree_, src_, Tfinal_, max_range);
    }
    const IVox& ivox() const { return *ivox_; }

private:
    void init_ivox() { ivox_.reset(new IVox(ivox_res_, nearby_, capacity_)); }

    // :256-324
    void planar_match(const Cloud& src) {
        const size_t N = n_planar_;
        nearest_.resize(N);
        double R[9], t[3];
        T_get_Rt(T_, R, t);
        const double thr = plane_thres_;
#pragma omp parallel for schedule(dynamic, 256)
        for (int64_t ii = 0; ii < int64_t(N); ++ii) {
            const size_t i = size_t(ii);
            const P4& sp = src[i];
            const P4 q = transform_point_d(sp, T_);  // :265-266
            P4 nn[5];
            const int found = ivox_->closest(q, 5, max_range_, nn);  // :269 (the map's max_range_, ivox_map.h:58)
            // DELIBERATE DEVIATION (DESIGN.md §8): upstream's IVoxMap::GetClosestPoint returns false WITHOUT clearing `closest_pt`
            // when the stencil holds no candidate at all (ivox_map.cpp:21-23), so nearest_points_[i] keeps what index i found in an
            // earlier iteration — or in an earlier Match, where index i was a different point — and a plane is fitted to those
            // stale neighbours.  Here (and on the GPU) a point without candidates has no neighbours: it is skipped, and the
            // mapping-mode insertion rule adds it unconditionally (:93-96).  tests/test_gpu_p2plane.py isolates the case.
            nearest_[i].assign(nn, nn + found);
            if (found < 5) continue;  // :271-273
            double A[15];
            const double b[5] = {-1, -1, -1, -1, -1};
            for (int j = 0; j < 5; ++j) { A[j * 3 + 0] = nn[j].x; A[j * 3 + 1] = nn[j].y; A[j * 3 + 2] = nn[j].z; }
            double c[3];
            lstsq_colpiv_qr<5, 3>(A, b, c);  // :283
            const double cn = norm3(c);
            bool valid = true;
            for (int j = 0; j < 5; ++j)
                if (std::fabs(dot3(A + j * 3, c) + 1.0) / cn > thr) { valid = false; break; }  // :286-293
            if (!valid) continue;
            const double n[3] = {c[0] / cn, c[1] / cn, c[2] / cn};
            const double ps[3] = {double(sp.x), double(sp.y), double(sp.z)};
            const double pt[3] = {double(q.x) - A[0], double(q.y) - A[1], double(q.z) - A[2]};
            const double d = dot3(pt, n);  // :306 measured from the NEAREST neighbour  [quirk 2]
            if (norm3(ps) < 81 * d * d) continue;  // :309 body-frame norm  [quirk 3]
            const double s = d > 0 ? 1.0 : -1.0;
            double Rp[3], J[6];
            mat3_vec(R, ps, Rp);
            cross3(Rp, n, J);  // -hat(Rp)^T n = Rp x n   (:315)
            for (int a = 0; a < 3; ++a) { J[a] *= s; J[3 + a] = n[a] * s; }
            flags_[i] = 1;
            const double ad = std::fabs(d);
            for (int a = 0; a < 6; ++a) {
                for (int bq = 0; bq < 6; ++bq) Hc_[i * 36 + a * 6 + bq] = J[a] * J[bq];
                gc_[i * 6 + a] = -J[a] * ad;
            }
            resid_[i] = ad;
        }
    }

    double plane_thres_, pos_thres_, rot_thres_;
    unsigned iters_;
    bool loc_;
    float ivox_res_;
    int nearby_;
    size_t capacity_;
    float max_range_;
    double filter_size_ = 0.5;  // filter_size_map_min_ (:351)
    bool is_first_ = true;      // upstream: function-local static (:62)  [quirk 7]
    std::unique_ptr<IVox> ivox_;
    ExactKnn tree_;
    Cloud src_;
    size_t n_planar_ = 0, n_valid_ = 0;
    double sum_res_ = 0;
    double T_[16], Tfinal_[16];
    std::vector<double> Hc_, gc_, resid_;
    std::vector<uint8_t> flags_;
    std::vector<std::vector<P4>> nearest_;
};

// =================================================================================================
class IncrementalNdt {
public:
    IncrementalNdt(double voxel_size, double outlier_thres, float src_leaf, double rot_thres, double pos_thres, int min_pts, int max_pts,
                   int min_effective, int capacity, int max_iter, bool localization)
        : voxel_(voxel_size), inv_voxel_(1.0 / voxel_size), outlier_(outlier_thres), src_leaf_(src_leaf), rot_thres_(rot_thres),
          pos_thres_(pos_thres), min_pts_(min_pts), max_pts_(max_pts), min_eff_(min_effective), capacity_(size_t(capacity)),
          max_iter_(max_iter), loc_(localization) {}

    struct Voxel {
        std::vector<double> pts;  // xyz triples awaiting estimation
        double mu[3] = {0, 0, 0};
        double sigma[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        double info[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        bool estimated = false;
        int num_points = 0;
    };

    // incremental_ndt.h:182-227
    void add_cloud(const Cloud& cloud_world_full) {
        const Cloud cloud = voxel_grid(cloud_world_full, src_leaf_);  // :186
        if (loc_) tree_.build(cloud);
        std::set<uint64_t> active;
        for (const P4& p : cloud) {
            const double pe[3] = {double(p.x), double(p.y), double(p.z)};
            const int k[3] = {int(pe[0] * inv_voxel_), int(pe[1] * inv_voxel_), int(pe[2] * inv_voxel_)};  // :195 truncation [quirk 5]
            const uint64_t key = pack(k);
            auto it = grids_.find(key);
            if (it == grids_.end()) {
                data_.emplace_front();
                data_.front().first = key;
                Voxel& v = data_.front().second;
                v.pts.assign(pe, pe + 3);
                v.num_points = 1;
                grids_[key] = data_.begin();
                if (data_.size() >= capacity_) {  // :203-206
                    grids_.erase(data_.back().first);
                    data_.pop_back();
                }
            } else {
                Voxel& v = it->second->second;
                v.pts.insert(v.pts.end(), pe, pe + 3);
                if (!v.estimated) v.num_points++;
                data_.splice(data_.begin(), data_, it->second);
                it->second = data_.begin();
            }
            active.insert(key);
        }
        for (uint64_t key : active) {
            auto it = grids_.find(key);
            if (it == grids_.end()) continue;  // upstream would default-insert (UB) — evicted voxel, skipped here
            update_voxel(it->second->second);
        }
        first_scan_ = loc_;  // :222-226
    }

    // incremental_ndt.h:229-337
    MatchResult match(const Cloud& ordered, double* T) {
        MatchResult res;
        src_ = voxel_grid(ordered, src_leaf_);  // :232
        double pose[16], Tin[16];
        std::memcpy(pose, T, sizeof(pose));
        std::memcpy(Tin, T, sizeof(Tin));
        const size_t N = src_.size(), total = N * 7;
        static const int S[7][3] = {{0, 0, 0}, {-1, 0, 0}, {1, 0, 0}, {0, 1, 0}, {0, -1, 0}, {0, 0, -1}, {0, 0, 1}};  // :122-127
        for (int iter = 0; iter < max_iter_; ++iter) {
            std::vector<double> err(total * 3), info(total * 9), jac(total * 18);  // :247-250 per-iteration allocations
            std::vector<uint8_t> eff(total, 0);
            double R[9], t[3];
            T_get_Rt(pose, R, t);
#pragma omp parallel for schedule(dynamic, 256)
            for (int64_t ii = 0; ii < int64_t(N); ++ii) {
                const size_t idx = size_t(ii);
                const double p[3] = {double(src_[idx].x), double(src_[idx].y), double(src_[idx].z)};
                double q[3];
                mat3_vec(R, p, q);
                for (int a = 0; a < 3; ++a) q[a] += t[a];  // :255 fp64
                const int key[3] = {int(q[0] * inv_voxel_), int(q[1] * inv_voxel_), int(q[2] * inv_voxel_)};  // :256
                double Sp[9], B[9];
                so3_hat(p, Sp);
                mat3_mul(R, Sp, B);
                for (int a = 0; a < 9; ++a) B[a] = -B[a];  // :274
                for (int s = 0; s < 7; ++s) {
                    const int kk[3] = {key[0] + S[s][0], key[1] + S[s][1], key[2] + S[s][2]};
                    auto it = grids_.find(pack(kk));
                    const size_t ri = idx * 7 + s;
                    if (it == grids_.end() || !it->second->second.estimated) continue;
                    const Voxel& v = it->second->second;
                    const double e[3] = {q[0] - v.mu[0], q[1] - v.mu[1], q[2] - v.mu[2]};
                    double Ie[3];
                    mat3_vec(v.info, e, Ie);
                    const double chi = dot3(e, Ie);
                    if (std::isnan(chi) || chi > outlier_) continue;  // :267-271
                    for (int r = 0; r < 3; ++r) {
                        for (int c = 0; c < 3; ++c) {
                            jac[ri * 18 + r * 6 + c] = B[r * 3 + c];
                            jac[ri * 18 + r * 6 + 3 + c] = (r == c) ? 1.0 : 0.0;
                        }
                        err[ri * 3 + r] = e[r];
                    }
                    for (int a = 0; a < 9; ++a) info[ri * 9 + a] = v.info[a];
                    eff[ri] = 1;
                }
            }
            IterLog lg{};
            double total_res = 0;
            int effective = 0;
            for (size_t ri = 0; ri < total; ++ri) {  // :294-304 serial
                if (!eff[ri]) continue;
                const double* e = &err[ri * 3];
                const double* I = &info[ri * 9];
                const double* J = &jac[ri * 18];
                double Ie[3];
                mat3_vec(I, e, Ie);
                total_res += dot3(e, Ie);
                effective++;
                double IJ[18];  // 3x6
                for (int r = 0; r < 3; ++r)
                    for (int c = 0; c < 6; ++c) IJ[r * 6 + c] = I[r * 3 + 0] * J[0 * 6 + c] + I[r * 3 + 1] * J[1 * 6 + c] + I[r * 3 + 2] * J[2 * 6 + c];
                for (int a = 0; a < 6; ++a) {
                    for (int c = 0; c < 6; ++c) lg.H[a * 6 + c] += J[0 * 6 + a] * IJ[0 * 6 + c] + J[1 * 6 + a] * IJ[1 * 6 + c] + J[2 * 6 + a] * IJ[2 * 6 + c];
                    lg.g[a] += -(J[0 * 6 + a] * Ie[0] + J[1 * 6 + a] * Ie[1] + J[2 * 6 + a] * Ie[2]);
                }
            }
            lg.n_valid = effective;
            lg.sum_res = total_res;
            res.n_valid = effective;
            res.sum_res = total_res;
            res.iters = iter + 1;
            if (effective < min_eff_) {  // :306-309
                res.log.push_back(lg);
                std::memcpy(T, pose, sizeof(pose));
                res.converged = false;
                return res;
            }
            solve_lu<6>(lg.H, lg.g, lg.dx);  // :311  H.inverse() * err
            double Rd[9], Rn[9];
            so3_exp(lg.dx, Rd);
            mat3_mul(R, Rd, Rn);  // :312 right update
            T_set_R(pose, Rn);
            for (int a = 0; a < 3; ++a) pose[a * 4 + 3] += lg.dx[3 + a];
            res.log.push_back(lg);
            if (norm3(lg.dx) < rot_thres_ && norm3(lg.dx + 3) < pos_thres_) break;  // :315
        }
        res.converged = true;  // :325  [quirk 6]
        if (!loc_) {
            const Cloud tc = transform_cloud_f(src_, Tin);  // :328 uses the INPUT guess  [quirk 6]
            add_cloud(tc);
        }
        std::memcpy(T, pose, sizeof(pose));
        std::memcpy(Tfinal_, pose, sizeof(pose));
        return res;
    }

    float fitness(float max_range) const {
        if (!loc_) return std::numeric_limits<float>::max();
        return fitness_score(tree_, src_, Tfinal_, max_range);
    }

    size_t num_voxels() const { return grids_.size(); }
    // export the voxels for tests, LRU order: key(3 int), mu(3), info(9), estimated flag, num_points_, points_.size()
    void dump(std::vector<int>& keys, std::vector<double>& mu, std::vector<double>& info, std::vector<int>& est, std::vector<int>& num_points,
              std::vector<int>& pending) const {
        for (const auto& kv : data_) {
            int k[3];
            unpack(kv.first, k);
            keys.insert(keys.end(), k, k + 3);
            mu.insert(mu.end(), kv.second.mu, kv.second.mu + 3);
            info.insert(info.end(), kv.second.info, kv.second.info + 9);
            est.push_back(kv.second.estimated ? 1 : 0);
            num_points.push_back(kv.second.num_points);
            pending.push_back(int(kv.second.pts.size() / 3));
        }
    }

private:
    static uint64_t pack(const int* k) {
        return (uint64_t(uint32_t(k[0]) & 0x1fffff) << 42) | (uint64_t(uint32_t(k[1]) & 0x1fffff) << 21) | uint64_t(uint32_t(k[2]) & 0x1fffff);
    }
    static void unpack(uint64_t key, int* k) {
        for (int a = 0; a < 3; ++a) {
            uint32_t v = uint32_t((key >> (42 - 21 * a)) & 0x1fffff);
            k[a] = (v & 0x100000) ? int(v | 0xffe00000u) : int(v);
        }
    }
    // incremental_ndt.h:92-110 — mean, covariance / (n-1), sequential accumulation
    static void mean_cov(const std::vector<double>& pts, double* mean, double* cov) {
        const size_t n = pts.size() / 3;
        double s[3] = {0, 0, 0};
        for (size_t i = 0; i < n; ++i)
            for (int a = 0; a < 3; ++a) s[a] += pts[i * 3 + a];
        for (int a = 0; a < 3; ++a) mean[a] = s[a] / double(n);
        double c[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        for (size_t i = 0; i < n; ++i) {
            const double v[3] = {pts[i * 3] - mean[0], pts[i * 3 + 1] - mean[1], pts[i * 3 + 2] - mean[2]};
            for (int a = 0; a < 3; ++a)
                for (int b = 0; b < 3; ++b) c[a * 3 + b] += v[a] * v[b];
        }
        for (int a = 0; a < 9; ++a) cov[a] = c[a] / double(n - 1);
    }
    // incremental_ndt.h:130-179
    void update_voxel(Voxel& v) const {
        if (first_scan_) {
            if (v.pts.size() / 3 > 1u) {
                mean_cov(v.pts, v.mu, v.sigma);
                double S[9];
                for (int a = 0; a < 9; ++a) S[a] = v.sigma[a] + (a % 4 == 0 ? 1.0e-3 : 0.0);
                inv3(S, v.info);
            } else {
                for (int a = 0; a < 3; ++a) v.mu[a] = v.pts[a];
                for (int a = 0; a < 9; ++a) v.info[a] = (a % 4 == 0) ? 1.0e2 : 0.0;
            }
            v.estimated = true;
            v.pts.clear();
            return;
        }
        if (v.estimated && v.num_points > max_pts_) return;  // :145-147
        const int np = int(v.pts.size() / 3);
        if (!v.estimated && np > min_pts_) {
            mean_cov(v.pts, v.mu, v.sigma);
            double S[9];
            for (int a = 0; a < 9; ++a) S[a] = v.sigma[a] + (a % 4 == 0 ? 1.0e-3 : 0.0);
            inv3(S, v.info);
            v.estimated = true;
            v.pts.clear();
        } else if (v.estimated && np > min_pts_) {
            double cm[3], cv[9], nm[3], nv[9];
            mean_cov(v.pts, cm, cv);
            const double m = double(v.num_points), n = double(np);  // :112-120
            for (int a = 0; a < 3; ++a) nm[a] = (m * v.mu[a] + n * cm[a]) / (m + n);
            for (int a = 0; a < 3; ++a)
                for (int b = 0; b < 3; ++b)
                    nv[a * 3 + b] = (m * (v.sigma[a * 3 + b] + (v.mu[a] - nm[a]) * (v.mu[b] - nm[b])) + n * (cv[a * 3 + b] + (cm[a] - nm[a]) * (cm[b] - nm[b]))) / (m + n);
            std::memcpy(v.mu, nm, sizeof(nm));
            std::memcpy(v.sigma, nv, sizeof(nv));
            v.num_points += np;
            v.pts.clear();
            double lam[3], V[9];
            sym_eig3(v.sigma, lam, V);  // :166 JacobiSVD of a symmetric PSD matrix
            if (lam[1] < lam[0] * 1e-3) lam[1] = lam[0] * 1e-3;
            if (lam[2] < lam[0] * 1e-3) lam[2] = lam[0] * 1e-3;
            for (int a = 0; a < 3; ++a)
                for (int b = 0; b < 3; ++b)
                    v.info[a * 3 + b] = V[a * 3 + 0] * V[b * 3 + 0] / lam[0] + V[a * 3 + 1] * V[b * 3 + 1] / lam[1] + V[a * 3 + 2] * V[b * 3 + 2] / lam[2];
        }
    }

    double voxel_, inv_voxel_, outlier_;
    float src_leaf_;
    double rot_thres_, pos_thres_;
    int min_pts_, max_pts_, min_eff_;
    size_t capacity_;
    int max_iter_;
    bool loc_;
    bool first_scan_ = true;
    std::list<std::pair<uint64_t, Voxel>> data_;
    std::unordered_map<uint64_t, std::list<std::pair<uint64_t, Voxel>>::iterator> grids_;
    ExactKnn tree_;
    Cloud src_;
    double Tfinal_[16];
};

// =================================================================================================
class IcpOptimized {
public:
    IcpOptimized(unsigned max_iter, unsigned local_map_size, float map_leaf, float src_leaf, double max_corr, double pos_thres,
                 double rot_thres, double rot_add, double dist_add, bool localization)
        : max_iter_(max_iter), local_map_size_(local_map_size), map_leaf_(map_leaf), src_leaf_(src_leaf), max_corr_(max_corr),
          pos_thres_(pos_thres), rot_thres_(rot_thres), rot_add_(rot_add), dist_add_(dist_add), loc_(localization) {}

    // icp_optimized.h:165-189
    void add_cloud(const Cloud& c) {
        Cloud merged;
        if (loc_) {
            merged = c;
        } else {
            deque_.push_back(c);
            if (deque_.size() > local_map_size_) deque_.pop_front();
            for (const Cloud& it : deque_) merged.insert(merged.end(), it.begin(), it.end());  // per-cloud downsample is discarded upstream (:182-183)
        }
        map_ = voxel_grid(merged, map_leaf_);
        tree_.build(map_);
    }

    // icp_optimized.h:54-163
    MatchResult match(const Cloud& ordered, double* T) {
        MatchResult res;
        converged_ = false;
        src_ = voxel_grid(ordered, src_leaf_);  // :57
        double Tt[16];
        std::memcpy(Tt, T, sizeof(Tt));
        const size_t N = src_.size();
        for (unsigned it = 0; it < max_iter_; ++it) {
            const Cloud tc = transform_cloud_f(src_, Tt);  // :64 fp32 transform, R/t cast to float first
            std::vector<double> Hall(N * 36, 0.0), Ball(N * 6, 0.0), errv(N * 3, 0.0);  // :70-73
            std::vector<uint8_t> eff(N, 0);
            double R[9], t[3];
            T_get_Rt(Tt, R, t);
#pragma omp parallel for schedule(dynamic, 256)
            for (int64_t ii = 0; ii < int64_t(N); ++ii) {
                const size_t i = size_t(ii);
                int idx;
                float d2;
                if (tree_.search(tc[i], 1, &idx, &d2) < 1) continue;
                if (double(d2) > max_corr_) continue;  // :87  [quirk 4] squared distance vs unsquared threshold
                const P4& m = tree_.point(idx);
                const double e[3] = {double(tc[i].x) - double(m.x), double(tc[i].y) - double(m.y), double(tc[i].z) - double(m.z)};
                const double p[3] = {double(src_[i].x), double(src_[i].y), double(src_[i].z)};
                double Sp[9], A[9];
                so3_hat(p, Sp);
                mat3_mul(R, Sp, A);
                double J[18];  // 3x6 = [I | -R p^]
                for (int r = 0; r < 3; ++r)
                    for (int c = 0; c < 3; ++c) {
                        J[r * 6 + c] = (r == c) ? 1.0 : 0.0;
                        J[r * 6 + 3 + c] = -A[r * 3 + c];
                    }
                for (int a = 0; a < 6; ++a) {
                    for (int b = 0; b < 6; ++b) Hall[i * 36 + a * 6 + b] = J[0 * 6 + a] * J[0 * 6 + b] + J[1 * 6 + a] * J[1 * 6 + b] + J[2 * 6 + a] * J[2 * 6 + b];
                    Ball[i * 6 + a] = -(J[0 * 6 + a] * e[0] + J[1 * 6 + a] * e[1] + J[2 * 6 + a] * e[2]);
                }
                for (int a = 0; a < 3; ++a) errv[i * 3 + a] = e[a];
                eff[i] = 1;
            }
            IterLog lg{};
            double total_res = 0;
            int effective = 0;
            for (size_t i = 0; i < N; ++i) {  // :117-127 serial
                if (!eff[i]) continue;
                for (int k = 0; k < 36; ++k) lg.H[k] += Hall[i * 36 + k];
                for (int k = 0; k < 6; ++k) lg.g[k] += Ball[i * 6 + k];
                effective++;
                total_res += norm3(&errv[i * 3]);
            }
            lg.n_valid = effective;
            lg.sum_res = total_res;
            res.n_valid = effective;
            res.sum_res = total_res;
            res.iters = int(it) + 1;
            const double det = solve_lu<6>(lg.H, lg.g, lg.dx);
            if (det == 0) {  // :129-131
                for (int a = 0; a < 6; ++a) lg.dx[a] = 0;
                res.log.push_back(lg);
                continue;
            }
            for (int a = 0; a < 3; ++a) Tt[a * 4 + 3] += lg.dx[a];  // :135  dx = [dt, dtheta]
            double Rd[9], Rn[9];
            so3_exp(lg.dx + 3, Rd);
            mat3_mul(R, Rd, Rn);  // :136 right update
            T_set_R(Tt, Rn);
            res.log.push_back(lg);
            if (norm3(lg.dx + 3) < rot_thres_ && norm3(lg.dx) < pos_thres_) {  // :138-139
                converged_ = true;
                break;
            }
        }
        std::memcpy(Tfinal_, Tt, sizeof(Tt));
        std::memcpy(T, Tt, sizeof(Tt));  // :152 always written
        if (converged_ && !loc_ && need_add_cloud(Tt)) {  // :154 (IsNeedAddCloud is evaluated before the mode test upstream; same effect on last_T only in mapping mode)
            add_cloud(transform_cloud_f(src_, Tt));
        }
        res.converged = converged_;
        return res;
    }

    float fitness(float max_range) const { return fitness_score(tree_, src_, Tfinal_, max_range); }
    const Cloud& map() const { return map_; }

private:
    // icp_optimized.h:218-236 — upstream keeps `static last_T` per template instantiation  [quirk 7]
    bool need_add_cloud(const double* T) {
        if (!have_last_) { std::memcpy(lastT_, T, sizeof(lastT_)); have_last_ = true; }
        double Rl[9], tl[3], R[9], t[3], Rli[9], Rd[9], rpy[3];
        T_get_Rt(lastT_, Rl, tl);
        T_get_Rt(T, R, t);
        inv3(Rl, Rli);
        mat3_mul(Rli, R, Rd);
        rot_to_rpy(Rd, rpy);
        const double dt[3] = {t[0] - tl[0], t[1] - tl[1], t[2] - tl[2]};
        if (norm3(dt) > dist_add_ || std::fabs(rpy[0]) > rot_add_ || std::fabs(rpy[1]) > rot_add_ || std::fabs(rpy[2]) > rot_add_) {
            std::memcpy(lastT_, T, sizeof(lastT_));
            return true;
        }
        return false;
    }

    unsigned max_iter_, local_map_size_;
    float map_leaf_, src_leaf_;
    double max_corr_, pos_thres_, rot_thres_, rot_add_, dist_add_;
    bool loc_;
    bool converged_ = false, have_last_ = false;
    double lastT_[16], Tfinal_[16];
    std::deque<Cloud> deque_;
    Cloud map_, src_;
    ExactKnn tree_;
};


// =================================================================================================
// Shared pieces of the kd-tree LOAM plug-ins.

// rigid key-frame gate shared by LoamPointToPlaneKdtree / LoamFull (loam_point_to_plane_kdtree.h:186-202,
// loam_full_kdtree.h:356-371): `static last_T = T` on the first call  [quirk 7]
struct KeyframeGate {
    bool have_last = false;
    double lastT[16];
    bool need(const double* T, double dist_add, double rot_add) {
        if (!have_last) { std::memcpy(lastT, T, sizeof(lastT)); have_last = true; }
        double Rl[9], tl[3], R[9], t[3], Rli[9], Rd[9], rpy[3];
        T_get_Rt(lastT, Rl, tl);
        T_get_Rt(T, R, t);
        inv3(Rl, Rli);
        mat3_mul(Rli, R, Rd);
        rot_to_rpy(Rd, rpy);
        const double dt[3] = {t[0] - tl[0], t[1] - tl[1], t[2] - tl[2]};
        if (norm3(dt) > dist_add || std::fabs(rpy[0]) > rot_add || std::fabs(rpy[1]) > rot_add || std::fabs(rpy[2]) > rot_add) {
            std::memcpy(lastT, T, sizeof(lastT));
            return true;
        }
        return false;
    }
};

// plane through 5 neighbours -> J (6), |d|; false when the point is rejected
// (loam_point_to_plane_kdtree.h:226-283 == loam_full_kdtree.h:295-343 == loam_point_to_plane_ivox.h:275-321)
inline bool plane_term(const P4* nn, const P4& sp, const P4& q, const double* R, double thr, double* J, double* ad) {
    double A[15];
    const double b[5] = {-1, -1, -1, -1, -1};
    for (int j = 0; j < 5; ++j) { A[j * 3 + 0] = nn[j].x; A[j * 3 + 1] = nn[j].y; A[j * 3 + 2] = nn[j].z; }
    double c[3];
    lstsq_colpiv_qr<5, 3>(A, b, c);
    const double cn = norm3(c);
    for (int j = 0; j < 5; ++j)
        if (std::fabs(dot3(A + j * 3, c) + 1.0) / cn > thr) return false;
    const double n[3] = {c[0] / cn, c[1] / cn, c[2] / cn};
    const double ps[3] = {double(sp.x), double(sp.y), double(sp.z)};
    const double pt[3] = {double(q.x) - A[0], double(q.y) - A[1], double(q.z) - A[2]};
    const double d = dot3(pt, n);  // measured from the NEAREST neighbour  [quirk 2]
    if (norm3(ps) < 81 * d * d) return false;  // body-frame norm  [quirk 3]
    const double s = d > 0 ? 1.0 : -1.0;
    double Rp[3];
    mat3_vec(R, ps, Rp);
    cross3(Rp, n, J);
    for (int a = 0; a < 3; ++a) { J[a] *= s; J[3 + a] = n[a] * s; }
    *ad = std::fabs(d);
    return true;
}

// per-class persistent H_i / g_i / res_i / flag arrays with the "reset once per Match" rule  [quirk 1]
struct TermStore {
    std::vector<double> Hc, gc, res;
    std::vector<uint8_t> flags;
    void reset(size_t N) { Hc.resize(N * 36); gc.resize(N * 6); res.resize(N); flags.assign(N, 0); }
    void set(size_t i, const double* J, double r) {
        flags[i] = 1;
        for (int a = 0; a < 6; ++a) {
            for (int b = 0; b < 6; ++b) Hc[i * 36 + a * 6 + b] = J[a] * J[b];
            gc[i * 6 + a] = -J[a] * r;
        }
        res[i] = r;
    }
    // serial sum over all flagged points, stale ones included; returns the count
    size_t sum_into(IterLog& lg, double& sum_res) const {
        size_t n = 0;
        sum_res = 0;
        for (size_t i = 0; i < flags.size(); ++i) {
            if (!flags[i]) continue;
            ++n;
            for (int k = 0; k < 36; ++k) lg.H[k] += Hc[i * 36 + k];
            for (int k = 0; k < 6; ++k) lg.g[k] += gc[i * 6 + k];
            sum_res += res[i];
        }
        return n;
    }
};

// one LOAM Gauss-Newton update + stop rule (loam_point_to_plane_kdtree.h:108-136, loam_full_kdtree.h:136-170)
inline bool loam_gn_update(IterLog& lg, double* T_, double& last_rot, double& last_pos, double rot_thres, double pos_thres) {
    solve_fullpiv<6>(lg.H, lg.g, lg.dx);
    double Rd[9], R[9], t[3], Rn[9];
    so3_exp(lg.dx, Rd);
    T_get_Rt(T_, R, t);
    mat3_mul(Rd, R, Rn);
    T_set_R(T_, Rn);
    for (int a = 0; a < 3; ++a) T_[a * 4 + 3] += lg.dx[3 + a];
    const double rn = norm3(lg.dx), pn = norm3(lg.dx + 3);
    const double drot = std::fabs(rn - last_rot), dpos = std::fabs(pn - last_pos);
    last_rot = rn;
    last_pos = pn;
    return (rn < rot_thres && pn < pos_thres) || (drot < 1.0e-4 && dpos < 1.0e-4);
}

// =================================================================================================
// LoamPointToPlaneKdtree<double>  (include/registration/loam_point_to_plane_kdtree.h:24-322)
class LoamP2PlaneKdtree {
public:
    LoamP2PlaneKdtree(double plane_thres, double pos_thres, double rot_thres, double rot_add, double dist_add, unsigned local_map_size,
                      float map_leaf, unsigned iters, bool localization)
        : plane_thres_(plane_thres), pos_thres_(pos_thres), rot_thres_(rot_thres), rot_add_(rot_add), dist_add_(dist_add),
          local_map_size_(local_map_size), map_leaf_(map_leaf), iters_(iters), loc_(localization) {}

    // :56-80 — the per-cloud down-sample inside the loop is computed and discarded upstream (:73)
    void add_cloud(const Cloud& planar) {
        Cloud merged;
        if (loc_) {
            merged = planar;
        } else {
            deque_.push_back(planar);
            if (deque_.size() > local_map_size_) deque_.pop_front();
            for (const Cloud& it : deque_) merged.insert(merged.end(), it.begin(), it.end());
        }
        map_ = voxel_grid(merged, map_leaf_);  // :78
        tree_.build(map_);
    }

    // :82-157
    MatchResult match(const Cloud& planar, double* T) {
        MatchResult res;
        src_ = planar;
        const size_t N = planar.size();
        store_.reset(N);  // :98 flags reset once per Match  [quirk 1]
        std::memcpy(T_, T, sizeof(T_));
        double last_rot = 0.0, last_pos = 0.0;
        size_t n_valid = 0;
        double sum_res = 0;
        for (unsigned it = 0; it < iters_; ++it) {
            double R[9], t[3];
            T_get_Rt(T_, R, t);
#pragma omp parallel for schedule(dynamic, 256)
            for (int64_t ii = 0; ii < int64_t(N); ++ii) {
                const size_t i = size_t(ii);
                const P4 q = transform_point_d(planar[i], T_);  // :211-212
                int idx[5];
                float d2[5];
                if (tree_.search(q, 5, idx, d2) < 5) continue;  // :217-221
                P4 nn[5];
                for (int j = 0; j < 5; ++j) nn[j] = tree_.point(idx[j]);
                double J[6], ad;
                if (plane_term(nn, planar[i], q, R, plane_thres_, J, &ad)) store_.set(i, J, ad);
            }
            IterLog lg{};
            n_valid = store_.sum_into(lg, sum_res);
            lg.n_valid = int64_t(n_valid);
            lg.sum_res = sum_res;
            const bool stop = loam_gn_update(lg, T_, last_rot, last_pos, rot_thres_, pos_thres_);
            res.log.push_back(lg);
            res.iters = int(it) + 1;
            if (stop) break;
        }
        std::memcpy(T, T_, sizeof(T_));  // :139
        std::memcpy(Tfinal_, T_, sizeof(T_));
        const bool ok = n_valid >= 50u;  // :142-144
        // :146-150 — IsNeedAddCloud is evaluated (and moves last_T) before the mode test
        if (ok && gate_.need(T_, dist_add_, rot_add_) && !loc_) add_cloud(transform_cloud_f(src_, T_));
        res.converged = ok;
        res.n_valid = int64_t(n_valid);
        res.sum_res = sum_res;
        return res;
    }

    float fitness(float max_range) const { return fitness_score(tree_, src_, Tfinal_, max_range); }  // :159-183
    const Cloud& map() const { return map_; }

private:
    double plane_thres_, pos_thres_, rot_thres_, rot_add_, dist_add_;
    unsigned local_map_size_;
    float map_leaf_;
    unsigned iters_;
    bool loc_;
    KeyframeGate gate_;
    double T_[16], Tfinal_[16];
    std::deque<Cloud> deque_;
    Cloud map_, src_;
    ExactKnn tree_;
    TermStore store_;
};

// =================================================================================================
// LoamFull<double>  (include/registration/loam_full_kdtree.h:24-435)
class LoamFull {
public:
    LoamFull(double plane_thres, double search_thres, double line_ratio, double pos_thres, double rot_thres, double dist_add, double rot_add,
             unsigned local_corner_size, unsigned local_planar_size, float corner_leaf, float planar_leaf, unsigned iters)
        : plane_thres_(plane_thres), search_thres_(search_thres), line_ratio_(line_ratio), pos_thres_(pos_thres), rot_thres_(rot_thres),
          dist_add_(dist_add), rot_add_(rot_add), local_corner_size_(local_corner_size), local_planar_size_(local_planar_size),
          corner_leaf_(corner_leaf), planar_leaf_(planar_leaf), iters_(iters) {}

    // :66-104 — {planar, corner}; the voxel filters only run once a deque holds more than 5 clouds
    void add_cloud(const Cloud& planar, const Cloud& corner) {
        corner_deque_.push_back(corner);
        planar_deque_.push_back(planar);
        if (planar_deque_.size() > local_planar_size_) planar_deque_.pop_front();
        if (corner_deque_.size() > local_corner_size_) corner_deque_.pop_front();
        planar_map_.clear();
        corner_map_.clear();
        for (const Cloud& c : planar_deque_) planar_map_.insert(planar_map_.end(), c.begin(), c.end());
        for (const Cloud& c : corner_deque_) corner_map_.insert(corner_map_.end(), c.begin(), c.end());
        if (planar_deque_.size() > 5) planar_map_ = voxel_grid(planar_map_, planar_leaf_);
        if (corner_deque_.size() > 5) corner_map_ = voxel_grid(corner_map_, corner_leaf_);
        planar_tree_.build(planar_map_);
        corner_tree_.build(corner_map_);
    }

    // :106-204
    MatchResult match(const Cloud& planar, const Cloud& corner, double* T) {
        MatchResult res;
        const size_t Nc = corner.size(), Np = planar.size();
        cstore_.reset(Nc);
        pstore_.reset(Np);
        std::memcpy(T_, T, sizeof(T_));
        double last_rot = 0.0, last_pos = 0.0;
        size_t nv_c = 0, nv_p = 0;
        double res_c = 0, res_p = 0;
        for (unsigned it = 0; it < iters_; ++it) {
            double R[9], t[3];
            T_get_Rt(T_, R, t);
            // CornerMatch :211-273
#pragma omp parallel for schedule(dynamic, 64)
            for (int64_t ii = 0; ii < int64_t(Nc); ++ii) {
                const size_t i = size_t(ii);
                const P4 q = transform_point_d(corner[i], T_);
                int idx[5];
                float d2[5];
                if (corner_tree_.search(q, 5, idx, d2) < 5) continue;  // upstream reads 5 indices unconditionally
                if (double(d2[4]) > search_thres_) continue;           // :227
                double P[15], c[3] = {0, 0, 0};
                for (int j = 0; j < 5; ++j) {
                    const P4& m = corner_tree_.point(idx[j]);
                    P[j * 3 + 0] = m.x; P[j * 3 + 1] = m.y; P[j * 3 + 2] = m.z;
                    for (int a = 0; a < 3; ++a) c[a] += P[j * 3 + a];
                }
                for (int a = 0; a < 3; ++a) c[a] /= 5.0;  // rowwise().mean()
                double S[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
                for (int j = 0; j < 5; ++j)
                    for (int a = 0; a < 3; ++a)
                        for (int b = 0; b < 3; ++b) S[a * 3 + b] += (P[j * 3 + a] - c[a]) * (P[j * 3 + b] - c[b]);
                for (int k = 0; k < 9; ++k) S[k] /= 5.0;  // :239-242
                double lam[3], V[9];
                sym_eig3(S, lam, V);  // JacobiSVD of a symmetric PSD matrix (:244)
                if (lam[0] <= line_ratio_ * lam[1]) continue;  // :249
                const double n[3] = {V[0], V[3], V[6]};        // V.col(0); J is invariant to its sign
                const double ps[3] = {double(corner[i].x), double(corner[i].y), double(corner[i].z)};
                const double v[3] = {double(q.x) - c[0], double(q.y) - c[1], double(q.z) - c[2]};
                double w[3];
                cross3(v, n, w);
                const double d = norm3(w);  // :260
                const double u[3] = {w[0] / d, w[1] / d, w[2] / d};
                // J.head = (n^ (Rp)^)^T u = (Rp)^T^ n^T^ u ... evaluated literally: M = n^ * (Rp)^ ; J.head = M^T u   (:264)
                double Rp[3], Nh[9], Ph[9], M[9], J[6];
                mat3_vec(R, ps, Rp);
                so3_hat(n, Nh);
                so3_hat(Rp, Ph);
                mat3_mul(Nh, Ph, M);
                for (int a = 0; a < 3; ++a) J[a] = M[0 * 3 + a] * u[0] + M[1 * 3 + a] * u[1] + M[2 * 3 + a] * u[2];
                // J.tail = (-n^)^T u = n^ u = n x u   (:265)
                cross3(n, u, J + 3);
                cstore_.set(i, J, d);  // g = -J d, res = d  (:267-270)
            }
            // PlanarMatch :275-345
#pragma omp parallel for schedule(dynamic, 256)
            for (int64_t ii = 0; ii < int64_t(Np); ++ii) {
                const size_t i = size_t(ii);
                const P4 q = transform_point_d(planar[i], T_);
                int idx[5];
                float d2[5];
                if (planar_tree_.search(q, 5, idx, d2) < 5) continue;
                if (double(d2[4]) > search_thres_) continue;  // :291
                P4 nn[5];
                for (int j = 0; j < 5; ++j) nn[j] = planar_tree_.point(idx[j]);
                double J[6], ad;
                if (plane_term(nn, planar[i], q, R, plane_thres_, J, &ad)) pstore_.set(i, J, ad);
            }
            IterLog lg{};
            nv_c = cstore_.sum_into(lg, res_c);  // :347-372 corners first
            nv_p = pstore_.sum_into(lg, res_p);
            lg.n_valid = int64_t(nv_p);
            lg.sum_res = res_p + res_c;
            const bool stop = loam_gn_update(lg, T_, last_rot, last_pos, rot_thres_, pos_thres_);
            res.log.push_back(lg);
            res.iters = int(it) + 1;
            if (stop) break;
        }
        std::memcpy(T, T_, sizeof(T_));  // :172
        const bool ok = nv_p >= 50;      // :174-176 planar count only
        if (ok && gate_.need(T_, dist_add_, rot_add_)) {  // :178-186 pcl::transformPointCloud with the double matrix
            Cloud tp(planar.size()), tc(corner.size());
            for (size_t i = 0; i < planar.size(); ++i) tp[i] = transform_point_d(planar[i], T_);
            for (size_t i = 0; i < corner.size(); ++i) tc[i] = transform_point_d(corner[i], T_);
            add_cloud(tp, tc);
        }
        res.converged = ok;
        res.n_valid = int64_t(nv_p);
        res.sum_res = res_p + res_c;
        n_valid_corner_ = nv_c;
        return res;
    }

    float fitness(float) const { return std::numeric_limits<float>::max(); }  // :206-208 FloatNaN
    const Cloud& planar_map() const { return planar_map_; }
    const Cloud& corner_map() const { return corner_map_; }
    size_t n_valid_corner() const { return n_valid_corner_; }

private:
    double plane_thres_, search_thres_, line_ratio_, pos_thres_, rot_thres_, dist_add_, rot_add_;
    unsigned local_corner_size_, local_planar_size_;
    float corner_leaf_, planar_leaf_;
    unsigned iters_;
    KeyframeGate gate_;
    double T_[16];
    std::deque<Cloud> corner_deque_, planar_deque_;
    Cloud corner_map_, planar_map_;
    ExactKnn corner_tree_, planar_tree_;
    TermStore cstore_, pstore_;
    size_t n_valid_corner_ = 0;
};

}  // namespace orc
