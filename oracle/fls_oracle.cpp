// ORACLE — TEST INFRASTRUCTURE ONLY.  parity unpinned (see orc_math.h header).
//
// extern "C" surface of the CPU oracle, loaded with ctypes by tests/, __graft_entry__.smoke() and
// bench.py's cpu_baseline / --impl reference legs.  It takes the product's fls_config struct
// (include/fls_b200.h — interface header only) so a test can hand the same configuration to both
// sides.  Poses cross this API as Eigen Mat4d memory (16 doubles, column-major).
#include <chrono>
#include <cstdio>
#include <cstring>
#include <memory>
#ifdef _OPENMP
#include <omp.h>
#endif

#include "../include/fls_b200.h"
#include "orc_cloud.h"
#include "orc_deskew.h"
#include "orc_features.h"
#include "orc_ivox.h"
#include "orc_math.h"
#include "orc_reg.h"

using namespace orc;

namespace {

Cloud load_cloud(const void* pts, size_t n, size_t stride) {
    Cloud c(n);
    const unsigned char* b = static_cast<const unsigned char*>(pts);
    const size_t ioff = (stride >= 32) ? 16 : 12;
    for (size_t k = 0; k < n; ++k) {
        const float* f = reinterpret_cast<const float*>(b + k * stride);
        c[k].x = f[0]; c[k].y = f[1]; c[k].z = f[2];
        std::memcpy(&c[k].i, b + k * stride + ioff, 4);
    }
    return c;
}
void col2row(const double* c, double* r) {
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) r[i * 4 + j] = c[j * 4 + i];
}
void row2col(const double* r, double* c) {
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) c[j * 4 + i] = r[i * 4 + j];
}

struct Reg {
    fls_config cfg;
    std::unique_ptr<LoamP2PlaneIvox> p2p;
    std::unique_ptr<IncrementalNdt> ndt;
    std::unique_ptr<IcpOptimized> icp;
    std::unique_ptr<LoamP2PlaneKdtree> kd;
    std::unique_ptr<LoamFull> full;
    MatchResult last;
};

}  // namespace

extern "C" {

int orc_num_threads() {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
void orc_set_num_threads(int n) {
#ifdef _OPENMP
    omp_set_num_threads(n);
#else
    (void)n;
#endif
}

// ---- math KAT hooks -------------------------------------------------------------------------------
void orc_so3_exp(const double* v, double* R) { so3_exp(v, R); }
void orc_se3_exp(const double* v, double* T) { se3_exp(v, T); }
void orc_rot_to_rpy(const double* R, double* rpy) { rot_to_rpy(R, rpy); }
float orc_fast_atan2f(float y, float x) { return fast_atan2f(y, x); }
void orc_lstsq53(const double* A, const double* b, double* x) { lstsq_colpiv_qr<5, 3>(A, b, x); }
void orc_solve6_fullpiv(const double* H, const double* g, double* x) { solve_fullpiv<6>(H, g, x); }
double orc_solve6_lu(const double* H, const double* g, double* x) { return solve_lu<6>(H, g, x); }
void orc_sym_eig3(const double* S, double* lam, double* V) { sym_eig3(S, lam, V); }
void orc_inv3(const double* A, double* Ai) { inv3(A, Ai); }

// ---- cloud primitives -----------------------------------------------------------------------------
size_t orc_voxel_grid(const void* pts, size_t n, size_t stride, float leaf, float* out) {
    const Cloud o = voxel_grid(load_cloud(pts, n, stride), leaf);
    std::memcpy(out, o.data(), o.size() * sizeof(P4));
    return o.size();
}
void orc_transform_d(const float* pts, size_t n, const double* T_col, float* out) {
    double T[16];
    col2row(T_col, T);
    for (size_t k = 0; k < n; ++k) {
        const P4 o = transform_point_d(P4{pts[k * 4], pts[k * 4 + 1], pts[k * 4 + 2], pts[k * 4 + 3]}, T);
        std::memcpy(out + k * 4, &o, sizeof(P4));
    }
}
void orc_transform_f(const float* pts, size_t n, const double* T_col, float* out) {
    double T[16];
    col2row(T_col, T);
    const Cloud o = transform_cloud_f(load_cloud(pts, n, 16), T);
    std::memcpy(out, o.data(), o.size() * sizeof(P4));
}

void* orc_knn_build(const float* pts, size_t n, float cell) {
    auto* t = new ExactKnn();
    t->build(load_cloud(pts, n, 16), cell);
    return t;
}
void orc_knn_search(void* h, const float* q, size_t nq, int k, int* idx, float* d2, int* found) {
    auto* t = static_cast<ExactKnn*>(h);
#pragma omp parallel for schedule(dynamic, 64)
    for (int64_t i = 0; i < int64_t(nq); ++i) {
        const P4 qq{q[i * 4], q[i * 4 + 1], q[i * 4 + 2], q[i * 4 + 3]};
        found[i] = t->search(qq, k, idx + i * k, d2 + i * k);
    }
}
void orc_knn_free(void* h) { delete static_cast<ExactKnn*>(h); }

// ---- iVox -----------------------------------------------------------------------------------------
void* orc_ivox_create(float res, int nearby, size_t capacity) { return new IVox(res, nearby, capacity); }
void orc_ivox_add(void* h, const float* pts, size_t n) { static_cast<IVox*>(h)->add_points(load_cloud(pts, n, 16)); }
void orc_ivox_closest(void* h, const float* q, size_t nq, int K, float max_range, float* out, int* found) {
    auto* iv = static_cast<IVox*>(h);
#pragma omp parallel for schedule(dynamic, 64)
    for (int64_t i = 0; i < int64_t(nq); ++i) {
        const P4 qq{q[i * 4], q[i * 4 + 1], q[i * 4 + 2], q[i * 4 + 3]};
        P4 tmp[16];
        const int f = iv->closest(qq, K, max_range, tmp);
        found[i] = f;
        std::memset(out + i * K * 4, 0, sizeof(float) * 4 * K);
        std::memcpy(out + i * K * 4, tmp, sizeof(P4) * f);
    }
}
size_t orc_ivox_num_voxels(void* h) { return static_cast<IVox*>(h)->num_voxels(); }
size_t orc_ivox_num_points(void* h) { return static_cast<IVox*>(h)->num_points(); }
void orc_ivox_free(void* h) { delete static_cast<IVox*>(h); }

// ---- registration plug-ins --------------------------------------------------------------------------
void* orc_reg_create(const fls_config* c) {
    auto* r = new Reg();
    r->cfg = *c;
    switch (c->method) {
        case FLS_P2PLANE_IVOX:
            r->p2p.reset(new LoamP2PlaneIvox(c->point_to_planar_thres, c->position_converge_thres, c->rotation_converge_thres,
                                             unsigned(c->max_iterations), c->localization_mode != 0, c->ivox_resolution, c->ivox_nearby,
                                             size_t(c->ivox_capacity), c->ivox_max_range));
            break;
        case FLS_NDT:
            r->ndt.reset(new IncrementalNdt(c->ndt_voxel_size, c->ndt_outlier_thres, c->source_cloud_filter_size, c->rotation_converge_thres,
                                            c->position_converge_thres, c->ndt_min_points_in_voxel, c->ndt_max_points_in_voxel,
                                            c->ndt_min_effective_pts, c->ndt_capacity, c->max_iterations, c->localization_mode != 0));
            break;
        case FLS_ICP_P2P:
            r->icp.reset(new IcpOptimized(unsigned(c->max_iterations), unsigned(c->local_map_size), c->map_cloud_filter_size,
                                          c->source_cloud_filter_size, c->icp_max_correspond_distance, c->position_converge_thres,
                                          c->rotation_converge_thres, c->rot_thre_add_cloud, c->dist_thre_add_cloud, c->localization_mode != 0));
            break;
        case FLS_P2PLANE_KNN:
            r->kd.reset(new LoamP2PlaneKdtree(c->point_to_planar_thres, c->position_converge_thres, c->rotation_converge_thres,
                                              c->rot_thre_add_cloud, c->dist_thre_add_cloud, unsigned(c->local_map_size), c->map_cloud_filter_size,
                                              unsigned(c->max_iterations), c->localization_mode != 0));
            break;
        case FLS_LOAM_FULL:
            r->full.reset(new LoamFull(c->point_to_planar_thres, c->point_search_thres, c->line_ratio_thres, c->position_converge_thres,
                                       c->rotation_converge_thres, c->dist_thre_add_cloud, c->rot_thre_add_cloud,
                                       unsigned(c->corner_local_map_size), unsigned(c->local_map_size), c->corner_map_filter_size,
                                       c->map_cloud_filter_size, unsigned(c->max_iterations)));
            break;
        default:
            delete r;
            return nullptr;
    }
    return r;
}
void orc_reg_free(void* h) { delete static_cast<Reg*>(h); }

int orc_reg_add_cloud(void* h, const void* pts, size_t n, size_t stride) {
    auto* r = static_cast<Reg*>(h);
    const Cloud c = load_cloud(pts, n, stride);
    if (r->p2p) r->p2p->add_cloud(c);
    else if (r->ndt) r->ndt->add_cloud(c);
    else if (r->icp) r->icp->add_cloud(c);
    else if (r->kd) r->kd->add_cloud(c);
    else return -1;  // LoamFull takes {planar, corner}: orc_reg_add_cloud2
    return 0;
}
int orc_reg_add_cloud2(void* h, const void* planar, size_t n_planar, const void* corner, size_t n_corner, size_t stride) {
    auto* r = static_cast<Reg*>(h);
    if (!r->full) return -1;
    r->full->add_cloud(load_cloud(planar, n_planar, stride), load_cloud(corner, n_corner, stride));
    return 0;
}

// returns wall seconds spent inside Match (steady_clock) through *seconds
int orc_reg_match(void* h, const void* pts, size_t n, size_t stride, double* T_col, int* converged, fls_match_stats* st, double* seconds) {
    auto* r = static_cast<Reg*>(h);
    const Cloud c = load_cloud(pts, n, stride);
    double T[16];
    col2row(T_col, T);
    const auto t0 = std::chrono::steady_clock::now();
    if (r->p2p) r->last = r->p2p->match(c, T);
    else if (r->ndt) r->last = r->ndt->match(c, T);
    else if (r->icp) r->last = r->icp->match(c, T);
    else if (r->kd) r->last = r->kd->match(c, T);
    else return -1;
    const auto t1 = std::chrono::steady_clock::now();
    row2col(T, T_col);
    if (converged) *converged = r->last.converged ? 1 : 0;
    if (st) {
        std::memset(st, 0, sizeof(*st));
        st->iterations = r->last.iters;
        st->converged = r->last.converged;
        st->n_valid = r->last.n_valid;
        st->sum_residual = r->last.sum_res;
        st->n_source = int64_t(n);
    }
    if (seconds) *seconds = std::chrono::duration<double>(t1 - t0).count();
    return 0;
}
// LoamFull: {planar, corner} feature clouds of one scan
int orc_reg_match2(void* h, const void* planar, size_t n_planar, const void* corner, size_t n_corner, size_t stride, double* T_col, int* converged,
                   fls_match_stats* st, double* seconds) {
    auto* r = static_cast<Reg*>(h);
    if (!r->full) return -1;
    const Cloud cp = load_cloud(planar, n_planar, stride), cc = load_cloud(corner, n_corner, stride);
    double T[16];
    col2row(T_col, T);
    const auto t0 = std::chrono::steady_clock::now();
    r->last = r->full->match(cp, cc, T);
    const auto t1 = std::chrono::steady_clock::now();
    row2col(T, T_col);
    if (converged) *converged = r->last.converged ? 1 : 0;
    if (st) {
        std::memset(st, 0, sizeof(*st));
        st->iterations = r->last.iters;
        st->converged = r->last.converged;
        st->n_valid = r->last.n_valid;
        st->sum_residual = r->last.sum_res;
        st->n_source = int64_t(n_planar + n_corner);
    }
    if (seconds) *seconds = std::chrono::duration<double>(t1 - t0).count();
    return 0;
}
int orc_reg_get_iter_log(void* h, fls_iter_log* out, int cap) {
    auto* r = static_cast<Reg*>(h);
    const int n = std::min<int>(cap, int(r->last.log.size()));
    for (int i = 0; i < n; ++i) {
        std::memcpy(out[i].H, r->last.log[i].H, sizeof(out[i].H));
        std::memcpy(out[i].g, r->last.log[i].g, sizeof(out[i].g));
        std::memcpy(out[i].dx, r->last.log[i].dx, sizeof(out[i].dx));
        out[i].sum_residual = r->last.log[i].sum_res;
        out[i].n_valid = r->last.log[i].n_valid;
    }
    return n;
}
float orc_reg_fitness(void* h, float max_range) {
    auto* r = static_cast<Reg*>(h);
    if (r->p2p) return r->p2p->fitness(max_range);
    if (r->ndt) return r->ndt->fitness(max_range);
    if (r->kd) return r->kd->fitness(max_range);
    if (r->full) return r->full->fitness(max_range);
    return r->icp->fitness(max_range);
}
size_t orc_reg_map_voxels(void* h) {
    auto* r = static_cast<Reg*>(h);
    if (r->p2p) return r->p2p->ivox().num_voxels();
    if (r->ndt) return r->ndt->num_voxels();
    if (r->kd) return r->kd->map().size();
    if (r->full) return r->full->planar_map().size();
    return r->icp->map().size();
}
size_t orc_reg_map_points(void* h) {
    auto* r = static_cast<Reg*>(h);
    if (r->p2p) return r->p2p->ivox().num_points();
    if (r->icp) return r->icp->map().size();
    if (r->kd) return r->kd->map().size();
    if (r->full) return r->full->planar_map().size() + r->full->corner_map().size();
    return 0;
}
// copies the current local map (kd-tree plug-ins / ICP) into out (capacity cap points, packed xyzi); which = 0 planar / only map, 1 = corner map
size_t orc_reg_map_copy(void* h, int which, float* out, size_t cap) {
    auto* r = static_cast<Reg*>(h);
    const Cloud* m = nullptr;
    Cloud iv;
    if (r->p2p) {  // LOAM-iVox: every point the iVox map holds, voxels in LRU order
        r->p2p->ivox().dump(iv);
        m = &iv;
    }
    if (r->icp) m = &r->icp->map();
    else if (r->kd) m = &r->kd->map();
    else if (r->full) m = which ? &r->full->corner_map() : &r->full->planar_map();
    if (!m) return 0;
    const size_t n = std::min(cap, m->size());
    std::memcpy(out, m->data(), n * sizeof(P4));
    return m->size();
}
// NDT voxel dump in LRU order (front first): returns count; arrays sized by orc_reg_map_voxels.  num_points and pending (the
// points_ buffer awaiting an estimate) may be NULL.
size_t orc_reg_ndt_dump(void* h, int* keys, double* mu, double* info, int* est, int* num_points, int* pending) {
    auto* r = static_cast<Reg*>(h);
    if (!r->ndt) return 0;
    std::vector<int> k, e, np, pd;
    std::vector<double> m, i;
    r->ndt->dump(k, m, i, e, np, pd);
    std::memcpy(keys, k.data(), k.size() * sizeof(int));
    std::memcpy(mu, m.data(), m.size() * sizeof(double));
    std::memcpy(info, i.data(), i.size() * sizeof(double));
    std::memcpy(est, e.data(), e.size() * sizeof(int));
    if (num_points) std::memcpy(num_points, np.data(), np.size() * sizeof(int));
    if (pending) std::memcpy(pending, pd.data(), pd.size() * sizeof(int));
    return e.size();
}

// ---- pre-hot-path pipeline: range gate + IMU de-skew + jump span + voxel filter; projector with de-skew -------------------------
static ImuBuffer make_imu(const uint64_t* t, const double* q_xyzw, size_t m, uint64_t ref_time, const double* T_li) {
    ImuBuffer b;
    b.t.assign(t, t + m);
    b.q.resize(m);
    for (size_t i = 0; i < m; ++i) b.q[i] = Quat{q_xyzw[4 * i], q_xyzw[4 * i + 1], q_xyzw[4 * i + 2], q_xyzw[4 * i + 3]};
    b.ref_time = ref_time;
    std::memcpy(b.T_li, T_li, sizeof(b.T_li));
    return b;
}
// returns n_ordered; *n_planar set; outputs sized n (packed xyzi)
size_t orc_preprocess(const float* raw_xyzit, size_t n, const uint64_t* imu_t, const double* imu_q, size_t m, uint64_t ref_time, const double* T_li,
                      float min_d, float max_d, int jump_span, float leaf, float* ordered, float* planar, size_t* n_planar) {
    ImuBuffer b;
    if (imu_t) b = make_imu(imu_t, imu_q, m, ref_time, T_li);
    const Preprocessed p = preprocess(raw_xyzit, n, imu_t ? &b : nullptr, min_d, max_d, jump_span, leaf);
    std::memcpy(ordered, p.ordered.data(), p.ordered.size() * sizeof(P4));
    std::memcpy(planar, p.planar.data(), p.planar.size() * sizeof(P4));
    *n_planar = p.planar.size();
    return p.ordered.size();
}
size_t orc_project_imu(const float* raw, const int* ring, const float* time, size_t n, const uint64_t* imu_t, const double* imu_q, size_t m,
                       uint64_t ref_time, const double* T_li, int V, int H, float h_res, float min_d, float max_d, float* ordered, float* depth,
                       int* col, int* row_start, int* row_end) {
    std::vector<int> rg(ring, ring + n);
    ImuBuffer b;
    if (imu_t) b = make_imu(imu_t, imu_q, m, ref_time, T_li);
    const Projected p = project_imu(load_cloud(raw, n, 16), rg, time, imu_t ? &b : nullptr, V, H, h_res, min_d, max_d);
    std::memcpy(ordered, p.ordered.data(), p.ordered.size() * sizeof(P4));
    std::memcpy(depth, p.depth.data(), p.depth.size() * sizeof(float));
    std::memcpy(col, p.col.data(), p.col.size() * sizeof(int));
    std::memcpy(row_start, p.row_start.data(), V * sizeof(int));
    std::memcpy(row_end, p.row_end.data(), V * sizeof(int));
    return p.ordered.size();
}

// ---- LOAM features ----------------------------------------------------------------------------------
// project(): returns N (ordered points); outputs sized V*H (depth, col), V (row_start/end), ordered V*H*4 floats
size_t orc_project(const float* raw, const int* ring, size_t n, int V, int H, float h_res, float min_d, float max_d, float* ordered, float* depth,
                   int* col, int* row_start, int* row_end) {
    std::vector<int> rg(ring, ring + n);
    const Projected p = project(load_cloud(raw, n, 16), rg, V, H, h_res, min_d, max_d);
    std::memcpy(ordered, p.ordered.data(), p.ordered.size() * sizeof(P4));
    std::memcpy(depth, p.depth.data(), p.depth.size() * sizeof(float));
    std::memcpy(col, p.col.data(), p.col.size() * sizeof(int));
    std::memcpy(row_start, p.row_start.data(), V * sizeof(int));
    std::memcpy(row_end, p.row_end.data(), V * sizeof(int));
    return p.ordered.size();
}
int orc_extract_features(const float* depth, const int* col, size_t n, const int* row_start, const int* row_end, int V, float corner_thr,
                         float planar_thr, int* corner_idx, size_t* n_corner, int* planar_idx, size_t* n_planar, double* seconds) {
    const auto t0 = std::chrono::steady_clock::now();
    const Features f = extract_features(int(n), depth, col, V, row_start, row_end, corner_thr, planar_thr);
    const auto t1 = std::chrono::steady_clock::now();
    std::memcpy(corner_idx, f.corner_idx.data(), f.corner_idx.size() * sizeof(int));
    std::memcpy(planar_idx, f.planar_idx.data(), f.planar_idx.size() * sizeof(int));
    *n_corner = f.corner_idx.size();
    *n_planar = f.planar_idx.size();
    if (seconds) *seconds = std::chrono::duration<double>(t1 - t0).count();
    return 0;
}

}  // extern "C"
