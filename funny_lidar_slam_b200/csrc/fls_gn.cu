// fls_gn.cu — state initialisation of a single NDT or ICP Match's Gauss-Newton loop (every loop starts from gn_state_init, fls_gn.cuh:
// here, in a sub-grid launch's gn_start_kernel and in the LOAM-iVox batch prep kernel), and the per-device kernel attributes that size
// and prepare every persistent launch.  The solve / update / stop rule itself (K6) is device code in fls_gn.cuh: gn_step_pre, which every persistent
// kernel runs, and the single-level fold around it (gn_handover / gn_handover_rows), which every one but the LOAM-iVox batch kernel
// uses.
// fls_gn_step_probe runs gn_step_pre alone on constructed cases, for the tests that hold the step to a reference.
#include <map>
#include <utility>
#include <vector>

#include "fls_gn.cuh"
#include "fls_handle.h"

namespace fls {
namespace {

__global__ void gn_init_kernel(GnState* s, GnPose p) { gn_state_init(s, p); }

}  // namespace

void launch_gn_init(GnState* d_state, const double* T, cudaStream_t st) { gn_init_kernel<<<1, 1, 0, st>>>(d_state, gn_pose(T)); }

// ---- kernel attributes per device ----------------------------------------------------------------------------------------
// Handles on different threads size their kernels concurrently: one lock over every entry.
namespace {
struct KernelSlot {
    size_t smem_limit = 0;  // dynamic shared-memory limit raised so far (0: the default)
    int ctas = 0;           // co-resident CTAs (0: not queried yet)
};
std::mutex g_attr_mu;
std::map<std::pair<const void*, int>, KernelSlot> g_slots;  // (function, device)
int g_sms[kMaxDevices];

void raise_locked(KernelSlot& k, const void* fn, size_t bytes) {
    if (bytes <= k.smem_limit) return;
    FLS_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    k.smem_limit = bytes;
}

int sms_locked(int device) {
    if (!g_sms[device]) FLS_CUDA(cudaDeviceGetAttribute(&g_sms[device], cudaDevAttrMultiProcessorCount, device));
    return g_sms[device];
}
}  // namespace

void raise_smem_limit(const void* fn, size_t bytes, int device) {
    std::lock_guard<std::mutex> lock(g_attr_mu);
    raise_locked(g_slots[{fn, device}], fn, bytes);
}

int coresident_ctas(const void* fn, int block, size_t smem, int device) {
    std::lock_guard<std::mutex> lock(g_attr_mu);
    KernelSlot& k = g_slots[{fn, device}];
    if (!k.ctas) {
        raise_locked(k, fn, smem);
        int per_sm = 0;
        FLS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, block, smem));
        if (per_sm < 1) {
            set_last_error("cudaOccupancyMaxActiveBlocksPerMultiprocessor: no block of " + std::to_string(block) + " threads and " +
                           std::to_string(smem) + " B of shared memory fits on an SM of device " + std::to_string(device));
            throw CudaError{FLS_ERR_CUDA};
        }
        k.ctas = sms_locked(device) * per_sm;
    }
    return k.ctas;
}

int device_sms(int device) {
    std::lock_guard<std::mutex> lock(g_attr_mu);
    return sms_locked(device);
}

// ---- test hook: gn_step_pre on constructed cases (fls_gn_step_probe) ------------------------------------------------------
namespace {
__global__ void gn_step_probe_kernel(const fls_gn_step_case* in, fls_gn_step_out* out, GnState* states, uint4* ll, double* results, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const fls_gn_step_case& c = in[i];
    GnState* s = states + i;
    GnPre q;
    for (int k = 0; k < 9; ++k) q.R[k] = s->R[k] = s->R0[k] = s->Rprev[k] = c.R[k];
    for (int k = 0; k < 3; ++k) q.t[k] = s->t[k] = s->t0[k] = s->tprev[k] = c.t[k];
    q.last_rot = s->last_rot = c.last_rot;
    q.last_pos = s->last_pos = c.last_pos;
    q.cand0 = q.hits0 = 0.0;
    q.it = s->iter = c.iter;
    s->done = s->converged = s->failed = 0;
    GnParams p;
    p.method = c.method;
    p.max_iterations = c.max_iterations;
    p.min_effective = c.min_effective;
    p.rot_thres = c.rot_thres;
    p.pos_thres = c.pos_thres;
    const unsigned tag = 0x100u | (unsigned)((c.iter + 1) & 0xff);  // the tag of a first Match's iteration c.iter
    uint4* pose = ll + (size_t)i * kLlPoseLen;
    double* res = results + (size_t)i * kResultLen;
    gn_step_pre(s, q, c.tot, p, nullptr, 0, pose, tag, res);

    fls_gn_step_out& o = out[i];
    int ok = 1;
    for (int k = 0; k < 13; ++k) ok &= ll_load(pose + k, tag, o.published[k]) ? 1 : 0;
    o.published_ok = ok;
    for (int k = 0; k < 9; ++k) o.R[k] = s->R[k];
    for (int k = 0; k < 3; ++k) o.t[k] = s->t[k];
    for (int k = 0; k < 6; ++k) {
        o.dx[k] = s->dx[k];
        o.g[k] = s->g[k];
    }
    for (int k = 0; k < 36; ++k) o.H[k] = s->H[k];
    o.last_rot = s->last_rot;
    o.last_pos = s->last_pos;
    for (int k = 0; k < kResultLen; ++k) o.result[k] = res[k];
    o.n_valid = s->n_valid;
    o.iter = s->iter;
    o.converged = s->converged;
    o.failed = s->failed;
    o.done = s->done;
    // the fast-path decision, from a separate call of the same solver on the same system
    double H[36], g[6], x[6], det = 0.0;
    for (int r = 0; r < 6; ++r)
        for (int k = r; k < 6; ++k) H[r * 6 + k] = H[k * 6 + r] = c.tot[tri6(r, k)];
    for (int k = 0; k < 6; ++k) g[k] = c.tot[21 + k];
    o.spd = solve6_spd(H, g, x, &det) ? 1 : 0;
    o.det_spd = o.spd ? det : 0.0;
}
}  // namespace

}  // namespace fls

extern "C" int fls_gn_step_probe(fls_handle* hh, const fls_gn_step_case* cases, size_t n, fls_gn_step_out* out) {
    fls::Handle* h = reinterpret_cast<fls::Handle*>(hh);
    if (!h || (n && (!cases || !out)) || n > (1u << 20)) return FLS_ERR_INVALID_ARG;
    for (size_t i = 0; i < n; ++i)
        if (cases[i].method < FLS_ICP_P2P || cases[i].method > FLS_LOAM_FULL || cases[i].iter < 0) return FLS_ERR_INVALID_ARG;
    if (!n) return FLS_OK;
    FLS_TRY
    using namespace fls;
    h->begin_call();
    const size_t in_b = n * sizeof(fls_gn_step_case), out_b = n * sizeof(fls_gn_step_out), st_b = n * sizeof(GnState),
                 ll_b = n * kLlPoseLen * sizeof(uint4), res_b = n * kResultLen * sizeof(double);
    DevBuf<unsigned char> buf;
    unsigned char* d = buf.reserve(in_b + out_b + st_b + ll_b + res_b);
    fls_gn_step_case* d_in = reinterpret_cast<fls_gn_step_case*>(d);
    fls_gn_step_out* d_out = reinterpret_cast<fls_gn_step_out*>(d + in_b);
    GnState* d_st = reinterpret_cast<GnState*>(d + in_b + out_b);
    uint4* d_ll = reinterpret_cast<uint4*>(d + in_b + out_b + st_b);
    double* d_res = reinterpret_cast<double*>(d + in_b + out_b + st_b + ll_b);
    const std::vector<double> nan_fill(n * kResultLen, __builtin_nan(""));
    FLS_CUDA(cudaMemcpyAsync(d_in, cases, in_b, cudaMemcpyHostToDevice, h->call.stream));
    FLS_CUDA(cudaMemsetAsync(d_ll, 0, ll_b, h->call.stream));  // tag 0: no iteration's record
    FLS_CUDA(cudaMemcpyAsync(d_res, nan_fill.data(), res_b, cudaMemcpyHostToDevice, h->call.stream));
    gn_step_probe_kernel<<<(unsigned)((n + 127) / 128), 128, 0, h->call.stream>>>(d_in, d_out, d_st, d_ll, d_res, (int)n);
    FLS_CUDA(cudaGetLastError());
    FLS_CUDA(cudaMemcpyAsync(out, d_out, out_b, cudaMemcpyDeviceToHost, h->call.stream));
    h->call.end(nullptr);
    return FLS_OK;
    FLS_CATCH
}
