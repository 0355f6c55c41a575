// fls_gn.cu — state initialisation of a Gauss-Newton loop (NDT / ICP / kd-tree LOAM; the LOAM-iVox path initialises its
// states in its batch prep kernel), and the per-device kernel attributes that size and prepare every persistent launch.
// The solve / update / stop rule itself (K6) is device code in fls_gn.cuh: gn_step_pre, which every persistent kernel runs, and
// the single-level fold around it (gn_handover / gn_handover_rows), which every one but the LOAM-iVox batch kernel uses.
#include <map>
#include <utility>

#include "fls_gn.cuh"

namespace fls {
namespace {

__global__ void gn_init_kernel(GnState* s, double t00, double t10, double t20, double t01, double t11, double t21, double t02, double t12,
                               double t22, double t03, double t13, double t23) {
    if (threadIdx.x != 0) return;
    // arguments are the column-major Mat4d entries T(r,c) named t<r><c>
    const double R[9] = {t00, t01, t02, t10, t11, t12, t20, t21, t22};
    const double t[3] = {t03, t13, t23};
    for (int i = 0; i < 9; ++i) s->R[i] = s->R0[i] = s->Rprev[i] = R[i];
    for (int i = 0; i < 3; ++i) s->t[i] = s->t0[i] = s->tprev[i] = t[i];
    s->last_rot = s->last_pos = 0.0;
    for (int i = 0; i < 36; ++i) s->H[i] = 0;
    for (int i = 0; i < 6; ++i) s->g[i] = s->dx[i] = 0;
    s->sum_res = 0;
    s->cand_total = s->hits_total = 0;
    s->n_valid = 0;
    s->iter = 0;
    s->done = 0;
    s->converged = 0;
    s->failed = 0;
}

}  // namespace

void launch_gn_init(GnState* d_state, const double* T, cudaStream_t st) {
    // T is column-major: T[c*4 + r]
    gn_init_kernel<<<1, 32, 0, st>>>(d_state, T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10], T[12], T[13], T[14]);
}

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

}  // namespace fls
