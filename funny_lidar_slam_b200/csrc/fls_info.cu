// fls_info.cu — the fold of the information evaluation (fls_info.cuh) and fls_get_information.
#include "fls_info.cuh"

namespace fls {
namespace {

// One warp per scan: lane k adds sum k over the scan's CTA rows in CTA order, then lane 0 maps the plug-in's system to the fusion
// parameterization ([dθ; dp], R <- R Exp(dθ), p <- p + dp) and writes the record.  With the plug-in's dx = A [dθ; dp]:
//   NDT   dx = [dθ, dt], R <- R Exp(dθ), t += dt  ->  A = I;
//   ICP   dx = [dt, dθ], R <- R Exp(dθ), t += dt  ->  A swaps the blocks;
//   LOAM  dx = [dθ, dt], R <- Exp(dθ) R, t += dt  ->  Exp(dθ) R = R Exp(R^T dθ), so dθ = R δθ: A = blockdiag(R, I)
// (every update moves t in the world frame: gn_step_pre, fls_gn.cuh).  H_f = A^T H A and g_f = A^T g, where g = sum J^T W r is the
// negative of the accumulated right-hand side.
__global__ void info_fold_kernel(const __grid_constant__ InfoFold f, const double* __restrict__ part, fls_information* __restrict__ out) {
    __shared__ double tot[kAccStride];
    const int s = (int)blockIdx.x, k = (int)threadIdx.x;
    double v = 0.0;
    for (int c = f.cta0[s]; c < f.cta0[s + 1]; ++c) v += part[(size_t)c * kAccStride + k];
    tot[k] = v;
    __syncwarp();
    if (k != 0) return;
    double H[36], g[6], A[36];
    for (int r = 0; r < 6; ++r)
        for (int c = r; c < 6; ++c) H[r * 6 + c] = H[c * 6 + r] = tot[tri6(r, c)];
    for (int r = 0; r < 6; ++r) g[r] = -tot[21 + r];
    for (int i = 0; i < 36; ++i) A[i] = 0.0;
    if (f.method == FLS_NDT) {
        for (int i = 0; i < 6; ++i) A[i * 6 + i] = 1.0;
    } else if (f.method == FLS_ICP_P2P) {
        for (int i = 0; i < 6; ++i) A[i * 6 + (i + 3) % 6] = 1.0;
    } else {
        const GnState* st = f.state[s];
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) A[r * 6 + c] = st->R[r * 3 + c];
        for (int i = 3; i < 6; ++i) A[i * 6 + i] = 1.0;
    }
    fls_information& o = out[s];
    double HA[36];
    for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c) {
            double x = 0.0;
            for (int m = 0; m < 6; ++m) x += H[r * 6 + m] * A[m * 6 + c];
            HA[r * 6 + c] = x;
        }
    for (int r = 0; r < 6; ++r)
        for (int c = r; c < 6; ++c) {
            double x = 0.0;
            for (int m = 0; m < 6; ++m) x += A[m * 6 + r] * HA[m * 6 + c];
            o.H[r * 6 + c] = o.H[c * 6 + r] = x;  // symmetric by construction
        }
    for (int r = 0; r < 6; ++r) {
        double x = 0.0;
        for (int m = 0; m < 6; ++m) x += A[m * 6 + r] * g[m];
        o.g[r] = x;
    }
    o.sum_residual = tot[kAccRes];
    o.n_valid = (long long)(tot[kAccValid] + 0.5);
    o.valid = 1;
    o.pad = 0;
}

}  // namespace

void launch_info_fold(const InfoFold& f, int B, const double* part, fls_information* out, cudaStream_t st) {
    info_fold_kernel<<<B, 32, 0, st>>>(f, part, out);
    FLS_CUDA(cudaGetLastError());
}

}  // namespace fls

extern "C" int fls_get_information_scan(const fls_handle* hh, int scan, fls_information* out) {
    const fls::Handle* h = reinterpret_cast<const fls::Handle*>(hh);
    if (!h || !out || scan < 0 || scan >= (h->info_n > 0 ? h->info_n : 1)) return FLS_ERR_INVALID_ARG;
    if (h->info_n > 0) *out = h->h_info.p[scan];
    else std::memset(out, 0, sizeof(*out));
    return FLS_OK;
}

extern "C" int fls_get_information(const fls_handle* hh, fls_information* out) { return fls_get_information_scan(hh, 0, out); }
