// fls_common.cuh — shared device/host helpers of the H100 (sm_90a) scan-matching library.
// Nothing in this tree includes or links anything under oracle/.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <cstdio>
#include <cstring>
#include <mutex>
#include <new>
#include <string>

#include "../../include/fls_b200.h"

namespace fls {

// ---- error plumbing ---------------------------------------------------------------------------------
void set_last_error(const std::string& s);
struct CudaError { int status; };

#define FLS_CUDA(expr)                                                                                              \
    do {                                                                                                            \
        cudaError_t _e = (expr);                                                                                    \
        if (_e != cudaSuccess) {                                                                                    \
            ::fls::set_last_error(std::string(#expr) + " -> " + cudaGetErrorString(_e) + " (" + __FILE__ + ":" +    \
                                  std::to_string(__LINE__) + ")");                                                  \
            throw ::fls::CudaError{FLS_ERR_CUDA};                                                                   \
        }                                                                                                           \
    } while (0)

// The error boundary of every extern "C" entry whose body can throw: a CUDA or host allocation failure becomes its status.
#define FLS_TRY try {
#define FLS_CATCH                                              \
    }                                                          \
    catch (const fls::CudaError& e) { return e.status; }       \
    catch (const std::bad_alloc&) {                            \
        fls::set_last_error("host allocation failed");         \
        return FLS_ERR_CUDA;                                   \
    }

// per-device tables (workspaces, kernel attributes) have this many slots
constexpr int kMaxDevices = 64;

// FLS_OK when `device` is a visible CUDA device with a slot in the per-device tables, FLS_ERR_NO_DEVICE otherwise
int check_device(int device);

// ---- kernel attributes per device (fls_gn.cu), cached per (function, device) under one lock ------------------------------
// The caller has made `device` current.  A persistent (cooperatively launched) kernel is launched only after its sizing call
// on the same device — coresident_ctas, or raise_smem_limit for a kernel sized by SMs — since that call is what raises the
// kernel's dynamic shared-memory limit there.

// Raises fn's dynamic shared-memory limit on `device` to `bytes`; never lowers it.
void raise_smem_limit(const void* fn, size_t bytes, int device);
// CTAs of fn that can be resident at once on `device` (SMs x blocks per SM at this block and dynamic shared memory; a function
// is always sized with the same block and smem).  Raises fn's shared-memory limit first; no resident block is an error.
int coresident_ctas(const void* fn, int block, size_t smem, int device);
int device_sms(int device);
// grid of a persistent launch: what the work needs, at least one CTA and at most what can be co-resident
inline int clamp_grid(int need, int coresident) { return need < 1 ? 1 : need < coresident ? need : coresident; }

// Cooperative launch of fn; the arguments are taken by value with fn's own parameter types, so params[] points at exactly what
// the kernel reads.
template <class T>
struct same_type { using type = T; };
template <class... P>
void launch_cooperative(void (*fn)(P...), int grid, int block, size_t smem, cudaStream_t st, typename same_type<P>::type... args) {
    void* params[] = {&args...};
    FLS_CUDA(cudaLaunchCooperativeKernel((const void*)fn, dim3(grid), dim3(block), params, smem, st));
}

// caller record layouts: packed float4, or x y z at 0 / 4 / 8 and the intensity at 16 of a larger record
inline bool stride_ok(size_t stride) { return stride == 16 || (stride >= 20 && stride % 4 == 0); }

// ---- one call: its stream, the events that time it and what it reports ----------------------------------------------------
// launches and the bytes copied each way (h2d / d2h) are counted where they are enqueued, waits (stream synchronisations) by
// sync().  Its owner (Handle, Workspace, KeyframeStore) creates the stream and the events; every helper of the call takes the
// Call and counts into it.
struct Call {
    cudaStream_t stream = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    int launches = 0, waits = 0;
    long long h2d = 0, d2h = 0;

    // zeroes the counts and records e0
    void begin() {
        launches = waits = 0;
        h2d = d2h = 0;
        FLS_CUDA(cudaEventRecord(e0, stream));
    }
    void sync() {
        FLS_CUDA(cudaStreamSynchronize(stream));
        ++waits;
    }
    // records e1 and waits for it, then clears *st (when given) and fills the call-level figures: device time from e0 to e1,
    // launches and copies
    void end(fls_match_stats* st) {
        FLS_CUDA(cudaEventRecord(e1, stream));
        sync();
        if (!st) return;
        std::memset(st, 0, sizeof(*st));
        FLS_CUDA(cudaEventElapsedTime(&st->gpu_ms, e0, e1));
        st->gpu_launches = launches;
        st->h2d_bytes = h2d;
        st->d2h_bytes = d2h;
    }
};

// ---- device buffer (grow-only) ------------------------------------------------------------------------
template <typename T>
struct DevBuf {
    T* p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { release(); }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }
    // ensure capacity for n elements; contents are NOT preserved on growth
    T* reserve(size_t n) {
        if (n > cap) {
            release();
            size_t want = n + n / 4 + 64;
            FLS_CUDA(cudaMalloc(&p, want * sizeof(T)));
            cap = want;
        }
        return p;
    }
    size_t bytes() const { return cap * sizeof(T); }
};

// ---- CUB device passes ----------------------------------------------------------------------------------
// A pass is one CUB device call with its arguments bound, as a callable cudaError_t(void* tmp, size_t& bytes): with tmp null it
// only writes the temporary storage it needs to `bytes`, otherwise it runs in the `bytes` of storage at tmp.  Sizing from the
// same callable that runs keeps the two argument lists from drifting apart.
// cub_reserve grows tmp (grow-only, 256 bytes of slack) to what the largest of `passes` needs.  A pipeline sizes all its passes
// before the first one runs, so that its buffer is not reallocated between two of them.
template <class... P>
void cub_reserve(DevBuf<unsigned char>& tmp, P&&... passes) {
    size_t need = 0;
    auto size = [&need](auto&& pass) {
        size_t bytes = 0;
        pass(nullptr, bytes);
        if (bytes > need) need = bytes;
    };
    (size(passes), ...);
    tmp.reserve(need + 256);
}
// runs a pass in tmp, which cub_reserve has sized for it
template <class P>
void cub_run(DevBuf<unsigned char>& tmp, P&& pass) {
    size_t bytes = tmp.cap;
    FLS_CUDA(pass(tmp.p, bytes));
}
// sizes tmp for one pass and runs it
template <class P>
void cub_pass(DevBuf<unsigned char>& tmp, P&& pass) {
    cub_reserve(tmp, pass);
    cub_run(tmp, pass);
}

// blocks of `block` threads that cover n items
inline unsigned grid_for(size_t n, int block) { return (unsigned)((n + block - 1) / block); }

// ---- pinned host buffer (grow-only): staging whose copies do not make the enqueue wait ------------------
template <typename T>
struct PinnedBuf {
    T* p = nullptr;
    size_t cap = 0;
    PinnedBuf() = default;
    PinnedBuf(const PinnedBuf&) = delete;
    PinnedBuf& operator=(const PinnedBuf&) = delete;
    ~PinnedBuf() { release(); }
    void release() {
        if (p) cudaFreeHost(p);
        p = nullptr;
        cap = 0;
    }
    // ensure capacity for n elements; contents are NOT preserved on growth
    T* reserve(size_t n) {
        if (n > cap) {
            release();
            size_t want = n + n / 4 + 64;
            FLS_CUDA(cudaMallocHost(&p, want * sizeof(T)));
            cap = want;
        }
        return p;
    }
};

// ---- per-device workspaces of the handle-free entries ---------------------------------------------------
// W derives from Workspace and adds its stage buffers.  There is one W per device and entry type, so a call takes only its own
// entry's lock; buffers, stream and events survive across calls (allocating per call costs more than the kernels).
struct Workspace {
    std::mutex mu;
    bool ready = false;
    Call call;  // stream and events created on first use
};

// Runs body(W&) on `device` (checked by check_device) under the workspace's lock.
template <class W, class F>
int with_workspace(int device, F&& body) {
    static W ws[kMaxDevices];
    W& w = ws[device];
    std::lock_guard<std::mutex> lock(w.mu);
    FLS_CUDA(cudaSetDevice(device));
    if (!w.ready) {
        FLS_CUDA(cudaStreamCreateWithFlags(&w.call.stream, cudaStreamNonBlocking));
        FLS_CUDA(cudaEventCreate(&w.call.e0));
        FLS_CUDA(cudaEventCreate(&w.call.e1));
        w.ready = true;
    }
    return body(w);
}

// ---- voxel keys / hash table ---------------------------------------------------------------------------
// Hash slot = one 16-byte record so a probe is a single LDG.128:
//   {u64 packed key (21 bits per axis, two's complement), u32 start, u32 count}
// start/count address the voxel's points inside the voxel-contiguous point array (NdtMap: voxel index and estimated flag).
struct __align__(16) HashSlot {
    unsigned long long key;
    unsigned int start;
    unsigned int count;
};
static constexpr unsigned long long kEmptyKey = ~0ull;

__host__ __device__ __forceinline__ unsigned long long pack_key(int x, int y, int z) {
    return ((unsigned long long)((unsigned)x & 0x1fffffu) << 42) | ((unsigned long long)((unsigned)y & 0x1fffffu) << 21) |
           (unsigned long long)((unsigned)z & 0x1fffffu);
}
__host__ __device__ __forceinline__ unsigned hash_key(unsigned long long k) {  // murmur3 fmix64
    k ^= k >> 33;
    k *= 0xff51afd7ed558ccdULL;
    k ^= k >> 33;
    k *= 0xc4ceb9fe1a85ec53ULL;
    k ^= k >> 33;
    return (unsigned)k;
}
__host__ __device__ __forceinline__ unsigned long long spread21(unsigned v) {  // 21 bits -> every 3rd bit
    unsigned long long x = v & 0x1fffffu;
    x = (x | x << 32) & 0x1f00000000ffffULL;
    x = (x | x << 16) & 0x1f0000ff0000ffULL;
    x = (x | x << 8) & 0x100f00f00f00f00fULL;
    x = (x | x << 4) & 0x10c30c30c30c30c3ULL;
    x = (x | x << 2) & 0x1249249249249249ULL;
    return x;
}
// Morton code of a signed voxel key (biased by 2^20): sort order that keeps stencil neighbours close in memory
__host__ __device__ __forceinline__ unsigned long long morton_key(int x, int y, int z) {
    return spread21((unsigned)(x + (1 << 20))) | (spread21((unsigned)(y + (1 << 20))) << 1) | (spread21((unsigned)(z + (1 << 20))) << 2);
}

#ifdef __CUDACC__
// static_cast<int64_t> of a double as x86-64's cvttsd2si does it: toward zero, and INT64_MIN for NaN and for values outside the
// int64 range.  C++ leaves those cases undefined, so the rule is written out here rather than left to what a plain conversion
// happens to return.  Every time product of the pre-processing path (the scan window, the de-skew's point time) goes through it.
__device__ __forceinline__ long long trunc_i64(double v) {
    return (v >= -9.2233720368547758e18 && v < 9.2233720368547758e18) ? __double2ll_rz(v) : (long long)0x8000000000000000ull;
}

__device__ __forceinline__ bool table_find(const HashSlot* __restrict__ tab, unsigned mask, unsigned long long key, unsigned& start,
                                           unsigned& count) {
    unsigned h = hash_key(key) & mask;
#pragma unroll 1
    for (;;) {
        const uint4 raw = __ldg(reinterpret_cast<const uint4*>(tab + h));
        const unsigned long long k = ((unsigned long long)raw.y << 32) | raw.x;
        if (k == key) {
            start = raw.z;
            count = raw.w;
            return true;
        }
        if (k == kEmptyKey) return false;
        h = (h + 1) & mask;
    }
}

// Claims key's slot in a table being filled (VoxelTable, fls_maps.h): returns the slot and sets `created` when this thread inserted
// the key.  Only the key is written; start and count are the caller's.
__device__ __forceinline__ unsigned table_claim(HashSlot* tab, unsigned mask, unsigned long long key, bool& created) {
    unsigned h = hash_key(key) & mask;
    for (;;) {
        const unsigned long long prev = atomicCAS(&tab[h].key, kEmptyKey, key);
        if (prev == kEmptyKey || prev == key) {
            created = prev == kEmptyKey;
            return h;
        }
        h = (h + 1) & mask;
    }
}

// fp32 squared distance in the reference's evaluation order, no FMA contraction
// ((dx*dx + dy*dy) + dz*dz — include/common/pointcloud_utility.h:13-17 upstream)
__device__ __forceinline__ float dist2_ref(float ax, float ay, float az, float bx, float by, float bz) {
    const float dx = __fsub_rn(ax, bx), dy = __fsub_rn(ay, by), dz = __fsub_rn(az, bz);
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// pcl::transformPoint with a double transform: ((r0*x + r1*y) + r2*z) + t in fp64 without contraction,
// one rounding to float (loam_point_to_plane_ivox.h:265-266 upstream)
__device__ __forceinline__ float xform_row_d(double r0, double r1, double r2, double t, double x, double y, double z) {
    return (float)__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(r0, x), __dmul_rn(r1, y)), __dmul_rn(r2, z)), t);
}
// same in fp64 without the final rounding (IncrementalNDT: incremental_ndt.h:255 upstream)
__device__ __forceinline__ double xform_row_dd(double r0, double r1, double r2, double t, double x, double y, double z) {
    return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(r0, x), __dmul_rn(r1, y)), __dmul_rn(r2, z)), t);
}
// TransformPoint(pt, Mat3f, Vec3f): fp32, R and t already cast (pointcloud_utility.h:63-72 upstream)
__device__ __forceinline__ float xform_row_f(float r0, float r1, float r2, float t, float x, float y, float z) {
    return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(r0, x), __fmul_rn(r1, y)), __fmul_rn(r2, z)), t);
}
#endif

// ---- Gauss-Newton state resident in device memory --------------------------------------------------------
// 31 reduced quantities per iteration: 21 upper-triangular entries of H, 6 of g, n_valid, sum of residuals,
// and two traffic counters for the roofline accounting (map records scanned, table probes that hit).
static constexpr int kNumAcc = 31;
static constexpr int kAccValid = 27, kAccRes = 28, kAccCand = 29, kAccHits = 30;
static constexpr int kAccStride = 32;  // padded row of the per-block partial-sum matrix

struct GnState {
    double R[9];  // row-major rotation
    double t[3];
    double R0[9];  // pose the caller passed in (IncrementalNDT re-uses it after the loop)
    double t0[3];
    double Rprev[9];  // pose before the last update (LOAM-iVox map insertion rule)
    double tprev[3];
    double last_rot, last_pos;
    double H[36];
    double g[6];
    double dx[6];
    double sum_res;
    double cand_total;  // map records scanned, summed over the executed iterations (roofline accounting)
    double hits_total;  // table probes that hit, summed over the executed iterations
    long long n_valid;
    int iter;       // iterations executed so far
    int done;       // loop finished (converged / failed / cap reached)
    int converged;  // value Match returns
    int failed;     // early-out (NDT effective_num < min)
    int pad[2];
};

// upper-triangular index of a symmetric 6x6 (row <= col)
__host__ __device__ __forceinline__ int tri6(int r, int c) { return r * 6 - (r * (r - 1)) / 2 + (c - r); }

// ---- small dense maths, host + device --------------------------------------------------------------------
__host__ __device__ inline void mat3_mul(const double* A, const double* B, double* C) {
    double t[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) t[i * 3 + j] = A[i * 3 + 0] * B[0 * 3 + j] + A[i * 3 + 1] * B[1 * 3 + j] + A[i * 3 + 2] * B[2 * 3 + j];
    for (int i = 0; i < 9; ++i) C[i] = t[i];
}
__host__ __device__ inline double norm3(const double* a) { return sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]); }

// Rodrigues with the reference's epsilon guard (include/common/math_function.h:74-89 upstream)
__host__ __device__ inline void so3_exp(const double* v, double* R) {
    const double theta = norm3(v);
    for (int i = 0; i < 9; ++i) R[i] = (i % 4 == 0) ? 1.0 : 0.0;
    if (theta > 2.220446049250313e-16) {
        const double n[3] = {v[0] / theta, v[1] / theta, v[2] / theta};
        const double c = cos(theta), s = sin(theta);
        const double S[9] = {0, -n[2], n[1], n[2], 0, -n[0], -n[1], n[0], 0};
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) R[i * 3 + j] = c * (i == j ? 1.0 : 0.0) + (1.0 - c) * n[i] * n[j] + s * S[i * 3 + j];
    }
}

// 6x6 solve with complete pivoting; rank-deficient systems get the basic solution (zeros on dropped
// pivots), the behaviour of Eigen's FullPivHouseholderQR::solve used at loam_point_to_plane_ivox.h:167 upstream.
__host__ __device__ inline void solve6_fullpiv(const double* H, const double* g, double* x) {
    double A[36], b[6];
    int cperm[6];
    for (int i = 0; i < 36; ++i) A[i] = H[i];
    for (int i = 0; i < 6; ++i) {
        b[i] = g[i];
        cperm[i] = i;
    }
    double maxpiv = 0;
    int rank = 6;
    for (int k = 0; k < 6; ++k) {
        int pr = k, pc = k;
        double best = -1;
        for (int i = k; i < 6; ++i)
            for (int j = k; j < 6; ++j)
                if (fabs(A[i * 6 + j]) > best) {
                    best = fabs(A[i * 6 + j]);
                    pr = i;
                    pc = j;
                }
        if (k == 0) maxpiv = best;
        if (best <= 2.220446049250313e-16 * 6 * maxpiv || best == 0.0) {
            rank = k;
            break;
        }
        if (pr != k) {
            for (int j = 0; j < 6; ++j) {
                const double t = A[k * 6 + j];
                A[k * 6 + j] = A[pr * 6 + j];
                A[pr * 6 + j] = t;
            }
            const double t = b[k];
            b[k] = b[pr];
            b[pr] = t;
        }
        if (pc != k) {
            for (int i = 0; i < 6; ++i) {
                const double t = A[i * 6 + k];
                A[i * 6 + k] = A[i * 6 + pc];
                A[i * 6 + pc] = t;
            }
            const int t = cperm[k];
            cperm[k] = cperm[pc];
            cperm[pc] = t;
        }
        for (int i = k + 1; i < 6; ++i) {
            const double f = A[i * 6 + k] / A[k * 6 + k];
            if (f == 0.0) continue;
            for (int j = k; j < 6; ++j) A[i * 6 + j] -= f * A[k * 6 + j];
            b[i] -= f * b[k];
        }
    }
    double y[6] = {0, 0, 0, 0, 0, 0};
    for (int i = rank - 1; i >= 0; --i) {
        double s = b[i];
        for (int j = i + 1; j < rank; ++j) s -= A[i * 6 + j] * y[j];
        y[i] = s / A[i * 6 + i];
    }
    for (int i = 0; i < 6; ++i) x[i] = 0;
    for (int i = 0; i < rank; ++i) x[cperm[i]] = y[i];
}

// Fast path for the well-conditioned symmetric positive-definite case (H = sum J^T J): fully unrolled LDL^T with the
// 21 upper-triangular entries in registers.  Returns false — caller falls back to the pivoting solver that mirrors the
// reference's rank handling — when a pivot is not safely positive (min pivot <= 1e-8 * max pivot).
// Also returns the determinant (product of pivots) for IcpOptimized's `det == 0` test.
__host__ __device__ inline bool solve6_spd(const double* H, const double* g, double* x, double* det_out) {
    double a00 = H[0], a01 = H[1], a02 = H[2], a03 = H[3], a04 = H[4], a05 = H[5];
    double a11 = H[7], a12 = H[8], a13 = H[9], a14 = H[10], a15 = H[11];
    double a22 = H[14], a23 = H[15], a24 = H[16], a25 = H[17];
    double a33 = H[21], a34 = H[22], a35 = H[23];
    double a44 = H[28], a45 = H[29];
    double a55 = H[35];
    double b0 = g[0], b1 = g[1], b2 = g[2], b3 = g[3], b4 = g[4], b5 = g[5];
    double dmax = fmax(fmax(fmax(a00, a11), fmax(a22, a33)), fmax(a44, a55));
    if (!(dmax > 0.0)) return false;
    const double tiny = 1e-8 * dmax;
    // elimination of column 0
    if (!(a00 > tiny)) return false;
    double inv = 1.0 / a00;
    double l1 = a01 * inv, l2 = a02 * inv, l3 = a03 * inv, l4 = a04 * inv, l5 = a05 * inv;
    a11 -= l1 * a01; a12 -= l1 * a02; a13 -= l1 * a03; a14 -= l1 * a04; a15 -= l1 * a05;
    a22 -= l2 * a02; a23 -= l2 * a03; a24 -= l2 * a04; a25 -= l2 * a05;
    a33 -= l3 * a03; a34 -= l3 * a04; a35 -= l3 * a05;
    a44 -= l4 * a04; a45 -= l4 * a05;
    a55 -= l5 * a05;
    b1 -= l1 * b0; b2 -= l2 * b0; b3 -= l3 * b0; b4 -= l4 * b0; b5 -= l5 * b0;
    // column 1
    if (!(a11 > tiny)) return false;
    inv = 1.0 / a11;
    l2 = a12 * inv; l3 = a13 * inv; l4 = a14 * inv; l5 = a15 * inv;
    a22 -= l2 * a12; a23 -= l2 * a13; a24 -= l2 * a14; a25 -= l2 * a15;
    a33 -= l3 * a13; a34 -= l3 * a14; a35 -= l3 * a15;
    a44 -= l4 * a14; a45 -= l4 * a15;
    a55 -= l5 * a15;
    b2 -= l2 * b1; b3 -= l3 * b1; b4 -= l4 * b1; b5 -= l5 * b1;
    // column 2
    if (!(a22 > tiny)) return false;
    inv = 1.0 / a22;
    l3 = a23 * inv; l4 = a24 * inv; l5 = a25 * inv;
    a33 -= l3 * a23; a34 -= l3 * a24; a35 -= l3 * a25;
    a44 -= l4 * a24; a45 -= l4 * a25;
    a55 -= l5 * a25;
    b3 -= l3 * b2; b4 -= l4 * b2; b5 -= l5 * b2;
    // column 3
    if (!(a33 > tiny)) return false;
    inv = 1.0 / a33;
    l4 = a34 * inv; l5 = a35 * inv;
    a44 -= l4 * a34; a45 -= l4 * a35;
    a55 -= l5 * a35;
    b4 -= l4 * b3; b5 -= l5 * b3;
    // column 4
    if (!(a44 > tiny)) return false;
    inv = 1.0 / a44;
    l5 = a45 * inv;
    a55 -= l5 * a45;
    b5 -= l5 * b4;
    if (!(a55 > tiny)) return false;
    // back substitution on the upper-triangular factor
    const double x5 = b5 / a55;
    const double x4 = (b4 - a45 * x5) / a44;
    const double x3 = (b3 - a34 * x4 - a35 * x5) / a33;
    const double x2 = (b2 - a23 * x3 - a24 * x4 - a25 * x5) / a22;
    const double x1 = (b1 - a12 * x2 - a13 * x3 - a14 * x4 - a15 * x5) / a11;
    const double x0 = (b0 - a01 * x1 - a02 * x2 - a03 * x3 - a04 * x4 - a05 * x5) / a00;
    x[0] = x0; x[1] = x1; x[2] = x2; x[3] = x3; x[4] = x4; x[5] = x5;
    if (det_out) *det_out = a00 * a11 * a22 * a33 * a44 * a55;
    return true;
}

// 6x6 partial-pivot LU solve; returns det (0 => x untouched).  Stands for `H.inverse() * b` and
// `H.determinant() == 0` (icp_optimized.h:129-133, incremental_ndt.h:311 upstream).
__host__ __device__ inline double solve6_lu(const double* H, const double* g, double* x) {
    double A[36], b[6];
    for (int i = 0; i < 36; ++i) A[i] = H[i];
    for (int i = 0; i < 6; ++i) b[i] = g[i];
    double det = 1.0;
    for (int k = 0; k < 6; ++k) {
        int pr = k;
        double best = fabs(A[k * 6 + k]);
        for (int i = k + 1; i < 6; ++i)
            if (fabs(A[i * 6 + k]) > best) {
                best = fabs(A[i * 6 + k]);
                pr = i;
            }
        if (best == 0.0) return 0.0;
        if (pr != k) {
            for (int j = 0; j < 6; ++j) {
                const double t = A[k * 6 + j];
                A[k * 6 + j] = A[pr * 6 + j];
                A[pr * 6 + j] = t;
            }
            const double t = b[k];
            b[k] = b[pr];
            b[pr] = t;
            det = -det;
        }
        det *= A[k * 6 + k];
        for (int i = k + 1; i < 6; ++i) {
            const double f = A[i * 6 + k] / A[k * 6 + k];
            for (int j = k; j < 6; ++j) A[i * 6 + j] -= f * A[k * 6 + j];
            b[i] -= f * b[k];
        }
    }
    for (int i = 5; i >= 0; --i) {
        double s = b[i];
        for (int j = i + 1; j < 6; ++j) s -= A[i * 6 + j] * x[j];
        x[i] = s / A[i * 6 + i];
    }
    return det;
}

}  // namespace fls
