// fls_kernels.h — launch interfaces that more than one file uses: the LOAM-iVox batch kernel (generation 9, whose host half lives
// with generation 8 in fls_p2plane.cu).  Each plug-in's own argument structs and launchers sit in its file.
#pragma once
#include "fls_common.cuh"
#include "fls_gn.cuh"
#include "fls_ivox.cuh"
#include "fls_maps.h"

namespace fls {

static constexpr int kMaxBatch = 64;  // scans per fls_match_batch call

// One scan of a batch (device-resident descriptor read by the LoamPointToPlaneIVOX batch kernel, v9)
struct P2PlaneScan {
    const float4* src;  // body-frame scan in Morton order of the query voxel, packed float4
    int n;
    unsigned tag_base;         // Match epoch << 8 (hand-over tags, fls_gn.cuh)
    GnState* state;
    float4* rec0;  // persistent per-point record: J0..J3
    float4* rec1;  //                              J4, J5, |d|, 1
    unsigned char* flags;
    uint4* rows;     // [grid][32] LL records {lo, tag, hi, tag}: one per CTA and sum
    uint4* ll_pose;  // [kLlPoseLen] LL records: next pose + stop word, published by the scan's folder
    fls_iter_log* log;
    double* result;  // optional packed result (kResultLen doubles), written by the folder when the scan stops
    uint4* grows;    // [16][32] LL records: group rows of the two-level fold
};

// whole-loop arguments of the LoamPointToPlaneIVOX batch kernel (v9, K1 + fused K6); one launch = a batch of scans
struct P2PlaneLoopArgs {
    IvoxView map;
    double plane_thres;
    GnParams gp;
    int log_cap;
    const P2PlaneScan* scans;  // [n_scans]; CTAs draw chunks of any scan, the folder warp of CTA (12 s + 1) mod grid solves scan s
    int n_scans;
    unsigned* tickets;  // chunk ticket counters [n_scans][ticket_stride], zeroed before the launch
    int ticket_stride;  // >= max_iterations + 2
    unsigned* abort_word;  // watchdog: zeroed before the launch, non-zero when a wait loop gave up (protocol error)
};
// Each persistent kernel is sized by its *_grid call on the device it then runs on (see coresident_ctas, fls_common.cuh).
// generation 9 (fls_p2plane_v9.cu), batches: barrier-free dataflow, TMA-staged candidate runs, DMMA sums
int p2plane_v9_grid(int n_max, int device);  // also raises the kernel's shared-memory limit on `device`
void launch_p2plane_v9(const P2PlaneLoopArgs& a, int grid, cudaStream_t st);

}  // namespace fls
