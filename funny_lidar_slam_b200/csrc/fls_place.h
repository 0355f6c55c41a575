// fls_place.h — the Scan Context descriptors of the keyframe store and their exact search (fls_place.cu, DESIGN.md §3.12).
#pragma once
#include <vector>

#include "fls_maps.h"

namespace fls {

constexpr int kTile = 8192;  // points of one keyframe handled by one block of the segmented passes (assemble's and describe's)

// the ranges of include/fls_b200.h: 1..64 rings, 1..360 sectors, at most 4096 cells, finite R > 0, finite z_offset
bool sc_cfg_ok(const fls_sc_cfg& c);

// One descriptor per keyframe for one fls_sc_cfg, computed lazily: a pass describes the keyframes added since the last one (all of
// them after a cfg change) and, for a scan query, the scan into the slot after the last keyframe.  Slots hold n_rings x n_sectors
// cells (f2ord values during the pass, float bits after it) and n_sectors fp64 column norms.  The owner serializes calls.
struct PlaceIndex {
    fls_sc_cfg cfg{};
    size_t described = 0;  // keyframes [0, described) hold descriptors for cfg
    // grow geometrically, keeping what is described; how many descriptors they hold depends on the cfg (describe recomputes it)
    DevBuf<unsigned> cells;
    DevBuf<double> norms;
    DevBuf<unsigned char> table;       // per-pass [segments | tiles]
    PinnedBuf<unsigned char> h_table;  // its staging
    DevBuf<double> dist;               // per candidate: D
    DevBuf<int> shift;                 // per candidate: its best shift
    DevBuf<fls_place_match> pick;
    BuildScratch sc;                   // the sort of (D, id)

    size_t n_cells() const { return (size_t)cfg.n_rings * cfg.n_sectors; }
    const float* desc(size_t slot) const { return reinterpret_cast<const float*>(cells.p) + slot * n_cells(); }
    // Describes what is not described for c yet: keyframes [described, K) of the arena and, when with_query, the n_query packed
    // records at d_query into slot K.  Enqueued on call.stream (no wait): a memset, the binning kernel when any point is read, the
    // finalize.  Returns the points read.
    size_t describe(const fls_sc_cfg& c, const float4* arena, const std::vector<unsigned long long>& begin, const std::vector<unsigned>& count,
                  const float4* d_query, size_t n_query, bool with_query, Call& call);
    // Ranks candidates [0, n_cand) against the descriptor in slot q by (D, id) and enqueues the copy of the first n_out records to
    // h_out (pinned).  n_cand > 0.  Three launches: the search, the sort, the pick.
    void search(size_t q, size_t n_cand, size_t n_out, fls_place_match* h_out, Call& call, int device);
};

}  // namespace fls
