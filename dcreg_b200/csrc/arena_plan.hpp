// arena_plan.hpp - host-side planning of a grid arena: the dense grids of one or many clouds built side by side in one
// set of buffers (the context's target, the targets of dcreg_icp_run_pairs, the aligned sources of the metrics).
//
// Cloud b's points get one global cell numbering: its cells are [cell_off[b], cell_off[b] + cells[b]), in the x-fastest
// dense order of its own bounding box, and the clouds follow each other.  One count / scan / scatter / rank over all
// points then groups every cloud's points exactly as a build of that cloud alone would (by cell, then by index), only
// shifted by the points of the clouds before it.  Everything here is plain C++ so tests/test_arena_plan.py can check it
// on the CPU (tools/test_arena_plan.cpp).
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace arena_plan {

constexpr long long kMaxDenseCells = 1ll << 27;      // per dense grid (above it: a sparse row index, or an error)
constexpr int kCoordLimit = 1 << 19;                 // cell coordinates outside +-2^19: NaN / huge coordinates
constexpr long long kMaxCells = 1ll << 30;           // all grids of a call: cell ids and cell_start entries are int32
constexpr long long kMaxPoints = 0x1fffffffLL;       // points per side and call: int32 positions, the loop kernel's 2^29
constexpr int kMaxPairs = 65535;                     // pairs = trials = grid y of the loop kernel

struct Box {
    int ox, oy, oz;          // cell coordinates of the box's minimum corner
    int nx, ny, nz;
    long long cells;         // nx * ny * nz
    long long cell_off;      // first global cell id
};

// Offsets table of n segments (n + 1 entries): starts at 0, ascends strictly (no empty segment), total <= max_total.
// Returns an empty string when valid, else the reason.
inline std::string check_offsets(int n, const int64_t* off, long long max_total, const char* what) {
    if (off[0] != 0) return std::string(what) + " offsets must start at 0";
    for (int b = 0; b < n; ++b)
        if (off[b + 1] <= off[b])
            return std::string(what) + " " + std::to_string(b) + " is empty (offsets must ascend strictly)";
    if (off[n] > max_total)
        return std::string(what) + " points of one call exceed " + std::to_string(max_total) + " (int32 indexing)";
    return std::string();
}

enum Fit { kDense, kTooManyCells, kOutOfRange };

// The box of one cloud from its bounds hb[6] (min cell coordinates x, y, z, then the max): kOutOfRange when a
// coordinate lies outside the +-2^19 cell range, else *x (cell_off 0) and kDense when it has at most kMaxDenseCells
// cells, kTooManyCells when it has more.
inline Fit box_of(const int* hb, Box* x) {
    for (int k = 0; k < 3; ++k)
        if (hb[k] < -kCoordLimit || hb[3 + k] > kCoordLimit || hb[k] > hb[3 + k]) return kOutOfRange;
    const long long nx = (long long)hb[3] - hb[0] + 1, ny = (long long)hb[4] - hb[1] + 1, nz = (long long)hb[5] - hb[2] + 1;
    x->cells = nx * ny * nz;
    x->cell_off = 0;
    if (x->cells > kMaxDenseCells) return kTooManyCells;
    x->ox = hb[0]; x->oy = hb[1]; x->oz = hb[2];
    x->nx = (int)nx; x->ny = (int)ny; x->nz = (int)nz;
    return kDense;
}

inline std::string out_of_range(const char* what) {
    return std::string(what) + ": coordinates / cell_size exceed the +-2^19 cell range (NaN or huge coordinates?)";
}

// bounds: n x 6 ints, per segment as box_of reads them.  Fills boxes[n] and *total_cells.
// Returns an empty string when every segment gets a dense grid, else the reason (naming the segment).
inline std::string plan(int n, const int* bounds, std::vector<Box>& boxes, long long* total_cells, const char* what) {
    boxes.assign((size_t)n, Box{});
    long long off = 0;
    for (int b = 0; b < n; ++b) {
        Box& x = boxes[(size_t)b];
        const std::string seg = std::string(what) + " " + std::to_string(b);
        const Fit fit = box_of(bounds + 6 * (size_t)b, &x);
        if (fit == kOutOfRange) return out_of_range(seg.c_str());
        if (fit == kTooManyCells)
            return seg + ": bounding box of " + std::to_string(x.cells) +
                   " cells is too large for a dense grid at this cell size (dcreg_set_sparse_maps(1) builds a sparse row index instead)";
        x.cell_off = off;
        off += x.cells;
        if (off > kMaxCells)
            return std::string(what) + " grids of one call exceed 2^30 dense cells in total (int32 cell ids)";
    }
    *total_cells = off;
    return std::string();
}

// plan for a caller that may build sparse row indexes instead (dcreg_set_sparse_maps): when plan rejects the clouds only
// for their cell counts (a box over kMaxDenseCells, or over kMaxCells in all), *sparse is set and the reason is empty;
// a coordinate outside the +-2^19 cell range is still refused, naming the first such cloud.  The boxes are then unset:
// a sparse index takes its box from the bounds.
inline std::string plan_or_sparse(int n, const int* bounds, std::vector<Box>& boxes, long long* total_cells,
                                  const char* what, bool* sparse) {
    *sparse = false;
    const std::string why = plan(n, bounds, boxes, total_cells, what);
    if (why.empty()) return why;
    Box x;
    for (int b = 0; b < n; ++b)
        if (box_of(bounds + 6 * (size_t)b, &x) == kOutOfRange)
            return out_of_range((std::string(what) + " " + std::to_string(b)).c_str());
    *sparse = true;
    *total_cells = 0;
    return std::string();
}

}  // namespace arena_plan
