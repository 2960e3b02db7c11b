// arena_plan.hpp - host-side planning of a grid arena: the dense target grids of many scan/target pairs
// (dcreg_icp_run_pairs) built side by side in one set of buffers.
//
// Pair b's points get one global cell numbering: its cells are [cell_off[b], cell_off[b] + cells[b]), in the x-fastest
// dense order of its own bounding box, and the pairs follow each other.  One count / scan / scatter / rank over all
// points then groups every pair's points exactly as a build of that pair alone would (by cell, then by index), only
// shifted by the points of the pairs before it.  Everything here is plain C++ so tests/test_arena_plan.py can check it
// on the CPU (tools/test_arena_plan.cpp).
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace arena_plan {

constexpr long long kMaxDenseCells = 1ll << 27;      // per grid: corr::kMaxDenseCells
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

// bounds: n x 6 ints, per segment the min cell coordinates (x, y, z) then the max.  Fills boxes[n] and *total_cells.
// Returns an empty string when every segment gets a dense grid, else the reason (naming the segment).
inline std::string plan(int n, const int* bounds, std::vector<Box>& boxes, long long* total_cells, const char* what) {
    boxes.assign((size_t)n, Box{});
    long long off = 0;
    for (int b = 0; b < n; ++b) {
        const int* hb = bounds + 6 * (size_t)b;
        for (int k = 0; k < 3; ++k)
            if (hb[k] < -kCoordLimit || hb[3 + k] > kCoordLimit || hb[k] > hb[3 + k])
                return std::string(what) + " " + std::to_string(b) +
                       ": coordinates / cell_size exceed the +-2^19 cell range (NaN or huge coordinates?)";
        Box& x = boxes[(size_t)b];
        const long long nx = (long long)hb[3] - hb[0] + 1, ny = (long long)hb[4] - hb[1] + 1, nz = (long long)hb[5] - hb[2] + 1;
        x.cells = nx * ny * nz;
        if (x.cells > kMaxDenseCells)
            return std::string(what) + " " + std::to_string(b) + ": bounding box of " + std::to_string(x.cells) +
                   " cells is too large for a dense grid at this cell size (pairs use dense grids only)";
        x.ox = hb[0]; x.oy = hb[1]; x.oz = hb[2];
        x.nx = (int)nx; x.ny = (int)ny; x.nz = (int)nz;
        x.cell_off = off;
        off += x.cells;
        if (off > kMaxCells)
            return std::string(what) + " grids of one call exceed 2^30 dense cells in total (int32 cell ids)";
    }
    *total_cells = off;
    return std::string();
}

}  // namespace arena_plan
