// loop_plan.hpp - how the source slots of a run are cut into blocks of the iteration kernel (host logic, no CUDA).
//
// One block = one tile of `tile` <= block_threads consecutive source slots per pass (the OpenMP loop body of
// icp_test_runner.cpp:1714-1863, one slot per thread).  Every phase of the kernel is a latency chain per tile, so:
//   * a single run keeps all its tiles resident at once (<= 3 blocks per SM; more slots: the blocks loop over tiles);
//   * a single run of a SMALL cloud (fewer 256-slot tiles than SMs) is cut into >= 2 tiles per SM at 32-slot
//     granularity instead of leaving most SMs idle - measured 45.6 -> 36.0 us per iteration on the shipped 7 562-point
//     cloud on an H100 (with an earlier build that could force the tile size); no effect once there is a tile per SM;
//   * batched trials (grid y = trial) are throughput-bound: full tiles, at most 64 blocks per trial;
//   * a batch of different scans (ragged slot counts) follows its largest scan (plan_scan_tiles).
// Also which instantiation of the iteration kernel a plan runs (variant), with how much shared memory (smem_class).
// tests/test_host_la.py::test_loop_tile_plan and tests/test_scan_plan.py check the invariants on the CPU.
#pragma once
#include <algorithm>

namespace loop_plan {

struct Tiles {
    int tile;            // source slots per block and pass, 32 <= tile <= block_threads
    long long grid_x;    // blocks per trial
};

// reserved: resident slots a single run keeps for blocks without a tile (the solver block), not counted in grid_x.
inline Tiles plan_tiles(long long slots, int trials, int sm_count, int block_threads, int reserved = 0) {
    Tiles t{block_threads, std::max<long long>(1, (slots + block_threads - 1) / block_threads)};
    if (trials != 1) {
        t.grid_x = std::min<long long>(t.grid_x, 64);
        return t;
    }
    const long long cap = (long long)sm_count * 3 - reserved;
    if (t.grid_x > cap) { t.grid_x = cap; return t; }
    int tile = block_threads;
    if (t.grid_x < sm_count) tile = (int)std::max<long long>(32, (slots / (2LL * sm_count) + 31) / 32 * 32);
    if (tile < 32 || tile > block_threads || (slots + tile - 1) / tile > cap) tile = block_threads;
    t.tile = tile;
    t.grid_x = std::max<long long>(1, (slots + tile - 1) / tile);
    return t;
}

// A batch of different scans (trial = one scan with its own slot count, dcreg_icp_run_scans): one grid for all of them,
// sized by the largest scan with the batch rule above (full tiles, at most 64 blocks per trial), also for one scan.
// Block tb of scan b takes the tiles tb, tb + grid_x, ... below n_b; a block with tb * tile >= n_b takes none and only
// contributes a zero row to its scan's reduction.
inline Tiles plan_scan_tiles(long long max_slots, int block_threads) {
    return plan_tiles(max_slots, 2, 0, block_threads);
}

// The instantiations icp_iter2_kernel<kUseWd, kGrids, kSeq, kPlanes, kSparse> a plan can run.  Variants 0-15 are the
// loop bodies: bit 0 kUseWd, bit 1 kGrids, bit 2 kSeq, bit 3 kSparse.  16 and 17 are seam 1 (kPlanes, dcreg_find_planes)
// on a dense grid and on a sparse index, with no grid table, no lanes and no weight derivative.
struct Variant { bool use_wd, grids, seq, planes, sparse; };
constexpr int kVariants = 18;
constexpr Variant variant_flags(int v) {
    return v < 16 ? Variant{(v & 1) != 0, (v & 2) != 0, (v & 4) != 0, false, (v & 8) != 0}
                  : Variant{false, false, false, true, v == 17};
}

// The variant of a plan: planes_out set (seam 1), sparse row indexes, every trial its own grid (grid_table), sequence
// lanes, the weight derivative.  -1: seam 1 of a batch, which has none (plan_iteration refuses it before it asks).
constexpr int variant(bool planes, bool sparse, bool grid_table, bool lanes, bool use_wd) {
    if (planes) return grid_table || lanes ? -1 : 16 + (sparse ? 1 : 0);
    return (use_wd ? 1 : 0) + (grid_table ? 2 : 0) + (lanes ? 4 : 0) + (sparse ? 8 : 0);
}

// A variant's dynamic shared memory: Iter2Smem up to its per-trial grid copy, which only kGrids reads, up to odometry's
// radius fields, which only kGrids && kSeq reads, or all of it
enum SmemClass { kSmemNoGrid, kSmemGrid, kSmemFull };
constexpr SmemClass smem_class(int v) {
    return !variant_flags(v).grids ? kSmemNoGrid : variant_flags(v).seq ? kSmemFull : kSmemGrid;
}

}  // namespace loop_plan
