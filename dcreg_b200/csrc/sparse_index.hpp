// sparse_index.hpp - the sparse row index of a cloud whose cell bounding box is too large for a dense grid: the
// context's target (dcreg_set_target_sparse), odometry's local maps and dcreg_icp_run_pairs' targets
// (dcreg_set_sparse_maps), each a cloud of a grid arena built by build_sparse_arena.
//
// The loop's searches never read a cell's own table entry: they read cell_start of a row (z, y) at two x positions and
// scan the contiguous point range between them, [x0, x1) with x1 - x0 <= 2K + 1 <= kReach (K = rings <= 4).  The index
// keeps exactly that contract without the box:
//   * points ordered by cell (z, y, x), x fastest, then by original index: the dense grid's order of the same points;
//   * cs(z, y, x) = the number of points whose cell comes before (z, y, x) in that order (what cell_start holds on a
//     dense grid);
//   * an open-addressing table keyed by (z, y, x) that holds cs for every x of a row within [x' - kBack, x' + kReach]
//     of an occupied cell x' of that row (clipped to the box's [0, nx]).  A range of width <= kReach that holds an
//     occupied cell has both ends in the table, so a range is [cs(x0), cs(x1)) when both lookups hit and empty
//     otherwise.
// Coordinates are box-local (cell minus the box's minimum corner): every one lies in [0, 2^21), so a cell packs into
// 63 bits with z in the high bits and the keys' order is the point order.  Plain C++ (host and
// device): tests/test_sparse_index_twin.py builds it with tools/test_sparse_index.cpp.
#pragma once
#include <cstdint>

#ifdef __CUDACC__
#define SPARSE_HD __host__ __device__ __forceinline__
#else
#define SPARSE_HD inline
#endif

namespace sparse_index {

constexpr int kReach = 9;                            // widest range a search reads: 2 K + 1 cells, K <= 4
constexpr int kBack = kReach - 1;                    // an occupied cell x' puts x in [x' - kBack, x' + kReach]
constexpr int kBits = 21;                            // per box-local coordinate (the box spans at most 2^20 + 1 cells)
constexpr unsigned long long kEmpty = ~0ull;         // free table slot (never a 63-bit key)

// key of box-local cell (x, y, z): z, then y, then x, most significant first
SPARSE_HD unsigned long long key(int x, int y, int z) {
    return ((unsigned long long)(unsigned)z << (2 * kBits)) | ((unsigned long long)(unsigned)y << kBits) |
           (unsigned long long)(unsigned)x;
}
SPARSE_HD unsigned long long row_of(unsigned long long k) { return k >> kBits; }
SPARSE_HD int x_of(unsigned long long k) { return (int)(k & ((1ull << kBits) - 1ull)); }

// The entries the occupied cell of key k adds to its row, [*lo, *hi] (empty when *lo > *hi): its dilation clipped to
// [0, nx], minus what the previous occupied cell of the order (key prev; kEmpty: none) already covers when it lies in
// the same row.  Every (row, x) of the table is added by exactly one cell.
SPARSE_HD void new_entries(unsigned long long k, unsigned long long prev, int nx, int* lo, int* hi) {
    const int x = x_of(k);
    int a = x - kBack < 0 ? 0 : x - kBack;
    const int b = x + kReach > nx ? nx : x + kReach;
    if (prev != kEmpty && row_of(prev) == row_of(k)) {
        const int px = x_of(prev);
        const int pb = px + kReach > nx ? nx : px + kReach;
        if (pb + 1 > a) a = pb + 1;
    }
    *lo = a; *hi = b;
}

// cs of key k over the n sorted point keys: the number of them below k
SPARSE_HD long long cs(const unsigned long long* sorted, long long n, unsigned long long k) {
    long long lo = 0, hi = n;
    while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if (sorted[mid] < k) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// first probe of key k in a table of mask + 1 slots (MurmurHash3's 64-bit finaliser)
SPARSE_HD unsigned int slot(unsigned long long k, unsigned int mask) {
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
    return (unsigned int)k & mask;
}

// table slots for `entries` entries: a power of two at least twice the count (and at least 1024)
inline long long capacity(long long entries) {
    long long cap = 1024;
    while (cap < 2 * entries) cap <<= 1;
    return cap;
}

constexpr long long kMaxSlots = 1ll << 32;           // Grid::mask is 32 bits

// The tables of n clouds side by side in one buffer (a sparse arena: the context's target is n = 1, and its one
// table is capacity(entries[0]) slots at offset 0): cloud b's table is slots [off[b], off[b] + cap[b]), cap[b] = capacity(entries[b]);
// off has n + 1 entries, off[n] the total.  Returns the first cloud whose table would need more than kMaxSlots slots
// (cap and off then hold the clouds before it), or -1.
inline int layout(int n, const unsigned long long* entries, long long* cap, long long* off) {
    off[0] = 0;
    for (int b = 0; b < n; ++b) {
        cap[b] = capacity((long long)entries[b]);
        if (cap[b] > kMaxSlots) return b;
        off[b + 1] = off[b] + cap[b];
    }
    return -1;
}

}  // namespace sparse_index
