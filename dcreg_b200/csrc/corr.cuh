// corr.cuh - device correspondence stage: uniform-grid exact 5-NN within radius + 5x3 plane fit.
//
// Replaces (reference file:line):
//   ICPContext::setTargetCloud kd-tree build           DCReg/include/utils.hpp:393-424
//   kdtree.nearestKSearch(q, 5) + 5th-NN radius gate   DCReg/src/icp_test_runner.cpp:1720-1726
//   5x3 colPivHouseholderQr plane fit + gates          icp_test_runner.cpp:1727-1773
//
// The reference's accept rule is "the 5th nearest neighbour is closer than the search radius".
// With cubic cells of edge = radius, every point closer than the radius to q lies in the 27 cells
// around q's cell, so an exact 5-NN over those cells reproduces the accept set of the kd-tree
// (SURVEY.md §7 step 6).  Distances are float32 sums of float32 squared differences, as in FLANN's
// L2_Simple functor that PCL's KdTreeFLANN uses; ties are broken by original point index.
//
// Layout in HBM: target points grouped by cell (float4: x, y, z, bit-cast original index).
//   dense mode : cells of the target's bounding box in x-fastest linear order + cell_start[ncells + 1];
//                the 3 x-adjacent cells of a row are ONE contiguous point range, so a query scans 9 ranges.
//   sparse mode: (a bounding box of more than arena_plan::kMaxDenseCells cells) the dense order of the points, and
//                cell_start only where a search can read it: a table of row starts (sparse_index.hpp) replaces the
//                box's table, so the searches run the dense traversal with one table lookup per range end.  One build,
//                the sparse_seg_* kernels below, serves dcreg_set_target (one cloud), odometry's local maps and
//                dcreg_icp_run_pairs' targets (one cloud each).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "cr_fp64.cuh"
#include "small_la.cuh"
#include "sparse_index.hpp"

namespace corr {

constexpr unsigned long long kEmptyKey = ~0ull;

struct Grid {
    float4* pts;                // n target points grouped by cell
    int* pos_of;                // [n] position in pts of the point with original index i (inverse of pts[j].w)
    int n;
    int dense;                  // 1: dense mode, kSparseGrid: sparse mode
    int rings;                  // ceil(search radius / cell edge): cells per direction a query must look at
    double inv_cell;            // 1 / cell edge
    // dense mode (sparse mode: the box, no cell_start)
    int ox, oy, oz;             // cell coordinates of the bounding box's minimum corner
    int nx, ny, nz;
    int* cell_start;            // [nx*ny*nz + 1]
    // sparse mode: the row-start table
    unsigned long long* keys;   // capacity entries: sparse_index::key of (x, y, z) box-local, sparse_index::kEmpty = free
    int* hstart;                // capacity: cs of the key's cell
    unsigned int mask;          // capacity - 1 (capacity is a power of two)
};

constexpr int kSparseGrid = 2;  // Grid::dense of the sparse row index

__host__ __device__ __forceinline__ int cell_coord(float v, double inv_cell) {
    return (int)floor((double)v * inv_cell);
}

__host__ __device__ __forceinline__ unsigned long long pack_key(int ix, int iy, int iz) {
    const long long B = 1ll << 20;
    return ((unsigned long long)(ix + B) << 42) | ((unsigned long long)(iy + B) << 21) | (unsigned long long)(iz + B);
}

__host__ __device__ __forceinline__ unsigned int hash_key(unsigned long long k) {
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
    return (unsigned int)k;
}

__device__ __forceinline__ int dense_index(const Grid& g, int cx, int cy, int cz) {
    return ((cz - g.oz) * g.ny + (cy - g.oy)) * g.nx + (cx - g.ox);
}

// ---- build: the dense grids of one or many clouds in one set of buffers (arena_plan.hpp) --------------------------
// segment of point i of a concatenation: the largest b with seg[b] <= i
__device__ __forceinline__ int segment_of(const long long* __restrict__ seg, int nseg, long long i) {
    int lo = 0, hi = nseg;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (seg[mid] <= i) lo = mid; else hi = mid;
    }
    return lo;
}

// cell bounds per segment: grid y = segment b (points [seg[b], seg[b+1])); bounds[6 b ..] = min cell coords (x, y, z),
// then max cell coords (initialised to +-2^30 by the host)
__global__ void grid_bounds_seg_kernel(const float4* __restrict__ pts, const long long* __restrict__ seg, double inv_cell,
                                       int* __restrict__ bounds) {
    const int b = blockIdx.y;
    const long long e = seg[b + 1];
    int lo[3] = {1 << 30, 1 << 30, 1 << 30}, hi[3] = {-(1 << 30), -(1 << 30), -(1 << 30)};
    for (long long i = seg[b] + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < e; i += (long long)gridDim.x * blockDim.x) {
        const float4 p = pts[i];
        const int c[3] = {cell_coord(p.x, inv_cell), cell_coord(p.y, inv_cell), cell_coord(p.z, inv_cell)};
        for (int k = 0; k < 3; ++k) { lo[k] = min(lo[k], c[k]); hi[k] = max(hi[k], c[k]); }
    }
    for (int k = 0; k < 3; ++k) {
        for (int off = 16; off > 0; off >>= 1) {
            lo[k] = min(lo[k], __shfl_xor_sync(0xffffffffu, lo[k], off));
            hi[k] = max(hi[k], __shfl_xor_sync(0xffffffffu, hi[k], off));
        }
        if ((threadIdx.x & 31) == 0) { atomicMin(&bounds[6 * b + k], lo[k]); atomicMax(&bounds[6 * b + 3 + k], hi[k]); }
    }
}

// cell id of a point and the per-cell counts: the global cell id is the point's segment's first cell (cell_off) plus
// its dense linear index in that segment's own box (grids[b])
__global__ void grid_count_seg_kernel(const float4* __restrict__ pts, int n, const long long* __restrict__ seg, int nseg,
                                      const Grid* __restrict__ grids, const int* __restrict__ cell_off,
                                      int* __restrict__ pt_cell, int* __restrict__ counts) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int b = segment_of(seg, nseg, i);
    const Grid& g = grids[b];
    const float4 p = pts[i];
    const int c = cell_off[b] + dense_index(g, cell_coord(p.x, g.inv_cell), cell_coord(p.y, g.inv_cell), cell_coord(p.z, g.inv_cell));
    pt_cell[i] = c;
    atomicAdd(&counts[c], 1);
}

// exclusive scan of an int array, three phases (tile sums, scan of tile sums, tile rescan)
constexpr int kScanTile = 2048;   // 256 threads x 8
__global__ void scan_tile_sums_kernel(const int* __restrict__ in, int n, int* __restrict__ tile_sums) {
    __shared__ int sh[256];
    const long long base = (long long)blockIdx.x * kScanTile;
    int s = 0;
    for (int k = 0; k < 8; ++k) {
        const long long idx = base + threadIdx.x * 8 + k;
        if (idx < n) s += in[idx];
    }
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int off = 128; off > 0; off >>= 1) {
        if (threadIdx.x < off) sh[threadIdx.x] += sh[threadIdx.x + off];
        __syncthreads();
    }
    if (threadIdx.x == 0) tile_sums[blockIdx.x] = sh[0];
}
__global__ void scan_tile_offsets_kernel(int* tile_sums, int ntiles) {   // single block, 1024 threads
    __shared__ int sh[1024];
    __shared__ int carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < ntiles; base += 1024) {
        const int idx = base + threadIdx.x;
        const int v = idx < ntiles ? tile_sums[idx] : 0;
        sh[threadIdx.x] = v;
        __syncthreads();
        for (int off = 1; off < 1024; off <<= 1) {
            const int t = threadIdx.x >= off ? sh[threadIdx.x - off] : 0;
            __syncthreads();
            sh[threadIdx.x] += t;
            __syncthreads();
        }
        if (idx < ntiles) tile_sums[idx] = carry + sh[threadIdx.x] - v;   // exclusive
        __syncthreads();
        if (threadIdx.x == 1023) carry += sh[1023];
        __syncthreads();
    }
}
__global__ void scan_tile_apply_kernel(const int* __restrict__ in, int n, const int* __restrict__ tile_offsets,
                                       int* __restrict__ out) {
    __shared__ int sh[256];
    const long long base = (long long)blockIdx.x * kScanTile;
    int loc[8];
    int s = 0;
    for (int k = 0; k < 8; ++k) {
        const long long idx = base + threadIdx.x * 8 + k;
        loc[k] = idx < n ? in[idx] : 0;
        s += loc[k];
    }
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int off = 1; off < 256; off <<= 1) {
        const int t = threadIdx.x >= off ? sh[threadIdx.x - off] : 0;
        __syncthreads();
        sh[threadIdx.x] += t;
        __syncthreads();
    }
    int run = tile_offsets[blockIdx.x] + sh[threadIdx.x] - s;
    for (int k = 0; k < 8; ++k) {
        const long long idx = base + threadIdx.x * 8 + k;
        if (idx < n) out[idx] = run;
        run += loc[k];
    }
}

// scatter points into their cell's range; `start` is the exclusive scan of the per-cell counts
__global__ void grid_scatter_kernel(const float4* __restrict__ pts, int n, const int* __restrict__ pt_cell,
                                    const int* __restrict__ start, int* __restrict__ fill, float4* __restrict__ out,
                                    int keep_w) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int c = pt_cell[i];
    const int pos = start[c] + atomicAdd(&fill[c], 1);
    float4 p = pts[i];
    if (!keep_w) p.w = __int_as_float(i);
    out[pos] = p;
}

// Deterministic order inside every cell: ascending original index.  The scatter above fills a cell in atomic-arrival
// order; this pass moves every point to (cell start + number of points of its cell with a smaller index).  One thread
// per point, O(points in its cell) reads of a range its neighbours read too - parallel over POINTS, so a cell with
// thousands of points (dense map, cell = search radius) no longer serialises on one thread the way a per-cell insertion
// sort does.  `cell_of` is indexed by the original point index (p.w).
__global__ void grid_rank_cells_kernel(const float4* __restrict__ in, int n, const int* __restrict__ cell_of,
                                       const int* __restrict__ start, float4* __restrict__ out, int* __restrict__ pos_of) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const float4 p = in[j];
    const int me = __float_as_int(p.w);
    const int c = cell_of[me];
    const int s = start[c];
    const int e = start[c + 1];
    int rank = 0;
    for (int k = s; k < e; ++k) rank += (__float_as_int(__ldg(&in[k].w)) < me) ? 1 : 0;
    out[s + rank] = p;
    if (pos_of) pos_of[me] = s + rank;
}

// cell of a (transformed) source point for the spatial sort of the source cloud, clamped into the target box
// (T: the first 12 entries of a row-major 4x4 pose)
__device__ __forceinline__ int source_cell(const Grid& g, const double* __restrict__ T, float4 p) {
    const double px = p.x, py = p.y, pz = p.z;
    const float qx = (float)(T[0] * px + T[1] * py + T[2] * pz + T[3]);
    const float qy = (float)(T[4] * px + T[5] * py + T[6] * pz + T[7]);
    const float qz = (float)(T[8] * px + T[9] * py + T[10] * pz + T[11]);
    const int cx = min(max(cell_coord(qx, g.inv_cell) - g.ox, 0), g.nx - 1);
    const int cy = min(max(cell_coord(qy, g.inv_cell) - g.oy, 0), g.ny - 1);
    const int cz = min(max(cell_coord(qz, g.inv_cell) - g.oz, 0), g.nz - 1);
    return (cz * g.ny + cy) * g.nx + cx;
}

__global__ void source_cell_kernel(const float4* __restrict__ src, int n, Grid g, const double* __restrict__ T,
                                   int* __restrict__ pt_cell, int* __restrict__ counts) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int c = source_cell(g, T, src[i]);
    pt_cell[i] = c;
    atomicAdd(&counts[c], 1);
}

// ---- build: the sparse row indexes (sparse_index.hpp) of one or many clouds in one arena (segment b: points [seg[b],
// seg[b+1]), its index grids[b], box fields set).  A cloud's box-local key takes 63 bits, so the cloud id does not fit
// beside it: the order (cloud, z, y, x, index) comes from two stable passes.  Pass 0: key (y, x) of point i = j; pass
// 1: key (cloud, z) of point i = order[j], the order pass 0 left.
__global__ void sparse_seg_key_kernel(const float4* __restrict__ pts, int n, const long long* __restrict__ seg, int nseg,
                                      const Grid* __restrict__ grids, int pass, const int* __restrict__ order,
                                      unsigned long long* __restrict__ keys, int* __restrict__ vals) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const int i = pass ? order[j] : j;
    const int b = segment_of(seg, nseg, i);
    const Grid& g = grids[b];
    const float4 p = pts[i];
    if (pass == 0)
        keys[j] = sparse_index::key(cell_coord(p.x, g.inv_cell) - g.ox, cell_coord(p.y, g.inv_cell) - g.oy, 0);
    else
        keys[j] = ((unsigned long long)b << sparse_index::kBits) | (unsigned long long)(cell_coord(p.z, g.inv_cell) - g.oz);
    vals[j] = i;
}

// the points in sort order (w = index over all clouds, as arena_fill leaves it), the inverse permutation, and the
// box-local key of every sorted position in its cloud's box (sorted positions keep the clouds' segments)
__global__ void sparse_seg_gather_kernel(const float4* __restrict__ pts, const int* __restrict__ order, int n,
                                         const long long* __restrict__ seg, int nseg, const Grid* __restrict__ grids,
                                         float4* __restrict__ out, int* __restrict__ pos_of,
                                         unsigned long long* __restrict__ sorted) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const int i = order[j];
    const Grid& g = grids[segment_of(seg, nseg, j)];
    float4 p = pts[i];
    sorted[j] = sparse_index::key(cell_coord(p.x, g.inv_cell) - g.ox, cell_coord(p.y, g.inv_cell) - g.oy,
                                  cell_coord(p.z, g.inv_cell) - g.oz);
    p.w = __int_as_float(i);
    out[j] = p;
    pos_of[i] = j;
}

// every cloud's table entries (sparse_index::new_entries within its segment), summed into count[b]
__global__ void sparse_seg_count_kernel(const unsigned long long* __restrict__ sorted, int n,
                                        const long long* __restrict__ seg, int nseg, const Grid* __restrict__ grids,
                                        unsigned long long* __restrict__ count) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    int b = nseg - 1;
    unsigned c = 0;
    if (j < n) {
        b = segment_of(seg, nseg, j);
        const long long first = seg[b];
        if (j == first || sorted[j - 1] != sorted[j]) {
            int lo, hi;
            sparse_index::new_entries(sorted[j], j > first ? sorted[j - 1] : sparse_index::kEmpty, grids[b].nx, &lo, &hi);
            if (hi >= lo) c = (unsigned)(hi - lo + 1);
        }
    }
    const unsigned peers = __match_any_sync(0xffffffffu, b);
    c = __reduce_add_sync(peers, c);
    if ((int)(threadIdx.x & 31) == __ffs(peers) - 1 && c) atomicAdd(&count[b], (unsigned long long)c);
}

// ... and their cs in every cloud's own table, shifted by the cloud's first position
__global__ void sparse_seg_insert_kernel(const unsigned long long* __restrict__ sorted, int n,
                                         const long long* __restrict__ seg, int nseg, const Grid* __restrict__ grids) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const int b = segment_of(seg, nseg, j);
    const long long first = seg[b];
    if (j > first && sorted[j - 1] == sorted[j]) return;
    const Grid& g = grids[b];
    int lo, hi;
    sparse_index::new_entries(sorted[j], j > first ? sorted[j - 1] : sparse_index::kEmpty, g.nx, &lo, &hi);
    const unsigned long long row = sparse_index::row_of(sorted[j]) << sparse_index::kBits;
    for (int x = lo; x <= hi; ++x) {
        const unsigned long long k = row | (unsigned long long)x;
        unsigned int s = sparse_index::slot(k, g.mask);
        while (atomicCAS(&g.keys[s], sparse_index::kEmpty, k) != sparse_index::kEmpty) s = (s + 1) & g.mask;
        g.hstart[s] = (int)(first + sparse_index::cs(sorted + first, seg[b + 1] - first, k));
    }
}

// cs of box-local cell (x, yy, zz) of a sparse grid, or -1 when the table has no entry for it
__device__ __forceinline__ int sparse_cs(const Grid& g, int zz, int yy, int x) {
    const unsigned long long k = sparse_index::key(x, yy, zz);
    unsigned int s = sparse_index::slot(k, g.mask);
    while (true) {
        const unsigned long long kk = __ldg(&g.keys[s]);
        if (kk == k) return __ldg(&g.hstart[s]);
        if (kk == sparse_index::kEmpty) return -1;
        s = (s + 1) & g.mask;
    }
}

// point range of the cells [x0, x1) of row (yy, zz) of a sparse grid (x1 - x0 <= sparse_index::kReach): a range that
// holds a point has both ends in the table
__device__ __forceinline__ void sparse_span(const Grid& g, int zz, int yy, int x0, int x1, int& s, int& e) {
    s = sparse_cs(g, zz, yy, x0);
    e = sparse_cs(g, zz, yy, x1);
    if (s < 0 || e < 0) { s = 0; e = 0; }
}

// ---- query -----------------------------------------------------------------------------------
// The five best so far, ascending.  key = (bits of the squared distance) << 32 | original index: squared distances are
// non-negative floats, whose bit patterns order like unsigned integers, so ONE 64-bit unsigned compare is the (distance,
// then index) rule of the reference's tie handling - two instructions instead of four per compare in the insertion that
// dominates the per-thread search (ncu, lean iterations: 30 % of all warp instructions on that compare).
// The list carries no positions: a neighbour's position in g.pts is looked up from its index once, when the search is
// over (Grid::pos_of) - one register and two moves per insertion step less.
struct Knn5 {
    unsigned long long key[5];
};

__device__ __forceinline__ unsigned long long knn_key(float d2, int idx) {
    return ((unsigned long long)__float_as_uint(d2) << 32) | (unsigned long long)(unsigned)idx;
}
__device__ __forceinline__ float knn_d2(const Knn5& k, int i) { return __uint_as_float((unsigned)(k.key[i] >> 32)); }
// positions of the five (-1 where the list still holds a sentinel): five independent loads, one round trip
__device__ __forceinline__ void knn_positions(const Grid& g, const Knn5& k, int (&pos)[5]) {
#pragma unroll
    for (int i = 0; i < 5; ++i) {
        const int idx = (int)(unsigned)(k.key[i] & 0xffffffffull);
        pos[i] = idx == 0x7fffffff ? -1 : __ldg(&g.pos_of[idx]);
    }
}

__device__ __forceinline__ void knn_init(Knn5& k) {
#pragma unroll
    for (int i = 0; i < 5; ++i) k.key[i] = knn_key(3.0e38f, 0x7fffffff);
}

__device__ __forceinline__ void knn_insert(Knn5& k, unsigned long long key) {
    k.key[4] = key;
#pragma unroll
    for (int i = 4; i > 0; --i) {
        if (k.key[i] < k.key[i - 1]) { const unsigned long long tk = k.key[i]; k.key[i] = k.key[i - 1]; k.key[i - 1] = tk; }
    }
}

// FLANN L2_Simple: float differences, float accumulation, x then y then z (no FMA contraction)
__device__ __forceinline__ float dist2(float qx, float qy, float qz, const float4& p) {
    const float ex = __fsub_rn(qx, p.x), ey = __fsub_rn(qy, p.y), ez = __fsub_rn(qz, p.z);
    return __fadd_rn(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)), __fmul_rn(ez, ez));
}

__device__ __forceinline__ void knn_scan_range(const float4* __restrict__ pts, int s, int e, float qx, float qy,
                                               float qz, Knn5& k) {
    int j = s;
#pragma unroll 1
    for (; j + 3 < e; j += 4) {                       // four candidates per trip: four loads in flight (the scan is one
        const float4 p0 = __ldg(&pts[j]), p1 = __ldg(&pts[j + 1]), p2 = __ldg(&pts[j + 2]), p3 = __ldg(&pts[j + 3]);   // thread's latency chain)
        const unsigned long long k0 = knn_key(dist2(qx, qy, qz, p0), __float_as_int(p0.w)), k1 = knn_key(dist2(qx, qy, qz, p1), __float_as_int(p1.w));
        const unsigned long long k2 = knn_key(dist2(qx, qy, qz, p2), __float_as_int(p2.w)), k3 = knn_key(dist2(qx, qy, qz, p3), __float_as_int(p3.w));
        if (k0 < k.key[4]) knn_insert(k, k0);
        if (k1 < k.key[4]) knn_insert(k, k1);
        if (k2 < k.key[4]) knn_insert(k, k2);
        if (k3 < k.key[4]) knn_insert(k, k3);
    }
#pragma unroll 1
    for (; j < e; ++j) {
        const float4 p0 = __ldg(&pts[j]);
        const unsigned long long k0 = knn_key(dist2(qx, qy, qz, p0), __float_as_int(p0.w));
        if (k0 < k.key[4]) knn_insert(k, k0);
    }
}

// kSparse: g is a sparse row index (Grid::dense == kSparseGrid): the dense traversal, each range read from its table
template <bool kSparse = false>
__device__ __forceinline__ void knn_search(const Grid& g, float qx, float qy, float qz, Knn5& k) {
    const int cx = cell_coord(qx, g.inv_cell), cy = cell_coord(qy, g.inv_cell), cz = cell_coord(qz, g.inv_cell);
    // K = ceil(radius / cell) rings of cells cover the search radius (K = 1 when cell = radius; a finer grid,
    // cell = radius / 2, K = 2, scans ~3x fewer candidates because most cells are pruned by their box distance).
    // Rows (dy, dz) are visited in rings of growing max(|dy|, |dz|); inside a row the own column first, then
    // outwards.  A row / cell is skipped only when its box distance exceeds the current 5th-best distance
    // (strictly, with a 1e-5 relative margin for the float arithmetic of the bound), so the search stays exact.
    // Loops are deliberately NOT unrolled: one copy of the scan loop keeps the kernel inside the instruction
    // cache (a fully unrolled version stalls on instruction fetch).
    const int K = g.rings;
    const float cell = (float)(1.0 / g.inv_cell);
    const int lx = cx - g.ox, ly = cy - g.oy, lz = cz - g.oz;
    if (lx + K < 0 || lx - K >= g.nx) return;
    // position inside the own cell, in [0, cell) up to float rounding of cx * cell: every gap below is shrunk
    // by an absolute eps that covers that rounding, so a bound can only be too small (never prunes a hit)
    const float eps = 2e-6f * (fabsf(qx) + fabsf(qy) + fabsf(qz) + cell);
    const float fx = qx - (float)cx * cell, fy = qy - (float)cy * cell, fz = qz - (float)cz * cell;
    if (K == 1) {
        // cell = search radius (the usual set-up): 9 rows of 3 cells, own row first, rows pruned by the same test
        // as the general loop below; a visited row costs one fetch of its two outer cell boundaries and one scan
        // (the lanes of a warp prune differently, so a warp walks nearly all 27 cells and every dependent load is
        // on its critical path).
        const int xa = min(max(lx - 1, 0), g.nx), xd = min(max(lx + 2, 0), g.nx);
#pragma unroll 1
        for (int r = 0; r < 9; ++r) {
            // own row first, then the ring: (dz, dy) = (-1,-1) (-1,0) (-1,1) (0,-1) (0,1) (1,-1) (1,0) (1,1)
            const int q = r == 0 ? 4 : (r <= 4 ? r - 1 : r);
            const int dz = q / 3 - 1, dy = q % 3 - 1;
            const int zz = lz + dz, yy = ly + dy;
            if (zz < 0 || zz >= g.nz || yy < 0 || yy >= g.ny) continue;
            const float gz = dz == 0 ? 0.0f : fmaxf((dz < 0 ? fz : cell - fz) - eps, 0.0f);
            const float gy = dy == 0 ? 0.0f : fmaxf((dy < 0 ? fy : cell - fy) - eps, 0.0f);
            const float row_lb = (gy * gy + gz * gz) * 0.99999f;
            if (row_lb > knn_d2(k, 4)) continue;
            const int* rowp = g.cell_start + (size_t)(zz * g.ny + yy) * g.nx;
            // A row's three cells are one contiguous range: scanned in one pass, four loads in flight across the
            // cell boundaries (~3 points per cell on a surface at cell = radius, so three separate passes spent
            // most of their time in single-candidate trips, one memory round trip each).  The left / right cells
            // are no longer pruned: their box-distance test only ever skips cells holding nothing below the
            // current 5th key, so scanning them too leaves the list unchanged, bit for bit.
            if constexpr (kSparse) {
                int s, e;
                sparse_span(g, zz, yy, xa, xd, s, e);
                knn_scan_range(g.pts, s, e, qx, qy, qz, k);
            } else {
                knn_scan_range(g.pts, __ldg(rowp + xa), __ldg(rowp + xd), qx, qy, qz, k);
            }
        }
        return;
    }
#pragma unroll 1
    for (int ring = 0; ring <= K; ++ring) {
        // a whole ring is at least (ring - 1) * cell + (distance to the own cell's nearest face) away
        if (ring > 1) {
            const float m = fmaxf(fminf(fminf(fy, cell - fy), fminf(fz, cell - fz)) + (float)(ring - 1) * cell - eps, 0.0f);
            if (m * m * 0.99999f > knn_d2(k, 4)) break;
        }
#pragma unroll 1
        for (int dz = -ring; dz <= ring; ++dz) {
            const int zz = lz + dz;
            if (zz < 0 || zz >= g.nz) continue;
            const float gz = dz == 0 ? 0.0f : fmaxf((dz < 0 ? fz + (float)(-dz - 1) * cell : (cell - fz) + (float)(dz - 1) * cell) - eps, 0.0f);
            const int stepy = (dz == -ring || dz == ring) ? 1 : 2 * ring;     // only the ring's boundary rows
#pragma unroll 1
            for (int dy = -ring; dy <= ring; dy += (stepy > 0 ? stepy : 1)) {
                const int yy = ly + dy;
                if (yy < 0 || yy >= g.ny) continue;
                const float gy = dy == 0 ? 0.0f : fmaxf((dy < 0 ? fy + (float)(-dy - 1) * cell : (cell - fy) + (float)(dy - 1) * cell) - eps, 0.0f);
                const float row_lb = (gy * gy + gz * gz) * 0.99999f;
                if (row_lb > knn_d2(k, 4)) continue;
                const int* rowp = g.cell_start + (size_t)(zz * g.ny + yy) * g.nx;
                // own column, then +-1, +-2, ... : stop a side once its gap bound exceeds the 5th-best distance
                {
                    const int x0 = min(max(lx, 0), g.nx), x1 = min(max(lx + 1, 0), g.nx);
                    if constexpr (kSparse) {
                        int s, e;
                        sparse_span(g, zz, yy, x0, x1, s, e);
                        knn_scan_range(g.pts, s, e, qx, qy, qz, k);
                    } else {
                        knn_scan_range(g.pts, __ldg(rowp + x0), __ldg(rowp + x1), qx, qy, qz, k);
                    }
                }
#pragma unroll 1
                for (int dx = 1; dx <= K; ++dx) {
                    const float gl = fmaxf(fx + (float)(dx - 1) * cell - eps, 0.0f);
                    const float gr = fmaxf((cell - fx) + (float)(dx - 1) * cell - eps, 0.0f);
                    const bool left = (row_lb + gl * gl * 0.99999f) <= knn_d2(k, 4);
                    if (left) {
                        const int x0 = min(max(lx - dx, 0), g.nx), x1 = min(max(lx - dx + 1, 0), g.nx);
                        if constexpr (kSparse) {
                            int s, e;
                            sparse_span(g, zz, yy, x0, x1, s, e);
                            knn_scan_range(g.pts, s, e, qx, qy, qz, k);
                        } else {
                            knn_scan_range(g.pts, __ldg(rowp + x0), __ldg(rowp + x1), qx, qy, qz, k);
                        }
                    }
                    const bool right = (row_lb + gr * gr * 0.99999f) <= knn_d2(k, 4);
                    if (right) {
                        const int x0 = min(max(lx + dx, 0), g.nx), x1 = min(max(lx + dx + 1, 0), g.nx);
                        if constexpr (kSparse) {
                            int s, e;
                            sparse_span(g, zz, yy, x0, x1, s, e);
                            knn_scan_range(g.pts, s, e, qx, qy, qz, k);
                        } else {
                            knn_scan_range(g.pts, __ldg(rowp + x0), __ldg(rowp + x1), qx, qy, qz, k);
                        }
                    }
                    if (!left && !right) break;
                }
            }
        }
    }
}

// ---- bounded exact M-NN with a gap certificate (dense grid, one thread per query) ----------------------------------
// Same traversal as knn_search, three differences:
//   * it keeps the kSeeds (7) nearest, not 5: the first five are the answer, the extra two widen the certificate below;
//   * the list starts as sentinels at the caller's bound B (any value >= the true 7th squared distance keeps the
//     search exact: a candidate with d2 == B and a real index still beats a sentinel), so rows / cells / candidates
//     beyond B are never touched;
//   * lb collects a lower bound on the squared distance of every target point that does NOT end up in the list:
//     the d2 of every rejected or evicted candidate and the box distance of everything pruned.  The caller uses it
//     to prove, in later iterations, that the seven still contain the five nearest without searching
//     (icp_iter2_kernel).
constexpr int kSeeds = 7;

struct KnnM {                 // as Knn5: key = (bits of the squared distance) << 32 | original index, ascending
    unsigned long long key[kSeeds];
    int pos[kSeeds];
};
__device__ __forceinline__ float knn_d2(const KnnM& k, int i) { return __uint_as_float((unsigned)(k.key[i] >> 32)); }

__device__ __forceinline__ void knnm_insert(KnnM& k, unsigned long long key, int pos) {
    k.key[kSeeds - 1] = key; k.pos[kSeeds - 1] = pos;
#pragma unroll
    for (int i = kSeeds - 1; i > 0; --i) {
        if (k.key[i] < k.key[i - 1]) {
            const unsigned long long tk = k.key[i]; k.key[i] = k.key[i - 1]; k.key[i - 1] = tk;
            const int tp = k.pos[i]; k.pos[i] = k.pos[i - 1]; k.pos[i - 1] = tp;
        }
    }
}

__device__ __forceinline__ void knn_scan_range_lb(const float4* __restrict__ pts, int s, int e, float qx, float qy,
                                                  float qz, KnnM& k, float& lb) {
    constexpr int L = kSeeds - 1;
    int j = s;
#pragma unroll 1
    for (; j + 1 < e; j += 2) {                       // two candidates per trip: both loads in flight
        const float4 p0 = __ldg(&pts[j]), p1 = __ldg(&pts[j + 1]);
        const float a0 = dist2(qx, qy, qz, p0), a1 = dist2(qx, qy, qz, p1);
        const unsigned long long k0 = knn_key(a0, __float_as_int(p0.w)), k1 = knn_key(a1, __float_as_int(p1.w));
        if (k0 < k.key[L]) { lb = fminf(lb, knn_d2(k, L)); knnm_insert(k, k0, j); }
        else lb = fminf(lb, a0);                      // rejected candidates and evicted entries bound the outside
        if (k1 < k.key[L]) { lb = fminf(lb, knn_d2(k, L)); knnm_insert(k, k1, j + 1); }
        else lb = fminf(lb, a1);
    }
    if (j < e) {
        const float4 p0 = __ldg(&pts[j]);
        const float a0 = dist2(qx, qy, qz, p0);
        const unsigned long long k0 = knn_key(a0, __float_as_int(p0.w));
        if (k0 < k.key[L]) { lb = fminf(lb, knn_d2(k, L)); knnm_insert(k, k0, j); }
        else lb = fminf(lb, a0);
    }
}

template <bool kSparse = false>
__device__ __forceinline__ void knn_search_lb(const Grid& g, float qx, float qy, float qz, float B, KnnM& k, float& lb) {
    constexpr int L = kSeeds - 1;
#pragma unroll
    for (int i = 0; i < kSeeds; ++i) { k.key[i] = knn_key(B, 0x7fffffff); k.pos[i] = -1; }
    const int cx = cell_coord(qx, g.inv_cell), cy = cell_coord(qy, g.inv_cell), cz = cell_coord(qz, g.inv_cell);
    const int K = g.rings;
    const float cell = (float)(1.0 / g.inv_cell);
    const int lx = cx - g.ox, ly = cy - g.oy, lz = cz - g.oz;
    if (lx + K < 0 || lx - K >= g.nx) return;
    const float eps = 2e-6f * (fabsf(qx) + fabsf(qy) + fabsf(qz) + cell);
    const float fx = qx - (float)cx * cell, fy = qy - (float)cy * cell, fz = qz - (float)cz * cell;
#pragma unroll 1
    for (int ring = 0; ring <= K; ++ring) {
        if (ring > 1) {
            const float m = fmaxf(fminf(fminf(fy, cell - fy), fminf(fz, cell - fz)) + (float)(ring - 1) * cell - eps, 0.0f);
            if (m * m * 0.99999f > knn_d2(k, L)) { lb = fminf(lb, m * m * 0.99999f); break; }
        }
#pragma unroll 1
        for (int dz = -ring; dz <= ring; ++dz) {
            const int zz = lz + dz;
            if (zz < 0 || zz >= g.nz) continue;
            const float gz = dz == 0 ? 0.0f : fmaxf((dz < 0 ? fz + (float)(-dz - 1) * cell : (cell - fz) + (float)(dz - 1) * cell) - eps, 0.0f);
            const int stepy = (dz == -ring || dz == ring) ? 1 : 2 * ring;     // only the ring's boundary rows
#pragma unroll 1
            for (int dy = -ring; dy <= ring; dy += (stepy > 0 ? stepy : 1)) {
                const int yy = ly + dy;
                if (yy < 0 || yy >= g.ny) continue;
                const float gy = dy == 0 ? 0.0f : fmaxf((dy < 0 ? fy + (float)(-dy - 1) * cell : (cell - fy) + (float)(dy - 1) * cell) - eps, 0.0f);
                const float row_lb = (gy * gy + gz * gz) * 0.99999f;
                if (row_lb > knn_d2(k, L)) { lb = fminf(lb, row_lb); continue; }
                const int* rowp = g.cell_start + (size_t)(zz * g.ny + yy) * g.nx;
                {
                    const int x0 = min(max(lx, 0), g.nx), x1 = min(max(lx + 1, 0), g.nx);
                    if constexpr (kSparse) {
                        int s, e;
                        sparse_span(g, zz, yy, x0, x1, s, e);
                        knn_scan_range_lb(g.pts, s, e, qx, qy, qz, k, lb);
                    } else {
                        knn_scan_range_lb(g.pts, __ldg(rowp + x0), __ldg(rowp + x1), qx, qy, qz, k, lb);
                    }
                }
                bool left = true, right = true;
#pragma unroll 1
                for (int dx = 1; dx <= K; ++dx) {
                    if (left) {
                        const float gl = fmaxf(fx + (float)(dx - 1) * cell - eps, 0.0f);
                        const float b = row_lb + gl * gl * 0.99999f;
                        if (b <= knn_d2(k, L)) {
                            const int x0 = min(max(lx - dx, 0), g.nx), x1 = min(max(lx - dx + 1, 0), g.nx);
                            if constexpr (kSparse) {
                                int s, e;
                                sparse_span(g, zz, yy, x0, x1, s, e);
                                knn_scan_range_lb(g.pts, s, e, qx, qy, qz, k, lb);
                            } else {
                                knn_scan_range_lb(g.pts, __ldg(rowp + x0), __ldg(rowp + x1), qx, qy, qz, k, lb);
                            }
                        } else { lb = fminf(lb, b); left = false; }
                    }
                    if (right) {
                        const float gr = fmaxf((cell - fx) + (float)(dx - 1) * cell - eps, 0.0f);
                        const float b = row_lb + gr * gr * 0.99999f;
                        if (b <= knn_d2(k, L)) {
                            const int x0 = min(max(lx + dx, 0), g.nx), x1 = min(max(lx + dx + 1, 0), g.nx);
                            if constexpr (kSparse) {
                                int s, e;
                                sparse_span(g, zz, yy, x0, x1, s, e);
                                knn_scan_range_lb(g.pts, s, e, qx, qy, qz, k, lb);
                            } else {
                                knn_scan_range_lb(g.pts, __ldg(rowp + x0), __ldg(rowp + x1), qx, qy, qz, k, lb);
                            }
                        } else { lb = fminf(lb, b); right = false; }
                    }
                    if (!left && !right) break;
                }
            }
        }
    }
}


// ---- one query, one warp (dense grid) -----------------------------------------------------------------------------
// Same contract as knn_search_lb, executed by all 32 lanes for ONE query: used when only a few slots of a warp need a
// search, where the sequential search of one lane would keep the other 31 waiting for the whole search.  Lanes set up the cell
// rows in parallel, walk every row with stride 32 (coalesced), compact the candidates with d2 <= B into a 64-entry
// shared buffer and rank them ((d2, index) order): ranks 0..6 are the list, everything else feeds lb.
// Returns false (nothing usable) when more than 64 candidates survive the bound; the caller then searches sequentially.
constexpr int kWarpKnnCap = 64;

struct WarpKnnSmem {
    int rs[81], re[81];                              // point range per cell row (empty when pruned)
    int pref[82];                                    // exclusive prefix sums of the row lengths (+ total)
    unsigned long long key[kWarpKnnCap];             // candidates inside the bound: knn_key(d2, index), ...
    int pos[kWarpKnnCap];                            // ... and their position
    unsigned long long okey[kSeeds];                 // the list, ascending
    int opos[kSeeds];
};

// One row (r of (2K+1)^2, x-fastest over (dy, dz)) of a bounded query's set-up: the point range of the row's cells that can
// hold something within the squared bound B, and `lb`, a lower bound on the squared distance of everything it dropped
// (3e38: dropped nothing).  A tile's searches have their rows set up by ALL its threads at once before the warps start
// (icp_iter2_kernel): one memory round trip for the whole tile instead of one at the head of every search.
struct RowRange { int s, e; float lb; };

template <bool kSparse = false>
__device__ __forceinline__ RowRange knn_row_range(const Grid& g, float qx, float qy, float qz, float B, int r) {
    const int K = g.rings, W = 2 * K + 1;
    const float cell = (float)(1.0 / g.inv_cell);
    const int cx = cell_coord(qx, g.inv_cell), cy = cell_coord(qy, g.inv_cell), cz = cell_coord(qz, g.inv_cell);
    const int lx = cx - g.ox, ly = cy - g.oy, lz = cz - g.oz;
    const float eps = 2e-6f * (fabsf(qx) + fabsf(qy) + fabsf(qz) + cell);
    const float fx = qx - (float)cx * cell, fy = qy - (float)cy * cell, fz = qz - (float)cz * cell;
    RowRange out{0, 0, 3.0e38f};
    const int rz = r / W;
    const int dz = rz - K, dy = r - rz * W - K;
    const int zz = lz + dz, yy = ly + dy;
    if (zz >= 0 && zz < g.nz && yy >= 0 && yy < g.ny) {
        const float gz = dz == 0 ? 0.0f : fmaxf((dz < 0 ? fz + (float)(-dz - 1) * cell : (cell - fz) + (float)(dz - 1) * cell) - eps, 0.0f);
        const float gy = dy == 0 ? 0.0f : fmaxf((dy < 0 ? fy + (float)(-dy - 1) * cell : (cell - fy) + (float)(dy - 1) * cell) - eps, 0.0f);
        const float row_lb = (gy * gy + gz * gz) * 0.99999f;
        if (row_lb <= B) {
            int xa = lx - K, xb = lx + K;                  // drop end cells whose box distance exceeds the bound
#pragma unroll 1
            for (; xa < lx; ++xa) {
                const float gl = fmaxf(fx + (float)(lx - xa - 1) * cell - eps, 0.0f);
                const float b = row_lb + gl * gl * 0.99999f;
                if (b <= B) break;
                out.lb = fminf(out.lb, b);
            }
#pragma unroll 1
            for (; xb > lx; --xb) {
                const float gr = fmaxf((cell - fx) + (float)(xb - lx - 1) * cell - eps, 0.0f);
                const float b = row_lb + gr * gr * 0.99999f;
                if (b <= B) break;
                out.lb = fminf(out.lb, b);
            }
            xa = max(xa, 0); xb = min(xb, g.nx - 1);
            if (xa <= xb) {
                if constexpr (kSparse) {
                    sparse_span(g, zz, yy, xa, xb + 1, out.s, out.e);
                } else {
                    const int* rowp = g.cell_start + (size_t)(zz * g.ny + yy) * g.nx;
                    out.s = __ldg(rowp + xa); out.e = __ldg(rowp + xb + 1);
                }
            }
        } else {
            out.lb = row_lb;
        }
    }
    return out;
}

// prof (profiling only, may be null): [0] += cycles of the row set-up, [1] += prefix + candidate scan, [2] += selection,
// [3] += searches, [4] += candidates scanned
template <bool kSparse = false>
__device__ __forceinline__ bool knn_warp_search(const Grid& g, float qx, float qy, float qz, float B, WarpKnnSmem& S,
                                                KnnM& out, float& lb, long long* prof = nullptr, const RowRange* pre = nullptr) {
    const unsigned full = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    long long tc0 = 0, tc1 = 0, tc2 = 0;
    if (prof) tc0 = clock64();
    const int K = g.rings, W = 2 * K + 1, nrows = W * W;
    float lbl = lb;                                   // lane-local lower bound of everything this lane drops
    if (lane < kSeeds) { S.okey[lane] = knn_key(B, 0x7fffffff); S.opos[lane] = -1; }
#pragma unroll 1
    for (int r = lane; r < nrows; r += 32) {
        const RowRange rr = pre ? pre[r] : knn_row_range<kSparse>(g, qx, qy, qz, B, r);
        lbl = fminf(lbl, rr.lb);
        S.rs[r] = rr.s; S.re[r] = rr.e;
    }
    __syncwarp();
    if (prof) tc1 = clock64();
    // Candidates of ALL rows as one flat list (prefix sums of the row lengths): lane l takes candidates l, l + 32, ...
    // wherever their rows are, so the point loads of different rows are independent and in flight together (walking
    // the rows one after the other costs one dependent memory round trip per row: 9 for cell = radius, up to 81).
    int total = 0;
#pragma unroll 1
    for (int base = 0; base < nrows; base += 32) {
        const int r = base + lane;
        const int len = r < nrows ? S.re[r] - S.rs[r] : 0;
        int incl = len;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const int t = __shfl_up_sync(full, incl, off);
            if (lane >= off) incl += t;
        }
        if (r < nrows) S.pref[r] = total + incl - len;
        total += __shfl_sync(full, incl, 31);
    }
    if (lane == 0) S.pref[nrows] = total;
    __syncwarp();
    int cnt = 0;
    bool overflow = false;
    int row = 0;                                      // row of this lane's current candidate (candidates ascend per lane)
    // cell = radius (9 rows): the prefix sums in registers, so a candidate's row is nine compares instead of a walk
    // through shared memory with one dependent load per step
    const bool few_rows = nrows <= 9;
    int pr[9];
#pragma unroll
    for (int r = 0; r < 9; ++r) pr[r] = (few_rows && r < nrows) ? S.pref[r + 1] : 0x7fffffff;
    constexpr int kU = 4;                             // candidates per lane and trip: that many loads in flight
#pragma unroll 1
    for (int c0 = 0; c0 < total; c0 += 32 * kU) {
        int jj[kU];
        bool in[kU];
        float4 pp[kU];
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            const int c = c0 + u * 32 + lane;
            in[u] = c < total;
            jj[u] = 0;
            if (in[u]) {
                if (few_rows) {
                    row = 0;
#pragma unroll
                    for (int r = 0; r < 8; ++r) row += (c >= pr[r]) ? 1 : 0;
                } else {
                    while (c >= S.pref[row + 1]) ++row;
                }
                jj[u] = S.rs[row] + (c - S.pref[row]);
                pp[u] = __ldg(&g.pts[jj[u]]);
            }
        }
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            if (c0 + u * 32 >= total) break;          // (uniform) nothing left for this and the following slots
            bool hit = false;
            float d = 0.0f;
            int pi = 0;
            if (in[u]) {
                d = dist2(qx, qy, qz, pp[u]);
                pi = __float_as_int(pp[u].w);
                hit = d <= B;
                if (!hit) lbl = fminf(lbl, d);
            }
            const unsigned bits = __ballot_sync(full, hit);
            const int slot = cnt + __popc(bits & ((1u << lane) - 1u));
            if (hit && slot < kWarpKnnCap) { S.key[slot] = knn_key(d, pi); S.pos[slot] = jj[u]; }
            cnt += __popc(bits);
        }
        if (cnt > kWarpKnnCap) { overflow = true; break; }
    }
    __syncwarp();
    if (overflow) return false;
    if (prof) tc2 = clock64();
    // Rank of every candidate inside the bound = number of candidates that precede it in (d2, index) order; ranks 0..6 are
    // the list.  All-pairs over the (few: ~20 of ~45 scanned) hits with broadcast shared-memory reads: the iterations
    // are independent, so unrolled they pipeline.  Slower during development (clock64 per phase, tools/timeline.py; not
    // re-measured on H100): seven warp-wide minimum extractions with REDUX (a serial chain of collectives), this loop
    // not unrolled.
#pragma unroll 1
    for (int en = lane; en < cnt; en += 32) {
        const unsigned long long ke = S.key[en];
        int rank = 0;
#pragma unroll 4
        for (int f = 0; f < cnt; ++f) rank += (S.key[f] < ke) ? 1 : 0;
        if (rank < kSeeds) { S.okey[rank] = ke; S.opos[rank] = S.pos[en]; }
        else lbl = fminf(lbl, __uint_as_float((unsigned)(ke >> 32)));
    }
    lbl = __uint_as_float(__reduce_min_sync(full, __float_as_uint(lbl)));      // lbl >= 0: bit patterns order like the values
    __syncwarp();
#pragma unroll
    for (int i = 0; i < kSeeds; ++i) { out.key[i] = S.okey[i]; out.pos[i] = S.opos[i]; }
    lb = lbl;
    __syncwarp();
    if (prof && lane == 0) {
        const long long tc3 = clock64();
        prof[0] += tc1 - tc0; prof[1] += tc2 - tc1; prof[2] += tc3 - tc2; prof[3] += 1; prof[4] += total;
    }
    return true;
}

// ---- exact 1-NN (post-run point-to-point metrics, DCReg/include/utils.hpp:538-589) ---------------------------
// Nearest target point of q in a dense grid: rings of cells of growing Chebyshev radius around q's cell, clipped to
// the grid box, until the best distance found is no larger than the distance to the next ring.  FLANN-style float32
// squared distances.  Returns the squared distance (3e38 if the grid is empty).
__device__ __forceinline__ float nn1_search(const Grid& g, float qx, float qy, float qz) {
    const float cell = (float)(1.0 / g.inv_cell);
    const int lx = cell_coord(qx, g.inv_cell) - g.ox, ly = cell_coord(qy, g.inv_cell) - g.oy, lz = cell_coord(qz, g.inv_cell) - g.oz;
    // first ring that can touch the box, last ring that still does
    const int ox = lx < 0 ? -lx : (lx >= g.nx ? lx - g.nx + 1 : 0);
    const int oy = ly < 0 ? -ly : (ly >= g.ny ? ly - g.ny + 1 : 0);
    const int oz = lz < 0 ? -lz : (lz >= g.nz ? lz - g.nz + 1 : 0);
    const int r0 = max(ox, max(oy, oz));
    const int r1 = max(max(lx, g.nx - 1 - lx), max(max(ly, g.ny - 1 - ly), max(lz, g.nz - 1 - lz)));
    float best = 3.0e38f;
#pragma unroll 1
    for (int r = r0; r <= r1; ++r) {
        if (r > 0) {
            const float lb = (float)(r - 1) * cell * 0.99999f;      // every point of ring r is at least this far
            if (lb * lb > best) break;
        }
        const int z0 = max(-r, -lz), z1 = min(r, g.nz - 1 - lz);
        const int y0 = max(-r, -ly), y1 = min(r, g.ny - 1 - ly);
#pragma unroll 1
        for (int dz = z0; dz <= z1; ++dz) {
#pragma unroll 1
            for (int dy = y0; dy <= y1; ++dy) {
                const int* rowp = g.cell_start + (size_t)((lz + dz) * g.ny + (ly + dy)) * g.nx;
                const bool shell = (dz == -r) || (dz == r) || (dy == -r) || (dy == r);
                if (shell) {                                         // whole x-span of the ring, one contiguous range
                    const int xa = max(lx - r, 0), xb = min(lx + r, g.nx - 1);
                    if (xa > xb) continue;
                    const int s = __ldg(rowp + xa), e = __ldg(rowp + xb + 1);
                    for (int j = s; j < e; ++j) best = fminf(best, dist2(qx, qy, qz, __ldg(&g.pts[j])));
                } else {                                             // interior row: only the two end cells dx = +-r
                    for (int sgn = -1; sgn <= 1; sgn += 2) {
                        const int xx = lx + sgn * r;
                        if (xx < 0 || xx >= g.nx) continue;
                        const int s = __ldg(rowp + xx), e = __ldg(rowp + xx + 1);
                        for (int j = s; j < e; ++j) best = fminf(best, dist2(qx, qy, qz, __ldg(&g.pts[j])));
                    }
                }
            }
        }
    }
    return best;
}

// per-block partial sums: [0] sum of distances, [1] sum of squared distances below the threshold, [2] count below it.
// Grid y = pair b, whose queries are q[seg[b], seg[b+1]), searched in grids[b]; partials [b][gridDim.x][3].  When
// T != nullptr the query is fl32(T_b p) with the pose T_b = T[16 b ..] (row-major 4x4; pcl::transformPointCloud: FP64
// math, float32 store), else p itself.
__global__ void nn1_metrics_kernel(const float4* __restrict__ q, const long long* __restrict__ seg,
                                   const Grid* __restrict__ grids, const double* __restrict__ T, double threshold,
                                   double* __restrict__ partials) {
    __shared__ double sh[3][8];
    double sd = 0.0, ssq = 0.0, cnt = 0.0;
    const int b = blockIdx.y;
    const long long n = seg[b + 1];
    const Grid& g = grids[b];
    if (T) T += 16 * (size_t)b;
    for (long long i = seg[b] + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float4 p = __ldg(&q[i]);
        float x = p.x, y = p.y, z = p.z;
        if (T) {
            const double px = p.x, py = p.y, pz = p.z;
            x = (float)(T[0] * px + T[1] * py + T[2] * pz + T[3]);
            y = (float)(T[4] * px + T[5] * py + T[6] * pz + T[7]);
            z = (float)(T[8] * px + T[9] * py + T[10] * pz + T[11]);
        }
        const float d2 = nn1_search(g, x, y, z);
        const double dist = sqrt((double)d2);
        sd += dist;
        if (dist < threshold) { ssq += (double)d2; cnt += 1.0; }
    }
    for (int off = 16; off > 0; off >>= 1) {
        sd += __shfl_down_sync(0xffffffffu, sd, off);
        ssq += __shfl_down_sync(0xffffffffu, ssq, off);
        cnt += __shfl_down_sync(0xffffffffu, cnt, off);
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { sh[0][warp] = sd; sh[1][warp] = ssq; sh[2][warp] = cnt; }
    __syncthreads();
    if (threadIdx.x < 3) {
        double s = 0.0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += sh[threadIdx.x][w];
        partials[((size_t)b * gridDim.x + blockIdx.x) * 3 + threadIdx.x] = s;
    }
}

// transform + float32 store of clouds (aligned copies for the backward Chamfer pass): point i of segment b uses the
// pose T[16 b ..]
__global__ void transform_points_kernel(const float4* __restrict__ in, long long n, const double* __restrict__ T,
                                        float4* __restrict__ out, const long long* __restrict__ seg, int nseg) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    T += 16 * (size_t)segment_of(seg, nseg, i);
    const float4 p = in[i];
    const double px = p.x, py = p.y, pz = p.z;
    out[i] = make_float4((float)(T[0] * px + T[1] * py + T[2] * pz + T[3]), (float)(T[4] * px + T[5] * py + T[6] * pz + T[7]),
                         (float)(T[8] * px + T[9] * py + T[10] * pz + T[11]), p.w);
}

// The fit's divisions and square roots by the correctly rounded primitives of cr_fp64.cuh: each ORs "operand outside
// the exact range" into `bad` instead of branching to the library's slow path.
struct CrArith {
    bool& bad;
    __device__ __forceinline__ double div(double a, double b) const { return crf::div(a, b, bad); }
    __device__ __forceinline__ double rcp(double b) const { return crf::rcp_step(b, bad); }
    __device__ __forceinline__ double div_by(double a, double b, double y) const { return crf::div_by(a, b, y, bad); }
    __device__ __forceinline__ double sqrt(double a) const { return crf::sqrt(a, bad); }
};

// Plane through the 5 neighbours: least squares of [nb] x = -1, n = x/|x|, d = 1/|x|, gates
// |x| >= min_norm and max_j (n.nb_j + d)^2 < thickness^2 (icp_test_runner.cpp:1727-1773).
// Returns true and (n, d) when a valid plane exists; (n, d) is written whenever |x| >= min_norm.
// The QR is the register-resident one (small_la.cuh: the same operations in the same order as the generic
// colpiv_qr_solve, bit-identical results; tools/test_qr_reg.cu).  Every division and square root goes through `ar`.
template <class Ar>
__device__ __forceinline__ bool fit_plane_ar(const float4* pts, const int* kpos, double min_norm, double thickness,
                                             double& nx, double& ny, double& nz, double& d, Ar ar) {
    double A[5][3], b[5], x[3];
#pragma unroll
    for (int j = 0; j < 5; ++j) {
        const float4 p = __ldg(&pts[kpos[j]]);
        A[j][0] = (double)p.x;
        A[j][1] = (double)p.y;
        A[j][2] = (double)p.z;
        b[j] = -1.0;
    }
    dla::colpiv_qr_solve_reg<5, 3>(A, b, x, ar);
    const double ps = ar.sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
    if (!(ps >= min_norm)) return false;                 // :1752 (also rejects NaN)
    const double y = ar.rcp(ps);                         // the four divisions by ps share one reciprocal
    nx = ar.div_by(x[0], ps, y); ny = ar.div_by(x[1], ps, y); nz = ar.div_by(x[2], ps, y); d = ar.div_by(1.0, ps, y);
    double worst = 0.0;
#pragma unroll
    for (int j = 0; j < 5; ++j) {
        const float4 p = __ldg(&pts[kpos[j]]);
        double e = nx * (double)p.x + ny * (double)p.y + nz * (double)p.z + d;
        e *= e;
        worst = fmax(worst, e);
    }
    return worst < thickness * thickness;                // :1772-1773
}

// The loop's plane fit.  It runs fit_plane_ar with the correctly rounded primitives, whose values are exactly those of
// `/` and `sqrt` wherever their range flag stays clear, so the pivot choices, the rank cut and the gates see the same
// bits as with plain arithmetic.  A fit that set the flag (an operand outside the primitives' range: in practice a
// subnormal, huge or degenerate neighbourhood) discards what it computed and runs again with plain `/` and `sqrt`.
// The primitives have no branch per operation, so the fit's ~30 serial divisions and square roots form one straight
// dependent chain and the independent ones (the column norms, the downdates of two columns, the normalisation)
// overlap.  Inlined into the fit list of the loop kernel: as a separate function under the kernel's 80-register cap
// it saved and restored the caller's registers and its own spills through local memory on every fit's chain, and its
// key array (kpos) lived in the stack frame; kpos is the fit list's key row in shared memory (§3, "Fit keys from
// shared memory, fit inlined").
// Rejected: a variant of the QR with hardware reciprocal / rsqrt seeds instead of the ~30 IEEE divisions and square
// roots on the fit's dependent chain shortens a fit, but on exactly rank-deficient neighbourhoods (collinear lattice
// points) its 1-ulp differences flip the pivoted QR's rank decision and change a correspondence.
struct FitPlane { double nx, ny, nz, d; bool ok; };

// The fallback, out of line: inlined, its registers shaped the allocation of the fast fit and of the kernel around it
// (more spills in the loop kernel's per-trial-grid instantiations).  p carries the caller's (n, d) in and out, so an
// early rejection leaves them as they were.
__device__ __noinline__ FitPlane fit_plane_plain(const float4* pts, const int* kpos, double min_norm, double thickness,
                                                 FitPlane p) {
    p.ok = fit_plane_ar(pts, kpos, min_norm, thickness, p.nx, p.ny, p.nz, p.d, dla::PlainArith());
    return p;
}

__device__ __forceinline__ bool fit_plane_reg(const Grid& g, const int* kpos, double min_norm, double thickness,
                                           double& nx, double& ny, double& nz, double& d) {
    bool bad = false;
    double fx = nx, fy = ny, fz = nz, fd = d;
    const bool ok = fit_plane_ar(g.pts, kpos, min_norm, thickness, fx, fy, fz, fd, CrArith{bad});
    if (bad) {
        const FitPlane p = fit_plane_plain(g.pts, kpos, min_norm, thickness, FitPlane{nx, ny, nz, d, false});
        nx = p.nx; ny = p.ny; nz = p.nz; d = p.d;
        return p.ok;
    }
    nx = fx; ny = fy; nz = fz; d = fd;
    return ok;
}

}  // namespace corr
