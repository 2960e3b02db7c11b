// Device harness for the neighbour searches of dcreg_b200/csrc/corr.cuh, driven by tests/test_gpu_corr_search.py.
//
//   test_corr_search <input> <output>
//
// The input is one grid and a list of queries: the target points in their original order, the dense grid layout the
// test computed for them (points grouped by cell, x-fastest cells, ascending index inside a cell), and per query its
// position and squared bound B.  The harness runs the production device functions on it, unchanged:
//   knn_search      one thread per query, on the dense grid and on the sparse row index of the same points (built
//                   here with the production build, build_sparse);
//   knn_search_lb   one thread per query, bound B, starting lb = r2_up * 0.9999 (as icp_iter2_kernel);
//   knn_warp_search one warp per query, rows set up by the search itself and, when rings == 1, also from a table of
//                   rows every thread set up beforehand with knn_row_range (the loop kernel's `pre` path);
//   knn_row_range   the listed (query, row) pairs;
//   nn1_search      one thread per query;
// and builds the dense grid again from the raw points with corr.cuh's build kernels (bounds, count, three-phase scan,
// scatter, rank; the order of arena_fill for one cloud), reporting whether the result is byte-identical to the input
// layout.  Binary formats: see read_input / the writes at the end of main (little-endian, no padding).
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include <cub/device/device_radix_sort.cuh>
#include "../dcreg_b200/csrc/corr.cuh"

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(2); } } while (0)

constexpr int kMagic = 0x43525331;   // "CRS1"
constexpr int kWarpsPerBlock = 4;

struct Input {
    int n, nq, nrr, rings, ox, oy, oz, nx, ny, nz;
    float r2_up;
    double inv_cell;
    std::vector<float> xyz;              // [n][3], original order
    std::vector<float4> pts;             // [n], grouped by cell, .w = bit-cast original index
    std::vector<int> pos_of;             // [n]
    std::vector<int> cell_start;         // [nx ny nz + 1]
    std::vector<float> q;                // [nq][3]
    std::vector<float> B;                // [nq]
    std::vector<int> rr;                 // [nrr][2]: query, row
};

template <class T>
static void read_into(FILE* f, std::vector<T>& v, size_t count) {
    v.resize(count);
    if (count && fread(v.data(), sizeof(T), count, f) != count) { fprintf(stderr, "short input\n"); exit(2); }
}

// header: int32 magic, n, nq, nrr, rings, ox, oy, oz, nx, ny, nz, float32 r2_up, float64 inv_cell; then the arrays in
// the order of Input
static Input read_input(const char* path) {
    FILE* f = fopen(path, "rb");
    if (!f) { fprintf(stderr, "cannot read %s\n", path); exit(2); }
    int h[12];
    if (fread(h, sizeof(int), 12, f) != 12 || h[0] != kMagic) { fprintf(stderr, "bad header\n"); exit(2); }
    Input in;
    in.n = h[1]; in.nq = h[2]; in.nrr = h[3]; in.rings = h[4];
    in.ox = h[5]; in.oy = h[6]; in.oz = h[7]; in.nx = h[8]; in.ny = h[9]; in.nz = h[10];
    memcpy(&in.r2_up, &h[11], sizeof(float));
    if (fread(&in.inv_cell, sizeof(double), 1, f) != 1) { fprintf(stderr, "bad header\n"); exit(2); }
    const size_t cells = (size_t)in.nx * in.ny * in.nz;
    read_into(f, in.xyz, (size_t)in.n * 3);
    read_into(f, in.pts, (size_t)in.n);
    read_into(f, in.pos_of, (size_t)in.n);
    read_into(f, in.cell_start, cells + 1);
    read_into(f, in.q, (size_t)in.nq * 3);
    read_into(f, in.B, (size_t)in.nq);
    read_into(f, in.rr, (size_t)in.nrr * 2);
    fclose(f);
    return in;
}

template <class T>
static T* upload(const std::vector<T>& v) {
    T* d = nullptr;
    CK(cudaMalloc(&d, (v.size() ? v.size() : 1) * sizeof(T)));
    if (v.size()) CK(cudaMemcpy(d, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
    return d;
}
template <class T>
static T* alloc(size_t count) {
    T* d = nullptr;
    CK(cudaMalloc(&d, (count ? count : 1) * sizeof(T)));
    CK(cudaMemset(d, 0, (count ? count : 1) * sizeof(T)));
    return d;
}
template <class T>
static std::vector<T> download(const T* d, size_t count) {
    std::vector<T> v(count);
    if (count) CK(cudaMemcpy(v.data(), d, count * sizeof(T), cudaMemcpyDeviceToHost));
    return v;
}

struct ThreadOut {
    unsigned long long* knn5;     // [nq][5] dense knn_search
    unsigned long long* knn5s;    // [nq][5] sparse knn_search
    unsigned long long* lbk;      // [nq][7] knn_search_lb
    int* lbp;                     // [nq][7]
    float* lbv;                   // [nq]
    float* nn1;                   // [nq]
};

__global__ void thread_searches_kernel(corr::Grid g, corr::Grid s, const float* __restrict__ q, const float* __restrict__ B,
                                       int nq, float lb0, ThreadOut o) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq) return;
    const float qx = q[3 * i], qy = q[3 * i + 1], qz = q[3 * i + 2];
    corr::Knn5 k;
    corr::knn_init(k);
    corr::knn_search(g, qx, qy, qz, k);
    for (int j = 0; j < 5; ++j) o.knn5[5 * (size_t)i + j] = k.key[j];
    corr::knn_init(k);
    corr::knn_search<true>(s, qx, qy, qz, k);
    for (int j = 0; j < 5; ++j) o.knn5s[5 * (size_t)i + j] = k.key[j];
    corr::KnnM m;
    float lb = lb0;
    corr::knn_search_lb(g, qx, qy, qz, B[i], m, lb);
    for (int j = 0; j < corr::kSeeds; ++j) { o.lbk[7 * (size_t)i + j] = m.key[j]; o.lbp[7 * (size_t)i + j] = m.pos[j]; }
    o.lbv[i] = lb;
    o.nn1[i] = corr::nn1_search(g, qx, qy, qz);
}

// the loop kernel's row table (icp_iter2_kernel, rings == 1): every thread sets up rows of any listed query
__global__ void row_table_kernel(corr::Grid g, const float* __restrict__ q, const float* __restrict__ B, int nq,
                                 corr::RowRange* __restrict__ tab) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= nq * 9) return;
    const int i = e / 9, r = e - i * 9;
    tab[e] = corr::knn_row_range(g, q[3 * i], q[3 * i + 1], q[3 * i + 2], B[i], r);
}

__global__ void row_pairs_kernel(corr::Grid g, const float* __restrict__ q, const float* __restrict__ B,
                                 const int* __restrict__ rr, int nrr, int* __restrict__ out) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= nrr) return;
    const int i = rr[2 * e], r = rr[2 * e + 1];
    const corr::RowRange x = corr::knn_row_range(g, q[3 * i], q[3 * i + 1], q[3 * i + 2], B[i], r);
    out[3 * (size_t)e] = x.s; out[3 * (size_t)e + 1] = x.e; out[3 * (size_t)e + 2] = __float_as_int(x.lb);
}

struct WarpOut {
    int* got;                     // [nq]
    unsigned long long* key;      // [nq][7]
    int* pos;                     // [nq][7]
    float* lb;                    // [nq]
};

__global__ void warp_searches_kernel(corr::Grid g, const float* __restrict__ q, const float* __restrict__ B, int nq,
                                     float lb0, const corr::RowRange* __restrict__ pre, WarpOut o) {
    __shared__ corr::WarpKnnSmem S[kWarpsPerBlock];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = blockIdx.x * kWarpsPerBlock + warp; i < nq; i += gridDim.x * kWarpsPerBlock) {
        corr::KnnM r;
        float lb = lb0;
        const bool got = corr::knn_warp_search(g, q[3 * i], q[3 * i + 1], q[3 * i + 2], B[i], S[warp], r, lb, nullptr,
                                               pre ? pre + 9 * (size_t)i : nullptr);
        if (lane == 0) {
            o.got[i] = got ? 1 : 0;
            for (int j = 0; j < corr::kSeeds; ++j) {
                o.key[7 * (size_t)i + j] = got ? r.key[j] : 0ull;
                o.pos[7 * (size_t)i + j] = got ? r.pos[j] : 0;
            }
            o.lb[i] = got ? lb : 0.0f;
        }
        __syncwarp();
    }
}

// corr.cuh's build kernels on the raw points, in arena_fill's order for one cloud; flags: pts, pos_of, cell_start
// byte-identical to the input layout
static void grid_build_check(const Input& in, int (&bounds)[6], int (&same)[3]) {
    std::vector<float4> raw((size_t)in.n);
    for (int i = 0; i < in.n; ++i) raw[(size_t)i] = make_float4(in.xyz[3 * (size_t)i], in.xyz[3 * (size_t)i + 1], in.xyz[3 * (size_t)i + 2], 0.0f);
    float4* d_raw = upload(raw);
    const std::vector<long long> seg = {0, (long long)in.n};
    long long* d_seg = upload(seg);
    std::vector<int> hb = {1 << 30, 1 << 30, 1 << 30, -(1 << 30), -(1 << 30), -(1 << 30)};
    int* d_bounds = upload(hb);
    corr::grid_bounds_seg_kernel<<<dim3(64, 1), 256>>>(d_raw, d_seg, in.inv_cell, d_bounds);
    CK(cudaGetLastError());
    hb = download(d_bounds, 6);
    for (int k = 0; k < 6; ++k) bounds[k] = hb[(size_t)k];
    same[0] = same[1] = same[2] = 0;
    const int nx = hb[3] - hb[0] + 1, ny = hb[4] - hb[1] + 1, nz = hb[5] - hb[2] + 1;
    if (hb[0] != in.ox || hb[1] != in.oy || hb[2] != in.oz || nx != in.nx || ny != in.ny || nz != in.nz) {
        cudaFree(d_raw); cudaFree(d_seg); cudaFree(d_bounds);
        return;
    }
    const long long cells = (long long)nx * ny * nz;
    corr::Grid g{};
    g.n = in.n; g.dense = 1; g.rings = in.rings; g.inv_cell = in.inv_cell;
    g.ox = hb[0]; g.oy = hb[1]; g.oz = hb[2]; g.nx = nx; g.ny = ny; g.nz = nz;
    corr::Grid* d_grids = upload(std::vector<corr::Grid>{g});
    int* d_cell_off = upload(std::vector<int>{0, (int)cells});
    int* counts = alloc<int>((size_t)cells + 1);
    int* fill = alloc<int>((size_t)cells);
    int* start = alloc<int>((size_t)cells + 1);
    int* pt_cell = alloc<int>((size_t)in.n);
    float4* tmp = alloc<float4>((size_t)in.n);
    float4* out = alloc<float4>((size_t)in.n);
    int* pos_of = alloc<int>((size_t)in.n);
    const unsigned nb = (unsigned)((in.n + 255) / 256);
    corr::grid_count_seg_kernel<<<nb, 256>>>(d_raw, in.n, d_seg, 1, d_grids, d_cell_off, pt_cell, counts);
    const long long ns = cells + 1;
    const int ntiles = (int)((ns + corr::kScanTile - 1) / corr::kScanTile);
    int* tile_sums = alloc<int>((size_t)ntiles);
    corr::scan_tile_sums_kernel<<<ntiles, 256>>>(counts, (int)ns, tile_sums);
    corr::scan_tile_offsets_kernel<<<1, 1024>>>(tile_sums, ntiles);
    corr::scan_tile_apply_kernel<<<ntiles, 256>>>(counts, (int)ns, tile_sums, start);
    corr::grid_scatter_kernel<<<nb, 256>>>(d_raw, in.n, pt_cell, start, fill, tmp, 0);
    corr::grid_rank_cells_kernel<<<nb, 256>>>(tmp, in.n, pt_cell, start, out, pos_of);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    const std::vector<float4> hp = download(out, (size_t)in.n);
    const std::vector<int> hpos = download(pos_of, (size_t)in.n), hcs = download(start, (size_t)cells + 1);
    same[0] = memcmp(hp.data(), in.pts.data(), hp.size() * sizeof(float4)) == 0;
    same[1] = memcmp(hpos.data(), in.pos_of.data(), hpos.size() * sizeof(int)) == 0;
    same[2] = memcmp(hcs.data(), in.cell_start.data(), hcs.size() * sizeof(int)) == 0;
    for (void* p : {(void*)d_raw, (void*)d_seg, (void*)d_bounds, (void*)d_grids, (void*)d_cell_off, (void*)counts, (void*)fill,
                    (void*)start, (void*)pt_cell, (void*)tmp, (void*)out, (void*)pos_of, (void*)tile_sums})
        cudaFree(p);
}

// The sparse row index of the same points (box: the dense layout's g), built with the production build as
// build_sparse_arena runs it on a one-cloud arena: corr::sparse_seg_key_kernel and a stable radix sort over (y, x), then
// over (cloud, z); sparse_seg_gather_kernel, sparse_seg_count_kernel, sparse_index::layout, sparse_seg_insert_kernel.
// check: pts identical and pos_of identical to the dense layout, table entries.
static corr::Grid build_sparse(const Input& in, const corr::Grid& g, int (&check)[3]) {
    const int n = in.n;
    std::vector<float4> raw((size_t)n);
    for (int i = 0; i < n; ++i) raw[(size_t)i] = make_float4(in.xyz[3 * (size_t)i], in.xyz[3 * (size_t)i + 1], in.xyz[3 * (size_t)i + 2], 0.0f);
    float4* d_raw = upload(raw);
    corr::Grid s = g;
    s.dense = corr::kSparseGrid; s.cell_start = nullptr;
    s.pts = alloc<float4>((size_t)n); s.pos_of = alloc<int>((size_t)n);
    const long long* d_seg = upload(std::vector<long long>{0, n});
    corr::Grid* d_grids = upload(std::vector<corr::Grid>{s});
    unsigned long long* keys = alloc<unsigned long long>(2 * (size_t)n);
    int* vals = alloc<int>(2 * (size_t)n);
    // each pass sorts the bits of its largest key: (y, x) of the box's far corner, (cloud 0, z) of its top
    const unsigned long long top[2] = {sparse_index::key(s.nx - 1, s.ny - 1, 0), (unsigned long long)(s.nz - 1)};
    int end_bit[2] = {1, 1};
    for (int p = 0; p < 2; ++p)
        while (end_bit[p] < 64 && top[p] >> end_bit[p]) ++end_bit[p];
    size_t tmp0 = 0, tmp1 = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, tmp0, keys, keys + n, vals, vals + n, n, 0, end_bit[0]));
    CK(cub::DeviceRadixSort::SortPairs(nullptr, tmp1, keys, keys + n, vals, vals + n, n, 0, end_bit[1]));
    size_t tmp = std::max(tmp0, tmp1);
    unsigned char* d_tmp = alloc<unsigned char>(tmp);
    const unsigned nb = (unsigned)((n + 255) / 256);
    for (int pass = 0; pass < 2; ++pass) {
        corr::sparse_seg_key_kernel<<<nb, 256>>>(d_raw, n, d_seg, 1, d_grids, pass, vals + n, keys, vals);
        CK(cub::DeviceRadixSort::SortPairs(d_tmp, tmp, keys, keys + n, vals, vals + n, n, 0, end_bit[pass]));
    }
    unsigned long long* sorted = keys;                           // (the passes' input keys are spent)
    corr::sparse_seg_gather_kernel<<<nb, 256>>>(d_raw, vals + n, n, d_seg, 1, d_grids, s.pts, s.pos_of, sorted);
    unsigned long long* d_entries = alloc<unsigned long long>(1);
    corr::sparse_seg_count_kernel<<<nb, 256>>>(sorted, n, d_seg, 1, d_grids, d_entries);
    CK(cudaGetLastError());
    const unsigned long long entries = download(d_entries, 1)[0];
    long long cap, off[2];
    if (sparse_index::layout(1, &entries, &cap, off) >= 0) { fprintf(stderr, "sparse index over 2^32 slots\n"); exit(2); }
    s.keys = alloc<unsigned long long>((size_t)cap);
    CK(cudaMemset(s.keys, 0xff, (size_t)cap * sizeof(unsigned long long)));
    s.hstart = alloc<int>((size_t)cap); s.mask = (unsigned)(cap - 1);
    CK(cudaMemcpy(d_grids, &s, sizeof(s), cudaMemcpyHostToDevice));
    corr::sparse_seg_insert_kernel<<<nb, 256>>>(sorted, n, d_seg, 1, d_grids);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    const std::vector<float4> sp = download(s.pts, (size_t)n);
    const std::vector<int> spos = download(s.pos_of, (size_t)n);
    check[0] = memcmp(sp.data(), in.pts.data(), sp.size() * sizeof(float4)) == 0;
    check[1] = memcmp(spos.data(), in.pos_of.data(), spos.size() * sizeof(int)) == 0;
    check[2] = (int)entries;
    return s;
}

template <class T>
static void write(FILE* f, const std::vector<T>& v) {
    if (v.size() && fwrite(v.data(), sizeof(T), v.size(), f) != v.size()) { fprintf(stderr, "short write\n"); exit(2); }
}

#ifndef CORR_SEARCH_NO_MAIN      // tools/test_sparse_search.cu reuses the input format and helpers above
int main(int argc, char** argv) {
    if (argc != 3) { fprintf(stderr, "usage: %s <input> <output>\n", argv[0]); return 2; }
    const Input in = read_input(argv[1]);
    const int nq = in.nq;
    const size_t nq_ = (size_t)nq;
    // the bound every search starts from: nothing outside the rings of cells is nearer than the search radius
    const float lb0 = in.r2_up * 0.9999f;

    corr::Grid g{};
    g.pts = upload(in.pts); g.pos_of = upload(in.pos_of); g.n = in.n; g.dense = 1; g.rings = in.rings;
    g.inv_cell = in.inv_cell; g.ox = in.ox; g.oy = in.oy; g.oz = in.oz; g.nx = in.nx; g.ny = in.ny; g.nz = in.nz;
    g.cell_start = upload(in.cell_start);
    int sparse_check[3];
    const corr::Grid s = build_sparse(in, g, sparse_check);

    float* d_q = upload(in.q);
    float* d_B = upload(in.B);
    int* d_rr = upload(in.rr);

    ThreadOut to{alloc<unsigned long long>(nq_ * 5), alloc<unsigned long long>(nq_ * 5), alloc<unsigned long long>(nq_ * 7),
                 alloc<int>(nq_ * 7), alloc<float>(nq_), alloc<float>(nq_)};
    thread_searches_kernel<<<(nq + 127) / 128, 128>>>(g, s, d_q, d_B, nq, lb0, to);
    CK(cudaGetLastError());

    const unsigned wblocks = (unsigned)((nq + kWarpsPerBlock - 1) / kWarpsPerBlock);
    WarpOut wo{alloc<int>(nq_), alloc<unsigned long long>(nq_ * 7), alloc<int>(nq_ * 7), alloc<float>(nq_)};
    warp_searches_kernel<<<wblocks, 32 * kWarpsPerBlock>>>(g, d_q, d_B, nq, lb0, nullptr, wo);
    CK(cudaGetLastError());
    WarpOut po{alloc<int>(nq_), alloc<unsigned long long>(nq_ * 7), alloc<int>(nq_ * 7), alloc<float>(nq_)};
    if (in.rings == 1) {
        corr::RowRange* tab = alloc<corr::RowRange>(nq_ * 9);
        row_table_kernel<<<(nq * 9 + 255) / 256, 256>>>(g, d_q, d_B, nq, tab);
        warp_searches_kernel<<<wblocks, 32 * kWarpsPerBlock>>>(g, d_q, d_B, nq, lb0, tab, po);
        CK(cudaGetLastError());
    }
    int* d_rro = alloc<int>((size_t)in.nrr * 3);
    if (in.nrr) row_pairs_kernel<<<(in.nrr + 255) / 256, 256>>>(g, d_q, d_B, d_rr, in.nrr, d_rro);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());

    int bounds[6], same[3];
    grid_build_check(in, bounds, same);

    // output: knn5, knn5s (uint64 [nq][5]); lb search keys (uint64 [nq][7]), positions (int32 [nq][7]), lb (float32
    // [nq]); warp search got (int32 [nq]), keys, positions, lb; the same four with the row table (zeros unless
    // rings == 1); nn1 (float32 [nq]); row pairs (int32 [nrr][3]: s, e, bits of lb); grid build: bounds (int32 [6]),
    // identical pts / pos_of / cell_start (int32 [3])
    FILE* f = fopen(argv[2], "wb");
    if (!f) { fprintf(stderr, "cannot write %s\n", argv[2]); return 2; }
    write(f, download(to.knn5, nq_ * 5));
    write(f, download(to.knn5s, nq_ * 5));
    write(f, download(to.lbk, nq_ * 7));
    write(f, download(to.lbp, nq_ * 7));
    write(f, download(to.lbv, nq_));
    for (const WarpOut& w : {wo, po}) {
        write(f, download(w.got, nq_));
        write(f, download(w.key, nq_ * 7));
        write(f, download(w.pos, nq_ * 7));
        write(f, download(w.lb, nq_));
    }
    write(f, download(to.nn1, nq_));
    write(f, download(d_rro, (size_t)in.nrr * 3));
    write(f, std::vector<int>(bounds, bounds + 6));
    write(f, std::vector<int>(same, same + 3));
    fclose(f);
    printf("CORR_SEARCH_DONE %d queries, %d row pairs\n", nq, in.nrr);
    return 0;
}
#endif
