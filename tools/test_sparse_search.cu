// Device harness for the sparse row index (dcreg_set_target_sparse), driven by tests/test_gpu_sparse_search.py.
//
//   test_sparse_search <input> <output>
//
// The input is tools/test_corr_search.cu's: the target points, their dense grid layout and the queries.  The harness
// builds the sparse row index of the same points with the production build (test_corr_search.cu's build_sparse) and
// reports whether its points and positions are byte-identical to the dense layout.  Then it runs the searches of
// corr.cuh on the dense grid and on the sparse index (their kSparse instantiations), unchanged: knn_search, knn_search_lb,
// knn_warp_search without and (rings == 1) with the loop kernel's row table, and knn_row_range on the listed pairs.
// Output: the sparse build check (int32 [3]: pts identical, pos_of identical, table entries), then for the dense grid
// and then the sparse index: knn5 (uint64 [nq][5]), the bounded list keys (uint64 [nq][7]), positions (int32 [nq][7]),
// lb (float32 [nq]), the warp search and the warp search with the row table (got int32 [nq], keys, positions, lb),
// and the row pairs (int32 [nrr][3]: s, e, bits of lb).
#define CORR_SEARCH_NO_MAIN
#include "test_corr_search.cu"

struct Out {
    unsigned long long* knn5;     // [nq][5]
    unsigned long long* lbk;      // [nq][7]
    int* lbp;                     // [nq][7]
    float* lbv;                   // [nq]
    WarpOut warp, pre;
    int* rr;                      // [nrr][3]
};

template <bool kSparse>
__global__ void thread_kernel(corr::Grid g, const float* __restrict__ q, const float* __restrict__ B, int nq, float lb0,
                              Out o) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq) return;
    const float qx = q[3 * i], qy = q[3 * i + 1], qz = q[3 * i + 2];
    corr::Knn5 k;
    corr::knn_init(k);
    corr::knn_search<kSparse>(g, qx, qy, qz, k);
    for (int j = 0; j < 5; ++j) o.knn5[5 * (size_t)i + j] = k.key[j];
    corr::KnnM m;
    float lb = lb0;
    corr::knn_search_lb<kSparse>(g, qx, qy, qz, B[i], m, lb);
    for (int j = 0; j < corr::kSeeds; ++j) { o.lbk[7 * (size_t)i + j] = m.key[j]; o.lbp[7 * (size_t)i + j] = m.pos[j]; }
    o.lbv[i] = lb;
}

template <bool kSparse>
__global__ void table_kernel(corr::Grid g, const float* __restrict__ q, const float* __restrict__ B, int nq,
                             corr::RowRange* __restrict__ tab) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= nq * 9) return;
    const int i = e / 9, r = e - i * 9;
    tab[e] = corr::knn_row_range<kSparse>(g, q[3 * i], q[3 * i + 1], q[3 * i + 2], B[i], r);
}

template <bool kSparse>
__global__ void pairs_kernel(corr::Grid g, const float* __restrict__ q, const float* __restrict__ B,
                             const int* __restrict__ rr, int nrr, int* __restrict__ out) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= nrr) return;
    const int i = rr[2 * e], r = rr[2 * e + 1];
    const corr::RowRange x = corr::knn_row_range<kSparse>(g, q[3 * i], q[3 * i + 1], q[3 * i + 2], B[i], r);
    out[3 * (size_t)e] = x.s; out[3 * (size_t)e + 1] = x.e; out[3 * (size_t)e + 2] = __float_as_int(x.lb);
}

template <bool kSparse>
__global__ void warp_kernel(corr::Grid g, const float* __restrict__ q, const float* __restrict__ B, int nq, float lb0,
                            const corr::RowRange* __restrict__ pre, WarpOut o) {
    __shared__ corr::WarpKnnSmem S[kWarpsPerBlock];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = blockIdx.x * kWarpsPerBlock + warp; i < nq; i += gridDim.x * kWarpsPerBlock) {
        corr::KnnM r;
        float lb = lb0;
        const bool got = corr::knn_warp_search<kSparse>(g, q[3 * i], q[3 * i + 1], q[3 * i + 2], B[i], S[warp], r, lb,
                                                        nullptr, pre ? pre + 9 * (size_t)i : nullptr);
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

template <bool kSparse>
static Out run_searches(const corr::Grid& g, const Input& in, const float* d_q, const float* d_B, const int* d_rr, float lb0) {
    const int nq = in.nq;
    const size_t nq_ = (size_t)nq;
    auto warp_out = [&]() { return WarpOut{alloc<int>(nq_), alloc<unsigned long long>(nq_ * 7), alloc<int>(nq_ * 7), alloc<float>(nq_)}; };
    Out o{alloc<unsigned long long>(nq_ * 5), alloc<unsigned long long>(nq_ * 7), alloc<int>(nq_ * 7), alloc<float>(nq_),
          warp_out(), warp_out(), alloc<int>((size_t)in.nrr * 3)};
    thread_kernel<kSparse><<<(nq + 127) / 128, 128>>>(g, d_q, d_B, nq, lb0, o);
    const unsigned wblocks = (unsigned)((nq + kWarpsPerBlock - 1) / kWarpsPerBlock);
    warp_kernel<kSparse><<<wblocks, 32 * kWarpsPerBlock>>>(g, d_q, d_B, nq, lb0, nullptr, o.warp);
    if (in.rings == 1) {
        corr::RowRange* tab = alloc<corr::RowRange>(nq_ * 9);
        table_kernel<kSparse><<<(nq * 9 + 255) / 256, 256>>>(g, d_q, d_B, nq, tab);
        warp_kernel<kSparse><<<wblocks, 32 * kWarpsPerBlock>>>(g, d_q, d_B, nq, lb0, tab, o.pre);
    }
    if (in.nrr) pairs_kernel<kSparse><<<(in.nrr + 255) / 256, 256>>>(g, d_q, d_B, d_rr, in.nrr, o.rr);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    return o;
}

static void write_out(FILE* f, const Out& o, const Input& in) {
    const size_t nq_ = (size_t)in.nq;
    write(f, download(o.knn5, nq_ * 5));
    write(f, download(o.lbk, nq_ * 7));
    write(f, download(o.lbp, nq_ * 7));
    write(f, download(o.lbv, nq_));
    for (const WarpOut& w : {o.warp, o.pre}) {
        write(f, download(w.got, nq_));
        write(f, download(w.key, nq_ * 7));
        write(f, download(w.pos, nq_ * 7));
        write(f, download(w.lb, nq_));
    }
    write(f, download(o.rr, (size_t)in.nrr * 3));
}

int main(int argc, char** argv) {
    if (argc != 3) { fprintf(stderr, "usage: %s <input> <output>\n", argv[0]); return 2; }
    const Input in = read_input(argv[1]);
    const int n = in.n;
    const float lb0 = in.r2_up * 0.9999f;

    corr::Grid g{};
    g.pts = upload(in.pts); g.pos_of = upload(in.pos_of); g.n = n; g.dense = 1; g.rings = in.rings;
    g.inv_cell = in.inv_cell; g.ox = in.ox; g.oy = in.oy; g.oz = in.oz; g.nx = in.nx; g.ny = in.ny; g.nz = in.nz;
    g.cell_start = upload(in.cell_start);

    // the sparse row index of the same points
    int check[3];
    const corr::Grid s = build_sparse(in, g, check);

    float* d_q = upload(in.q);
    float* d_B = upload(in.B);
    int* d_rr = upload(in.rr);
    const Out od = run_searches<false>(g, in, d_q, d_B, d_rr, lb0);
    const Out os = run_searches<true>(s, in, d_q, d_B, d_rr, lb0);

    FILE* f = fopen(argv[2], "wb");
    if (!f) { fprintf(stderr, "cannot write %s\n", argv[2]); return 2; }
    write(f, std::vector<int>(check, check + 3));
    write_out(f, od, in);
    write_out(f, os, in);
    fclose(f);
    printf("SPARSE_SEARCH_DONE %d queries, %d row pairs, %d entries\n", in.nq, in.nrr, check[2]);
    return 0;
}
