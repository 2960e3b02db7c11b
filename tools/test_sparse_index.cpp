// Host check of sparse_index.hpp (tests/test_sparse_index_twin.py): a host twin of the sparse row index build
// (sort by box-local cell key, the entry count, the table inserts), the way corr::sparse_* run it on the device, against
// a literal reading of its contract:
//   * every table entry holds cs(z, y, x) counted point by point (the points whose cell comes before (z, y, x));
//   * the table holds exactly the union of every occupied cell's dilation [x' - 8, x' + 9], clipped to [0, nx];
//   * for every occupied cell and every window [x0, x1) of width 1..9 around it (clipped as the searches clip), the
//     range rule (both ends in the table: [cs(x0), cs(x1)), else empty) gives exactly the points of those cells.
// Clouds are cell coordinates: random ones with repeated cells, negative ones and ones at the +-2^19 edge, and rows whose
// occupied cells are 8, 9 and 10 apart.
#include <algorithm>
#include <cstdio>
#include <numeric>
#include <random>
#include <set>
#include <tuple>
#include <vector>
#include "../dcreg_b200/csrc/sparse_index.hpp"

static int fails = 0;
#define CHECK(c) do { if (!(c)) { std::printf("FAIL line %d: %s\n", __LINE__, #c); if (++fails > 20) return; } } while (0)

struct Cell { int x, y, z; };

struct Twin {
    int ox, oy, oz, nx, ny, nz;
    std::vector<int> order;                        // original index of sorted position j
    std::vector<unsigned long long> sorted;        // key of sorted position j
    std::vector<unsigned long long> keys;          // table
    std::vector<int> val;
    unsigned mask = 0;
    long long entries = 0;

    int lookup(int x, int y, int z) const {
        const unsigned long long k = sparse_index::key(x, y, z);
        unsigned s = sparse_index::slot(k, mask);
        while (true) {
            if (keys[s] == k) return val[s];
            if (keys[s] == sparse_index::kEmpty) return -1;
            s = (s + 1) & mask;
        }
    }
};

static Twin build(const std::vector<Cell>& c) {
    Twin t;
    int lo[3] = {1 << 30, 1 << 30, 1 << 30}, hi[3] = {-(1 << 30), -(1 << 30), -(1 << 30)};
    for (const Cell& p : c) {
        const int v[3] = {p.x, p.y, p.z};
        for (int k = 0; k < 3; ++k) { lo[k] = std::min(lo[k], v[k]); hi[k] = std::max(hi[k], v[k]); }
    }
    t.ox = lo[0]; t.oy = lo[1]; t.oz = lo[2];
    t.nx = hi[0] - lo[0] + 1; t.ny = hi[1] - lo[1] + 1; t.nz = hi[2] - lo[2] + 1;
    const long long n = (long long)c.size();
    std::vector<unsigned long long> k(n);
    for (long long i = 0; i < n; ++i) k[i] = sparse_index::key(c[i].x - t.ox, c[i].y - t.oy, c[i].z - t.oz);
    t.order.resize(n);
    std::iota(t.order.begin(), t.order.end(), 0);
    std::stable_sort(t.order.begin(), t.order.end(), [&](int a, int b) { return k[a] < k[b]; });
    t.sorted.resize(n);
    for (long long j = 0; j < n; ++j) t.sorted[j] = k[t.order[j]];
    for (long long j = 0; j < n; ++j) {
        if (j > 0 && t.sorted[j - 1] == t.sorted[j]) continue;
        int a, b;
        sparse_index::new_entries(t.sorted[j], j > 0 ? t.sorted[j - 1] : sparse_index::kEmpty, t.nx, &a, &b);
        if (b >= a) t.entries += b - a + 1;
    }
    const long long cap = sparse_index::capacity(t.entries);
    t.keys.assign(cap, sparse_index::kEmpty);
    t.val.assign(cap, -7);
    t.mask = (unsigned)(cap - 1);
    for (long long j = 0; j < n; ++j) {
        if (j > 0 && t.sorted[j - 1] == t.sorted[j]) continue;
        int a, b;
        sparse_index::new_entries(t.sorted[j], j > 0 ? t.sorted[j - 1] : sparse_index::kEmpty, t.nx, &a, &b);
        const unsigned long long row = sparse_index::row_of(t.sorted[j]) << sparse_index::kBits;
        for (int x = a; x <= b; ++x) {
            const unsigned long long kk = row | (unsigned long long)x;
            unsigned s = sparse_index::slot(kk, t.mask);
            while (t.keys[s] != sparse_index::kEmpty) s = (s + 1) & t.mask;
            t.keys[s] = kk;
            t.val[s] = (int)sparse_index::cs(t.sorted.data(), n, kk);
        }
    }
    return t;
}

static void check(const std::vector<Cell>& c) {
    const Twin t = build(c);
    const long long n = (long long)c.size();
    // literal cs and the literal dilation union, in box-local coordinates
    auto before = [&](int x, int y, int z) {
        long long m = 0;
        for (const Cell& p : c)
            if (std::make_tuple(p.z - t.oz, p.y - t.oy, p.x - t.ox) < std::make_tuple(z, y, x)) ++m;
        return m;
    };
    std::set<std::tuple<int, int, int>> occupied, dil;
    for (const Cell& p : c) occupied.insert({p.z - t.oz, p.y - t.oy, p.x - t.ox});
    for (const auto& o : occupied)
        for (int x = std::get<2>(o) - sparse_index::kBack; x <= std::get<2>(o) + sparse_index::kReach; ++x)
            if (x >= 0 && x <= t.nx) dil.insert({std::get<0>(o), std::get<1>(o), x});
    CHECK(t.entries == (long long)dil.size());
    long long in_table = 0;
    for (size_t s = 0; s < t.keys.size(); ++s) {
        if (t.keys[s] == sparse_index::kEmpty) continue;
        ++in_table;
        const unsigned long long k = t.keys[s];
        const int x = sparse_index::x_of(k), y = (int)(sparse_index::row_of(k) & ((1u << sparse_index::kBits) - 1)),
                  z = (int)(k >> (2 * sparse_index::kBits));
        CHECK(dil.count({z, y, x}) == 1);
        CHECK(t.val[s] == before(x, y, z));
    }
    CHECK(in_table == (long long)dil.size());
    CHECK((long long)t.keys.size() >= 2 * in_table && (t.keys.size() & (t.keys.size() - 1)) == 0);
    // the dense order: by cell (z, y, x), then by index
    for (long long j = 1; j < n; ++j) {
        const Cell &a = c[t.order[j - 1]], &b = c[t.order[j]];
        CHECK(std::make_tuple(a.z, a.y, a.x, t.order[j - 1]) < std::make_tuple(b.z, b.y, b.x, t.order[j]));
    }
    // the range rule around every occupied cell, in its row and the rows next to it
    for (const auto& o : occupied) {
        const int z = std::get<0>(o), y0 = std::get<1>(o), xo = std::get<2>(o);
        for (int y = y0 - 1; y <= y0 + 1; ++y) {
            if (y < 0 || y >= t.ny) continue;
            for (int w = 1; w <= sparse_index::kReach; ++w)
                for (int x0 = xo - w - 1; x0 <= xo + 1; ++x0) {
                    const int a = std::min(std::max(x0, 0), t.nx), b = std::min(std::max(x0 + w, 0), t.nx);
                    const int s = t.lookup(a, y, z), e = t.lookup(b, y, z);
                    std::vector<int> got, want;
                    if (s >= 0 && e >= 0)
                        for (int j = s; j < e; ++j) got.push_back(t.order[j]);
                    for (long long i = 0; i < n; ++i) {
                        const int px = c[i].x - t.ox, py = c[i].y - t.oy, pz = c[i].z - t.oz;
                        if (pz == z && py == y && px >= a && px < b) want.push_back((int)i);
                    }
                    std::sort(got.begin(), got.end());
                    CHECK(got == want);
                    if (fails) return;
                }
        }
    }
}

int main() {
    std::mt19937_64 rng(2026);
    // random clouds, many repeated cells, offsets negative and positive
    for (int trial = 0; trial < 40 && !fails; ++trial) {
        const int n = 1 + (int)(rng() % 300), span = 1 + (int)(rng() % 40);
        const int o[3] = {(int)(rng() % 2001) - 1000, (int)(rng() % 2001) - 1000, (int)(rng() % 201) - 100};
        std::vector<Cell> c((size_t)n);
        for (Cell& p : c) {
            p.x = o[0] + (int)(rng() % span);
            p.y = o[1] + (int)(rng() % 4);
            p.z = o[2] + (int)(rng() % 3);
        }
        check(c);
    }
    // the +-2^19 edge: a box 2^20 + 1 cells wide in x (and tall in z), so box-local x reaches 2^20
    {
        const int L = 1 << 19;
        std::vector<Cell> c = {{-L, 0, -L}, {-L, 0, -L}, {-L + 3, 0, -L}, {L, 0, L}, {L - 9, 0, L}, {L, 1, L}, {0, 0, 0},
                               {-5, -1, 0}, {-L, 1, L}};
        check(c);
    }
    // rows whose occupied cells are 8, 9 and 10 apart (and 17, 18, 19: where two dilations just meet or leave a gap)
    for (int gap : {8, 9, 10, 17, 18, 19}) {
        std::vector<Cell> c;
        for (int k = 0; k < 4; ++k) {
            c.push_back({-30 + k * gap, 2, -1});
            c.push_back({-30 + k * gap, 2, -1});
            c.push_back({-30 + k * gap + (k == 3 ? 1 : 0), 3, -1});
        }
        c.push_back({-40, 0, 5});
        check(c);
    }
    // one point, and everything in one cell
    check({{7, -7, 7}});
    check(std::vector<Cell>(12, Cell{-3, 4, -5}));
    if (fails) { std::printf("%d failure(s)\n", fails); return 1; }
    std::printf("SPARSE_INDEX_OK\n");
    return 0;
}
