// Host check of the sparse arena (tests/test_sparse_arena_twin.py): the sparse row indexes of many clouds in one set of
// buffers, the way build_sparse_arena and corr::sparse_seg_* run it on the device (two stable passes, (y, x) then
// (cloud, z); per-cloud entry counts; sparse_index::layout; inserts with cs shifted by the cloud's first position),
// against a literal per-cloud build of sparse_index.hpp, each cloud alone:
//   * the point order is every cloud's own dense order, the clouds in order, positions shifted by the cloud's offset;
//   * the entry counts, capacities and table offsets are the per-cloud builds', laid out back to back;
//   * every cloud's table slice is slot for slot its own table, with every cs shifted by the cloud's offset.
// Also arena_plan::plan_or_sparse (sparse only for cell counts, never for coordinates outside +-2^19) and
// odom_plan::map_failure given its empty reason.  Clouds: zero extra entries (a cloud whose cells all share one row
// dilation), single points, +-2^19-edge coordinates, rows whose occupied cells are 8-10 and 17-19 apart.
#include <algorithm>
#include <cstdio>
#include <numeric>
#include <random>
#include <vector>
#include "../dcreg_b200/csrc/sparse_index.hpp"
#include "../dcreg_b200/csrc/arena_plan.hpp"
#include "../dcreg_b200/csrc/odom_plan.hpp"

static int fails = 0;
#define CHECK(c) do { if (!(c)) { std::printf("FAIL line %d: %s\n", __LINE__, #c); if (++fails > 20) return; } } while (0)

struct Cell { int x, y, z; };
typedef unsigned long long u64;

// one cloud alone, literally: bounds, its order (stable by key), entries, table
struct Alone {
    int ox, oy, oz, nx;
    std::vector<int> order;
    std::vector<u64> sorted, keys;
    std::vector<int> val;
    long long entries = 0, cap = 0;
};

static Alone alone(const std::vector<Cell>& c) {
    Alone a;
    int lo[3] = {1 << 30, 1 << 30, 1 << 30}, hi[3] = {-(1 << 30), -(1 << 30), -(1 << 30)};
    for (const Cell& p : c) {
        const int v[3] = {p.x, p.y, p.z};
        for (int k = 0; k < 3; ++k) { lo[k] = std::min(lo[k], v[k]); hi[k] = std::max(hi[k], v[k]); }
    }
    a.ox = lo[0]; a.oy = lo[1]; a.oz = lo[2]; a.nx = hi[0] - lo[0] + 1;
    const long long n = (long long)c.size();
    std::vector<u64> k((size_t)n);
    for (long long i = 0; i < n; ++i) k[(size_t)i] = sparse_index::key(c[(size_t)i].x - a.ox, c[(size_t)i].y - a.oy, c[(size_t)i].z - a.oz);
    a.order.resize((size_t)n);
    std::iota(a.order.begin(), a.order.end(), 0);
    std::stable_sort(a.order.begin(), a.order.end(), [&](int p, int q) { return k[(size_t)p] < k[(size_t)q]; });
    for (long long j = 0; j < n; ++j) a.sorted.push_back(k[(size_t)a.order[(size_t)j]]);
    for (long long j = 0; j < n; ++j) {
        if (j > 0 && a.sorted[(size_t)j - 1] == a.sorted[(size_t)j]) continue;
        int l, h;
        sparse_index::new_entries(a.sorted[(size_t)j], j > 0 ? a.sorted[(size_t)j - 1] : sparse_index::kEmpty, a.nx, &l, &h);
        if (h >= l) a.entries += h - l + 1;
    }
    a.cap = sparse_index::capacity(a.entries);
    a.keys.assign((size_t)a.cap, sparse_index::kEmpty);
    a.val.assign((size_t)a.cap, -7);
    for (long long j = 0; j < n; ++j) {
        if (j > 0 && a.sorted[(size_t)j - 1] == a.sorted[(size_t)j]) continue;
        int l, h;
        sparse_index::new_entries(a.sorted[(size_t)j], j > 0 ? a.sorted[(size_t)j - 1] : sparse_index::kEmpty, a.nx, &l, &h);
        const u64 row = sparse_index::row_of(a.sorted[(size_t)j]) << sparse_index::kBits;
        for (int x = l; x <= h; ++x) {
            const u64 kk = row | (u64)x;
            unsigned s = sparse_index::slot(kk, (unsigned)(a.cap - 1));
            while (a.keys[s] != sparse_index::kEmpty) s = (s + 1) & (unsigned)(a.cap - 1);
            a.keys[s] = kk;
            a.val[s] = (int)sparse_index::cs(a.sorted.data(), n, kk);
        }
    }
    return a;
}

// the arena build of clouds cl, as the device runs it
static void check(const std::vector<std::vector<Cell>>& cl) {
    const int n = (int)cl.size();
    std::vector<long long> seg(1, 0);
    std::vector<Cell> pts;
    std::vector<Alone> ref;
    for (const auto& c : cl) {
        pts.insert(pts.end(), c.begin(), c.end());
        seg.push_back((long long)pts.size());
        ref.push_back(alone(c));
    }
    const long long m = seg.back();
    auto cloud = [&](long long i) { return (int)(std::upper_bound(seg.begin(), seg.end(), i) - seg.begin()) - 1; };
    // two stable passes: (y, x) of point i, then (cloud, z) of the order pass 0 left
    std::vector<int> ord((size_t)m);
    std::iota(ord.begin(), ord.end(), 0);
    auto local = [&](long long i) {
        const Alone& a = ref[(size_t)cloud(i)];
        const Cell& p = pts[(size_t)i];
        return sparse_index::key(p.x - a.ox, p.y - a.oy, p.z - a.oz);
    };
    std::stable_sort(ord.begin(), ord.end(), [&](int p, int q) {
        return (local(p) & ((1ull << (2 * sparse_index::kBits)) - 1)) < (local(q) & ((1ull << (2 * sparse_index::kBits)) - 1));
    });
    std::stable_sort(ord.begin(), ord.end(), [&](int p, int q) {
        const u64 kp = ((u64)cloud(p) << sparse_index::kBits) | (local(p) >> (2 * sparse_index::kBits));
        const u64 kq = ((u64)cloud(q) << sparse_index::kBits) | (local(q) >> (2 * sparse_index::kBits));
        return kp < kq;
    });
    std::vector<u64> sorted((size_t)m);
    for (long long j = 0; j < m; ++j) sorted[(size_t)j] = local(ord[(size_t)j]);
    // the order: every cloud's own, shifted
    for (int b = 0; b < n; ++b)
        for (long long j = seg[(size_t)b]; j < seg[(size_t)b + 1]; ++j) {
            CHECK(ord[(size_t)j] == seg[(size_t)b] + ref[(size_t)b].order[(size_t)(j - seg[(size_t)b])]);
            CHECK(sorted[(size_t)j] == ref[(size_t)b].sorted[(size_t)(j - seg[(size_t)b])]);
        }
    if (fails) return;
    // per-cloud counts within their segments
    std::vector<u64> entries((size_t)n, 0);
    for (long long j = 0; j < m; ++j) {
        const int b = cloud(j);
        const long long first = seg[(size_t)b];
        if (j > first && sorted[(size_t)j - 1] == sorted[(size_t)j]) continue;
        int l, h;
        sparse_index::new_entries(sorted[(size_t)j], j > first ? sorted[(size_t)j - 1] : sparse_index::kEmpty, ref[(size_t)b].nx, &l, &h);
        if (h >= l) entries[(size_t)b] += (u64)(h - l + 1);
    }
    std::vector<long long> cap((size_t)n), off((size_t)n + 1);
    CHECK(sparse_index::layout(n, entries.data(), cap.data(), off.data()) == -1);
    long long at = 0;
    for (int b = 0; b < n; ++b) {
        CHECK((long long)entries[(size_t)b] == ref[(size_t)b].entries);
        CHECK(cap[(size_t)b] == ref[(size_t)b].cap);
        CHECK(off[(size_t)b] == at);
        at += ref[(size_t)b].cap;
    }
    CHECK(off[(size_t)n] == at);
    // inserts into the one buffer
    std::vector<u64> keys((size_t)at, sparse_index::kEmpty);
    std::vector<int> val((size_t)at, -7);
    for (long long j = 0; j < m; ++j) {
        const int b = cloud(j);
        const long long first = seg[(size_t)b];
        if (j > first && sorted[(size_t)j - 1] == sorted[(size_t)j]) continue;
        int l, h;
        sparse_index::new_entries(sorted[(size_t)j], j > first ? sorted[(size_t)j - 1] : sparse_index::kEmpty, ref[(size_t)b].nx, &l, &h);
        const u64 row = sparse_index::row_of(sorted[(size_t)j]) << sparse_index::kBits;
        const unsigned mask = (unsigned)(cap[(size_t)b] - 1);
        for (int x = l; x <= h; ++x) {
            const u64 kk = row | (u64)x;
            unsigned s = sparse_index::slot(kk, mask);
            while (keys[(size_t)(off[(size_t)b] + s)] != sparse_index::kEmpty) s = (s + 1) & mask;
            keys[(size_t)(off[(size_t)b] + s)] = kk;
            val[(size_t)(off[(size_t)b] + s)] =
                (int)(first + sparse_index::cs(sorted.data() + first, seg[(size_t)b + 1] - first, kk));
        }
    }
    // (slots are claimed in cell order in both builds, so the probe sequences, and the slots, agree)
    for (int b = 0; b < n; ++b)
        for (long long s = 0; s < cap[(size_t)b]; ++s) {
            CHECK(keys[(size_t)(off[(size_t)b] + s)] == ref[(size_t)b].keys[(size_t)s]);
            const int want = ref[(size_t)b].keys[(size_t)s] == sparse_index::kEmpty ? -7 : (int)seg[(size_t)b] + ref[(size_t)b].val[(size_t)s];
            CHECK(val[(size_t)(off[(size_t)b] + s)] == want);
            if (fails) return;
        }
}

static void check_layout_limit() {
    const u64 e[3] = {10, (1ull << 31) + 1, 5};      // capacity(2^31 + 1) = 2^33 > kMaxSlots
    long long cap[3], off[4];
    CHECK(sparse_index::layout(3, e, cap, off) == 1);
    CHECK(cap[0] == 1024 && off[1] == 1024);
    const u64 f[2] = {1ull << 31, 0};                // exactly 2^32 slots: allowed
    CHECK(sparse_index::layout(2, f, cap, off) == -1);
    CHECK(cap[0] == sparse_index::kMaxSlots && cap[1] == 1024 && off[2] == sparse_index::kMaxSlots + 1024);
}

static void check_plan() {
    std::vector<arena_plan::Box> boxes;
    long long cells = -1;
    bool sparse = true;
    // dense: plan's result, not sparse
    const int small[12] = {0, 0, 0, 9, 9, 9, -5, -5, -5, 5, 5, 5};
    CHECK(arena_plan::plan_or_sparse(2, small, boxes, &cells, "lane", &sparse).empty());
    CHECK(!sparse && cells == 1000 + 1331);
    // a box over 2^27 cells: sparse, no reason
    const int big[12] = {0, 0, 0, 9, 9, 9, -4000, -4000, 0, 4000, 4000, 9};
    CHECK(!arena_plan::plan(2, big, boxes, &cells, "lane").empty());
    CHECK(arena_plan::plan_or_sparse(2, big, boxes, &cells, "lane", &sparse).empty());
    CHECK(sparse && cells == 0);
    // over 2^30 in all, each box dense: sparse
    std::vector<int> many;
    for (int b = 0; b < 9; ++b) {
        const int x[6] = {0, 0, 0, 511, 511, 499};         // 1.31e8 cells each, 1.18e9 in all
        many.insert(many.end(), x, x + 6);
    }
    CHECK(arena_plan::plan(9, many.data(), boxes, &cells, "lane").find("2^30") != std::string::npos);
    CHECK(arena_plan::plan_or_sparse(9, many.data(), boxes, &cells, "lane", &sparse).empty() && sparse);
    // coordinates outside +-2^19: refused, naming the cloud, even behind a sparse one
    const int far[18] = {0, 0, 0, 9, 9, 9, -4000, -4000, 0, 4000, 4000, 9, 0, 0, 0, (1 << 19) + 1, 0, 0};
    const std::string why = arena_plan::plan_or_sparse(3, far, boxes, &cells, "lane", &sparse);
    CHECK(!sparse && why == arena_plan::out_of_range("lane 2"));
    // map_failure passes an empty reason through: no "dense grid" message for a sparse step
    odom_plan::MapInput in;
    in.add_piece(0, 0, 10);
    in.center.push_back(-1);
    in.end_segment(0);
    int at = -1;
    CHECK(odom_plan::map_failure(in, 1, 4, arena_plan::kMaxPoints, {}, {}, std::vector<int>(big, big + 6), "", &at).empty());
}

int main() {
    std::mt19937_64 rng(2027);
    for (int trial = 0; trial < 30 && !fails; ++trial) {
        const int n = 1 + (int)(rng() % 6);
        std::vector<std::vector<Cell>> cl((size_t)n);
        for (auto& c : cl) {
            const int np = 1 + (int)(rng() % 120), span = 1 + (int)(rng() % 40);
            const int o[3] = {(int)(rng() % 2001) - 1000, (int)(rng() % 2001) - 1000, (int)(rng() % 201) - 100};
            for (int i = 0; i < np; ++i)
                c.push_back({o[0] + (int)(rng() % span), o[1] + (int)(rng() % 4), o[2] + (int)(rng() % 3)});
        }
        check(cl);
    }
    const int L = 1 << 19;
    std::vector<std::vector<Cell>> edge = {
        {{7, -7, 7}},                                                    // a single point
        {{-L, 0, -L}, {-L, 0, -L}, {-L + 3, 0, -L}, {L, 0, L}, {L - 9, 0, L}, {L, 1, L}, {0, 0, 0}, {-L, 1, L}},
        std::vector<Cell>(12, Cell{-3, 4, -5}),                          // one cell: no entry beyond its own dilation
        {{L, L, L}},
    };
    check(edge);
    for (int gap : {8, 9, 10, 17, 18, 19}) {
        std::vector<std::vector<Cell>> cl(3);
        for (int k = 0; k < 4; ++k) {
            cl[0].push_back({-30 + k * gap, 2, -1});
            cl[0].push_back({-30 + k * gap + (k == 3 ? 1 : 0), 3, -1});
            cl[1].push_back({100 + k * gap, -2, 4});
        }
        cl[2].push_back({-40, 0, 5});
        check(cl);
    }
    check_layout_limit();
    check_plan();
    if (fails) { std::printf("%d failure(s)\n", fails); return 1; }
    std::printf("SPARSE_ARENA_OK\n");
    return 0;
}
