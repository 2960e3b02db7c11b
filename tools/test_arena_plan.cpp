// Host check of arena_plan.hpp (tests/test_arena_plan.py): the planning of a grid arena, the dense grids of many
// clouds in one set of buffers (dcreg_icp_run_pairs).  Per-cloud boxes and dims from the bounds, cell offsets that
// follow each other, the +-2^19 cell range, the dense-cell limit per cloud and in total, the one-cloud decision of the
// context's target (dense, sparse row index or error), the offset tables; and a replay of the arena's grouping (one stable
// order by global cell id) against every cloud grouped alone.
#include <algorithm>
#include <cstdio>
#include <numeric>
#include <random>
#include <vector>
#include "../dcreg_b200/csrc/arena_plan.hpp"

static int fails = 0;
#define CHECK(c) do { if (!(c)) { std::printf("FAIL line %d: %s\n", __LINE__, #c); ++fails; } } while (0)

int main() {
    std::mt19937_64 rng(2024);
    std::vector<arena_plan::Box> boxes;
    long long cells = 0;
    // dims and offsets of random boxes
    for (int trial = 0; trial < 300; ++trial) {
        const int n = 1 + (int)(rng() % 80);
        std::vector<int> hb((size_t)n * 6);
        for (int b = 0; b < n; ++b)
            for (int k = 0; k < 3; ++k) {
                const int lo = (int)(rng() % 2001) - 1000, w = (int)(rng() % (k == 2 ? 8 : 120));
                hb[6 * b + k] = lo; hb[6 * b + 3 + k] = lo + w;
            }
        CHECK(arena_plan::plan(n, hb.data(), boxes, &cells, "cloud").empty());
        long long off = 0;
        for (int b = 0; b < n; ++b) {
            const arena_plan::Box& x = boxes[b];
            CHECK(x.ox == hb[6 * b] && x.oy == hb[6 * b + 1] && x.oz == hb[6 * b + 2]);
            CHECK(x.nx == hb[6 * b + 3] - hb[6 * b] + 1 && x.ny == hb[6 * b + 4] - hb[6 * b + 1] + 1 &&
                  x.nz == hb[6 * b + 5] - hb[6 * b + 2] + 1);
            CHECK(x.cells == (long long)x.nx * x.ny * x.nz);
            CHECK(x.cell_off == off);
            off += x.cells;
        }
        CHECK(cells == off);
    }
    // the +-2^19 cell range (inclusive), per cloud, on every axis and both sides
    const int L = arena_plan::kCoordLimit;
    for (int k = 0; k < 3; ++k) {
        int hb[12] = {0, 0, 0, 1, 1, 1, -L, -L, -L, -L + 3, -L + 3, -L + 3};
        CHECK(arena_plan::plan(2, hb, boxes, &cells, "cloud").empty());
        arena_plan::Box one;                                    // box_of: the context's target alone
        CHECK(arena_plan::box_of(hb + 6, &one) == arena_plan::kDense && one.ox == -L && one.cells == 64);
        hb[6 + k] = -L - 1;
        const std::string why = arena_plan::plan(2, hb, boxes, &cells, "cloud");
        CHECK(why.find("cloud 1") != std::string::npos && why.find("2^19") != std::string::npos);
        int hi[6] = {L - 2, L - 2, L - 2, L, L, L};
        CHECK(arena_plan::plan(1, hi, boxes, &cells, "cloud").empty());
        CHECK(arena_plan::box_of(hi, &one) == arena_plan::kDense && one.cells == 27 && one.cell_off == 0);
        hi[3 + k] = L + 1;
        CHECK(arena_plan::plan(1, hi, boxes, &cells, "cloud").find("2^19") != std::string::npos);
        CHECK(arena_plan::box_of(hi, &one) == arena_plan::kOutOfRange);                // the context's target: an error
        CHECK(arena_plan::box_of(hb + 6, &one) == arena_plan::kOutOfRange);
    }
    // NaN / infinite coordinates come back as INT_MIN cell coordinates
    {
        int hb[6] = {-2147483647 - 1, 0, 0, 5, 5, 5};
        CHECK(!arena_plan::plan(1, hb, boxes, &cells, "cloud").empty());
    }
    // dense cells per cloud: 2^27 fits, one row more does not
    {
        int ok[6] = {0, 0, 0, 1023, 1023, 127};                     // 1024 * 1024 * 128 = 2^27
        CHECK(arena_plan::plan(1, ok, boxes, &cells, "cloud").empty() && cells == (1ll << 27));
        int big[6] = {0, 0, 0, 1023, 1023, 128};
        const std::string why = arena_plan::plan(1, big, boxes, &cells, "cloud");
        CHECK(why.find("dense") != std::string::npos && why.find("cloud 0") != std::string::npos);
        // the same limit for the context's target alone, where one row more means a sparse row index, not an error
        arena_plan::Box one;
        CHECK(arena_plan::box_of(ok, &one) == arena_plan::kDense && one.cells == (1ll << 27));
        CHECK(one.ox == 0 && one.nx == 1024 && one.ny == 1024 && one.nz == 128 && one.cell_off == 0);
        CHECK(arena_plan::box_of(big, &one) == arena_plan::kTooManyCells && one.cells == (1ll << 27) + (1ll << 20));
    }
    // all clouds of a call: 8 x 2^27 = 2^30 cells fit, a ninth does not
    {
        std::vector<int> hb;
        for (int b = 0; b < 9; ++b) { int r[6] = {0, 0, 0, 1023, 1023, 127}; hb.insert(hb.end(), r, r + 6); }
        CHECK(arena_plan::plan(8, hb.data(), boxes, &cells, "cloud").empty() && cells == (1ll << 30));
        CHECK(arena_plan::plan(8, hb.data(), boxes, &cells, "cloud").empty());
        CHECK(arena_plan::plan(9, hb.data(), boxes, &cells, "cloud").find("2^30") != std::string::npos);
    }
    // offset tables
    {
        const int64_t good[4] = {0, 3, 4, 10}, from1[4] = {1, 3, 4, 10}, desc[4] = {0, 5, 4, 10}, empty[4] = {0, 3, 3, 10};
        CHECK(arena_plan::check_offsets(3, good, 10, "source").empty());
        CHECK(arena_plan::check_offsets(3, good, 9, "source").find("int32") != std::string::npos);
        CHECK(arena_plan::check_offsets(3, from1, 10, "source").find("start at 0") != std::string::npos);
        CHECK(arena_plan::check_offsets(3, desc, 10, "source").find("source 1 is empty") != std::string::npos);
        CHECK(arena_plan::check_offsets(3, empty, 10, "target").find("target 1 is empty") != std::string::npos);
        const int64_t limit[2] = {0, arena_plan::kMaxPoints}, over[2] = {0, arena_plan::kMaxPoints + 1};
        CHECK(arena_plan::check_offsets(1, limit, arena_plan::kMaxPoints, "source").empty());
        CHECK(!arena_plan::check_offsets(1, over, arena_plan::kMaxPoints, "source").empty());
    }
    // the arena's grouping: a stable order of all points by global cell id (cell_off + dense index) puts every cloud's
    // points exactly where a grouping of that cloud alone puts them, shifted by the cloud's first point
    for (int trial = 0; trial < 100; ++trial) {
        const int n = 1 + (int)(rng() % 12);
        std::vector<long long> seg(1, 0);
        std::vector<int> cx, cy, cz, hb((size_t)n * 6);
        for (int b = 0; b < n; ++b) {
            const int m = 1 + (int)(rng() % 300), ox = (int)(rng() % 50) - 25, w = 1 + (int)(rng() % 6);
            int lo[3] = {1 << 30, 1 << 30, 1 << 30}, hi[3] = {-(1 << 30), -(1 << 30), -(1 << 30)};
            for (int i = 0; i < m; ++i) {
                const int c[3] = {ox + (int)(rng() % w), (int)(rng() % w), (int)(rng() % 3)};
                cx.push_back(c[0]); cy.push_back(c[1]); cz.push_back(c[2]);
                for (int k = 0; k < 3; ++k) { lo[k] = std::min(lo[k], c[k]); hi[k] = std::max(hi[k], c[k]); }
            }
            for (int k = 0; k < 3; ++k) { hb[6 * b + k] = lo[k]; hb[6 * b + 3 + k] = hi[k]; }
            seg.push_back(seg.back() + m);
        }
        CHECK(arena_plan::plan(n, hb.data(), boxes, &cells, "cloud").empty());
        auto local = [&](int b, long long i) {
            const arena_plan::Box& x = boxes[b];
            return ((long long)(cz[i] - x.oz) * x.ny + (cy[i] - x.oy)) * x.nx + (cx[i] - x.ox);
        };
        std::vector<long long> key((size_t)seg[n]);
        for (int b = 0; b < n; ++b)
            for (long long i = seg[b]; i < seg[b + 1]; ++i) {
                key[i] = boxes[b].cell_off + local(b, i);
                CHECK(key[i] >= boxes[b].cell_off && key[i] < boxes[b].cell_off + boxes[b].cells);
            }
        std::vector<long long> order((size_t)seg[n]);
        std::iota(order.begin(), order.end(), 0);
        std::stable_sort(order.begin(), order.end(), [&](long long a, long long c) { return key[a] < key[c]; });
        for (int b = 0; b < n; ++b) {
            std::vector<long long> alone((size_t)(seg[b + 1] - seg[b]));
            std::iota(alone.begin(), alone.end(), 0);
            std::stable_sort(alone.begin(), alone.end(),
                             [&](long long a, long long c) { return local(b, seg[b] + a) < local(b, seg[b] + c); });
            for (size_t j = 0; j < alone.size(); ++j) CHECK(order[seg[b] + j] == seg[b] + alone[j]);
        }
    }
    std::printf("%d failures\n", fails);
    if (!fails) std::printf("ARENA_PLAN_OK\n");
    return fails ? 1 : 0;
}
