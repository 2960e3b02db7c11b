// Host check of loop_plan.hpp (tests/test_host_la.py::test_loop_tile_plan).  plan_tiles: every slot is covered exactly
// once per pass structure, tiles stay within the block, a single run never asks for more than the resident blocks.
// variant / smem_class: the instantiation of the iteration kernel and its shared memory, against launch_plan's former
// if-ladder, transcribed below, so that the table keeps launching what the ladder launched.  With --flags it prints
// variant_flags of every variant instead.
#include <cstdio>
#include <cstdlib>
#include <set>
#include <string>
#include <tuple>
#include "../dcreg_b200/csrc/loop_plan.hpp"

static int fails = 0;
#define CHECK(c) do { if (!(c)) { std::printf("FAIL line %d: %s\n", __LINE__, #c); ++fails; } } while (0)

using loop_plan::SmemClass;
using loop_plan::kSmemNoGrid;
using loop_plan::kSmemGrid;
using loop_plan::kSmemFull;

// launch_plan's former if-ladder, one row per launch in it, first match wins: the inputs it tested (-1: not tested) and
// the icp_iter2_kernel<kUseWd, kGrids, kSeq, kPlanes, kSparse> it launched (kUseWd -1: the input's weight derivative)
// with its dynamic shared memory (kIter2SmemNoGrid, kIter2SmemGrid, sizeof(Iter2Smem))
struct LadderRow {
    int planes, sparse, table, lanes, wd;
    int k_wd, k_grids, k_seq, k_planes, k_sparse;
    SmemClass smem;
};
static const LadderRow kLadder[] = {
    {1, 1, -1, -1, -1,   0, 0, 0, 1, 1, kSmemNoGrid},
    {1, 0, -1, -1, -1,   0, 0, 0, 1, 0, kSmemNoGrid},
    {0, 1, 1, 1, -1,    -1, 1, 1, 0, 1, kSmemFull},
    {0, 1, 1, 0, -1,    -1, 1, 0, 0, 1, kSmemGrid},
    {0, 1, 0, 1, -1,    -1, 0, 1, 0, 1, kSmemNoGrid},
    {0, 1, 0, 0, -1,    -1, 0, 0, 0, 1, kSmemNoGrid},
    {0, 0, 1, 1, -1,    -1, 1, 1, 0, 0, kSmemFull},
    {0, 0, 1, 0, -1,    -1, 1, 0, 0, 0, kSmemGrid},
    {0, 0, 0, 1, -1,    -1, 0, 1, 0, 0, kSmemNoGrid},
    {0, 0, 0, 0, -1,    -1, 0, 0, 0, 0, kSmemNoGrid},
};

static bool matches(int want, bool have) { return want < 0 || want == (have ? 1 : 0); }

static void check_variants() {
    // every variant is its own instantiation, and takes the shared memory of the kGrids / kSeq rule
    std::set<std::tuple<bool, bool, bool, bool, bool>> insts;
    for (int v = 0; v < loop_plan::kVariants; ++v) {
        const loop_plan::Variant f = loop_plan::variant_flags(v);
        insts.insert(std::make_tuple(f.use_wd, f.grids, f.seq, f.planes, f.sparse));
        const SmemClass want = f.grids && f.seq ? kSmemFull : f.grids ? kSmemGrid : kSmemNoGrid;
        CHECK(loop_plan::smem_class(v) == want);
        if (f.planes) CHECK(!f.use_wd && !f.grids && !f.seq);
    }
    CHECK((int)insts.size() == loop_plan::kVariants);
    // every input combination: the ladder's launch, except seam 1 of a batch (no instantiation: plan_iteration refuses it
    // before it picks one); exactly kVariants variants are reached
    std::set<int> reached;
    for (int bits = 0; bits < 32; ++bits) {
        const bool planes = bits & 1, sparse = bits & 2, table = bits & 4, lanes = bits & 8, wd = bits & 16;
        const int v = loop_plan::variant(planes, sparse, table, lanes, wd);
        if (planes && (table || lanes)) { CHECK(v == -1); continue; }
        CHECK(v >= 0 && v < loop_plan::kVariants);
        if (v < 0 || v >= loop_plan::kVariants) continue;
        reached.insert(v);
        const loop_plan::Variant f = loop_plan::variant_flags(v);
        CHECK(f.planes == planes);                                   // seam 1 only for planes, with either weight derivative
        if (planes) CHECK(v == loop_plan::variant(true, sparse, false, false, !wd));
        const LadderRow* row = nullptr;
        for (const LadderRow& r : kLadder)
            if (!row && matches(r.planes, planes) && matches(r.sparse, sparse) && matches(r.table, table) &&
                matches(r.lanes, lanes) && matches(r.wd, wd))
                row = &r;
        CHECK(row != nullptr);
        if (!row) continue;
        CHECK(f.use_wd == (row->k_wd < 0 ? wd : row->k_wd == 1));
        CHECK(f.grids == (row->k_grids == 1) && f.seq == (row->k_seq == 1) && f.planes == (row->k_planes == 1) &&
              f.sparse == (row->k_sparse == 1));
        CHECK(loop_plan::smem_class(v) == row->smem);
    }
    CHECK((int)reached.size() == loop_plan::kVariants);
}

int main(int argc, char** argv) {
    if (argc > 1 && std::string(argv[1]) == "--flags") {
        // the instantiation table alone, one line per variant: v use_wd grids seq planes sparse
        // (tests/test_gpu_loop_variants.py reads it to check its cases' expected variants)
        for (int v = 0; v < loop_plan::kVariants; ++v) {
            const loop_plan::Variant f = loop_plan::variant_flags(v);
            std::printf("%d %d %d %d %d %d\n", v, f.use_wd, f.grids, f.seq, f.planes, f.sparse);
        }
        return 0;
    }
    check_variants();
    const int sms[] = {1, 8, 132, 148, 160};
    long long cases = 0;
    for (int sm : sms) {
        for (long long n = 1; n <= 400000; n += (n < 3000 ? 1 : 997)) {
            for (int trials : {1, 2, 5000}) {
                const loop_plan::Tiles t = loop_plan::plan_tiles(n, trials, sm, 256);
                ++cases;
                CHECK(t.tile >= 32 && t.tile <= 256 && t.tile % 32 == 0);
                CHECK(t.grid_x >= 1);
                if (trials == 1) {
                    CHECK(t.grid_x <= 3LL * sm);
                    if (t.grid_x < 3LL * sm) CHECK(t.grid_x * t.tile >= n);                  // one pass covers the cloud
                    if (t.grid_x * (long long)t.tile >= n) CHECK((t.grid_x - 1) * t.tile < n);   // no empty block
                    if (n >= 256LL * sm) CHECK(t.tile == 256);                                // a tile per SM: full tiles
                    if (n < 256LL * (sm - 1) && n >= 64LL * sm) CHECK(t.grid_x >= sm);        // small cloud: every SM gets work
                } else {
                    CHECK(t.tile == 256 && t.grid_x <= 64);
                }
            }
        }
    }
    // the shipped cloud and C2 on an H100 (132 SMs)
    loop_plan::Tiles a = loop_plan::plan_tiles(7562, 1, 132, 256);
    CHECK(a.tile == 32 && a.grid_x == 237);
    a = loop_plan::plan_tiles(100000, 1, 132, 256);
    CHECK(a.tile == 256 && a.grid_x == 391);
    a = loop_plan::plan_tiles(10000000, 1, 132, 256);
    CHECK(a.tile == 256 && a.grid_x == 396);
    a = loop_plan::plan_tiles(7562, 5000, 132, 256);
    CHECK(a.tile == 256 && a.grid_x == 30);
    // a single folded run keeps one resident slot for the solver block: at most 3 SMs - 1 tile blocks
    for (int sm : sms)
        for (long long n = 1; n <= 400000; n += (n < 3000 ? 1 : 997)) {
            const loop_plan::Tiles t = loop_plan::plan_tiles(n, 1, sm, 256, 1);
            ++cases;
            CHECK(t.tile >= 32 && t.tile <= 256 && t.tile % 32 == 0);
            CHECK(t.grid_x >= 1 && t.grid_x <= 3LL * sm - 1);
            if (t.grid_x < 3LL * sm - 1) CHECK(t.grid_x * t.tile >= n);
            if (t.grid_x * (long long)t.tile >= n) CHECK((t.grid_x - 1) * t.tile < n);
        }
    a = loop_plan::plan_tiles(100000, 1, 132, 256, 1);
    CHECK(a.tile == 256 && a.grid_x == 391);                                  // C2: 391 tiles + the solver = 392 blocks
    a = loop_plan::plan_tiles(10000000, 1, 132, 256, 1);
    CHECK(a.tile == 256 && a.grid_x == 395);                                  // C4: 395 looping tile blocks
    a = loop_plan::plan_tiles(7562, 1, 132, 256, 1);
    CHECK(a.tile == 32 && a.grid_x == 237);
    std::printf("%lld cases, %d failures\n", cases, fails);
    if (!fails) std::printf("LOOP_PLAN_OK\n");
    return fails ? 1 : 0;
}
