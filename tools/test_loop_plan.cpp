// Host check of loop_plan::plan_tiles (tests/test_host_la.py::test_loop_tile_plan): every slot is covered exactly once
// per pass structure, tiles stay within the block, a single run never asks for more than the resident blocks.
#include <cstdio>
#include <cstdlib>
#include "../dcreg_b200/csrc/loop_plan.hpp"

static int fails = 0;
#define CHECK(c) do { if (!(c)) { std::printf("FAIL line %d: %s\n", __LINE__, #c); ++fails; } } while (0)

int main() {
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
