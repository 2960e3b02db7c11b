// Host check of loop_plan::plan_scan_tiles (tests/test_scan_plan.py): a batch of scans with ragged slot counts shares one
// grid sized by its largest scan.  Replays the iteration kernel's tile loop for every scan and block: every slot of every
// scan is taken by exactly one block, blocks past a smaller scan's end take nothing, tiles are full, <= 64 blocks per scan.
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>
#include "../dcreg_b200/csrc/loop_plan.hpp"

static int fails = 0;
#define CHECK(c) do { if (!(c)) { std::printf("FAIL line %d: %s\n", __LINE__, #c); ++fails; } } while (0)

// the tile loop of icp_iter2_kernel for one scan of n slots: how often each slot is taken, and how many blocks take none
static void replay(long long n, const loop_plan::Tiles& t, std::vector<int>& hits, long long& idle_blocks) {
    hits.assign((size_t)n, 0);
    idle_blocks = 0;
    for (long long tb = 0; tb < t.grid_x; ++tb) {
        bool any = false;
        for (long long base = tb * t.tile; base < n; base += t.grid_x * t.tile) {
            for (long long i = base; i < base + t.tile && i < n; ++i) ++hits[(size_t)i];
            any = true;
        }
        if (!any) ++idle_blocks;
    }
}

int main() {
    std::mt19937_64 rng(12345);
    long long cases = 0;
    std::vector<int> hits;
    for (int trial = 0; trial < 400; ++trial) {
        // a batch of 1..70 scans; sizes from a single slot to a few tiles past the 64-block cap
        const int nb = 1 + (int)(rng() % 70);
        const long long top = (trial % 4 == 0) ? 40000 : 9000;
        std::vector<long long> n(nb);
        long long mx = 0;
        for (int b = 0; b < nb; ++b) {
            n[b] = 1 + (long long)(rng() % top);
            if (rng() % 5 == 0) n[b] = 256LL * (1 + (long long)(rng() % 30));          // exact multiples of the tile
            mx = n[b] > mx ? n[b] : mx;
        }
        const loop_plan::Tiles t = loop_plan::plan_scan_tiles(mx, 256);
        CHECK(t.tile == 256);
        CHECK(t.grid_x >= 1 && t.grid_x <= 64);
        if (mx <= 64LL * 256) CHECK(t.grid_x * t.tile >= mx && (t.grid_x - 1) * t.tile < mx);   // one pass, no idle block
        for (int b = 0; b < nb; ++b) {
            long long idle = 0;
            replay(n[b], t, hits, idle);
            ++cases;
            bool once = true;
            for (int h : hits) once = once && h == 1;
            CHECK(once);                                                                     // every slot exactly once
            const long long busy = (n[b] + t.tile - 1) / t.tile < t.grid_x ? (n[b] + t.tile - 1) / t.tile : t.grid_x;
            CHECK(idle == t.grid_x - busy);                                                  // the rest write zero rows
            if (n[b] == mx) CHECK(mx > 64LL * 256 || idle == 0);
        }
    }
    // C3-shaped frames (about 6 000 points): 24 blocks per scan; a scan below one tile uses block 0 only
    loop_plan::Tiles a = loop_plan::plan_scan_tiles(6100, 256);
    CHECK(a.tile == 256 && a.grid_x == 24);
    long long idle = 0;
    replay(40, a, hits, idle);
    CHECK(idle == 23 && hits.size() == 40);
    a = loop_plan::plan_scan_tiles(256 * 31, 256);
    CHECK(a.grid_x == 31);
    a = loop_plan::plan_scan_tiles(100000, 256);                                             // the cap: blocks loop
    CHECK(a.tile == 256 && a.grid_x == 64);
    a = loop_plan::plan_scan_tiles(1, 256);
    CHECK(a.tile == 256 && a.grid_x == 1);
    // the same grid as a same-source batch of the largest scan
    for (long long m : {1LL, 255LL, 256LL, 257LL, 7562LL, 16384LL, 16385LL, 1000000LL}) {
        const loop_plan::Tiles s = loop_plan::plan_scan_tiles(m, 256), b = loop_plan::plan_tiles(m, 64, 132, 256);
        CHECK(s.tile == b.tile && s.grid_x == b.grid_x);
    }
    std::printf("%lld scans, %d failures\n", cases, fails);
    if (!fails) std::printf("SCAN_PLAN_OK\n");
    return fails ? 1 : 0;
}
