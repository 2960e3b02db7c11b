// Host test of odom_plan.hpp (tests/test_odom_plan.py compiles and runs it): device numbering, lanes, windows, map
// offsets and the per-step point limit of dcreg_icp_run_odometry, a push onto the empty history, against a direct
// reading of the window rule.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../dcreg_b200/csrc/odom_plan.hpp"

static int fails = 0;
#define CHECK(c)                                                            \
    do {                                                                    \
        if (!(c)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++fails; } \
    } while (0)

// The plan of a one-shot call: one push of the whole recording onto the empty history
static std::string plan(int S, const int* so, int n, const int64_t* fo, int map_frames, long long max_points,
                        odom_plan::Plan* p) {
    odom_plan::Push u;
    const std::string why = odom_plan::make_push(S, so, n, fo, map_frames, max_points, odom_plan::History(S), &u);
    *p = u.plan;
    return why;
}

static void check_case(const std::vector<int>& lens, int map_frames, unsigned seed) {
    const int S = (int)lens.size();
    std::vector<int> so(1, 0);
    for (int l : lens) so.push_back(so.back() + l);
    const int n = so.back();
    std::vector<int64_t> fo(1, 0);
    srand(seed);
    for (int k = 0; k < n; ++k) fo.push_back(fo.back() + 1 + rand() % 50);
    odom_plan::Plan p;
    CHECK(plan(S, so.data(), n, fo.data(), map_frames, 1ll << 40, &p).empty());
    int longest = 0;
    for (int l : lens) longest = l > longest ? l : longest;
    CHECK((int)p.steps.size() == longest);
    // a permutation, numbered step by step, lanes in ascending sequence order
    std::vector<int> seen(n, 0);
    for (int k = 0; k < n; ++k) { CHECK(p.dev[k] >= 0 && p.dev[k] < n); seen[p.dev[k]]++; CHECK(p.input[p.dev[k]] == k); }
    for (int d = 0; d < n; ++d) CHECK(seen[d] == 1);
    CHECK(p.dev_off[0] == 0 && p.dev_off[n] == fo[n]);
    for (int d = 0; d < n; ++d) CHECK(p.dev_off[d + 1] - p.dev_off[d] == fo[p.input[d] + 1] - fo[p.input[d]]);
    long long max_map = 0;
    for (int i = 0; i < longest; ++i) {
        const odom_plan::Step& st = p.steps[i];
        int j = 0;
        for (int s = 0; s < S; ++s) {
            if (lens[s] <= i) continue;
            CHECK(j < st.active && st.seq[j] == s);
            const int k = so[s] + i;
            CHECK(p.dev[k] == st.first + j);
            if (i > 0) {
                CHECK(st.prev[j] == p.dev[k - 1]);
                CHECK(st.prev2[j] == (i >= 2 ? p.dev[k - 2] : -1));
            }
            ++j;
        }
        CHECK(st.active == j);
        if (i == 0) { CHECK(st.map.piece_frame.empty() && st.map.seg.size() == 1 && st.map.seq.empty()); continue; }
        CHECK(st.map.seq == st.seq && st.map.center.empty());     // one segment per lane, nothing pruned
        // every lane's map: the window frames in ascending order, each frame's points contiguous
        size_t q = 0;
        long long m = 0;
        CHECK(st.map.seg[0] == 0 && st.map.piece_dst[0] == 0);
        for (int l = 0; l < st.active; ++l) {
            const int s = st.seq[l], k = so[s] + i;
            const int w0 = k - map_frames > so[s] ? k - map_frames : so[s];
            CHECK(st.map.seg[l] == m);
            for (int w = w0; w < k; ++w, ++q) {
                CHECK(q < st.map.piece_frame.size());
                CHECK(st.map.piece_frame[q] == p.dev[w]);
                CHECK(st.map.piece_src[q] == p.dev_off[p.dev[w]]);
                CHECK(st.map.piece_dst[q] == m);
                m += fo[w + 1] - fo[w];
                CHECK(st.map.piece_dst[q + 1] == m);
            }
            CHECK(st.map.seg[l + 1] == m);
        }
        CHECK(q == st.map.piece_frame.size() && st.map.piece_dst.size() == q + 1);
        max_map = m > max_map ? m : max_map;
    }
    CHECK(p.max_map == max_map);
    // the point limit: exactly the largest step's map points pass, one less fails naming a step
    if (longest > 1) {
        odom_plan::Plan p2;
        CHECK(plan(S, so.data(), n, fo.data(), map_frames, max_map, &p2).empty());
        const std::string why = plan(S, so.data(), n, fo.data(), map_frames, max_map - 1, &p2);
        CHECK(!why.empty() && why.find("step") != std::string::npos);
    }
}

int main() {
    check_case({256}, 10, 1);
    check_case({64, 64, 64, 64, 64, 64, 64, 64}, 10, 2);
    check_case({1, 7, 24}, 10, 3);                     // a one-frame sequence: only an anchor
    check_case({5, 1, 9, 3}, 1, 4);                    // map_frames = 1: the previous frame alone
    check_case({5, 2, 9, 3}, 100, 5);                  // map_frames past every sequence: all frames before k
    check_case({1}, 3, 6);                             // nothing to register
    // the window of frame 7 of a sequence starting at frame 0 with map_frames 3: frames 4, 5, 6
    {
        const int so[2] = {0, 8};
        std::vector<int64_t> fo;
        for (int k = 0; k <= 8; ++k) fo.push_back(10 * k);
        odom_plan::Plan p;
        CHECK(plan(1, so, 8, fo.data(), 3, 1000, &p).empty());
        const odom_plan::Step& st = p.steps[7];
        CHECK(st.map.piece_frame.size() == 3 && st.map.piece_frame[0] == 4 && st.map.piece_frame[2] == 6);
        CHECK(st.map.seg[1] == 30 && p.max_map == 30);
    }
    if (fails) { std::printf("%d failures\n", fails); return 1; }
    std::printf("ODOM_PLAN_OK\n");
    return 0;
}
