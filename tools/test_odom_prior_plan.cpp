// Host test of odom_plan.hpp's prior-map plan (tests/test_odom_prior_plan.py compiles and runs it): make_push with
// prior = true and map_frames = 0 has no anchors and no maps.  Step j holds frame j of every sequence that has one
// (since the sequence started, pushed or retained), a first frame has prev = prev2 = -1, a second prev2 = -1, and the
// history keeps the last two frames of each sequence as poses alone; any chunking of a recording gives, frame for
// frame, the same sequence positions and references as one push.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../dcreg_b200/csrc/odom_plan.hpp"

static int fails = 0;
#define CHECK(c)                                                            \
    do {                                                                    \
        if (!(c)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++fails; } \
    } while (0)


// Push the recording (lens frames per sequence) in `chunks` (per push, frames of every sequence); check every push's
// plan against the prior-map rule, and return every frame's (prev, prev2) as positions in its sequence (-1: none)
static std::vector<std::pair<long long, long long>> run(const std::vector<int>& lens,
                                                        const std::vector<std::vector<int>>& chunks, unsigned seed) {
    const int S = (int)lens.size();
    std::vector<int> so0(1, 0);
    for (int l : lens) so0.push_back(so0.back() + l);
    std::vector<std::pair<long long, long long>> out((size_t)so0.back(), {-2, -2});
    odom_plan::History h(S);
    std::vector<int> done((size_t)S, 0);
    srand(seed);
    // retained frame e of the history: (sequence, position)
    std::vector<std::pair<int, long long>> ret;
    for (const std::vector<int>& cnt : chunks) {
        std::vector<int> so(1, 0);
        for (int s = 0; s < S; ++s) so.push_back(so.back() + cnt[(size_t)s]);
        const int n = so.back();
        std::vector<int64_t> fo(1, 0);
        for (int k = 0; k < n; ++k) fo.push_back(fo.back() + 1 + rand() % 50);
        odom_plan::Push u;
        CHECK(odom_plan::make_push(S, so.data(), n, fo.data(), 0, 1ll << 40, h, &u, nullptr, true).empty());
        const odom_plan::Plan& p = u.plan;
        // no anchors: as many steps as the most frames one sequence pushes, step j holding the j-th of each
        int most = 0;
        for (int c : cnt) most = c > most ? c : most;
        CHECK((int)p.steps.size() == most);
        auto pos = [&](int s, int k) { return (long long)done[(size_t)s] + (k - so[(size_t)s]); };
        auto where = [&](int r) -> std::pair<int, long long> {     // a reference's (sequence, position)
            if (r < n) {
                const int k = p.input[(size_t)r];
                int s = 0;
                while (so[(size_t)s + 1] <= k) ++s;
                return {s, pos(s, k)};
            }
            return ret[(size_t)(r - n)];
        };
        for (size_t i = 0; i < p.steps.size(); ++i) {
            const odom_plan::Step& st = p.steps[i];
            CHECK(st.map.piece_frame.empty() && st.map.center.empty() && st.map.seg.back() == 0);   // empty maps
            CHECK((int)st.prev.size() == st.active && (int)st.prev2.size() == st.active);
            for (int j = 0; j < st.active; ++j) {
                const int s = st.seq[(size_t)j], k = p.input[(size_t)(st.first + j)];
                CHECK(k - so[(size_t)s] == (int)i);
                const long long w = pos(s, k);
                const int r1 = st.prev[(size_t)j], r2 = st.prev2[(size_t)j];
                CHECK((w == 0) == (r1 < 0));
                CHECK((w <= 1) == (r2 < 0));
                if (r1 >= 0) CHECK(where(r1) == std::make_pair(s, w - 1));
                if (r2 >= 0) CHECK(where(r2) == std::make_pair(s, w - 2));
                out[(size_t)(so0[(size_t)s] + w)] = {r1 < 0 ? -1 : w - 1, r2 < 0 ? -1 : w - 2};
            }
        }
        CHECK(p.max_map == 0 && p.max_pieces == 0);
        // the history after the push: poses alone, the last min(seen, 2) frames of each sequence
        CHECK(u.keep_ref.empty() && u.keep_dst.size() == 1 && u.keep_dst[0] == 0);
        std::vector<std::pair<int, long long>> next;
        for (int s = 0; s < S; ++s) {
            const long long c = done[(size_t)s] + cnt[(size_t)s];
            CHECK(u.next.seen[(size_t)s] == c);
            const int keep = u.next.off[(size_t)s + 1] - u.next.off[(size_t)s];
            CHECK(keep == (int)(c < 2 ? c : 2));
            for (int e = u.next.off[(size_t)s]; e < u.next.off[(size_t)s + 1]; ++e) {
                CHECK(u.next.n[(size_t)e] == 0);
                const std::pair<int, long long> x = where(u.next_ref[(size_t)e]);
                CHECK(x == std::make_pair(s, c - keep + (e - u.next.off[(size_t)s])));
                next.push_back(x);
            }
        }
        ret.swap(next);
        h = u.next;
        for (int s = 0; s < S; ++s) done[(size_t)s] += cnt[(size_t)s];
    }
    for (int s = 0; s < S; ++s) CHECK(done[(size_t)s] == lens[(size_t)s]);
    return out;
}

int main() {
    const std::vector<int> lens = {1, 7, 12};
    const auto one = run(lens, {{1, 7, 12}}, 1);
    for (size_t k = 0; k < one.size(); ++k) CHECK(one[k].first >= -1);
    std::vector<std::vector<int>> per_frame;
    for (int k = 0; k < 12; ++k) per_frame.push_back({k < 1 ? 1 : 0, k < 7 ? 1 : 0, 1});
    CHECK(run(lens, per_frame, 2) == one);
    CHECK(run(lens, {{1, 2, 0}, {0, 0, 5}, {0, 3, 1}, {0, 2, 6}}, 3) == one);
    CHECK(run(lens, {{0, 0, 1}, {0, 0, 0}, {1, 7, 0}, {0, 0, 11}}, 4) == one);
    // the window plan is unchanged by the new argument's default: step 0 holds the anchors, prev from step 1
    {
        const int so[3] = {0, 2, 5};
        const int64_t fo[6] = {0, 3, 6, 9, 12, 15};
        odom_plan::Push u;
        CHECK(odom_plan::make_push(2, so, 5, fo, 2, 1ll << 40, odom_plan::History(2), &u).empty());
        CHECK(u.plan.steps.size() == 3 && u.plan.steps[0].prev.empty() && u.plan.steps[1].prev.size() == 2);
    }
    if (fails) return 1;
    std::printf("ODOM_PRIOR_PLAN_OK\n");
    return 0;
}
