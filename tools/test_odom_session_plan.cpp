// Host test of odom_plan::make_push (tests/test_odom_session_plan.py compiles and runs it): random recordings pushed to
// a session in random chunks, against one push of the whole recording onto the empty history (the one-call plan, which
// tools/test_odom_plan.cpp checks against the window rule).  Every frame is named by (sequence, frame of the sequence)
// and every point by its global index in the recording, so a push's window pieces, previous frames and retained window
// can be compared with the one-call plan whatever the chunking.  The device buffers are simulated as arrays of point
// ids: the push's packed frames in device order, and the window buffer the retain step gathers.
#include <cstdio>
#include <cstdlib>
#include <utility>
#include <vector>

#include "../dcreg_b200/csrc/odom_plan.hpp"

static int fails = 0;
#define CHECK(c)                                                                        \
    do {                                                                                \
        if (!(c)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++fails; } \
    } while (0)

typedef std::pair<int, long long> Name;      // (sequence, frame of the sequence)

static unsigned rnd(unsigned& state) {
    state = state * 1664525u + 1013904223u;
    return state >> 8;
}

static void check_case(const std::vector<int>& lens, int map_frames, unsigned seed, int max_push) {
    const int S = (int)lens.size();
    unsigned state = seed;
    // the whole recording, as one call sees it
    std::vector<int> so(1, 0);
    for (int l : lens) so.push_back(so.back() + l);
    const int n = so.back();
    std::vector<int64_t> fo(1, 0);
    for (int k = 0; k < n; ++k) fo.push_back(fo.back() + 1 + rnd(state) % 40);
    odom_plan::Push one;
    CHECK(odom_plan::make_push(S, so.data(), n, fo.data(), map_frames, 1ll << 40, odom_plan::History(S), &one).empty());
    const odom_plan::Plan& full = one.plan;
    auto full_name = [&](int d) {
        const int k = full.input[(size_t)d];
        int s = 0;
        while (so[s + 1] <= k) ++s;
        return Name(s, k - so[s]);
    };
    auto global = [&](int s, long long w) { return so[s] + (int)w; };
    // the session
    odom_plan::History h(S);
    std::vector<Name> h_name;                // the retained frames' names
    std::vector<long long> window;           // the window buffer: point ids
    std::vector<long long> done((size_t)S, 0);
    int pushes = 0;
    while (true) {
        int left = 0;
        for (int s = 0; s < S; ++s) left += lens[s] - (int)done[(size_t)s];
        if (left == 0) break;
        // a random chunk: every sequence 0 .. max_push frames (often none), at least one frame in all
        std::vector<int> cnt((size_t)S, 0);
        int total = 0;
        while (total == 0)
            for (int s = 0; s < S; ++s) {
                const int rest = lens[s] - (int)done[(size_t)s];
                cnt[(size_t)s] = rnd(state) % 3 == 0 ? 0 : std::min(rest, (int)(rnd(state) % (max_push + 1)));
                total += cnt[(size_t)s];
            }
        std::vector<int> pso(1, 0);
        std::vector<int64_t> pfo(1, 0);
        std::vector<Name> pushed;            // input frame k of the push
        for (int s = 0; s < S; ++s) {
            pso.push_back(pso.back() + cnt[(size_t)s]);
            for (int j = 0; j < cnt[(size_t)s]; ++j) {
                const int g = global(s, done[(size_t)s] + j);
                pfo.push_back(pfo.back() + (fo[g + 1] - fo[g]));
                pushed.push_back(Name(s, done[(size_t)s] + j));
            }
        }
        odom_plan::Push u;
        CHECK(odom_plan::make_push(S, pso.data(), total, pfo.data(), map_frames, 1ll << 40, h, &u).empty());
        const odom_plan::Plan& p = u.plan;
        // the push's packed frames in device order
        std::vector<long long> packed;
        CHECK((int)p.dev_off.size() == total + 1 && p.dev_off[0] == 0);
        for (int d = 0; d < total; ++d) {
            const int k = p.input[(size_t)d];
            CHECK(k >= 0 && k < total && p.dev[(size_t)k] == d);
            const Name nm = pushed[(size_t)k];
            const int g = global(nm.first, nm.second);
            for (long long q = fo[g]; q < fo[g + 1]; ++q) packed.push_back(q);
            CHECK(p.dev_off[(size_t)d + 1] == (long long)packed.size());
        }
        auto name_of = [&](int r) { return r < total ? pushed[(size_t)p.input[(size_t)r]] : h_name[(size_t)(r - total)]; };
        auto point_at = [&](int r, long long at) { return r < total ? packed[(size_t)at] : window[(size_t)at]; };
        // every pushed frame: its step, previous frames and window equal the one-call plan's
        for (int i = 0; i < (int)p.steps.size(); ++i) {
            const odom_plan::Step& st = p.steps[(size_t)i];
            int prev_s = -1;
            for (int j = 0; j < st.active; ++j) {
                const int d = st.first + j, s = st.seq[(size_t)j];
                CHECK(s > prev_s);
                prev_s = s;
                const Name nm = name_of(d);
                CHECK(nm.first == s);
                CHECK((nm.second == 0) == (i == 0));                 // step 0: exactly the anchors
                CHECK(i == nm.second - h.seen[(size_t)s] + (h.seen[(size_t)s] > 0 ? 1 : 0));
                if (i == 0) continue;
                const int fd = full.dev[(size_t)global(s, nm.second)];
                const odom_plan::Step& fs = full.steps[(size_t)nm.second];
                const int fj = fd - fs.first;
                CHECK(name_of(st.prev[(size_t)j]) == full_name(fs.prev[(size_t)fj]));
                CHECK((st.prev2[(size_t)j] < 0) == (fs.prev2[(size_t)fj] < 0));
                if (st.prev2[(size_t)j] >= 0) CHECK(name_of(st.prev2[(size_t)j]) == full_name(fs.prev2[(size_t)fj]));
                // window pieces: the same frames in the same order, and the points they read are those frames' points
                CHECK(st.map.seg[(size_t)j + 1] - st.map.seg[(size_t)j] == fs.map.seg[(size_t)fj + 1] - fs.map.seg[(size_t)fj]);
                size_t q0 = 0, f0 = 0;
                while (q0 < st.map.piece_dst.size() && st.map.piece_dst[q0] < st.map.seg[(size_t)j]) ++q0;
                while (f0 < fs.map.piece_dst.size() && fs.map.piece_dst[f0] < fs.map.seg[(size_t)fj]) ++f0;
                for (; f0 + 1 < fs.map.piece_dst.size() && fs.map.piece_dst[f0] < fs.map.seg[(size_t)fj + 1]; ++f0, ++q0) {
                    CHECK(q0 + 1 < st.map.piece_dst.size());
                    if (q0 + 1 >= st.map.piece_dst.size()) break;
                    const int r = st.map.piece_frame[q0];
                    const Name w = name_of(r);
                    CHECK(w == full_name(fs.map.piece_frame[f0]));
                    const long long len = st.map.piece_dst[q0 + 1] - st.map.piece_dst[q0];
                    CHECK(len == fs.map.piece_dst[f0 + 1] - fs.map.piece_dst[f0]);
                    const int g = global(w.first, w.second);
                    CHECK(len == fo[g + 1] - fo[g]);
                    for (long long t = 0; t < len; ++t) CHECK(point_at(r, st.map.piece_src[q0] + t) == fo[g] + t);
                }
            }
        }
        // the per-step point limit: the largest step's map passes, one point less fails naming a step
        if (p.max_map > 0) {
            odom_plan::Push u2;
            CHECK(odom_plan::make_push(S, pso.data(), total, pfo.data(), map_frames, p.max_map, h, &u2).empty());
            const std::string why = odom_plan::make_push(S, pso.data(), total, pfo.data(), map_frames, p.max_map - 1, h, &u2);
            CHECK(!why.empty() && why.find("step") != std::string::npos);
        }
        // retain: gather the new window, then check it holds the last min(map_frames, c) frames of every sequence with
        // their points, behind the frame before them as a pose alone when map_frames = 1
        std::vector<long long> win2((size_t)u.keep_dst.back());
        for (size_t q = 0; q + 1 < u.keep_dst.size(); ++q)
            for (long long t = u.keep_dst[q]; t < u.keep_dst[q + 1]; ++t)
                win2[(size_t)t] = point_at(u.keep_ref[q], u.keep_src[q] + (t - u.keep_dst[q]));
        std::vector<Name> name2;
        for (int r : u.next_ref) name2.push_back(name_of(r));
        const odom_plan::History& x = u.next;
        CHECK(x.off.size() == (size_t)S + 1 && x.off[0] == 0 && (size_t)x.off[S] == x.n.size());
        long long at = 0;
        for (int s = 0; s < S; ++s) {
            done[(size_t)s] += cnt[(size_t)s];
            const long long c = done[(size_t)s];
            CHECK(x.seen[(size_t)s] == c);
            const long long keep = std::min<long long>(c, std::max(map_frames, 2));
            CHECK(x.off[s + 1] - x.off[s] == keep);
            for (int e = x.off[s]; e < x.off[s + 1]; ++e) {
                const long long w = c - (x.off[s + 1] - e);
                CHECK(name2[(size_t)e] == Name(s, w));
                const int g = global(s, w);
                if (w < c - map_frames) { CHECK(x.n[(size_t)e] == 0); continue; }
                CHECK(x.n[(size_t)e] == fo[g + 1] - fo[g] && x.at[(size_t)e] == at);
                for (long long t = 0; t < x.n[(size_t)e]; ++t) CHECK(win2[(size_t)(at + t)] == fo[g] + t);
                at += x.n[(size_t)e];
            }
        }
        CHECK(at == (long long)win2.size());
        h = x;
        h_name = name2;
        window = win2;
        ++pushes;
    }
    CHECK(pushes >= 1);
}

int main() {
    unsigned state = 12345u;
    for (int c = 0; c < 60; ++c) {
        const int S = 1 + (int)(rnd(state) % 4);
        std::vector<int> lens;
        for (int s = 0; s < S; ++s) lens.push_back(1 + (int)(rnd(state) % 40));
        const int mf[3] = {1, 3, 100};
        const int max_push[3] = {1, 3, 12};
        check_case(lens, mf[c % 3], 1000u + c, max_push[(c / 3) % 3]);
    }
    check_case({1, 7, 12}, 3, 7, 1);         // the GPU tests' recording, one frame per sequence per push
    check_case({40}, 100, 8, 40);            // everything in one push: the plan of one call
    if (fails) { std::printf("%d failures\n", fails); return 1; }
    std::printf("ODOM_SESSION_PLAN_OK\n");
    return 0;
}
