// Host test of odom_plan.hpp's two point ranges per frame (tests/test_odom_map_input_plan.py compiles and runs it): with
// dcreg_set_map_input_voxel a frame registers with one set of points (Plan::dev_off, the loop's segments) and gives the
// maps another (Plan::map_off: the window pieces, the voxel-map updates and a session's history).  Without it the two
// are one table and the plan is the one make_push made before.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../dcreg_b200/csrc/odom_plan.hpp"

static int fails = 0;
#define CHECK(c)                                                            \
    do {                                                                    \
        if (!(c)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++fails; } \
    } while (0)

static bool same_input(const odom_plan::MapInput& a, const odom_plan::MapInput& b) {
    return a.seq == b.seq && a.center == b.center && a.seg == b.seg && a.piece_dst == b.piece_dst &&
           a.piece_src == b.piece_src && a.piece_frame == b.piece_frame;
}

static bool same_push(const odom_plan::Push& a, const odom_plan::Push& b) {
    const odom_plan::Plan &p = a.plan, &q = b.plan;
    bool ok = p.dev == q.dev && p.input == q.input && p.dev_off == q.dev_off && p.map_off == q.map_off &&
              p.max_map == q.max_map && p.max_pieces == q.max_pieces && p.steps.size() == q.steps.size();
    for (size_t i = 0; ok && i < p.steps.size(); ++i) {
        const odom_plan::Step &s = p.steps[i], &t = q.steps[i];
        ok = s.first == t.first && s.active == t.active && s.seq == t.seq && s.prev == t.prev && s.prev2 == t.prev2 &&
             same_input(s.map, t.map);
    }
    return ok && a.next.seen == b.next.seen && a.next.off == b.next.off && a.next.at == b.next.at &&
           a.next.n == b.next.n && a.next_ref == b.next_ref && a.keep_dst == b.keep_dst && a.keep_src == b.keep_src &&
           a.keep_ref == b.keep_ref;
}

// Offsets of n frames of 1 .. 50 points, and of a subset of each (the source: F_s of the map input)
static void frames(int n, unsigned seed, std::vector<int64_t>* in, std::vector<int64_t>* src) {
    srand(seed);
    in->assign(1, 0);
    src->assign(1, 0);
    for (int k = 0; k < n; ++k) {
        const int m = 1 + rand() % 50;
        in->push_back(in->back() + m);
        src->push_back(src->back() + 1 + rand() % m);
    }
}

// One recording pushed in `chunks` (frames per sequence per push) onto the empty history, with and without the split:
// every push's source ranges are the unsplit plan's, its map ranges those of a plan made from the map-input offsets
static void check_pushes(const std::vector<int>& lens, const std::vector<std::vector<int>>& chunks, int map_frames,
                         unsigned seed) {
    const int S = (int)lens.size();
    int n = 0;
    for (int l : lens) n += l;
    std::vector<int64_t> in, src;
    frames(n, seed, &in, &src);
    std::vector<int> first(1, 0);
    for (int l : lens) first.push_back(first.back() + l);
    odom_plan::History h_split(S), h_src(S), h_in(S);
    std::vector<int> done((size_t)S, 0);
    for (const std::vector<int>& cnt : chunks) {
        // the push's frames in the caller's order: sequence by sequence
        std::vector<int> so(1, 0);
        std::vector<int64_t> fo_in(1, 0), fo_src(1, 0);
        for (int s = 0; s < S; ++s) {
            for (int j = 0; j < cnt[(size_t)s]; ++j) {
                const int k = first[(size_t)s] + done[(size_t)s] + j;
                fo_in.push_back(fo_in.back() + (in[k + 1] - in[k]));
                fo_src.push_back(fo_src.back() + (src[k + 1] - src[k]));
            }
            so.push_back(so.back() + cnt[(size_t)s]);
        }
        const int m = so.back();
        odom_plan::Push u_same, u_null, u_split, u_src, u_in;
        // off: the same table twice, or none, is the plan of one table
        CHECK(odom_plan::make_push(S, so.data(), m, fo_src.data(), map_frames, 1ll << 40, h_src, &u_null).empty());
        CHECK(odom_plan::make_push(S, so.data(), m, fo_src.data(), map_frames, 1ll << 40, h_src, &u_same,
                                   fo_src.data()).empty());
        CHECK(same_push(u_null, u_same));
        CHECK(u_null.plan.map_off == u_null.plan.dev_off);
        // split: the loop's ranges from the source, everything the maps read from the map input
        CHECK(odom_plan::make_push(S, so.data(), m, fo_src.data(), map_frames, 1ll << 40, h_split, &u_split,
                                   fo_in.data()).empty());
        CHECK(odom_plan::make_push(S, so.data(), m, fo_in.data(), map_frames, 1ll << 40, h_in, &u_in).empty());
        const odom_plan::Plan &p = u_split.plan, &q = u_in.plan;
        CHECK(p.dev == q.dev && p.input == q.input && p.dev_off == u_null.plan.dev_off && p.map_off == q.dev_off);
        CHECK(p.max_map == q.max_map && p.max_pieces == q.max_pieces && p.steps.size() == q.steps.size());
        for (size_t i = 0; i < p.steps.size(); ++i) {
            const odom_plan::Step &s = p.steps[i], &t = q.steps[i];
            CHECK(s.first == t.first && s.active == t.active && s.seq == t.seq && s.prev == t.prev && s.prev2 == t.prev2);
            CHECK(same_input(s.map, t.map));
            for (size_t c = 0; c < s.map.piece_frame.size(); ++c) {
                const int r = s.map.piece_frame[c];
                if (r < m) CHECK(s.map.piece_src[c] == p.map_off[(size_t)r]);
            }
        }
        CHECK(u_split.next.at == u_in.next.at && u_split.next.n == u_in.next.n && u_split.next.off == u_in.next.off);
        CHECK(u_split.keep_dst == u_in.keep_dst && u_split.keep_src == u_in.keep_src && u_split.keep_ref == u_in.keep_ref);
        // the voxel map's updates: a pending frame's piece is its map-input range
        if (map_frames == 0 && !p.steps.empty()) {
            odom_plan::MapState a = odom_plan::map_start(S, m, h_split, nullptr), b = odom_plan::map_start(S, m, h_in, nullptr);
            for (int i = 1; i <= (int)p.steps.size(); ++i) {
                odom_plan::MapInput x, y;
                odom_plan::map_step(p, i, true, a, &x);
                odom_plan::map_step(q, i, true, b, &y);
                CHECK(same_input(x, y));
                odom_plan::map_commit(x, x.seg.data(), a);
                odom_plan::map_commit(y, y.seg.data(), b);
            }
        }
        h_split = u_split.next;
        h_src = u_null.next;
        h_in = u_in.next;
        for (int s = 0; s < S; ++s) done[(size_t)s] += cnt[(size_t)s];
    }
}

int main() {
    check_pushes({1, 7, 12}, {{1, 7, 12}}, 3, 1);                                  // one call
    check_pushes({1, 7, 12}, {{1, 2, 0}, {0, 0, 5}, {0, 3, 1}, {0, 2, 6}}, 3, 2);   // ragged pushes
    check_pushes({5, 5}, {{1, 1}, {1, 1}, {1, 1}, {1, 1}, {1, 1}}, 1, 3);           // one frame per push, map_frames 1
    check_pushes({6, 9, 2}, {{6, 9, 2}}, 100, 4);                                  // a window past every sequence
    check_pushes({1, 7, 12}, {{1, 7, 12}}, 0, 5);                                  // the voxel map
    check_pushes({1, 7, 12}, {{1, 2, 0}, {0, 0, 5}, {0, 3, 1}, {0, 2, 6}}, 0, 6);
    // the point limit counts map-input points: a limit the sources pass but the map inputs do not fails
    {
        const int so[2] = {0, 4};
        const std::vector<int64_t> in = {0, 10, 20, 30, 40}, src = {0, 1, 2, 3, 4};
        odom_plan::Push u;
        CHECK(odom_plan::make_push(1, so, 4, src.data(), 3, 29, odom_plan::History(1), &u, in.data()).find("step") !=
              std::string::npos);
        CHECK(odom_plan::make_push(1, so, 4, src.data(), 3, 30, odom_plan::History(1), &u, in.data()).empty());
        CHECK(u.plan.max_map == 30 && u.plan.dev_off.back() == 4 && u.plan.map_off.back() == 40);
    }
    if (fails) { std::printf("%d failures\n", fails); return 1; }
    std::printf("ODOM_MAP_INPUT_PLAN_OK\n");
    return 0;
}
