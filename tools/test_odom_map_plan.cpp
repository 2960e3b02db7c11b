// Host test of the voxel map's step layout (odom_plan::map_start / map_step / map_commit; tests/test_odom_map_plan.py
// compiles and runs it).  Random recordings, pushed to a session in random chunks or run as one call, against the rule:
// the map frame k of sequence s registers against holds frames 0 .. k-1 of s, and a session's map after a push holds
// every frame pushed so far.  Points are named by their global index in the recording; the device is simulated as
// arrays of point ids (the push's packed frames in device order, the old maps, each update's output), and the update's
// filter as a fixed rule that drops some points (an id divisible by 3), which keeps the layout honest without the
// geometry: every point the rule keeps must show up once, in frame order, in the right segment.
#include <cstdio>
#include <utility>
#include <vector>

#include "../dcreg_b200/csrc/odom_plan.hpp"

static int fails = 0;
#define CHECK(c)                                                                        \
    do {                                                                                \
        if (!(c)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++fails; } \
    } while (0)

static unsigned rnd(unsigned& state) {
    state = state * 1664525u + 1013904223u;
    return state >> 8;
}

static bool kept(long long id) { return id % 3 != 0; }

struct Recording {
    std::vector<int> lens;                   // frames per sequence
    std::vector<int> so;                     // sequence offsets over the frames
    std::vector<int64_t> fo;                 // point offsets of the frames
    int global(int s, long long w) const { return so[(size_t)s] + (int)w; }
    // the map of frame k of sequence s (frames 0 .. k-1, kept points, in order)
    std::vector<long long> map_of(int s, long long k) const {
        std::vector<long long> m;
        for (long long w = 0; w < k; ++w)
            for (long long q = fo[(size_t)global(s, w)]; q < fo[(size_t)global(s, w) + 1]; ++q)
                if (kept(q)) m.push_back(q);
        return m;
    }
};

// One push: cnt[s] frames of every sequence after done[s]; h / map_off / maps: the session before it (maps: point ids
// packed by sequence, map_off[S + 1]; carry: a session).  Checks every lane's map, and with carry the maps after it.
static void run_push(const Recording& rec, const std::vector<int>& cnt, std::vector<long long>& done, odom_plan::History& h,
                     std::vector<long long>& map_off, std::vector<long long>& maps, bool carry) {
    const int S = (int)rec.lens.size();
    std::vector<int> pso(1, 0);
    std::vector<int64_t> pfo(1, 0);
    std::vector<std::pair<int, long long>> pushed;          // input frame k of the push: (sequence, frame since open)
    for (int s = 0; s < S; ++s) {
        pso.push_back(pso.back() + cnt[(size_t)s]);
        for (int j = 0; j < cnt[(size_t)s]; ++j) {
            const int g = rec.global(s, done[(size_t)s] + j);
            pfo.push_back(pfo.back() + (rec.fo[(size_t)g + 1] - rec.fo[(size_t)g]));
            pushed.push_back({s, done[(size_t)s] + j});
        }
    }
    const int n = pso.back();
    odom_plan::Push u;
    CHECK(odom_plan::make_push(S, pso.data(), n, pfo.data(), 0, 1ll << 40, h, &u).empty());
    const odom_plan::Plan& p = u.plan;
    CHECK(p.max_map == 0 && u.keep_ref.empty());             // map_frames = 0: no window, nothing retained with points
    std::vector<long long> packed;
    for (int d = 0; d < n; ++d) {
        const auto nm = pushed[(size_t)p.input[(size_t)d]];
        const int g = rec.global(nm.first, nm.second);
        for (long long q = rec.fo[(size_t)g]; q < rec.fo[(size_t)g + 1]; ++q) packed.push_back(q);
    }
    odom_plan::MapState ms = odom_plan::map_start(S, n, h, carry ? map_off.data() : nullptr);
    std::vector<long long> old = carry ? maps : std::vector<long long>();
    const int n_steps = (int)p.steps.size();
    for (int i = 1; i <= n_steps; ++i) {
        if (i == n_steps && !carry) break;
        odom_plan::MapInput m;
        odom_plan::map_step(p, i, carry, ms, &m);
        const int segs = (int)m.seq.size();
        CHECK((int)m.seg.size() == segs + 1 && (int)m.center.size() == segs && m.seg[0] == 0);
        CHECK(m.piece_dst.size() == m.piece_src.size() + 1 && m.piece_frame.size() == m.piece_src.size());
        CHECK(m.piece_dst.back() == m.seg.back());
        // the update's input, then the filter: every segment keeps the points the rule keeps, in order
        std::vector<long long> in((size_t)m.seg.back());
        for (size_t q = 0; q + 1 < m.piece_dst.size(); ++q) {
            const int r = m.piece_frame[q];
            CHECK(r < n);
            for (long long t = m.piece_dst[q]; t < m.piece_dst[q + 1]; ++t)
                in[(size_t)t] = r < 0 ? old[(size_t)(m.piece_src[q] + t - m.piece_dst[q])]
                                      : packed[(size_t)(m.piece_src[q] + t - m.piece_dst[q])];
        }
        std::vector<long long> out;
        std::vector<int64_t> kept_off(1, 0);
        for (int b = 0; b < segs; ++b) {
            for (long long t = m.seg[(size_t)b]; t < m.seg[(size_t)b + 1]; ++t)
                if (kept(in[(size_t)t])) out.push_back(in[(size_t)t]);
            kept_off.push_back((int64_t)out.size());
        }
        if (i < n_steps) {
            // the lanes come first, in lane order, each pruned at its previous frame, holding frames 0 .. k-1
            const odom_plan::Step& st = p.steps[(size_t)i];
            CHECK(segs >= st.active);
            for (int j = 0; j < st.active && j < segs; ++j) {
                const int s = st.seq[(size_t)j];
                CHECK(m.seq[(size_t)j] == s);
                CHECK(m.center[(size_t)j] == st.prev[(size_t)j]);
                const long long k = pushed[(size_t)p.input[(size_t)(st.first + j)]].second;
                const std::vector<long long> want = rec.map_of(s, k);
                CHECK(std::vector<long long>(out.begin() + kept_off[(size_t)j], out.begin() + kept_off[(size_t)j + 1]) == want);
            }
            if (!carry) CHECK(segs == st.active);
        } else {
            CHECK(segs == S);
            for (int b = 0; b < S; ++b) CHECK(m.seq[(size_t)b] == b);
        }
        // the lanes ascend, then the carried sequences ascend; only an empty segment has no center
        const int lanes = i < n_steps ? p.steps[(size_t)i].active : 0;
        for (int b = 0; b < segs; ++b) {
            const int s = m.seq[(size_t)b];
            CHECK(b == 0 || b == lanes || s > m.seq[(size_t)b - 1]);
            CHECK((m.center[(size_t)b] < 0) == (m.seg[(size_t)b + 1] == m.seg[(size_t)b]));
        }
        odom_plan::map_commit(m, kept_off.data(), ms);
        old.swap(out);
    }
    for (int s = 0; s < S; ++s) done[(size_t)s] += cnt[(size_t)s];
    if (carry) {
        // the session's maps after the push: every frame pushed so far, packed by sequence
        std::vector<long long> want_off(1, 0), want;
        for (int s = 0; s < S; ++s) {
            const std::vector<long long> m = rec.map_of(s, done[(size_t)s]);
            want.insert(want.end(), m.begin(), m.end());
            want_off.push_back((long long)want.size());
            CHECK(ms.at[(size_t)s] == want_off[(size_t)s] && ms.n[(size_t)s] == (long long)m.size());
            CHECK(!ms.pending[(size_t)s]);
        }
        CHECK(old == want);
        map_off = want_off;
        maps = old;
    }
    h = u.next;
}

static void check_case(const std::vector<int>& lens, unsigned seed, int max_push) {
    const int S = (int)lens.size();
    unsigned state = seed;
    Recording rec;
    rec.lens = lens;
    rec.so.assign(1, 0);
    for (int l : lens) rec.so.push_back(rec.so.back() + l);
    rec.fo.assign(1, 0);
    for (int k = 0; k < rec.so.back(); ++k) rec.fo.push_back(rec.fo.back() + 1 + rnd(state) % 20);
    // one call (no carry, every map starting empty)
    {
        std::vector<long long> done((size_t)S, 0), off((size_t)S + 1, 0), maps;
        odom_plan::History h(S);
        run_push(rec, lens, done, h, off, maps, false);
    }
    // a session, in random chunks with empty entries
    std::vector<long long> done((size_t)S, 0), off((size_t)S + 1, 0), maps;
    odom_plan::History h(S);
    int pushes = 0;
    while (true) {
        int left = 0;
        for (int s = 0; s < S; ++s) left += lens[(size_t)s] - (int)done[(size_t)s];
        if (left == 0) break;
        std::vector<int> cnt((size_t)S, 0);
        int total = 0;
        while (total == 0)
            for (int s = 0; s < S; ++s) {
                const int rest = lens[(size_t)s] - (int)done[(size_t)s];
                cnt[(size_t)s] = rnd(state) % 3 == 0 ? 0 : std::min(rest, (int)(rnd(state) % (max_push + 1)));
                total += cnt[(size_t)s];
            }
        run_push(rec, cnt, done, h, off, maps, true);
        ++pushes;
    }
    CHECK(pushes >= 1);
}

// odom_plan::pack and odom_plan::map_failure on hand-made layouts: 3 segments (segs 0, 1: the lanes of a step; 2: a
// carried sequence) over a push of 6 frames
static void check_failures() {
    const std::string range = "a voxel coordinate of the map filter outside [-2^20, 2^20)";
    odom_plan::MapInput in;
    in.add_piece(0, -1, 4); in.add_piece(40, 2, 3); in.end_segment(1);       // sequence 1: its old map and frame 2
    in.add_piece(4, -1, 2); in.add_piece(50, 5, 2); in.end_segment(3);       // sequence 3: its old map and frame 5
    in.add_piece(6, -1, 3); in.end_segment(4);                               // sequence 4: its old map alone
    in.center = {2, 5, 7};                                                   // 7: a retained frame
    std::vector<long long> ll;
    std::vector<int> ints;
    odom_plan::pack(in, ll, ints);
    CHECK(ll == std::vector<long long>({0, 7, 11, 14, 0, 4, 7, 9, 11, 14, 0, 40, 4, 50, 6}));
    CHECK(ints == std::vector<int>({-1, 2, -1, 5, -1, 2, 5, 7}));
    const std::vector<int> none, ok3 = {0, 0, 0};
    const std::vector<int64_t> kept = {0, 5, 9, 11};
    int at = -1;
    CHECK(odom_plan::map_failure(in, 2, 6, 14, ok3, kept, none, "", &at).empty() && at == 0);
    CHECK(odom_plan::map_failure(in, 0, 6, 14, ok3, kept, none, "", &at).empty());
    // the point limit: a step names its first lane, the final update its first sequence with a pushed frame
    odom_plan::MapInput fin = in;
    fin.center = {-1, 7, 5};
    CHECK(odom_plan::map_failure(in, 2, 6, 13, none, {}, none, "", &at) ==
              "the maps of its step and their new frames hold 14 points, more than 13 (int32 indexing)" && at == 0);
    CHECK(odom_plan::map_failure(fin, 0, 6, 13, none, {}, none, "", &at) ==
              "the maps after the push and their new frames hold 14 points, more than 13 (int32 indexing)" && at == 2);
    // the map filter's range: a lane's map, or a carried sequence's last frame at its pose; before an empty map
    CHECK(odom_plan::map_failure(in, 2, 6, 14, {0, 1, 1}, {0, 5, 5, 9}, none, "", &at) == "its local map has " + range &&
          at == 1);
    CHECK(odom_plan::map_failure(in, 2, 6, 14, {0, 0, 1}, {0, 0, 5, 9}, none, "", &at) ==
              "its points at its pose have " + range && at == 2);
    CHECK(odom_plan::map_failure(in, 0, 6, 14, {0, 1, 0}, kept, none, "", &at) == "its points at its pose have " + range &&
          at == 1);
    // a lane's map that the prune left empty (the voxel map only; a carried sequence's may be empty)
    const std::string empty = "its local map is empty: every voxel lies max_distance or more from the last pose";
    CHECK(odom_plan::map_failure(in, 2, 6, 14, ok3, {0, 5, 5, 5}, none, "x", &at) == empty && at == 1);
    CHECK(odom_plan::map_failure(in, 2, 6, 14, ok3, {0, 5, 9, 9}, none, "", &at).empty());
    CHECK(odom_plan::map_failure(in, 0, 6, 14, ok3, {0, 0, 0, 0}, none, "", &at).empty());
    odom_plan::MapInput win = in;
    win.center.clear();
    CHECK(odom_plan::map_failure(win, 2, 6, 14, ok3, {0, 0, 5, 9}, none, "", &at).empty());
    // the grids' plan: named at the first lane whose box is not dense, else the last lane
    std::vector<int> hb = {0, 0, 0, 3, 3, 3, 0, 0, 0, 1 << 20, 1, 1, 5, 5, 5, 6, 6, 6};
    std::vector<arena_plan::Box> boxes;
    long long cells = 0;
    const std::string why = arena_plan::plan(3, hb.data(), boxes, &cells, "local map of lane");
    CHECK(!why.empty() && why.find("local map of lane 1") != std::string::npos);
    CHECK(odom_plan::map_failure(win, 3, 6, 14, none, {}, hb, why, &at) == why && at == 1);
    CHECK(odom_plan::map_failure(in, 3, 6, 14, ok3, {0, 5, 9, 11}, hb, why, &at) == why && at == 1);
    hb[9] = 1;
    CHECK(arena_plan::plan(3, hb.data(), boxes, &cells, "local map of lane").empty());
    CHECK(odom_plan::map_failure(win, 3, 6, 14, none, {}, hb, "all grids too large", &at) == "all grids too large" &&
          at == 2);
    CHECK(odom_plan::map_failure(win, 2, 6, 14, none, {}, hb, "all grids too large", &at) == "all grids too large" &&
          at == 1);
}

int main() {
    check_failures();
    unsigned state = 4242u;
    for (int c = 0; c < 60; ++c) {
        const int S = 1 + (int)(rnd(state) % 4);
        std::vector<int> lens;
        for (int s = 0; s < S; ++s) lens.push_back(1 + (int)(rnd(state) % 30));
        const int max_push[3] = {1, 3, 12};
        check_case(lens, 2000u + c, max_push[c % 3]);
    }
    check_case({1, 7, 12}, 7, 1);            // a sequence of one frame: its anchor only
    check_case({30}, 8, 30);                 // everything in one push
    if (fails) { std::printf("%d failures\n", fails); return 1; }
    std::printf("ODOM_MAP_PLAN_OK\n");
    return 0;
}
