// odom_plan.hpp - host-side planning of scan-to-map odometry (dcreg_icp_run_odometry, dcreg_odometry_push): which
// frames run side by side, where every frame lives on the device, and which points make each frame's local map.
//
// One plan serves both: a one-shot call is a push onto the empty history (History(n_seqs): no sequence has a frame yet).
// Step i registers the i-th registrable frame of every sequence that has one (step 0: the anchors, the first frames of
// sequences that start in the push, which are not registered).  On the device the frames are numbered step by step: the
// frames of step i are [Step::first, Step::first + Step::active), one per lane, the lanes in ascending sequence order.
// So a step's frames are one contiguous lane table, and the loop's frame cursor stops at the end of a lane's only frame.
// The map of frame k (since its sequence started) is the window frames [max(0, k - map_frames), k) of its sequence in
// ascending order, each frame's points in their input order; the lanes' maps follow each other in one buffer.  Every
// map input, a step's windows or a voxel-map update's, is one piece table (MapInput), which map_points_kernel lays out.
// A frame has two point ranges in device order: the points it registers with (Plan::dev_off, the loop's segments) and
// the points it gives the maps (Plan::map_off, the map input's pieces and a session's window).  They are one table
// unless dcreg_set_map_input_voxel splits them: then a frame's map input is F_in(frame), its source F_s(F_in(frame)).
// With a prior map (dcreg_set_prior_map) there are no anchors and no maps: every frame registers against the context's
// target, step 0 holds every sequence's first frame in the push, a prev of -1 means "start from T_init", and the
// history keeps poses alone (make_push with prior = true and map_frames = 0).
// Everything here is plain C++ so tests/test_odom_plan.py, tests/test_odom_session_plan.py,
// tests/test_odom_map_plan.py and tests/test_odom_prior_plan.py can check it on the CPU (tools/test_odom_*plan.cpp).
#pragma once
#include <algorithm>
#include <cstdint>
#include <string>
#include <vector>

#include "arena_plan.hpp"

namespace odom_plan {

// A piece table: segment b (one map) is points [seg[b], seg[b + 1]) of the input, piece p (a run of points) is points
// [piece_dst[p], piece_dst[p + 1]) = points piece_src[p] .. of frame reference r = piece_frame[p] (see Push) under its
// final pose, or, for r = -1, of the last voxel-map update's output, copied.
struct MapInput {
    std::vector<int> seq;               // [segs] sequence of segment b (a step's lanes first, in lane order)
    std::vector<int> center;            // [segs] (voxel map) the frame reference whose pose prunes segment b (-1: empty)
    std::vector<int64_t> seg = {0};     // [segs + 1]
    std::vector<long long> piece_dst = {0};     // [pieces + 1]
    std::vector<long long> piece_src;   // [pieces]
    std::vector<int> piece_frame;       // [pieces]
    void add_piece(long long src, int r, long long n) {
        piece_src.push_back(src); piece_frame.push_back(r); piece_dst.push_back(piece_dst.back() + n);
    }
    void end_segment(int s) { seq.push_back(s); seg.push_back(piece_dst.back()); }
};

// A piece table's device layout, appended: long long seg, piece_dst, piece_src; int piece_frame, center
inline void pack(const MapInput& in, std::vector<long long>& ll, std::vector<int>& ints) {
    ll.insert(ll.end(), in.seg.begin(), in.seg.end());
    ll.insert(ll.end(), in.piece_dst.begin(), in.piece_dst.end());
    ll.insert(ll.end(), in.piece_src.begin(), in.piece_src.end());
    ints.insert(ints.end(), in.piece_frame.begin(), in.piece_frame.end());
    ints.insert(ints.end(), in.center.begin(), in.center.end());
}

struct Step {
    int first = 0;                      // device index of the step's first frame; lane j runs first + j
    int active = 0;                     // lanes: the sequences with a frame at this step
    std::vector<int> seq;               // [active] sequence of lane j
    std::vector<int> prev, prev2;       // [active] device index of frame k - 1, and of k - 2 (-1: k - 1 is the anchor;
                                        // prior map: prev -1, frame k is its sequence's first and starts from T_init)
    MapInput map;                       // the lanes' window maps, one segment per lane (the voxel map: none)
};

struct Plan {
    std::vector<int> dev;               // [n_frames] device index of input frame k
    std::vector<int> input;             // [n_frames] input frame of device index d
    std::vector<int64_t> dev_off;       // [n_frames + 1] point offsets of the frames in device order
    std::vector<int64_t> map_off;       // [n_frames + 1] ... of their map-input points (dev_off's values when not split)
    std::vector<Step> steps;            // steps[0]: the anchors (no map; prior map: registered like every step)
    long long max_map = 0;              // the most map points of one step
    int max_pieces = 0;                 // the most window frames of one step
};

// What a session carries, per sequence, from one push to the next: the frames pushed so far and the last of them: the
// window frames the next frames' maps need, with their points, and the frames the constant-velocity model needs, by
// pose alone.  Sequence s retains its last min(seen, max(map_frames, 2)) frames; the last min(seen, map_frames) of them
// carry their map-input points (map_frames = 1 keeps the frame before the last as a pose alone).
struct History {
    std::vector<long long> seen;        // [n_seqs] frames of the sequence since the session opened
    std::vector<int> off;               // [n_seqs + 1] retained frames of sequence s: [off[s], off[s + 1]), oldest first
    std::vector<long long> at, n;       // [retained] first point in the window buffer, and points (0: a pose alone)
    History() = default;
    explicit History(int n_seqs) : seen((size_t)n_seqs, 0), off((size_t)n_seqs + 1, 0) {}   // no frame yet
};

// The retained frames act as anchors that are not in the push: fixed poses, not registered, no outputs.  A frame
// reference r (Step::prev, prev2, MapInput::piece_frame, and keep_ref below) is the device index of a pushed frame when
// r < n_frames, else retained frame r - n_frames of the history; piece_src is then a point of the push's packed frames
// or of the window buffer.  On the empty history every reference is a pushed frame.
struct Push {
    Plan plan;
    History next;                       // the history after the push, its window packed sequence by sequence
    std::vector<int> next_ref;          // [next retained] the frame each retained frame is
    std::vector<long long> keep_dst;    // [keep + 1] the retained frames with points: where each goes in the new window
    std::vector<long long> keep_src;    // [keep] its first point (push or window buffer, by keep_ref)
    std::vector<int> keep_ref;          // [keep] its frame reference
};

inline int retained_frames(long long seen, int map_frames) {
    return (int)std::min<long long>(seen, std::max(map_frames, 2));
}

// seq_off: n_seqs + 1 non-decreasing frame offsets of the pushed frames (a sequence may have none), frame_off: n_frames
// + 1 point offsets, both validated; h: the history before the push.  map_frame_off: n_frames + 1 offsets of the
// frames' map-input points (null: frame_off, the points they register with).  Fails (returns the reason) when the maps
// of one step hold more than max_points points.  prior (with map_frames = 0): no anchors, as described at the top.
inline std::string make_push(int n_seqs, const int* seq_off, int n_frames, const int64_t* frame_off, int map_frames,
                             long long max_points, const History& h, Push* out, const int64_t* map_frame_off = nullptr,
                             bool prior = false) {
    Push& u = *out;
    u = Push{};
    Plan& p = u.plan;
    // sequence s's pushed frame j is its frame seen[s] + j, at step j (a new sequence: j = 0 is its anchor) or j + 1
    // (prior map: at step j)
    auto step_of = [&](int s, int j) { return !prior && h.seen[(size_t)s] > 0 ? j + 1 : j; };
    int n_steps = 0;
    for (int s = 0; s < n_seqs; ++s)
        if (seq_off[s + 1] > seq_off[s]) n_steps = std::max(n_steps, step_of(s, seq_off[s + 1] - seq_off[s] - 1) + 1);
    p.dev.assign((size_t)n_frames, -1);
    p.input.assign((size_t)n_frames, -1);
    p.steps.resize((size_t)n_steps);
    int d = 0;
    for (int i = 0; i < n_steps; ++i) {
        Step& st = p.steps[(size_t)i];
        st.first = d;
        for (int s = 0; s < n_seqs; ++s) {
            const int j = i - step_of(s, 0);
            if (j >= 0 && j < seq_off[s + 1] - seq_off[s]) {
                const int k = seq_off[s] + j;
                p.dev[(size_t)k] = d;
                p.input[(size_t)d] = k;
                st.seq.push_back(s);
                ++d;
            }
        }
        st.active = (int)st.seq.size();
    }
    auto device_order = [&](const int64_t* off) {
        std::vector<int64_t> o((size_t)n_frames + 1, 0);
        for (int e = 0; e < n_frames; ++e) {
            const int k = p.input[(size_t)e];
            o[(size_t)e + 1] = o[(size_t)e] + (off[k + 1] - off[k]);
        }
        return o;
    };
    p.dev_off = device_order(frame_off);
    p.map_off = map_frame_off ? device_order(map_frame_off) : p.dev_off;
    // frame w (since open) of sequence s: a pushed frame, or one the history retains
    auto ref = [&](int s, long long w) {
        const long long seen = h.seen[(size_t)s];
        return w >= seen ? p.dev[(size_t)(seq_off[s] + (w - seen))] : n_frames + h.off[(size_t)s + 1] - (int)(seen - w);
    };
    auto points = [&](int r) { return r < n_frames ? p.map_off[(size_t)r + 1] - p.map_off[(size_t)r] : h.n[(size_t)(r - n_frames)]; };
    auto first_point = [&](int r) { return r < n_frames ? p.map_off[(size_t)r] : h.at[(size_t)(r - n_frames)]; };
    for (int i = prior ? 0 : 1; i < n_steps; ++i) {
        Step& st = p.steps[(size_t)i];
        for (int j = 0; j < st.active; ++j) {
            const int s = st.seq[(size_t)j];
            const long long k = h.seen[(size_t)s] + (i - step_of(s, 0));
            st.prev.push_back(k > 0 ? ref(s, k - 1) : -1);
            st.prev2.push_back(k - 1 > 0 ? ref(s, k - 2) : -1);
            for (long long w = std::max<long long>(0, k - map_frames); w < k; ++w) {
                const int r = ref(s, w);
                st.map.add_piece(first_point(r), r, points(r));
            }
            st.map.end_segment(s);
        }
        const long long m = st.map.seg.back();
        if (m > max_points)
            return "the maps of step " + std::to_string(i) + " hold " + std::to_string(m) +
                   " points, more than " + std::to_string(max_points) + " (int32 indexing)";
        p.max_map = std::max(p.max_map, m);
        p.max_pieces = std::max(p.max_pieces, (int)st.map.piece_frame.size());
    }
    // the history after the push
    History& x = u.next;
    x.seen.resize((size_t)n_seqs);
    x.off.assign(1, 0);
    u.keep_dst.assign(1, 0);
    for (int s = 0; s < n_seqs; ++s) {
        const long long c = h.seen[(size_t)s] + (seq_off[s + 1] - seq_off[s]);
        x.seen[(size_t)s] = c;
        const long long with_points = c - std::min<long long>(c, map_frames);
        for (long long w = c - retained_frames(c, map_frames); w < c; ++w) {
            const int r = ref(s, w);
            u.next_ref.push_back(r);
            x.at.push_back(u.keep_dst.back());
            x.n.push_back(w >= with_points ? points(r) : 0);
            if (w >= with_points) {
                u.keep_ref.push_back(r);
                u.keep_src.push_back(first_point(r));
                u.keep_dst.push_back(u.keep_dst.back() + points(r));
            }
        }
        x.off.push_back((int)x.n.size());
    }
    return std::string();
}

// ---- the voxel map (dcreg_icp_run_odometry_map, dcreg_odometry_open_map) -------------------------------------------
// Instead of a window, every sequence carries one map from frame to frame, KISS-ICP's VoxelHashMap: after frame k is
// registered, M_{k+1} = prune(cap(M_k ++ map_points(T_out[k], frame k)), t_k).  make_push then runs with map_frames = 0:
// the history keeps the motion model's two poses and no points, and the steps have no window pieces.  Instead, before
// its registrations, step i >= 1 runs one map update over segments: segment b is [the current map of its sequence | the
// sequence's last frame, when that frame is not in the map yet], capped and pruned at the pose of that last frame.  The
// segments are the step's lanes in lane order (so the first `active` segments of the update's output are the lanes'
// maps, as the grids need them), then, with `carry`, every other sequence with a map or a frame to insert, ascending, so
// that the update's output holds every map and the previous one can be overwritten.  The final update (i = n_steps,
// after the last registration) has one segment per sequence in sequence order: a session's maps after the push.  The
// sizes come back from the device after every update (map_commit), so the layout of a step is only known at that step.
struct MapState {
    std::vector<long long> at, n;       // [n_seqs] sequence s's map: points [at[s], at[s] + n[s]) of the last update's output
    std::vector<int> last;              // [n_seqs] frame reference of its last frame so far (-1: none)
    std::vector<char> pending;          // [n_seqs] that frame is not in the map yet
};

// The maps before a push: map_off[n_seqs + 1], the session's maps packed by sequence (null: every map empty); h: the
// history before the push (a sequence's last frame is its last retained frame, already in its map)
inline MapState map_start(int n_seqs, int n_frames, const History& h, const long long* map_off) {
    MapState ms;
    ms.at.assign((size_t)n_seqs, 0);
    ms.n.assign((size_t)n_seqs, 0);
    ms.last.assign((size_t)n_seqs, -1);
    ms.pending.assign((size_t)n_seqs, 0);
    for (int s = 0; s < n_seqs; ++s) {
        if (map_off) { ms.at[(size_t)s] = map_off[s]; ms.n[(size_t)s] = map_off[s + 1] - map_off[s]; }
        if (h.off[(size_t)s + 1] > h.off[(size_t)s]) ms.last[(size_t)s] = n_frames + h.off[(size_t)s + 1] - 1;
    }
    return ms;
}

// The update before step i of plan p (1 <= i < steps), or the final update (i = steps)
inline void map_step(const Plan& p, int i, bool carry, MapState& ms, MapInput* out) {
    MapInput& m = *out;
    m = MapInput{};
    const int n_seqs = (int)ms.at.size(), n_steps = (int)p.steps.size();
    const Step& pv = p.steps[(size_t)i - 1];        // its frames are now their sequences' last frames, not in the maps
    for (int j = 0; j < pv.active; ++j) {
        ms.last[(size_t)pv.seq[(size_t)j]] = pv.first + j;
        ms.pending[(size_t)pv.seq[(size_t)j]] = 1;
    }
    std::vector<int> seq;
    if (i < n_steps) {
        seq = p.steps[(size_t)i].seq;
        if (carry) {
            std::vector<char> lane((size_t)n_seqs, 0);
            for (int s : seq) lane[(size_t)s] = 1;
            for (int s = 0; s < n_seqs; ++s)
                if (!lane[(size_t)s] && (ms.n[(size_t)s] > 0 || ms.pending[(size_t)s])) seq.push_back(s);
        }
    } else {
        for (int s = 0; s < n_seqs; ++s) seq.push_back(s);
    }
    for (int s : seq) {
        const int r = ms.last[(size_t)s];
        if (ms.n[(size_t)s] > 0) m.add_piece(ms.at[(size_t)s], -1, ms.n[(size_t)s]);
        if (ms.pending[(size_t)s]) m.add_piece(p.map_off[(size_t)r], r, p.map_off[(size_t)r + 1] - p.map_off[(size_t)r]);
        m.center.push_back(m.piece_dst.back() > m.seg.back() ? r : -1);
        m.end_segment(s);
    }
}

// After the update m ran: kept[segs + 1], its output's offsets; every sequence of m has its map there, its last frame in
// it.  A sequence that is not in m keeps its state (a one-shot call without carry never reads it again).
inline void map_commit(const MapInput& m, const int64_t* kept, MapState& ms) {
    for (size_t b = 0; b < m.seq.size(); ++b) {
        const int s = m.seq[b];
        ms.at[(size_t)s] = kept[b];
        ms.n[(size_t)s] = kept[b + 1] - kept[b];
        ms.pending[(size_t)s] = 0;
    }
}

// Why the maps of `in` (a step's, its first `lanes` segments the lanes', or a session's final voxel-map update, lanes =
// 0) cannot be searched ("": they can), and the segment the message names (*at; a lane by its frame of the step, else by
// center[b]).  From the host data, each empty when the call has none (bad[segs], kept[segs + 1]: the map filter's range
// flags and kept offsets; hb[lanes * 6], plan_why: the grids' bounds, arena_plan::plan's result), in order: more than
// max_points points (not built); a voxel coordinate out of range; a lane's map the prune left empty; the grids' plan.
inline std::string map_failure(const MapInput& in, int lanes, int n_frames, long long max_points,
                               const std::vector<int>& bad, const std::vector<int64_t>& kept, const std::vector<int>& hb,
                               const std::string& plan_why, int* at) {
    int& b = *at;
    b = 0;
    if (in.seg.back() > max_points) {
        while (lanes == 0 && (in.center[(size_t)b] < 0 || in.center[(size_t)b] >= n_frames)) ++b;
        return std::string(lanes > 0 ? "the maps of its step" : "the maps after the push") + " and their new frames hold " +
               std::to_string(in.seg.back()) + " points, more than " + std::to_string(max_points) + " (int32 indexing)";
    }
    for (b = 0; b < (int)bad.size(); ++b)
        if (bad[(size_t)b])
            return b < lanes ? "its local map has a voxel coordinate of the map filter outside [-2^20, 2^20)"
                             : "its points at its pose have a voxel coordinate of the map filter outside [-2^20, 2^20)";
    for (b = 0; !in.center.empty() && !kept.empty() && b < lanes; ++b)
        if (kept[(size_t)b + 1] == kept[(size_t)b])
            return "its local map is empty: every voxel lies max_distance or more from the last pose";
    arena_plan::Box x;
    for (b = 0; !plan_why.empty() && b < lanes - 1 && arena_plan::box_of(hb.data() + 6 * (size_t)b, &x) == arena_plan::kDense;)
        ++b;
    return plan_why;
}

}  // namespace odom_plan
