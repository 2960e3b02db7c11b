// odom_plan.hpp - host-side planning of scan-to-map odometry (dcreg_icp_run_odometry, dcreg_odometry_push): which
// frames run side by side, where every frame lives on the device, and which points make each frame's local map.
//
// One plan serves both: a one-shot call is a push onto the empty history (History(n_seqs): no sequence has a frame yet).
// Step i registers the i-th registrable frame of every sequence that has one (step 0: the anchors, the first frames of
// sequences that start in the push, which are not registered).  On the device the frames are numbered step by step: the
// frames of step i are [Step::first, Step::first + Step::active), one per lane, the lanes in ascending sequence order.
// So a step's frames are one contiguous lane table, and the loop's frame cursor stops at the end of a lane's only frame.
// The map of frame k (since its sequence started) is the window frames [max(0, k - map_frames), k) of its sequence in
// ascending order, each frame's points in their input order; the lanes' maps follow each other in one buffer.
// Everything here is plain C++ so tests/test_odom_plan.py and tests/test_odom_session_plan.py can check it on the CPU
// (tools/test_odom_plan.cpp, tools/test_odom_session_plan.cpp).
#pragma once
#include <algorithm>
#include <cstdint>
#include <string>
#include <vector>

namespace odom_plan {

struct Step {
    int first = 0;                      // device index of the step's first frame; lane j runs first + j
    int active = 0;                     // lanes: the sequences with a frame at this step
    std::vector<int> seq;               // [active] sequence of lane j
    std::vector<int> prev, prev2;       // [active] device index of frame k - 1, and of k - 2 (-1: k - 1 is the anchor)
    std::vector<int64_t> map_seg;       // [active + 1] lane j's map is points [map_seg[j], map_seg[j + 1]) of the step
    std::vector<long long> piece_dst;   // [pieces + 1] where each window frame's points go in the step's maps
    std::vector<long long> piece_src;   // [pieces] first point of the window frame (device order)
    std::vector<int> piece_frame;       // [pieces] device index of the window frame (its pose)
};

struct Plan {
    std::vector<int> dev;               // [n_frames] device index of input frame k
    std::vector<int> input;             // [n_frames] input frame of device index d
    std::vector<int64_t> dev_off;       // [n_frames + 1] point offsets of the frames in device order
    std::vector<Step> steps;            // steps[0]: the anchors (no map, no pieces)
    long long max_map = 0;              // the most map points of one step
    int max_pieces = 0;                 // the most window frames of one step
};

// What a session carries, per sequence, from one push to the next: the frames pushed so far and the last of them: the
// window frames the next frames' maps need, with their points, and the frames the constant-velocity model needs, by
// pose alone.  Sequence s retains its last min(seen, max(map_frames, 2)) frames; the last min(seen, map_frames) of them
// carry points (map_frames = 1 keeps the frame before the last as a pose alone).
struct History {
    std::vector<long long> seen;        // [n_seqs] frames of the sequence since the session opened
    std::vector<int> off;               // [n_seqs + 1] retained frames of sequence s: [off[s], off[s + 1]), oldest first
    std::vector<long long> at, n;       // [retained] first point in the window buffer, and points (0: a pose alone)
    History() = default;
    explicit History(int n_seqs) : seen((size_t)n_seqs, 0), off((size_t)n_seqs + 1, 0) {}   // no frame yet
};

// The retained frames act as anchors that are not in the push: fixed poses, not registered, no outputs.  A frame
// reference r (Step::prev, prev2, piece_frame, and keep_ref below) is the device index of a pushed frame when
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
// + 1 point offsets, both validated; h: the history before the push.  Fails (returns the reason) when the maps of one
// step hold more than max_points points.
inline std::string make_push(int n_seqs, const int* seq_off, int n_frames, const int64_t* frame_off, int map_frames,
                             long long max_points, const History& h, Push* out) {
    Push& u = *out;
    u = Push{};
    Plan& p = u.plan;
    // sequence s's pushed frame j is its frame seen[s] + j, at step j (a new sequence: j = 0 is its anchor) or j + 1
    auto step_of = [&](int s, int j) { return h.seen[(size_t)s] > 0 ? j + 1 : j; };
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
    p.dev_off.assign((size_t)n_frames + 1, 0);
    for (int e = 0; e < n_frames; ++e) {
        const int k = p.input[(size_t)e];
        p.dev_off[(size_t)e + 1] = p.dev_off[(size_t)e] + (frame_off[k + 1] - frame_off[k]);
    }
    // frame w (since open) of sequence s: a pushed frame, or one the history retains
    auto ref = [&](int s, long long w) {
        const long long seen = h.seen[(size_t)s];
        return w >= seen ? p.dev[(size_t)(seq_off[s] + (w - seen))] : n_frames + h.off[(size_t)s + 1] - (int)(seen - w);
    };
    auto points = [&](int r) { return r < n_frames ? p.dev_off[(size_t)r + 1] - p.dev_off[(size_t)r] : h.n[(size_t)(r - n_frames)]; };
    auto first_point = [&](int r) { return r < n_frames ? p.dev_off[(size_t)r] : h.at[(size_t)(r - n_frames)]; };
    for (int i = 1; i < n_steps; ++i) {
        Step& st = p.steps[(size_t)i];
        st.map_seg.push_back(0);
        st.piece_dst.push_back(0);
        long long m = 0;
        for (int j = 0; j < st.active; ++j) {
            const int s = st.seq[(size_t)j];
            const long long k = h.seen[(size_t)s] + (i - step_of(s, 0));
            st.prev.push_back(ref(s, k - 1));
            st.prev2.push_back(k - 1 > 0 ? ref(s, k - 2) : -1);
            for (long long w = std::max<long long>(0, k - map_frames); w < k; ++w) {
                const int r = ref(s, w);
                st.piece_src.push_back(first_point(r));
                st.piece_frame.push_back(r);
                m += points(r);
                st.piece_dst.push_back(m);
            }
            st.map_seg.push_back(m);
        }
        if (m > max_points)
            return "the maps of step " + std::to_string(i) + " hold " + std::to_string(m) +
                   " points, more than " + std::to_string(max_points) + " (int32 indexing)";
        p.max_map = std::max(p.max_map, m);
        p.max_pieces = std::max(p.max_pieces, (int)st.piece_frame.size());
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

struct MapStep {
    std::vector<int> seq;               // [segs] sequence of segment b (the lanes first)
    std::vector<int> center;            // [segs] the frame reference whose pose prunes segment b (-1: an empty segment)
    std::vector<int64_t> seg;           // [segs + 1] segment b is points [seg[b], seg[b + 1]) of the update's input
    std::vector<long long> piece_dst;   // [pieces + 1] where each piece goes in the update's input
    std::vector<long long> piece_src;   // [pieces] its first point: in the old maps, or in the push's packed frames
    std::vector<int> piece_frame;       // [pieces] -1: an old map, copied; else the pushed frame, under its pose
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
inline void map_step(const Plan& p, int i, bool carry, MapState& ms, MapStep* out) {
    MapStep& m = *out;
    m = MapStep{};
    const int n_seqs = (int)ms.at.size(), n_steps = (int)p.steps.size();
    const Step& pv = p.steps[(size_t)i - 1];        // its frames are now their sequences' last frames, not in the maps
    for (int j = 0; j < pv.active; ++j) {
        ms.last[(size_t)pv.seq[(size_t)j]] = pv.first + j;
        ms.pending[(size_t)pv.seq[(size_t)j]] = 1;
    }
    if (i < n_steps) {
        m.seq = p.steps[(size_t)i].seq;
        if (carry) {
            std::vector<char> lane((size_t)n_seqs, 0);
            for (int s : m.seq) lane[(size_t)s] = 1;
            for (int s = 0; s < n_seqs; ++s)
                if (!lane[(size_t)s] && (ms.n[(size_t)s] > 0 || ms.pending[(size_t)s])) m.seq.push_back(s);
        }
    } else {
        for (int s = 0; s < n_seqs; ++s) m.seq.push_back(s);
    }
    m.seg.push_back(0);
    m.piece_dst.push_back(0);
    long long at = 0;
    for (int s : m.seq) {
        const int r = ms.last[(size_t)s];
        if (ms.n[(size_t)s] > 0) {
            m.piece_src.push_back(ms.at[(size_t)s]);
            m.piece_frame.push_back(-1);
            at += ms.n[(size_t)s];
            m.piece_dst.push_back(at);
        }
        if (ms.pending[(size_t)s]) {
            m.piece_src.push_back(p.dev_off[(size_t)r]);
            m.piece_frame.push_back(r);
            at += p.dev_off[(size_t)r + 1] - p.dev_off[(size_t)r];
            m.piece_dst.push_back(at);
        }
        m.center.push_back(at > m.seg.back() ? r : -1);
        m.seg.push_back(at);
    }
}

// After the update m ran: kept[segs + 1], its output's offsets; every sequence of m has its map there, its last frame in
// it.  A sequence that is not in m keeps its state (a one-shot call without carry never reads it again).
inline void map_commit(const MapStep& m, const int64_t* kept, MapState& ms) {
    for (size_t b = 0; b < m.seq.size(); ++b) {
        const int s = m.seq[b];
        ms.at[(size_t)s] = kept[b];
        ms.n[(size_t)s] = kept[b + 1] - kept[b];
        ms.pending[(size_t)s] = 0;
    }
}

}  // namespace odom_plan
