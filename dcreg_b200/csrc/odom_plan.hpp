// odom_plan.hpp - host-side planning of scan-to-map odometry (dcreg_icp_run_odometry): which frames run side by side,
// where every frame lives on the device, and which points make each frame's local map.
//
// Step i registers frame i of every sequence that has more than i frames (step 0: the anchors, which are not
// registered).  On the device the frames are numbered step by step: the frames of step i are [Step::first, Step::first +
// Step::active), one per lane, the lanes in ascending sequence order.  So a step's frames are one contiguous lane table,
// and the loop's frame cursor stops at the end of a lane's only frame.  The map of lane j is the window frames
// [max(first of the sequence, k - map_frames), k) of its sequence in ascending order, each frame's points in their input
// order; the lanes' maps follow each other in one buffer.  Everything here is plain C++ so tests/test_odom_plan.py can
// check it on the CPU (tools/test_odom_plan.cpp).
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

// seq_off: n_seqs + 1 frame offsets, frame_off: n_frames + 1 point offsets, both already validated (ascending strictly
// from 0).  Fails (returns the reason) when the maps of one step hold more than max_points points.
inline std::string make(int n_seqs, const int* seq_off, int n_frames, const int64_t* frame_off, int map_frames,
                        long long max_points, Plan* out) {
    Plan& p = *out;
    p = Plan{};
    int n_steps = 0;
    for (int s = 0; s < n_seqs; ++s) n_steps = std::max(n_steps, seq_off[s + 1] - seq_off[s]);
    p.dev.assign((size_t)n_frames, -1);
    p.input.assign((size_t)n_frames, -1);
    p.steps.resize((size_t)n_steps);
    int d = 0;
    for (int i = 0; i < n_steps; ++i) {
        Step& st = p.steps[(size_t)i];
        st.first = d;
        for (int s = 0; s < n_seqs; ++s)
            if (seq_off[s + 1] - seq_off[s] > i) {
                const int k = seq_off[s] + i;
                p.dev[(size_t)k] = d;
                p.input[(size_t)d] = k;
                st.seq.push_back(s);
                ++d;
            }
        st.active = (int)st.seq.size();
    }
    p.dev_off.assign((size_t)n_frames + 1, 0);
    for (int e = 0; e < n_frames; ++e) {
        const int k = p.input[(size_t)e];
        p.dev_off[(size_t)e + 1] = p.dev_off[(size_t)e] + (frame_off[k + 1] - frame_off[k]);
    }
    for (int i = 1; i < n_steps; ++i) {
        Step& st = p.steps[(size_t)i];
        st.map_seg.push_back(0);
        st.piece_dst.push_back(0);
        long long m = 0;
        for (int j = 0; j < st.active; ++j) {
            const int s = st.seq[(size_t)j], f0 = seq_off[s], k = f0 + i;
            st.prev.push_back(p.dev[(size_t)k - 1]);
            st.prev2.push_back(k - 1 > f0 ? p.dev[(size_t)k - 2] : -1);
            for (int w = std::max(f0, k - map_frames); w < k; ++w) {
                const int dw = p.dev[(size_t)w];
                st.piece_src.push_back(p.dev_off[(size_t)dw]);
                st.piece_frame.push_back(dw);
                m += frame_off[w + 1] - frame_off[w];
                st.piece_dst.push_back(m);
            }
            st.map_seg.push_back(m);
        }
        if (m > max_points)
            return "icp_run_odometry: the maps of step " + std::to_string(i) + " hold " + std::to_string(m) +
                   " points, more than " + std::to_string(max_points) + " (int32 indexing)";
        p.max_map = std::max(p.max_map, m);
        p.max_pieces = std::max(p.max_pieces, (int)st.piece_frame.size());
    }
    return std::string();
}

}  // namespace odom_plan
