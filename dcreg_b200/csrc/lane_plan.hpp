// Per-lane solver settings of a batched call (dcreg_set_lane_params): which fields may differ between the lanes of one
// call, and where each lane's solve step runs.  Plain host C++ (tools/test_lane_plan.cpp checks it on the CPU).
//
// A lane's settings split in two.  The common fields feed the host plan (ring count, chunking), the search, the rows or
// a template instantiation of the loop kernel, so every entry must hold entry 0's bytes.  The other fields are read only
// by the solve step and the log fill, so each lane may have its own.  The solve step of a lane that runs "Ours" (Schur
// detection + PCG) is folded into the iteration kernel's last block; every other lane's runs in the separate K2 kernel.
#pragma once

#include <cstddef>
#include <cstring>
#include <string>

#include "../../include/dcreg_b200.h"

namespace lane_plan {

struct Field { const char* name; size_t offset, size; };

#define DCREG_LANE_FIELD(f) Field{#f, offsetof(dcreg_icp_params, f), sizeof(dcreg_icp_params::f)}
// must equal entry 0's byte for byte (reserved0 is neither common nor per lane: it is ignored)
constexpr Field kCommon[] = {
    DCREG_LANE_FIELD(search_radius),  DCREG_LANE_FIELD(max_iterations), DCREG_LANE_FIELD(fixed_iterations),
    DCREG_LANE_FIELD(use_weight_derivative), DCREG_LANE_FIELD(plane_thickness), DCREG_LANE_FIELD(weight_slope),
    DCREG_LANE_FIELD(weight_gate),    DCREG_LANE_FIELD(min_normal_norm),
};
// read only by the solve step and the log fill: each lane its own
constexpr Field kPerLane[] = {
    DCREG_LANE_FIELD(detection),      DCREG_LANE_FIELD(handling),     DCREG_LANE_FIELD(conv_thresh_rot),
    DCREG_LANE_FIELD(conv_thresh_trans), DCREG_LANE_FIELD(cond_thresh), DCREG_LANE_FIELD(eig_thresh),
    DCREG_LANE_FIELD(kappa_target),   DCREG_LANE_FIELD(pcg_tol),      DCREG_LANE_FIELD(pcg_max_iter),
    DCREG_LANE_FIELD(std_reg_gamma),  DCREG_LANE_FIELD(min_effective_points),
};
#undef DCREG_LANE_FIELD

inline bool same(const dcreg_icp_params& a, const dcreg_icp_params& b, const Field& f) {
    return std::memcmp(reinterpret_cast<const char*>(&a) + f.offset, reinterpret_cast<const char*>(&b) + f.offset,
                       f.size) == 0;
}

// The solve step of these settings is the warp-cooperative "Ours" step, which the iteration kernel folds
inline bool folds(const dcreg_icp_params& p) {
    return p.detection == DCREG_DET_SCHUR_CONDITION_NUMBER && p.handling == DCREG_HAND_PRECONDITIONED_CG;
}

// "<name>: entry <i>: <field> differs from entry 0 (...)" for the first entry and field that break the common rule, or
// empty
inline std::string check_common(const dcreg_icp_params* p, int n, const char* name) {
    for (int i = 1; i < n; ++i)
        for (const Field& f : kCommon)
            if (!same(p[i], p[0], f))
                return std::string(name) + ": entry " + std::to_string(i) + ": " + f.name +
                       " differs from entry 0 (per-lane settings may differ only in the solve step's fields)";
    return std::string();
}

// Every entry has entry 0's settings: the call runs exactly as with one params (no lane table)
inline bool uniform(const dcreg_icp_params* p, int n) {
    for (int i = 1; i < n; ++i)
        for (const Field& f : kPerLane)
            if (!same(p[i], p[0], f)) return false;
    return true;
}

// Where the lanes' solve steps run.  fold: some lane folds into the iteration kernel; k2: some lane needs the K2 kernel
// after it.  can_fold = false (the sum over ranks goes through NCCL, or the caller wants no fold): none folds.
struct Mix { bool fold = false, k2 = false; };
inline Mix mix(const dcreg_icp_params* p, int n, bool can_fold) {
    Mix m;
    for (int i = 0; i < n; ++i) {
        if (can_fold && folds(p[i])) m.fold = true;
        else m.k2 = true;
    }
    return m;
}

}  // namespace lane_plan
