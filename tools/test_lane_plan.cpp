// Host check of lane_plan.hpp (tests/test_lane_plan.py): the common-field rule of per-lane settings
// (dcreg_set_lane_params), the uniform case, and the fold mix of a call.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include "../dcreg_b200/csrc/lane_plan.hpp"

static int fails = 0;
#define CHECK(c) do { if (!(c)) { std::printf("FAIL line %d: %s\n", __LINE__, #c); ++fails; } } while (0)

static dcreg_icp_params base() {
    dcreg_icp_params p;
    std::memset(&p, 0, sizeof(p));
    p.search_radius = 1.0; p.max_iterations = 30; p.detection = DCREG_DET_SCHUR_CONDITION_NUMBER;
    p.handling = DCREG_HAND_PRECONDITIONED_CG; p.conv_thresh_rot = 1e-5; p.conv_thresh_trans = 1e-3; p.cond_thresh = 10;
    p.eig_thresh = 120; p.kappa_target = 1; p.pcg_tol = 1e-6; p.pcg_max_iter = 10; p.std_reg_gamma = 0.01;
    p.plane_thickness = 0.2; p.weight_slope = 0.9; p.weight_gate = 0.1; p.min_normal_norm = 1e-6;
    p.min_effective_points = 10;
    return p;
}

int main() {
    // every byte of the struct is in exactly one list, except reserved0
    {
        std::vector<int> owner(sizeof(dcreg_icp_params), 0);
        for (const lane_plan::Field& f : lane_plan::kCommon)
            for (size_t b = 0; b < f.size; ++b) owner[f.offset + b]++;
        for (const lane_plan::Field& f : lane_plan::kPerLane)
            for (size_t b = 0; b < f.size; ++b) owner[f.offset + b]++;
        for (size_t b = 0; b < owner.size(); ++b) {
            const bool reserved = b >= offsetof(dcreg_icp_params, reserved0) &&
                                  b < offsetof(dcreg_icp_params, reserved0) + sizeof(int32_t);
            CHECK(owner[b] == (reserved ? 0 : 1));
        }
    }
    // one differing common field: named with its entry; per-lane fields and reserved0 may differ
    for (const lane_plan::Field& f : lane_plan::kCommon) {
        std::vector<dcreg_icp_params> p(4, base());
        reinterpret_cast<unsigned char*>(&p[2])[f.offset] ^= 1;
        const std::string why = lane_plan::check_common(p.data(), 4, "icp_run_batch");
        CHECK(why.find("icp_run_batch: entry 2: ") == 0);
        CHECK(why.find(f.name) != std::string::npos);
        CHECK(lane_plan::check_common(p.data(), 2, "x").empty());                   // entries past n are not read
    }
    {
        std::vector<dcreg_icp_params> p(3, base());
        p[1].kappa_target = 100; p[1].cond_thresh = 100; p[2].detection = DCREG_DET_NONE_DETE;
        p[2].handling = DCREG_HAND_NONE_HAND; p[2].reserved0 = 7;
        CHECK(lane_plan::check_common(p.data(), 3, "x").empty());
        CHECK(!lane_plan::uniform(p.data(), 3));
        CHECK(lane_plan::uniform(p.data(), 1));
        p[1] = p[0];
        p[1].reserved0 = 9;
        CHECK(lane_plan::uniform(p.data(), 2));                                     // reserved0 ignored
        // -0.0 and 0.0 are different bytes: a common field compares bytes, not values
        p[1].weight_gate = 0.0; p[0].weight_gate = -0.0;
        CHECK(!lane_plan::check_common(p.data(), 2, "x").empty());
    }
    for (const lane_plan::Field& f : lane_plan::kPerLane) {
        std::vector<dcreg_icp_params> p(2, base());
        reinterpret_cast<unsigned char*>(&p[1])[f.offset] ^= 1;
        CHECK(!lane_plan::uniform(p.data(), 2));
        CHECK(lane_plan::check_common(p.data(), 2, "x").empty());
    }
    // the fold mix: all "Ours", none, mixed; without folding (NCCL) every lane needs K2
    {
        std::vector<dcreg_icp_params> p(5, base());
        lane_plan::Mix m = lane_plan::mix(p.data(), 5, true);
        CHECK(m.fold && !m.k2);
        m = lane_plan::mix(p.data(), 5, false);
        CHECK(!m.fold && m.k2);
        p[3].handling = DCREG_HAND_TRUNCATED_SVD;
        m = lane_plan::mix(p.data(), 5, true);
        CHECK(m.fold && m.k2);
        for (auto& q : p) q.detection = DCREG_DET_FULL_EVD_MIN_EIGENVALUE;
        m = lane_plan::mix(p.data(), 5, true);
        CHECK(!m.fold && m.k2);
        p[0].detection = DCREG_DET_SCHUR_CONDITION_NUMBER;                          // Schur detection, CG handling only
        m = lane_plan::mix(p.data(), 5, true);
        CHECK(m.fold && m.k2);
        CHECK(lane_plan::folds(p[0]) && !lane_plan::folds(p[1]) && !lane_plan::folds(p[3]));
    }
    if (fails) return 1;
    std::printf("LANE_PLAN_OK\n");
    return 0;
}
