// k2_solve.cuh - K2: degeneracy analysis + solve + SE(3) update, device side.
//
// What it replaces (reference file:line, relative to the DCReg checkout):
//   DCReg::analyzeDegeneracy            DCReg/include/dcreg.hpp:45-166
//   released Schur-complement block     DCReg/src/icp_test_runner.cpp:2418-2469
//   Schur detection / preconditioner /  stubs at dcreg.hpp:96-98,186-193,267-287; algorithm from the
//   PCG ("Ours")                        paper's Alg. 1-3, Eq. 18-21, 43-46 (SURVEY.md §3.4)
//   DCReg::solveDegenerateSystem        dcreg.hpp:168-264 (TReg / SR / TSVD / QR handlers)
//   SE3State::boxplus, MathUtils::exp   DCReg/include/math_utils.hpp:158-166, 20-33
//   convergence / abort rules           icp_test_runner.cpp:1847-1854, 1942-1950, 1958-2003
#pragma once
#include "../../include/dcreg_b200.h"
#include "small_la.cuh"
#include "k2_fast.cuh"

namespace k2 {

// accumulator layout shared by K1 and K2 (hessian_computer.h:62-123 order + stats)
constexpr int kAcc = 32;        // 21 upper-tri + 6 rhs + sum r^2 + N_eff + N_corr_pt + sum b^2 (+1 pad)
constexpr int kAccUsed = 31;
constexpr int kAccSumR2 = 27;
constexpr int kAccNeff = 28;
constexpr int kAccNpt = 29;
constexpr int kAccSumB2 = 30;

struct IcpState {               // device-resident loop state, written only by K2
    double R[9];
    double t[3];
    int iter;                   // iterations completed
    int done;                   // 1: stop (converged, aborted or max_iterations reached)
    int converged;
    int status;                 // dcreg_status
    double H_last[36];
    long long n_source_total;   // denominator of fitness (global count when sharded)
    // temporal coherence of the correspondence stage (dcreg_b200.cu, icp_iter2_kernel): written here by K2
    double step_rot, step_trans; // |omega| and |v| of the last update
    int seeds;                  // 1: the iteration kernel that just ran left neighbour records behind
    int coherent_used;          // mode the iteration kernel that just ran was in (it reads it from `coherent`)
    int coherent;               // 1: the next iteration may use the records (the last update was small)
    int warm;                   // 1: V_warm holds the Schur eigenvectors of the previous iteration (k2_fast.cuh)
    unsigned long long t_last;  // globaltimer (ns) at the end of the previous solve step / at run start (iter_time_ms)
    double V_warm[2][9];        // [0] rotation block, [1] translation block, eigenvectors in columns
};

__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

// IterationLogData::iter_time_ms (icp_test_runner.cpp:1695 tic, :1973 toc): device time since the previous step ended
__device__ __forceinline__ double stamp_iteration(IcpState* st) {
    const unsigned long long now = globaltimer_ns();
    const double ms = (double)(now - st->t_last) * 1e-6;
    st->t_last = now;
    return ms;
}

// after the pose update: decide the next iteration's mode (see icp_iter2_kernel)
__device__ __forceinline__ void note_step(IcpState* st, const double* dx, double lever, double max_step) {
    const double dR = sqrt(dx[0] * dx[0] + dx[1] * dx[1] + dx[2] * dx[2]);
    const double dT = sqrt(dx[3] * dx[3] + dx[4] * dx[4] + dx[5] * dx[5]);
    st->step_rot = dR; st->step_trans = dT;
    st->seeds = st->coherent;                                   // records exist iff the iteration just done was coherent
    st->coherent = (dR * lever + dT) < max_step ? 1 : 0;         // largest displacement of any source point
}

__device__ inline void unpack_H(const double* v27, double* H, double* g) {
    int k = 0;
    for (int i = 0; i < 6; ++i)
        for (int j = i; j < 6; ++j) { H[i * 6 + j] = v27[k]; H[j * 6 + i] = v27[k]; ++k; }
    for (int i = 0; i < 6; ++i) g[i] = v27[21 + i];
}

__device__ inline double cond3(const double* lam) {   // lambda ascending
    return lam[2] / fmax(lam[0], 1e-12);               // icp_test_runner.cpp:2454-2457
}

// paper Alg. 2 (log only): greedy assignment of eigenvectors to the reference axes, sign fix,
// Gram-Schmidt in slot order.  indices[j] = column of V_raw that landed in slot j.
__device__ __noinline__ void align_axes(const double* V, double* Va, int* indices) {
    bool used_v[3] = {false, false, false}, used_e[3] = {false, false, false};
    for (int round = 0; round < 3; ++round) {
        double best = -1.0; int bi = 0, bj = 0;
        for (int j = 0; j < 3; ++j) {
            if (used_e[j]) continue;
            for (int i = 0; i < 3; ++i) {
                if (used_v[i]) continue;
                const double a = fabs(V[j * 3 + i]);     // |v_i . e_j| = |V[j][i]|
                if (a > best) { best = a; bi = i; bj = j; }
            }
        }
        used_v[bi] = true; used_e[bj] = true; indices[bj] = bi;
    }
    for (int j = 0; j < 3; ++j) {
        double v[3] = {V[0 * 3 + indices[j]], V[1 * 3 + indices[j]], V[2 * 3 + indices[j]]};
        if (v[j] < 0.0) { v[0] = -v[0]; v[1] = -v[1]; v[2] = -v[2]; }
        for (int k = 0; k < j; ++k) {
            const double d = v[0] * Va[0 * 3 + k] + v[1] * Va[1 * 3 + k] + v[2] * Va[2 * 3 + k];
            v[0] -= d * Va[0 * 3 + k]; v[1] -= d * Va[1 * 3 + k]; v[2] -= d * Va[2 * 3 + k];
        }
        const double nrm = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
        const double inv = nrm > 0.0 ? 1.0 / nrm : 0.0;
        Va[0 * 3 + j] = v[0] * inv; Va[1 * 3 + j] = v[1] * inv; Va[2 * 3 + j] = v[2] * inv;
    }
}

// PCG on H x = g, x0 = 0 (paper Alg. 3; stub DCReg::solvePCG dcreg.hpp:279-287).
// Stops when ||r||_2 < tol or after max_iter iterations.  Returns iterations used.
__device__ __noinline__ int pcg6(const double* H, const double* g, const double* P, int max_iter,
                           double tol, double* x, double* res_out) {
    double r[6], z[6], p[6], Hp[6];
    for (int i = 0; i < 6; ++i) { x[i] = 0.0; r[i] = g[i]; }
    dla::mat6_vec(P, r, z);
    double rz = 0.0;
    for (int i = 0; i < 6; ++i) { p[i] = z[i]; rz += r[i] * z[i]; }
    int it = 0;
    double rn = 0.0;
    for (int i = 0; i < 6; ++i) rn += r[i] * r[i];
    rn = sqrt(rn);
    for (it = 1; it <= max_iter; ++it) {
        dla::mat6_vec(H, p, Hp);
        double pHp = 0.0;
        for (int i = 0; i < 6; ++i) pHp += p[i] * Hp[i];
        const double alpha = rz / pHp;
        rn = 0.0;
        for (int i = 0; i < 6; ++i) { x[i] += alpha * p[i]; r[i] -= alpha * Hp[i]; rn += r[i] * r[i]; }
        rn = sqrt(rn);
        if (rn < tol) break;
        dla::mat6_vec(P, r, z);
        double rz_new = 0.0;
        for (int i = 0; i < 6; ++i) rz_new += r[i] * z[i];
        const double beta = rz_new / rz;
        for (int i = 0; i < 6; ++i) p[i] = z[i] + beta * p[i];
        rz = rz_new;
    }
    if (it > max_iter) it = max_iter;
    *res_out = rn;
    return it;
}

__device__ __noinline__ void qr6(const double* H, const double* g, double* x) {
    double A[36], b[6];
    for (int i = 0; i < 36; ++i) A[i] = H[i];
    for (int i = 0; i < 6; ++i) b[i] = g[i];
    dla::colpiv_qr_solve<6, 6>(A, b, x);
}

// analysis + solve for one 6x6 system.  Single thread.
// kFull = true : everything DegeneracyAnalysisResult holds (the host-callable seam, and the post-run log fill).
// kFull = false: only what the chosen (detection, handling) pair needs to produce dx - the per-iteration critical
//                path of the loop; the log-only quantities (full EVD/SVD, diagonal blocks, alignment report, and the
//                Schur blocks when the method does not use them) are filled after the run, one thread per iteration.
template <bool kFull>
__device__ inline void analyze_and_solve(const double* v27, const dcreg_icp_params& prm,
                                         dcreg_analysis* a, double* dx) {
    double H[36], g[6];
    unpack_H(v27, H, g);
    const double NaN = nan("");
    const bool need_evd6 = kFull || prm.detection == DCREG_DET_FULL_EVD_MIN_EIGENVALUE ||
                           prm.detection == DCREG_DET_FULL_SVD_CONDITION ||
                           prm.handling == DCREG_HAND_SOLUTION_REMAPPING || prm.handling == DCREG_HAND_TRUNCATED_SVD;
    const bool need_schur = kFull || prm.detection == DCREG_DET_SCHUR_CONDITION_NUMBER;

    // ---- defaults of DegeneracyAnalysisResult (utils.hpp:427-448) ----
    a->is_degenerate = 0; a->pcg_iterations = 0; a->pcg_residual = 0.0;
    for (int i = 0; i < 6; ++i) a->degenerate_mask[i] = 0;
    for (int i = 0; i < 36; ++i) a->P_preconditioner[i] = (i % 7 == 0) ? 1.0 : 0.0;
    for (int i = 0; i < 9; ++i) {
        const double e = (i % 4 == 0) ? 1.0 : 0.0;
        a->aligned_V_rot[i] = a->aligned_V_trans[i] = a->schur_V_rot[i] = a->schur_V_trans[i] = e;
    }
    for (int i = 0; i < 3; ++i) { a->rot_indices[i] = a->trans_indices[i] = i; }
    a->schur_singular = 0; a->reserved1 = 0;
    for (int i = 0; i < 36; ++i) a->W_adaptive[i] = 0.0;                  // dcreg.hpp:52: reset, never written by a released handler

    // ---- full EVD / "SVD" of H (dcreg.hpp:62-89) ----
    double W[36], lam[6], V[36];
    if (need_evd6) {
        for (int i = 0; i < 36; ++i) W[i] = H[i];
        dla::jacobi_eigh<6>(W, lam, V);
    } else {
        for (int i = 0; i < 6; ++i) lam[i] = NaN;
    }
    for (int i = 0; i < 6; ++i) a->eigenvalues_full[i] = lam[i];
    a->cond_full_sub_trans = fabs(lam[2]) / fmax(fabs(lam[0]), 1e-12);
    a->cond_full_sub_rot = fabs(lam[5]) / fmax(fabs(lam[3]), 1e-12);
    // singular values of a symmetric matrix = |eigenvalues|, descending; order[] maps
    // singular index -> eigen index (needed by the TSVD handler)
    int order[6];
    for (int i = 0; i < 6; ++i) order[i] = i;
    for (int i = 0; i < 5; ++i) {
        int m = i;
        for (int j = i + 1; j < 6; ++j)
            if (fabs(lam[order[j]]) > fabs(lam[order[m]])) m = j;
        const int t = order[i]; order[i] = order[m]; order[m] = t;
    }
    for (int i = 0; i < 6; ++i) a->singular_values[i] = fabs(lam[order[i]]);
    a->cond_full = (a->singular_values[5] > 1e-12) ? a->singular_values[0] / a->singular_values[5]
                                                   : (double)INFINITY;
    if (!need_evd6) a->cond_full = NaN;

    // ---- diagonal blocks + Schur complements (icp_test_runner.cpp:2418-2469, paper Eq. 18) ----
    double HRR[9], Htt[9], HRt[9], HtR[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            HRR[i * 3 + j] = H[i * 6 + j];
            Htt[i * 3 + j] = H[(i + 3) * 6 + j + 3];
            HRt[i * 3 + j] = H[i * 6 + j + 3];
            HtR[i * 3 + j] = H[(i + 3) * 6 + j];
        }
    double tmpA[9], tmpV[9];
    if (kFull) {
        dla::jacobi_eigh3(HRR, a->lambda_sub_rot, tmpV);
        dla::jacobi_eigh3(Htt, a->lambda_sub_trans, tmpV);
        a->cond_diag_rot = cond3(a->lambda_sub_rot);
        a->cond_diag_trans = cond3(a->lambda_sub_trans);
    } else {
        for (int i = 0; i < 3; ++i) a->lambda_sub_rot[i] = a->lambda_sub_trans[i] = NaN;
        a->cond_diag_rot = a->cond_diag_trans = NaN;
    }

    double HttInv[9], HRRInv[9];
    bool schur_ok = false;
    if (need_schur) {
        for (int i = 0; i < 9; ++i) tmpA[i] = Htt[i];
        const bool ok_t = dla::fullpiv_inverse<3>(tmpA, HttInv);
        for (int i = 0; i < 9; ++i) tmpA[i] = HRR[i];
        const bool ok_r = dla::fullpiv_inverse<3>(tmpA, HRRInv);
        schur_ok = ok_t && ok_r;
    }
    if (!need_schur) {
        for (int i = 0; i < 3; ++i) a->lambda_schur_rot[i] = a->lambda_schur_trans[i] = NaN;
        a->cond_schur_rot = a->cond_schur_trans = NaN;
    } else if (schur_ok) {
        double T1[9], T2[9], SR[9], St[9];
        dla::mat3_mul(HRt, HttInv, T1); dla::mat3_mul(T1, HtR, T2);
        for (int i = 0; i < 9; ++i) SR[i] = HRR[i] - T2[i];
        dla::mat3_mul(HtR, HRRInv, T1); dla::mat3_mul(T1, HRt, T2);
        for (int i = 0; i < 9; ++i) St[i] = Htt[i] - T2[i];
        // SelfAdjointEigenSolver reads one triangle only; symmetrise so Jacobi sees the same matrix
        for (int i = 0; i < 3; ++i)
            for (int j = i + 1; j < 3; ++j) {
                const double m1 = 0.5 * (SR[i * 3 + j] + SR[j * 3 + i]); SR[i * 3 + j] = SR[j * 3 + i] = m1;
                const double m2 = 0.5 * (St[i * 3 + j] + St[j * 3 + i]); St[i * 3 + j] = St[j * 3 + i] = m2;
            }
        dla::jacobi_eigh3(SR, a->lambda_schur_rot, a->schur_V_rot);
        dla::jacobi_eigh3(St, a->lambda_schur_trans, a->schur_V_trans);
        a->cond_schur_rot = cond3(a->lambda_schur_rot);
        a->cond_schur_trans = cond3(a->lambda_schur_trans);
        if (kFull) {
            align_axes(a->schur_V_rot, a->aligned_V_rot, a->rot_indices);
            align_axes(a->schur_V_trans, a->aligned_V_trans, a->trans_indices);
        }
    } else {
        for (int i = 0; i < 3; ++i) a->lambda_schur_rot[i] = a->lambda_schur_trans[i] = NaN;
        a->cond_schur_rot = a->cond_schur_trans = (double)INFINITY;
        a->schur_singular = 1;                               // icp_test_runner.cpp:2464 (a warning there)
    }

    // ---- detection (dcreg.hpp:94-162 + paper Eq. 20-21 for the Schur case) ----
    switch (prm.detection) {
        case DCREG_DET_SCHUR_CONDITION_NUMBER:
            if (schur_ok) {
                for (int blk = 0; blk < 2; ++blk) {
                    const double* l = blk ? a->lambda_schur_trans : a->lambda_schur_rot;
                    const double* Vb = blk ? a->schur_V_trans : a->schur_V_rot;
                    double lt[3];
                    for (int i = 0; i < 3; ++i) {
                        if (l[2] / fmax(l[i], 1e-12) > prm.cond_thresh) {
                            a->degenerate_mask[blk * 3 + i] = 1; a->is_degenerate = 1;
                        }
                        lt[i] = fmax(l[i], l[2] / prm.kappa_target);     // Eq. 46
                    }
                    for (int i = 0; i < 3; ++i)
                        for (int j = 0; j < 3; ++j) {
                            double s = 0.0;
                            for (int k = 0; k < 3; ++k) s += Vb[i * 3 + k] * Vb[j * 3 + k] / lt[k];
                            a->P_preconditioner[(blk * 3 + i) * 6 + blk * 3 + j] = s;   // Eq. 43-44
                        }
                }
            }
            break;
        case DCREG_DET_FULL_EVD_MIN_EIGENVALUE:
            for (int i = 0; i < 6; ++i)
                if (lam[i] < prm.eig_thresh) { a->is_degenerate = 1; a->degenerate_mask[i] = 1; }
            break;
        case DCREG_DET_EVD_SUB_CONDITION:
            // dcreg.hpp:112-126 tests cond_diag_* which the released analyzeDegeneracy leaves NaN:
            // the comparison is always false.  Kept as released.
            break;
        case DCREG_DET_FULL_SVD_CONDITION:
            a->is_degenerate = (a->cond_full > prm.cond_thresh) ? 1 : 0;
            if (a->is_degenerate) {
                const double mx = lam[5];
                for (int i = 0; i < 6; ++i)
                    if (mx / lam[i] > prm.cond_thresh) a->degenerate_mask[i] = 1;
            }
            break;
        default: break;
    }

    // ---- handling (dcreg.hpp:168-264) ----
    switch (prm.handling) {
        case DCREG_HAND_STANDARD_REGULARIZATION: {
            double Hr[36];
            for (int i = 0; i < 36; ++i) Hr[i] = H[i];
            if (a->is_degenerate) for (int i = 0; i < 6; ++i) Hr[i * 7] += prm.std_reg_gamma;
            qr6(Hr, g, dx);
            break;
        }
        case DCREG_HAND_PRECONDITIONED_CG:
            if (a->is_degenerate) {
                a->pcg_iterations = pcg6(H, g, a->P_preconditioner, prm.pcg_max_iter, prm.pcg_tol, dx,
                                         &a->pcg_residual);
            } else {
                qr6(H, g, dx);
            }
            break;
        case DCREG_HAND_SOLUTION_REMAPPING: {
            double x0[6];
            qr6(H, g, x0);
            if (a->is_degenerate) {
                int good = 0;
                for (int i = 0; i < 6; ++i) dx[i] = 0.0;
                for (int k = 0; k < 6; ++k) {
                    if (a->degenerate_mask[k]) continue;
                    ++good;
                    double d = 0.0;
                    for (int i = 0; i < 6; ++i) d += V[i * 6 + k] * x0[i];
                    for (int i = 0; i < 6; ++i) dx[i] += V[i * 6 + k] * d;
                }
                if (good == 0) for (int i = 0; i < 6; ++i) dx[i] = 0.0;
            } else {
                for (int i = 0; i < 6; ++i) dx[i] = x0[i];
            }
            break;
        }
        case DCREG_HAND_TRUNCATED_SVD: {
            // mask[i] (ascending-eigenvalue index) is paired with sigma_i (descending) exactly as
            // the reference does (dcreg.hpp:232-237) - a quirk of the baseline, kept.
            int kept = 0;
            for (int i = 0; i < 6; ++i) dx[i] = 0.0;
            for (int i = 0; i < 6; ++i) {
                const double sig = a->singular_values[i];
                if (!a->degenerate_mask[i] && sig > 1e-9) {
                    ++kept;
                    const int e = order[i];
                    double d = 0.0;
                    for (int r = 0; r < 6; ++r) d += V[r * 6 + e] * g[r];
                    const double sc = (lam[e] >= 0.0 ? 1.0 : -1.0) * d / sig;
                    for (int r = 0; r < 6; ++r) dx[r] += V[r * 6 + e] * sc;
                }
            }
            if (kept == 0) for (int i = 0; i < 6; ++i) dx[i] = 0.0;
            break;
        }
        default:
            qr6(H, g, dx);
            break;
    }
}

// R <- R exp(w), t <- t + R_old v  (math_utils.hpp:158-166, 20-33)
__device__ __noinline__ void boxplus(double* R, double* t, const double* dx) {
    const double wx = dx[0], wy = dx[1], wz = dx[2];
    const double theta = sqrt(wx * wx + wy * wy + wz * wz);
    double E[9];
    if (theta < 1e-10) {
        E[0] = 1.0; E[1] = -wz; E[2] = wy;
        E[3] = wz;  E[4] = 1.0; E[5] = -wx;
        E[6] = -wy; E[7] = wx;  E[8] = 1.0;
    } else {
        const double ax = wx / theta, ay = wy / theta, az = wz / theta;
        const double K[9] = {0.0, -az, ay, az, 0.0, -ax, -ay, ax, 0.0};
        double K2[9];
        dla::mat3_mul(K, K, K2);
        double s, c;
        sincos(theta, &s, &c);
        const double c1 = 1.0 - c;
        for (int i = 0; i < 9; ++i) E[i] = ((i % 4 == 0) ? 1.0 : 0.0) + s * K[i] + c1 * K2[i];
    }
    double Rn[9];
    dla::mat3_mul(R, E, Rn);
    const double v0 = dx[3], v1 = dx[4], v2 = dx[5];
    t[0] += R[0] * v0 + R[1] * v1 + R[2] * v2;
    t[1] += R[3] * v0 + R[4] * v1 + R[5] * v2;
    t[2] += R[6] * v0 + R[7] * v1 + R[8] * v2;
    for (int i = 0; i < 9; ++i) R[i] = Rn[i];
}

// One full K2 step on the reduced accumulators: abort rules, analysis, solve, pose update,
// convergence flag and log record.  Single thread.
__device__ inline void icp_step(const double* acc, IcpState* st, const dcreg_icp_params& prm,
                                dcreg_iter_log* log, int log_cap, double lever, double max_step) {
    const int iter = st->iter;
    dcreg_iter_log* rec = (log != nullptr && iter < log_cap) ? &log[iter] : nullptr;
    dcreg_analysis scratch;
    dcreg_analysis* an = rec ? &rec->analysis : &scratch;
    const int n_eff = (int)(acc[kAccNeff] + 0.5);
    const int n_pt = (int)(acc[kAccNpt] + 0.5);
    if (rec) {
        rec->iter = iter; rec->n_effective = n_eff; rec->n_corr_pt = n_pt; rec->status = DCREG_OK;
        for (int i = 0; i < 27; ++i) rec->H27[i] = acc[i];
    }
    if (n_eff < prm.min_effective_points) {                 // icp_test_runner.cpp:1847-1854
        st->iter = iter + 1; st->done = 1; st->converged = 0; st->status = DCREG_NOT_ENOUGH_POINTS;
        const double ms = stamp_iteration(st);
        if (rec) {
            rec->status = DCREG_NOT_ENOUGH_POINTS; rec->rmse = 0.0; rec->fitness = 0.0; rec->objective = 0.0;
            rec->iter_time_ms = ms;
            for (int i = 0; i < 6; ++i) { rec->gradient[i] = 0.0; rec->dx[i] = 0.0; }
            for (int r = 0; r < 3; ++r) {
                for (int c = 0; c < 3; ++c) rec->T[r * 4 + c] = st->R[r * 3 + c];
                rec->T[r * 4 + 3] = st->t[r];
            }
            rec->T[12] = rec->T[13] = rec->T[14] = 0.0; rec->T[15] = 1.0;
        }
        return;
    }
    double dx[6];
    analyze_and_solve<false>(acc, prm, an, dx);
    bool finite = true;
    for (int i = 0; i < 6; ++i) finite = finite && isfinite(dx[i]);
    const double fitness = st->n_source_total > 0 ? (double)n_pt / (double)st->n_source_total : 0.0;
    const double rmse = sqrt(acc[kAccSumR2] / (double)n_eff);
    if (rec) {
        rec->rmse = rmse; rec->fitness = fitness;
        for (int i = 0; i < 6; ++i) rec->gradient[i] = -acc[21 + i];
    }
    if (!finite) {                                          // icp_test_runner.cpp:1942-1950
        st->done = 1; st->converged = 0; st->status = DCREG_NONFINITE_UPDATE;
        const double ms = stamp_iteration(st);
        if (rec) {
            rec->status = DCREG_NONFINITE_UPDATE; rec->objective = 0.5 * acc[kAccSumB2]; rec->iter_time_ms = ms;
            for (int i = 0; i < 6; ++i) rec->dx[i] = 0.0;
            for (int r = 0; r < 3; ++r) {
                for (int c = 0; c < 3; ++c) rec->T[r * 4 + c] = st->R[r * 3 + c];
                rec->T[r * 4 + 3] = st->t[r];
            }
            rec->T[12] = rec->T[13] = rec->T[14] = 0.0; rec->T[15] = 1.0;
        }
        return;
    }
    boxplus(st->R, st->t, dx);                              // icp_test_runner.cpp:1953
    note_step(st, dx, lever, max_step);
    {
        double gtmp[6];
        unpack_H(acc, st->H_last, gtmp);                    // matAtA_last, icp_test_runner.cpp:1965
    }
    if (rec) {
        rec->objective = 0.5 * acc[kAccSumB2];              // icp_test_runner.cpp:1919
        for (int i = 0; i < 6; ++i) rec->dx[i] = dx[i];
        for (int r = 0; r < 3; ++r) {
            for (int c = 0; c < 3; ++c) rec->T[r * 4 + c] = st->R[r * 3 + c];
            rec->T[r * 4 + 3] = st->t[r];
        }
        rec->T[12] = rec->T[13] = rec->T[14] = 0.0; rec->T[15] = 1.0;
    }
    const double dR = sqrt(dx[0] * dx[0] + dx[1] * dx[1] + dx[2] * dx[2]);
    const double dT = sqrt(dx[3] * dx[3] + dx[4] * dx[4] + dx[5] * dx[5]);
    st->iter = iter + 1;
    if (!prm.fixed_iterations && dR < prm.conv_thresh_rot && dT < prm.conv_thresh_trans) {
        st->converged = 1; st->done = 1;                    // icp_test_runner.cpp:1998-2002
    } else if (st->iter >= prm.max_iterations) {
        st->done = 1;
    }
    const double ms = stamp_iteration(st);                  // icp_test_runner.cpp:1973
    if (rec) rec->iter_time_ms = ms;
}

// ------------------------------------------------------------------------------------------------------------------
// Warp-cooperative K2 step for the "Ours" method (SCHUR_CONDITION_NUMBER + PRECONDITIONED_CG), the per-iteration
// critical path of the loop.  Why: executed by a single thread the step is ~7 k dependent FP64 instructions, each
// waiting for the previous one, and the straight-line code is fetched cold on every launch.  Here the 32 lanes share the work: the two 3x3 inverses and
// the two 3x3 Jacobi EVDs run on lanes 0/1 side by side, Schur products and the preconditioner are one entry per
// lane, and the PCG mat-vecs are row-per-lane with shuffle broadcasts and butterfly dot products.  Its arithmetic is
// not the seam's (MUFU-seeded reciprocals, warm Jacobi, L D L^T pivots, FMAs, the squared stop rule), so a decision
// whose margin is within rounding can go the other way here.  The in-loop record therefore gets, besides the
// non-analysis fields, the decisions of the step that moved the pose: is_degenerate, degenerate_mask, schur_singular,
// pcg_iterations and pcg_residual.  log_fill_kernel keeps those and fills the rest of the analysis block (eigenvalues,
// eigenvectors, P, conditions) from the record's H27 with the host seam's single-thread code.
// ------------------------------------------------------------------------------------------------------------------
struct WarpSmem {
    double H[36], g[6];
    double inv[2][9];        // [0] = H_tt^-1, [1] = H_RR^-1
    double S[2][9];          // [0] = S_R, [1] = S_t
    double lam[2][3], V[2][9];
    double P[36];
    double dx[6];
    double Rt[12];           // pose copy: boxplus works on shared memory, lanes write it back in parallel
    double ilam[2][3];       // 1 / clamped Schur eigenvalues (preconditioner)
    double Vw[2][9];         // warm-start bases (previous iteration's Schur eigenvectors), fetched with the first loads
    int ok[2];
};

// The PCG runs on lanes 0..7 only (components live in lanes 0..5): 3 shuffle rounds per dot product instead of 5.
constexpr unsigned kPcgMask = 0xffu;
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int off = 4; off > 0; off >>= 1) v += __shfl_xor_sync(kPcgMask, v, off);
    return v;
}
__device__ __forceinline__ double row_dot_bcast(const double (&row)[6], double v) {   // sum_j row[j] * v(lane j)
    double s = 0.0;
#pragma unroll
    for (int j = 0; j < 6; ++j) s = fma(row[j], __shfl_sync(kPcgMask, v, j), s);
    return s;
}

// PCG on H x = g (paper Alg. 3): lanes 0..5 own rows/components, lanes 0..7 execute.  Returns iterations used;
// rn2_out = ||r||^2 at exit.
__device__ __forceinline__ int pcg6_warp(const WarpSmem& sm, int lane, int max_iter, double tol, double& x_out,
                                         double& rn2_out) {
    double Hrow[6], Prow[6];
#pragma unroll
    for (int j = 0; j < 6; ++j) { Hrow[j] = lane < 6 ? sm.H[lane * 6 + j] : 0.0; Prow[j] = lane < 6 ? sm.P[lane * 6 + j] : 0.0; }
    double x = 0.0, r = lane < 6 ? sm.g[lane] : 0.0;
    double z = row_dot_bcast(Prow, r);
    double p = z;
    double rz = warp_sum(r * z);
    int it;
    // ||r|| < tol  <=>  ||r||^2 < tol^2: no square root on the chain.  Exact only while tol^2 is a normal number: below
    // tol ~1.5e-154 the square rounds (to 0 under ~1e-162) and the two rules part; the documented tolerances are far above.
    const double tol2 = tol * tol;
    double rn2 = max_iter < 1 ? warp_sum(r * r) : 0.0;
    for (it = 1; it <= max_iter; ++it) {
        const double Hp = row_dot_bcast(Hrow, p);
        const double alpha = k2f::fast_div(rz, warp_sum(p * Hp));
        x = fma(alpha, p, x);
        r = fma(-alpha, Hp, r);
        rn2 = warp_sum(r * r);
        if (rn2 < tol2) break;                               // identical in every lane: uniform branch
        z = row_dot_bcast(Prow, r);
        const double rz_new = warp_sum(r * z);
        p = fma(k2f::fast_div(rz_new, rz), p, z);
        rz = rz_new;
    }
    x_out = x;
    rn2_out = rn2;
    return it > max_iter ? max_iter : it;
}

// One K2 step by one warp.  Same observable behaviour as icp_step for the "Ours" method.
// dbg (profiling only, may be null): globaltimer stamps [0] entry, [1] after the block inverses, [2] after the Schur
// eigen-decompositions, [3] after the preconditioner, [4] after the solve, [5] after the pose update.
#define K2_STAMP(k) do { if (dbg && lane == 0) dbg[k] = globaltimer_ns(); } while (0)
__device__ inline void icp_step_warp_ours(const double* acc, IcpState* st, const dcreg_icp_params& prm,
                                          dcreg_iter_log* log, int log_cap, WarpSmem& sm, double lever, double max_step,
                                          unsigned long long* dbg = nullptr) {
    const int lane = threadIdx.x & 31;
    K2_STAMP(0);
    // loop state (global memory): requested first, consumed only after the block inverses, which need nothing but the sums
    const int iter = st->iter;
    const int warm_flag = st->warm;
    double pre = 0.0;                                        // lanes 0..17: warm-start bases, lanes 18..29: pose
    if (lane < 18) pre = st->V_warm[lane / 9][lane % 9];
    else if (lane < 30) pre = lane < 27 ? st->R[lane - 18] : st->t[lane - 27];
    const int n_eff = (int)(acc[kAccNeff] + 0.5);
    const int n_pt = (int)(acc[kAccNpt] + 0.5);
    for (int e = lane; e < 36; e += 32) {
        const int i = e / 6, j = e % 6, a = i < j ? i : j, b = i < j ? j : i;
        sm.H[e] = acc[a * 6 - (a * (a - 1)) / 2 + (b - a)];
    }
    if (lane < 6) sm.g[lane] = acc[21 + lane];
    __syncwarp();
    // ---- block inverses (FullPivLU semantics), lanes 0 / 1 ----
    if (lane < 2 && n_eff >= prm.min_effective_points) {
        double M[9];
        const int o = lane == 0 ? 3 : 0;                     // lane 0: H_tt, lane 1: H_RR
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) M[i * 3 + j] = sm.H[(i + o) * 6 + j + o];
        sm.ok[lane] = k2f::spd_inverse3(M, sm.inv[lane]) ? 1 : 0;   // FullPivLU::isInvertible + inverse (k2_fast.cuh)
    }
    // now the state: pose, warm start of the two Jacobi iterations (k2_fast.cuh; a cold start every 64 iterations bounds
    // the drift of the accumulated rotations in 5000-iteration runs, icp_iter.yaml), log record
    dcreg_iter_log* rec = (log != nullptr && iter < log_cap) ? &log[iter] : nullptr;
    {
        const bool warm = warm_flag != 0 && (iter & 63) != 0;
        if (lane < 18) sm.Vw[lane / 9][lane % 9] = warm ? pre : ((lane % 9) % 4 == 0 ? 1.0 : 0.0);
        else if (lane < 30) sm.Rt[lane - 18] = pre;
    }
    if (rec) {
        if (lane < 27) rec->H27[lane] = acc[lane];
        if (lane == 0) { rec->iter = iter; rec->n_effective = n_eff; rec->n_corr_pt = n_pt; rec->status = DCREG_OK; }
    }
    __syncwarp();
    if (n_eff < prm.min_effective_points) {                 // icp_test_runner.cpp:1847-1854 (uniform branch)
        if (lane == 0) {
            st->iter = iter + 1; st->done = 1; st->converged = 0; st->status = DCREG_NOT_ENOUGH_POINTS;
            const double ms = stamp_iteration(st);
            if (rec) {
                rec->status = DCREG_NOT_ENOUGH_POINTS; rec->rmse = 0.0; rec->fitness = 0.0; rec->objective = 0.0;
                rec->iter_time_ms = ms;
                for (int i = 0; i < 6; ++i) { rec->gradient[i] = 0.0; rec->dx[i] = 0.0; }
                for (int r = 0; r < 3; ++r) {
                    for (int c = 0; c < 3; ++c) rec->T[r * 4 + c] = st->R[r * 3 + c];
                    rec->T[r * 4 + 3] = st->t[r];
                }
                rec->T[12] = rec->T[13] = rec->T[14] = 0.0; rec->T[15] = 1.0;
            }
        }
        return;
    }
    __syncwarp();
    K2_STAMP(1);
    const bool schur_ok = sm.ok[0] && sm.ok[1];
    int degenerate = 0;
    bool deg = false;                                        // lanes 0..5: this eigenvalue's flag of the mask
    if (schur_ok) {
        // ---- Schur complements (icp_test_runner.cpp:2443-2447, paper Eq. 18): one entry per lane ----
        double sval = 0.0;
        if (lane < 18) {
            const int blk = lane / 9, e = lane % 9, i = e / 3, j = e % 3;
            // blk 0: S_R = H_RR - (H_Rt Htt^-1) H_tR ; blk 1: S_t = H_tt - (H_tR HRR^-1) H_Rt
            const int ro = blk == 0 ? 0 : 3, co = blk == 0 ? 3 : 0;
            const double* Inv = sm.inv[blk];
            double t2 = 0.0;
#pragma unroll
            for (int m = 0; m < 3; ++m) {
                double t1 = 0.0;
#pragma unroll
                for (int k = 0; k < 3; ++k) t1 += sm.H[(ro + i) * 6 + co + k] * Inv[k * 3 + m];
                t2 += t1 * sm.H[(co + m) * 6 + ro + j];
            }
            sval = sm.H[(ro + i) * 6 + ro + j] - t2;
            sm.S[blk][e] = sval;
        }
        __syncwarp();
        if (lane < 18) {
            const int blk = lane / 9, e = lane % 9, i = e / 3, j = e % 3;
            sval = 0.5 * (sval + sm.S[blk][j * 3 + i]);
        }
        __syncwarp();
        if (lane < 18) sm.S[lane / 9][lane % 9] = sval;
        __syncwarp();
        if (lane < 2) {
            double Vw[9], Vn[9], ln[3], Sl[9];
#pragma unroll
            for (int e = 0; e < 9; ++e) { Sl[e] = sm.S[lane][e]; Vw[e] = sm.Vw[lane][e]; }
            k2f::jacobi_eigh3_warm(Sl, Vw, ln, Vn);
#pragma unroll
            for (int e = 0; e < 9; ++e) { sm.V[lane][e] = Vn[e]; st->V_warm[lane][e] = Vn[e]; }
#pragma unroll
            for (int e = 0; e < 3; ++e) sm.lam[lane][e] = ln[e];
            if (lane == 0) st->warm = 1;
        }
        __syncwarp();
        K2_STAMP(2);
        // ---- detection (Eq. 20-21) and preconditioner (Eq. 43-46) ----
        if (lane < 6) {
            const double* l = sm.lam[lane / 3];
            deg = l[2] / fmax(l[lane % 3], 1e-12) > prm.cond_thresh;
        }
        degenerate = __ballot_sync(0xffffffffu, deg) != 0u;
        if (lane < 6) {
            const double* l = sm.lam[lane / 3];
            sm.ilam[lane / 3][lane % 3] = k2f::fast_rcp(fmax(l[lane % 3], l[2] * k2f::fast_rcp(prm.kappa_target)));
        }
        __syncwarp();
        for (int e = lane; e < 36; e += 32) {
            const int i = e / 6, j = e % 6;
            double v = 0.0;
            if (i / 3 == j / 3) {
                const int blk = i / 3;
                const double* il = sm.ilam[blk];
                const double* Vb = sm.V[blk];
#pragma unroll
                for (int k = 0; k < 3; ++k) v = fma(Vb[(i % 3) * 3 + k] * Vb[(j % 3) * 3 + k], il[k], v);
            }
            sm.P[e] = v;
        }
        __syncwarp();
    }
    K2_STAMP(3);
    // ---- solve ----
    int pcg_it = 0;
    double pcg_rn2 = 0.0;
    if (degenerate) {
        if (lane < 8) {
            double xi;
            pcg_it = pcg6_warp(sm, lane, prm.pcg_max_iter, prm.pcg_tol, xi, pcg_rn2);
            if (lane < 6) sm.dx[lane] = xi;
        }
    } else if (lane == 0) {
        qr6(sm.H, sm.g, sm.dx);                              // dcreg.hpp:190
    }
    __syncwarp();
    K2_STAMP(4);
    if (rec) {                                               // the decisions this step took (log_fill_kernel keeps them)
        dcreg_analysis* an = &rec->analysis;
        if (lane < 6) an->degenerate_mask[lane] = deg ? 1 : 0;
        if (lane == 0) {
            an->is_degenerate = degenerate; an->schur_singular = schur_ok ? 0 : 1;
            an->pcg_iterations = pcg_it; an->pcg_residual = degenerate ? sqrt(pcg_rn2) : 0.0;
        }
    }
    const double dxi = lane < 6 ? sm.dx[lane] : 0.0;
    const bool finite = __ballot_sync(0xffffffffu, !isfinite(dxi)) == 0u;
    if (rec) {                                               // log only: off the pose's dependent chain
        if (lane == 0) {
            rec->rmse = sqrt(acc[kAccSumR2] / (double)n_eff);
            rec->fitness = st->n_source_total > 0 ? (double)n_pt / (double)st->n_source_total : 0.0;
            rec->objective = 0.5 * acc[kAccSumB2];
        }
        if (lane < 6) rec->gradient[lane] = -acc[21 + lane];
    }
    if (!finite) {                                          // icp_test_runner.cpp:1942-1950
        if (lane == 0) {
            st->done = 1; st->converged = 0; st->status = DCREG_NONFINITE_UPDATE;
            const double ms = stamp_iteration(st);
            if (rec) { rec->status = DCREG_NONFINITE_UPDATE; rec->iter_time_ms = ms; }
        }
        if (rec) {
            if (lane < 6) rec->dx[lane] = 0.0;
            if (lane < 16) {
                const int r = lane / 4, c = lane % 4;
                rec->T[lane] = r == 3 ? (c == 3 ? 1.0 : 0.0) : (c == 3 ? sm.Rt[9 + r] : sm.Rt[r * 3 + c]);
            }
        }
        return;
    }
    for (int e = lane; e < 36; e += 32) st->H_last[e] = sm.H[e];     // matAtA_last, icp_test_runner.cpp:1965
    // ---- boxplus (math_utils.hpp:158-166, 20-33), spread over the lanes: R <- R exp(w), t <- t + R_old v.
    // exp(w) = c I + (1 - c) a a^T + s [a]x with a = w / theta (the same matrix as I + s K + (1 - c) K^2); lane 0 owns
    // the only long chain (theta, sincos), lanes 0..8 one entry of R exp(w) each, lanes 9..11 one entry of t.
    {
        const double wx = sm.dx[0], wy = sm.dx[1], wz = sm.dx[2];
        const double th2 = wx * wx + wy * wy + wz * wz;
        const double v2 = sm.dx[3] * sm.dx[3] + sm.dx[4] * sm.dx[4] + sm.dx[5] * sm.dx[5];
        const double theta = sqrt(th2), dT = sqrt(v2);       // every lane (same instructions, no exchange needed)
        double e_[9];                                        // exp(w), row-major
        if (theta < 1e-10) {
            e_[0] = 1.0; e_[1] = -wz; e_[2] = wy;
            e_[3] = wz;  e_[4] = 1.0; e_[5] = -wx;
            e_[6] = -wy; e_[7] = wx;  e_[8] = 1.0;
        } else {
            const double ax = wx / theta, ay = wy / theta, az = wz / theta;
            double sn, cs;
            sincos(theta, &sn, &cs);
            const double c1 = 1.0 - cs;
            // K = [a]x, K^2 = a a^T - I (|a| = 1): I + s K + c1 K^2, written entry by entry as the reference's formula
            const double K[9] = {0.0, -az, ay, az, 0.0, -ax, -ay, ax, 0.0};
            const double K2[9] = {-(ay * ay + az * az), ax * ay, ax * az, ax * ay, -(ax * ax + az * az), ay * az,
                                  ax * az, ay * az, -(ax * ax + ay * ay)};
#pragma unroll
            for (int i = 0; i < 9; ++i) e_[i] = ((i % 4 == 0) ? 1.0 : 0.0) + sn * K[i] + c1 * K2[i];
        }
        double outv = 0.0;
        if (lane < 9) {
            const int r = lane / 3, c = lane % 3;
            outv = sm.Rt[r * 3 + 0] * e_[0 * 3 + c] + sm.Rt[r * 3 + 1] * e_[1 * 3 + c] + sm.Rt[r * 3 + 2] * e_[2 * 3 + c];
        } else if (lane < 12) {
            const int r = lane - 9;
            outv = sm.Rt[9 + r] + (sm.Rt[r * 3 + 0] * sm.dx[3] + sm.Rt[r * 3 + 1] * sm.dx[4] + sm.Rt[r * 3 + 2] * sm.dx[5]);
        }
        __syncwarp();
        if (lane < 12) sm.Rt[lane] = outv;
        if (lane == 0) {
            st->step_rot = theta; st->step_trans = dT;
            st->seeds = st->coherent;                        // records exist iff the iteration just done was coherent
            st->coherent = (theta * lever + dT) < max_step ? 1 : 0;   // largest displacement of any source point (note_step)
            st->iter = iter + 1;
            if (!prm.fixed_iterations && theta < prm.conv_thresh_rot && dT < prm.conv_thresh_trans) {
                st->converged = 1; st->done = 1;             // icp_test_runner.cpp:1998-2002
            } else if (iter + 1 >= prm.max_iterations) {
                st->done = 1;
            }
            const double ms = stamp_iteration(st);           // icp_test_runner.cpp:1973
            if (rec) rec->iter_time_ms = ms;
        }
    }
    __syncwarp();
    K2_STAMP(5);
    if (lane < 9) st->R[lane] = sm.Rt[lane];
    else if (lane < 12) st->t[lane - 9] = sm.Rt[lane];
    if (rec) {
        if (lane < 6) rec->dx[lane] = sm.dx[lane];
        if (lane < 16) {
            const int r = lane / 4, c = lane % 4;
            rec->T[lane] = r == 3 ? (c == 3 ? 1.0 : 0.0) : (c == 3 ? sm.Rt[9 + r] : sm.Rt[r * 3 + c]);
        }
    }
}

}  // namespace k2
