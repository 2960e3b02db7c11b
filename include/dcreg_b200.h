/*
 * dcreg_b200.h - C ABI of the H100 (sm_90a) point-to-plane ICP + Schur-decoupled degeneracy engine.
 *
 * This is the drop-in boundary for ONE hot path of JokerJohn/DCReg (SURVEY.md §8b).  The
 * reference has no FFI layer; each entry point below names the C++ member / code block of the
 * reference it replaces (paths relative to the reference checkout).  Plain pointers and sizes
 * only: no torch, Eigen or PCL types cross this boundary.  Nothing here ever throws; every
 * function returns a dcreg_status and dcreg_last_error() holds the text.
 *
 * State-vector order everywhere: [wx wy wz | x y z] (rotation first, right perturbation),
 * as on the reference's SO(3) path (DCReg/src/icp_test_runner.cpp:1611-2060).
 * 4x4 / 3x3 / 6x6 matrices are ROW-major doubles.
 */
#ifndef DCREG_B200_H
#define DCREG_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DCREG_ABI_VERSION 2

/* -------------------------------------------------------------------------------------------
 * Status codes.  Reference convention: bool return + std::cerr text
 * (icp_test_runner.cpp:1635-1646, 1847-1854, 1942-1950; dcreg.hpp:259-262).
 * ----------------------------------------------------------------------------------------- */
typedef enum dcreg_status {
    DCREG_OK = 0,
    DCREG_NOT_ENOUGH_POINTS = 1,   /* < 10 effective correspondences (icp_test_runner.cpp:1847) */
    DCREG_NONFINITE_UPDATE = 2,    /* solver returned non-finite dx (icp_test_runner.cpp:1942)  */
    DCREG_SINGULAR_BLOCK = 3,      /* never RETURNED: the reference only warns when H_RR or H_tt is not invertible
                                      (icp_test_runner.cpp:2464) and carries on with cond = inf; the warning is
                                      surfaced per iteration as dcreg_analysis.schur_singular.  Value kept reserved. */
    DCREG_CUDA_ERROR = 4,
    DCREG_NCCL_ERROR = 5,
    DCREG_BAD_ARG = 6,
    DCREG_NO_DEVICE = 7            /* no CUDA device: the product has no CPU fallback            */
} dcreg_status;

/* DetectionMethod / HandlingMethod, DCReg/include/utils.hpp:106-121 (same order, same names). */
typedef enum dcreg_detection {
    DCREG_DET_NONE_DETE = 0,
    DCREG_DET_SCHUR_CONDITION_NUMBER = 1,
    DCREG_DET_FULL_EVD_MIN_EIGENVALUE = 2,
    DCREG_DET_EVD_SUB_CONDITION = 3,
    DCREG_DET_FULL_SVD_CONDITION = 4
} dcreg_detection;

typedef enum dcreg_handling {
    DCREG_HAND_NONE_HAND = 0,
    DCREG_HAND_STANDARD_REGULARIZATION = 1,
    DCREG_HAND_ADAPTIVE_REGULARIZATION = 2, /* parsed by the reference, no handler: plain QR */
    DCREG_HAND_PRECONDITIONED_CG = 3,
    DCREG_HAND_SOLUTION_REMAPPING = 4,
    DCREG_HAND_TRUNCATED_SVD = 5
} dcreg_handling;

/* Motion model of dcreg_icp_run_odometry: how frame k's prior follows from frame k-1's result. */
typedef enum dcreg_motion { DCREG_MOTION_INCREMENTS = 0, DCREG_MOTION_CONSTANT_VELOCITY = 1 } dcreg_motion;

/* -------------------------------------------------------------------------------------------
 * Parameters: POD mirror of ICPRunner::Config + ICPParameters
 * (DCReg/include/utils.hpp:82-103, 132-171), passed by pointer, no global state
 * (the reference re-sets them every iteration through DCReg::setConfig, dcreg.hpp:36-38).
 * dcreg_default_params() fills the reference defaults.
 * ----------------------------------------------------------------------------------------- */
typedef struct dcreg_icp_params {
    double search_radius;          /* icp.search_radius                       (1.0)   */
    int32_t max_iterations;        /* icp.max_iterations                      (30)    */
    int32_t detection;             /* dcreg_detection                                  */
    int32_t handling;              /* dcreg_handling                                   */
    int32_t use_weight_derivative; /* USE_WEIGHT_DERIVATIVE, icp_test_runner.cpp:1691 (0) */
    double conv_thresh_rot;        /* CONVERGENCE_THRESH_ROT                  (1e-5)  */
    double conv_thresh_trans;      /* CONVERGENCE_THRESH_TRANS                (1e-3)  */
    double cond_thresh;            /* DEGENERACY_THRES_COND                   (10)    */
    double eig_thresh;             /* DEGENERACY_THRES_EIG                    (120)   */
    double kappa_target;           /* KAPPA_TARGET                            (1)     */
    double pcg_tol;                /* PCG_TOLERANCE                           (1e-6)  */
    int32_t pcg_max_iter;          /* PCG_MAX_ITER                            (10)    */
    int32_t reserved0;
    double std_reg_gamma;          /* STD_REG_GAMMA                           (0.01)  */
    /* compile-time constants of the reference, exposed with the reference values */
    double plane_thickness;        /* 0.2   icp_test_runner.cpp:1772 */
    double weight_slope;           /* 0.9   icp_test_runner.cpp:1776: s = 1 - weight_slope |r|              */
    double weight_gate;            /* 0.1   icp_test_runner.cpp:1785: slot kept when s > weight_gate         */
    double min_normal_norm;        /* 1e-6  icp_test_runner.cpp:1750 */
    int32_t min_effective_points;  /* 10    icp_test_runner.cpp:1847 */
    int32_t fixed_iterations;      /* 1: ignore the convergence test and always run max_iterations
                                      (BASELINE config "50 ICP iterations"); default 0 */
} dcreg_icp_params;

/* POD mirror of DegeneracyAnalysisResult (DCReg/include/utils.hpp:427-448). */
typedef struct dcreg_analysis {
    int32_t is_degenerate;
    int32_t degenerate_mask[6];    /* eigen-index order (ascending lambda), NOT physical axes */
    int32_t pcg_iterations;        /* iterations the PCG solve used (0 when the direct solve ran) */
    double cond_schur_rot, cond_schur_trans;
    double cond_diag_rot, cond_diag_trans;
    double cond_full;
    double cond_full_sub_rot, cond_full_sub_trans;
    double eigenvalues_full[6];    /* ascending */
    double singular_values[6];     /* descending */
    double lambda_schur_rot[3], lambda_schur_trans[3];   /* ascending */
    double lambda_sub_rot[3], lambda_sub_trans[3];       /* diagonal blocks, ascending */
    double schur_V_rot[9], schur_V_trans[9];             /* eigenvectors in columns */
    double aligned_V_rot[9], aligned_V_trans[9];         /* paper Alg. 2 (log only) */
    int32_t rot_indices[3], trans_indices[3];
    int32_t schur_singular;        /* 1: H_tt or H_RR not invertible, Schur complements skipped (icp_test_runner.cpp:2464) */
    int32_t reserved1;
    double P_preconditioner[36];   /* paper Eq. 43-46; identity unless SCHUR detection */
    double W_adaptive[36];         /* utils.hpp:446; zero: no released handler writes it (dcreg.hpp:52) */
    double pcg_residual;           /* ||g - H dx||_2 at exit of the PCG solve */
} dcreg_analysis;

/* Per-iteration record: the numeric part of IterationLogData (DCReg/include/utils.hpp:174-249)
 * that pins the path (columns of iteration_details_with_dx.csv, SURVEY.md Appendix B.4). */
typedef struct dcreg_iter_log {
    int32_t iter;
    int32_t status;                /* dcreg_status of this iteration */
    int32_t n_effective;           /* corr_num / effective_points */
    int32_t n_corr_pt;             /* correspondence_pt_count (5th NN within radius) */
    double rmse, fitness, objective;
    double iter_time_ms;           /* IterationLogData::iter_time_ms (utils.hpp:174-249; tic at the top of the iteration,
                                      toc after the update, icp_test_runner.cpp:1695, 1973): device time between the
                                      end of the previous solve step (run start for iteration 0) and the end of this
                                      one, from the GPU's globaltimer */
    double gradient[6];            /* -A^T b */
    double H27[27];                /* 21 upper-tri of A^T A (row-major upper) + 6 rhs A^T b */
    double dx[6];
    double T[16];                  /* pose AFTER the update */
    dcreg_analysis analysis;
} dcreg_iter_log;

typedef struct dcreg_ctx dcreg_ctx;   /* opaque: owns device buffers, stream, (optional) NCCL comm */

/* ---- lifetime ---------------------------------------------------------------------------- */
int dcreg_abi_version(void);
/* Replaces: TestRunner ctor + ICPContext (icp_test_runner.cpp:10-17, utils.hpp:340-425). */
int dcreg_create(int device_id, dcreg_ctx** out);
int dcreg_destroy(dcreg_ctx* ctx);
const char* dcreg_last_error(const dcreg_ctx* ctx);
void dcreg_default_params(dcreg_icp_params* p);
/* cudaStream_t the context launches on (for CUDA-event timing by the caller). */
void* dcreg_stream(dcreg_ctx* ctx);

/* ---- clouds ------------------------------------------------------------------------------ */
/* Source (measure) cloud: n points, `stride` floats between points (3 for xyz, 4 for xyzi).
 * Copied to the device as float4.  Replaces the measure_cloud argument of
 * Point2PlaneICP_SO3_OpenMP (icp_test_runner.h:92-102). */
int dcreg_set_source(dcreg_ctx* ctx, const float* xyz, int64_t n, int stride);
/* Target cloud + its spatial index.  Replaces ICPContext::setTargetCloud's kd-tree build
 * (utils.hpp:393-424): a device dense grid with cell = `cell_size` (pass the search radius;
 * exact 5-NN-within-radius then only needs the 27 surrounding cells).  A map too large for a dense grid (a bounding box
 * of more than 2^27 cells: city-scale prior maps) gets a sparse row index instead: the points in the dense grid's order
 * (by cell z, y, x, then index) and an open-addressing table of the row starts the searches read, about 12 B per table
 * slot with at most 18 entries per occupied cell (2 slots per entry, rounded up to a power of two), instead of 12 B per
 * cell of the box.  On it dcreg_icp_run, _enqueue / _fetch (records and coherent mode as on a dense grid),
 * dcreg_icp_run_batch, _scans, _sequences, dcreg_find_planes and dcreg_time_iteration work as on a dense grid: for
 * sources whose query cells stay inside a dense grid's box, a target whose extra points lie outside every search returns
 * that grid's results bit for bit.  dcreg_point_to_point_metrics refuses it (DCREG_BAD_ARG).  A cell coordinate outside
 * +-2^19, or a sparse index that would need more than 2^32 table slots, gives DCREG_BAD_ARG. */
int dcreg_set_target(dcreg_ctx* ctx, const float* xyz, int64_t m, int stride, double cell_size);
/* Identical to dcreg_set_target (kept for compatibility; its error texts name dcreg_set_target_sparse). */
int dcreg_set_target_sparse(dcreg_ctx* ctx, const float* xyz, int64_t m, int stride, double cell_size);
/* Sparse row indexes for the grids the library builds itself: the local maps of dcreg_icp_run_odometry* and of the
 * odometry sessions, and the targets of dcreg_icp_run_pairs.  enable = 0 (the default): such a map or target whose
 * bounding box has more than 2^27 cells at cell_size, or a step's or call's grids with more than 2^30 cells in all, is
 * DCREG_BAD_ARG, as documented at those calls.  enable = 1: that step (every lane of it) or that call (every pair of
 * it) builds sparse row indexes instead (those of dcreg_set_target, one per map or target, in one set of buffers;
 * one more host sync), and returns what the dense grids would return on the same points: a search of a sparse index
 * gives the dense grid's results bit for bit.  A step or call that fits dense grids runs exactly as with enable = 0;
 * there is no other choice between the two.  Still DCREG_BAD_ARG with enable = 1: a cell coordinate outside +-2^19, a
 * map or target whose index would need more than 2^32 table slots, and, for dcreg_icp_run_pairs with metrics, a call
 * whose targets are sparse (after the poses are written, naming the pair).  An odometry session keeps the value it had
 * at dcreg_odometry_open*: changing it later does not change that session's pushes.  enable other than 0 or 1:
 * DCREG_BAD_ARG. */
int dcreg_set_sparse_maps(dcreg_ctx* ctx, int enable);
/* Per-lane solver settings: compare methods or sweep a threshold across the lanes of one batched call.  enable = 0 (the
 * default): every call takes one dcreg_icp_params.  enable = 1: the params argument of the batched calls points to one
 * dcreg_icp_params per lane: n_trials for dcreg_icp_run_batch, n_scans for _scans, n_pairs for _pairs, and n_seqs for
 * _sequences, every dcreg_icp_run_odometry* and dcreg_odometry_open, _open_map and _open_adaptive (every frame of
 * sequence s uses entry s).  Single-run calls (dcreg_icp_run, _enqueue, _host_planes, dcreg_find_planes,
 * dcreg_analyze_and_solve, dcreg_time_* and the timeline) read entry 0 only.
 *   Per lane: detection, handling, conv_thresh_rot, conv_thresh_trans, cond_thresh, eig_thresh, kappa_target, pcg_tol,
 *   pcg_max_iter, std_reg_gamma, min_effective_points (the fields only the solve step and the log read).
 *   Common: search_radius, max_iterations, fixed_iterations, use_weight_derivative, plane_thickness, weight_slope,
 *   weight_gate and min_normal_norm must equal entry 0's byte for byte; otherwise the call is DCREG_BAD_ARG before
 *   anything runs, and dcreg_last_error names the call, the first differing entry and the field.  reserved0 is ignored.
 * Lane b of a call returns byte for byte what the same call returns for lane b when every entry is a copy of entry b
 * (every output but iter_time_ms), and a call whose entries are all alike is the call with one params (same bytes, same
 * launches).  In one call the lanes running "Ours" (Schur detection + PCG) solve inside the iteration kernel and the
 * others in a second kernel after it.  An odometry session copies the entries at open and keeps the setting it had
 * then; changing the setting later does not change its pushes.  enable other than 0 or 1: DCREG_BAD_ARG. */
int dcreg_set_lane_params(dcreg_ctx* ctx, int enable);
/* Minimum point spacing of scan-to-map odometry's map filter (KISS-ICP's VoxelHashMap::AddPoints): with min_spacing > 0,
 * F_m(P) = dcreg_voxel_downsample_spaced(P, map_voxel, map_max_points, min_spacing) instead of dcreg_voxel_downsample_n,
 * for the window and the voxel map of every dcreg_icp_run_odometry_voxel, _voxel_n, _deskew, _map and _adaptive call and
 * of sessions.  KISS-ICP's value is map_voxel / sqrt(map_max_points).  It leaves the source filter F_s,
 * dcreg_icp_run_odometry and _sequences, and maps with map_voxel = 0 or map_max_points = 1 unchanged (same launches,
 * same bytes), and so does 0, the default.  A step keeps its launches and its one host sync.  An odometry session keeps
 * the value it had at dcreg_odometry_open*: changing it later does not change that session's pushes, and
 * dcreg_odometry_local_map returns the spaced map.  min_spacing NaN, negative or infinite: DCREG_BAD_ARG. */
int dcreg_set_map_spacing(dcreg_ctx* ctx, double min_spacing);

/* ---- seam 1: correspondence stage (icp_test_runner.cpp:1714-1813) -------------------------
 * For every source slot: q = fl32(R p + t), exact 5-NN in the target, 5th d^2 < radius^2,
 * 5x3 least-squares plane, normalisation, thickness gate.  Writes plane[i] = (nx,ny,nz,d) as
 * doubles (all-zero = no plane) into a device buffer owned by ctx and optionally copies it to
 * `planes_out` (host, 4*n doubles, may be NULL).  n_corr_pt = correspondence_pt_count. */
int dcreg_find_planes(dcreg_ctx* ctx, const double T[16], double search_radius,
                      double* planes_out, int64_t* n_corr_pt);

/* ---- seam 2: fused residual / weight / Jacobian / normal-equation reduction (K1) ----------
 * Replaces icp_test_runner.cpp:1774-1803 + 1863-1919 and the SymmetricHessianComputer functor
 * (hessian_computer.h:62-123): out27 = 21 upper-triangular entries of A^T A in the functor's
 * order followed by the 6 entries of A^T b (= -J^T r); stats = { sum r^2, N_eff, N_slots_with_plane }.
 * d_src / d_plane are DEVICE pointers to n float4 (x,y,z,-) and n float4 (nx,ny,nz,d); a slot
 * with an all-zero normal is skipped.  pose_Rt = R (9, row-major) then t (3). */
int dcreg_reduce_normal_equations(dcreg_ctx* ctx, const void* d_src, const void* d_plane,
                                  int64_t n, const double pose_Rt[12], int use_weight_derivative,
                                  double out27[27], double stats[3]);
/* Same with n double4 planes (48 B/slot): the precision the reference itself uses for the plane. */
int dcreg_reduce_normal_equations_f64plane(dcreg_ctx* ctx, const void* d_src, const void* d_plane,
                                           int64_t n, const double pose_Rt[12],
                                           int use_weight_derivative, double out27[27],
                                           double stats[3]);
/* Host-buffer convenience of the above (copies in, reduces, copies out). plane_is_f64: 0/1. */
int dcreg_reduce_normal_equations_host(dcreg_ctx* ctx, const float* src4, const void* plane4,
                                       int plane_is_f64, int64_t n, const double pose_Rt[12],
                                       int use_weight_derivative, double out27[27], double stats[3]);

/* ---- seam 3: degeneracy analysis + solve (K2) ---------------------------------------------
 * Replaces DCReg::analyzeDegeneracy (dcreg.hpp:45-166), DCReg::solveDegenerateSystem
 * (dcreg.hpp:168-264), the released Schur block (icp_test_runner.cpp:2418-2469) and the
 * stubbed alignAndOrthonormalize / solvePCG (dcreg.hpp:267-287; paper Alg. 1-3).
 * Runs on the device (single-warp kernel); H27 and outputs are HOST pointers. */
int dcreg_analyze_and_solve(dcreg_ctx* ctx, const double H27[27], const dcreg_icp_params* params,
                            dcreg_analysis* out, double dx[6]);
/* DCReg::solvePCG (dcreg.hpp:279-283): A (36, row-major), b (6), P (36) -> x (6). */
int dcreg_solve_pcg(dcreg_ctx* ctx, const double A[36], const double b[6], const double P[36],
                    int max_iterations, double tolerance, double x[6], int* iterations);

/* ---- the outer loop ------------------------------------------------------------------------
 * Replaces TestRunner::Point2PlaneICP_SO3_OpenMP (icp_test_runner.h:92-102,
 * icp_test_runner.cpp:1611-2060).  Uses the clouds set on ctx.  All iterations (correspondences,
 * reduction, analysis, solve, pose update, convergence test) run on the device with no host
 * round trip; the host reads the final pose and the per-iteration log afterwards.
 * log may be NULL (log_cap 0).  *converged mirrors the reference's bool return.
 * Returns DCREG_OK also when not converged; DCREG_NOT_ENOUGH_POINTS / DCREG_NONFINITE_UPDATE
 * when the reference would abort (T_out then holds the last pose, as in the reference). */
int dcreg_icp_run(dcreg_ctx* ctx, const dcreg_icp_params* params, const double T_init[16],
                  double T_out[16], dcreg_iter_log* log, int log_cap, int* n_iterations,
                  int* converged);
/* The same run split in two for callers that pipeline scans: dcreg_icp_enqueue puts the whole run (all max_iterations
 * loop bodies; iterations past convergence exit at once on the device) on the context's stream and returns without any
 * host synchronisation; dcreg_icp_fetch waits for the stream and returns the pose / iteration count / flags of the LAST
 * enqueued run with dcreg_icp_run's return value.  No per-iteration log on this path. */
int dcreg_icp_enqueue(dcreg_ctx* ctx, const dcreg_icp_params* params, const double T_init[16]);
int dcreg_icp_fetch(dcreg_ctx* ctx, double T_out[16], int* n_iterations, int* converged);
/* Many registrations of the SAME source against the SAME target from different initial poses, side by side in one
 * sequence of launches (trial = grid y-dimension; each trial owns its loop state, neighbour records and log slice, and
 * stops on its own convergence test).  Replaces the `num_runs` loop of TestRunner::runSingleTest
 * (icp_test_runner.cpp:331-345: `for run in 0..num_runs: runSingleTest`) and is what a perturbation Monte-Carlo
 * (BASELINE.json configs[4]) calls.  T_init / T_out: n_trials row-major 4x4 matrices; n_iterations / converged / status:
 * n_trials ints (status[t] = what dcreg_icp_run would have returned for trial t; any may be NULL except T_init, T_out);
 * log: n_trials x log_cap records (trial-major) or NULL.  Every trial runs the kernels a dcreg_icp_run from the same
 * T_init runs (at most 65535 trials: the grid's y-dimension): counts, masks and iteration counts are identical, poses
 * equal up to the order of the FP64 sums (the source is sorted by target cell once, under trial 0's pose, and a single
 * run of a small cloud uses smaller tiles; 1e-8 on the poses in the tests; a batch itself is reproducible bit for
 * bit).  Not
 * available on a sharded context: trials are independent, distribute them over ranks instead. */
int dcreg_icp_run_batch(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_trials, const double* T_init,
                        double* T_out, int* n_iterations, int* converged, int* status, dcreg_iter_log* log,
                        int log_cap);
/* Many DIFFERENT source scans (e.g. the LiDAR frames of a sequence) against the context's target, side by side in one
 * sequence of launches, with one set of parameters.  xyz: HOST memory, all scans concatenated, `stride` floats per
 * point as in dcreg_set_source; scan b is points [scan_offsets[b], scan_offsets[b+1]) (n_scans + 1 entries, ascending
 * from 0, no empty scan; at most 2^29 - 1 points and 65535 scans).  T_init / T_out: n_scans row-major 4x4 matrices;
 * n_iterations / converged / status: n_scans ints (status[b] = what dcreg_icp_run would have returned for scan b alone;
 * may be NULL); cov: n_scans x 36 doubles, scan b's post-loop covariance as dcreg_last_covariance gives it after a
 * single run, or NULL; log: n_scans x log_cap records (scan-major) or NULL.  Each scan is sorted by target cell under
 * its own initial pose and stops on its own convergence test; it differs from dcreg_set_source(scan b) + dcreg_icp_run
 * only in how the FP64 partial sums are grouped (counts, masks and iteration counts identical, poses equal to rounding;
 * a batch itself is reproducible bit for bit).  The scans go to buffers of their own: the context's source and what
 * dcreg_icp_run computes from it are left as they were. Not available on a sharded context (distribute scans over ranks
 * instead). */
int dcreg_icp_run_scans(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_scans, const float* xyz,
                        const int64_t* scan_offsets, int stride, const double* T_init, double* T_out,
                        int* n_iterations, int* converged, int* status, double* cov, dcreg_iter_log* log,
                        int log_cap);
/* Many scan/target pairs, EACH SOURCE AGAINST ITS OWN TARGET (scan-to-submap odometry, loop-closure candidates), side by
 * side in one sequence of launches, with one set of parameters.  src_xyz / tgt_xyz: HOST memory, concatenated, `stride`
 * floats per point; pair b is source points [src_offsets[b], src_offsets[b+1]) against target points
 * [tgt_offsets[b], tgt_offsets[b+1]) (n_pairs + 1 entries each, ascending strictly from 0: no empty source or target;
 * at most 2^29 - 1 points per side, at most 65535 pairs).  cell_size: as in dcreg_set_target (search_radius / cell_size
 * in (0, 4]); every target needs a dense grid (at most 2^27 cells in its bounding box, 2^30 over the call), unless
 * dcreg_set_sparse_maps(1): then a call past those limits gives every target a sparse row index, and pair b equals
 * dcreg_set_target(tgt_b) + dcreg_set_source(src_b) + dcreg_icp_run(T_init[b]) up to the FP64 grouping.
 * T_init / T_out / n_iterations / converged / status / cov / log: as in dcreg_icp_run_scans, one per pair.
 * metrics: n_pairs x 4 doubles or NULL; pair b's dcreg_point_to_point_metrics(T_out[b], error_threshold) = rmse, fitness,
 * chamfer, n_valid (an aligned source too large for a dense grid, or a call whose targets are sparse row indexes:
 * DCREG_BAD_ARG after the poses are written, naming the pair).
 * Pair b gives what dcreg_set_target(tgt_b, cell_size) + dcreg_set_source(src_b) + dcreg_icp_run(T_init[b]) gives up to
 * the grouping of the FP64 partial sums; a call reproduces bit for bit.  Needs no dcreg_set_target / dcreg_set_source
 * beforehand and leaves the context's source, target and grid as they were.  Not available on a sharded context. */
int dcreg_icp_run_pairs(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_pairs, const float* src_xyz,
                        const int64_t* src_offsets, const float* tgt_xyz, const int64_t* tgt_offsets, int stride,
                        double cell_size, const double* T_init, double* T_out, int* n_iterations, int* converged,
                        int* status, double* cov, double error_threshold, double* metrics, dcreg_iter_log* log,
                        int log_cap);
/* S independent SEQUENCES OF FRAMES against the context's target (map-based localisation: frame k+1 starts from frame
 * k's registered pose composed with the odometry increment between the two).  Inside a sequence the frames run strictly
 * one after another, entirely on the device: frame k+1's initial pose is T_out[k] * delta[k], composed on the device when
 * frame k stops (converged, max_iterations reached or aborted), with no host round trip in between.  Different sequences
 * run side by side (the loop kernel's grid y).
 * xyz / frame_offsets / stride: all frames concatenated in HOST memory, as in dcreg_icp_run_scans (n_frames + 1 entries,
 * ascending strictly from 0: no empty frame; at most 2^29 - 1 points and 65535 frames in one call).
 * seq_offsets: n_seqs + 1 ascending ints over the frames (0 .. n_frames); sequence s is frames
 * [seq_offsets[s], seq_offsets[s+1]), and every sequence has at least one frame.
 * T_init: n_seqs row-major 4x4 poses, the prior of each sequence's first frame.  deltas: n_frames row-major 4x4
 * increments (entry k maps frame k's result to frame k+1's prior; the entry of a sequence's last frame is ignored), or
 * NULL for identity (the constant-position model).  T_prior (out, may be NULL): n_frames x 16, the prior each frame
 * actually started from.  T_out / n_iterations / converged / status / cov / log: one per frame, as in
 * dcreg_icp_run_scans (status[k] = what dcreg_icp_run returns for frame k alone from T_prior[k]).
 * - Abort and non-convergence do not stop a sequence: the next prior is composed from the pose the frame returned (on an
 *   abort the last pose, as dcreg_icp_run leaves it); the caller sees it in status / converged.
 * - Composition rule: R' = R R_delta, t' = R t_delta + t in FP64, every entry rounded as ((a0 b0 + a1 b1) + a2 b2), then
 *   + t, with no FMA contraction and no re-orthonormalisation.  dcreg_b200.api.compose_prior reproduces the bits.
 * - Each frame is sorted by target cell under its dead-reckoned prior (T_init composed with the increments alone), so a
 *   frame differs from dcreg_set_source(frame k) + dcreg_icp_run(T_prior[k]) only in how the FP64 partial sums are
 *   grouped (counts, masks and iteration counts identical, poses equal to rounding); a call reproduces bit for bit.
 * - Device memory grows with the points of the call (about 100 B per point, as for scans): process a long recording in
 *   calls of a few thousand frames, each call's T_init being the previous call's last T_out * delta.
 * The frames go to buffers of their own: the context's source and what dcreg_icp_run, trial batches and scan batches
 * compute are left as they were.  Needs max_iterations >= 1; not available on a sharded context
 * (give every rank its own sequences).  Errors: DCREG_BAD_ARG with dcreg_last_error, as dcreg_icp_run_scans. */
int dcreg_icp_run_sequences(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_seqs, const int* seq_offsets,
                            int n_frames, const float* xyz, const int64_t* frame_offsets, int stride,
                            const double* T_init, const double* deltas, double* T_prior, double* T_out,
                            int* n_iterations, int* converged, int* status, double* cov, dcreg_iter_log* log,
                            int log_cap);
/* S independent sequences of SCAN-TO-MAP ODOMETRY (a LiDAR front end with no prebuilt map): frame k registers against a
 * local map made from the results of the frames before it in its sequence, all on the device (no dcreg_set_target, no
 * host round trip between frames).  Different sequences run side by side.
 * xyz / frame_offsets / stride / seq_offsets / T_init and the outputs T_prior / T_out / n_iterations / converged /
 * status / cov / log: as in dcreg_icp_run_sequences (one entry per frame, in the caller's frame order).
 * cell_size: the dense-grid cell of the local maps; search_radius / cell_size must be in (0, 4].
 * - Anchor: the first frame of sequence s is not registered.  T_out = T_prior = T_init[s], n_iterations = 0,
 *   converged = 0, status = DCREG_OK, no log records, cov = 1e6 I (the rule for a run that did not converge).
 * - Map of frame k: the frames j in [max(first frame of the sequence, k - map_frames), k), ascending j, each frame's
 *   points in input order.  Point p of frame j becomes fl32(R_j p + t_j) with (R_j, t_j) = T_out[j]; each coordinate is
 *   ((r0 x + r1 y) + r2 z) + t in FP64 with one rounding per operation and no FMA, then one float32 rounding
 *   (dcreg_b200.api.map_points gives the same bits).  Every frame of the window goes in, aborted ones included, at the
 *   pose it returned; no downsampling (dcreg_icp_run_odometry_voxel adds voxel filters), cropping or keyframe selection.
 * - Prior of frame k: compose_prior(T_out[k-1], D) with the rounding rule of dcreg_icp_run_sequences.
 *   motion = DCREG_MOTION_INCREMENTS: D = deltas[k-1], or the identity when deltas is NULL.
 *   motion = DCREG_MOTION_CONSTANT_VELOCITY (deltas must be NULL): D = identity when frame k-1 is the anchor, else
 *   inv(T_out[k-2]) T_out[k-1], i.e. R_D = R_{k-2}^T R_{k-1}, t_D = R_{k-2}^T (t_{k-1} - t_{k-2}), the differences
 *   rounded first, every entry ((a0 b0 + a1 b1) + a2 b2) with no FMA (dcreg_b200.api.constant_velocity_increment).
 * - Frame k returns what dcreg_set_target(map_k, cell_size) + dcreg_set_source(frame k) + dcreg_icp_run(T_prior[k])
 *   returns, up to how the FP64 partial sums are grouped (the frames are sorted once per call by their own cells in the
 *   sensor frame): counts, masks, iteration counts and status identical, poses equal to rounding.  A call reproduces bit
 *   for bit.
 * - Execution: step i registers frame i of every sequence that has one; before it, the device assembles the step's maps
 *   from the poses in device memory and builds their dense grids (one host sync for the grids' bounds per step).
 * Limits (DCREG_BAD_ARG before anything is launched): map_frames >= 1, max_iterations >= 1, a valid motion (constant
 * velocity with deltas == NULL), no sharded context, at most 65535 frames and 2^29 - 1 frame points, and at every step at
 * most 2^29 - 1 map points over all sequences.  A map whose bounding box is too large for a dense grid at cell_size (over
 * 2^27 cells, or coordinates outside +-2^19 cells) is only found at its step: the call then returns DCREG_BAD_ARG with
 * dcreg_last_error naming the sequence and frame, the frames of the earlier steps have their outputs, and the context
 * stays usable.  With dcreg_set_sparse_maps(1) a step whose maps are over 2^27 cells each, or 2^30 in all, gives every
 * lane a sparse row index instead (one more host sync at that step) and returns the same results as dense grids would;
 * coordinates outside +-2^19 cells are still refused.  The context's source, target and grid, and what the other calls compute, are left as they were.
 * A recording that arrives frame by frame, or is too long for one call (about 100 B of device memory per point of the
 * call), goes through an odometry session (dcreg_odometry_open / _push / _close): pushed in any chunks, it returns
 * exactly what one call over the whole recording returns. */
int dcreg_icp_run_odometry(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_seqs, const int* seq_offsets,
                           int n_frames, const float* xyz, const int64_t* frame_offsets, int stride,
                           double cell_size, int map_frames, int motion, const double* T_init, const double* deltas,
                           double* T_prior, double* T_out, int* n_iterations, int* converged, int* status,
                           double* cov, dcreg_iter_log* log, int log_cap);
/* dcreg_icp_run_odometry with voxel-filtered frames and local maps.  F_s(P) = dcreg_voxel_downsample(P, source_voxel),
 * F_m(P) = dcreg_voxel_downsample(P, map_voxel); a voxel size of 0 means no filter (P itself).
 * - Frame k's source is F_s(frame k), filtered in its own sensor frame.  frame_points (out, may be NULL): n_frames
 *   counts, the size of F_s(frame k), anchors included (their kept points enter the maps too).
 * - Map of frame k: F_m(concatenation over the window frames j of map_points(T_out[j], F_s(frame j))), with the window,
 *   order and transform of dcreg_icp_run_odometry, filtered per sequence in world coordinates.
 * - Frame k returns what dcreg_set_target(map_k, cell_size) + dcreg_set_source(F_s(frame k)) + dcreg_icp_run(T_prior[k])
 *   returns, up to how the FP64 partial sums are grouped; priors, anchors, aborts, reproducibility and the untouched
 *   context as in dcreg_icp_run_odometry, which is this call with source_voxel = map_voxel = 0 (same launches, same bytes).
 * - Cost: the frames are filtered once per call (one extra host sync for the kept counts); each step's maps are
 *   filtered on the device (six more launches per step whatever the number of sequences) and their kept counts come
 *   back in the copy of the grids' bounds, so a step keeps its one host sync.
 * Errors (DCREG_BAD_ARG, dcreg_last_error naming the sequence and frame): a negative or non-finite voxel size (before
 * anything is launched); a frame with no finite point, or a voxel coordinate of the source filter outside [-2^20, 2^20)
 * (after the frames' filter, before any loop launch); a step's map with a voxel coordinate outside that range (at its
 * step, like a map too large for a dense grid: the earlier steps keep their outputs, the context stays usable).
 * dcreg_set_sparse_maps applies as in dcreg_icp_run_odometry. */
int dcreg_icp_run_odometry_voxel(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_seqs, const int* seq_offsets,
                                 int n_frames, const float* xyz, const int64_t* frame_offsets, int stride,
                                 double cell_size, int map_frames, int motion, double source_voxel, double map_voxel,
                                 const double* T_init, const double* deltas, int64_t* frame_points, double* T_prior,
                                 double* T_out, int* n_iterations, int* converged, int* status, double* cov,
                                 dcreg_iter_log* log, int log_cap);
/* dcreg_icp_run_odometry_voxel with a cap on the points each voxel keeps: F_s(P) = dcreg_voxel_downsample_n(P,
 * source_voxel, source_max_points), F_m(P) = dcreg_voxel_downsample_n(P, map_voxel, map_max_points); everything else
 * as in dcreg_icp_run_odometry_voxel, which is this call with source_max_points = map_max_points = 1 (same launches,
 * same bytes).  A map cap of KISS-ICP's default 20 keeps a map's density where a cap of 1 thins it to about one frame's
 * worth of points.  The map window is built in frame order and each frame's points in input order, so a voxel of the
 * map keeps the points of its oldest window frames.  Cost of a cap above 1: the filter's radix sort and one more launch
 * (see dcreg_voxel_downsample_n), once per call for the frames and once per step for the maps; the sort's scratch is
 * sized once per call for the largest step, so a step keeps its one host sync and the chunk graphs are captured once.
 * A cap below 1 is DCREG_BAD_ARG before anything is launched, whatever the voxel sizes. */
int dcreg_icp_run_odometry_voxel_n(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_seqs, const int* seq_offsets,
                                   int n_frames, const float* xyz, const int64_t* frame_offsets, int stride,
                                   double cell_size, int map_frames, int motion, double source_voxel, double map_voxel,
                                   int source_max_points, int map_max_points, const double* T_init,
                                   const double* deltas, int64_t* frame_points, double* T_prior, double* T_out,
                                   int* n_iterations, int* converged, int* status, double* cov, dcreg_iter_log* log,
                                   int log_cap);
/* dcreg_icp_run_odometry_voxel_n with motion compensation (deskewing) of every registered frame, KISS-ICP's DeSkewScan.
 * timestamps (HOST, one float per input point, indexed like xyz; NULL: this call is dcreg_icp_run_odometry_voxel_n
 * itself, same launches, same bytes): tau, the point's fraction of its sweep in [0, 1], normalised by the caller; the
 * reference time is mid-sweep, tau = 0.5, so T_out[k] is the sensor pose at the middle of frame k's sweep.
 * - Motion: D_k, the increment frame k's prior is composed with (T_prior[k] = compose_prior(T_out[k-1], D_k)): deltas[k-1]
 *   (or the identity) with DCREG_MOTION_INCREMENTS, constant_velocity_increment(T_out[k-2], T_out[k-1]) (identity right
 *   after the anchor) with DCREG_MOTION_CONSTANT_VELOCITY - the same bytes.  xi_k = Log(D_k) (SE(3), Sophus's
 *   convention: the rotation through its quaternion and atan2, exact on [0, pi]).
 * - Deskew: every kept point p of frame k becomes fl32(Exp((tau - 0.5) xi_k) p), in FP64 with one float32 rounding
 *   (Rodrigues and the V matrix; dcreg_b200/csrc/se3.cuh, and dcreg_b200.api.deskew_points for the NumPy twin).  A point
 *   is copied bit for bit, with no arithmetic, when tau = 0.5, when xi_k is exactly zero or not finite, when it has a
 *   non-finite coordinate, or when the result would have one: deskewing adds no non-finite coordinate.  Anchors are
 *   never deskewed (nothing is known of their motion).  Accuracy: within one float32 ulp of the exact value or 1e-12 m,
 *   whichever is larger (the device's sincos and libm's differ in the last FP64 bit).
 * - Order: the source filter runs first, on the raw points (the plan needs every frame's kept count before the loop);
 *   each kept point is then deskewed at its frame's step with its own timestamp.  KISS-ICP deskews, then filters; this
 *   call filters, then deskews.
 * - The deskewed frame is what frame k registers with, what enters the later maps (at T_out[k]) and what a session
 *   retains.  deskewed_xyz (out, may be NULL): every frame's kept points after deskewing, 3 floats each, frame_points[k]
 *   rows per frame in the caller's frame order, anchors included.
 * - Cost: one timestamp upload and one gather launch per call, two launches per step (the lanes' twists, then every point
 *   of the step's frames), outside the loop's CUDA graphs; deskewed_xyz costs one copy of the kept points.
 * Errors (DCREG_BAD_ARG before anything is launched, dcreg_last_error naming the sequence, frame and point): a
 * timestamp that is not finite, or outside [0, 1]; everything else as in dcreg_icp_run_odometry_voxel_n. */
int dcreg_icp_run_odometry_deskew(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_seqs, const int* seq_offsets,
                                  int n_frames, const float* xyz, const int64_t* frame_offsets, int stride,
                                  double cell_size, int map_frames, int motion, double source_voxel, double map_voxel,
                                  int source_max_points, int map_max_points, const double* T_init, const double* deltas,
                                  const float* timestamps, int64_t* frame_points, double* T_prior, double* T_out,
                                  int* n_iterations, int* converged, int* status, double* cov, float* deskewed_xyz,
                                  dcreg_iter_log* log, int log_cap);
/* dcreg_icp_run_odometry_deskew with a PERSISTENT VOXEL MAP per sequence instead of the window of map_frames frames
 * (KISS-ICP's VoxelHashMap): the map is carried from frame to frame, so it covers the space around the sensor rather than
 * the last W frames.  Same arguments, without map_frames, plus max_distance; timestamps and deskewed_xyz may be NULL
 * (NULL timestamps: no deskewing, as in dcreg_icp_run_odometry_voxel_n).
 * - Update: U(M, P, T) = prune(cap(M ++ map_points(T, P)), t_T), with cap(X) = dcreg_voxel_downsample_n(X, map_voxel,
 *   map_max_points) (each voxel keeps its map_max_points points of smallest index, bit for bit, in order: M comes first,
 *   so older points win, KISS-ICP's AddPoints) and prune(X, t) dropping every point of every voxel whose first point q
 *   has ((qx - tx)^2 + (qy - ty)^2) + (qz - tz)^2 >= max_distance^2 (KISS-ICP's RemovePointsFarFromLocation), in FP64
 *   from the float32 coordinates, one rounding per operation, no FMA, max_distance^2 = max_distance * max_distance in
 *   FP64.  Survivors keep their order.  dcreg_b200.api.voxel_map_update gives the same bits.
 * - Maps: M_1 = U(empty, F_s(anchor), T_init[s]), M_{k+1} = U(M_k, F_s(frame k), T_out[k]): every frame goes in at the
 *   pose it returned, aborted ones included, deskewed when timestamps are given.  Frame k registers against M_k and
 *   returns what dcreg_set_target(M_k, cell_size) + dcreg_set_source(F_s(frame k)) + dcreg_icp_run(T_prior[k]) returns,
 *   up to how the FP64 partial sums are grouped; priors, anchors, deskewing, covariances and logs as in
 *   dcreg_icp_run_odometry_deskew.
 * - max_distance = +inf prunes nothing; then, since cap(cap(A) ++ B) = cap(A ++ B), M_k is the window map of
 *   dcreg_icp_run_odometry_deskew with map_frames >= the longest sequence, and every output is the same bytes.
 * - Cost per step: one launch that lays out [old map | new frame] for every sequence, the capped filter and one prune
 *   launch, whatever the number of sequences; the new maps' sizes come back in the copy of the grids' bounds, so a step
 *   keeps its one host sync.  Buffers are sized from the sizes read back so far and grow with headroom.
 * Errors (DCREG_BAD_ARG before anything is launched): map_voxel not finite and > 0, map_max_points < 1, max_distance NaN
 * or <= 0 (+inf is allowed); everything else as in dcreg_icp_run_odometry_deskew.  At its step (dcreg_last_error naming
 * the sequence and frame; the earlier steps keep their outputs, the context stays usable): a map with no dense grid
 * (without dcreg_set_sparse_maps(1), as in dcreg_icp_run_odometry), an empty map (every voxel pruned), a map voxel
 * coordinate outside [-2^20, 2^20), more than 2^29 - 1 map points over a step's sequences.  An unpruned map
 * (max_distance = +inf) of a long drive outgrows the dense grid: dcreg_set_sparse_maps(1) keeps it running. */
int dcreg_icp_run_odometry_map(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_seqs, const int* seq_offsets,
                               int n_frames, const float* xyz, const int64_t* frame_offsets, int stride, double cell_size,
                               int motion, double source_voxel, double map_voxel, int source_max_points,
                               int map_max_points, double max_distance, const double* T_init, const double* deltas,
                               const float* timestamps, int64_t* frame_points, double* T_prior, double* T_out,
                               int* n_iterations, int* converged, int* status, double* cov, float* deskewed_xyz,
                               dcreg_iter_log* log, int log_cap);
/* ODOMETRY SESSION: scan-to-map odometry of S sequences fed as the frames arrive.  The session keeps each sequence's
 * last map_frames registered frames (their filtered points in sensor coordinates and their poses) on the device
 * between pushes, with the motion model's state, so no frame is uploaded or filtered twice.
 * Contract: pushing a recording's frames in any chunking (one frame at a time, ragged pushes, sequences advancing at
 * different rates) gives byte for byte the outputs of one dcreg_icp_run_odometry_voxel_n call over the whole recording
 * with the session's settings: T_prior, T_out, n_iterations, converged, status, cov, frame_points and the log records
 * (all but iter_time_ms).
 * dcreg_odometry_open: the settings of that call (params is copied; cell_size, map_frames, motion, voxel sizes and caps,
 *   T_init: n_seqs x 16), checked as that call checks them, and dcreg_set_sparse_maps as it is at open (every push
 *   uses that value, so any chunking still gives the one call's bytes; _open_map and _open_adaptive record it too).  One session per context: open while one is open is
 *   DCREG_BAD_ARG, as is a sharded context.  dcreg_destroy frees an open session.
 * dcreg_odometry_push: the next frames of the sequences.  seq_offsets: n_seqs + 1 NON-DECREASING ints from 0 to
 *   n_frames (n_frames >= 1; a sequence may get no frame, and then keeps its window untouched); xyz / frame_offsets /
 *   stride and the outputs as in dcreg_icp_run_odometry_voxel_n, for the pushed frames in the caller's order.  Frame
 *   numbers count from open: the first frame ever pushed to sequence s is its anchor (T_out = T_prior = T_init[s], cov
 *   = 1e6 I, its points enter the maps).  deltas (n_frames x 16, or NULL for identity) has the one call's meaning: entry
 *   k maps pushed frame k's result to the prior of the next frame of its sequence, which may come in a later push (the
 *   session keeps each sequence's last entry), so the pushes' deltas concatenated are the one call's deltas.  With
 *   DCREG_MOTION_CONSTANT_VELOCITY deltas must be NULL; the increment comes from the two previous results, wherever
 *   they were pushed.
 *   A push that fails returns DCREG_BAD_ARG with dcreg_last_error naming the sequence and its frame number since open
 *   (bad tables, a frame the source filter leaves empty, a voxel coordinate out of range, a step's map with no dense
 *   grid) and leaves the session exactly as it was: outputs of completed steps may have been written, but nothing is
 *   committed, so the caller may split the push and retry.
 *   Cost: a push costs what its frames cost in a one-shot call (the source filter's sync, one bounds copy per step, the
 *   read-back) plus one launch that gathers the next windows; equal-shaped pushes reuse the buffers and the loop's CUDA
 *   graphs.  Other calls may run between pushes without changing the session's results, and a push leaves the
 *   context's source, target and grid as they were.
 * dcreg_odometry_close: ends the session and frees its buffers; push or close without an open session is
 *   DCREG_BAD_ARG. */
int dcreg_odometry_open(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_seqs, double cell_size, int map_frames,
                        int motion, double source_voxel, double map_voxel, int source_max_points, int map_max_points,
                        const double* T_init);
int dcreg_odometry_push(dcreg_ctx* ctx, const int* seq_offsets, int n_frames, const float* xyz,
                        const int64_t* frame_offsets, int stride, const double* deltas, int64_t* frame_points,
                        double* T_prior, double* T_out, int* n_iterations, int* converged, int* status, double* cov,
                        dcreg_iter_log* log, int log_cap);
/* dcreg_odometry_push with motion compensation: timestamps and deskewed_xyz as in dcreg_icp_run_odometry_deskew, for the
 * pushed frames (NULL timestamps: dcreg_odometry_push itself).  The session contract extends to it: any chunking gives
 * byte for byte what one dcreg_icp_run_odometry_deskew call over the recording gives, deskewed_xyz included.  The
 * increments are the one call's, so a pushed frame whose previous frames came in earlier pushes is deskewed with the
 * retained poses or the sequence's last delta.  Pushes may mix: the frames of a push without timestamps are those of a
 * call with every tau = 0.5 (copied), and the frames a session retains are the deskewed ones.  A timestamp that is not
 * finite or outside [0, 1] is DCREG_BAD_ARG naming the sequence, its frame number since open and the point, before
 * anything is launched, and leaves the session unchanged. */
int dcreg_odometry_push_deskew(dcreg_ctx* ctx, const int* seq_offsets, int n_frames, const float* xyz,
                               const int64_t* frame_offsets, int stride, const double* deltas, const float* timestamps,
                               int64_t* frame_points, double* T_prior, double* T_out, int* n_iterations, int* converged,
                               int* status, double* cov, float* deskewed_xyz, dcreg_iter_log* log, int log_cap);
/* dcreg_odometry_open for the voxel map of dcreg_icp_run_odometry_map: the settings of that call (no map_frames; the
 * same checks), and dcreg_odometry_push / _push_deskew push onto it unchanged.  The session keeps every sequence's map
 * (its last frame already in it) and the motion model's two last poses on the device; the contract carries over: any
 * chunking gives byte for byte the outputs of one dcreg_icp_run_odometry_map call over the recording, and a push that
 * fails (also at its step: a map with no dense grid, an empty map, a voxel coordinate out of range, too many points)
 * commits nothing.  One exception to the contract: the 2^29 - 1 point limit counts an update's whole input, which in a
 * session also holds the maps carried along (in the push's final update, every sequence's map), so near that limit a
 * session can fail a push that the one call over the same recording accepts.  Cost: a push's steps as in the one call, with the maps of the sequences without a frame at a step
 * carried through its update, plus one final update that puts the push's last frames in their maps (one more sync). */
int dcreg_odometry_open_map(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_seqs, double cell_size, int motion,
                            double source_voxel, double map_voxel, int source_max_points, int map_max_points,
                            double max_distance, const double* T_init);
/* The current voxel map of sequence seq of the session dcreg_odometry_open_map opened: M after the sequence's last
 * committed frame (empty before its first), copied to the HOST as 3 floats per point in map order.  *n always receives
 * its size; a cap below it (or a null xyz for a non-empty map) is DCREG_BAD_ARG and writes nothing else.  DCREG_BAD_ARG
 * also without a session, for a window session, a null n or a seq outside [0, n_seqs). */
int dcreg_odometry_local_map(dcreg_ctx* ctx, int seq, float* xyz, int64_t cap, int64_t* n);
int dcreg_odometry_close(dcreg_ctx* ctx);
/* THE ADAPTIVE THRESHOLD (KISS-ICP's AdaptiveThreshold): every frame's search radius follows how far registration has had
 * to correct its sequence's motion model so far, so a model that is sometimes wrong (constant velocity through a turn)
 * widens the basin only while it is wrong.  The radius of frame k+1 depends on T_prior[k] and T_out[k], which exist only
 * on the device until the call returns: it cannot be done from outside without one call per frame.
 * initial_threshold: sigma before a sequence has a sample; min_motion: errors at or below it are not samples;
 * max_range: the lever arm that turns the rotation error into metres.  KISS-ICP's defaults are 2.0, 0.1 and 100.0. */
typedef struct dcreg_adaptive_threshold {
    double initial_threshold, min_motion, max_range;
} dcreg_adaptive_threshold;
/* Scan-to-map odometry with every setting of dcreg_icp_run_odometry_deskew and dcreg_icp_run_odometry_map, plus the
 * adaptive threshold.  map_frames >= 1: the window of dcreg_icp_run_odometry_deskew (max_distance is not read);
 * map_frames = 0: the voxel map of dcreg_icp_run_odometry_map, pruned at max_distance.  adaptive == NULL is that call
 * itself: same launches, same bytes, search_radius filled with params->search_radius.
 * - State, per sequence: (sse, n), FP64 and integer, (0, 0) at the sequence's anchor.  sigma = initial_threshold when
 *   n = 0, else sqrt(sse / n).  Frame k registers with radius_k = min(3 sigma, params->search_radius): the parameter
 *   becomes the ceiling, and search_radius / cell_size in (0, 4] is still what is checked.  sqrt, the division, 3 sigma
 *   and the min are single IEEE operations: radius_k is a bit-exact function of (sse, n).
 * - Update, after frame k has stopped (converged, not converged or aborted; anchors never): D =
 *   constant_velocity_increment(T_prior[k], T_out[k]) = inv(T_prior[k]) T_out[k] with that function's rounding rule;
 *   theta = the rotation angle of R_D through its quaternion, 2 atan2(|v|, w) (the route of the deskew's Log);
 *   e = 2 max_range sin(theta / 2) + |t_D| in FP64.  If e is finite and e > min_motion: sse += e e, n += 1; otherwise
 *   the state stays (a frame that returns its prior contributes nothing).  dcreg_b200.api.adaptive_threshold_error /
 *   _update / _radius are the NumPy twin: the radius bit for bit from (sse, n); e to a few FP64 ulp (the device's sin
 *   and atan2 and libm's differ in the last bit), so compare a frame with the radius the call returned.
 * - Everything that follows the radius follows the frame's own: the 5-NN-within-radius rule, the rings of grid cells a
 *   search visits (ceil(radius_k / cell_size), at least 1; lanes of one step may differ), the step limit of coherent
 *   mode, the fitness count.  Frame k returns what dcreg_set_target(map_k, cell_size) + dcreg_set_source(frame k) +
 *   dcreg_icp_run(T_prior[k]) returns with params.search_radius = radius_k, up to how the FP64 sums are grouped.
 * - search_radius (out, may be NULL): n_frames doubles in the caller's frame order, radius_k; anchors get 0.
 * - Cost: one launch per step whatever the number of sequences (one thread per lane, after the step's loop, outside
 *   the loop's CUDA graphs); the next step's radii come back in the copy of the grids' bounds, so a step keeps its one
 *   host sync, and the chunk graphs are still captured once per call.
 * Errors (DCREG_BAD_ARG before anything is launched): initial_threshold or max_range not finite or <= 0, min_motion not
 * finite or < 0; everything else as in the call the map selects. */
int dcreg_icp_run_odometry_adaptive(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_seqs, const int* seq_offsets,
                                    int n_frames, const float* xyz, const int64_t* frame_offsets, int stride,
                                    double cell_size, int map_frames, int motion, double source_voxel, double map_voxel,
                                    int source_max_points, int map_max_points, double max_distance,
                                    const dcreg_adaptive_threshold* adaptive, const double* T_init, const double* deltas,
                                    const float* timestamps, int64_t* frame_points, double* T_prior, double* T_out,
                                    int* n_iterations, int* converged, int* status, double* cov, float* deskewed_xyz,
                                    double* search_radius, dcreg_iter_log* log, int log_cap);
/* dcreg_odometry_open (map_frames >= 1) or dcreg_odometry_open_map (map_frames = 0) with the adaptive threshold
 * (adaptive == NULL: that call itself).  Every sequence's (sse, n) is session state: a push starts from the committed
 * state, a push that fails commits nothing, and any chunking of a recording gives byte for byte what one
 * dcreg_icp_run_odometry_adaptive call over it gives, search_radius included.  dcreg_odometry_push and _push_deskew push
 * onto it unchanged; dcreg_odometry_push_adaptive is dcreg_odometry_push_deskew that also returns search_radius (on a
 * session without the threshold: params->search_radius). */
int dcreg_odometry_open_adaptive(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_seqs, double cell_size,
                                 int map_frames, int motion, double source_voxel, double map_voxel, int source_max_points,
                                 int map_max_points, double max_distance, const dcreg_adaptive_threshold* adaptive,
                                 const double* T_init);
int dcreg_odometry_push_adaptive(dcreg_ctx* ctx, const int* seq_offsets, int n_frames, const float* xyz,
                                 const int64_t* frame_offsets, int stride, const double* deltas, const float* timestamps,
                                 int64_t* frame_points, double* T_prior, double* T_out, int* n_iterations, int* converged,
                                 int* status, double* cov, float* deskewed_xyz, double* search_radius, dcreg_iter_log* log,
                                 int log_cap);
/* Voxel downsampling of many clouds in one call (KISS-ICP's VoxelDownsample rule: the first point of every voxel).
 * xyz / offsets / stride: HOST memory as in dcreg_icp_run_scans (n_clouds + 1 offsets, ascending strictly from 0, at
 * most 2^29 - 1 points).  With inv = 1.0 / voxel in FP64, point i's voxel is (floor((double)x inv), floor((double)y inv),
 * floor((double)z inv)); a point with a non-finite coordinate has none and is dropped.  Each voxel keeps its point of
 * smallest index, its coordinates copied bit for bit; the kept points stay in input order.  dcreg_b200.api.voxel_downsample
 * gives the same selection.  Every voxel coordinate must lie in [-2^20, 2^20) (checked in FP64): a cloud outside it is
 * DCREG_BAD_ARG naming the cloud.  out_xyz: room for offsets[n_clouds] x 3 floats, cloud b's kept points being
 * [out_offsets[b], out_offsets[b+1]) (n_clouds + 1 entries); out_index (may be NULL): each kept point's index inside its
 * own cloud.  One host sync; the launches do not depend on n_clouds.  The context's source, target and grid are left
 * as they were. */
int dcreg_voxel_downsample(dcreg_ctx* ctx, int n_clouds, const float* xyz, const int64_t* offsets, int stride,
                           double voxel, float* out_xyz, int64_t* out_offsets, int64_t* out_index);
/* dcreg_voxel_downsample keeping up to max_points points per voxel (KISS-ICP's VoxelHashMap::AddPoints rule with
 * max_points_per_voxel, points inserted in index order): within each cloud, each voxel keeps its max_points points of
 * smallest index; voxels, dropped points, bit-for-bit copies, input order, out_index and errors as in
 * dcreg_voxel_downsample, which is this call with max_points = 1 (same launches, same bytes).
 * dcreg_b200.api.voxel_downsample(P, voxel, max_points) gives the same selection.  max_points < 1 is DCREG_BAD_ARG before
 * anything is launched.
 * Cost: max_points = 1 takes the cheaper path of one atomicMin per point.  max_points > 1 replaces it by a stable radix
 * sort of the points by their voxel's table slot (32-bit keys, as many radix passes as the slot count has bits) and one
 * O(1) pass per point whatever a voxel's occupancy: seven launches besides the sort's, whatever n_clouds. */
int dcreg_voxel_downsample_n(dcreg_ctx* ctx, int n_clouds, const float* xyz, const int64_t* offsets, int stride,
                             double voxel, int max_points, float* out_xyz, int64_t* out_offsets, int64_t* out_index);
/* dcreg_voxel_downsample_n with a minimum point spacing (KISS-ICP's AddPoints, which skips a point closer than
 * voxel / sqrt(max_points_per_voxel) to a point already in its voxel).  Within each cloud and voxel, in ascending index,
 * point p is kept iff fewer than max_points points of its voxel are kept before it and every kept point q before it has
 * ((px - qx)^2 + (py - qy)^2) + (pz - qz)^2 >= min_spacing^2, in FP64 from the float32 coordinates with one rounding
 * per operation and min_spacing^2 = min_spacing * min_spacing (a point exactly min_spacing away is kept).  A voxel's
 * first point is always kept; the result is idempotent, and filtering filter(A) ++ B gives filter(A ++ B).  Voxels,
 * dropped points, bit-for-bit copies, input order, out_index and errors as in dcreg_voxel_downsample_n, which is this
 * call with min_spacing = 0; max_points = 1 or min_spacing = 0 runs it (same launches, same bytes), and min_spacing
 * above twice the voxel size keeps what max_points = 1 keeps.  dcreg_b200.api.voxel_downsample(P, voxel, max_points,
 * min_spacing) gives the same selection.  min_spacing NaN, negative or infinite is DCREG_BAD_ARG before anything is
 * launched.  Cost: the radix sort of dcreg_voxel_downsample_n and the same launches, whatever n_clouds; its O(1) flag
 * pass becomes one in which a warp settles each voxel's points in order, O(points x max_points) per voxel. */
int dcreg_voxel_downsample_spaced(dcreg_ctx* ctx, int n_clouds, const float* xyz, const int64_t* offsets, int stride,
                                  double voxel, int max_points, double min_spacing, float* out_xyz, int64_t* out_offsets,
                                  int64_t* out_index);
/* Same loop, but correspondences are supplied by the caller each iteration through a callback
 * (host kd-tree mode, "PR1"): planes are 4*n doubles (nx,ny,nz,d), all-zero = none. */
typedef int (*dcreg_plane_callback)(void* user, const double T[16], double* planes4,
                                    int64_t* n_corr_pt);
int dcreg_icp_run_host_planes(dcreg_ctx* ctx, const dcreg_icp_params* params,
                              const double T_init[16], dcreg_plane_callback cb, void* user,
                              double T_out[16], dcreg_iter_log* log, int log_cap,
                              int* n_iterations, int* converged);
/* Post-loop covariance (icp_test_runner.cpp:2014-2037): inverse of the last H with the 1e-9
 * eigenvalue floor, or 1e6*I when not converged.  cov: 36 doubles. */
int dcreg_last_covariance(dcreg_ctx* ctx, double cov[36]);

/* Post-run point-to-point metrics on the device.  Replaces calculatePointToPointError
 * (DCReg/include/utils.hpp:538-589; callers icp_test_runner.cpp:506-510 and :1463-1470): aligned = fl32(T * source);
 * out = { P2P RMSE (over all source points, distances below error_threshold), P2P fitness, Chamfer distance,
 * number of source points within the threshold }.  Needs dcreg_set_source + dcreg_set_target. */
int dcreg_point_to_point_metrics(dcreg_ctx* ctx, const double T[16], double error_threshold, double out[4]);

/* ---- multi-GPU: point-block sharding (SURVEY.md §8e) ---------------------------------------
 * Each rank holds a contiguous block of source slots; the 27+5 accumulators are summed over ranks
 * once per iteration (inside the reducing kernel over peer memory, see dcreg_comm_mode; one
 * ncclAllReduce of 32 doubles on the context's stream as the fallback), then every rank runs K2
 * redundantly on bit-identical sums.  nccl_unique_id is the 128-byte ncclUniqueId created by dcreg_comm_unique_id on
 * rank 0 and distributed by the caller (e.g. torch.distributed broadcast). */
int dcreg_comm_unique_id(dcreg_ctx* ctx, uint8_t id_out[128]);
int dcreg_comm_init(dcreg_ctx* ctx, const uint8_t nccl_unique_id[128], int rank, int nranks);
int dcreg_comm_destroy(dcreg_ctx* ctx);
/* How the per-iteration sum over ranks is carried: 0 = no communicator, 1 = ncclAllReduce behind the reducing kernel
 * (fallback), 2 = peer-memory mailboxes over NVLink inside the reducing kernel's last block (one kernel per iteration,
 * bit-identical sums on every rank).  dcreg_comm_init picks 2 when every rank could map every peer (cudaIpc). */
int dcreg_comm_mode(const dcreg_ctx* ctx);
/* Total number of source points over all ranks (denominator of `fitness`); defaults to local n. */
int dcreg_set_global_source_count(dcreg_ctx* ctx, int64_t n_total);

/* ---- instrumentation ----------------------------------------------------------------------- */
/* Number of kernels this context has launched since creation (bench.py's gpu_launches). */
int64_t dcreg_launch_count(const dcreg_ctx* ctx);
/* Device pointers of the ctx-owned source float4 array and plane arrays (for the K1 seam). */
void* dcreg_device_source(dcreg_ctx* ctx);
void* dcreg_device_planes_f64(dcreg_ctx* ctx);
void* dcreg_device_planes_f32(dcreg_ctx* ctx);   /* filled by dcreg_freeze_planes_f32 */
/* Round the ctx's double planes to float4 on the device (the 32 B/slot K1 layout). */
int dcreg_freeze_planes_f32(dcreg_ctx* ctx);
/* Enqueue `reps` K1 launches over the ctx-owned source + planes (plane_is_f64 0/1) and return
 * the average device time per launch in milliseconds, measured with CUDA events on ctx's stream.
 * If flush_l2 != 0 a >L2-sized buffer is rewritten before every launch (outside the events). */
int dcreg_time_reduce(dcreg_ctx* ctx, int plane_is_f64, const double pose_Rt[12],
                      int use_weight_derivative, int reps, int flush_l2, float* ms_per_launch);
/* Profiling aid for the fused loop: enqueue `reps` loop bodies from pose T (source sorted as dcreg_icp_run does) and
 * return the average device time per body in milliseconds.  what = 0: the iteration kernel alone at the fixed
 * pose T; what = 1: iteration kernel + solve/update kernel, i.e. `reps` real iterations (no convergence stop). */
int dcreg_time_iteration(dcreg_ctx* ctx, const dcreg_icp_params* params, const double T[16], int what,
                         int reps, float* ms_per_body);
/* Profiling aid: run `iters` real loop iterations from pose T and record the phase time stamps (GPU globaltimer, ns) of
 * the LAST one.  out: (n_blocks + 1) x 16 values; row b < n_blocks, thread 0 of block b: [0] start (pose loaded),
 * [1] certificates done, [2] searches done, [3] fit list built, [4] fits done, [5] rows / Gram done, and for the block
 * that finished the reduction [6] partials summed, [7] sums ready, [8] solve step done; row n_blocks: the solve step's
 * own stamps [0] entry, [1] block inverses, [2] Schur eigen-decompositions, [3] preconditioner, [4] solve, [5] pose
 * update, and [15] = index of the block that ran it. */
int dcreg_iteration_timeline(dcreg_ctx* ctx, const dcreg_icp_params* params, const double T[16], int iters,
                             uint64_t* out, int out_cap_blocks, int* n_blocks);
/* Profiling counters of the loop's iteration kernel since the last call: out = { source slots that ran a neighbour
 * search, source slots that ran a plane fit } (the others reused the previous iteration's result, see DESIGN.md).
 * enable != 0 switches the counting on (off by default), 0 switches it off. */
int dcreg_iteration_counters(dcreg_ctx* ctx, int enable, uint64_t out[2]);

#ifdef __cplusplus
}
#endif
#endif /* DCREG_B200_H */
