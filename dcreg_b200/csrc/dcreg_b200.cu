// dcreg_b200.cu - kernels + C ABI of the H100 (sm_90a) ICP / degeneracy engine (see include/dcreg_b200.h).
//
// Data layout in HBM (per context):
//   src      float4[N]   body-frame source points (x,y,z,-), uploaded once per scan
//   tgt grid float4[M]   target points grouped by grid cell + cell_start table (dense grid) or row-start table (sparse)
//   planes64 double4[N]  (nx,ny,nz,d) per source slot, only materialised for the seams / host-plane mode
//   planes32 float4[N]   the 32 B/slot frozen-plane layout of the K1 benchmark
//   per trial (dcreg_icp_run: one, dcreg_icp_run_batch: many): neighbour records / plane cache (100 B per slot),
//   partials double[grid.x][32], acc double[32], ticket, state (pose, flags, warm-start bases), log records
// One ICP iteration = ONE kernel (icp_iter2_kernel): correspondences + residual + Jacobian + 27-sum reduction; the block
// that finishes a trial's reduction sums the block partials, [adds the other ranks' sums through peer-memory mailboxes,
// peer_reduce.cuh,] and its first warp runs the K2 step (analysis, solve, pose update, convergence flag), so nothing
// returns to the host inside the loop and the loop bodies of a run are replayed as one CUDA graph.  Baseline methods
// and the NCCL fallback of a sharded run keep K2 as a second kernel (k2_step_kernel).
#include <cub/device/device_radix_sort.cuh>
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <array>
#include <cstddef>
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "../../include/dcreg_b200.h"
#include "adaptive_threshold.cuh"
#include "arena_plan.hpp"
#include "corr.cuh"
#include "k1_reduce.cuh"
#include "k1_stream.cuh"
#include "k2_solve.cuh"
#include "lane_plan.hpp"
#include "loop_plan.hpp"
#include "odom_plan.hpp"
#include "se3.cuh"
#include "peer_reduce.cuh"

using k2::IcpState;
using k2::kAcc;

// ------------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------------
namespace {

constexpr int kBlock = 256;

// Programmatic dependent launch (sm_90+): the loop's two kernels are launched with the programmatic-stream-
// serialization attribute, so kernel k+1 is scheduled while kernel k still runs; pdl_wait() blocks until kernel k
// has completed and its writes are visible, pdl_release() lets kernel k+2 be scheduled.  Hides the launch
// latency of every kernel on the loop's critical path.  Without the attribute both are no-ops.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_release() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

__device__ __forceinline__ k1::Pose load_pose(const IcpState* st) {
    k1::Pose P;
#pragma unroll
    for (int i = 0; i < 9; ++i) P.R[i] = st->R[i];
#pragma unroll
    for (int i = 0; i < 3; ++i) P.t[i] = st->t[i];
    return P;
}

// K2 executed by warp 0 of the block that finished a trial's reduction (k2_solve.cuh).  A separate function with its
// own register allocation and stack frame: the iteration kernels are capped at 85 registers for 3 blocks per SM and
// must not pay for the solve's live state.  acc: the body-frame sums in shared memory.
static_assert(sizeof(k2::WarpSmem) <= 8 * k1::kTRow * sizeof(double), "k2::WarpSmem must fit one warp's transpose buffer");
static_assert(sizeof(corr::WarpKnnSmem) <= 8 * k1::kTRow * sizeof(double), "corr::WarpKnnSmem must fit one warp's transpose buffer");
__device__ __noinline__ void solve_step_in_kernel(const double* acc, IcpState* st, const dcreg_icp_params* prm,
                                                  dcreg_iter_log* log, int log_cap, k2::WarpSmem* sm, const float* src_radius,
                                                  double coherent_step, unsigned int* n_active, unsigned long long* dbg) {
    // only the "Ours" method (Schur detection + PCG, the warp-cooperative step) is folded; the baseline methods' generic
    // single-thread step needs a 3.7 KB stack frame, which every thread of the iteration kernel would have to reserve:
    // they keep the separate solve kernel (k2_step_kernel)
    const int lane = threadIdx.x & 31;
    const double lever = src_radius ? (double)*src_radius : 1.0e30;
    const double max_step = coherent_step * prm->search_radius;
    k2::icp_step_warp_ours(acc, st, *prm, log, log_cap, *sm, lever, max_step, dbg);    // all 32 lanes cooperate
    __syncwarp();
    if (lane == 0 && n_active && st->done) atomicSub(n_active, 1u);
}

// ---- sequences of frames (dcreg_icp_run_sequences) --------------------------------------------------------------
// Grid y is the sequence LANE s; it runs the frames [first[s], first[s+1]) one after another, frame cursor[s] now.  The
// reduction's working set (partials, ticket, sums) belongs to the lane; everything a registration owns (loop state,
// record slices, lever arm, log slice, covariance) to the frame.  The cursor lives in device memory like the pose and
// the mode flags, since a captured chunk of the loop freezes its kernel arguments.
struct SeqView {
    int* cursor;              // [lanes] frame the lane runs now (>= first[s + 1]: the lane is finished); null: no sequences
    const int* first;         // [lanes + 1] frame ranges
    const double* delta;      // [frames][16] row-major increments (frame k's result -> frame k+1's prior), or null (identity)
    double* T_prior;          // [frames][16] the prior each frame started from
    const long long* seg;     // [frames + 1] point offsets of the frames
    unsigned int* n_active;   // lanes still running
};

// A fresh loop state at pose T (row-major 4x4) over n_source points: a trial of a batch before its first iteration, or
// a frame of a sequence when the frame before it stops.  Unseeded, lean mode: the records of the slot range are unused.
__device__ __forceinline__ void init_loop_state(IcpState* st, const double* T, long long n_source) {
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) st->R[r * 3 + c] = T[r * 4 + c];
        st->t[r] = T[r * 4 + 3];
    }
    st->iter = 0; st->done = 0; st->converged = 0; st->status = DCREG_OK;
    for (int i = 0; i < 36; ++i) st->H_last[i] = (i % 7 == 0) ? 1.0 : 0.0;
    st->n_source_total = n_source;
    st->step_rot = 1.0e30; st->step_trans = 1.0e30; st->seeds = 0; st->coherent_used = 0; st->coherent = 0; st->warm = 0;
    st->t_last = k2::globaltimer_ns();                      // tic of iteration 0 (icp_test_runner.cpp:1695)
}

// Prior of the next frame, T' = T D: R' = R R_D, t' = R t_D + t, every entry ((a0 b0 + a1 b1) + a2 b2) [+ t] rounded in
// that order with no FMA contraction and no re-orthonormalisation (dcreg_b200.api.compose_prior gives the same bits).
// The host uses it for the dead-reckoned priors (plain x86-64 double arithmetic, which has no FMA to contract to).
__host__ __device__ __forceinline__ void compose_prior(const double* R, const double* t, const double* D, double* T) {
#ifdef __CUDA_ARCH__
#define DCREG_MUL(x, y) __dmul_rn(x, y)
#define DCREG_ADD(x, y) __dadd_rn(x, y)
#else
#define DCREG_MUL(x, y) ((x) * (y))
#define DCREG_ADD(x, y) ((x) + (y))
#endif
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            double s = DCREG_ADD(DCREG_ADD(DCREG_MUL(R[3 * r], D[c]), DCREG_MUL(R[3 * r + 1], D[4 + c])),
                                 DCREG_MUL(R[3 * r + 2], D[8 + c]));
            if (c == 3) s = DCREG_ADD(s, t[r]);
            T[4 * r + c] = s;
        }
#undef DCREG_MUL
#undef DCREG_ADD
    T[12] = 0.0; T[13] = 0.0; T[14] = 0.0; T[15] = 1.0;
}

// The constant-velocity increment of dcreg_icp_run_odometry, D = inv(T_a) T_b for the poses (Ra, ta) of frame k-2 and
// (Rb, tb) of frame k-1: R_D = Ra^T Rb, t_D = Ra^T (tb - ta), the differences rounded first, every entry
// ((a0 b0 + a1 b1) + a2 b2) with no FMA contraction (dcreg_b200.api.constant_velocity_increment gives the same bits).
__host__ __device__ __forceinline__ void constant_velocity_increment(const double* Ra, const double* ta, const double* Rb,
                                                                     const double* tb, double* D) {
#ifdef __CUDA_ARCH__
#define DCREG_MUL(x, y) __dmul_rn(x, y)
#define DCREG_ADD(x, y) __dadd_rn(x, y)
#define DCREG_SUB(x, y) __dsub_rn(x, y)
#else
#define DCREG_MUL(x, y) ((x) * (y))
#define DCREG_ADD(x, y) ((x) + (y))
#define DCREG_SUB(x, y) ((x) - (y))
#endif
    const double dt[3] = {DCREG_SUB(tb[0], ta[0]), DCREG_SUB(tb[1], ta[1]), DCREG_SUB(tb[2], ta[2])};
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int c = 0; c < 3; ++c)
            D[4 * r + c] = DCREG_ADD(DCREG_ADD(DCREG_MUL(Ra[r], Rb[c]), DCREG_MUL(Ra[3 + r], Rb[3 + c])),
                                     DCREG_MUL(Ra[6 + r], Rb[6 + c]));
        D[4 * r + 3] = DCREG_ADD(DCREG_ADD(DCREG_MUL(Ra[r], dt[0]), DCREG_MUL(Ra[3 + r], dt[1])), DCREG_MUL(Ra[6 + r], dt[2]));
    }
#undef DCREG_MUL
#undef DCREG_ADD
#undef DCREG_SUB
    D[12] = 0.0; D[13] = 0.0; D[14] = 0.0; D[15] = 1.0;
}

// Lane s's frame `frame` has stopped (converged, max_iterations or aborted): start the next frame of the lane from the
// pose this one returned composed with its increment, or, after the lane's last frame, count the lane as finished.  One
// thread, right after the solve step; the next launch reads the cursor after pdl_wait.  Own register allocation, like
// solve_step_in_kernel: the tile code does not pay for it.
__device__ __noinline__ void advance_frame(SeqView q, IcpState* states, int s, int frame) {
    const int next = frame + 1;
    if (next < q.first[s + 1]) {
        const IcpState* st = states + frame;
        double D[16] = {1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, 1.0};
        if (q.delta)
            for (int i = 0; i < 16; ++i) D[i] = q.delta[(size_t)frame * 16 + i];
        double T[16];
        compose_prior(st->R, st->t, D, T);
        double* P = q.T_prior + (size_t)next * 16;
        for (int i = 0; i < 16; ++i) P[i] = T[i];
        init_loop_state(states + next, T, q.seg[next + 1] - q.seg[next]);
    } else {
        atomicSub(q.n_active, 1u);
    }
    q.cursor[s] = next;
}

struct IterArgs {
    const float4* src;        // source points, w = bit-cast original index (spatially sorted copy or the original)
    long long n;
    corr::Grid grid;
    IcpState* state;
    double* partials;
    unsigned int* counter;
    double* acc;
    double4* planes_out;      // seam 1: the planes at the ORIGINAL slot index (only icp_iter2_kernel<., ., ., true> writes them)
    dcreg_icp_params prm;
};

// ---- the loop's iteration kernel -----------------------------------------------------------------------------------
// One thread per source slot (on a dense grid the source is sorted by target cell once per run).  Coherent mode:
//   1. q = fl32(R p + t); squared distances from q to the slot's SEVEN nearest target points of its last search.
//   2. skip test.  That search also left lb8, a lower bound on the squared distance from q_scan (where the query then
//      was) to every target point outside the seven.  The query has moved by delta = |q - q_scan|; while
//          (5th smallest of the seven new distances) + delta < sqrt(lb8)
//      (with margins that dwarf the float32 evaluation error of a squared distance) no outside point can be among
//      the five nearest, so the seven are only re-ranked by their new distances (index rule on ties) and no cell is
//      touched.  On a uniform surface the 8th neighbour is ~26 % farther than the 5th, so once the pose moves by
//      less than a few centimetres per iteration almost every slot takes this path.
//   3. otherwise an exact bounded 7-NN search (corr::knn_search_lb): bound = 1.21 x the largest of the seven new
//      distances (seven distinct real points bound the 7th distance; the look-ahead is what finds a gap even when
//      the 8th candidate is far), or the search radius on the first iteration.
//   4. neighbour record to HBM (next iteration's seeds); plane fit to the first five, reused while the ordered
//      list of five stays the same (same five rows in the same order give the same QR bit for bit); residual /
//      weight / Jacobian row; DMMA Gram accumulation.  Searches and fits of a tile (<= 256 slots, Iter2Args::tile) go through work lists.
// Tail: packed per-block partial, atomic ticket, last block reduces (k1s::finish_packed).
// Record per slot (3 int4): {pos0..pos3}, {pos4..pos6, bits(lb8)}, {bits(q_scan.xyz), flags};
// pos = position in the grid's point array (ascending (d2, index) at the time of writing), -1 = none.
constexpr int kNnRec = 3;
constexpr float kNnLook = 1.21f;              // squared-distance look-ahead beyond the seed bound (any value >= 1 is exact)
constexpr double kCoherentStep = 0.05;        // records are used once no source point moves more than this x search radius per iteration

constexpr int kStampSlots = 16;                // per-block phase time stamps of the loop kernel (profiling only)
#define DCREG_STAMP(k) do { if (a.stamps && tid == 0) a.stamps[(size_t)blockIdx.x * kStampSlots + (k)] = k2::globaltimer_ns(); } while (0)

constexpr int kSearchListMax = 96;            // more searching slots than this in a tile: every thread searches for itself

struct Iter2Smem {
    double tbuf[kBlock / 32][8 * k1::kTRow];    // per-warp DMMA transpose buffers (also: corr::WarpKnnSmem, the warp's Gram,
                                                // and - in the last block, after the reduction - k2::WarpSmem)
    k1s::TailSmem tail;
    // coherent mode, per tile (<= kBlock slots)
    float4 q[kBlock];                           // query (x, y, z), w = search bound B
    int res[kBlock][10];                        // pos0..pos6, bits(lb), bits(d2 of the 5th), 1 = no search / 0 = searched / 2 = search pending
    int key[kBlock][5];                         // the five positions in distance order (slots that need a fit)
    double4 plane[kBlock];
    signed char fitres[kBlock];
    int listS[kBlock], listF[kBlock];
    corr::RowRange rowtab[kSearchListMax][9];   // cell rows of the tile's listed searches (cell = radius)
    int nS, nF;
    corr::Grid grid;                            // this trial's own target grid (Iter2Args::grids)
    // odometry (kGrids and kSeq): the search radius of the lane's frame (Iter2Args::lane_radius, or the parameters'), its
    // square rounded up to float, and for the solve step the parameters with that radius
    double radius;
    float r2_up;
    dcreg_icp_params prm;
};

// Grid = (blocks per trial, trials).  A trial is one registration (one initial pose) of the context's source against
// its target (icp_test_runner.cpp:331-345 runs `num_runs` of them back to back; dcreg_icp_run_batch runs them side by
// side).  Everything a trial owns is an array indexed by blockIdx.y: loop state, ticket, partials, sums, neighbour
// records, plane cache, log.  dcreg_icp_run is the one-trial case.
struct Iter2Args {
    IterArgs it;              // it.state / it.partials / it.counter / it.acc: per-trial arrays ([B], [B][grid.x][32], [B], [B][32])
    int4* nn;                 // [B][kNnRec n] neighbour records
    double4* plane_cache;     // [B][n] plane fitted to the slot's current five neighbours (reused while the set stays)
    signed char* fit_state;   // [B][n] 0 = nothing cached, 1 = cached fit failed its gates, 2 = cached plane valid
    int* plane_key;           // [B][5 n] the five positions (in distance order) the cached plane was fitted to
    // the solve / update step (K2) runs in the last block of every trial: no second launch, no host, no acc round trip
    int fold_k2;              // 0: stop after writing the sums (sharded run over NCCL: all-reduce + k2_step_kernel follow)
    dcreg_iter_log* log;      // [B][log_cap] or null
    int log_cap;
    const float* src_radius;  // max |p| over the source (lever arm of a rotation step)
    double coherent_step;
    unsigned int* n_active;   // trials still running (decremented by the step that finishes one); host polls it
    peer::View peer;          // multi-GPU: the sum over ranks, inside the last block (peer_reduce.cuh)
    unsigned long long* stamps;   // profiling only (dcreg_iteration_timeline): [grid.x][kStampSlots] globaltimer values, or null
    int force;                // 0: mode and seeds from the loop state (written by K2); 1: coherent mode, seeds = use_seeds
    int use_seeds;            // (force) records of the previous launch are valid
    float r2_up;              // search radius^2 rounded up to float
    unsigned int* stats;      // optional [2]: slots that searched, slots that refitted (profiling)
    int tile;                 // source slots per block and pass (<= kBlock; plan_iteration: chosen so the blocks fill whole SM rounds)
    // single-trial folded run with a solver block (row_flags != null): block 0 sums the rows and solves (solver_block),
    // blocks 1.. work on the tiles; no ticket
    unsigned long long* row_flags;   // [grid.x - 1] row b is published with the value row_epoch + 1 of its launch
    unsigned long long* row_epoch;   // per-context launch counter (device memory: graph-captured arguments are frozen)
    IcpState* warm_state;            // scratch state of the solver block's warm-up step
    // a batch of different scans (dcreg_icp_run_scans): trial b owns the source slots [seg[b], seg[b+1]) of it.src and the
    // record slices at the same offsets (sized by the total slot count), and its own lever arm src_radius[b].
    // null: every trial runs the it.n slots of it.src, with record slices [b][it.n] and the one src_radius
    const long long* seg;
    // many scan/target pairs (dcreg_icp_run_pairs, with seg): trial b searches its own target grid grids[b] (device
    // memory, rings set) instead of it.grid.  Only the kGrids instantiations read it
    const corr::Grid* grids;
    // sequences of frames (dcreg_icp_run_sequences, with seg: the frames' slot ranges): grid y is the lane, the trial the
    // frame seq.cursor[lane].  Only the kSeq instantiations read it
    SeqView seq;
    // odometry with the adaptive threshold (dcreg_icp_run_odometry_adaptive): [lanes] the search radius of the frame each
    // lane runs at this step, in device memory (a captured chunk freezes its arguments), or null: prm.search_radius.
    // Only the kGrids && kSeq instantiations read it
    const double* lane_radius;
    // per-lane solver settings (dcreg_set_lane_params): [lanes] in device memory, grid y's entry lane_prm[ys], or with
    // lane_seq (odometry, whose steps compact the lanes) lane_prm[lane_seq[ys]]; null: it.prm for every lane.  Only a
    // lane whose settings run "Ours" folds its solve step; k2_step_kernel runs the others'
    const dcreg_icp_params* lane_prm;
    const int* lane_seq;
};

__device__ __forceinline__ void cswap5(unsigned long long& ka, int& pa, unsigned long long& kb, int& pb) {
    if (kb < ka) {                                    // one 64-bit compare = (distance, then index) order (corr::knn_key)
        const unsigned long long tk = ka; ka = kb; kb = tk;
        const int tp = pa; pa = pb; pb = tp;
    }
}

// The solver block of a single-trial folded run (blockIdx.x == 0, so it is dispatched first).  Without it the iteration
// ends in a serial chain that starts only when the last tile block wins the ticket: sum of all rows, then a solve step
// of a few thousand warp instructions fetched cold on whichever SM finished last.  Here, while the tile blocks work,
// warp 0 runs one step on a scratch copy of the state with the previous iteration's sums (everything it reads is stable
// after pdl_wait; it writes only the scratch state), which pulls the step's instructions into this SM's caches; then all
// warps sum the rows as they land (k1s::stream_rows_to_fin: the same additions as the ticket path, bit for bit), and
// the real step follows at once.  A row that never lands ends the trial with DCREG_CUDA_ERROR instead of hanging.
constexpr unsigned long long kRowTimeoutNs = 4000000000ull;
__device__ __noinline__ void solver_block(const Iter2Args& a, IcpState* st, Iter2Smem& sm, unsigned long long row_epoch,
                                          unsigned int peer_epoch) {
    const IterArgs& A = a.it;
    const int tid = threadIdx.x, warp = tid >> 5;
    k2::WarpSmem* wsm = reinterpret_cast<k2::WarpSmem*>(sm.tbuf[0]);
    if (warp == 0) {
        for (int e = tid; e < (int)(sizeof(IcpState) / sizeof(int)); e += 32)
            reinterpret_cast<int*>(a.warm_state)[e] = reinterpret_cast<const int*>(st)[e];
        __syncwarp();
        solve_step_in_kernel(A.acc, a.warm_state, &A.prm, nullptr, 0, wsm, a.src_radius, a.coherent_step, nullptr, nullptr);
        DCREG_STAMP(1);
    }
    const bool ok = k1s::stream_rows_to_fin(sm.tail, A.partials, a.row_flags, row_epoch + 1, (int)gridDim.x - 1,
                                            kRowTimeoutNs);
    if (tid == 0) *a.row_epoch = row_epoch + 1;     // the next launch reads it after pdl_wait
    DCREG_STAMP(6);
    if (!ok) {
        if (tid == 0) {
            st->done = 1; st->converged = 0; st->status = DCREG_CUDA_ERROR;
            if (a.n_active) atomicSub(a.n_active, 1u);
        }
        return;
    }
    peer::all_reduce32(a.peer, sm.tail.fin, sm.tail.red, peer_epoch);
    k1s::congruence(sm.tail.fin, st->R, sm.tail.acc);
    __syncthreads();
    DCREG_STAMP(7);
    if (tid < kAcc) A.acc[tid] = sm.tail.acc[tid];
    if (warp == 0) {
        solve_step_in_kernel(sm.tail.acc, st, &A.prm, a.log, a.log_cap, wsm, a.src_radius, a.coherent_step, a.n_active,
                             a.stamps ? a.stamps + (size_t)gridDim.x * kStampSlots : nullptr);
        DCREG_STAMP(8);
        if (a.stamps && tid == 0) {
            a.stamps[(size_t)gridDim.x * kStampSlots + 14] = 1;     // timeline: block 0 is the solver block
            a.stamps[(size_t)gridDim.x * kStampSlots + 15] = 0;
        }
    }
}

// kGrids: every trial has its own target grid (Iter2Args::grids), copied into shared memory once per block; the other
// paths keep reading it.grid from the kernel parameters, untouched by the table.  kSeq: grid y is a sequence lane
// (Iter2Args::seq) whose trial is the frame it runs now; the reduction's working set is the lane's.  Both (odometry,
// dcreg_icp_run_odometry): the grid is the lane's, grids[lane], a local map rebuilt before every step.  kPlanes (seam 1,
// dcreg_find_planes): every slot's plane goes to it.planes_out; a flag of its own, since the store costs the other
// instantiations spills.  kSparse: it.grid is the context's sparse row index (dcreg_set_target_sparse), whose searches
// read their ranges from its table (corr::sparse_span)
template <bool kUseWd, bool kGrids, bool kSeq, bool kPlanes = false, bool kSparse = false>
__global__ void __launch_bounds__(kBlock, 3) icp_iter2_kernel(const __grid_constant__ Iter2Args a) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    Iter2Smem& sm = *reinterpret_cast<Iter2Smem*>(smem_raw);
    const IterArgs& A = a.it;
    pdl_wait();                                   // the pose / mode flags come from the previous iteration's solve step
    pdl_release();
    const int ys = (int)blockIdx.y;               // owner of partials / ticket / sums: the trial, or (kSeq) the lane
    int trial = ys;
    if constexpr (kSeq) {                         // (the cursor too: written by the previous launch's frame advance)
        trial = a.seq.cursor[ys];
        if (trial >= a.seq.first[ys + 1]) return;
    }
    IcpState* const st = A.state + trial;
    if (st->done) return;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const bool solver_path = !kSeq && a.row_flags != nullptr;
    if (solver_path && blockIdx.x == 0) {
        DCREG_STAMP(0);
        solver_block(a, st, sm, *a.row_epoch, peer::load_epoch(a.peer));
        return;
    }
    const k1::Pose P = load_pose(st);
    if constexpr (kGrids) {
        static_assert(sizeof(corr::Grid) % sizeof(int) == 0 && sizeof(corr::Grid) / sizeof(int) <= kBlock, "grid copy");
        if (tid < (int)(sizeof(corr::Grid) / sizeof(int)))
            reinterpret_cast<int*>(&sm.grid)[tid] = reinterpret_cast<const int*>(a.grids + (kSeq ? ys : trial))[tid];
        if constexpr (kSeq) {
            if (tid == kBlock - 1) {              // r2_up: plan_iteration's round-up of the squared radius
                const double r = a.lane_radius ? a.lane_radius[ys] : A.prm.search_radius;
                sm.radius = r;
                sm.r2_up = a.lane_radius ? __double2float_ru(__dmul_rn(r, r)) : a.r2_up;
            }
        }
        __syncthreads();
    }
    const corr::Grid& g = kGrids ? sm.grid : A.grid;
    const unsigned int epoch0 = peer::load_epoch(a.peer);     // (after pdl_wait: the previous launch has advanced it)
    DCREG_STAMP(0);
    const int tb = (int)blockIdx.x - (solver_path ? 1 : 0), ntb = (int)gridDim.x - (solver_path ? 1 : 0);   // tile block
    // this trial's source slots and its slices of the per-slot records (Iter2Args::seg)
    long long n = A.n, rec0 = (long long)trial * A.n;
    const float4* src = A.src;
    if (a.seg) { rec0 = a.seg[trial]; n = a.seg[trial + 1] - rec0; src += rec0; }
    int4* const rec_nn = a.nn + (size_t)kNnRec * rec0;
    double4* const rec_plane = a.plane_cache + rec0;
    signed char* const rec_fit = a.fit_state + rec0;
    int* const rec_key = a.plane_key + (size_t)5 * rec0;
    // mode (uniform over the grid): while the pose still moves by more than ~5 % of the search radius per iteration
    // nothing can be reused; the lean path (plain 5-NN search, no records) is ~25 % cheaper than searching with a
    // certificate.  K2 flips `coherent` from the size of its update; a lean-only plan (coherent_step 0, plan_iteration)
    // never enters coherent mode and has no records.
    const bool coherent = a.force ? true : (st->coherent != 0);
    const bool use_seeds = a.force ? (a.use_seeds != 0) : (coherent && st->seeds != 0);
    double c0 = 0.0, c1 = 0.0, e0 = 0.0, e1 = 0.0;
    int neff = 0, npt = 0;
    unsigned n_search = 0, n_fit = 0;
    double radius = A.prm.search_radius;
    if constexpr (kGrids && kSeq) radius = sm.radius;
    const double r2max = radius * radius;
    {
        // ---- tiles of a.tile (<= 256) slots with per-tile work lists, so that searches and fits run densely packed.  Lean mode (the
        // pose still moves a lot) uses the same phases: every slot searches (plain 5-NN), every accepted slot fits.
        for (long long base = (long long)tb * a.tile; base < n; base += (long long)ntb * a.tile) {
            const long long i = base + tid;
            const bool valid = tid < a.tile && i < n;
            if (tid == 0) { sm.nS = 0; sm.nF = 0; }
            __syncthreads();
            // -- 1. query, previous seven, certificate
            double px = 0.0, py = 0.0, pz = 0.0;
            bool need = false;
            if (valid) {
                const float4 p4 = __ldg(&src[i]);
                px = (double)p4.x; py = (double)p4.y; pz = (double)p4.z;
                // q = fl32(R p + t)  (utils.hpp:630-636)
                const float qx = (float)(P.R[0] * px + P.R[1] * py + P.R[2] * pz + P.t[0]);
                const float qy = (float)(P.R[3] * px + P.R[4] * py + P.R[5] * pz + P.t[1]);
                const float qz = (float)(P.R[6] * px + P.R[7] * py + P.R[8] * pz + P.t[2]);
                float B = (kGrids && kSeq) ? sm.r2_up : a.r2_up;
                need = true;
                if (use_seeds) {
                    const int4 s0 = rec_nn[kNnRec * i], s1 = rec_nn[kNnRec * i + 1], s2 = rec_nn[kNnRec * i + 2];   // one round trip
                    if (s1.z >= 0) {                                          // all seven seeds exist
                        corr::KnnM nn;
                        nn.pos[0] = s0.x; nn.pos[1] = s0.y; nn.pos[2] = s0.z; nn.pos[3] = s0.w;
                        nn.pos[4] = s1.x; nn.pos[5] = s1.y; nn.pos[6] = s1.z;
#pragma unroll
                        for (int k = 0; k < corr::kSeeds; ++k) {
                            const float4 t = __ldg(&g.pts[nn.pos[k]]);
                            nn.key[k] = corr::knn_key(corr::dist2(qx, qy, qz, t), __float_as_int(t.w));
                        }
                        // 16-exchange sorting network on (d2, index)
#define DCREG_CS(x, y) cswap5(nn.key[x], nn.pos[x], nn.key[y], nn.pos[y])
                        DCREG_CS(0, 6); DCREG_CS(2, 3); DCREG_CS(4, 5); DCREG_CS(0, 2); DCREG_CS(1, 4); DCREG_CS(3, 6);
                        DCREG_CS(0, 1); DCREG_CS(2, 5); DCREG_CS(3, 4); DCREG_CS(1, 2); DCREG_CS(4, 6); DCREG_CS(2, 3);
                        DCREG_CS(4, 5); DCREG_CS(1, 2); DCREG_CS(3, 4); DCREG_CS(5, 6);
#undef DCREG_CS
                        B = fminf(B, corr::knn_d2(nn, 6) * kNnLook);
                        const float ex = qx - __int_as_float(s2.x), ey = qy - __int_as_float(s2.y), ez = qz - __int_as_float(s2.z);
                        const float delta = sqrtf(ex * ex + ey * ey + ez * ez);
                        const float lb = __int_as_float(s1.w);
                        // nothing outside the seven was closer than sqrt(lb) to q_scan; it is now at least sqrt(lb) - delta away
                        need = !((sqrtf(corr::knn_d2(nn, 4)) + delta) * 1.00002f + 1e-7f < sqrtf(lb) * 0.99998f);
                        if (!need) {
#pragma unroll
                            for (int k = 0; k < corr::kSeeds; ++k) sm.res[tid][k] = nn.pos[k];
                            sm.res[tid][7] = s1.w; sm.res[tid][8] = __float_as_int(corr::knn_d2(nn, 4)); sm.res[tid][9] = 1;
                        }
                    }
                }
                sm.q[tid] = make_float4(qx, qy, qz, B);
                if (need) { sm.res[tid][9] = 2; ++n_search; }
            }
            {   // search list of the tile (slot order)
                const unsigned bits = __ballot_sync(0xffffffffu, need);
                int wbase = 0;
                if (lane == 0 && bits) wbase = atomicAdd(&sm.nS, __popc(bits));
                wbase = __shfl_sync(0xffffffffu, wbase, 0);
                if (need) sm.listS[wbase + __popc(bits & ((1u << lane) - 1u))] = tid;
            }
            DCREG_STAMP(1);
            __syncthreads();
            // -- 2. searches: few -> one warp per listed slot (the other slots' threads are not held up by a
            //       long sequential search); many -> every thread searches for its own slot
            const int nS = sm.nS;
            if (coherent && nS <= kSearchListMax) {
                corr::WarpKnnSmem& W = *reinterpret_cast<corr::WarpKnnSmem*>(sm.tbuf[warp]);
                // cell = radius: the 9 cell rows of EVERY listed search are set up by all threads first (one memory round
                // trip for the tile instead of one at the head of each of a warp's searches)
                const bool pre_rows = g.rings == 1;
                if (pre_rows) {
                    for (int e = tid; e < nS * 9; e += kBlock) {
                        const int sidx = e / 9, r = e - sidx * 9;
                        const float4 q = sm.q[sm.listS[sidx]];
                        sm.rowtab[sidx][r] = corr::knn_row_range<kSparse>(g, q.x, q.y, q.z, q.w, r);
                    }
                    __syncthreads();
                }
                for (int w = warp; w < nS; w += kBlock / 32) {
                    const int t = sm.listS[w];
                    const float4 q = sm.q[t];
                    corr::KnnM r;
                    float lbq = ((kGrids && kSeq) ? sm.r2_up : a.r2_up) * 0.9999f;    // nothing beyond the rings of cells is closer than the radius
                    const bool got = corr::knn_warp_search<kSparse>(g, q.x, q.y, q.z, q.w, W, r, lbq,
                                                           (a.stamps && warp == 0) ? reinterpret_cast<long long*>(a.stamps + (size_t)blockIdx.x * kStampSlots + 9) : nullptr,
                                                           pre_rows ? sm.rowtab[w] : nullptr);
                    if (got) {
                        if (lane < corr::kSeeds) sm.res[t][lane] = W.opos[lane];
                        if (lane == 7) sm.res[t][7] = __float_as_int(lbq);
                        if (lane == 8) sm.res[t][8] = __float_as_int(corr::knn_d2(r, 4));
                        if (lane == 9) sm.res[t][9] = 0;
                    }
                    __syncwarp();
                }
                __syncthreads();
            }
            DCREG_STAMP(2);
            if (valid && sm.res[tid][9] == 2) {       // too many for the list, or more than 64 candidates inside the bound
                const float4 q = sm.q[tid];
                if (coherent) {
                    corr::KnnM r;
                    float lbq = ((kGrids && kSeq) ? sm.r2_up : a.r2_up) * 0.9999f;
                    corr::knn_search_lb<kSparse>(g, q.x, q.y, q.z, q.w, r, lbq);
#pragma unroll
                    for (int k = 0; k < corr::kSeeds; ++k) sm.res[tid][k] = r.pos[k];
                    sm.res[tid][7] = __float_as_int(lbq); sm.res[tid][8] = __float_as_int(corr::knn_d2(r, 4));
                } else {                              // lean: plain exact 5-NN, nothing kept for the next iteration
                    corr::Knn5 r;
                    corr::knn_init(r);
                    corr::knn_search<kSparse>(g, q.x, q.y, q.z, r);
                    int rpos[5];
                    corr::knn_positions(g, r, rpos);
#pragma unroll
                    for (int k = 0; k < 5; ++k) sm.res[tid][k] = rpos[k];
                    sm.res[tid][5] = -1; sm.res[tid][6] = -1; sm.res[tid][7] = 0; sm.res[tid][8] = __float_as_int(corr::knn_d2(r, 4));
                }
                sm.res[tid][9] = 0;
            }
            // -- 3a. record; which five; cached plane?
            double nx = 0.0, ny = 0.0, nz = 0.0, d = 0.0;
            bool ok = false, want_fit = false, have5 = false;
            float d5 = 0.0f;
            if (valid) {
                int pos[corr::kSeeds];
#pragma unroll
                for (int k = 0; k < corr::kSeeds; ++k) pos[k] = sm.res[tid][k];
                d5 = __int_as_float(sm.res[tid][8]);
                if (coherent) {
                    rec_nn[kNnRec * i] = make_int4(pos[0], pos[1], pos[2], pos[3]);
                    rec_nn[kNnRec * i + 1] = make_int4(pos[4], pos[5], pos[6], sm.res[tid][7]);
                    if (sm.res[tid][9] == 0) {                                // searched: remember where
                        const float4 q = sm.q[tid];
                        rec_nn[kNnRec * i + 2] = make_int4(__float_as_int(q.x), __float_as_int(q.y), __float_as_int(q.z), 0);
                    }
                }
                // (a lean search is not bounded by the radius: its five may lie outside and then need no plane)
                have5 = pos[4] >= 0 && (coherent || (double)d5 < r2max);
                // The plane is a function of the five target points IN THEIR ORDER (the rows of the 5x3 system keep the
                // reference's distance order, so the QR rounds exactly as a fresh fit would): the cache key is the
                // ordered list.  A pure re-ranking therefore refits; the fit list keeps that cheap.
                const int key[5] = {pos[0], pos[1], pos[2], pos[3], pos[4]};
                int fit = 0;                                                  // 1 = gates failed, 2 = plane valid
                if (have5) {
                    int cached = 0;
                    if (use_seeds) {
                        const int* kp = rec_key + 5 * i;
                        if (kp[0] == key[0] && kp[1] == key[1] && kp[2] == key[2] && kp[3] == key[3] && kp[4] == key[4])
                            cached = (int)rec_fit[i];
                    }
                    if (cached == 2) {
                        const double4 c = rec_plane[i];
                        nx = c.x; ny = c.y; nz = c.z; d = c.w;
                        fit = 2;
                    } else if (cached == 1) {
                        fit = 1;
                    } else {
                        want_fit = true;
#pragma unroll
                        for (int k = 0; k < 5; ++k) sm.key[tid][k] = key[k];
                    }
                }
                if (!want_fit) { if (coherent) rec_fit[i] = (signed char)fit; ok = fit == 2; }
            }
            {   // fit list of the tile
                const unsigned bits = __ballot_sync(0xffffffffu, want_fit);
                int wbase = 0;
                if (lane == 0 && bits) wbase = atomicAdd(&sm.nF, __popc(bits));
                wbase = __shfl_sync(0xffffffffu, wbase, 0);
                if (want_fit) sm.listF[wbase + __popc(bits & ((1u << lane) - 1u))] = tid;
            }
            DCREG_STAMP(3);
            __syncthreads();
            // -- 3b. fits, densely packed into the first warps
            const int nF = sm.nF;
            for (int f = tid; f < nF; f += kBlock) {
                const int t = sm.listF[f];
                double fx = 0.0, fy = 0.0, fz = 0.0, fd = 0.0;
                const int fit = corr::fit_plane_reg(g, sm.key[t], A.prm.min_normal_norm, A.prm.plane_thickness, fx, fy, fz, fd) ? 2 : 1;
                sm.plane[t] = make_double4(fx, fy, fz, fd);
                sm.fitres[t] = (signed char)fit;
                if (coherent) {
                    const long long it = base + t;
                    if (fit == 2) rec_plane[it] = make_double4(fx, fy, fz, fd);
                    int* kp = rec_key + 5 * it;
#pragma unroll
                    for (int k = 0; k < 5; ++k) kp[k] = sm.key[t][k];
                    rec_fit[it] = (signed char)fit;
                }
                ++n_fit;
            }
            __syncthreads();
            DCREG_STAMP(4);
            // -- 3c. gate, row, Gram
            if (valid) {
                if (want_fit) {
                    const double4 c = sm.plane[tid];
                    nx = c.x; ny = c.y; nz = c.z; d = c.w;
                    ok = sm.fitres[tid] == 2;
                }
                if (have5 && (double)d5 < r2max) npt += 1;                    // icp_test_runner.cpp:1726, 1731
                else ok = false;
                if (!ok) { nx = 0.0; ny = 0.0; nz = 0.0; d = 0.0; }
                if constexpr (kPlanes) A.planes_out[__float_as_int(src[i].w)] = make_double4(nx, ny, nz, d);
            }
            double c[8];
            k1::slot_front<kUseWd>(P, px, py, pz, nx, ny, nz, d, ok, c, neff, A.prm.weight_slope, A.prm.weight_gate);
            __syncwarp();
            k1::gram_accumulate_dmma(sm.tbuf[warp], lane, c, c0, c1, e0, e1);
            __syncthreads();
        }
    }
    DCREG_STAMP(5);
    // (the solver block advances the counter only after it has seen this block's flag, which carries the value read here)
    const unsigned long long row_want = solver_path ? *a.row_epoch + 1 : 0ull;
    if (a.stats) {
        n_search = __reduce_add_sync(0xffffffffu, n_search);
        n_fit = __reduce_add_sync(0xffffffffu, n_fit);
        if (lane == 0 && (n_search | n_fit)) { atomicAdd(&a.stats[0], n_search); atomicAdd(&a.stats[1], n_fit); }
    }
    // ---- tail: the warp's 8x8 Gram -> packed totals (k1s::kPk layout), then the grid reduction
    c0 += e0; c1 += e1;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        neff += __shfl_xor_sync(0xffffffffu, neff, off);
        npt += __shfl_xor_sync(0xffffffffu, npt, off);
    }
    double* G = sm.tbuf[warp];
    G[2 * lane] = c0; G[2 * lane + 1] = c1;
    __syncwarp();
    double mine = 0.0;
    if (lane < 21) {
        int i = 0, rem = lane;
        while (rem >= 6 - i) { rem -= 6 - i; ++i; }
        const int j = i + rem;
        mine = 0.5 * (G[i * 8 + j] + G[j * 8 + i]);
    } else if (lane < 27) {
        const int i = lane - 21;
        mine = 0.5 * (G[i * 8 + 6] + G[6 * 8 + i]);
    } else if (lane == k1s::kPkR2) mine = G[7 * 8 + 7];
    else if (lane == k1s::kPkB2) mine = G[6 * 8 + 6];
    else if (lane == k1s::kPkNeff) mine = (double)neff;
    else if (lane == k1s::kPkNpt) mine = (double)npt;
    if (solver_path) {
        k1s::publish_row(mine, sm.tail, A.partials + (size_t)tb * k1s::kPk, a.row_flags + tb, row_want);
        DCREG_STAMP(6);
        return;
    }
    // ---- grid reduction of this trial, [sum over ranks], congruence, solve + pose update: all in the last block
    if (!k1s::reduce_to_fin(mine, sm.tail, A.partials + (size_t)ys * gridDim.x * k1s::kPk, A.counter + ys,
                            (int)blockIdx.x, (int)gridDim.x)) return;
    DCREG_STAMP(6);
    peer::all_reduce32(a.peer, sm.tail.fin, sm.tail.red, epoch0);
    k1s::congruence(sm.tail.fin, st->R, sm.tail.acc);
    __syncthreads();
    DCREG_STAMP(7);
    if (tid < kAcc) A.acc[(size_t)ys * kAcc + tid] = sm.tail.acc[tid];
    if (a.fold_k2 && warp == 0) {
        const dcreg_icp_params* prm = &A.prm;
        if (a.lane_prm) {                         // per-lane settings: this lane's, and k2_step_kernel steps a baseline lane
            prm = a.lane_prm + (a.lane_seq ? a.lane_seq[ys] : ys);
            if (!(prm->detection == DCREG_DET_SCHUR_CONDITION_NUMBER && prm->handling == DCREG_HAND_PRECONDITIONED_CG))
                return;
        }
        if constexpr (kGrids && kSeq) {           // the step limit of coherent mode follows the frame's own radius
            if (a.lane_radius) {
                static_assert(sizeof(dcreg_icp_params) % sizeof(int) == 0, "parameter copy");
                for (int e = lane; e < (int)(sizeof(dcreg_icp_params) / sizeof(int)); e += 32)
                    reinterpret_cast<int*>(&sm.prm)[e] = reinterpret_cast<const int*>(prm)[e];
                __syncwarp();
                if (lane == 0) sm.prm.search_radius = sm.radius;
                __syncwarp();
                prm = &sm.prm;
            }
        }
        solve_step_in_kernel(sm.tail.acc, st, prm, a.log ? a.log + (size_t)trial * a.log_cap : nullptr, a.log_cap,
                             reinterpret_cast<k2::WarpSmem*>(sm.tbuf[0]), a.seg ? a.src_radius + trial : a.src_radius,
                             a.coherent_step, a.n_active,
                             a.stamps ? a.stamps + (size_t)gridDim.x * kStampSlots : nullptr);
        if constexpr (kSeq) {                     // (a.n_active is null here: the advance counts finished lanes)
            __syncwarp();
            if (lane == 0 && st->done) advance_frame(a.seq, A.state, ys, trial);
        }
        DCREG_STAMP(8);
        if (a.stamps && tid == 0) a.stamps[(size_t)gridDim.x * kStampSlots + 15] = blockIdx.x;      // which block was last
    }
}

// A kernel instantiation and the dynamic shared memory it is launched with
template <typename Args>
struct KernelEntry { void (*kernel)(Args); size_t smem; };
using LoopKernel = KernelEntry<Iter2Args>;

static cudaError_t loop_kernel_attributes(const LoopKernel& k) {
    cudaError_t e = cudaFuncSetAttribute(k.kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k.smem);
    // the smallest shared-memory carveout that keeps 3 blocks resident (each also reserves 1 KB), so that the rest of the
    // SM's unified data cache is L1 for the searches' and certificates' target reads.  The percentage is of the largest
    // carveout and is rounded up to the next capacity the SM supports.
    int dev = 0, max_smem = 0;
    if (e == cudaSuccess) e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev);
    if (e == cudaSuccess) {
        const size_t need = 3 * (k.smem + 1024);
        const int pct = (int)std::min<size_t>(100, (need * 100 + (size_t)max_smem - 1) / (size_t)max_smem);
        e = cudaFuncSetAttribute(k.kernel, cudaFuncAttributePreferredSharedMemoryCarveout, pct);
    }
    return e;
}

// K2 as its own kernel: baseline methods (their generic single-thread step), the host-plane loop and the NCCL fallback
// of a sharded run.  One warp per trial (blockIdx.x).
// K2 executes a few thousand warp instructions exactly once per launch, so it stalls on instruction fetch.  Thanks to the programmatic dependent launch it starts while the
// iteration kernel is still running, so it first executes the SAME code on a scratch copy of the state with the
// previous iteration's sums (same branches, harmless stores), which pulls the instructions into the SM's caches;
// only then does it wait for the iteration kernel and do the real step.
static_assert(kAcc == 32, "k2_step_kernel copies acc with one element per lane");
struct K2Scratch {
    double acc_prev[kAcc];
    IcpState state;
};

// One warp per trial (blockIdx.x): acc_all [B][kAcc], st_all [B], log_all [B][log_cap].  scratch (rehearsal) only for B = 1.
// radius_per_trial: src_radius is [B] (a batch of different scans) instead of one value for every trial.
// seq.cursor set (sequences of frames): blockIdx.x is a lane with acc_all [lanes][kAcc]; its trial is the frame it runs
// now, and the step that stops a frame advances the lane (no rehearsal: scratch is null).  lane_radius: Iter2Args's, or null
// lane_prm, lane_seq: Iter2Args's (per-lane settings; prm is entry 0); folded: the iteration kernel has run the step of
// every lane whose settings run "Ours", so their blocks return at once
__global__ void __launch_bounds__(32) k2_step_kernel(const double* acc_all, IcpState* st_all, dcreg_icp_params prm,
                                                     dcreg_iter_log* log_all, int log_cap, const float* src_radius,
                                                     double coherent_step, K2Scratch* scratch, unsigned int* n_active,
                                                     int radius_per_trial, SeqView seq, const double* lane_radius,
                                                     const dcreg_icp_params* lane_prm, const int* lane_seq, int folded) {
    __shared__ k2::WarpSmem sm;
    pdl_release();
    const int lane = threadIdx.x;
    const double* acc = acc_all + (size_t)blockIdx.x * kAcc;
    int trial = (int)blockIdx.x;
    if (seq.cursor) {
        pdl_wait();                                       // the cursor comes from the previous launch's advance
        trial = seq.cursor[blockIdx.x];
        if (trial >= seq.first[blockIdx.x + 1]) return;
    }
    // the lane's settings in shared memory: its entry (read after the cursor, since a lane past its last frame may be
    // past the step's lanes of lane_seq too), or prm.  The step reads them there in both cases
    __shared__ dcreg_icp_params P;
    if (lane_prm) {
        const int* from = reinterpret_cast<const int*>(lane_prm + (lane_seq ? lane_seq[blockIdx.x] : blockIdx.x));
        for (int e = lane; e < (int)(sizeof(dcreg_icp_params) / sizeof(int)); e += 32) reinterpret_cast<int*>(&P)[e] = from[e];
    } else if (lane == 0) {
        P = prm;
    }
    __syncwarp();
    const bool warp_path = P.detection == DCREG_DET_SCHUR_CONDITION_NUMBER && P.handling == DCREG_HAND_PRECONDITIONED_CG;
    if (folded && warp_path) return;
    IcpState* st = st_all + trial;
    dcreg_iter_log* log = log_all ? log_all + (size_t)trial * log_cap : nullptr;
    if (src_radius && radius_per_trial) src_radius += trial;
    // (odometry's adaptive threshold: the lane's own search radius, Iter2Args::lane_radius)
    const double max_step = coherent_step * (lane_radius ? lane_radius[blockIdx.x] : prm.search_radius);
#pragma unroll 1
    for (int pass = scratch ? 0 : 1; pass < 2; ++pass) {
        const double* acc_use = acc;
        IcpState* st_use = st;
        dcreg_iter_log* log_use = log;
        if (pass == 0) {                                  // rehearsal: nothing the previous kernels still write is read
            for (int e = lane; e < (int)(sizeof(IcpState) / sizeof(int)); e += 32)
                reinterpret_cast<int*>(&scratch->state)[e] = reinterpret_cast<const int*>(st)[e];
            __syncwarp();
            acc_use = scratch->acc_prev; st_use = &scratch->state; log_use = nullptr;
        } else {
            pdl_wait();                                   // acc comes from the iteration kernel (or the all-reduce) before
            if (st->done) return;
        }
        // mode of the next iteration kernel: records pay off once no source point moves more than ~5 % of the search radius
        const double lever = src_radius ? (double)*src_radius : 1.0e30;
        if (warp_path) {
            k2::icp_step_warp_ours(acc_use, st_use, P, log_use, log_cap, sm, lever, max_step);   // all 32 lanes cooperate
        } else if (lane == 0) {
            k2::icp_step(acc_use, st_use, P, log_use, log_cap, lever, max_step);    // baseline methods: generic single-thread path
        }
        __syncwarp();
        if (pass == 1 && scratch) scratch->acc_prev[lane] = acc[lane];              // kAcc == 32: next launch's rehearsal input
        if (pass == 1 && lane == 0 && n_active && st->done) atomicSub(n_active, 1u);
        if (pass == 1 && lane == 0 && seq.cursor && st->done) advance_frame(seq, st_all, (int)blockIdx.x, trial);
    }
}

__global__ void k2_analyze_kernel(const double* v27, dcreg_icp_params prm, dcreg_analysis* out, double* dx) {
    if (threadIdx.x != 0) return;
    k2::analyze_and_solve<true>(v27, prm, out, dx);
}

// Post-run log fill: one thread per iteration record recomputes the FULL analysis from the record's H27 with the seam's
// code and thereby adds the log-only quantities without putting them on the loop's critical path.  The baseline
// methods' step (k2::icp_step) runs that same code on the same inputs, so its record is rewritten with identical
// values.  The "Ours" step (k2::icp_step_warp_ours) has its own arithmetic: the decisions it wrote (mask, is_degenerate,
// schur_singular, PCG iterations and residual) are kept, so the record describes the step that moved the pose even
// where a decision sits within rounding of its threshold and the seam's code would have gone the other way.
// lane_prm (per-lane settings, prm is entry 0): trial y's record uses lane_prm[trial_lane[y]], or without trial_lane
// lane_prm[y]; null: prm.
__global__ void log_fill_kernel(dcreg_iter_log* logs, int log_cap, const IcpState* states, dcreg_icp_params prm,
                                const dcreg_icp_params* lane_prm, const int* trial_lane) {
    // the trial's settings in shared memory (every thread of the block fills the same trial's records)
    __shared__ dcreg_icp_params P;
    if (lane_prm) {
        const int* from = reinterpret_cast<const int*>(lane_prm + (trial_lane ? trial_lane[blockIdx.y] : blockIdx.y));
        for (int e = threadIdx.x; e < (int)(sizeof(dcreg_icp_params) / sizeof(int)); e += blockDim.x)
            reinterpret_cast<int*>(&P)[e] = from[e];
    } else if (threadIdx.x == 0) {
        P = prm;
    }
    __syncthreads();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const IcpState* st = states + blockIdx.y;
    dcreg_iter_log* log = logs + (size_t)blockIdx.y * log_cap;
    const int n = st->iter < log_cap ? st->iter : log_cap;
    if (i >= n) return;
    if (log[i].status != DCREG_OK) return;
    dcreg_analysis* a = &log[i].analysis;
    const bool ours = P.detection == DCREG_DET_SCHUR_CONDITION_NUMBER && P.handling == DCREG_HAND_PRECONDITIONED_CG;
    int mask[6];
    for (int k = 0; k < 6; ++k) mask[k] = a->degenerate_mask[k];
    const int is_deg = a->is_degenerate, singular = a->schur_singular, pcg_it = a->pcg_iterations;
    const double pcg_res = a->pcg_residual;
    double dx[6];
    k2::analyze_and_solve<true>(log[i].H27, P, a, dx);
    if (ours) {
        for (int k = 0; k < 6; ++k) a->degenerate_mask[k] = mask[k];
        a->is_degenerate = is_deg; a->schur_singular = singular;
        a->pcg_iterations = pcg_it; a->pcg_residual = pcg_res;
    }
}

__global__ void pcg_kernel(const double* A, const double* b, const double* P, int max_it, double tol, double* x,
                           int* iters) {
    if (threadIdx.x != 0) return;
    double res;
    *iters = k2::pcg6(A, b, P, max_it, tol, x, &res);
}

// icp_test_runner.cpp:2014-2037.  One block per trial: st [B], cov [B][36]
__global__ void covariance_kernel(const IcpState* st, double* cov) {
    if (threadIdx.x != 0) return;
    st += blockIdx.x;
    cov += (size_t)blockIdx.x * 36;
    bool ok = false;
    if (st->converged) {
        double A[36], Inv[36];
        for (int i = 0; i < 36; ++i) A[i] = st->H_last[i];
        if (dla::fullpiv_inverse<6>(A, Inv)) {
            ok = true;
            double W[36], lam[6], V[36];
            for (int i = 0; i < 6; ++i)
                for (int j = 0; j < 6; ++j) W[i * 6 + j] = 0.5 * (Inv[i * 6 + j] + Inv[j * 6 + i]);
            dla::jacobi_eigh<6>(W, lam, V);
            if (lam[0] <= 1e-12) {
                for (int i = 0; i < 6; ++i) lam[i] = fmax(lam[i], 1e-9);
                for (int i = 0; i < 6; ++i)
                    for (int j = 0; j < 6; ++j) {
                        double s = 0.0;
                        for (int k = 0; k < 6; ++k) s += V[i * 6 + k] * lam[k] * V[j * 6 + k];
                        cov[i * 6 + j] = s;
                    }
            } else {
                for (int i = 0; i < 36; ++i) cov[i] = Inv[i];
            }
        }
    }
    if (!ok)
        for (int i = 0; i < 36; ++i) cov[i] = (i % 7 == 0) ? 1e6 : 0.0;
}

// Pack host points (`stride` floats each) into float4 with w = the point's index inside its segment, and take each
// segment's max |p| into radius[b] (the lever arm that turns a rotation step into metres; NaN / Inf points count as 0).
// One segment (seg null, n_seg = 1): w is the global index and radius, when given, the max over all points.
__global__ void pack_points_kernel(const float* __restrict__ in, long long n, int stride, const long long* __restrict__ seg,
                                   int n_seg, float4* __restrict__ out, float* __restrict__ radius) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    int b = -1;
    float r = 0.0f;
    if (i < n) {
        b = corr::segment_of(seg, n_seg, i);     // one segment reads no table: seg may be null
        const float x = in[i * stride], y = in[i * stride + 1], z = in[i * stride + 2];
        out[i] = make_float4(x, y, z, __int_as_float((int)(i - (b > 0 ? seg[b] : 0))));
        r = sqrtf(x * x + y * y + z * z);
        if (!(r < 3.0e38f)) r = 0.0f;
    }
    if (radius) {                               // the lanes of a warp that hold points of the same segment reduce together
        const unsigned peers = __match_any_sync(0xffffffffu, b);
        const unsigned rmax = __reduce_max_sync(peers, __float_as_uint(r));  // r >= 0: the bits order like the values
        if (b >= 0 && (int)(threadIdx.x & 31) == __ffs(peers) - 1 && rmax > 0u)
            atomicMax(reinterpret_cast<unsigned int*>(radius + b), rmax);
    }
}

// Key of the scans' spatial sort (sort_sources) of packed points: (scan b, target cell of fl32(T_b p)) with
// T_b = T[16 b ..], and the point's index as the value.  A stable sort on that key orders each segment exactly as
// sort_source_by_cell orders the scan alone: by cell, then index.  Against the context's grid g the key is
// b * ncells + cell.  grids (scan/target pairs, dcreg_icp_run_pairs): scan b's cell is taken in its own target's grid
// grids[b], and the key is that cell's global id in the grid arena, cell_off[b] + cell (the pairs' cell ranges follow
// each other in pair order, so the key still sorts by scan first); g and ncells are then unused.
__global__ void cell_key_kernel(const float4* __restrict__ pts, long long n, const long long* __restrict__ seg, int n_seg,
                                const double* __restrict__ T, corr::Grid g, long long ncells,
                                const corr::Grid* __restrict__ grids, const int* __restrict__ cell_off,
                                unsigned long long* __restrict__ keys, int* __restrict__ vals) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int b = corr::segment_of(seg, n_seg, i);
    const float4 p = pts[i];
    if (grids) keys[i] = (unsigned long long)cell_off[b] + (unsigned long long)corr::source_cell(grids[b], T + (size_t)b * 16, p);
    else keys[i] = (unsigned long long)b * (unsigned long long)ncells + (unsigned long long)corr::source_cell(g, T + (size_t)b * 16, p);
    vals[i] = (int)i;
}

// Keys of the spatial sort against a sparse row index (sort_by_sparse_cell), whose box is too large for one cell id:
// the cell (x, y, z) of fl32(T_b p) unclamped, in two stable passes.  Pass 0: key (y, x) of point i = j.  Pass 1: key
// (segment b, z) of point i = order[j], the order pass 0 left.  Signed coordinates are flipped into unsigned order.
__global__ void sparse_source_key_kernel(const float4* __restrict__ pts, long long n, const long long* __restrict__ seg,
                                         int n_seg, const double* __restrict__ T, double inv_cell, int pass,
                                         const int* __restrict__ order, unsigned long long* __restrict__ keys,
                                         int* __restrict__ vals) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const long long i = pass ? order[j] : j;
    const int b = corr::segment_of(seg, n_seg, i);
    const double* Tb = T + (size_t)b * 16;
    const float4 p = pts[i];
    const double px = p.x, py = p.y, pz = p.z;
    if (pass == 0) {
        const float qx = (float)(Tb[0] * px + Tb[1] * py + Tb[2] * pz + Tb[3]);
        const float qy = (float)(Tb[4] * px + Tb[5] * py + Tb[6] * pz + Tb[7]);
        keys[j] = ((unsigned long long)((unsigned)corr::cell_coord(qy, inv_cell) ^ 0x80000000u) << 32) |
                  (unsigned long long)((unsigned)corr::cell_coord(qx, inv_cell) ^ 0x80000000u);
    } else {
        const float qz = (float)(Tb[8] * px + Tb[9] * py + Tb[10] * pz + Tb[11]);
        keys[j] = ((unsigned long long)b << 32) | (unsigned long long)((unsigned)corr::cell_coord(qz, inv_cell) ^ 0x80000000u);
    }
    vals[j] = (int)i;
}

__global__ void gather_points_kernel(const float4* __restrict__ in, const int* __restrict__ idx, long long n,
                                     float4* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = in[idx[i]];
}

__global__ void planes_to_f32_kernel(const double4* __restrict__ in, long long n, float4* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double4 v = in[i];
    out[i] = make_float4((float)v.x, (float)v.y, (float)v.z, (float)v.w);
}

__global__ void flush_l2_kernel(float4* buf, long long n, float v) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        buf[i] = make_float4(v, v, v, v);
}

// one thread per trial: T = [n_trials][16] row-major 4x4 initial poses.  seg (a batch of scans, Iter2Args::seg): trial b
// has seg[b+1] - seg[b] source points instead of n_total.  running: the start value of n_active (trials, or lanes)
__global__ void init_state_kernel(IcpState* states, const double* T, long long n_total, unsigned int* counters, int n_trials,
                                  unsigned int* n_active, const long long* seg, int running) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b == 0 && n_active) *n_active = (unsigned)running;
    if (b >= n_trials) return;
    init_loop_state(states + b, T + (size_t)b * 16, seg ? seg[b + 1] - seg[b] : n_total);
    counters[b] = 0u;
}

// ---- voxel filter (dcreg_voxel_downsample, dcreg_icp_run_odometry_voxel) -------------------------------------------
// n points (`stride` floats each: host layout, or float4) in n_seg clouds, cloud b being points [seg[b], seg[b+1]).
// Point i's voxel is floor((double)p * inv) per axis (corr::cell_coord before the integer conversion); the survivor of a
// voxel is its point of smallest index (with a cap of max_points: its max_points points of smallest index), kept bit for
// bit, and the survivors keep their input order.  Four passes for all clouds at once: hash, flag, exclusive scan, scatter.
constexpr double kVoxelLimit = 1048576.0;   // voxel coordinates must lie in [-2^20, 2^20): the range of corr::pack_key

// Pass 1: cloud b owns the slots [tab[b], tab[b+1]) (a power of two) of the open-addressing table keys / first; point i
// claims its voxel's slot and atomicMin's its index into it (the minimum does not depend on the order threads arrive
// in).  slot_of[i] = the slot, or -1 for a point with a non-finite coordinate (no voxel) or out of range (bad[b] = 1).
__global__ void voxel_hash_kernel(const float* __restrict__ in, long long n, int stride, const long long* __restrict__ seg,
                                  int n_seg, const long long* __restrict__ tab, double inv, unsigned long long* __restrict__ keys,
                                  int* __restrict__ first, long long* __restrict__ slot_of, int* __restrict__ bad) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int b = corr::segment_of(seg, n_seg, i);
    slot_of[i] = -1;
    const float x = in[i * stride], y = in[i * stride + 1], z = in[i * stride + 2];
    if (!isfinite(x) || !isfinite(y) || !isfinite(z)) return;
    const double fx = floor(__dmul_rn((double)x, inv)), fy = floor(__dmul_rn((double)y, inv)),
                 fz = floor(__dmul_rn((double)z, inv));
    if (!(fx >= -kVoxelLimit && fx < kVoxelLimit && fy >= -kVoxelLimit && fy < kVoxelLimit && fz >= -kVoxelLimit &&
          fz < kVoxelLimit)) {
        bad[b] = 1;
        return;
    }
    const unsigned long long key = corr::pack_key((int)fx, (int)fy, (int)fz);
    const long long base = tab[b];
    const unsigned int mask = (unsigned int)(tab[b + 1] - base - 1);
    unsigned int s = corr::hash_key(key) & mask;
    while (true) {
        const unsigned long long prev = atomicCAS(&keys[base + s], corr::kEmptyKey, key);
        if (prev == corr::kEmptyKey || prev == key) break;
        s = (s + 1) & mask;
    }
    atomicMin(&first[base + s], (int)i);
    slot_of[i] = base + s;
}

// Pass 2: keep[i] = 1 iff point i is the first of its voxel; keep[n] = 0 (the scan's total)
__global__ void voxel_flag_kernel(const long long* __restrict__ slot_of, long long n, const int* __restrict__ first,
                                  int* __restrict__ keep) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    const long long s = i < n ? slot_of[i] : -1;
    keep[i] = s >= 0 && first[s] == (int)i;
}

// A cap of max_points > 1 points per voxel (dcreg_voxel_downsample_n) replaces pass 2 by a stable radix sort of the
// points by slot and a flag pass over the sorted order.  The sort's input: key[i] = point i's slot as a uint32, or
// `dropped` (the table's slot count: it sorts last) for a point with none; val[i] = i
__global__ void voxel_sort_keys_kernel(const long long* __restrict__ slot_of, long long n, unsigned int dropped,
                                       unsigned int* __restrict__ key, int* __restrict__ val) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long long s = slot_of[i];
    key[i] = s >= 0 ? (unsigned int)s : dropped;
    val[i] = (int)i;
}

// key / val sorted stably by key, so a voxel's points are one run with their indices ascending: the point at sorted
// position p has rank p - (start of its run) in its voxel, which is below max_points iff p < max_points or the key
// max_points positions back differs.  keep[val[p]] = that for a point with a slot; keep[n] = 0.  n + 1 threads, O(1)
// each whatever a voxel's occupancy.
__global__ void voxel_cap_flag_kernel(const unsigned int* __restrict__ key, const int* __restrict__ val, long long n,
                                      unsigned int dropped, int max_points, int* __restrict__ keep) {
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (p > n) return;
    if (p == n) { keep[n] = 0; return; }
    const unsigned int k = key[p];
    keep[val[p]] = k != dropped && (p < max_points || key[p - max_points] != k);
}

// The capped filter with a minimum point spacing (dcreg_voxel_downsample_spaced, dcreg_set_map_spacing; KISS-ICP's
// AddPoints): over the same sorted key / val, a voxel's point is kept iff fewer than max_points of its voxel are kept
// before it and every kept point q before it has ((px - qx)^2 + (py - qy)^2) + (pz - qz)^2 >= s2, in FP64 from the
// float32 coordinates with one rounding per operation (the prune's arithmetic).  Warp w owns every run that starts in
// sorted positions [32 w, 32 w + 32) and walks it in batches of 32: each lane tests its candidate against the run's
// kept points so far, then the batch settles one kept point per round (ballot, ffs, shuffle of its coordinates to the
// lanes after it), at most max_points rounds per run.  Each run is settled in index order by one warp, so the flags
// are a function of the points alone.  kept_at: scratch of n ints (the sort's consumed input values), run [a, b)
// listing its kept points' input indices at [a, a + kept); keep[n] = 0.  O(run length x max_points) per run.
__global__ void voxel_space_flag_kernel(const float* __restrict__ in, int stride, const unsigned int* __restrict__ key,
                                        const int* __restrict__ val, long long n, unsigned int dropped, int max_points,
                                        double s2, int* __restrict__ kept_at, int* __restrict__ keep) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t == 0) keep[n] = 0;
    const int lane = threadIdx.x & 31;
    const long long w0 = t - lane;
    if (w0 >= n) return;                                         // whole warps: n is the same for every lane
    const long long q0 = w0 + lane;
    unsigned int starts = __ballot_sync(~0u, q0 < n && (q0 == 0 || key[q0 - 1] != key[q0]));
    while (starts) {
        const long long a = w0 + __ffs(starts) - 1;
        starts &= starts - 1;
        const unsigned int k = key[a];
        int n_kept = 0;
        for (long long b = a;; b += 32) {
            const long long p = b + lane;
            const bool in_run = p < n && key[p] == k;
            const unsigned int run = __ballot_sync(~0u, in_run);
            const int i = in_run ? val[p] : 0;
            bool ok = in_run && k != dropped && n_kept < max_points;
            double px = 0.0, py = 0.0, pz = 0.0;
            if (ok) {
                px = (double)in[(long long)i * stride]; py = (double)in[(long long)i * stride + 1];
                pz = (double)in[(long long)i * stride + 2];
                for (int j = 0; j < n_kept && ok; ++j) {
                    const long long q = (long long)kept_at[a + j] * stride;
                    const double dx = __dsub_rn(px, (double)in[q]), dy = __dsub_rn(py, (double)in[q + 1]),
                                 dz = __dsub_rn(pz, (double)in[q + 2]);
                    ok = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)) >= s2;
                }
            }
            unsigned int cand = __ballot_sync(~0u, ok), kept = 0u;
            while (cand && n_kept < max_points) {
                const int l = __ffs(cand) - 1;
                kept |= 1u << l;
                const double lx = __shfl_sync(~0u, px, l), ly = __shfl_sync(~0u, py, l), lz = __shfl_sync(~0u, pz, l);
                if (lane == l) kept_at[a + n_kept] = i;
                ++n_kept;
                if (ok && lane > l) {
                    const double dx = __dsub_rn(px, lx), dy = __dsub_rn(py, ly), dz = __dsub_rn(pz, lz);
                    ok = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)) >= s2;
                }
                cand = __ballot_sync(~0u, ok && lane > l);
            }
            if (in_run) keep[i] = (int)((kept >> lane) & 1u);
            if (run != ~0u) break;                               // the run ends in this batch
            __syncwarp();                                        // this batch's kept_at entries, for the next
        }
    }
}

// Pass 4 (pos: the exclusive scan of keep): kept point i goes to out[pos[i]] (out_stride 3: x y z; 4: x y z and w = its
// index over all kept points, as pack_points_kernel packs one cloud), index[pos[i]] = its index in its own cloud (index
// may be null); out_seg[b] = pos[seg[b]] for b <= n_seg, the kept points' offsets.  max(n, n_seg) + 1 threads.
__global__ void voxel_scatter_kernel(const float* __restrict__ in, long long n, int stride, const long long* __restrict__ seg,
                                     int n_seg, const int* __restrict__ keep, const int* __restrict__ pos,
                                     float* __restrict__ out, int out_stride, long long* __restrict__ index,
                                     long long* __restrict__ out_seg) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= n_seg) out_seg[i] = pos[seg[i]];
    if (i >= n || !keep[i]) return;
    const long long p = pos[i];
    float* o = out + p * out_stride;
    o[0] = in[i * stride]; o[1] = in[i * stride + 1]; o[2] = in[i * stride + 2];
    if (out_stride == 4) o[3] = __int_as_float((int)p);
    if (index) index[p] = i - seg[corr::segment_of(seg, n_seg, i)];
}

// ---- odometry (dcreg_icp_run_odometry, dcreg_odometry_push; odom_plan.hpp) ------------------------------------------
// Frame reference r (odom_plan::Push): r < n_frames is a frame of the call (device index d = r: points in its packed
// frames, pose in states[d]); otherwise retained frame r - n_frames of a session (points in the window buffer, pose the
// row-major 4x4 T_out the call that registered it returned, hist_T[16 (r - n_frames) ..], whose R and t are the bytes
// of that frame's final loop state).  A one-shot call has no retained frame: its hist_T and window are null.
__device__ __forceinline__ void ref_pose(int r, int n_frames, const IcpState* __restrict__ states,
                                         const double* __restrict__ hist_T, double* R, double* t) {
    if (r < n_frames) {
        const IcpState* st = states + r;
#pragma unroll
        for (int i = 0; i < 9; ++i) R[i] = st->R[i];
#pragma unroll
        for (int i = 0; i < 3; ++i) t[i] = st->t[i];
    } else {
        const double* T = hist_T + (size_t)(r - n_frames) * 16;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
#pragma unroll
            for (int b = 0; b < 3; ++b) R[3 * a + b] = T[4 * a + b];
            t[a] = T[4 * a + 3];
        }
    }
}

// The maps of one step, or the input of one voxel-map update (odom_plan::MapInput): m points in all, piece p being map
// points [dst[p], dst[p+1]) = the points src_at[p] .. of frame reference r = frame[p]: an old voxel map copied from `old`
// (r < 0), or a frame's packed input (input order) under its final pose (ref_pose).  Every transformed coordinate is
// ((r0 x + r1 y) + r2 z) + t in FP64, one rounding per operation, then one float32 rounding (dcreg_b200.api.map_points
// gives the same bits); w = the point's index over the maps, as a packed target.
__global__ void map_points_kernel(const float4* __restrict__ src, const float4* __restrict__ win,
                                  const float4* __restrict__ old, int n_frames, const long long* __restrict__ dst,
                                  int pieces, const long long* __restrict__ src_at, const int* __restrict__ frame,
                                  long long m, const IcpState* __restrict__ states, const double* __restrict__ hist_T,
                                  float4* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const int p = corr::segment_of(dst, pieces, i);
    const int r = frame[p];
    const long long at = src_at[p] + (i - dst[p]);
    if (r < 0) {
        const float4 q = old[at];
        out[i] = make_float4(q.x, q.y, q.z, __int_as_float((int)i));
        return;
    }
    double R[9], t[3];
    ref_pose(r, n_frames, states, hist_T, R, t);
    const float4 q = (r < n_frames ? src : win)[at];
    const double x = q.x, y = q.y, z = q.z;
    float v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c)
        v[c] = (float)__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(R[3 * c], x), __dmul_rn(R[3 * c + 1], y)),
                                          __dmul_rn(R[3 * c + 2], z)),
                                t[c]);
    out[i] = make_float4(v[0], v[1], v[2], __int_as_float((int)i));
}

// Accelerometer input (dcreg_icp_run_odometry_imu): device frame d's (start, span, tm, tm_prev) ft[4 d ..] and its
// (alpha, beta, gamma) abg[9 d ..] (odom_gyro_kernel), every frame reference r's velocity v[3 r ..] (world frame; a
// step's velocity kernel writes its frames'), gravity in the world frame.  v null: gyro input alone.
struct OdomImu {
    const double* ft = nullptr;
    const double* abg = nullptr;
    double* v = nullptr;
    double gravity[3] = {0.0, 0.0, 0.0};
};

// The increment D lane j's prior is composed with: delta[prev[j]] (null: identity), or with constant velocity the
// increment from frame k-2 to frame k-1 (identity after the anchor); the identity for a first frame (prev[j] < 0).  The start kernel and odom_twist_kernel both take
// it from here, so the deskew twist is the increment the prior used, bit for bit.
__device__ __forceinline__ void odom_increment(int j, const IcpState* __restrict__ states, const int* __restrict__ prev,
                                               const int* __restrict__ prev2, const double* __restrict__ delta, int motion,
                                               int n_frames, const double* __restrict__ hist_T, double* D) {
    for (int i = 0; i < 16; ++i) D[i] = (i % 5 == 0) ? 1.0 : 0.0;
    if (motion == DCREG_MOTION_CONSTANT_VELOCITY) {
        if (prev2[j] >= 0) {
            double Ra[9], ta[3], Rb[9], tb[3];
            ref_pose(prev[j], n_frames, states, hist_T, Ra, ta);
            ref_pose(prev2[j], n_frames, states, hist_T, Rb, tb);
            constant_velocity_increment(Rb, tb, Ra, ta, D);
        }
    } else if (delta && prev[j] >= 0) {
        for (int i = 0; i < 16; ++i) D[i] = delta[(size_t)prev[j] * 16 + i];
    }
}

// Start of step `step_first` (one thread per lane of `lanes`): lane j < active runs frame step_first + j and nothing
// after it (its frame range is that one frame, so the frame advance ends the lane), the other lanes run nothing.  The
// frame's prior is compose_prior(frame prev[j]'s pose, odom_increment); delta holds one entry per frame reference, or is
// null.  kGyro (odom_start_gyro_kernel): the increment's rotation is the frame's gyro rotation G[9 f ..] instead, and
// with tD the increment's translation goes to tD[3 j ..] and the frame's lever arm is zeroed, for
// odom_deskew_gyro_kernel.  With accelerometer input (imu.v not null) the increment's translation is
// se3::imu_translation's instead, from frame prev[j]'s pose and velocity and the frame's beta.  (prior map) A lane whose
// prev[j] < 0 runs its sequence's first frame from the state and prior start_loop gave it, T_init: only its frame range
// is set.
template <bool kGyro>
__device__ __forceinline__ void odom_start(IcpState* states, const long long* __restrict__ seg, double* T_prior,
                                           int* cursor, int* first, unsigned int* n_active, int lanes, int step_first,
                                           int active, const int* __restrict__ prev, const int* __restrict__ prev2,
                                           const double* __restrict__ delta, int motion, int n_frames,
                                           const double* __restrict__ hist_T, const double* __restrict__ G,
                                           double* __restrict__ tD, float* __restrict__ radius,
                                           const OdomImu& imu) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j == 0) { *n_active = (unsigned)active; first[lanes] = step_first + active; }
    if (j >= lanes) return;
    const int f = step_first + min(j, active);
    first[j] = f; cursor[j] = f;
    if (j >= active || prev[j] < 0) return;
    double D[16], Ra[9], ta[3];
    odom_increment(j, states, prev, prev2, delta, motion, n_frames, hist_T, D);
    ref_pose(prev[j], n_frames, states, hist_T, Ra, ta);
    if (kGyro) {
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) D[4 * r + c] = G[(size_t)f * 9 + 3 * r + c];
        if (imu.v) {
            const double* ft = imu.ft + 4 * (size_t)f;
            double t[3];
            se3::imu_translation(Ra, imu.v + 3 * (size_t)prev[j], imu.gravity, imu.abg + 9 * (size_t)f + 3,
                                 __dsub_rn(ft[2], ft[3]), t);
            for (int r = 0; r < 3; ++r) D[4 * r + 3] = t[r];
        }
        if (tD) {
            for (int r = 0; r < 3; ++r) tD[3 * (size_t)j + r] = D[4 * r + 3];
            radius[f] = 0.0f;
        }
    }
    double T[16];
    compose_prior(Ra, ta, D, T);
    for (int i = 0; i < 16; ++i) T_prior[(size_t)f * 16 + i] = T[i];
    init_loop_state(states + f, T, seg[f + 1] - seg[f]);
}

__global__ void odom_start_kernel(IcpState* states, const long long* __restrict__ seg, double* T_prior, int* cursor,
                                  int* first, unsigned int* n_active, int lanes, int step_first, int active,
                                  const int* __restrict__ prev, const int* __restrict__ prev2,
                                  const double* __restrict__ delta, int motion, int n_frames,
                                  const double* __restrict__ hist_T) {
    odom_start<false>(states, seg, T_prior, cursor, first, n_active, lanes, step_first, active, prev, prev2, delta,
                      motion, n_frames, hist_T, nullptr, nullptr, nullptr, OdomImu{});
}

__global__ void odom_start_gyro_kernel(IcpState* states, const long long* __restrict__ seg, double* T_prior, int* cursor,
                                       int* first, unsigned int* n_active, int lanes, int step_first, int active,
                                       const int* __restrict__ prev, const int* __restrict__ prev2, int n_frames,
                                       const double* __restrict__ hist_T, const double* __restrict__ G,
                                       double* __restrict__ tD, float* __restrict__ radius, OdomImu imu) {
    odom_start<true>(states, seg, T_prior, cursor, first, n_active, lanes, step_first, active, prev, prev2, nullptr,
                     DCREG_MOTION_CONSTANT_VELOCITY, n_frames, hist_T, G, tD, radius, imu);
}

// The session's window after a push: m points in `pieces` retained frames, piece p being out[dst[p], dst[p+1]) = the
// packed points (src_at[p] ..) of the push (ref[p] < n_frames) or of the old window.  One launch for every sequence.
__global__ void retain_points_kernel(const float4* __restrict__ src, const float4* __restrict__ win, int n_frames,
                                     const long long* __restrict__ dst, int pieces, const long long* __restrict__ src_at,
                                     const int* __restrict__ ref, long long m, float4* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const int p = corr::segment_of(dst, pieces, i);
    out[i] = (ref[p] < n_frames ? src : win)[src_at[p] + (i - dst[p])];
}

// ---- the voxel map (dcreg_icp_run_odometry_map, dcreg_odometry_open_map; odom_plan::map_step) ----------------------
// The voxel map's prune, between the voxel filter's flag pass and its scan (KISS-ICP's RemovePointsFarFromLocation): a
// kept point i whose voxel's first point q (first[slot_of[i]], the voxel's smallest index) has ((qx - tx)^2 + (qy -
// ty)^2) + (qz - tz)^2 >= max_d2 is dropped, in FP64 from the float32 coordinates with one rounding per operation.  t:
// the translation of frame reference center[b] (ref_pose's rule) for segment b.  O(1) per point: every point of a
// voxel reads the same first point, so a voxel goes or stays whole.
__global__ void voxel_prune_kernel(const float* __restrict__ in, long long n, int stride, const long long* __restrict__ seg,
                                   int n_seg, const long long* __restrict__ slot_of, const int* __restrict__ first,
                                   const int* __restrict__ center, int n_frames, const IcpState* __restrict__ states,
                                   const double* __restrict__ hist_T, double max_d2, int* __restrict__ keep) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !keep[i]) return;
    const int r = center[corr::segment_of(seg, n_seg, i)];
    double t[3];
    if (r < n_frames) {
        for (int c = 0; c < 3; ++c) t[c] = states[r].t[c];
    } else {
        for (int c = 0; c < 3; ++c) t[c] = hist_T[(size_t)(r - n_frames) * 16 + 4 * c + 3];
    }
    const long long q = first[slot_of[i]];
    const double dx = __dsub_rn((double)in[q * stride], t[0]), dy = __dsub_rn((double)in[q * stride + 1], t[1]),
                 dz = __dsub_rn((double)in[q * stride + 2], t[2]);
    if (__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)) >= max_d2) keep[i] = 0;
}

// ---- motion compensation (dcreg_icp_run_odometry_deskew, dcreg_odometry_push_deskew; se3.cuh) ---------------------
// Once per call: ts[i] = the timestamp of packed point i (device order, segments seg[n_seg + 1]) from the caller's
// timestamps ts_in.  Device frame b is the caller's frame whose input points start at in_at[b]; its point j is input
// point j of that frame, or, after the source filter (index: d_vox_index), the input point index[kept_at[b] + j].
__global__ void odom_ts_gather_kernel(const float* __restrict__ ts_in, long long n, const long long* __restrict__ seg,
                                      int n_seg, const long long* __restrict__ in_at, const long long* __restrict__ kept_at,
                                      const long long* __restrict__ index, float* __restrict__ ts) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int b = corr::segment_of(seg, n_seg, i);
    const long long j = i - seg[b];
    ts[i] = ts_in[in_at[b] + (index ? index[kept_at[b] + j] : j)];
}

// Per step, after the start kernel (one thread per lane j < active): xi[6 j ..] = Log(D) of the lane's increment, and
// the lever arm of its frame step_first + j zeroed for odom_deskew_kernel to take again
__global__ void odom_twist_kernel(const IcpState* __restrict__ states, int step_first, int active,
                                  const int* __restrict__ prev, const int* __restrict__ prev2,
                                  const double* __restrict__ delta, int motion, int n_frames,
                                  const double* __restrict__ hist_T, double* __restrict__ xi, float* __restrict__ radius) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= active) return;
    double D[16];
    odom_increment(j, states, prev, prev2, delta, motion, n_frames, hist_T, D);
    const double R[9] = {D[0], D[1], D[2], D[4], D[5], D[6], D[8], D[9], D[10]}, t[3] = {D[3], D[7], D[11]};
    se3::se3_log(R, t, xi + 6 * (size_t)j);
    radius[step_first + j] = 0.0f;
}

// Per step: the step's frames [step_first, step_first + active), points [base, base + n) of the packed (src) and the
// sorted copy, deskewed in place by se3::deskew_point with their lane's twist.  A packed point's timestamp is ts[i]; a
// sorted point's is that of its index in the frame (.w).  A point that does not move is not written.  The frame's lever
// arm is taken again from the deskewed packed points with pack_points_kernel's rule.  kSource = false (the map-input
// points of dcreg_set_map_input_voxel, segments seg): the packed points alone, no sorted copy, no lever arm.
template <bool kSource>
__global__ void odom_deskew_kernel(float4* __restrict__ src, float4* __restrict__ sorted, const long long* __restrict__ seg,
                                   int step_first, int active, long long base, long long n, const float* __restrict__ ts,
                                   const double* __restrict__ xi, float* __restrict__ radius) {
    const long long i = base + (long long)blockIdx.x * blockDim.x + threadIdx.x;
    int b = -1;
    float r = 0.0f;
    if (i < base + n) {
        const int j = corr::segment_of(seg + step_first, active, i);
        b = step_first + j;
        const double* x = xi + 6 * (size_t)j;
        float o[3];
        float4 p = src[i];
        const float pi[3] = {p.x, p.y, p.z};
        if (se3::deskew_point(x, ts[i], pi, o)) {
            p.x = o[0]; p.y = o[1]; p.z = o[2];
            src[i] = p;
        }
        if (!kSource) return;
        float4 q = sorted[i];
        const float qi[3] = {q.x, q.y, q.z};
        if (se3::deskew_point(x, ts[seg[b] + __float_as_int(q.w)], qi, o)) {
            q.x = o[0]; q.y = o[1]; q.z = o[2];
            sorted[i] = q;
        }
        const float px = p.x, py = p.y, pz = p.z;
        r = sqrtf(px * px + py * py + pz * pz);
        if (!(r < 3.0e38f)) r = 0.0f;
    }
    if (!kSource) return;
    const unsigned peers = __match_any_sync(0xffffffffu, b);
    const unsigned rmax = __reduce_max_sync(peers, __float_as_uint(r));
    if (b >= 0 && (int)(threadIdx.x & 31) == __ffs(peers) - 1 && rmax > 0u)
        atomicMax(reinterpret_cast<unsigned int*>(radius + b), rmax);
}

// ---- gyroscope input (dcreg_icp_run_odometry_gyro, dcreg_odometry_push_gyro; se3.cuh) -----------------------------
// Device frame d's sweep: ft[4 d ..] = (start, span, tm, tm_prev), tm = start + 0.5 span its mid-sweep time and tm_prev
// the previous frame's; its sequence's samples are rows [range[2 d], range[2 d + 1]) of smp; its knot table is knots
// [kKnotStride knot_off[d] ..], empty for an anchor.
//
// Once per call, before the steps (one thread per device frame; the poses play no part): every non-anchor frame's
// G(tm_prev -> tm), the rotation of its prior's increment, into G[9 d ..], and its sweep's knot table; samples `stride`
// doubles a row.  With abg (IMU samples) the same walk's (alpha, beta, gamma) into abg[9 d ..], the specific force less
// acc_bias.
struct AccelBias { double b[3]; };
__global__ void odom_gyro_kernel(se3::Gyro g, int stride, AccelBias acc, const double* __restrict__ smp,
                                 const double* __restrict__ ft, const long long* __restrict__ range,
                                 const long long* __restrict__ knot_off, int n_frames, double* __restrict__ G,
                                 double* __restrict__ abg, double* __restrict__ knots) {
    const int d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= n_frames || knot_off[d + 1] == knot_off[d]) return;
    const double* s = smp + (size_t)range[2 * d] * stride;
    const long long n = range[2 * d + 1] - range[2 * d];
    const double* f = ft + 4 * (size_t)d;
    se3::gyro_rotation(g, s, n, f[3], f[2], G + 9 * (size_t)d, stride, abg ? acc.b : nullptr,
                       abg ? abg + 9 * (size_t)d : nullptr);
    se3::gyro_knots(g, s, n, f[0], f[2], __dadd_rn(f[0], f[1]), knots + (size_t)knot_off[d] * se3::kKnotStride, stride);
}

// (IMU) Per step, after its loop has ended (one thread per lane j < active): the velocity of the lane's frame
// step_first + j, which has stopped, from its pose and frame prev[j]'s (se3::imu_velocity).  A sequence's first frame
// (prior map: prev[j] < 0) keeps the velocity it was given.
__global__ void odom_velocity_kernel(const IcpState* __restrict__ states, int step_first, int active,
                                     const int* __restrict__ prev, int n_frames, const double* __restrict__ hist_T,
                                     OdomImu imu) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= active || prev[j] < 0) return;
    const int f = step_first + j;
    double Ra[9], ta[3], R[9], t[3];
    ref_pose(prev[j], n_frames, states, hist_T, Ra, ta);
    ref_pose(f, n_frames, states, hist_T, R, t);
    const double* ft = imu.ft + 4 * (size_t)f;
    se3::imu_velocity(Ra, ta, t, imu.gravity, imu.abg + 9 * (size_t)f + 6, __dsub_rn(ft[2], ft[3]), imu.v + 3 * (size_t)f);
}

// Per step, after odom_start_gyro_kernel: odom_deskew_kernel with se3::deskew_point_gyro, the lane's increment
// translation tD[3 j ..] and its frame's knot table; the lever arm is taken again the same way (kSource as there).  A
// frame without knots (prior map: a sequence's first frame) is left as it is.
template <bool kSource>
__global__ void odom_deskew_gyro_kernel(float4* __restrict__ src, float4* __restrict__ sorted,
                                        const long long* __restrict__ seg, int step_first, int active, long long base,
                                        long long n, const float* __restrict__ ts, const double* __restrict__ ft,
                                        const long long* __restrict__ knot_off, const double* __restrict__ knots,
                                        const double* __restrict__ tD, float* __restrict__ radius) {
    const long long i = base + (long long)blockIdx.x * blockDim.x + threadIdx.x;
    int b = -1;
    float r = 0.0f;
    if (i < base + n) {
        const int j = corr::segment_of(seg + step_first, active, i);
        b = step_first + j;
        const double* f = ft + 4 * (size_t)b;
        const double* K = knots + (size_t)knot_off[b] * se3::kKnotStride;
        const int nk = (int)(knot_off[b + 1] - knot_off[b]);
        const double* t = tD + 3 * (size_t)j;
        float o[3];
        float4 p = src[i];
        const float pi[3] = {p.x, p.y, p.z};
        if (nk > 0 && se3::deskew_point_gyro(K, nk, f[0], f[1], f[2], f[3], t, ts[i], pi, o)) {
            p.x = o[0]; p.y = o[1]; p.z = o[2];
            src[i] = p;
        }
        if (!kSource) return;
        float4 q = sorted[i];
        const float qi[3] = {q.x, q.y, q.z};
        if (nk > 0 && se3::deskew_point_gyro(K, nk, f[0], f[1], f[2], f[3], t, ts[seg[b] + __float_as_int(q.w)], qi, o)) {
            q.x = o[0]; q.y = o[1]; q.z = o[2];
            sorted[i] = q;
        }
        const float px = p.x, py = p.y, pz = p.z;
        r = sqrtf(px * px + py * py + pz * pz);
        if (!(r < 3.0e38f)) r = 0.0f;
    }
    if (!kSource) return;
    const unsigned peers = __match_any_sync(0xffffffffu, b);
    const unsigned rmax = __reduce_max_sync(peers, __float_as_uint(r));
    if (b >= 0 && (int)(threadIdx.x & 31) == __ffs(peers) - 1 && rmax > 0u)
        atomicMax(reinterpret_cast<unsigned int*>(radius + b), rmax);
}

// ---- the adaptive threshold (dcreg_icp_run_odometry_adaptive; adaptive_threshold.cuh) -----------------------------
// Per step, after its loop has ended (one thread per lane j < active): the lane's frame step_first + j, which has
// stopped, is folded into its sequence's state, state[seq[j]], with the correction inv(T_prior) T_out, and the
// sequence's next radius goes to lane_radius[next_lane[j]], the lane that runs the sequence at the next step (-1: none).
// The lanes of a step keep their order into the next one, so next_lane[j] <= j is written by one thread and read by
// none here.  (prior map) seq[j] < 0: the lane ran sequence ~seq[j]'s first frame, whose prior was the caller's guess,
// not a prediction; its state is not folded.
__global__ void odom_threshold_kernel(const IcpState* __restrict__ states, const double* __restrict__ T_prior,
                                      int step_first, int active, const int* __restrict__ seq,
                                      const int* __restrict__ next_lane, adaptive::Settings set, double ceiling,
                                      adaptive::State* __restrict__ state, double* lane_radius) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= active) return;
    const IcpState* st = states + step_first + j;
    const double* P = T_prior + (size_t)(step_first + j) * 16;
    const double Ra[9] = {P[0], P[1], P[2], P[4], P[5], P[6], P[8], P[9], P[10]}, ta[3] = {P[3], P[7], P[11]};
    double D[16];
    constant_velocity_increment(Ra, ta, st->R, st->t, D);
    const int s = seq[j] < 0 ? ~seq[j] : seq[j];
    adaptive::State x = state[s];
    if (seq[j] >= 0) {
        adaptive::fold(&x, adaptive::model_error(D, set.max_range), set.min_motion);
        state[s] = x;
    }
    if (next_lane[j] >= 0) lane_radius[next_lane[j]] = adaptive::radius(x, set.initial_threshold, ceiling);
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// NCCL through dlopen (so the library loads without it; torch's bundled copy is reused when present)
// ------------------------------------------------------------------------------------------------
namespace {
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
struct NcclApi {
    void* lib = nullptr;
    int (*GetUniqueId)(ncclUniqueId*) = nullptr;
    int (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    int (*CommDestroy)(ncclComm_t) = nullptr;
    int (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    bool load(std::string& err) {
        if (lib) return true;
        const char* names[] = {"libnccl.so.2", "libnccl.so"};
        for (const char* nm : names) {
            lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
            if (lib) break;
        }
        if (!lib) { err = std::string("dlopen libnccl failed: ") + dlerror(); return false; }
        GetUniqueId = (int (*)(ncclUniqueId*))dlsym(lib, "ncclGetUniqueId");
        CommInitRank = (int (*)(ncclComm_t*, int, ncclUniqueId, int))dlsym(lib, "ncclCommInitRank");
        CommDestroy = (int (*)(ncclComm_t))dlsym(lib, "ncclCommDestroy");
        AllReduce = (int (*)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t))dlsym(lib, "ncclAllReduce");
        AllGather = (int (*)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t))dlsym(lib, "ncclAllGather");
        GetErrorString = (const char* (*)(int))dlsym(lib, "ncclGetErrorString");
        if (!GetUniqueId || !CommInitRank || !CommDestroy || !AllReduce) { err = "libnccl: missing symbols"; return false; }
        return true;
    }
};
NcclApi g_nccl;
constexpr int kNcclFloat64 = 8;   // ncclDouble
constexpr int kNcclInt8 = 0;      // ncclInt8 / ncclChar
constexpr int kNcclSum = 0;
}  // namespace

// ------------------------------------------------------------------------------------------------
// context
// ------------------------------------------------------------------------------------------------
// A grow-only allocation with one owner: ensure(n) reallocates, at exactly n elements, only when the capacity is below
// n (the old contents are lost), and the destructor frees it; grow(n) reallocates with a quarter of headroom, for sizes
// that follow results.  kPinned: page-locked host memory.
template <typename T, bool kPinned = false>
struct DevBuf {
    T* p = nullptr;
    long long cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { release(); }
    operator T*() const { return p; }
    void release() {
        if (p) {
            if (kPinned) cudaFreeHost(p);
            else cudaFree(p);
        }
        p = nullptr; cap = 0;
    }
    cudaError_t ensure(long long n) {
        if (cap >= n) return cudaSuccess;
        release();
        void* q = nullptr;
        const cudaError_t e = kPinned ? cudaMallocHost(&q, (size_t)n * sizeof(T)) : cudaMalloc(&q, (size_t)n * sizeof(T));
        if (e == cudaSuccess) { p = (T*)q; cap = n; }
        return e;
    }
    cudaError_t grow(long long n) { return cap >= n ? cudaSuccess : ensure(n + n / 4); }
};
template <typename T>
using PinnedBuf = DevBuf<T, true>;

// The settings of scan-to-map odometry: a one-shot call's, or those dcreg_odometry_open gives every push of a session
struct OdomSettings {
    dcreg_icp_params params{};
    int n_seqs = 0, map_frames = 1, motion = 0, source_max_points = 1, map_max_points = 1;
    double cell_size = 0.0, source_voxel = 0.0, map_voxel = 0.0;
    std::vector<double> T_init;                                        // [n_seqs][16]
    // the voxel map (dcreg_icp_run_odometry_map, dcreg_odometry_open_map) instead of the window (map_frames unused):
    // every sequence's map carried from frame to frame, pruned at max_distance (+inf: never)
    bool voxel_map = false;
    double max_distance = 0.0;
    // the adaptive threshold (dcreg_icp_run_odometry_adaptive, dcreg_odometry_open_adaptive): every frame's search radius
    // follows its sequence's motion-model error, under the ceiling params.search_radius
    bool adaptive = false;
    adaptive::Settings threshold{};
    // gyroscope input (dcreg_icp_run_odometry_gyro, dcreg_odometry_open_gyro): every non-anchor frame's prior rotation
    // and deskew rotation come from integrated gyro rates
    bool gyro = false;
    se3::Gyro gyro_set{};
    // accelerometer input (dcreg_icp_run_odometry_imu, dcreg_odometry_open_imu; gyro is set too): every non-anchor
    // frame's prior translation from the previous frame's velocity and the preintegrated specific force (IMU samples:
    // se3::kImuStride doubles a row).  v_init [n_seqs][3]: the velocity of every sequence's first frame
    bool imu = false;
    double accel_bias[3] = {0.0, 0.0, 0.0}, gravity[3] = {0.0, 0.0, 0.0};
    std::vector<double> v_init;
    // (a session) dcreg_set_sparse_maps and dcreg_set_map_spacing as they were at open; a one-shot call reads the
    // context's
    bool sparse_maps = false;
    double map_spacing = 0.0;
    // dcreg_set_map_input_voxel (at open, for a session; at the call for the filtered one-shot calls; 0 for
    // dcreg_icp_run_odometry): the frames enter the maps as F_in(frame), and register with F_s(F_in(frame))
    double map_input_voxel = 0.0;
    // dcreg_set_lane_params on (at open, for a session): every sequence's settings [n_seqs], params being entry 0; off:
    // empty
    std::vector<dcreg_icp_params> lanes;
    // (a session) dcreg_set_prior_map as it was at open; a one-shot call reads the context's
    bool prior_map = false;
};

struct dcreg_ctx {
    int device = 0;
    int sm_count = 132;
    cudaStream_t stream = nullptr;
    std::string err;
    long long launches = 0;

    DevBuf<float4> d_src; long long n_src = 0; long long n_src_total = 0;
    DevBuf<float> d_stage;                                                 // host point uploads before packing

    DevBuf<float4> d_tgt; long long n_tgt = 0;                             // exactly n_tgt: every set_target reallocates it
    corr::Grid grid{}; long long grid_cells = 0; bool has_grid = false;
    DevBuf<double4> d_plane_cache; DevBuf<signed char> d_fit_state;        // plane of the slot's current five neighbours
    DevBuf<int> d_plane_key;                                               // ... and which five (ascending positions)
    bool force_coherent = false;                                           // profiling (dcreg_time_iteration what = 0)
    DevBuf<float> d_src_radius;                                            // max |p| over the source cloud (device)
    DevBuf<unsigned int> d_iter_stats;                                     // profiling counters of the iteration kernel (while enabled)
    DevBuf<int4> d_nn; bool nn_valid = false;                              // neighbours of the sorted source (seeds of the next iteration)
    long long nn_slots = 0; int nn_trials = 0;                             // shape of the per-slot records (d_nn, d_plane_cache, ...)
    DevBuf<float4> d_src_sorted;                                           // source in target-cell order (w = original index)
    DevBuf<float4> d_sort_tmp;                                             // ... before the in-cell ranking
    DevBuf<int> d_cell_tmp;                                                // counts / fill cursors for the source sort
    DevBuf<int> d_pt_cell;
    DevBuf<int> d_tile_sums;
    double cell_size = 0.0;

    DevBuf<double4> d_planes64; DevBuf<float4> d_planes32;

    // per-trial arrays (dcreg_icp_run = 1 trial, dcreg_icp_run_batch = many)
    DevBuf<double> d_partials;            // [blocks][kPartialDoubles]
    DevBuf<unsigned int> d_counter;
    DevBuf<double> d_acc;
    DevBuf<IcpState> d_state;
    DevBuf<unsigned int> d_n_active;      // trials still running
    DevBuf<double> d_T_init;
    DevBuf<dcreg_iter_log> d_log;         // records, [trials][log_cap of the run]
    bool loop_attr_done = false, k1_attr_done[4] = {};     // k1: one per kReduceKernels entry
    // CUDA graphs of one chunk of loop iterations, keyed on the kernel arguments (a few shapes alternate in practice:
    // with / without a log, one trial / a batch); most recently used first
    struct LoopGraph { std::vector<unsigned char> key; cudaGraphExec_t exec; };
    std::vector<LoopGraph> graphs; bool graph_off = false;
    long long graph_launches = 0;
    void drop_graphs() { for (auto& g : graphs) if (g.exec) cudaGraphExecDestroy(g.exec); graphs.clear(); }
    DevBuf<double> d_small;              // scratch for the seams (1024 doubles)
    DevBuf<K2Scratch> d_k2_scratch;      // K2's rehearsal state (see k2_step_kernel)
    // solver block of a single-trial folded run (solver_block): row flags, launch counter, warm-up state.  The counter
    // and the flags are never reset, so no flag written by an earlier launch can match a later one
    DevBuf<unsigned long long> d_row_flags;
    DevBuf<unsigned long long> d_row_epoch;
    DevBuf<IcpState> d_warm_state;
    // the sources of a batched call (dcreg_icp_run_scans, _pairs, _sequences, _odometry) in buffers of their own: the
    // context's source stays as it was.  [points] packed / in sort order, [2][points] sort keys and values in / out,
    // [sources + 1] offsets, [sources] lever arms and covariances
    DevBuf<float4> d_scan_src, d_scan_sorted;
    DevBuf<unsigned long long> d_scan_keys; DevBuf<int> d_scan_vals;
    DevBuf<unsigned char> d_scan_sort_tmp;
    DevBuf<long long> d_scan_seg; DevBuf<float> d_scan_radius; DevBuf<double> d_scan_cov;
    // sequences of frames (dcreg_icp_run_sequences, _odometry; the frames are the batch's sources): lane cursors and
    // frame ranges [lanes] / [lanes + 1], increments and priors [frames][16]
    DevBuf<int> d_seq_cursor, d_seq_first;
    DevBuf<double> d_seq_delta, d_seq_prior;
    // odometry (dcreg_icp_run_odometry): every step's tables (odom_plan.hpp) in one upload, the step's local maps (or a
    // voxel-map update's input), and their grids in an arena of their own
    DevBuf<long long> d_odom_ll; DevBuf<int> d_odom_int;
    DevBuf<float4> d_odom_map;
    // the voxel map: one update's tables (odom_plan::MapInput), uploaded per update.  The maps after the voxel filter:
    // a window's in d_vmap[0], the voxel map's updates in turns (an update reads the previous one's output)
    DevBuf<long long> d_vmap_ll; DevBuf<int> d_vmap_int;
    DevBuf<float4> d_vmap[2];
    // motion compensation (dcreg_icp_run_odometry_deskew): the caller's timestamps [input points], the packed points'
    // [points], and the step's twists [lanes][6]
    DevBuf<float> d_odom_ts_in, d_odom_ts;
    DevBuf<double> d_odom_xi;
    // the map-input filter with a source filter after it (dcreg_set_map_input_voxel, voxel_filter_chain): F_in's kept
    // xyz [input points][3] (NaN past the kept ones), their indices in their frames, its kept offsets [n_frames + 1];
    // F_in's points packed in device order, and (timestamps) theirs
    DevBuf<float> d_in_xyz; DevBuf<long long> d_in_index, d_in_seg;
    DevBuf<float4> d_odom_in;
    DevBuf<float> d_odom_ts_map;
    // gyroscope input: the call's samples [rows][4], every device frame's (start, span, tm, tm_prev) [n_frames][4], its
    // prior's rotation [n_frames][9] and the knot tables [knots][16] (odom_gyro_kernel)
    DevBuf<double> d_gyro_smp, d_gyro_ft, d_gyro_G, d_gyro_knots;
    // accelerometer input: every device frame's (alpha, beta, gamma) [n_frames][9], and every frame reference's
    // velocity [n_frames + retained][3] (OdomImu)
    DevBuf<double> d_imu_abg, d_imu_v;
    // the adaptive threshold: every sequence's (sse, n) [n_seqs], and the radii of the coming step's lanes [lanes]
    DevBuf<adaptive::State> d_thr_state;
    DevBuf<double> d_lane_radius;
    // the odometry session (dcreg_odometry_open .. _close), if one is open: the settings of its pushes, and what every
    // sequence carries from one push to the next (odom_plan::History): the retained frames' kept points, packed and in
    // input order as d_scan_src holds them, in win[cur] (the other buffer receives the next push's window), their poses
    // (the T_out the host returned) and the last increment of every sequence
    struct OdomSession {
        OdomSettings set;
        odom_plan::History hist;
        std::vector<double> hist_T;                                    // [retained][16]
        std::vector<double> last_delta;                                // [n_seqs][16]
        DevBuf<float4> win[2]; int cur = 0;
        DevBuf<double> d_hist_T;                                       // hist_T on the device
        // the voxel map (set.voxel_map): win[cur] holds every sequence's map instead of a window, sequence s's being
        // points [map_off[s], map_off[s + 1]), its last frame in it (the push's final update gathers them in win[1 - cur])
        std::vector<long long> map_off;                                // [n_seqs + 1]
        // (set.adaptive) every sequence's threshold state after its last committed frame; a push uploads it
        std::vector<adaptive::State> thr_state;                        // [n_seqs]
        // (set.gyro) every sequence's last committed mid-sweep time (NaN: none yet, or pushed without frame times)
        std::vector<double> last_mid;                                  // [n_seqs]
        // (set.imu) every sequence's last committed velocity (its v_init before its first frame)
        std::vector<double> last_v;                                    // [n_seqs][3]
        // (set.prior_map) every sequence's dead-reckoned pose (T_init and the increments alone) of its last frame, the
        // pose its next frame's points are sorted under
        std::vector<double> dr_T;                                      // [n_seqs][16]
    };
    std::unique_ptr<OdomSession> odom;
    // the voxel filter (voxel_filter): table [slots] keys / first indices, [points] slots, [points + 1] flags and their
    // scan, [clouds + 1] table offsets, input and kept offsets, [clouds] range flags, [points][3] kept xyz and indices
    DevBuf<unsigned long long> d_vox_keys; DevBuf<int> d_vox_first;
    DevBuf<long long> d_vox_slot; DevBuf<int> d_vox_keep, d_vox_pos;
    DevBuf<long long> d_vox_tab, d_vox_in_seg, d_vox_seg; DevBuf<int> d_vox_bad;
    DevBuf<float> d_vox_xyz; DevBuf<long long> d_vox_index;
    // ... and with a cap above one point per voxel: [2][points] sort keys (slots) and values (indices) in / out
    DevBuf<unsigned int> d_vox_skey; DevBuf<int> d_vox_sval;
    DevBuf<unsigned char> d_vox_sort_tmp;
    // Grow-only arenas of dense grids (build_grid_arena) or sparse row indexes (build_sparse_arena): the context's
    // target (one cloud; `grid` points into it), the targets of dcreg_icp_run_pairs (the context's target and grid stay
    // as they were), the grids over the aligned sources of the point-to-point metrics, and odometry's local maps
    struct GridArena {
        DevBuf<float4> pts, tmp; DevBuf<int> pos_of, pt_cell;               // [points]
        DevBuf<int> cell_start, counts, fill;                               // [cells + 1], [cells + 1], [cells]
        DevBuf<corr::Grid> d_grids; DevBuf<int> d_cell_off, d_bounds;       // [clouds], [clouds + 1], [clouds][6]
        // sparse row indexes instead (build_sparse_arena): [2][points] sort keys and values, the sort's scratch,
        // [clouds] entry counts, and every cloud's table side by side
        DevBuf<unsigned long long> skeys, entries, tab_keys; DevBuf<int> svals, tab_start;
        DevBuf<unsigned char> sort_tmp;
        // room for m points in `cells` cells
        cudaError_t reserve(long long m, long long cells) {
            cudaError_t e;
            if ((e = pts.ensure(m)) || (e = pos_of.ensure(m)) || (e = tmp.ensure(m)) || (e = pt_cell.ensure(m)) ||
                (e = cell_start.ensure(cells + 1)) || (e = counts.ensure(cells + 1)) || (e = fill.ensure(cells)))
                return e;
            return cudaSuccess;
        }
    };
    GridArena tgt_arena, pair_tgt, aligned, odom_maps;
    // dcreg_set_sparse_maps: odometry's local maps and the pairs' targets past the dense-grid limits get sparse row
    // indexes instead of a refusal (a session keeps the value it had at open)
    bool sparse_maps = false;
    // dcreg_set_map_spacing: the minimum point spacing of odometry's map filter (0: the cap rule; a session keeps the
    // value it had at open)
    double map_spacing = 0.0;
    // dcreg_set_map_input_voxel: the voxel of odometry's map-input filter F_in (0: none; a session keeps the value it
    // had at open)
    double map_input_voxel = 0.0;
    // dcreg_set_lane_params: the batched calls' params point to one entry per lane (a session keeps the value it had at
    // open).  A call's entries [lanes] (plan_iteration), an odometry step's device lane -> sequence [lanes], and the log
    // fill's device trial -> lane [trials]
    bool lane_params = false;
    // dcreg_set_prior_map: odometry registers every frame against the context's target instead of a local map (a
    // session keeps the value it had at open)
    bool prior_map = false;
    DevBuf<dcreg_icp_params> d_lane_prm;
    DevBuf<int> d_lane_seq, d_trial_lane;
    DevBuf<float4> d_pair_tgt;                                   // targets, packed (w = global index)
    DevBuf<long long> d_pair_tgt_seg; DevBuf<double> d_pair_T;   // [n + 1] / [n][16] final poses
    DevBuf<float4> d_aligned;                                    // sources under their final poses
    DevBuf<dcreg_analysis> d_analysis;
    DevBuf<float4> d_flush;

    PinnedBuf<unsigned char> h_pinned;

    ncclComm_t comm = nullptr; int rank = 0, nranks = 1;
    // peer mailboxes for the in-kernel sum over ranks (peer_reduce.cuh); NCCL all-reduce is the fallback
    peer::Mailbox* d_mailbox = nullptr; void* peer_ptr[peer::kMaxRanks] = {nullptr}; bool peer_ok = false;
    peer::View peer_view{};
};

namespace {

#define CK(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess) {                                                                   \
            ctx->err = std::string(#call) + ": " + cudaGetErrorString(e_);                         \
            return DCREG_CUDA_ERROR;                                                               \
        }                                                                                          \
    } while (0)

constexpr long long kPartialDoubles = 72;   // d_partials per block: >= k1s::kPart and kAcc

int ensure_row_flags(dcreg_ctx* ctx, int rows) {
    if (!ctx->d_row_epoch) {
        CK(ctx->d_row_epoch.ensure(1));
        CK(cudaMemsetAsync(ctx->d_row_epoch, 0, sizeof(unsigned long long), ctx->stream));
        CK(ctx->d_warm_state.ensure(1));
        CK(cudaMemsetAsync(ctx->d_warm_state, 0, sizeof(IcpState), ctx->stream));
    }
    if (ctx->d_row_flags.cap >= rows) return DCREG_OK;
    CK(ctx->d_row_flags.ensure(rows));
    CK(cudaMemsetAsync(ctx->d_row_flags, 0, (size_t)rows * sizeof(unsigned long long), ctx->stream));   // below every epoch + 1
    return DCREG_OK;
}

// per-trial loop state: IcpState, ticket, sums, initial poses
int ensure_trials(dcreg_ctx* ctx, int trials) {
    if (ctx->d_state.cap >= trials) return DCREG_OK;
    CK(ctx->d_counter.ensure(trials));
    CK(cudaMemsetAsync(ctx->d_counter, 0, (size_t)trials * sizeof(unsigned int), ctx->stream));
    CK(ctx->d_acc.ensure((long long)trials * kAcc));
    CK(cudaMemsetAsync(ctx->d_acc, 0, (size_t)trials * kAcc * sizeof(double), ctx->stream));   // the solver block's warm-up input
    CK(ctx->d_state.ensure(trials));
    CK(cudaMemsetAsync(ctx->d_state, 0, (size_t)trials * sizeof(IcpState), ctx->stream));
    CK(ctx->d_T_init.ensure((long long)trials * 16));
    ctx->drop_graphs();
    return DCREG_OK;
}

// launch with the programmatic-stream-serialization attribute (see pdl_wait)
template <typename... KArgs, typename... Args>
static cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}

// host points -> d_out, packed by pack_points_kernel (d_seg: device table of n_seg segments, or null for one; d_radius:
// [n_seg] per-segment max |p|, or null)
// order / in_off (odometry): segment b of the device copy is host segment order[b], points [in_off[order[b]], ..) of xyz;
// null: xyz in order.  kind: cudaMemcpyDeviceToDevice when xyz is device memory (the voxel filter's output)
int upload_points(dcreg_ctx* ctx, const float* xyz, long long n, int stride, const long long* d_seg, int n_seg,
                  float4* d_out, float* d_radius, const int* order = nullptr, const int64_t* in_off = nullptr,
                  cudaMemcpyKind kind = cudaMemcpyHostToDevice) {
    const size_t bytes = (size_t)n * stride * sizeof(float);
    CK(ctx->d_stage.ensure(n * stride));
    if (!order) {
        CK(cudaMemcpyAsync(ctx->d_stage, xyz, bytes, kind, ctx->stream));
    } else {
        long long at = 0;                              // one copy per run of segments that are also consecutive on the host
        for (int b = 0; b < n_seg;) {
            int e = b + 1;
            while (e < n_seg && order[e] == order[e - 1] + 1) ++e;
            const long long a0 = in_off[order[b]], a1 = in_off[order[e - 1] + 1];
            CK(cudaMemcpyAsync(ctx->d_stage + (size_t)at * stride, xyz + (size_t)a0 * stride,
                               (size_t)(a1 - a0) * stride * sizeof(float), kind, ctx->stream));
            at += a1 - a0;
            b = e;
        }
    }
    if (d_radius) CK(cudaMemsetAsync(d_radius, 0, (size_t)n_seg * sizeof(float), ctx->stream));
    pack_points_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(ctx->d_stage, n, stride, d_seg, n_seg, d_out,
                                                                            d_radius);
    ctx->launches++;
    CK(cudaGetLastError());
    return DCREG_OK;
}

// The K1 streaming reduction's instantiations, entry (f64 planes ? 2 : 0) + (weight derivative ? 1 : 0).  Team size
// (k1_stream.cuh): 1 CTA per contiguous range; larger teams were no faster during development (not re-measured on H100)
using ReduceKernel = KernelEntry<k1s::Args>;
static constexpr ReduceKernel kReduceKernels[] = {
    {k1s::reduce_stream_kernel<float4, false, 1>, sizeof(k1s::Smem<float4>)},
    {k1s::reduce_stream_kernel<float4, true, 1>, sizeof(k1s::Smem<float4>)},
    {k1s::reduce_stream_kernel<double4, false, 1>, sizeof(k1s::Smem<double4>)},
    {k1s::reduce_stream_kernel<double4, true, 1>, sizeof(k1s::Smem<double4>)},
};
static_assert(std::size(kReduceKernels) == sizeof(dcreg_ctx::k1_attr_done), "one attribute flag per K1 kernel");

// The loop kernel's instantiations, entry v = loop_plan variant v, with the bytes of its loop_plan::smem_class.  Defined
// after every kernel: where a template kernel is instantiated sets the order of the module's functions, and with the
// loop kernels ahead of k2_step_kernel ptxas scheduled k2_step_kernel differently
template <int v>
constexpr LoopKernel loop_kernel() {
    constexpr loop_plan::Variant f = loop_plan::variant_flags(v);
    constexpr size_t smem[] = {offsetof(Iter2Smem, grid), offsetof(Iter2Smem, radius), sizeof(Iter2Smem)};
    static_assert(loop_plan::kSmemNoGrid == 0 && loop_plan::kSmemGrid == 1 && loop_plan::kSmemFull == 2,
                  "smem[] is indexed by loop_plan::SmemClass");
    return LoopKernel{icp_iter2_kernel<f.use_wd, f.grids, f.seq, f.planes, f.sparse>, smem[loop_plan::smem_class(v)]};
}
template <int... v>
constexpr std::array<LoopKernel, sizeof...(v)> loop_kernel_table(std::integer_sequence<int, v...>) {
    return {loop_kernel<v>()...};
}
static constexpr auto kLoopKernels = loop_kernel_table(std::make_integer_sequence<int, loop_plan::kVariants>{});
static_assert(kLoopKernels.size() == loop_plan::kVariants, "one loop kernel per loop_plan variant");

// slope / gate: dcreg_icp_params::weight_slope / weight_gate (0.9 / 0.1 in the reference, icp_test_runner.cpp:1776, 1785)
int launch_reduce(dcreg_ctx* ctx, const float4* d_src, const void* d_plane, bool f64, long long n,
                  const k1::Pose* pose, int use_wd, double slope = 0.9, double gate = 0.1, double npt_override = -1.0) {
    k1s::Args a{};
    a.src = d_src; a.plane = d_plane; a.n = n;
    if (pose) a.pose = *pose;
    for (int i = 0; i < 9; ++i) a.Rs[i] = ldexp(a.pose.R[i], 896);      // exact: see k1s::f32_raw
    a.slope = slope; a.gate = gate;
    a.npt_override = npt_override;
    if (ctx->peer_ok) a.peer = ctx->peer_view;                          // the sum over ranks happens inside the kernel
    a.counter = ctx->d_counter; a.acc = ctx->d_acc;
    // persistent grid: every SM holds 2 CTAs (launch bounds; 2 x (32 KB / 48 KB ring) fits H100's 227 KB carveout)
    const long long nchunks = (a.n + 31) / 32;
    long long g = (long long)ctx->sm_count * 2;
    const long long need = (nchunks + k1s::kWarpsPerBlock - 1) / k1s::kWarpsPerBlock;
    if (g > need) g = need;
    if (g < 1) g = 1;
    CK(ctx->d_partials.ensure(g * kPartialDoubles));
    a.partials = ctx->d_partials;
    const int v = (f64 ? 2 : 0) + (use_wd ? 1 : 0);
    const ReduceKernel& k = kReduceKernels[v];
    if (!ctx->k1_attr_done[v]) {        // function attributes are per device: per context (= per device), not per process
        CK(cudaFuncSetAttribute(k.kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k.smem));
        CK(cudaFuncSetAttribute(k.kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
        ctx->k1_attr_done[v] = true;
    }
    k.kernel<<<(int)g, k1s::kThreads, k.smem, ctx->stream>>>(a);
    ctx->launches++;
    CK(cudaGetLastError());
    return DCREG_OK;
}

// Fallback exchange (no peer mapping): one ncclAllReduce of the 32 sums behind the reducing kernel.
int nccl_allreduce_acc(dcreg_ctx* ctx) {
    if (!ctx->comm || ctx->peer_ok) return DCREG_OK;
    int r = g_nccl.AllReduce(ctx->d_acc, ctx->d_acc, kAcc, kNcclFloat64, kNcclSum, ctx->comm, ctx->stream);
    if (r != 0) {
        ctx->err = std::string("ncclAllReduce: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "error");
        return DCREG_NCCL_ERROR;
    }
    return DCREG_OK;
}

// Results of `trials` registrations: final poses, iteration counts, flags, and up to log_cap records per trial.
// status_out[t] = dcreg_status of trial t.
int read_results(dcreg_ctx* ctx, int trials, double* T_out, dcreg_iter_log* log, int log_cap, int* n_iterations,
                 int* converged, int* status_out) {
    CK(ctx->h_pinned.ensure((long long)trials * sizeof(IcpState)));
    IcpState* hs = (IcpState*)ctx->h_pinned.p;
    CK(cudaMemcpyAsync(hs, ctx->d_state, (size_t)trials * sizeof(IcpState), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    for (int t = 0; t < trials; ++t) {
        if (T_out) {
            double* To = T_out + (size_t)t * 16;
            for (int r = 0; r < 3; ++r) {
                for (int c = 0; c < 3; ++c) To[r * 4 + c] = hs[t].R[r * 3 + c];
                To[r * 4 + 3] = hs[t].t[r];
            }
            To[12] = To[13] = To[14] = 0.0; To[15] = 1.0;
        }
        if (n_iterations) n_iterations[t] = hs[t].iter;
        if (converged) converged[t] = hs[t].converged;
        if (status_out) status_out[t] = hs[t].status;
        if (hs[t].status == DCREG_CUDA_ERROR) ctx->err = "loop: the solver block timed out waiting for the block rows";
    }
    if (log && log_cap > 0) {
        if (trials == 1) {
            const int iters = hs[0].iter;
            int nrec = iters < log_cap ? iters : log_cap;
            // a NOT_ENOUGH_POINTS abort still wrote a record at index iters-1; a NONFINITE abort at index iters
            if (hs[0].status == DCREG_NONFINITE_UPDATE && iters < log_cap) nrec = iters + 1;
            if (nrec > 0)
                CK(cudaMemcpyAsync(log, ctx->d_log, (size_t)nrec * sizeof(dcreg_iter_log), cudaMemcpyDeviceToHost, ctx->stream));
        } else {
            CK(cudaMemcpyAsync(log, ctx->d_log, (size_t)trials * log_cap * sizeof(dcreg_iter_log), cudaMemcpyDeviceToHost,
                               ctx->stream));
        }
        CK(cudaStreamSynchronize(ctx->stream));
    }
    if (ctx->peer_ok) {                                 // a peer that never posted (timeout in peer::all_reduce32)
        unsigned int perr = 0;
        CK(cudaMemcpyAsync(&perr, &ctx->d_mailbox->error, sizeof(perr), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        if (perr) { ctx->err = "peer all-reduce timed out waiting for rank " + std::to_string((int)perr - 1); return DCREG_NCCL_ERROR; }
    }
    return DCREG_OK;
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------
extern "C" {

int dcreg_abi_version(void) { return DCREG_ABI_VERSION; }

void dcreg_default_params(dcreg_icp_params* p) {
    if (!p) return;
    memset(p, 0, sizeof(*p));
    p->search_radius = 1.0; p->max_iterations = 30;
    p->detection = DCREG_DET_SCHUR_CONDITION_NUMBER; p->handling = DCREG_HAND_PRECONDITIONED_CG;
    p->use_weight_derivative = 0;
    p->conv_thresh_rot = 1e-5; p->conv_thresh_trans = 1e-3;
    p->cond_thresh = 10.0; p->eig_thresh = 120.0; p->kappa_target = 1.0;
    p->pcg_tol = 1e-6; p->pcg_max_iter = 10; p->std_reg_gamma = 0.01;
    p->plane_thickness = 0.2; p->weight_slope = 0.9; p->weight_gate = 0.1; p->min_normal_norm = 1e-6;
    p->min_effective_points = 10; p->fixed_iterations = 0;
}

int dcreg_create(int device_id, dcreg_ctx** out) {
    if (!out) return DCREG_BAD_ARG;
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) return DCREG_NO_DEVICE;   // no CPU fallback
    if (device_id < 0 || device_id >= ndev) return DCREG_BAD_ARG;
    dcreg_ctx* ctx = new dcreg_ctx();
    ctx->device = device_id;
    *out = ctx;   // returned even on failure so the caller can read dcreg_last_error
    CK(cudaSetDevice(device_id));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device_id));
    ctx->sm_count = prop.multiProcessorCount;
    CK(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
    {
        const int rc = ensure_trials(ctx, 1);
        if (rc) return rc;
    }
    CK(ctx->d_n_active.ensure(1));
    CK(cudaMemsetAsync(ctx->d_n_active, 0, sizeof(unsigned int), ctx->stream));
    CK(ctx->d_small.ensure(1024));
    CK(ctx->d_k2_scratch.ensure(1));
    CK(cudaMemsetAsync(ctx->d_k2_scratch, 0, sizeof(K2Scratch), ctx->stream));
    CK(ctx->d_analysis.ensure(1));
    CK(cudaStreamSynchronize(ctx->stream));
    return DCREG_OK;
}

// Nothing may be queued or captured when the buffers go: the stream is drained, the communicator and the CUDA graphs
// released, and the buffers then freed by their owners as the context is deleted (the device is still current).
int dcreg_destroy(dcreg_ctx* ctx) {
    if (!ctx) return DCREG_BAD_ARG;
    cudaSetDevice(ctx->device);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    dcreg_comm_destroy(ctx);
    ctx->drop_graphs();
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
    return DCREG_OK;
}

const char* dcreg_last_error(const dcreg_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }
void* dcreg_stream(dcreg_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }
int64_t dcreg_launch_count(const dcreg_ctx* ctx) { return ctx ? ctx->launches : 0; }
void* dcreg_device_source(dcreg_ctx* ctx) { return ctx ? ctx->d_src.p : nullptr; }
void* dcreg_device_planes_f64(dcreg_ctx* ctx) { return ctx ? ctx->d_planes64.p : nullptr; }
void* dcreg_device_planes_f32(dcreg_ctx* ctx) { return ctx ? ctx->d_planes32.p : nullptr; }

int dcreg_set_source(dcreg_ctx* ctx, const float* xyz, int64_t n, int stride) {
    if (!ctx) return DCREG_BAD_ARG;
    if (!xyz || n <= 0 || stride < 3) { ctx->err = "dcreg_set_source: empty cloud or stride < 3"; return DCREG_BAD_ARG; }
    CK(cudaSetDevice(ctx->device));
    CK(ctx->d_src.ensure(n));
    ctx->n_src = n;
    if (ctx->nranks == 1) ctx->n_src_total = n;
    CK(ctx->d_src_radius.ensure(1));
    return upload_points(ctx, xyz, n, stride, nullptr, 1, ctx->d_src, ctx->d_src_radius);
}

int dcreg_set_global_source_count(dcreg_ctx* ctx, int64_t n_total) {
    if (!ctx || n_total <= 0) return DCREG_BAD_ARG;
    ctx->n_src_total = n_total;
    return DCREG_OK;
}

// exclusive scan of `n` ints (in -> out) on ctx's stream; tile_sums is ctx-owned scratch
static int device_exclusive_scan(dcreg_ctx* ctx, const int* in, long long n, int* out) {
    const int ntiles = (int)((n + corr::kScanTile - 1) / corr::kScanTile);
    CK(ctx->d_tile_sums.ensure(ntiles));
    corr::scan_tile_sums_kernel<<<ntiles, 256, 0, ctx->stream>>>(in, (int)n, ctx->d_tile_sums);
    corr::scan_tile_offsets_kernel<<<1, 1024, 0, ctx->stream>>>(ctx->d_tile_sums, ntiles);
    corr::scan_tile_apply_kernel<<<ntiles, 256, 0, ctx->stream>>>(in, (int)n, ctx->d_tile_sums, out);
    ctx->launches += 3;
    CK(cudaGetLastError());
    return DCREG_OK;
}

// ---- the voxel filter on the device (voxel_hash_kernel .. voxel_scatter_kernel) ---------------------------------------
// Cloud b's table region: the least power of two >= 2 n_b slots.  tab[n + 1] gets the regions' offsets; returns the total.
static long long voxel_tables(int n, const int64_t* h_seg, std::vector<long long>& tab) {
    tab.assign((size_t)n + 1, 0);
    for (int b = 0; b < n; ++b) {
        long long cap = 2;
        while (cap < 2 * (h_seg[b + 1] - h_seg[b])) cap <<= 1;
        tab[(size_t)b + 1] = tab[(size_t)b] + cap;
    }
    return tab[(size_t)n];
}

// The radix sort's end bit for a table of `slots` slots: the bit width of `slots`, the key of a point with no slot (below
// 4 n + 2 n_seg < 2^32 for n <= 2^29 - 1 points)
static int voxel_key_bits(long long slots) {
    int bits = 1;
    while (slots >> bits) ++bits;
    return bits;
}

// Room for a filter of n points in n_seg clouds over `slots` table slots, keeping up to max_points points per voxel.
// The sort's scratch only grows with n and slots, so room for the largest of several filters is room for each of them
static int voxel_reserve(dcreg_ctx* ctx, long long n, int n_seg, long long slots, int max_points = 1) {
    CK(ctx->d_vox_keys.ensure(slots));
    CK(ctx->d_vox_first.ensure(slots));
    CK(ctx->d_vox_slot.ensure(n));
    CK(ctx->d_vox_keep.ensure(n + 1));
    CK(ctx->d_vox_pos.ensure(n + 1));
    CK(ctx->d_vox_tab.ensure(n_seg + 1));
    CK(ctx->d_vox_seg.ensure(n_seg + 1));
    CK(ctx->d_vox_bad.ensure(n_seg));
    if (max_points > 1) {
        CK(ctx->d_vox_skey.ensure(2 * n));
        CK(ctx->d_vox_sval.ensure(2 * n));
        size_t tmp = 0;
        CK(cub::DeviceRadixSort::SortPairs(nullptr, tmp, (const unsigned int*)nullptr, (unsigned int*)nullptr,
                                           (const int*)nullptr, (int*)nullptr, (int)n, 0, voxel_key_bits(slots),
                                           ctx->stream));
        CK(ctx->d_vox_sort_tmp.ensure(std::max<long long>((long long)tmp, 1)));
    }
    return DCREG_OK;
}

// The voxel filter of n_seg clouds, n points of `stride` floats at d_in, with offsets d_seg (device) and h_seg (host),
// keeping up to max_points points per voxel.  The kept points go to d_out (out_stride 3 or 4, see voxel_scatter_kernel)
// and their indices in their own cloud to d_index (null: not wanted); the kept offsets to ctx->d_vox_seg [n_seg + 1], and
// bad[b] != 0 in ctx->d_vox_bad when cloud b has a voxel coordinate outside [-2^20, 2^20).  No host sync; whatever
// n_seg, six launches for max_points = 1, and for max_points > 1 seven and the radix sort's own.  min_spacing > 0 with
// max_points > 1: voxel_space_flag_kernel instead of voxel_cap_flag_kernel, same launches; 0 is the cap rule.  prune
// (the voxel map): voxel_prune_kernel between the flags and the scan, one launch more.
struct VoxelPrune {
    const int* center;                  // [n_seg] the frame reference whose translation prunes each cloud
    int n_frames;                       // ... read as ref_pose reads it
    const IcpState* states;
    const double* hist_T;
    double max_d2;                      // max_distance * max_distance
};
static int voxel_filter(dcreg_ctx* ctx, const float* d_in, long long n, int stride, const long long* d_seg,
                        const int64_t* h_seg, int n_seg, double voxel, float* d_out, int out_stride, long long* d_index,
                        int max_points = 1, double min_spacing = 0.0, const VoxelPrune* prune = nullptr) {
    std::vector<long long> tab;
    const long long slots = voxel_tables(n_seg, h_seg, tab);
    int rc = voxel_reserve(ctx, n, n_seg, slots, max_points);
    if (rc) return rc;
    CK(cudaMemcpyAsync(ctx->d_vox_tab, tab.data(), tab.size() * sizeof(long long), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemsetAsync(ctx->d_vox_keys, 0xff, (size_t)slots * sizeof(unsigned long long), ctx->stream));   // kEmptyKey
    CK(cudaMemsetAsync(ctx->d_vox_first, 0x7f, (size_t)slots * sizeof(int), ctx->stream));   // above every index
    CK(cudaMemsetAsync(ctx->d_vox_bad, 0, (size_t)n_seg * sizeof(int), ctx->stream));
    const unsigned nb = (unsigned)((n + 255) / 256), nb1 = (unsigned)((n + 256) / 256);
    voxel_hash_kernel<<<nb, 256, 0, ctx->stream>>>(d_in, n, stride, d_seg, n_seg, ctx->d_vox_tab, 1.0 / voxel,
                                                   ctx->d_vox_keys, ctx->d_vox_first, ctx->d_vox_slot, ctx->d_vox_bad);
    if (max_points == 1) {
        voxel_flag_kernel<<<nb1, 256, 0, ctx->stream>>>(ctx->d_vox_slot, n, ctx->d_vox_first, ctx->d_vox_keep);
        ctx->launches += 2;
        CK(cudaGetLastError());
    } else {
        unsigned int* key = ctx->d_vox_skey;
        int* val = ctx->d_vox_sval;
        const unsigned int dropped = (unsigned int)slots;
        voxel_sort_keys_kernel<<<nb, 256, 0, ctx->stream>>>(ctx->d_vox_slot, n, dropped, key, val);
        ctx->launches += 2;
        CK(cudaGetLastError());
        size_t tmp = (size_t)ctx->d_vox_sort_tmp.cap;
        CK(cub::DeviceRadixSort::SortPairs(ctx->d_vox_sort_tmp.p, tmp, key, key + n, val, val + n, (int)n, 0,
                                           voxel_key_bits(slots), ctx->stream));
        if (min_spacing > 0.0)      // val [0, n), the sort's consumed input, lists each run's kept points
            voxel_space_flag_kernel<<<nb1, 256, 0, ctx->stream>>>(d_in, stride, key + n, val + n, n, dropped, max_points,
                                                                  min_spacing * min_spacing, val, ctx->d_vox_keep);
        else
            voxel_cap_flag_kernel<<<nb1, 256, 0, ctx->stream>>>(key + n, val + n, n, dropped, max_points, ctx->d_vox_keep);
        ctx->launches++;                                         // (the radix sort's own kernels are not counted)
        CK(cudaGetLastError());
    }
    if (prune) {
        voxel_prune_kernel<<<nb, 256, 0, ctx->stream>>>(d_in, n, stride, d_seg, n_seg, ctx->d_vox_slot, ctx->d_vox_first,
                                                        prune->center, prune->n_frames, prune->states, prune->hist_T,
                                                        prune->max_d2, ctx->d_vox_keep);
        ctx->launches++;
        CK(cudaGetLastError());
    }
    if ((rc = device_exclusive_scan(ctx, ctx->d_vox_keep, n + 1, ctx->d_vox_pos))) return rc;
    // the scatter's threads also write the n_seg + 1 kept offsets: with empty clouds (the voxel map's updates) there may
    // be more of those than points
    const unsigned nbs = (unsigned)((std::max<long long>(n, n_seg) + 256) / 256);
    voxel_scatter_kernel<<<nbs, 256, 0, ctx->stream>>>(d_in, n, stride, d_seg, n_seg, ctx->d_vox_keep, ctx->d_vox_pos, d_out,
                                                       out_stride, d_index, ctx->d_vox_seg);
    ctx->launches++;
    CK(cudaGetLastError());
    return DCREG_OK;
}

// The voxel filter of n clouds of host points (xyz / offsets / stride as in dcreg_icp_run_scans, validated), up to
// max_points points per voxel at least min_spacing apart (0: no spacing): the kept points' xyz go to ctx->d_vox_xyz (3 floats a point, input order), their indices
// to ctx->d_vox_index when `index`.  One host sync, after which kept[n + 1] holds the kept offsets and bad[n] the range
// flags; fetch: *h_xyz (and *h_index) then point at host copies of the kept xyz (and indices) in ctx->h_pinned.
static int voxel_filter_host(dcreg_ctx* ctx, int n, const float* xyz, const int64_t* offsets, int stride, double voxel,
                             int max_points, double min_spacing, bool index, bool fetch, int64_t* kept, int* bad,
                             const float** h_xyz = nullptr, const long long** h_index = nullptr) {
    const long long total = offsets[n];
    CK(ctx->d_stage.ensure(total * stride));
    CK(ctx->d_vox_in_seg.ensure(n + 1));
    CK(ctx->d_vox_xyz.ensure(total * 3));
    if (index) CK(ctx->d_vox_index.ensure(total));
    CK(cudaMemcpyAsync(ctx->d_stage, xyz, (size_t)total * stride * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->d_vox_in_seg, offsets, (size_t)(n + 1) * sizeof(long long), cudaMemcpyHostToDevice, ctx->stream));
    int rc = voxel_filter(ctx, ctx->d_stage, total, stride, ctx->d_vox_in_seg, offsets, n, voxel, ctx->d_vox_xyz, 3,
                          index ? ctx->d_vox_index.p : nullptr, max_points, min_spacing);
    if (rc) return rc;
    // pinned: [n + 1] kept offsets, [n] flags (padded to 8 B), then (fetch) xyz [total][3] and indices [total]
    const size_t b_seg = (size_t)(n + 1) * sizeof(long long), b_bad = ((size_t)n * sizeof(int) + 7) / 8 * 8;
    const size_t b_xyz = fetch ? ((size_t)total * 3 * sizeof(float) + 7) / 8 * 8 : 0;
    const size_t b_idx = fetch && index ? (size_t)total * sizeof(long long) : 0;
    CK(ctx->h_pinned.ensure((long long)(b_seg + b_bad + b_xyz + b_idx)));
    unsigned char* h = ctx->h_pinned.p;
    CK(cudaMemcpyAsync(h, ctx->d_vox_seg, b_seg, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(h + b_seg, ctx->d_vox_bad, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    if (b_xyz) CK(cudaMemcpyAsync(h + b_seg + b_bad, ctx->d_vox_xyz, (size_t)total * 3 * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    if (b_idx) CK(cudaMemcpyAsync(h + b_seg + b_bad + b_xyz, ctx->d_vox_index, b_idx, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    memcpy(kept, h, b_seg);
    memcpy(bad, h + b_seg, (size_t)n * sizeof(int));
    if (h_xyz) *h_xyz = (const float*)(h + b_seg + b_bad);
    if (h_index) *h_index = (const long long*)(h + b_seg + b_bad + b_xyz);
    return DCREG_OK;
}

// Odometry's map-input filter and the source filter after it (dcreg_set_map_input_voxel, KISS-ICP's Voxelize) on n
// frames of host points, validated: F_in = the filter at voxel_in, one point per voxel, into ctx->d_in_xyz (indices in
// the frame to ctx->d_in_index when `index`); then F_s = the filter at voxel with max_points over F_in's kept points,
// through F_in's kept offsets on the device (ctx->d_in_seg), into ctx->d_vox_xyz (indices in F_in(frame) to
// ctx->d_vox_index).  F_s runs over as many points as the input has: the rest of d_in_xyz is NaN, which has no voxel
// and is never kept, so nothing waits for F_in's counts.  One host sync, after which kept_in / bad_in and kept / bad
// ([n + 1] / [n]) hold F_in's and F_s's kept offsets and range flags.
static int voxel_filter_chain(dcreg_ctx* ctx, int n, const float* xyz, const int64_t* offsets, int stride,
                              double voxel_in, double voxel, int max_points, bool index, int64_t* kept_in, int* bad_in,
                              int64_t* kept, int* bad) {
    const long long total = offsets[n];
    CK(ctx->d_stage.ensure(total * stride));
    CK(ctx->d_vox_in_seg.ensure(n + 1));
    CK(ctx->d_in_seg.ensure(n + 1));
    CK(ctx->d_in_xyz.ensure(total * 3));
    CK(ctx->d_vox_xyz.ensure(total * 3));
    if (index) {
        CK(ctx->d_in_index.ensure(total));
        CK(ctx->d_vox_index.ensure(total));
    }
    // pinned: F_in's [n + 1] kept offsets and [n] flags (padded to 8 B), then F_s's
    const size_t b_seg = (size_t)(n + 1) * sizeof(long long), b_bad = ((size_t)n * sizeof(int) + 7) / 8 * 8;
    CK(ctx->h_pinned.ensure((long long)(2 * (b_seg + b_bad))));
    unsigned char* h = ctx->h_pinned.p;
    CK(cudaMemcpyAsync(ctx->d_stage, xyz, (size_t)total * stride * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->d_vox_in_seg, offsets, b_seg, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemsetAsync(ctx->d_in_xyz, 0xff, (size_t)total * 3 * sizeof(float), ctx->stream));   // NaN
    int rc = voxel_filter(ctx, ctx->d_stage, total, stride, ctx->d_vox_in_seg, offsets, n, voxel_in, ctx->d_in_xyz, 3,
                          index ? ctx->d_in_index.p : nullptr);
    if (rc) return rc;
    CK(cudaMemcpyAsync(ctx->d_in_seg, ctx->d_vox_seg, b_seg, cudaMemcpyDeviceToDevice, ctx->stream));
    CK(cudaMemcpyAsync(h, ctx->d_vox_seg, b_seg, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(h + b_seg, ctx->d_vox_bad, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    // the input offsets bound F_in's kept ones, so they size F_s's tables
    if ((rc = voxel_filter(ctx, ctx->d_in_xyz, total, 3, ctx->d_in_seg, offsets, n, voxel, ctx->d_vox_xyz, 3,
                           index ? ctx->d_vox_index.p : nullptr, max_points)))
        return rc;
    CK(cudaMemcpyAsync(h + b_seg + b_bad, ctx->d_vox_seg, b_seg, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(h + 2 * b_seg + b_bad, ctx->d_vox_bad, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    memcpy(kept_in, h, b_seg);
    memcpy(bad_in, h + b_seg, (size_t)n * sizeof(int));
    memcpy(kept, h + b_seg + b_bad, b_seg);
    memcpy(bad, h + 2 * b_seg + b_bad, (size_t)n * sizeof(int));
    return DCREG_OK;
}

// Grid arenas (dcreg_ctx::GridArena, planned by arena_plan.hpp): the dense grids of n clouds at once, cloud b being
// d_pts[h_seg[b], h_seg[b+1]) (d_seg: the same offsets on the device).  One segmented bounds pass and one copy of the
// n x 6 bounds to the host (arena_bounds: the only host sync), then one count, one exclusive scan, one scatter and one
// in-cell rank over all clouds (arena_fill): the number of launches and syncs does not grow with n.  Inside every cloud
// the points are grouped by cell, then by index, and positions and .w (the global index) are shifted by the constant
// h_seg[b]: the (distance, then index) order of the neighbour search and the equality of position lists are those of
// the cloud built alone.  Replaces the kd-tree build of ICPContext::setTargetCloud (utils.hpp:393-424).

// Device bytes a caller wants back in the same sync as the bounds
struct Readback { const void* dev; size_t bytes; void* host; };

// hb[n * 6]: per cloud the min cell coordinates (x, y, z), then the max (arena_plan::box_of).  h_seg sizes the pass:
// the clouds' point counts or upper bounds of them (d_seg is what the pass reads).  more: copied back before the sync
static int arena_bounds(dcreg_ctx* ctx, dcreg_ctx::GridArena& A, const float4* d_pts, const int64_t* h_seg,
                        const long long* d_seg, int n, double inv_cell, std::vector<int>& hb,
                        const std::vector<Readback>& more = {}) {
    CK(A.d_grids.ensure(n));
    CK(A.d_cell_off.ensure(n + 1));
    CK(A.d_bounds.ensure((long long)n * 6));
    size_t pinned = ((size_t)n * 6 * sizeof(int) + 7) / 8 * 8;
    for (const Readback& r : more) pinned += (r.bytes + 7) / 8 * 8;
    CK(ctx->h_pinned.ensure((long long)pinned));
    hb.resize((size_t)n * 6);
    long long max_m = 0;
    for (int b = 0; b < n; ++b) {
        for (int k = 0; k < 3; ++k) { hb[6 * (size_t)b + k] = 1 << 30; hb[6 * (size_t)b + 3 + k] = -(1 << 30); }
        max_m = std::max<long long>(max_m, h_seg[b + 1] - h_seg[b]);
    }
    CK(cudaMemcpyAsync(A.d_bounds, hb.data(), hb.size() * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    // blocks per cloud: one cloud (a target of up to 10 M points) gets the whole GPU, many up to 64 each
    const unsigned bx = n == 1 ? (unsigned)ctx->sm_count * 4 : (unsigned)std::min<long long>(64, (max_m + 2047) / 2048);
    corr::grid_bounds_seg_kernel<<<dim3(bx, (unsigned)n), 256, 0, ctx->stream>>>(d_pts, d_seg, inv_cell, A.d_bounds);
    ctx->launches++;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(ctx->h_pinned, A.d_bounds, hb.size() * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    size_t at = ((size_t)n * 6 * sizeof(int) + 7) / 8 * 8;
    for (const Readback& r : more) {
        CK(cudaMemcpyAsync(ctx->h_pinned.p + at, r.dev, r.bytes, cudaMemcpyDeviceToHost, ctx->stream));
        at += (r.bytes + 7) / 8 * 8;
    }
    CK(cudaStreamSynchronize(ctx->stream));
    memcpy(hb.data(), ctx->h_pinned.p, hb.size() * sizeof(int));
    at = ((size_t)n * 6 * sizeof(int) + 7) / 8 * 8;
    for (const Readback& r : more) {
        memcpy(r.host, ctx->h_pinned.p + at, r.bytes);
        at += (r.bytes + 7) / 8 * 8;
    }
    return DCREG_OK;
}

// the grid of the arena's cloud with box x (arena_plan::plan), over m points in all
static corr::Grid arena_grid(const dcreg_ctx::GridArena& A, const arena_plan::Box& x, long long m, double inv_cell,
                             int rings) {
    corr::Grid g{};
    g.pts = A.pts; g.pos_of = A.pos_of; g.n = (int)m; g.dense = 1; g.rings = rings; g.inv_cell = inv_cell;
    g.ox = x.ox; g.oy = x.oy; g.oz = x.oz; g.nx = x.nx; g.ny = x.ny; g.nz = x.nz;
    g.cell_start = A.cell_start + x.cell_off;
    return g;
}

// groups the m points of the n clouds with boxes[n] (`cells` in all); on return A.d_grids[b] is cloud b's grid.
// cloud_rings: [n] every cloud's own ring count instead of `rings`, or null
static int arena_fill(dcreg_ctx* ctx, dcreg_ctx::GridArena& A, const float4* d_pts, const long long* d_seg, int n,
                      long long m, const arena_plan::Box* boxes, long long cells, double inv_cell, int rings,
                      const int* cloud_rings = nullptr) {
    int rc;
    CK(A.reserve(m, cells));
    std::vector<corr::Grid> hg((size_t)n);
    std::vector<int> off((size_t)n + 1);
    for (int b = 0; b < n; ++b) {
        hg[(size_t)b] = arena_grid(A, boxes[b], m, inv_cell, cloud_rings ? cloud_rings[b] : rings);
        off[(size_t)b] = (int)boxes[b].cell_off;
    }
    off[(size_t)n] = (int)cells;
    CK(cudaMemcpyAsync(A.d_grids, hg.data(), hg.size() * sizeof(corr::Grid), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(A.d_cell_off, off.data(), off.size() * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemsetAsync(A.counts, 0, (size_t)(cells + 1) * sizeof(int), ctx->stream));
    CK(cudaMemsetAsync(A.fill, 0, (size_t)cells * sizeof(int), ctx->stream));
    const unsigned nb = (unsigned)((m + 255) / 256);
    corr::grid_count_seg_kernel<<<nb, 256, 0, ctx->stream>>>(d_pts, (int)m, d_seg, n, A.d_grids, A.d_cell_off, A.pt_cell, A.counts);
    ctx->launches++;
    if ((rc = device_exclusive_scan(ctx, A.counts, cells + 1, A.cell_start))) return rc;
    corr::grid_scatter_kernel<<<nb, 256, 0, ctx->stream>>>(d_pts, (int)m, A.pt_cell, A.cell_start, A.fill, A.tmp, 0);
    corr::grid_rank_cells_kernel<<<nb, 256, 0, ctx->stream>>>(A.tmp, (int)m, A.pt_cell, A.cell_start, A.pts, A.pos_of);
    ctx->launches += 2;
    CK(cudaGetLastError());
    return DCREG_OK;
}

// The arena's clouds as sparse row indexes (sparse_index.hpp) instead of dense grids, for a step or call whose boxes are
// too large for them (arena_plan::plan_or_sparse): the m points of the n clouds with the bounds hb[n * 6] (host offsets
// h_seg[n + 1]).  The points end in the order arena_fill gives them (by cloud, then cell z, y, x, then index; positions
// and .w over all clouds) from two stable radix passes, (y, x) then (cloud, z); one count of every cloud's table entries
// comes back in one sync (the only one); the tables lie side by side (sparse_index::layout), and on return A.d_grids[b]
// is cloud b's index.  Five launches and one sync, whatever n.  *bad: the first cloud whose table would need more than
// sparse_index::kMaxSlots slots (nothing is inserted), else -1.  cloud_rings: as in arena_fill.  grid0: if given, gets
// cloud 0's index (the host copy of A.d_grids[0]).
static int build_sparse_arena(dcreg_ctx* ctx, dcreg_ctx::GridArena& A, const float4* d_pts, const long long* d_seg,
                              const std::vector<long long>& h_seg, int n, const int* hb, double inv_cell, int rings,
                              const int* cloud_rings, int* bad, corr::Grid* grid0 = nullptr) {
    *bad = -1;
    const long long m = h_seg[(size_t)n];
    CK(A.pts.ensure(m));
    CK(A.pos_of.ensure(m));
    CK(A.skeys.ensure(2 * m));
    CK(A.svals.ensure(2 * m));
    CK(A.entries.ensure(n));
    std::vector<corr::Grid> hg((size_t)n);
    for (int b = 0; b < n; ++b) {
        const int* x = hb + 6 * (size_t)b;
        corr::Grid& g = hg[(size_t)b];
        g.pts = A.pts; g.pos_of = A.pos_of; g.n = (int)m; g.dense = corr::kSparseGrid;
        g.rings = cloud_rings ? cloud_rings[b] : rings; g.inv_cell = inv_cell;
        g.ox = x[0]; g.oy = x[1]; g.oz = x[2];
        g.nx = x[3] - x[0] + 1; g.ny = x[4] - x[1] + 1; g.nz = x[5] - x[2] + 1;
    }
    CK(cudaMemcpyAsync(A.d_grids, hg.data(), hg.size() * sizeof(corr::Grid), cudaMemcpyHostToDevice, ctx->stream));
    unsigned long long* keys = A.skeys;
    int* vals = A.svals;
    // each pass sorts only the bits its keys use: up to the largest (y, x) of any box, and (last cloud, its top z)
    unsigned long long top[2] = {0, 0};
    for (int b = 0; b < n; ++b) {
        const corr::Grid& g = hg[(size_t)b];
        top[0] = std::max(top[0], sparse_index::key(g.nx - 1, g.ny - 1, 0));
        top[1] = std::max(top[1], ((unsigned long long)b << sparse_index::kBits) | (unsigned long long)(g.nz - 1));
    }
    int end_bit[2] = {1, 1};
    for (int p = 0; p < 2; ++p)
        while (end_bit[p] < 64 && top[p] >> end_bit[p]) ++end_bit[p];
    size_t tmp0 = 0, tmp1 = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, tmp0, keys, keys + m, vals, vals + m, (int)m, 0, end_bit[0], ctx->stream));
    CK(cub::DeviceRadixSort::SortPairs(nullptr, tmp1, keys, keys + m, vals, vals + m, (int)m, 0, end_bit[1], ctx->stream));
    CK(A.sort_tmp.ensure((long long)std::max(tmp0, tmp1)));
    const unsigned nb = (unsigned)((m + 255) / 256);
    for (int pass = 0; pass < 2; ++pass) {
        corr::sparse_seg_key_kernel<<<nb, 256, 0, ctx->stream>>>(d_pts, (int)m, d_seg, n, A.d_grids, pass, vals + m, keys,
                                                                  vals);
        CK(cudaGetLastError());
        size_t tmp = (size_t)A.sort_tmp.cap;
        CK(cub::DeviceRadixSort::SortPairs(A.sort_tmp.p, tmp, keys, keys + m, vals, vals + m, (int)m, 0, end_bit[pass],
                                           ctx->stream));
    }
    unsigned long long* sorted = keys;                           // (the passes' input keys are spent)
    corr::sparse_seg_gather_kernel<<<nb, 256, 0, ctx->stream>>>(d_pts, vals + m, (int)m, d_seg, n, A.d_grids, A.pts,
                                                                 A.pos_of, sorted);
    CK(cudaMemsetAsync(A.entries, 0, (size_t)n * sizeof(unsigned long long), ctx->stream));
    corr::sparse_seg_count_kernel<<<nb, 256, 0, ctx->stream>>>(sorted, (int)m, d_seg, n, A.d_grids, A.entries);
    CK(cudaGetLastError());
    CK(ctx->h_pinned.ensure((long long)n * (long long)sizeof(unsigned long long)));
    std::vector<unsigned long long> entries((size_t)n);
    CK(cudaMemcpyAsync(ctx->h_pinned.p, A.entries, entries.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost,
                       ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    memcpy(entries.data(), ctx->h_pinned.p, entries.size() * sizeof(unsigned long long));
    std::vector<long long> cap((size_t)n), off((size_t)n + 1);
    ctx->launches += 4;                                          // (the radix sorts' own kernels are not counted)
    if ((*bad = sparse_index::layout(n, entries.data(), cap.data(), off.data())) >= 0) return DCREG_OK;
    CK(A.tab_keys.ensure(off[(size_t)n]));
    CK(A.tab_start.ensure(off[(size_t)n]));
    for (int b = 0; b < n; ++b) {
        corr::Grid& g = hg[(size_t)b];
        g.keys = A.tab_keys.p + off[(size_t)b]; g.hstart = A.tab_start.p + off[(size_t)b];
        g.mask = (unsigned)(cap[(size_t)b] - 1);
    }
    CK(cudaMemcpyAsync(A.d_grids, hg.data(), hg.size() * sizeof(corr::Grid), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemsetAsync(A.tab_keys, 0xff, (size_t)off[(size_t)n] * sizeof(unsigned long long), ctx->stream));
    corr::sparse_seg_insert_kernel<<<nb, 256, 0, ctx->stream>>>(sorted, (int)m, d_seg, n, A.d_grids);
    ctx->launches++;
    CK(cudaGetLastError());
    if (grid0) *grid0 = hg[0];
    return DCREG_OK;
}

// Both steps; a cloud whose box needs more than arena_plan::kMaxDenseCells cells is rejected, unless sparse_at is
// given: then such clouds (or more than kMaxCells in all) make every cloud a sparse row index (build_sparse_arena), and
// *sparse_at is the first cloud over kMaxDenseCells (n: none, only the total is over), or -1 when the grids are dense.
static int build_grid_arena(dcreg_ctx* ctx, dcreg_ctx::GridArena& A, const float4* d_pts, const int64_t* h_seg,
                            const long long* d_seg, int n, double cell_size, int rings, const char* what,
                            long long* cells_out, int* sparse_at = nullptr) {
    const double inv_cell = 1.0 / cell_size;
    std::vector<int> hb;
    int rc = arena_bounds(ctx, A, d_pts, h_seg, d_seg, n, inv_cell, hb);
    if (rc) return rc;
    std::vector<arena_plan::Box> boxes;
    long long cells = 0;
    bool sparse = false;
    const std::string why = sparse_at ? arena_plan::plan_or_sparse(n, hb.data(), boxes, &cells, what, &sparse)
                                      : arena_plan::plan(n, hb.data(), boxes, &cells, what);
    if (!why.empty()) { ctx->err = why; return DCREG_BAD_ARG; }
    if (cells_out) *cells_out = cells;
    if (!sparse) {
        if (sparse_at) *sparse_at = -1;
        return arena_fill(ctx, A, d_pts, d_seg, n, h_seg[n], boxes.data(), cells, inv_cell, rings);
    }
    arena_plan::Box x;
    for (*sparse_at = 0; *sparse_at < n && arena_plan::box_of(hb.data() + 6 * (size_t)*sparse_at, &x) == arena_plan::kDense;)
        ++*sparse_at;
    int bad = -1;
    if ((rc = build_sparse_arena(ctx, A, d_pts, d_seg, std::vector<long long>(h_seg, h_seg + n + 1), n, hb.data(),
                                 inv_cell, rings, nullptr, &bad)))
        return rc;
    if (bad >= 0) {
        ctx->err = std::string(what) + " " + std::to_string(bad) + ": its sparse index would need more than 2^32 table slots";
        return DCREG_BAD_ARG;
    }
    return DCREG_OK;
}

// one-segment offset tables of the context's own clouds (device, in d_small): [0, 1] = {0, n_tgt}, [2, 3] = {0, n_src}
static long long* own_segs(dcreg_ctx* ctx) { return (long long*)(ctx->d_small + 512); }

// dcreg_set_target and its alias dcreg_set_target_sparse (`name`, for the error texts): a dense grid, or past
// arena_plan::kMaxDenseCells cells a sparse row index
static int set_target(dcreg_ctx* ctx, const float* xyz, int64_t m, int stride, double cell_size, const char* name) {
    if (!ctx) return DCREG_BAD_ARG;
    if (!xyz || m <= 0 || stride < 3 || !(cell_size > 0.0) || m > 0x7fffffffLL) {
        ctx->err = std::string(name) + ": empty cloud, stride < 3, cell_size <= 0 or too many points";
        return DCREG_BAD_ARG;
    }
    CK(cudaSetDevice(ctx->device));
    ctx->d_tgt.release();                               // not grow-only: exactly m points
    ctx->grid = corr::Grid{}; ctx->grid_cells = 0;
    ctx->has_grid = false;
    CK(ctx->d_tgt.ensure(m));
    ctx->n_tgt = m;
    int rc = upload_points(ctx, xyz, m, stride, nullptr, 1, ctx->d_tgt, nullptr);
    if (rc) return rc;
    ctx->cell_size = cell_size;
    // the target is the one cloud of tgt_arena
    const int64_t seg[2] = {0, m};
    long long* d_seg = own_segs(ctx);
    CK(cudaMemcpyAsync(d_seg, seg, sizeof(seg), cudaMemcpyHostToDevice, ctx->stream));
    const double inv_cell = 1.0 / cell_size;
    std::vector<int> hb;
    if ((rc = arena_bounds(ctx, ctx->tgt_arena, ctx->d_tgt, seg, d_seg, 1, inv_cell, hb))) return rc;
    arena_plan::Box box;
    const arena_plan::Fit fit = arena_plan::box_of(hb.data(), &box);
    if (fit == arena_plan::kOutOfRange) { ctx->err = arena_plan::out_of_range("grid build"); return DCREG_BAD_ARG; }
    if (fit == arena_plan::kDense) {
        if ((rc = arena_fill(ctx, ctx->tgt_arena, ctx->d_tgt, d_seg, 1, m, &box, box.cells, inv_cell, 1))) return rc;
        ctx->grid = arena_grid(ctx->tgt_arena, box, m, inv_cell, 1);
        ctx->grid_cells = box.cells;
    } else {
        int bad = -1;
        if ((rc = build_sparse_arena(ctx, ctx->tgt_arena, ctx->d_tgt, d_seg, {0, m}, 1, hb.data(), inv_cell, 1, nullptr,
                                     &bad, &ctx->grid)))
            return rc;
        if (bad >= 0) { ctx->err = std::string(name) + ": the sparse index needs more than 2^32 table slots"; return DCREG_BAD_ARG; }
    }
    const cudaError_t e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { ctx->err = std::string("grid build: ") + cudaGetErrorString(e); return DCREG_CUDA_ERROR; }
    ctx->has_grid = true;
    return DCREG_OK;
}

int dcreg_set_target(dcreg_ctx* ctx, const float* xyz, int64_t m, int stride, double cell_size) {
    return set_target(ctx, xyz, m, stride, cell_size, "dcreg_set_target");
}

int dcreg_set_target_sparse(dcreg_ctx* ctx, const float* xyz, int64_t m, int stride, double cell_size) {
    return set_target(ctx, xyz, m, stride, cell_size, "dcreg_set_target_sparse");
}

int dcreg_set_sparse_maps(dcreg_ctx* ctx, int enable) {
    if (!ctx) return DCREG_BAD_ARG;
    if (enable != 0 && enable != 1) { ctx->err = "set_sparse_maps: enable must be 0 or 1"; return DCREG_BAD_ARG; }
    ctx->sparse_maps = enable == 1;
    return DCREG_OK;
}

int dcreg_set_map_spacing(dcreg_ctx* ctx, double min_spacing) {
    if (!ctx) return DCREG_BAD_ARG;
    if (!(min_spacing >= 0.0 && min_spacing < INFINITY)) {
        ctx->err = "set_map_spacing: min_spacing must be finite and >= 0 (0: no spacing)";
        return DCREG_BAD_ARG;
    }
    ctx->map_spacing = min_spacing;
    return DCREG_OK;
}

int dcreg_set_map_input_voxel(dcreg_ctx* ctx, double voxel) {
    if (!ctx) return DCREG_BAD_ARG;
    if (!(voxel >= 0.0 && voxel < INFINITY)) {
        ctx->err = "set_map_input_voxel: voxel must be finite and >= 0 (0: the maps take the source)";
        return DCREG_BAD_ARG;
    }
    ctx->map_input_voxel = voxel;
    return DCREG_OK;
}

int dcreg_set_prior_map(dcreg_ctx* ctx, int enable) {
    if (!ctx) return DCREG_BAD_ARG;
    if (enable != 0 && enable != 1) { ctx->err = "set_prior_map: enable must be 0 or 1"; return DCREG_BAD_ARG; }
    ctx->prior_map = enable == 1;
    return DCREG_OK;
}

int dcreg_set_lane_params(dcreg_ctx* ctx, int enable) {
    if (!ctx) return DCREG_BAD_ARG;
    if (enable != 0 && enable != 1) { ctx->err = "set_lane_params: enable must be 0 or 1"; return DCREG_BAD_ARG; }
    ctx->lane_params = enable == 1;
    return DCREG_OK;
}

// Post-run point-to-point metrics of n pairs, replaces calculatePointToPointError (DCReg/include/utils.hpp:538-589;
// called at icp_test_runner.cpp:506-510 and once per CSV row at :1463-1470).  Pair b: source d_src[src_off[b],
// src_off[b+1]) under the pose d_T[16 b ..], target d_tgt[tgt_off[b], tgt_off[b+1]) with the dense grid fwd_grids[b]
// (d_src_seg / d_tgt_seg: the offsets on the device).  Forward exact 1-NN aligned source -> target (RMSE over ALL
// source points of the distances below the threshold, fitness, mean distance), grids over the aligned sources
// (ctx->aligned, same cell size), backward exact 1-NN target -> aligned source, Chamfer = mean of the two mean
// distances.  A pair's block partials are added on the host in block order, so a call reproduces bit for bit.
// out: [n][4] = rmse, fitness, chamfer, n_valid.
static int p2p_metrics(dcreg_ctx* ctx, int n, const float4* d_src, const long long* d_src_seg, const int64_t* src_off,
                       const float4* d_tgt, const long long* d_tgt_seg, const int64_t* tgt_off,
                       const corr::Grid* fwd_grids, const double* d_T, double cell_size, double threshold,
                       const char* what, double* out) {
    const long long ns = src_off[n];
    long long max_s = 0, max_t = 0;
    for (int b = 0; b < n; ++b) {
        max_s = std::max<long long>(max_s, src_off[b + 1] - src_off[b]);
        max_t = std::max<long long>(max_t, tgt_off[b + 1] - tgt_off[b]);
    }
    // blocks per pair: what the largest cloud needs, at most about 8 per SM over the whole call
    auto blocks = [&](long long mx) {
        const long long cap = std::max<long long>(1, (long long)ctx->sm_count * 8 / n);
        return (int)std::max<long long>(1, std::min<long long>((mx + kBlock - 1) / kBlock, cap));
    };
    const int gf = blocks(max_s), gb = blocks(max_t);
    CK(ctx->d_partials.ensure((long long)n * (gf + gb) * kPartialDoubles));   // 3 doubles per block and pair, forward then backward
    CK(ctx->d_aligned.ensure(ns));
    int rc;
    double* fwd = ctx->d_partials;
    double* bwd = ctx->d_partials + (size_t)3 * n * gf;
    corr::nn1_metrics_kernel<<<dim3((unsigned)gf, (unsigned)n), kBlock, 0, ctx->stream>>>(d_src, d_src_seg, fwd_grids, d_T,
                                                                                        threshold, fwd);
    corr::transform_points_kernel<<<(unsigned)((ns + 255) / 256), 256, 0, ctx->stream>>>(d_src, ns, d_T, ctx->d_aligned,
                                                                                        d_src_seg, n);
    ctx->launches += 2;
    CK(cudaGetLastError());
    if ((rc = build_grid_arena(ctx, ctx->aligned, ctx->d_aligned, src_off, d_src_seg, n, cell_size, 1, what, nullptr)))
        return rc;
    corr::nn1_metrics_kernel<<<dim3((unsigned)gb, (unsigned)n), kBlock, 0, ctx->stream>>>(d_tgt, d_tgt_seg, ctx->aligned.d_grids,
                                                                                        nullptr, threshold, bwd);
    ctx->launches++;
    CK(cudaGetLastError());
    std::vector<double> hp((size_t)3 * n * (gf + gb));
    CK(cudaMemcpyAsync(hp.data(), ctx->d_partials, hp.size() * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    const double* hf = hp.data();
    const double* hb = hp.data() + (size_t)3 * n * gf;
    for (int b = 0; b < n; ++b) {
        double sum_fwd = 0, sum_sq = 0, valid = 0, sum_bwd = 0;
        for (int k = 0; k < gf; ++k) {
            const double* p = hf + 3 * ((size_t)b * gf + k);
            sum_fwd += p[0]; sum_sq += p[1]; valid += p[2];
        }
        for (int k = 0; k < gb; ++k) sum_bwd += hb[3 * ((size_t)b * gb + k)];
        const double ns_b = (double)(src_off[b + 1] - src_off[b]), nt_b = (double)(tgt_off[b + 1] - tgt_off[b]);
        double* o = out + 4 * (size_t)b;
        o[0] = sqrt(sum_sq / ns_b);
        o[1] = valid / ns_b;
        o[2] = 0.5 * (sum_fwd / ns_b + sum_bwd / nt_b);
        o[3] = valid;
    }
    return DCREG_OK;
}

// out = { rmse, fitness, chamfer, n_valid } of the context's source under T against its target
int dcreg_point_to_point_metrics(dcreg_ctx* ctx, const double T[16], double error_threshold, double out[4]) {
    if (!ctx) return DCREG_BAD_ARG;
    if (!T || !out) { ctx->err = "p2p metrics: null pointer"; return DCREG_BAD_ARG; }
    if (!ctx->d_src || !ctx->has_grid || !ctx->d_tgt) { ctx->err = "p2p metrics: set source and target first"; return DCREG_BAD_ARG; }
    if (ctx->grid.dense == corr::kSparseGrid) {          // nn1_search expands rings over the whole box
        ctx->err = "p2p metrics need the dense grid (the target is a sparse row index: its bounding box is too large for "
                   "this cell size)";
        return DCREG_BAD_ARG;
    }
    CK(cudaSetDevice(ctx->device));
    const int64_t seg[4] = {0, ctx->n_tgt, 0, ctx->n_src};
    long long* d_seg = own_segs(ctx);
    double* dT = ctx->d_small + 640;
    CK(cudaMemcpyAsync(d_seg, seg, sizeof(seg), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(dT, T, 12 * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    return p2p_metrics(ctx, 1, ctx->d_src, d_seg + 2, seg + 2, ctx->d_tgt, d_seg, seg, ctx->tgt_arena.d_grids, dT,
                       ctx->cell_size, error_threshold, "p2p metrics: the aligned source", out);
}

// Spatial sort against the context's sparse row index, whose box is too large for one cell id: the n points of every
// segment b (d_seg, n_seg; null and 1: one cloud) by the cell of fl32(T_b p) (d_T [n_seg][16]), z, then y, then x, then
// by index, unclamped - the order a dense grid's sort gives whenever those cells lie inside its box.  Two stable radix
// passes, (y, x) then (segment, z), through the batch's key buffers; into out, w kept.
static int sort_by_sparse_cell(dcreg_ctx* ctx, const float4* pts, long long n, const long long* d_seg, int n_seg,
                               const double* d_T, double inv_cell, float4* out) {
    CK(ctx->d_scan_keys.ensure(2 * n));
    CK(ctx->d_scan_vals.ensure(2 * n));
    unsigned long long* keys = ctx->d_scan_keys;
    int* vals = ctx->d_scan_vals;
    int end_bit = 33;                                            // pass 1: segment above the 32 bits of z
    while (end_bit < 64 && ((unsigned long long)(n_seg - 1) >> (end_bit - 32))) ++end_bit;
    size_t tmp0 = 0, tmp1 = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, tmp0, keys, keys + n, vals, vals + n, (int)n, 0, 64, ctx->stream));
    CK(cub::DeviceRadixSort::SortPairs(nullptr, tmp1, keys, keys + n, vals, vals + n, (int)n, 0, end_bit, ctx->stream));
    CK(ctx->d_scan_sort_tmp.ensure((long long)std::max(tmp0, tmp1)));
    const unsigned nb = (unsigned)((n + 255) / 256);
    for (int pass = 0; pass < 2; ++pass) {
        sparse_source_key_kernel<<<nb, 256, 0, ctx->stream>>>(pts, n, d_seg, n_seg, d_T, inv_cell, pass, vals + n,
                                                               keys, vals);
        CK(cudaGetLastError());
        size_t tmp = (size_t)ctx->d_scan_sort_tmp.cap;
        CK(cub::DeviceRadixSort::SortPairs(ctx->d_scan_sort_tmp.p, tmp, keys, keys + n, vals, vals + n, (int)n, 0,
                                           pass ? end_bit : 64, ctx->stream));
    }
    gather_points_kernel<<<nb, 256, 0, ctx->stream>>>(pts, vals + n, n, out);
    ctx->launches += 3;                                          // (the radix sorts' own kernels are not counted)
    CK(cudaGetLastError());
    return DCREG_OK;
}

// Spatial sort of the source by the target cell of T*p (dense grids and sparse row indexes): consecutive threads of the
// iteration kernel then query neighbouring cells, so their candidate loads hit the same lines and their trip counts
// agree.  The sorted copy carries the original index in .w; the pose moves little during ICP, so one sort per run suffices.
static int sort_source_by_cell(dcreg_ctx* ctx, const double T[16], const float4** src_out) {
    *src_out = ctx->d_src;
    if (ctx->n_src > 0x7fffffffLL) return DCREG_OK;
    if (ctx->grid.dense == corr::kSparseGrid) {
        CK(ctx->d_src_sorted.ensure(ctx->n_src));
        double* dT = ctx->d_small + 640;
        CK(cudaMemcpyAsync(dT, T, 12 * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        const int rc = sort_by_sparse_cell(ctx, ctx->d_src, ctx->n_src, nullptr, 1, dT, ctx->grid.inv_cell, ctx->d_src_sorted);
        if (rc) return rc;
        *src_out = ctx->d_src_sorted;
        return DCREG_OK;
    }
    const long long n = ctx->n_src, ncells = ctx->grid_cells;
    CK(ctx->d_src_sorted.ensure(n));
    CK(ctx->d_sort_tmp.ensure(n));
    CK(ctx->d_pt_cell.ensure(n));
    CK(ctx->d_cell_tmp.ensure(3 * (ncells + 1)));
    int* counts = ctx->d_cell_tmp;
    int* start = counts + (ncells + 1);
    int* fill = start + (ncells + 1);
    CK(cudaMemsetAsync(counts, 0, (size_t)(ncells + 1) * sizeof(int), ctx->stream));
    CK(cudaMemsetAsync(fill, 0, (size_t)ncells * sizeof(int), ctx->stream));
    double* dT = ctx->d_small + 640;
    CK(cudaMemcpyAsync(dT, T, 12 * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    const unsigned nb = (unsigned)((n + 255) / 256);
    corr::source_cell_kernel<<<nb, 256, 0, ctx->stream>>>(ctx->d_src, (int)n, ctx->grid, dT, ctx->d_pt_cell, counts);
    int rc = device_exclusive_scan(ctx, counts, ncells + 1, start);
    if (rc) return rc;
    corr::grid_scatter_kernel<<<nb, 256, 0, ctx->stream>>>(ctx->d_src, (int)n, ctx->d_pt_cell, start, fill, ctx->d_sort_tmp, 0);
    corr::grid_rank_cells_kernel<<<nb, 256, 0, ctx->stream>>>(ctx->d_sort_tmp, (int)n, ctx->d_pt_cell, start, ctx->d_src_sorted, nullptr);
    ctx->launches += 3;
    CK(cudaGetLastError());
    *src_out = ctx->d_src_sorted;
    return DCREG_OK;
}

// A batch of sources registered side by side, one trial each (dcreg_icp_run_scans, _pairs, _sequences, _odometry): what
// the loop needs to know about it.  The sources live in buffers of their own (ctx->d_scan_*): the context's source stays.
struct Batch {
    // the sources: n clouds of host points (`stride` floats each); offsets (host, [n + 1]): source b is points
    // [offsets[b], offsets[b+1]) of the device copy.  order / in_off (odometry): source b is host frame order[b], points
    // [in_off[order[b]], ..) of xyz; null: xyz in order
    int n;
    const float* xyz;
    int stride;
    const int64_t* offsets;
    const int* order = nullptr;
    const int64_t* in_off = nullptr;
    cudaMemcpyKind kind = cudaMemcpyHostToDevice;   // cudaMemcpyDeviceToDevice: xyz is device memory
    // the sort (locality only): every source by the cells of its points under ...
    enum Sort {
        kContextGrid,   // ... its trial's initial pose, in the context's grid
        kGridTable,     // ... its trial's initial pose, in its own grid of the table (cell_off, `cells` in all)
        kBox,           // ... the poses sort_T (device [n][16]), in the box sort_box of sort_cells cells
    } sort = kContextGrid;
    const double* sort_T = nullptr;
    corr::Grid sort_box{};
    long long sort_cells = 0;
    // the grid each trial searches: the context's grid, or (grid_table) its own entry of the device table `grids`, built
    // with cell_size from the arena whose first cells are cell_off [n + 1]
    bool grid_table = false;
    const corr::Grid* grids = nullptr;
    const int* cell_off = nullptr;
    long long cells = 0;
    double cell_size = 0.0;
    // the table's grids are sparse row indexes (build_sparse_arena): the kSparse instantiations, and kGridTable sorts
    // by the unclamped cell (sort_by_sparse_cell)
    bool sparse = false;
    // lanes: none (0), or the sources are frames that run one after another in `lanes` lanes (grid y of the loop kernel),
    // at most max_bodies loop bodies in all
    int lanes = 0;
    SeqView seq{};
    long long max_bodies = 0;

    long long total() const { return offsets[n]; }
    long long max_n() const {
        long long m = 0;
        for (int b = 0; b < n; ++b) m = std::max<long long>(m, offsets[b + 1] - offsets[b]);
        return m;
    }
};

// Room for a batch's sources on the device and its offsets in ctx->d_scan_seg (the trials' states read them)
static int stage_sources(dcreg_ctx* ctx, const Batch& S) {
    const long long total = S.total();
    CK(ctx->d_scan_seg.ensure(S.n + 1));
    CK(ctx->d_scan_radius.ensure(S.n));
    CK(ctx->d_scan_cov.ensure((long long)S.n * 36));
    CK(ctx->d_scan_src.ensure(total));
    CK(ctx->d_scan_sorted.ensure(total));
    CK(ctx->d_scan_keys.ensure(2 * total));
    CK(ctx->d_scan_vals.ensure(2 * total));
    CK(cudaMemcpyAsync(ctx->d_scan_seg, S.offsets, (size_t)(S.n + 1) * sizeof(long long), cudaMemcpyHostToDevice, ctx->stream));
    return DCREG_OK;
}

// The lanes' device tables (after stage_sources): cursors, frame ranges, increments (delta null: identity) and priors
static int stage_lanes(dcreg_ctx* ctx, int lanes, int frames, SeqView* v) {
    CK(ctx->d_seq_cursor.ensure(lanes));
    CK(ctx->d_seq_first.ensure(lanes + 1));
    CK(ctx->d_seq_delta.ensure((long long)frames * 16));
    CK(ctx->d_seq_prior.ensure((long long)frames * 16));
    *v = SeqView{ctx->d_seq_cursor, ctx->d_seq_first, nullptr, ctx->d_seq_prior, ctx->d_scan_seg, ctx->d_n_active};
    return DCREG_OK;
}

// Upload the staged sources, pack them with their lever arms, and sort every source by cell (Batch::sort): the batch's
// counterpart of dcreg_set_source + sort_source_by_cell.  One stable radix sort of the (source, cell) keys keeps the
// segments contiguous and in order and needs no per-source cell tables.
static int sort_sources(dcreg_ctx* ctx, const Batch& S, const float4** src_out) {
    const long long n = S.total();
    int rc = upload_points(ctx, S.xyz, n, S.stride, ctx->d_scan_seg, S.n, ctx->d_scan_src, ctx->d_scan_radius, S.order,
                           S.in_off, S.kind);
    if (rc) return rc;
    const bool sparse_ctx = S.sort == Batch::kContextGrid && ctx->grid.dense == corr::kSparseGrid;
    if (sparse_ctx || (S.sort == Batch::kGridTable && S.sparse)) {
        if ((rc = sort_by_sparse_cell(ctx, ctx->d_scan_src, n, ctx->d_scan_seg, S.n, ctx->d_T_init,
                                      sparse_ctx ? ctx->grid.inv_cell : 1.0 / S.cell_size, ctx->d_scan_sorted)))
            return rc;
        *src_out = ctx->d_scan_sorted;
        return DCREG_OK;
    }
    unsigned long long* keys = ctx->d_scan_keys;
    int* vals = ctx->d_scan_vals;
    // keys below n * the cells of the context's grid or of the box, or below the table arena's cell count
    const double* T = ctx->d_T_init;
    corr::Grid g = ctx->grid;
    long long ncells = ctx->grid_cells;
    const corr::Grid* grids = nullptr;
    const int* cell_off = nullptr;
    unsigned long long key_end = (unsigned long long)S.n * (unsigned long long)ctx->grid_cells;
    if (S.sort == Batch::kGridTable) {
        grids = S.grids; cell_off = S.cell_off;
        key_end = (unsigned long long)S.cells;
    } else if (S.sort == Batch::kBox) {
        T = S.sort_T; g = S.sort_box; ncells = S.sort_cells;
        key_end = (unsigned long long)S.n * (unsigned long long)S.sort_cells;
    }
    const unsigned nb = (unsigned)((n + 255) / 256);
    cell_key_kernel<<<nb, 256, 0, ctx->stream>>>(ctx->d_scan_src, n, ctx->d_scan_seg, S.n, T, g, ncells, grids, cell_off,
                                                 keys, vals);
    ctx->launches++;
    CK(cudaGetLastError());
    int end_bit = 1;
    while (end_bit < 64 && (key_end - 1ull) >> end_bit) ++end_bit;
    size_t tmp = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, tmp, keys, keys + n, vals, vals + n, (int)n, 0, end_bit, ctx->stream));
    CK(ctx->d_scan_sort_tmp.ensure((long long)tmp));
    tmp = (size_t)ctx->d_scan_sort_tmp.cap;
    CK(cub::DeviceRadixSort::SortPairs(ctx->d_scan_sort_tmp.p, tmp, keys, keys + n, vals, vals + n, (int)n, 0, end_bit,
                                       ctx->stream));
    gather_points_kernel<<<nb, 256, 0, ctx->stream>>>(ctx->d_scan_src, vals + n, n, ctx->d_scan_sorted);
    ctx->launches++;                                             // (the radix sort's own kernels are not counted)
    CK(cudaGetLastError());
    *src_out = ctx->d_scan_sorted;
    return DCREG_OK;
}

// rings of cells that cover the search radius (exactness of the 5-NN-within-radius rule); valid in [1, 4]
static int search_rings(double search_radius, double cell_size) {
    return (int)ceil(search_radius / cell_size - 1e-9);
}

// What one loop body looks like for this context: the loop kernel's arguments and grid, and whether the solve step is
// inside it.
struct LoopPlan {
    bool fold_k2 = false;     // the solve / update step runs in the iteration kernel's last block (of some lanes)
    bool k2 = true;           // k2_step_kernel follows the iteration kernel (the step of some lanes is not folded)
    int grid_x = 1, trials = 1;
    Iter2Args b{};            // arguments of icp_iter2_kernel
    int variant = 0;          // its instantiation (loop_plan::variant), an index into kLoopKernels
    bool lanes = false;       // a batch in sequence lanes (b.seq)
    const float* scan_radius = nullptr;   // the lever arms of a batch's sources, or null (the context's source)
};

// The per-lane settings of a batched call (dcreg_set_lane_params): its n entries, one per lane, or none (n = 0: every
// lane runs the call's params)
struct Lanes {
    const dcreg_icp_params* p = nullptr;
    int n = 0;
};

// params' lanes when the setting is on: none when every entry has entry 0's settings, so that such a call is the call
// with one params (the same launches, graphs and bytes)
static Lanes call_lanes(const dcreg_icp_params* params, int n, bool on) {
    if (!on || n < 2 || lane_plan::uniform(params, n)) return Lanes{};
    return Lanes{params, n};
}

// batch: a batch of sources (trial b = source b, or lane b; src = the sources in sort order), or null (the context's
// source).  lanes: the call's per-lane settings (prm is entry 0), written to the context's lane table
static int plan_iteration(dcreg_ctx* ctx, const dcreg_icp_params* prm, const float4* src, double4* planes_out, int trials,
                          dcreg_iter_log* dlog, int log_cap, bool want_fold, LoopPlan* plan, const Batch* batch = nullptr,
                          const Lanes& lanes = Lanes{}) {
    LoopPlan& L = *plan;
    L.trials = trials;
    const bool grid_table = batch && batch->grid_table;       // the trials search their own grids
    L.lanes = batch && batch->lanes > 0;
    L.scan_radius = batch ? ctx->d_scan_radius.p : nullptr;
    Iter2Args& b = L.b;
    IterArgs& a = b.it;
    a.src = src; a.n = batch ? batch->total() : ctx->n_src; a.grid = grid_table ? corr::Grid{} : ctx->grid; a.state = ctx->d_state;
    a.counter = ctx->d_counter; a.acc = ctx->d_acc;
    a.planes_out = planes_out; a.prm = *prm;
    {   // rings of cells that cover the search radius (exactness of the 5-NN-within-radius rule)
        const int rings = search_rings(prm->search_radius, grid_table ? batch->cell_size : ctx->cell_size);
        if (rings < 1 || rings > 4) {
            ctx->err = "search_radius / target cell_size must be in (0, 4]: rebuild the target index with a larger cell";
            return DCREG_BAD_ARG;
        }
        a.grid.rings = rings;
    }
    // Lean only: a plain 5-NN search and a fresh fit for every slot in every iteration, no records (coherent_step 0:
    // the solve step never switches to coherent mode).  Seam 1 (planes_out) fits every slot once; more than 2^29 - 1
    // slots would need more than 54 GB of records (101 B per slot); DCREG_FUSED_SEARCH (a single run of the context's
    // source) is the reference the record-reusing loop is tested against.
    const bool lean_only = planes_out || a.n > arena_plan::kMaxPoints || (!batch && getenv("DCREG_FUSED_SEARCH"));
    if ((trials > 1 || batch) && lean_only) {   // only dcreg_icp_run_batch: a batch's sources total at most kMaxPoints
        ctx->err = "batched trials need per-slot records (more than 2^29 - 1 source points, or DCREG_FUSED_SEARCH set)";
        return DCREG_BAD_ARG;
    }
    // (seam 1 has no batch here, so the variant is one of kLoopKernels)
    const bool sparse = grid_table ? batch->sparse : ctx->grid.dense == corr::kSparseGrid;
    L.variant = loop_plan::variant(planes_out != nullptr, sparse, grid_table, L.lanes, prm->use_weight_derivative != 0);
    const long long slots = ctx->n_src;
    if (!lean_only) {
        // per-slot records: [trials][slots], or one slice per source at its segment offset (total slots); reallocated
        // at exactly this shape when either side of it grows
        const long long rec_slots = batch ? a.n : slots;
        const int rec_trials = batch ? 1 : trials;
        if (ctx->nn_slots < rec_slots || ctx->nn_trials < rec_trials) {
            const long long tot = rec_slots * rec_trials;
            ctx->d_nn.release(); ctx->d_plane_cache.release(); ctx->d_fit_state.release(); ctx->d_plane_key.release();
            ctx->nn_slots = 0; ctx->nn_trials = 0;
            CK(ctx->d_nn.ensure(tot * kNnRec));
            CK(ctx->d_plane_cache.ensure(tot));
            CK(ctx->d_fit_state.ensure(tot));
            CK(ctx->d_plane_key.ensure(tot * 5));
            ctx->nn_slots = rec_slots; ctx->nn_trials = rec_trials;
            ctx->nn_valid = false;
        }
        b.nn = ctx->d_nn; b.plane_cache = ctx->d_plane_cache; b.fit_state = ctx->d_fit_state; b.plane_key = ctx->d_plane_key;
    }
    // the solve step inside the kernel unless the sum over ranks has to go through NCCL, for the lanes that run "Ours"
    // (lane_plan.hpp): all of them, none, or a mix, which runs K2 after the iteration kernel as well
    const bool can_fold = want_fold && !(ctx->comm && !ctx->peer_ok);
    const lane_plan::Mix mix = lanes.n ? lane_plan::mix(lanes.p, lanes.n, can_fold) : lane_plan::mix(prm, 1, can_fold);
    L.fold_k2 = mix.fold; L.k2 = mix.k2;
    if (lanes.n) {
        CK(ctx->d_lane_prm.ensure(lanes.n));
        CK(cudaMemcpyAsync(ctx->d_lane_prm, lanes.p, (size_t)lanes.n * sizeof(dcreg_icp_params), cudaMemcpyHostToDevice,
                           ctx->stream));
        b.lane_prm = ctx->d_lane_prm;
    }
    // a single folded run: block 0 is a dedicated solver block (solver_block); batches keep the ticket, since a
    // solver block per trial in a multi-wave grid could fill every resident slot with waiting blocks
    const bool solver = L.fold_k2 && trials == 1 && !batch && !lanes.n && !getenv("DCREG_NO_SOLVER_BLOCK");
    // blocks per trial and slots per block: loop_plan.hpp
    const loop_plan::Tiles tp = batch ? loop_plan::plan_scan_tiles(batch->max_n(), kBlock)
                                      : loop_plan::plan_tiles(slots, trials, ctx->sm_count, kBlock, solver ? 1 : 0);
    L.grid_x = (int)tp.grid_x + (solver ? 1 : 0);
    b.tile = tp.tile;
    CK(ctx->d_partials.ensure((long long)L.grid_x * trials * kPartialDoubles));
    int rc;
    if (solver && (rc = ensure_row_flags(ctx, (int)tp.grid_x))) return rc;
    a.partials = ctx->d_partials;
    if (solver) {
        b.row_flags = ctx->d_row_flags; b.row_epoch = ctx->d_row_epoch;
        b.warm_state = ctx->d_warm_state;
    }
    b.force = ctx->force_coherent && !lean_only ? 1 : 0;
    b.use_seeds = ctx->nn_valid ? 1 : 0;
    b.stats = ctx->d_iter_stats;
    const double r2 = prm->search_radius * prm->search_radius;
    float r2f = (float)r2;
    if ((double)r2f < r2) r2f = nextafterf(r2f, INFINITY);
    b.r2_up = r2f;
    b.fold_k2 = L.fold_k2 ? 1 : 0;
    b.log = dlog; b.log_cap = log_cap;
    b.src_radius = batch ? ctx->d_scan_radius.p : ctx->d_src_radius.p;
    b.coherent_step = lean_only ? 0.0 : kCoherentStep;
    b.seg = batch ? ctx->d_scan_seg.p : nullptr;
    // (a CUDA graph of the loop freezes this pointer, not the table: the entries are rewritten before every pairs call
    // and read at every launch, and a regrown table has a new pointer and so a new graph key)
    b.grids = grid_table ? batch->grids : nullptr;
    // lanes: trials = lanes; the frame advance, not the solve step, counts the lanes still running
    b.seq = L.lanes ? batch->seq : SeqView{};
    b.n_active = L.lanes ? nullptr : ctx->d_n_active.p;
    if (ctx->peer_ok && !planes_out) b.peer = ctx->peer_view;       // seam 1 counts this rank's slots only
    if (!ctx->loop_attr_done) {          // per device (= per context), not per process
        for (const LoopKernel& k : kLoopKernels) CK(loop_kernel_attributes(k));
        ctx->loop_attr_done = true;
    }
    return DCREG_OK;
}

// enqueue the iteration kernel of a plan (inside or outside a stream capture)
static int launch_plan(dcreg_ctx* ctx, LoopPlan& L) {
    L.b.use_seeds = ctx->nn_valid ? 1 : 0;
    ctx->nn_valid = true;
    const LoopKernel& k = kLoopKernels[L.variant];
    CK(launch_pdl(k.kernel, dim3((unsigned)L.grid_x, (unsigned)L.trials), dim3(kBlock), k.smem, ctx->stream, L.b));
    ctx->launches++;
    CK(cudaGetLastError());
    return DCREG_OK;
}

// the separate solve kernel (one warp per trial): baseline methods, the host-plane loop, NCCL fallback of a sharded run
// coherent_step: the plan's (Iter2Args::coherent_step).  scan_radius: the lever arms of a batch's sources, or null (the
// context's source).  seq: the lanes of a batch (trials = lanes), or null; lane_radius: Iter2Args's
static int launch_k2(dcreg_ctx* ctx, const dcreg_icp_params* prm, dcreg_iter_log* dlog, int log_cap, double coherent_step,
                     int trials = 1, const float* scan_radius = nullptr, const SeqView* seq = nullptr,
                     const double* lane_radius = nullptr, const LoopPlan* L = nullptr) {
    CK(launch_pdl(k2_step_kernel, dim3((unsigned)trials), dim3(32), 0, ctx->stream, (const double*)ctx->d_acc.p, ctx->d_state.p, *prm,
                  dlog, log_cap, scan_radius ? scan_radius : (const float*)ctx->d_src_radius.p, coherent_step,
                  trials == 1 && !seq ? ctx->d_k2_scratch.p : (K2Scratch*)nullptr, seq ? nullptr : ctx->d_n_active.p,
                  scan_radius ? 1 : 0, seq ? *seq : SeqView{}, lane_radius, L ? L->b.lane_prm : nullptr,
                  L ? L->b.lane_seq : nullptr, L && L->fold_k2 ? 1 : 0));
    ctx->launches++;
    return DCREG_OK;
}

// one loop body: iteration kernel [+ all-reduce + solve kernel when the step is not folded]
static int launch_body(dcreg_ctx* ctx, LoopPlan& L, const dcreg_icp_params* prm, dcreg_iter_log* dlog, int log_cap, bool with_k2) {
    int rc = launch_plan(ctx, L);
    if (rc) return rc;
    if (with_k2 && L.k2) {
        if ((rc = nccl_allreduce_acc(ctx))) return rc;          // no-op on one GPU / with peer mailboxes
        if ((rc = launch_k2(ctx, prm, dlog, log_cap, L.b.coherent_step, L.trials, L.scan_radius, L.lanes ? &L.b.seq : nullptr,
                            L.b.lane_radius, &L)))
            return rc;
    }
    return DCREG_OK;
}

// running: the start value of the running-trials counter n_active (0: trials)
static int init_state(dcreg_ctx* ctx, const double* T, int trials = 1, const long long* scan_seg = nullptr, int running = 0) {
    ctx->nn_valid = false;            // a new run: no neighbours of a previous iteration to seed the search with
    int rc = ensure_trials(ctx, trials);
    if (rc) return rc;
    CK(cudaMemcpyAsync(ctx->d_T_init, T, (size_t)trials * 16 * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    init_state_kernel<<<(trials + 127) / 128, 128, 0, ctx->stream>>>(ctx->d_state, ctx->d_T_init, ctx->n_src_total, ctx->d_counter,
                                                                   trials, ctx->d_n_active, scan_seg,
                                                                   running > 0 ? running : trials);
    ctx->launches++;
    CK(cudaGetLastError());
    return DCREG_OK;
}

int dcreg_find_planes(dcreg_ctx* ctx, const double T[16], double search_radius, double* planes_out,
                      int64_t* n_corr_pt) {
    if (!ctx || !T) return DCREG_BAD_ARG;
    if (!ctx->d_src || !ctx->has_grid) { ctx->err = "dcreg_find_planes: set source and target first"; return DCREG_BAD_ARG; }
    CK(cudaSetDevice(ctx->device));
    CK(ctx->d_planes64.ensure(ctx->n_src));
    CK(ctx->d_planes32.ensure(ctx->n_src));
    int rc;
    dcreg_icp_params prm;
    dcreg_default_params(&prm);
    prm.search_radius = search_radius;
    prm.min_effective_points = 0;
    if ((rc = init_state(ctx, T))) return rc;
    LoopPlan L;
    if ((rc = plan_iteration(ctx, &prm, ctx->d_src, ctx->d_planes64, 1, nullptr, 0, false, &L))) return rc;
    if ((rc = launch_plan(ctx, L))) return rc;
    double acc[kAcc];
    CK(cudaMemcpyAsync(acc, ctx->d_acc, sizeof(acc), cudaMemcpyDeviceToHost, ctx->stream));
    if (planes_out)
        CK(cudaMemcpyAsync(planes_out, ctx->d_planes64, (size_t)ctx->n_src * sizeof(double4), cudaMemcpyDeviceToHost,
                           ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (n_corr_pt) *n_corr_pt = (int64_t)(acc[k2::kAccNpt] + 0.5);
    return DCREG_OK;
}

static int reduce_common(dcreg_ctx* ctx, const void* d_src, const void* d_plane, bool f64, int64_t n,
                         const double pose_Rt[12], int use_wd, double out27[27], double stats[3]) {
    if (!ctx) return DCREG_BAD_ARG;
    if (!d_src || !d_plane || n <= 0 || !pose_Rt || !out27) { ctx->err = "reduce: null pointer or n <= 0"; return DCREG_BAD_ARG; }
    CK(cudaSetDevice(ctx->device));
    k1::Pose P;
    for (int i = 0; i < 9; ++i) P.R[i] = pose_Rt[i];
    for (int i = 0; i < 3; ++i) P.t[i] = pose_Rt[9 + i];
    int rc = launch_reduce(ctx, (const float4*)d_src, d_plane, f64, n, &P, use_wd);
    if (rc) return rc;
    if ((rc = nccl_allreduce_acc(ctx))) return rc;
    double acc[kAcc];
    CK(cudaMemcpyAsync(acc, ctx->d_acc, sizeof(acc), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    for (int i = 0; i < 27; ++i) out27[i] = acc[i];
    if (stats) { stats[0] = acc[k2::kAccSumR2]; stats[1] = acc[k2::kAccNeff]; stats[2] = acc[k2::kAccNpt]; }
    return DCREG_OK;
}

int dcreg_reduce_normal_equations(dcreg_ctx* ctx, const void* d_src, const void* d_plane, int64_t n,
                                  const double pose_Rt[12], int use_weight_derivative, double out27[27],
                                  double stats[3]) {
    return reduce_common(ctx, d_src, d_plane, false, n, pose_Rt, use_weight_derivative, out27, stats);
}

int dcreg_reduce_normal_equations_f64plane(dcreg_ctx* ctx, const void* d_src, const void* d_plane, int64_t n,
                                           const double pose_Rt[12], int use_weight_derivative, double out27[27],
                                           double stats[3]) {
    return reduce_common(ctx, d_src, d_plane, true, n, pose_Rt, use_weight_derivative, out27, stats);
}

int dcreg_reduce_normal_equations_host(dcreg_ctx* ctx, const float* src4, const void* plane4, int plane_is_f64,
                                       int64_t n, const double pose_Rt[12], int use_weight_derivative,
                                       double out27[27], double stats[3]) {
    if (!ctx) return DCREG_BAD_ARG;
    if (!src4 || !plane4 || n <= 0) { ctx->err = "reduce_host: null pointer or n <= 0"; return DCREG_BAD_ARG; }
    CK(cudaSetDevice(ctx->device));
    int rc = dcreg_set_source(ctx, src4, n, 4);
    if (rc) return rc;
    CK(ctx->d_planes64.ensure(n));
    CK(ctx->d_planes32.ensure(n));
    if (plane_is_f64)
        CK(cudaMemcpyAsync(ctx->d_planes64, plane4, (size_t)n * sizeof(double4), cudaMemcpyHostToDevice, ctx->stream));
    else
        CK(cudaMemcpyAsync(ctx->d_planes32, plane4, (size_t)n * sizeof(float4), cudaMemcpyHostToDevice, ctx->stream));
    return reduce_common(ctx, ctx->d_src, plane_is_f64 ? (const void*)ctx->d_planes64 : (const void*)ctx->d_planes32,
                         plane_is_f64 != 0, n, pose_Rt, use_weight_derivative, out27, stats);
}

int dcreg_freeze_planes_f32(dcreg_ctx* ctx) {
    if (!ctx || !ctx->d_planes64 || ctx->n_src <= 0) return DCREG_BAD_ARG;
    CK(cudaSetDevice(ctx->device));
    planes_to_f32_kernel<<<(unsigned)((ctx->n_src + 255) / 256), 256, 0, ctx->stream>>>(ctx->d_planes64, ctx->n_src,
                                                                                        ctx->d_planes32);
    ctx->launches++;
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(ctx->stream));
    return DCREG_OK;
}

int dcreg_time_reduce(dcreg_ctx* ctx, int plane_is_f64, const double pose_Rt[12], int use_weight_derivative,
                      int reps, int flush_l2, float* ms_per_launch) {
    if (!ctx || !pose_Rt || reps <= 0 || !ms_per_launch) return DCREG_BAD_ARG;
    if (!ctx->d_src || !ctx->d_planes64) { ctx->err = "time_reduce: no source/planes on the context"; return DCREG_BAD_ARG; }
    CK(cudaSetDevice(ctx->device));
    k1::Pose P;
    for (int i = 0; i < 9; ++i) P.R[i] = pose_Rt[i];
    for (int i = 0; i < 3; ++i) P.t[i] = pose_Rt[9 + i];
    const long long flush_n = (256ll << 20) / sizeof(float4);   // 256 MiB > 50 MB L2
    if (flush_l2) CK(ctx->d_flush.ensure(flush_n));
    const void* plane = plane_is_f64 ? (const void*)ctx->d_planes64 : (const void*)ctx->d_planes32;
    int rc = DCREG_OK;
    double total = 0.0;
    if (!flush_l2) {
        // one event pair around the whole batch of back-to-back launches (inputs larger than L2 need no flush)
        cudaEvent_t b0, b1;
        CK(cudaEventCreate(&b0)); CK(cudaEventCreate(&b1));
        CK(cudaEventRecord(b0, ctx->stream));
        for (int i = 0; i < reps && rc == DCREG_OK; ++i) {
            rc = launch_reduce(ctx, ctx->d_src, plane, plane_is_f64 != 0, ctx->n_src, &P, use_weight_derivative);
            if (rc == DCREG_OK) rc = nccl_allreduce_acc(ctx);      // sharded: the 32-double all-reduce is part of the step
        }
        CK(cudaEventRecord(b1, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        float ms = 0.f;
        cudaEventElapsedTime(&ms, b0, b1);
        total = ms;
        cudaEventDestroy(b0); cudaEventDestroy(b1);
    } else {
        std::vector<cudaEvent_t> e0(reps), e1(reps);
        for (int i = 0; i < reps; ++i) { CK(cudaEventCreate(&e0[i])); CK(cudaEventCreate(&e1[i])); }
        for (int i = 0; i < reps && rc == DCREG_OK; ++i) {
            flush_l2_kernel<<<ctx->sm_count * 4, 256, 0, ctx->stream>>>(ctx->d_flush, flush_n, (float)i);
            ctx->launches++;
            CK(cudaEventRecord(e0[i], ctx->stream));
            rc = launch_reduce(ctx, ctx->d_src, plane, plane_is_f64 != 0, ctx->n_src, &P, use_weight_derivative);
            if (rc == DCREG_OK) rc = nccl_allreduce_acc(ctx);
            CK(cudaEventRecord(e1[i], ctx->stream));
        }
        CK(cudaStreamSynchronize(ctx->stream));
        for (int i = 0; i < reps; ++i) {
            float ms = 0.f;
            cudaEventElapsedTime(&ms, e0[i], e1[i]);
            total += ms;
            cudaEventDestroy(e0[i]); cudaEventDestroy(e1[i]);
        }
    }
    *ms_per_launch = (float)(total / reps);
    return rc;
}

int dcreg_iteration_counters(dcreg_ctx* ctx, int enable, uint64_t out[2]) {
    if (!ctx || !out) return DCREG_BAD_ARG;
    CK(cudaSetDevice(ctx->device));
    out[0] = out[1] = 0;
    if (ctx->d_iter_stats) {
        unsigned int h[2] = {0, 0};
        CK(cudaMemcpyAsync(h, ctx->d_iter_stats, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        out[0] = h[0]; out[1] = h[1];
    }
    if (enable) CK(ctx->d_iter_stats.ensure(2));
    else ctx->d_iter_stats.release();
    if (ctx->d_iter_stats) CK(cudaMemsetAsync(ctx->d_iter_stats, 0, 2 * sizeof(unsigned int), ctx->stream));
    return DCREG_OK;
}

int dcreg_time_iteration(dcreg_ctx* ctx, const dcreg_icp_params* params, const double T[16], int what, int reps,
                         float* ms_per_body) {
    if (!ctx || !params || !T || reps <= 0 || !ms_per_body) return DCREG_BAD_ARG;
    if (!ctx->d_src || !ctx->has_grid) { ctx->err = "time_iteration: set source and target first"; return DCREG_BAD_ARG; }
    CK(cudaSetDevice(ctx->device));
    dcreg_icp_params prm = *params;
    prm.fixed_iterations = 1;
    prm.max_iterations = reps + 8;
    int rc;
    if ((rc = init_state(ctx, T))) return rc;
    const float4* src_iter = ctx->d_src;
    if ((rc = sort_source_by_cell(ctx, T, &src_iter))) return rc;
    ctx->force_coherent = (what == 0);                                     // fixed pose: measure the record-reusing mode
    LoopPlan L;
    rc = plan_iteration(ctx, &prm, src_iter, nullptr, 1, nullptr, 0, what == 1, &L);
    ctx->force_coherent = false;
    if (rc) return rc;
    for (int warm = 0; warm < 2; ++warm)                                   // instruction caches, lazy module load
        if ((rc = launch_body(ctx, L, &prm, nullptr, 0, false))) return rc;
    cudaEvent_t b0, b1;
    CK(cudaEventCreate(&b0)); CK(cudaEventCreate(&b1));
    CK(cudaEventRecord(b0, ctx->stream));
    for (int i = 0; i < reps; ++i)
        if ((rc = launch_body(ctx, L, &prm, nullptr, 0, what == 1))) return rc;
    CK(cudaEventRecord(b1, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    float ms = 0.f;
    cudaEventElapsedTime(&ms, b0, b1);
    cudaEventDestroy(b0); cudaEventDestroy(b1);
    *ms_per_body = ms / reps;
    return DCREG_OK;
}

int dcreg_iteration_timeline(dcreg_ctx* ctx, const dcreg_icp_params* params, const double T[16], int iters, uint64_t* out,
                             int out_cap_blocks, int* n_blocks) {
    if (!ctx || !params || !T || iters < 1 || !out || !n_blocks) return DCREG_BAD_ARG;
    if (!ctx->d_src || !ctx->has_grid) { ctx->err = "iteration_timeline: set source and target first"; return DCREG_BAD_ARG; }
    CK(cudaSetDevice(ctx->device));
    dcreg_icp_params prm = *params;
    prm.fixed_iterations = 1;
    prm.max_iterations = iters + 8;
    int rc;
    if ((rc = init_state(ctx, T))) return rc;
    const float4* src_iter = ctx->d_src;
    if ((rc = sort_source_by_cell(ctx, T, &src_iter))) return rc;
    LoopPlan L;
    if ((rc = plan_iteration(ctx, &prm, src_iter, nullptr, 1, nullptr, 0, true, &L))) return rc;
    *n_blocks = L.grid_x;
    if (out_cap_blocks < L.grid_x + 1) { ctx->err = "iteration_timeline: output too small"; return DCREG_BAD_ARG; }
    const size_t bytes = (size_t)(L.grid_x + 1) * kStampSlots * sizeof(unsigned long long);
    unsigned long long* d_st = nullptr;
    CK(cudaMalloc(&d_st, bytes));
    CK(cudaMemsetAsync(d_st, 0, bytes, ctx->stream));
    for (int i = 0; i + 1 < iters && rc == DCREG_OK; ++i) rc = launch_body(ctx, L, &prm, nullptr, 0, true);
    L.b.stamps = d_st;
    if (rc == DCREG_OK) rc = launch_body(ctx, L, &prm, nullptr, 0, true);
    if (rc == DCREG_OK) {
        cudaMemcpyAsync(out, d_st, bytes, cudaMemcpyDeviceToHost, ctx->stream);
        if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) { ctx->err = "iteration_timeline: stream error"; rc = DCREG_CUDA_ERROR; }
    }
    cudaFree(d_st);
    return rc;
}

int dcreg_analyze_and_solve(dcreg_ctx* ctx, const double H27[27], const dcreg_icp_params* params,
                            dcreg_analysis* out, double dx[6]) {
    if (!ctx) return DCREG_BAD_ARG;
    if (!H27 || !params || !out || !dx) { ctx->err = "analyze_and_solve: null pointer"; return DCREG_BAD_ARG; }
    CK(cudaSetDevice(ctx->device));
    CK(cudaMemcpyAsync(ctx->d_small, H27, 27 * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    k2_analyze_kernel<<<1, 32, 0, ctx->stream>>>(ctx->d_small, *params, ctx->d_analysis, ctx->d_small + 32);
    ctx->launches++;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out, ctx->d_analysis, sizeof(dcreg_analysis), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(dx, ctx->d_small + 32, 6 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    for (int i = 0; i < 6; ++i)
        if (!isfinite(dx[i])) return DCREG_NONFINITE_UPDATE;
    return DCREG_OK;
}

int dcreg_solve_pcg(dcreg_ctx* ctx, const double A[36], const double b[6], const double P[36], int max_iterations,
                    double tolerance, double x[6], int* iterations) {
    if (!ctx) return DCREG_BAD_ARG;
    if (!A || !b || !P || !x) { ctx->err = "solve_pcg: null pointer"; return DCREG_BAD_ARG; }
    CK(cudaSetDevice(ctx->device));
    double* d = ctx->d_small;
    CK(cudaMemcpyAsync(d, A, 36 * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(d + 36, b, 6 * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(d + 48, P, 36 * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    pcg_kernel<<<1, 32, 0, ctx->stream>>>(d, d + 36, d + 48, max_iterations, tolerance, d + 96, (int*)(d + 128));
    ctx->launches++;
    CK(cudaGetLastError());
    int it = 0;
    CK(cudaMemcpyAsync(x, d + 96, 6 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(&it, d + 128, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (iterations) *iterations = it;
    return DCREG_OK;
}

// FNV-1a over the bytes that define a captured chunk of the loop
static void key_bytes(std::vector<unsigned char>& k, const void* p, size_t n) {
    const unsigned char* c = (const unsigned char*)p;
    k.insert(k.end(), c, c + n);
}

// Enqueue `iters` loop bodies.  The bodies are identical launches (pose, mode flags and the done flag live on the
// device), so a chunk is captured once into a CUDA graph and replayed: one host call per chunk instead of one or two
// launches per iteration - what keeps independent ranks from queueing behind the host.  Falls back to plain launches if capture is unavailable.
static int enqueue_iterations(dcreg_ctx* ctx, LoopPlan& L, const dcreg_icp_params* prm, dcreg_iter_log* dlog, int log_cap, int iters) {
    const bool graphable = !ctx->graph_off && !L.b.force && iters > 1 &&
                           (!L.k2 || !(ctx->comm && !ctx->peer_ok));              // no NCCL call inside a capture
    if (graphable) {
        std::vector<unsigned char> key;
        Iter2Args kb = L.b;
        kb.use_seeds = 0;
        key_bytes(key, &kb, sizeof(kb));
        // (the variant: the kernel, e.g. kSparse at the same Iter2Args; k2: whether a K2 launch follows every iteration
        // kernel, which a mix of per-lane settings decides at the same Iter2Args)
        const int meta[5] = {L.grid_x, L.trials, L.variant, iters, L.k2 ? 1 : 0};
        key_bytes(key, meta, sizeof(meta));
        key_bytes(key, prm, sizeof(*prm));
        cudaGraphExec_t exec = nullptr;
        for (size_t gi = 0; gi < ctx->graphs.size(); ++gi)
            if (ctx->graphs[gi].key == key) {
                if (gi != 0) std::swap(ctx->graphs[gi], ctx->graphs[0]);
                exec = ctx->graphs[0].exec;
                break;
            }
        if (!exec) {
            cudaGraph_t graph = nullptr;
            const bool nn_valid0 = ctx->nn_valid;
            const long long launches0 = ctx->launches;
            cudaError_t e = cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeRelaxed);
            int rc = DCREG_OK;
            if (e == cudaSuccess) {
                for (int k = 0; k < iters && rc == DCREG_OK; ++k) rc = launch_body(ctx, L, prm, dlog, log_cap, true);
                e = cudaStreamEndCapture(ctx->stream, &graph);
            }
            ctx->nn_valid = nn_valid0; ctx->launches = launches0;      // nothing has run yet
            if (e == cudaSuccess && rc == DCREG_OK && graph) e = cudaGraphInstantiate(&exec, graph, 0);
            if (graph) cudaGraphDestroy(graph);
            if (e != cudaSuccess || rc != DCREG_OK || !exec) {
                cudaGetLastError();                                    // clear; run without a graph from now on
                exec = nullptr; ctx->graph_off = true;
            } else {
                if (ctx->graphs.size() >= 4) { cudaGraphExecDestroy(ctx->graphs.back().exec); ctx->graphs.pop_back(); }
                ctx->graphs.insert(ctx->graphs.begin(), dcreg_ctx::LoopGraph{key, exec});
            }
        }
        if (exec) {
            CK(cudaGraphLaunch(exec, ctx->stream));
            ctx->nn_valid = true;
            ctx->launches += (long long)iters * (L.k2 ? 2 : 1); ctx->graph_launches++;
            return DCREG_OK;
        }
    }
    for (int k = 0; k < iters; ++k) {
        const int rc = launch_body(ctx, L, prm, dlog, log_cap, true);
        if (rc) return rc;
    }
    return DCREG_OK;
}

// Enqueue up to `cap` loop bodies in chunks of `chunk`, with a peek at the number of running trials between chunks when
// `peek` (the only host sync inside a run; bodies past a trial's end exit at once on the device).  After the first
// chunk, a short last chunk is padded to `chunk` bodies, so each run shape has one graph.  The peek reads through
// h_pinned (start_loop).
static int run_chunks(dcreg_ctx* ctx, LoopPlan& L, const dcreg_icp_params* prm, dcreg_iter_log* dlog, int log_cap,
                      long long cap, int chunk, bool peek) {
    for (long long issued = 0; issued < cap;) {
        const long long todo = std::min<long long>(cap - issued, chunk);
        const int bodies = (todo < chunk && issued > 0) ? chunk : (int)todo;
        const int rc = enqueue_iterations(ctx, L, prm, dlog, log_cap, bodies);
        if (rc) return rc;
        issued += bodies;
        if (peek && issued < cap) {
            unsigned int* flag = (unsigned int*)ctx->h_pinned.p;       // every solve step that finishes a trial decrements it
            CK(cudaMemcpyAsync(flag, ctx->d_n_active, sizeof(unsigned int), cudaMemcpyDeviceToHost, ctx->stream));
            CK(cudaStreamSynchronize(ctx->stream));
            if (*flag == 0u) break;
        }
    }
    return DCREG_OK;
}

// Where a call's per-trial outputs go, in the caller's order (null: not wanted)
struct Results {
    double* T_out = nullptr;
    int* n_iterations = nullptr;
    int* converged = nullptr;
    int* status = nullptr;
    dcreg_iter_log* log = nullptr;
    int log_cap = 0;                 // records per trial
    double* cov = nullptr;           // [trials][36] by covariance_kernel's rule
    double* T_prior = nullptr;       // [trials][16] the prior each frame started from (lanes)
};

// The device log of `trials` registrations when the call wants one (*dlog = null otherwise), zeroed: aborted iterations
// leave fields untouched
static int setup_log(dcreg_ctx* ctx, const Results& r, int trials, dcreg_iter_log** dlog) {
    *dlog = nullptr;
    if (!r.log || r.log_cap <= 0) return DCREG_OK;
    const long long records = (long long)trials * r.log_cap;
    CK(ctx->d_log.ensure(records));
    CK(cudaMemsetAsync(ctx->d_log, 0, (size_t)records * sizeof(dcreg_iter_log), ctx->stream));
    *dlog = ctx->d_log;
    return DCREG_OK;
}

// Before a loop: the log, every trial's state, the sources in sort order (the context's source, or the staged sources of
// a batch), the lanes' first priors, and the pinned buffer of the peeks and read_results
static int start_loop(dcreg_ctx* ctx, int trials, const double* T_init, const Results& r, const Batch* batch,
                      dcreg_iter_log** dlog, const float4** src) {
    const bool lanes = batch && batch->lanes > 0;
    int rc;
    if ((rc = setup_log(ctx, r, trials, dlog))) return rc;
    if ((rc = init_state(ctx, T_init, trials, batch ? ctx->d_scan_seg.p : nullptr, lanes ? batch->lanes : trials))) return rc;
    if (batch) rc = sort_sources(ctx, *batch, src);
    else rc = sort_source_by_cell(ctx, T_init, src);             // locality only: any pose of the batch will do
    if (rc) return rc;
    if (lanes)         // a lane's first prior is its T_init; the frame advance writes the others
        CK(cudaMemcpyAsync(batch->seq.T_prior, ctx->d_T_init, (size_t)trials * 16 * sizeof(double), cudaMemcpyDeviceToDevice,
                           ctx->stream));
    CK(ctx->h_pinned.ensure((long long)trials * sizeof(IcpState)));
    return DCREG_OK;
}

// The end of a call, after its loop: the log's fill-in, the results, then the covariances and the priors when asked for.
// dev (odometry): the caller's trial k is device trial dev[k], and only the device trials below `done` are returned;
// null: the same order, every trial.  lanes (per-lane settings, in the context's lane table): device trial t's record
// takes lane trial_lane[t]'s, or lane t's without trial_lane.
static int finish_call(dcreg_ctx* ctx, const dcreg_icp_params* prm, int trials, dcreg_iter_log* dlog, const Results& r,
                       const int* dev = nullptr, int done = 0, const Lanes& lanes = Lanes{},
                       const int* trial_lane = nullptr) {
    if (dlog) {
        const int* d_trial_lane = nullptr;
        if (lanes.n && trial_lane) {
            CK(ctx->d_trial_lane.ensure(trials));
            CK(cudaMemcpyAsync(ctx->d_trial_lane, trial_lane, (size_t)trials * sizeof(int), cudaMemcpyHostToDevice,
                               ctx->stream));
            d_trial_lane = ctx->d_trial_lane;
        }
        log_fill_kernel<<<dim3((r.log_cap + 31) / 32, trials), 32, 0, ctx->stream>>>(
            dlog, r.log_cap, ctx->d_state, *prm, lanes.n ? ctx->d_lane_prm.p : nullptr, d_trial_lane);
        ctx->launches++;
    }
    // device order: straight into the caller's arrays, or into host copies that are put in the caller's order below
    Results d = r;
    std::vector<double> To, cv, Tp;
    std::vector<int> it, cg, st;
    std::vector<dcreg_iter_log> lg;
    if (dev) {
        To.resize((size_t)trials * 16); it.resize(trials); cg.resize(trials); st.resize(trials);
        d.T_out = To.data(); d.n_iterations = it.data(); d.converged = cg.data(); d.status = st.data();
        if (dlog) { lg.resize((size_t)trials * r.log_cap); d.log = lg.data(); }
        if (r.cov) { cv.resize((size_t)trials * 36); d.cov = cv.data(); }
        if (r.T_prior) { Tp.resize((size_t)trials * 16); d.T_prior = Tp.data(); }
    }
    int rc = read_results(ctx, trials, d.T_out, dlog ? d.log : nullptr, r.log_cap, d.n_iterations, d.converged, d.status);
    if (rc) return rc;
    if (r.cov) {
        covariance_kernel<<<trials, 32, 0, ctx->stream>>>(ctx->d_state, ctx->d_scan_cov);
        ctx->launches++;
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(d.cov, ctx->d_scan_cov, (size_t)trials * 36 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    }
    if (r.T_prior)
        CK(cudaMemcpyAsync(d.T_prior, ctx->d_seq_prior, (size_t)trials * 16 * sizeof(double), cudaMemcpyDeviceToHost,
                           ctx->stream));
    if (r.cov || r.T_prior) CK(cudaStreamSynchronize(ctx->stream));
    if (!dev) return DCREG_OK;
    for (int k = 0; k < trials; ++k) {
        const size_t t = (size_t)dev[k];
        if ((int)t >= done) continue;
        memcpy(r.T_out + (size_t)k * 16, &To[t * 16], 16 * sizeof(double));
        if (r.n_iterations) r.n_iterations[k] = it[t];
        if (r.converged) r.converged[k] = cg[t];
        if (r.status) r.status[k] = st[t];
        if (dlog) memcpy(r.log + (size_t)k * r.log_cap, &lg[t * r.log_cap], (size_t)r.log_cap * sizeof(dcreg_iter_log));
        if (r.cov) memcpy(r.cov + (size_t)k * 36, &cv[t * 36], 36 * sizeof(double));
        if (r.T_prior) memcpy(r.T_prior + (size_t)k * 16, &Tp[t * 16], 16 * sizeof(double));
    }
    return DCREG_OK;
}

// The loop for `trials` registrations side by side: of the context's source (batch null), or of the staged sources of a
// batch (stage_sources), whose lanes, if any, run the trials as frames.  fetch = false: enqueue only (no host
// synchronisation at all: no peek between chunks, no read-back).  lane_set: per-lane settings (params is entry 0), one per
// trial, or (batch lanes) one per lane with trial_lane the lane of every trial
static int run_loop(dcreg_ctx* ctx, const dcreg_icp_params* params, int trials, const double* T_init, const Results& r,
                    bool fetch = true, const Batch* batch = nullptr, const Lanes& lane_set = Lanes{},
                    const int* trial_lane = nullptr) {
    dcreg_iter_log* dlog = nullptr;
    const float4* src = nullptr;
    int rc = start_loop(ctx, trials, T_init, r, batch, &dlog, &src);
    if (rc) return rc;
    const bool lanes = batch && batch->lanes > 0;
    LoopPlan L;
    if ((rc = plan_iteration(ctx, params, src, nullptr, lanes ? batch->lanes : trials, dlog, dlog ? r.log_cap : 0, true, &L,
                             batch, lane_set)))
        return rc;
    // fixed iteration count: the whole run is one chunk; otherwise chunks of 16 with a peek in between.  Lanes: chunks
    // of 16 with a peek at the lanes still running, up to max_bodies (a frame never needs more than max_iterations
    // bodies), whatever fixed_iterations says
    const long long cap = lanes ? batch->max_bodies : params->max_iterations;
    const int chunk = params->fixed_iterations && !lanes ? std::min(params->max_iterations, 64) : 16;
    const bool peek = fetch && (lanes || !params->fixed_iterations);
    if ((rc = run_chunks(ctx, L, params, dlog, dlog ? r.log_cap : 0, cap, chunk, peek))) return rc;
    if (!fetch) return DCREG_OK;
    return finish_call(ctx, params, trials, dlog, r, nullptr, 0, lane_set, trial_lane);
}

// need_source = false: the run brings its own source points (dcreg_icp_run_scans); need_target = false: and its own
// targets (dcreg_icp_run_pairs)
static int check_run_args(dcreg_ctx* ctx, const dcreg_icp_params* params, bool need_source = true, bool need_target = true) {
    if (need_source && (!ctx->d_src || ctx->n_src <= 0)) { ctx->err = "[ICP Error] Input measure cloud is null or empty."; return DCREG_BAD_ARG; }
    if (need_target && !ctx->has_grid) { ctx->err = "[ICP Error] Target index is not set up in context."; return DCREG_BAD_ARG; }
    if (params->max_iterations < 0) { ctx->err = "icp_run: max_iterations < 0"; return DCREG_BAD_ARG; }
    if (!(params->weight_slope > 0.0) || !(params->weight_gate >= 0.0) || !(params->weight_gate < 1.0)) {
        ctx->err = "icp_run: weight_slope must be > 0 and weight_gate in [0, 1)";
        return DCREG_BAD_ARG;
    }
    return DCREG_OK;
}

int dcreg_icp_run(dcreg_ctx* ctx, const dcreg_icp_params* params, const double T_init[16], double T_out[16],
                  dcreg_iter_log* log, int log_cap, int* n_iterations, int* converged) {
    if (!ctx) return DCREG_BAD_ARG;
    if (!params || !T_init || !T_out) { ctx->err = "icp_run: null pointer"; return DCREG_BAD_ARG; }
    int rc = check_run_args(ctx, params);
    if (rc) return rc;
    CK(cudaSetDevice(ctx->device));
    int status = DCREG_OK;
    if ((rc = run_loop(ctx, params, 1, T_init, Results{T_out, n_iterations, converged, &status, log, log_cap}))) return rc;
    return status;
}

int dcreg_icp_enqueue(dcreg_ctx* ctx, const dcreg_icp_params* params, const double T_init[16]) {
    if (!ctx) return DCREG_BAD_ARG;
    if (!params || !T_init) { ctx->err = "icp_enqueue: null pointer"; return DCREG_BAD_ARG; }
    int rc = check_run_args(ctx, params);
    if (rc) return rc;
    CK(cudaSetDevice(ctx->device));
    return run_loop(ctx, params, 1, T_init, Results{}, false);
}

int dcreg_icp_fetch(dcreg_ctx* ctx, double T_out[16], int* n_iterations, int* converged) {
    if (!ctx) return DCREG_BAD_ARG;
    if (!T_out) { ctx->err = "icp_fetch: null pointer"; return DCREG_BAD_ARG; }
    CK(cudaSetDevice(ctx->device));
    int status = DCREG_OK;
    const int rc = read_results(ctx, 1, T_out, nullptr, 0, n_iterations, converged, &status);
    return rc ? rc : status;
}

// What a batched call (dcreg_icp_run_batch, _scans, _pairs, _sequences, _odometry) needs checked before anything is
// launched.  Every message of its own starts with the call's name.
struct BatchCheck {
    const char* name;                   // "icp_run_scans"
    bool args_ok;                       // no null pointer, positive counts ...
    const char* args_msg;               // ... or what is wrong
    const char* shard_msg;              // why a sharded context is refused
    int n;                              // trials: at most kMaxPairs (the loop kernel's grid y)
    const int64_t* offsets = nullptr;   // the sources' table (null: trials of the context's source) ...
    const char* item = nullptr;         // ... and what a source is called in its messages
    int stride = 3;
    bool own_cell = false;              // the call builds its own grids with cell_size (search rings in [1, 4])
    double cell_size = 0.0;
    const char* own_msg = nullptr;      // a check of the call's own that failed, reported after the cell size
    bool need_source = false, need_target = true;    // check_run_args
    bool one_iteration = false;         // max_iterations >= 1
    int n_seqs = 0;                     // the sequence table [n_seqs + 1]: from 0, ascending strictly, up to n
    const int* seq_offsets = nullptr;
    bool empty_seqs = false;            // ... or only non-decreasing (dcreg_odometry_push: a sequence may have no frame)
    int lanes = 0;                      // dcreg_set_lane_params: params holds this many entries (0: one)
};

static int check_batch_call(dcreg_ctx* ctx, const dcreg_icp_params* params, const BatchCheck& c) {
    const std::string name(c.name);
    auto bad = [ctx](const std::string& why) { ctx->err = why; return (int)DCREG_BAD_ARG; };
    if (!c.args_ok) return bad(name + ": " + c.args_msg);
    if (c.offsets && c.stride < 3) return bad(name + ": stride < 3");
    if (c.own_cell && !(c.cell_size > 0.0)) return bad(name + ": cell_size <= 0");
    if (c.own_msg) return bad(name + ": " + c.own_msg);
    if (ctx->comm) return bad(name + ": " + c.shard_msg);
    const std::string what = c.item ? name + ": " + c.item : name;
    const std::string too_many = what + ": more than " + std::to_string(arena_plan::kMaxPairs) + " trials in one call";
    if (!c.offsets && c.n > arena_plan::kMaxPairs) return bad(too_many);   // trials of the context's source: no table
    const int rc = check_run_args(ctx, params, c.need_source, c.need_target);
    if (rc) return rc;
    if (c.one_iteration && params->max_iterations < 1) return bad(name + ": max_iterations must be >= 1");
    if (c.own_cell) {
        const int rings = search_rings(params->search_radius, c.cell_size);
        if (rings < 1 || rings > 4) return bad(name + ": search_radius / cell_size must be in (0, 4]");
    }
    if (c.offsets) {
        if (c.n > arena_plan::kMaxPairs) return bad(too_many);
        const std::string why = arena_plan::check_offsets(c.n, c.offsets, arena_plan::kMaxPoints, what.c_str());
        if (!why.empty()) return bad(why);
    }
    if (c.seq_offsets) {
        const int* so = c.seq_offsets;
        if (so[0] != 0) return bad(name + ": seq_offsets must start at 0");
        for (int s = 0; s < c.n_seqs; ++s)
            if (c.empty_seqs ? so[s + 1] < so[s] : so[s + 1] <= so[s])
                return bad(name + ": sequence " + std::to_string(s) +
                           (c.empty_seqs ? " has a negative frame count (seq_offsets must not decrease)"
                                         : " is empty (seq_offsets must ascend strictly)"));
        if (so[c.n_seqs] != c.n)
            return bad(name + ": seq_offsets[n_seqs] = " + std::to_string(so[c.n_seqs]) + " but n_frames = " + std::to_string(c.n));
    }
    // the fields every lane shares equal entry 0's, whose checks above are then every entry's
    const std::string why = lane_plan::check_common(params, c.lanes, c.name);
    if (!why.empty()) return bad(why);
    return DCREG_OK;
}

int dcreg_icp_run_batch(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_trials, const double* T_init,
                        double* T_out, int* n_iterations, int* converged, int* status, dcreg_iter_log* log, int log_cap) {
    if (!ctx) return DCREG_BAD_ARG;
    BatchCheck c{"icp_run_batch", params && T_init && T_out && n_trials > 0, "null pointer or n_trials <= 0",
                 "trials are independent - distribute them over ranks, do not shard them", n_trials};
    c.need_source = true;
    c.lanes = ctx->lane_params ? n_trials : 0;
    int rc = check_batch_call(ctx, params, c);
    if (rc) return rc;
    CK(cudaSetDevice(ctx->device));
    return run_loop(ctx, params, n_trials, T_init, Results{T_out, n_iterations, converged, status, log, log_cap}, true,
                    nullptr, call_lanes(params, n_trials, ctx->lane_params));
}

int dcreg_icp_run_scans(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_scans, const float* xyz,
                        const int64_t* scan_offsets, int stride, const double* T_init, double* T_out, int* n_iterations,
                        int* converged, int* status, double* cov, dcreg_iter_log* log, int log_cap) {
    if (!ctx) return DCREG_BAD_ARG;
    BatchCheck c{"icp_run_scans", params && n_scans > 0 && xyz && scan_offsets && T_init && T_out,
                 "null pointer or n_scans <= 0", "scans are independent - distribute them over ranks, do not shard them",
                 n_scans};
    c.offsets = scan_offsets; c.item = "scan"; c.stride = stride;
    c.lanes = ctx->lane_params ? n_scans : 0;
    int rc = check_batch_call(ctx, params, c);
    if (rc) return rc;
    CK(cudaSetDevice(ctx->device));
    const Batch S{n_scans, xyz, stride, scan_offsets};
    if ((rc = stage_sources(ctx, S))) return rc;
    return run_loop(ctx, params, n_scans, T_init, Results{T_out, n_iterations, converged, status, log, log_cap, cov}, true,
                    &S, call_lanes(params, n_scans, ctx->lane_params));
}

int dcreg_icp_run_sequences(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_seqs, const int* seq_offsets,
                            int n_frames, const float* xyz, const int64_t* frame_offsets, int stride,
                            const double* T_init, const double* deltas, double* T_prior, double* T_out,
                            int* n_iterations, int* converged, int* status, double* cov, dcreg_iter_log* log,
                            int log_cap) {
    if (!ctx) return DCREG_BAD_ARG;
    BatchCheck c{"icp_run_sequences", params && n_seqs > 0 && n_frames > 0 && seq_offsets && xyz && frame_offsets && T_init && T_out,
                 "null pointer, n_seqs <= 0 or n_frames <= 0",
                 "sequences are independent - give each rank its own, do not shard them", n_frames};
    c.offsets = frame_offsets; c.item = "frame"; c.stride = stride; c.one_iteration = true;
    c.n_seqs = n_seqs; c.seq_offsets = seq_offsets;
    c.lanes = ctx->lane_params ? n_seqs : 0;
    int rc = check_batch_call(ctx, params, c);
    if (rc) return rc;
    CK(cudaSetDevice(ctx->device));
    // every frame is sorted by target cell under its dead-reckoned prior (T_init composed with the increments alone):
    // the sort only buys locality, and the chained prior is not known before the frame before it has run
    static const double kIdentity[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    std::vector<double> T_dr((size_t)n_frames * 16);
    Batch S{n_frames, xyz, stride, frame_offsets};
    S.lanes = n_seqs;
    for (int s = 0; s < n_seqs; ++s) {
        const int f0 = seq_offsets[s], f1 = seq_offsets[s + 1];
        memcpy(&T_dr[(size_t)f0 * 16], T_init + (size_t)s * 16, 16 * sizeof(double));
        for (int f = f0 + 1; f < f1; ++f) {
            const double* T = &T_dr[(size_t)(f - 1) * 16];
            const double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]}, t[3] = {T[3], T[7], T[11]};
            compose_prior(R, t, deltas ? deltas + (size_t)(f - 1) * 16 : kIdentity, &T_dr[(size_t)f * 16]);
        }
        S.max_bodies = std::max<long long>(S.max_bodies, (long long)(f1 - f0) * params->max_iterations);
    }
    if ((rc = stage_sources(ctx, S)) || (rc = stage_lanes(ctx, n_seqs, n_frames, &S.seq))) return rc;
    CK(cudaMemcpyAsync(ctx->d_seq_first, seq_offsets, (size_t)(n_seqs + 1) * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->d_seq_cursor, seq_offsets, (size_t)n_seqs * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    if (deltas) {
        CK(cudaMemcpyAsync(ctx->d_seq_delta, deltas, (size_t)n_frames * 16 * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        S.seq.delta = ctx->d_seq_delta;
    }
    // (per-lane settings) every frame's record takes its sequence's
    std::vector<int> frame_seq((size_t)n_frames);
    for (int s = 0; s < n_seqs; ++s)
        for (int f = seq_offsets[s]; f < seq_offsets[s + 1]; ++f) frame_seq[(size_t)f] = s;
    return run_loop(ctx, params, n_frames, T_dr.data(),
                    Results{T_out, n_iterations, converged, status, log, log_cap, cov, T_prior}, true, &S,
                    call_lanes(params, n_seqs, ctx->lane_params), frame_seq.data());
}

// The settings of a one-shot call (dcreg_icp_run_odometry: source_voxel = map_voxel = 0, caps of 1; _voxel: caps of 1)
// or of a session (dcreg_odometry_open).  A voxel size of 0 leaves its filter out entirely: no launch, no copy, no sync.
// T_init stays empty when params or T_init is null or n_seqs <= 0, which the checks report as a null pointer; no valid
// call has more than kMaxPairs sequences, so no more are read before the checks reject it.  lanes: params holds one
// entry per sequence (dcreg_set_lane_params), read the same way.
static OdomSettings odom_settings(const dcreg_icp_params* params, int n_seqs, double cell_size, int map_frames,
                                  int motion, double source_voxel, double map_voxel, int source_max_points,
                                  int map_max_points, const double* T_init, bool lanes) {
    OdomSettings set{params ? *params : dcreg_icp_params{}, n_seqs, map_frames, motion, source_max_points, map_max_points,
                     cell_size, source_voxel, map_voxel};
    if (params && T_init && n_seqs > 0) {
        set.T_init.assign(T_init, T_init + (size_t)std::min(n_seqs, arena_plan::kMaxPairs) * 16);
        if (lanes) set.lanes.assign(params, params + std::min(n_seqs, arena_plan::kMaxPairs));
    }
    return set;
}

// The settings of a filtered one-shot call (every dcreg_icp_run_odometry_* but dcreg_icp_run_odometry itself) with the
// context's dcreg_set_map_input_voxel
static OdomSettings with_map_input(OdomSettings set, const dcreg_ctx* ctx) {
    if (ctx) set.map_input_voxel = ctx->map_input_voxel;
    return set;
}

// How far R_sensor_imu^T R_sensor_imu may be from I, entry by entry
constexpr double kGyroOrthoTol = 1e-6;

// What is wrong with the settings of an odometry call or session, or null
static const char* odometry_settings_error(const OdomSettings& set, bool deltas) {
    if (!set.voxel_map && set.map_frames < 1) return "map_frames must be >= 1";
    if (set.motion != DCREG_MOTION_INCREMENTS && set.motion != DCREG_MOTION_CONSTANT_VELOCITY)
        return "motion must be DCREG_MOTION_INCREMENTS or DCREG_MOTION_CONSTANT_VELOCITY";
    if (set.motion == DCREG_MOTION_CONSTANT_VELOCITY && deltas) return "the constant-velocity model takes no deltas (pass NULL)";
    if (!(set.source_voxel >= 0.0 && set.source_voxel < INFINITY) || !(set.map_voxel >= 0.0 && set.map_voxel < INFINITY))
        return "source_voxel and map_voxel must be finite and >= 0 (0: no filter)";
    if (set.source_max_points < 1 || set.map_max_points < 1) return "source_max_points and map_max_points must be >= 1";
    if (set.voxel_map && !(set.map_voxel > 0.0)) return "the voxel map needs a map_voxel > 0";
    if (set.voxel_map && !(set.max_distance > 0.0)) return "max_distance must be > 0 (+inf: no pruning), not NaN";
    const adaptive::Settings& a = set.threshold;
    if (set.adaptive && !(a.initial_threshold > 0.0 && a.initial_threshold < INFINITY && a.min_motion >= 0.0 &&
                          a.min_motion < INFINITY && a.max_range > 0.0 && a.max_range < INFINITY))
        return "adaptive: initial_threshold and max_range must be finite and > 0, min_motion finite and >= 0";
    if (set.gyro) {
        if (set.motion != DCREG_MOTION_CONSTANT_VELOCITY || deltas)
            return "gyro input needs DCREG_MOTION_CONSTANT_VELOCITY and deltas == NULL (the gyro gives the rotation)";
        const se3::Gyro& g = set.gyro_set;
        bool finite = true;
        for (int i = 0; i < 9; ++i) finite = finite && std::isfinite(g.R_si[i]);
        if (!finite) return "gyro: R_sensor_imu has an entry that is not finite";
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) {
                const double e = (g.R_si[r] * g.R_si[c] + g.R_si[3 + r] * g.R_si[3 + c]) + g.R_si[6 + r] * g.R_si[6 + c];
                if (!(std::fabs(e - (r == c ? 1.0 : 0.0)) <= kGyroOrthoTol))
                    return "gyro: R_sensor_imu is not a rotation (an entry of R^T R - I exceeds 1e-6)";
            }
        if (!(std::isfinite(g.bias[0]) && std::isfinite(g.bias[1]) && std::isfinite(g.bias[2])))
            return "gyro: bias has an entry that is not finite";
    }
    if (set.imu) {
        bool finite = true;
        for (int i = 0; i < 3; ++i) finite = finite && std::isfinite(set.accel_bias[i]);
        if (!finite) return "imu: accel_bias has an entry that is not finite";
        for (int i = 0; i < 3; ++i) finite = finite && std::isfinite(set.gravity[i]);
        if (!finite) return "imu: gravity has an entry that is not finite";
    }
    return nullptr;
}

// (IMU) The sequence whose v_init has an entry that is not finite, as a message, or empty
static std::string v_init_error(const OdomSettings& set) {
    for (size_t i = 0; set.imu && i < set.v_init.size(); ++i)
        if (!std::isfinite(set.v_init[i]))
            return "imu: v_init of sequence " + std::to_string(i / 3) + " has an entry that is not finite";
    return std::string();
}

// A step's maps (or a session's final voxel-map update): segment b is points [d_seg[b], d_seg[b + 1]) of `map` (null:
// not built); with a map filter its kept offsets and range flags come back with the next copy of `more`
struct StepMap {
    const float4* map = nullptr;
    const long long* d_seg = nullptr;
    std::vector<int64_t> kept;          // (map filter) [segs + 1]
    std::vector<int> bad;               // (map filter) [segs]
    std::vector<Readback> more;
};

// The gyro input of a call or push (dcreg_icp_run_odometry_gyro, dcreg_odometry_push_gyro): frame_times [n_frames][2]
// (start, span), samples [rows][4] (t, wx, wy, wz), sequence s's rows [sample_offsets[s], sample_offsets[s + 1])
// (dcreg_icp_run_odometry_imu, dcreg_odometry_push_imu) samples [rows][7] (t, wx, wy, wz, ax, ay, az): stride
// se3::kImuStride, and velocity (out, may be null) [n_frames][3]
struct GyroInput {
    const double* frame_times = nullptr;
    const double* samples = nullptr;
    const int64_t* sample_offsets = nullptr;
    int stride = se3::kSampleStride;
    double* velocity = nullptr;
};

// One odometry call or push (run_odometry): its arguments, what its phases share, and the phases, in the order they run
struct OdomCall {
    dcreg_ctx* ctx; const char* name; const OdomSettings& set; dcreg_ctx::OdomSession* sess;
    const int* seq_offsets; int n_frames; const float* xyz; const int64_t* frame_offsets; int stride;
    const double* deltas; const float* timestamps; const Results& R; int64_t* frame_points; float* deskewed_xyz;
    double* search_radius;                          // (out, may be null) the radius every frame registered with; anchors 0
    GyroInput gi;                                   // (set.gyro) the frames' times and the samples, or all null
    const int n_seqs = set.n_seqs;
    const dcreg_icp_params* params = &set.params;
    // (dcreg_set_lane_params) every sequence's settings, indexed through the step's lane -> sequence table d_lane_seq
    const Lanes lanes = call_lanes(set.lanes.data(), (int)set.lanes.size(), true);
    odom_plan::History none;                        // a one-shot call's history, once check() has validated n_seqs
    const odom_plan::History& hist = sess ? sess->hist : none;
    // the frames as the device gets them: the caller's, or the source filter's kept points (src_off: kept offsets)
    const float* src_xyz = xyz; int src_stride = stride; const int64_t* src_off = frame_offsets;
    std::vector<int64_t> kept;
    // (dcreg_set_prior_map) every frame registers against the context's target: no anchors, no maps (odom_plan.hpp)
    const bool prior = sess ? set.prior_map : ctx->prior_map;
    std::vector<double> next_dr;                    // (prior, sess) every sequence's dead-reckoned pose after the push
    std::vector<double> first_r;                    // (prior, adaptive) the radii of step 0's lanes, from the host
    // (dcreg_set_map_input_voxel, not read with a prior map) the frames' filter is the map-input filter F_in, whose
    // kept points are the maps' input; split: a source filter F_s runs over them (voxel_filter_chain), and in_off
    // (F_in's kept offsets) differs from src_off.  d_map_src: the points the maps and a session's window take, the
    // packed sources or (split) d_odom_in
    const double in_voxel = prior ? 0.0 : set.map_input_voxel;
    const bool split = in_voxel > 0.0 && set.source_voxel > 0.0;
    const bool filtered = in_voxel > 0.0 || set.source_voxel > 0.0;
    const int64_t* in_off = frame_offsets;
    std::vector<int64_t> in_kept;
    size_t in_ll = 0;                               // (split) where the map-input offsets are in d_odom_ll
    const float4* d_map_src = nullptr;
    odom_plan::Push U;
    const odom_plan::Plan& P = U.plan;
    // where the tables are in d_odom_ll / d_odom_int: step i's map's (odom_plan::pack), then its int prev, prev2 and
    // (adaptive) the threshold kernel's seq, next_lane; the retain step's and the timestamp gather's
    std::vector<size_t> at_ll, at_int;
    size_t keep_ll = 0, keep_int = 0, ts_ll = 0;
    Batch S{};
    const double* d_delta = nullptr;                // one increment per frame reference (null: every one the identity)
    const double* d_hist_T = nullptr;               // the retained frames' poses and points (null: none)
    const float4* d_win = nullptr;
    dcreg_iter_log* dlog = nullptr; const float4* src_iter = nullptr;
    LoopPlan L; bool planned = false;
    // (sparse_maps) the plan of the steps whose maps are sparse row indexes, made at the first such step
    const bool sparse_maps = sess ? set.sparse_maps : ctx->sparse_maps;
    LoopPlan L_sparse; bool planned_sparse = false;
    bool sparse = false;            // the step's grids are sparse row indexes (sparse_maps: a lane's box, or the step's
                                    // boxes in all, too large for dense grids; prior: the target is one)
    std::vector<int> lane_rings;    // (window, adaptive) the step's lanes' rings
    const double map_spacing = sess ? set.map_spacing : ctx->map_spacing;   // the map filter's minimum spacing
    int failed = -1;                                // the step whose maps failed (-1: none)
    // (voxel map) where every sequence's map is: the session's maps before the first update, then each update's output
    odom_plan::MapState MS;
    const float4* d_old = nullptr;
    std::vector<double> frame_radius;               // [n_frames] the caller's frames' radii, as their steps run
    // (set.gyro) every frame's (start, span, tm, tm_prev) and whether it is an anchor, in the caller's order; every
    // sequence's last mid-sweep time after the push; where the knot offsets and sample ranges are in d_odom_ll
    std::vector<double> gyro_ft;
    std::vector<char> gyro_anchor;
    std::vector<double> next_mid;
    size_t gyro_ll = 0;
    long long gyro_knots = 0;
    // (set.imu) every frame reference's velocity in device order [n_frames + retained][3]: v_init (a first frame), the
    // session's last (a sequence's last retained frame), then the frames' as the call computed them (finish)
    std::vector<double> imu_v;
    OdomImu imu_dev;                                // (set.imu, samples given) what the kernels read

    int check(), check_gyro(), upload(), start(), step(int i), finish();
    int prior_grids(int i), window_grids(int i), step_run(int i);
    const char* prior_error() const;
    int build_map(const odom_plan::MapInput& in, const long long* ll, const int* ints, DevBuf<float4>& out, StepMap* sm);

    // the sequence of the caller's frame k
    int frame_seq_of(int k) const {
        return (int)(std::upper_bound(seq_offsets, seq_offsets + n_seqs + 1, k) - seq_offsets) - 1;
    }
    // "sequence s, frame k (frame j of the sequence)": the caller's frame k, j-th of sequence s in the call, or its
    // number since the session opened
    std::string frame_name(int s, int k) const {
        const int j = k - seq_offsets[s];
        if (!sess)
            return "sequence " + std::to_string(s) + ", frame " + std::to_string(k) + " (frame " + std::to_string(j) +
                   " of the sequence)";
        return "sequence " + std::to_string(s) + ", frame " + std::to_string(k) + " of the push (frame " +
               std::to_string(hist.seen[(size_t)s] + j) + " of the sequence since open)";
    }
    // odom_plan::map_failure's reason, if any, into ctx->err: segment `b` of `in`, a lane of step st or (st null) a
    // session's final update
    bool map_failed(const odom_plan::MapInput& in, const odom_plan::Step* st, const std::string& why, int b) {
        if (why.empty()) return false;
        const int d = st && b < st->active ? st->first + b : in.center[(size_t)b];
        ctx->err = std::string(name) + ": " + frame_name(in.seq[(size_t)b], P.input[(size_t)d]) + ": " + why;
        return true;
    }
};

// The maps of `in`, its tables on the device at ll / ints (null: a voxel-map update's, whose sizes follow the last
// update's results, packed and uploaded here): map_points_kernel into d_odom_map, then with a map filter the capped
// voxel filter into `out`, pruned in the voxel map.  The buffers grow with headroom (a window reserved them for its
// largest step).  An input over arena_plan::kMaxPoints is not built (odom_plan::map_failure names it).  No sync.
int OdomCall::build_map(const odom_plan::MapInput& in, const long long* ll, const int* ints, DevBuf<float4>& out,
                        StepMap* sm) {
    const int segs = (int)in.seq.size(), pieces = (int)in.piece_frame.size();
    const long long m = in.seg.back();
    const bool filter = set.map_voxel > 0.0;
    int rc;
    if (m > arena_plan::kMaxPoints) return DCREG_OK;
    if (!ll) {
        std::vector<long long> hll;
        std::vector<int> hint;
        odom_plan::pack(in, hll, hint);
        CK(ctx->d_vmap_ll.grow((long long)hll.size()));
        CK(ctx->d_vmap_int.grow(std::max<long long>((long long)hint.size(), 1)));
        CK(cudaMemcpyAsync(ctx->d_vmap_ll, hll.data(), hll.size() * sizeof(long long), cudaMemcpyHostToDevice, ctx->stream));
        if (!hint.empty())
            CK(cudaMemcpyAsync(ctx->d_vmap_int, hint.data(), hint.size() * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
        ll = ctx->d_vmap_ll;
        ints = ctx->d_vmap_int;
    }
    CK(ctx->d_odom_map.grow(std::max<long long>(m, 1)));
    if (filter) CK(out.grow(std::max<long long>(m, 1)));
    if (m == 0) {           // no map and no frame to insert anywhere
        CK(ctx->d_vox_seg.ensure(segs + 1));
        CK(ctx->d_vox_bad.ensure(std::max(segs, 1)));
        CK(cudaMemsetAsync(ctx->d_vox_seg, 0, (size_t)(segs + 1) * sizeof(long long), ctx->stream));
        CK(cudaMemsetAsync(ctx->d_vox_bad, 0, (size_t)segs * sizeof(int), ctx->stream));
    } else {
        std::vector<long long> tab;
        const long long slots = filter ? voxel_tables(segs, in.seg.data(), tab) : 0;
        if (filter && (ctx->d_vox_slot.cap < m || ctx->d_vox_keys.cap < slots ||
                       (set.map_max_points > 1 && ctx->d_vox_skey.cap < 2 * m)) &&
            (rc = voxel_reserve(ctx, m + m / 4, n_seqs, slots + slots / 4, set.map_max_points)))
            return rc;
        const long long* d_dst = ll + segs + 1;
        map_points_kernel<<<(unsigned)((m + 255) / 256), 256, 0, ctx->stream>>>(
            d_map_src, d_win, d_old, n_frames, d_dst, pieces, d_dst + pieces + 1, ints, m, ctx->d_state, d_hist_T,
            ctx->d_odom_map);
        ctx->launches++;
        CK(cudaGetLastError());
        const VoxelPrune prune{ints + pieces, n_frames, ctx->d_state, d_hist_T, set.max_distance * set.max_distance};
        if (filter && (rc = voxel_filter(ctx, (const float*)ctx->d_odom_map.p, m, 4, ll, in.seg.data(), segs,
                                         set.map_voxel, (float*)out.p, 4, nullptr, set.map_max_points, map_spacing,
                                         in.center.empty() ? nullptr : &prune)))
            return rc;
    }
    sm->map = filter ? out.p : ctx->d_odom_map.p;
    sm->d_seg = filter ? ctx->d_vox_seg.p : ll;
    if (filter) {
        sm->kept.resize((size_t)segs + 1);
        sm->bad.resize((size_t)segs);
        sm->more = {Readback{ctx->d_vox_seg.p, sm->kept.size() * sizeof(int64_t), sm->kept.data()},
                    Readback{ctx->d_vox_bad.p, sm->bad.size() * sizeof(int), sm->bad.data()}};
    }
    return DCREG_OK;
}

// A push that succeeded becomes the session's state: the history after it, the retained frames' poses (the T_out bytes
// just returned for this push's frames), every sequence's last increment (deltas' entry of its last pushed frame, or
// the identity without deltas; a sequence with no frame keeps its own), and the window the retain step gathered.
static void commit_push(dcreg_ctx::OdomSession& ss, const odom_plan::Push& u, int n_frames, const int* seq_offsets,
                        const double* T_out, const double* deltas) {
    std::vector<double> T((size_t)u.next_ref.size() * 16);
    for (size_t e = 0; e < u.next_ref.size(); ++e) {
        const int r = u.next_ref[e];
        const double* from = r < n_frames ? T_out + (size_t)u.plan.input[(size_t)r] * 16 : &ss.hist_T[(size_t)(r - n_frames) * 16];
        memcpy(&T[e * 16], from, 16 * sizeof(double));
    }
    static const double kIdentity[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    for (int s = 0; s < ss.set.n_seqs; ++s)
        if (seq_offsets[s + 1] > seq_offsets[s])
            memcpy(&ss.last_delta[(size_t)s * 16], deltas ? deltas + (size_t)(seq_offsets[s + 1] - 1) * 16 : kIdentity,
                   16 * sizeof(double));
    ss.hist_T.swap(T);
    ss.hist = u.next;
    ss.cur = 1 - ss.cur;
}

// The call and its frames: the timestamps, and the frames' voxel filter (once per call, on the staged points in input
// order, before the pack and the sort; one sync for the kept counts).  From here on a frame is its kept points
int OdomCall::check() {
    BatchCheck c{name, !set.T_init.empty() && n_frames > 0 && seq_offsets && xyz && frame_offsets && R.T_out,
                 "null pointer, n_seqs <= 0 or n_frames <= 0",
                 "sequences are independent - give each rank its own, do not shard them", n_frames};
    c.offsets = frame_offsets; c.item = "frame"; c.stride = stride; c.own_cell = true; c.cell_size = set.cell_size;
    c.need_target = false; c.one_iteration = true; c.n_seqs = n_seqs; c.seq_offsets = seq_offsets;
    c.empty_seqs = sess != nullptr;
    c.own_msg = prior ? prior_error() : nullptr;
    if (!c.own_msg) c.own_msg = odometry_settings_error(set, deltas != nullptr);
    c.lanes = (int)set.lanes.size();
    int rc = check_batch_call(ctx, set.lanes.empty() ? params : set.lanes.data(), c);
    if (rc) return rc;
    if (!sess) {
        const std::string why = v_init_error(set);
        if (!why.empty()) { ctx->err = std::string(name) + ": " + why; return DCREG_BAD_ARG; }
        none = odom_plan::History(n_seqs);
    }
    CK(cudaSetDevice(ctx->device));
    if (timestamps)             // every point's fraction of its sweep, before anything is launched
        for (int s = 0; s < n_seqs; ++s)
            for (int k = seq_offsets[s]; k < seq_offsets[s + 1]; ++k)
                for (int64_t i = frame_offsets[k]; i < frame_offsets[k + 1]; ++i) {
                    const float tau = timestamps[i];
                    if (tau >= 0.0f && tau <= 1.0f) continue;
                    ctx->err = std::string(name) + ": " + frame_name(s, k) + ": the timestamp of point " +
                               std::to_string(i - frame_offsets[k]) + " is " +
                               (std::isfinite(tau) ? std::to_string(tau) + ", outside [0, 1]" : std::string("not finite"));
                    return DCREG_BAD_ARG;
                }
    if ((set.gyro || gi.frame_times || gi.samples || gi.sample_offsets) && (rc = check_gyro())) return rc;
    if (filtered) {
        kept.resize((size_t)n_frames + 1);
        std::vector<int> bad((size_t)n_frames), bad_in;
        if (split) {
            in_kept.resize((size_t)n_frames + 1);
            bad_in.resize((size_t)n_frames);
            rc = voxel_filter_chain(ctx, n_frames, xyz, frame_offsets, stride, set.map_input_voxel, set.source_voxel,
                                    set.source_max_points, timestamps != nullptr, in_kept.data(), bad_in.data(),
                                    kept.data(), bad.data());
        } else if (in_voxel > 0.0) {                // F_s = none: the source is F_in(frame)
            rc = voxel_filter_host(ctx, n_frames, xyz, frame_offsets, stride, in_voxel, 1, 0.0,
                                   timestamps != nullptr, false, kept.data(), bad.data());
        } else {
            rc = voxel_filter_host(ctx, n_frames, xyz, frame_offsets, stride, set.source_voxel, set.source_max_points,
                                   0.0, timestamps != nullptr, false, kept.data(), bad.data());
        }
        if (rc) return rc;
        auto why = [](const std::vector<int64_t>& kp, const std::vector<int>& bd, int k, bool map_input) -> std::string {
            const std::string f = map_input ? "the map-input filter" : "the source filter";
            return bd[(size_t)k] ? "a voxel coordinate of " + f + " lies outside [-2^20, 2^20)"
                   : kp[(size_t)k + 1] == kp[(size_t)k] ? "no point is left by " + f + " (no finite point)"
                                                        : std::string();
        };
        for (int s = 0; s < n_seqs; ++s)
            for (int k = seq_offsets[s]; k < seq_offsets[s + 1]; ++k) {
                std::string w = split ? why(in_kept, bad_in, k, true) : std::string();
                if (w.empty()) w = why(kept, bad, k, in_voxel > 0.0 && !split);
                if (!w.empty()) {
                    ctx->err = std::string(name) + ": " + frame_name(s, k) + ": " + w;
                    return DCREG_BAD_ARG;
                }
            }
        src_xyz = ctx->d_vox_xyz; src_stride = 3; src_off = kept.data();
        in_off = split ? in_kept.data() : src_off;
    }
    if (frame_points)
        for (int k = 0; k < n_frames; ++k) frame_points[k] = src_off[k + 1] - src_off[k];
    return DCREG_OK;
}

// (prior) What the prior map refuses, or null: the voxel map, a context without a target, a cell size other than the
// target's, and a sharded context
const char* OdomCall::prior_error() const {
    if (set.voxel_map) return "the prior map (dcreg_set_prior_map) registers against the target: no voxel map (map_frames >= 1)";
    if (!ctx->has_grid) return "the prior map (dcreg_set_prior_map) needs a target (dcreg_set_target)";
    if (set.cell_size != ctx->cell_size) return "with the prior map (dcreg_set_prior_map) cell_size must be the target's";
    if (ctx->comm) return "the prior map (dcreg_set_prior_map) does not run on a sharded context";
    return nullptr;
}

// (gyro) The frame times and samples, before anything is launched: the samples finite and strictly ascending in time
// within each sequence; every frame's span finite and > 0, its start, mid-sweep tm = start + 0.5 span and end = start +
// span distinct; and every non-anchor frame's tm after the previous frame's, with a sample at or before min(tm_prev,
// start) and one at or after its end.  A push without gyro input (all null) on a gyro session may hold anchors only.
int OdomCall::check_gyro() {
    auto bad = [&](const std::string& why) { ctx->err = std::string(name) + ": " + why; return DCREG_BAD_ARG; };
    const bool given = gi.frame_times && gi.samples && gi.sample_offsets;
    if (!set.gyro) return bad("frame_times, samples and sample_offsets need a session opened with gyro input");
    if (!given && (gi.frame_times || gi.samples || gi.sample_offsets))
        return bad("frame_times, samples and sample_offsets are given together or not at all");
    if (!given && !sess) return bad("gyro input needs frame_times, samples and sample_offsets");
    const int sw = gi.stride;
    if (given && set.imu && sw != se3::kImuStride)
        return bad("a session opened with IMU input takes 7-column samples (dcreg_odometry_push_imu)");
    if (given && !set.imu && sw != se3::kSampleStride)
        return bad("7-column IMU samples need a session opened with IMU input (dcreg_odometry_open_imu)");
    const int64_t* so = gi.sample_offsets;
    if (given) {
        if (so[0] != 0) return bad("sample_offsets[0] must be 0");
        for (int s = 0; s < n_seqs; ++s) {
            if (so[s + 1] < so[s]) return bad("sample_offsets must be non-decreasing");
            for (int64_t i = so[s]; i < so[s + 1]; ++i) {
                const double* r = gi.samples + (size_t)i * sw;
                const std::string at = "sequence " + std::to_string(s) + ", sample " + std::to_string(i - so[s]) +
                                       " (row " + std::to_string(i) + ")";
                if (!(std::isfinite(r[0]) && std::isfinite(r[1]) && std::isfinite(r[2]) && std::isfinite(r[3])))
                    return bad(at + ": a value that is not finite");
                for (int c = 4; c < sw; ++c)
                    if (!std::isfinite(r[c])) return bad(at + ": an accelerometer value that is not finite");
                if (i > so[s] && !(r[0] > r[-sw]))
                    return bad(at + ": its time is not after the previous sample's (times must be strictly ascending)");
            }
        }
    }
    gyro_ft.assign((size_t)n_frames * 4, NAN);
    gyro_anchor.assign((size_t)n_frames, 1);
    next_mid.assign((size_t)n_seqs, NAN);
    for (int s = 0; s < n_seqs; ++s) {
        const bool started = sess && hist.seen[(size_t)s] > 0;
        double prev = sess ? sess->last_mid[(size_t)s] : NAN;
        const double* sm = given ? gi.samples + (size_t)so[s] * sw : nullptr;
        const long long ns = given ? so[s + 1] - so[s] : 0;
        for (int k = seq_offsets[s]; k < seq_offsets[s + 1]; ++k) {
            const bool anchor = !started && k == seq_offsets[s];
            gyro_anchor[(size_t)k] = anchor;
            if (!given) {
                if (!anchor)
                    return bad(frame_name(s, k) + ": its prior needs gyro samples (dcreg_odometry_push_gyro)");
                continue;
            }
            const double start = gi.frame_times[2 * (size_t)k], span = gi.frame_times[2 * (size_t)k + 1];
            const double tm = start + 0.5 * span, end = start + span;
            if (!(std::isfinite(start) && std::isfinite(span) && span > 0.0))
                return bad(frame_name(s, k) + ": its start and span must be finite and its span > 0");
            if (!(start < tm && tm < end && std::isfinite(end)))
                return bad(frame_name(s, k) + ": its span is too small to separate start, mid-sweep and end in FP64");
            if (!anchor) {
                if (std::isnan(prev))
                    return bad(frame_name(s, k) + ": the previous frame's mid-sweep time is unknown (it was pushed "
                                                  "without frame times)");
                if (!(tm > prev))
                    return bad(frame_name(s, k) + ": its mid-sweep time " + std::to_string(tm) +
                               " is not after the previous frame's, " + std::to_string(prev));
                const double lo = std::min(prev, start);
                if (se3::gyro_last(sm, ns, lo, false, sw) < 0)
                    return bad(frame_name(s, k) + ": no gyro sample at or before " + std::to_string(lo) +
                               " (the previous mid-sweep time or the sweep's start)");
                if (ns == 0 || sm[(size_t)(ns - 1) * sw] < end)
                    return bad(frame_name(s, k) + ": no gyro sample at or after the sweep's end, " + std::to_string(end));
            }
            const double f[4] = {start, span, tm, prev};
            std::copy(f, f + 4, &gyro_ft[(size_t)k * 4]);
            prev = tm;
        }
        next_mid[(size_t)s] = prev;
    }
    return DCREG_OK;
}

// The plan, and what the steps read that is known before them: every step's tables in one upload, the frames, the
// increments, the retained frames' poses, and room for the largest step's maps and (sess) the next window
int OdomCall::upload() {
    int rc;
    {
        const std::string why = odom_plan::make_push(n_seqs, seq_offsets, n_frames, src_off,
                                                     set.voxel_map || prior ? 0 : set.map_frames, arena_plan::kMaxPoints,
                                                     hist, &U, split ? in_off : nullptr, prior);
        if (!why.empty()) { ctx->err = std::string(name) + ": " + why; return DCREG_BAD_ARG; }
    }
    const int n_steps = (int)P.steps.size();
    const int n_hist = (int)hist.n.size();
    std::vector<long long> hll;
    std::vector<int> hint;
    at_ll.assign((size_t)n_steps, 0); at_int.assign((size_t)n_steps, 0);
    for (int i = prior ? 0 : 1; i < n_steps; ++i) {
        const odom_plan::Step& st = P.steps[(size_t)i];
        at_ll[(size_t)i] = hll.size(); at_int[(size_t)i] = hint.size();
        odom_plan::pack(st.map, hll, hint);
        hint.insert(hint.end(), st.prev.begin(), st.prev.end());
        hint.insert(hint.end(), st.prev2.begin(), st.prev2.end());
        if (set.adaptive) {     // lane j's sequence (~ it: a first frame), and the lane that runs it at the next step
            for (int j = 0; j < st.active; ++j) hint.push_back(st.prev[(size_t)j] < 0 ? ~st.seq[(size_t)j] : st.seq[(size_t)j]);
            for (int s : st.seq) {
                int next = -1;
                if (i + 1 < n_steps) {
                    const std::vector<int>& ns = P.steps[(size_t)i + 1].seq;
                    const auto it = std::lower_bound(ns.begin(), ns.end(), s);
                    if (it != ns.end() && *it == s) next = (int)(it - ns.begin());
                }
                hint.push_back(next);
            }
        }
    }
    // (sess) then the retain step's: long long keep_dst [K + 1], keep_src [K]; int keep_ref [K]
    keep_ll = hll.size(); keep_int = hint.size();
    if (sess) {
        hll.insert(hll.end(), U.keep_dst.begin(), U.keep_dst.end());
        hll.insert(hll.end(), U.keep_src.begin(), U.keep_src.end());
        hint.insert(hint.end(), U.keep_ref.begin(), U.keep_ref.end());
    }
    // (timestamps) then the timestamp gather's: long long in_at [n_frames], kept_at [n_frames] (odom_ts_gather_kernel)
    ts_ll = hll.size();
    if (timestamps) {
        for (int d = 0; d < n_frames; ++d) hll.push_back(frame_offsets[P.input[(size_t)d]]);
        for (int d = 0; d < n_frames; ++d) hll.push_back(src_off[P.input[(size_t)d]]);
    }
    // (split) then the map-input points' device offsets [n_frames + 1] and, with timestamps, F_in's kept offsets in
    // device order [n_frames] (the first timestamp gather's kept_at)
    in_ll = hll.size();
    if (split) {
        hll.insert(hll.end(), P.map_off.begin(), P.map_off.end());
        if (timestamps)
            for (int d = 0; d < n_frames; ++d) hll.push_back(in_off[P.input[(size_t)d]]);
    }
    // (gyro input) then odom_gyro_kernel's: long long knot_off [n_frames + 1], range [n_frames][2] (device order)
    gyro_ll = hll.size();
    if (set.gyro && gi.samples) {
        hll.push_back(0);
        for (int d = 0; d < n_frames; ++d) {
            const int k = P.input[(size_t)d];
            int nb = 0;
            const double* f = &gyro_ft[(size_t)k * 4];
            const int64_t* so = gi.sample_offsets;
            const int s = frame_seq_of(k);
            hll.push_back(hll.back() + (gyro_anchor[(size_t)k] ? 0
                                        : se3::gyro_knot_count(gi.samples + (size_t)so[s] * gi.stride,
                                                               so[s + 1] - so[s], f[0], f[2], f[0] + f[1], &nb,
                                                               gi.stride)));
        }
        gyro_knots = hll.back();
        for (int d = 0; d < n_frames; ++d) {
            const int s = frame_seq_of(P.input[(size_t)d]);
            hll.push_back(gi.sample_offsets[s]);
            hll.push_back(gi.sample_offsets[s + 1]);
        }
    }
    // the frames in device order, each sorted by its own cell in the sensor frame (identity poses, a box of 1024^3 cells
    // around the sensor: locality only, the chained priors are not known yet); lanes: grid y of the loop kernel, a
    // lane's frame range set by odom_start_kernel at every step; grids: the step's local maps.  (prior) Sorted as
    // dcreg_icp_run_sequences sorts them, in the target's cells under their dead-reckoned poses (start()); grids: the
    // target with each lane's rings
    S = Batch{n_frames, src_xyz, src_stride, P.dev_off.data()};
    S.order = P.input.data(); S.in_off = src_off;
    if (filtered) S.kind = cudaMemcpyDeviceToDevice;
    if (prior) {
        S.sparse = ctx->grid.dense == corr::kSparseGrid;
        CK(ctx->odom_maps.d_grids.ensure(n_seqs));
    } else {
        S.sort = Batch::kBox;
        S.sort_box.inv_cell = 1.0 / set.cell_size;
        S.sort_box.ox = S.sort_box.oy = S.sort_box.oz = -512;
        S.sort_box.nx = S.sort_box.ny = S.sort_box.nz = 1024;
        S.sort_cells = 1ll << 30;
    }
    S.grid_table = true; S.cell_size = set.cell_size;
    S.lanes = n_seqs;
    if ((rc = stage_sources(ctx, S)) || (rc = stage_lanes(ctx, n_seqs, n_frames, &S.seq))) return rc;
    S.sort_T = ctx->d_seq_prior;
    if (split) CK(ctx->d_odom_in.ensure(std::max<long long>(P.map_off[(size_t)n_frames], 1)));
    d_map_src = split ? ctx->d_odom_in.p : ctx->d_scan_src.p;
    CK(ctx->d_odom_ll.ensure(std::max<long long>((long long)hll.size(), 1)));
    CK(ctx->d_odom_int.ensure(std::max<long long>((long long)hint.size(), 1)));
    CK(ctx->d_odom_map.ensure(std::max<long long>(P.max_map, 1)));
    if (set.map_voxel > 0.0 && !set.voxel_map && !prior) {  // the maps' filter at its largest step: no regrowth inside
                                                              // the loop
        CK(ctx->d_vmap[0].ensure(std::max<long long>(P.max_map, 1)));
        long long slots = 0;
        std::vector<long long> tab;
        for (int i = 1; i < n_steps; ++i)
            slots = std::max(slots, voxel_tables(P.steps[(size_t)i].active, P.steps[(size_t)i].map.seg.data(), tab));
        if ((rc = voxel_reserve(ctx, P.max_map, n_seqs, slots, set.map_max_points))) return rc;
    }
    if (!hll.empty()) {
        CK(cudaMemcpyAsync(ctx->d_odom_ll, hll.data(), hll.size() * sizeof(long long), cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaMemcpyAsync(ctx->d_odom_int, hint.data(), hint.size() * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    }
    // one increment per frame reference: the frames' (identity without deltas), then the retained frames' (a sequence's
    // last one carries the increment its push left; only a session retains frames); null: every increment is the identity
    if (set.motion == DCREG_MOTION_INCREMENTS && (deltas || n_hist > 0)) {
        std::vector<double> D_dev((size_t)(n_frames + n_hist) * 16, 0.0);
        for (int e = 0; e < n_frames + n_hist; ++e)
            for (int c4 = 0; c4 < 4; ++c4) D_dev[(size_t)e * 16 + 5 * c4] = 1.0;
        if (deltas)
            for (int k = 0; k < n_frames; ++k)
                memcpy(&D_dev[(size_t)P.dev[(size_t)k] * 16], deltas + (size_t)k * 16, 16 * sizeof(double));
        for (int s = 0; s < n_seqs; ++s)
            if (hist.off[(size_t)s + 1] > hist.off[(size_t)s])
                memcpy(&D_dev[(size_t)(n_frames + hist.off[(size_t)s + 1] - 1) * 16], &sess->last_delta[(size_t)s * 16],
                       16 * sizeof(double));
        CK(ctx->d_seq_delta.ensure((long long)D_dev.size()));
        CK(cudaMemcpyAsync(ctx->d_seq_delta, D_dev.data(), D_dev.size() * sizeof(double), cudaMemcpyHostToDevice,
                           ctx->stream));
        d_delta = ctx->d_seq_delta;
    }
    // the retained frames' poses and points (none on the empty history: nothing reads them), and (sess) room for the
    // next window, grown with headroom: a window whose frames vary in size does not reallocate (and synchronise) at
    // every push
    if (n_hist) {
        CK(sess->d_hist_T.ensure((long long)n_hist * 16));
        CK(cudaMemcpyAsync(sess->d_hist_T, sess->hist_T.data(), (size_t)n_hist * 16 * sizeof(double),
                           cudaMemcpyHostToDevice, ctx->stream));
        d_hist_T = sess->d_hist_T;
        d_win = sess->win[sess->cur];
    }
    if (sess) CK(sess->win[1 - sess->cur].grow(std::max<long long>(U.keep_dst.back(), 1)));
    return DCREG_OK;
}

// The loop's start: every frame's loop state at its sequence's T_init (device order; an anchor keeps it: T_out = T_prior
// = T_init, no iteration, not converged), and (timestamps) the caller's timestamps beside the packed points
int OdomCall::start() {
    int rc;
    if (set.imu) {
        const int n_hist = (int)hist.n.size();
        imu_v.assign((size_t)(n_frames + n_hist) * 3, 0.0);
        for (int s = 0; s < n_seqs; ++s) {
            for (int k = seq_offsets[s]; k < seq_offsets[s + 1]; ++k)
                std::copy(&set.v_init[(size_t)s * 3], &set.v_init[(size_t)s * 3] + 3, &imu_v[(size_t)P.dev[(size_t)k] * 3]);
            if (hist.off[(size_t)s + 1] > hist.off[(size_t)s])
                std::copy(&sess->last_v[(size_t)s * 3], &sess->last_v[(size_t)s * 3] + 3,
                          &imu_v[(size_t)(n_frames + hist.off[(size_t)s + 1] - 1) * 3]);
        }
    }
    std::vector<double> T_dev((size_t)n_frames * 16), ident((size_t)n_frames * 16, 0.0);
    for (int s = 0; s < n_seqs; ++s)
        for (int k = seq_offsets[s]; k < seq_offsets[s + 1]; ++k)
            memcpy(&T_dev[(size_t)P.dev[(size_t)k] * 16], &set.T_init[(size_t)s * 16], 16 * sizeof(double));
    if (prior) {    // frame k's dead-reckoned pose: T_init (a sequence's first frame), then compose_prior with D_{k-1}
        static const double kIdentity[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
        const bool inc = set.motion == DCREG_MOTION_INCREMENTS;
        if (sess) next_dr = sess->dr_T;
        for (int s = 0; s < n_seqs; ++s)
            for (int k = seq_offsets[s]; k < seq_offsets[s + 1]; ++k) {
                double* T = &T_dev[(size_t)P.dev[(size_t)k] * 16];
                const bool first = k == seq_offsets[s] && hist.seen.at((size_t)s) == 0;
                if (!first) {
                    const double* A = k > seq_offsets[s] ? &T_dev[(size_t)P.dev[(size_t)(k - 1)] * 16] : &sess->dr_T[(size_t)s * 16];
                    const double* D = !inc ? kIdentity
                                      : k > seq_offsets[s] ? (deltas ? deltas + (size_t)(k - 1) * 16 : kIdentity)
                                                           : &sess->last_delta[(size_t)s * 16];
                    const double R[9] = {A[0], A[1], A[2], A[4], A[5], A[6], A[8], A[9], A[10]}, t[3] = {A[3], A[7], A[11]};
                    compose_prior(R, t, D, T);
                }
                if (sess && k + 1 == seq_offsets[s + 1]) memcpy(&next_dr[(size_t)s * 16], T, 16 * sizeof(double));
            }
    } else {
        for (int d = 0; d < n_frames; ++d)
            for (int c4 = 0; c4 < 4; ++c4) ident[(size_t)d * 16 + 5 * c4] = 1.0;
        CK(cudaMemcpyAsync(ctx->d_seq_prior, ident.data(), ident.size() * sizeof(double), cudaMemcpyHostToDevice,
                           ctx->stream));
    }
    if ((rc = start_loop(ctx, n_frames, T_dev.data(), R, &S, &dlog, &src_iter))) return rc;
    const long long n_points = P.dev_off[(size_t)n_frames], n_map_points = P.map_off[(size_t)n_frames];
    const long long* d_map_seg = ctx->d_odom_ll + in_ll;
    if (split &&                // F_in's kept points packed in device order, as the sources are
        (rc = upload_points(ctx, ctx->d_in_xyz, n_map_points, 3, d_map_seg, n_frames, ctx->d_odom_in, nullptr,
                            P.input.data(), in_off, cudaMemcpyDeviceToDevice)))
        return rc;
    if (timestamps) {
        CK(ctx->d_odom_ts_in.ensure(std::max<long long>(frame_offsets[n_frames], 1)));
        CK(ctx->d_odom_ts.ensure(std::max<long long>(n_points, 1)));
        CK(ctx->d_odom_xi.ensure((long long)n_seqs * 6));
        CK(cudaMemcpyAsync(ctx->d_odom_ts_in, timestamps, (size_t)frame_offsets[n_frames] * sizeof(float),
                           cudaMemcpyHostToDevice, ctx->stream));
        const long long* d_in_at = ctx->d_odom_ll + ts_ll;
        if (split) {            // the map-input points' timestamps, then the sources' from theirs
            CK(ctx->d_odom_ts_map.ensure(std::max<long long>(n_map_points, 1)));
            odom_ts_gather_kernel<<<(unsigned)((n_map_points + 255) / 256), 256, 0, ctx->stream>>>(
                ctx->d_odom_ts_in, n_map_points, d_map_seg, n_frames, d_in_at, d_map_seg + n_frames + 1,
                ctx->d_in_index, ctx->d_odom_ts_map);
            odom_ts_gather_kernel<<<(unsigned)((n_points + 255) / 256), 256, 0, ctx->stream>>>(
                ctx->d_odom_ts_map, n_points, ctx->d_scan_seg, n_frames, d_map_seg, d_in_at + n_frames,
                ctx->d_vox_index, ctx->d_odom_ts);
            ctx->launches += 2;
        } else {
            odom_ts_gather_kernel<<<(unsigned)((n_points + 255) / 256), 256, 0, ctx->stream>>>(
                ctx->d_odom_ts_in, n_points, ctx->d_scan_seg, n_frames, d_in_at, d_in_at + n_frames,
                filtered ? ctx->d_vox_index.p : nullptr, ctx->d_odom_ts);
            ctx->launches++;
        }
        CK(cudaGetLastError());
    }
    if (set.gyro && gi.samples) {   // every non-anchor frame's prior rotation and knot table, from one upload
        const int64_t rows = gi.sample_offsets[n_seqs];
        std::vector<double> ft((size_t)n_frames * 4);
        for (int d = 0; d < n_frames; ++d)
            std::copy(&gyro_ft[(size_t)P.input[(size_t)d] * 4], &gyro_ft[(size_t)P.input[(size_t)d] * 4] + 4, &ft[(size_t)d * 4]);
        CK(ctx->d_gyro_smp.ensure(std::max<long long>(rows * gi.stride, 1)));
        CK(ctx->d_gyro_ft.ensure((long long)ft.size()));
        CK(ctx->d_gyro_G.ensure((long long)n_frames * 9));
        CK(ctx->d_gyro_knots.ensure(std::max<long long>(gyro_knots * se3::kKnotStride, 1)));
        if (rows)
            CK(cudaMemcpyAsync(ctx->d_gyro_smp, gi.samples, (size_t)rows * gi.stride * sizeof(double),
                               cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaMemcpyAsync(ctx->d_gyro_ft, ft.data(), ft.size() * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        if (set.imu) {          // (IMU) the preintegrals' room, and every frame reference's velocity as it starts
            CK(ctx->d_imu_abg.ensure((long long)n_frames * 9));
            CK(ctx->d_imu_v.ensure((long long)imu_v.size()));
            CK(cudaMemcpyAsync(ctx->d_imu_v, imu_v.data(), imu_v.size() * sizeof(double), cudaMemcpyHostToDevice,
                               ctx->stream));
            imu_dev.ft = ctx->d_gyro_ft;
            imu_dev.abg = ctx->d_imu_abg;
            imu_dev.v = ctx->d_imu_v;
            std::copy(set.gravity, set.gravity + 3, imu_dev.gravity);
        }
        AccelBias acc{};
        std::copy(set.accel_bias, set.accel_bias + 3, acc.b);
        const long long* d_knot_off = ctx->d_odom_ll + gyro_ll;
        odom_gyro_kernel<<<(unsigned)((n_frames + 127) / 128), 128, 0, ctx->stream>>>(
            set.gyro_set, gi.stride, acc, ctx->d_gyro_smp, ctx->d_gyro_ft, d_knot_off + n_frames + 1, d_knot_off,
            n_frames, ctx->d_gyro_G, set.imu ? ctx->d_imu_abg.p : nullptr, ctx->d_gyro_knots);
        ctx->launches++;
        CK(cudaGetLastError());
    }
    if (set.voxel_map) {
        MS = odom_plan::map_start(n_seqs, n_frames, hist, sess ? sess->map_off.data() : nullptr);
        if (sess) d_old = sess->win[sess->cur];
    }
    frame_radius.assign((size_t)n_frames, 0.0);
    if (set.adaptive) {         // the sequences' committed states, and the radii step 1's (prior: step 0's) lanes use
        const std::vector<adaptive::State> h =
            sess ? sess->thr_state : std::vector<adaptive::State>((size_t)n_seqs, adaptive::State{0.0, 0});
        std::vector<double> r;
        const size_t i0 = prior ? 0 : 1;
        if (P.steps.size() > i0)
            for (int s : P.steps[i0].seq)
                r.push_back(adaptive::radius(h[(size_t)s], set.threshold.initial_threshold, params->search_radius));
        if (prior) first_r = r;
        CK(ctx->d_thr_state.ensure(n_seqs));
        CK(ctx->d_lane_radius.ensure(n_seqs));
        CK(cudaMemcpyAsync(ctx->d_thr_state, h.data(), h.size() * sizeof(adaptive::State), cudaMemcpyHostToDevice, ctx->stream));
        if (!r.empty())
            CK(cudaMemcpyAsync(ctx->d_lane_radius, r.data(), r.size() * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    }
    return DCREG_OK;
}

// Step i >= 1 (prior: i >= 0); when its maps fail, ctx->err names the frame, `failed` the step, and nothing of it runs
int OdomCall::step(int i) {
    const odom_plan::Step& st = P.steps[(size_t)i];
    int rc;
    if (prior && (rc = prior_grids(i))) return rc;
    else if (!prior && (rc = window_grids(i))) return rc;
    if (failed >= 0) return DCREG_OK;
    // 1. the lanes' local maps from the window frames' device-resident results and the retained frames, or (voxel map)
    // one update: every lane's map becomes its previous one with frame k-1 inserted at its pose, capped and pruned (with
    // a session, every other sequence's map is carried along); then the map filter, if any
    return step_run(i);
}

// (prior) The step's grid table: the context's target with the rings of each lane's radius; with the adaptive threshold
// the radii of step i >= 1 come back first (the step's one sync; step 0's are start()'s), else the table is the same at
// every step and goes up once
int OdomCall::prior_grids(int i) {
    const odom_plan::Step& st = P.steps[(size_t)i];
    std::vector<double> lane_r((size_t)st.active, params->search_radius);
    if (set.adaptive && i == 0) {
        lane_r = first_r;
    } else if (set.adaptive) {
        CK(cudaMemcpyAsync(lane_r.data(), ctx->d_lane_radius, lane_r.size() * sizeof(double), cudaMemcpyDeviceToHost,
                           ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
    }
    sparse = ctx->grid.dense == corr::kSparseGrid;
    for (int j = 0; j < st.active; ++j) frame_radius[(size_t)P.input[(size_t)(st.first + j)]] = lane_r[(size_t)j];
    if (!set.adaptive && planned + planned_sparse > 0) return DCREG_OK;
    std::vector<corr::Grid> g((size_t)st.active, ctx->grid);
    for (int j = 0; j < st.active; ++j) g[(size_t)j].rings = std::max(1, search_rings(lane_r[(size_t)j], set.cell_size));
    CK(cudaMemcpyAsync(ctx->odom_maps.d_grids, g.data(), g.size() * sizeof(corr::Grid), cudaMemcpyHostToDevice, ctx->stream));
    return DCREG_OK;
}

// (window, voxel map) The step's maps and their grids; when the maps fail, ctx->err names the frame and `failed` the step
int OdomCall::window_grids(int i) {
    const odom_plan::Step& st = P.steps[(size_t)i];
    int rc;
    odom_plan::MapInput update;
    const odom_plan::MapInput& in = set.voxel_map ? update : st.map;
    if (set.voxel_map) odom_plan::map_step(P, i, sess != nullptr, MS, &update);
    StepMap sm;
    if ((rc = set.voxel_map ? build_map(update, nullptr, nullptr, ctx->d_vmap[i % 2], &sm)
                            : build_map(st.map, ctx->d_odom_ll + at_ll[(size_t)i], ctx->d_odom_int + at_int[(size_t)i],
                                        ctx->d_vmap[0], &sm)))
        return rc;
    // 2. their dense grids, one arena segment per lane (the bounds copy is the step's sync besides the loop's peeks, and
    // brings the filter's kept offsets back; the unfiltered map sizes bound the kept ones).  (adaptive) the lanes' radii,
    // which the last step's threshold kernel left, ride the same copy; each lane's grid gets its own ring count
    const double inv_cell = 1.0 / set.cell_size;
    std::vector<double> lane_r((size_t)st.active, params->search_radius);
    lane_rings.clear();
    if (set.adaptive) sm.more.push_back(Readback{ctx->d_lane_radius.p, lane_r.size() * sizeof(double), lane_r.data()});
    std::vector<int> hb;
    std::vector<arena_plan::Box> boxes;
    long long cells = 0;
    std::string plan_why;
    sparse = false;
    if (sm.map) {
        if ((rc = arena_bounds(ctx, ctx->odom_maps, sm.map, in.seg.data(), sm.d_seg, st.active, inv_cell, hb, sm.more)))
            return rc;
        plan_why = sparse_maps ? arena_plan::plan_or_sparse(st.active, hb.data(), boxes, &cells, "local map of lane", &sparse)
                               : arena_plan::plan(st.active, hb.data(), boxes, &cells, "local map of lane");
    }
    int b = 0;
    const std::string why = odom_plan::map_failure(in, st.active, n_frames, arena_plan::kMaxPoints, sm.bad, sm.kept, hb,
                                                   plan_why, &b);
    if (map_failed(in, &st, why, b)) {
        failed = i;
        return DCREG_OK;
    }
    if (set.voxel_map) {
        odom_plan::map_commit(update, sm.kept.data(), MS);
        d_old = sm.map;
    }
    const long long m = sm.kept.empty() ? in.seg[(size_t)st.active] : sm.kept[(size_t)st.active];
    for (int j = 0; j < st.active; ++j) {
        frame_radius[(size_t)P.input[(size_t)(st.first + j)]] = lane_r[(size_t)j];
        if (set.adaptive) lane_rings.push_back(std::max(1, search_rings(lane_r[(size_t)j], set.cell_size)));
    }
    const int rings = search_rings(params->search_radius, set.cell_size);
    if (sparse) {           // every lane a sparse row index (one more sync, for the tables' sizes)
        std::vector<long long> seg((size_t)st.active + 1);
        for (int j = 0; j <= st.active; ++j) seg[(size_t)j] = sm.kept.empty() ? in.seg[(size_t)j] : sm.kept[(size_t)j];
        int bad = -1;
        if ((rc = build_sparse_arena(ctx, ctx->odom_maps, sm.map, sm.d_seg, seg, st.active, hb.data(), inv_cell, rings,
                                     set.adaptive ? lane_rings.data() : nullptr, &bad)))
            return rc;
        if (map_failed(in, &st, bad < 0 ? "" : "its local map's sparse index would need more than 2^32 table slots", bad)) {
            failed = i;
            return DCREG_OK;
        }
    } else if ((rc = arena_fill(ctx, ctx->odom_maps, sm.map, sm.d_seg, st.active, m, boxes.data(), cells, inv_cell, rings,
                                set.adaptive ? lane_rings.data() : nullptr))) {
        return rc;
    }
    return DCREG_OK;
}

// Step i's frames, after its grids: their priors, deskew, the loop, and (adaptive) the threshold states
int OdomCall::step_run(int i) {
    const odom_plan::Step& st = P.steps[(size_t)i];
    int rc;
    // 3. every lane's frame of this step: its prior and a fresh loop state
    const int* d_prev = ctx->d_odom_int + at_int[(size_t)i] + st.map.piece_frame.size() + st.map.center.size();
    const int* d_prev2 = d_prev + st.active;
    if (set.gyro)       // (gyro) the increment's rotation from the gyro, its translation kept for the deskew
        odom_start_gyro_kernel<<<(unsigned)((n_seqs + 127) / 128), 128, 0, ctx->stream>>>(
            ctx->d_state, ctx->d_scan_seg, ctx->d_seq_prior, ctx->d_seq_cursor, ctx->d_seq_first, ctx->d_n_active,
            n_seqs, st.first, st.active, d_prev, d_prev2, n_frames, d_hist_T, ctx->d_gyro_G,
            timestamps ? ctx->d_odom_xi.p : nullptr, ctx->d_scan_radius, imu_dev);
    else
        odom_start_kernel<<<(unsigned)((n_seqs + 127) / 128), 128, 0, ctx->stream>>>(
            ctx->d_state, ctx->d_scan_seg, ctx->d_seq_prior, ctx->d_seq_cursor, ctx->d_seq_first, ctx->d_n_active, n_seqs,
            st.first, st.active, d_prev, d_prev2, d_delta, set.motion, n_frames, d_hist_T);
    ctx->launches++;
    CK(cudaGetLastError());
    // 3b. (timestamps) the step's frames deskewed with the increments their priors used, outside the loop's graphs.
    // (gyro) A push without gyro input holds first frames alone (check_gyro), which are not deskewed: no knot table
    if (timestamps && set.gyro && gi.samples) {
        const long long a = P.dev_off[(size_t)st.first], np = P.dev_off[(size_t)(st.first + st.active)] - a;
        const long long* d_knot_off = ctx->d_odom_ll + gyro_ll;
        odom_deskew_gyro_kernel<true><<<(unsigned)((np + 255) / 256), 256, 0, ctx->stream>>>(
            ctx->d_scan_src, ctx->d_scan_sorted, ctx->d_scan_seg, st.first, st.active, a, np, ctx->d_odom_ts,
            ctx->d_gyro_ft, d_knot_off, ctx->d_gyro_knots, ctx->d_odom_xi, ctx->d_scan_radius);
        ctx->launches++;
        CK(cudaGetLastError());
    } else if (timestamps && !set.gyro) {
        odom_twist_kernel<<<(unsigned)((st.active + 127) / 128), 128, 0, ctx->stream>>>(
            ctx->d_state, st.first, st.active, d_prev, d_prev2, d_delta, set.motion, n_frames, d_hist_T,
            ctx->d_odom_xi, ctx->d_scan_radius);
        const long long a = P.dev_off[(size_t)st.first], np = P.dev_off[(size_t)(st.first + st.active)] - a;
        odom_deskew_kernel<true><<<(unsigned)((np + 255) / 256), 256, 0, ctx->stream>>>(
            ctx->d_scan_src, ctx->d_scan_sorted, ctx->d_scan_seg, st.first, st.active, a, np, ctx->d_odom_ts,
            ctx->d_odom_xi, ctx->d_scan_radius);
        ctx->launches += 2;
        CK(cudaGetLastError());
    }
    // 3c. (split, timestamps) the step's map-input points deskewed with the same increments: every source point is a
    // copy of one of them with the same timestamp, so the two passes agree on it bit for bit
    if (timestamps && split) {
        const long long a = P.map_off[(size_t)st.first], np = P.map_off[(size_t)(st.first + st.active)] - a;
        const long long* d_map_seg = ctx->d_odom_ll + in_ll;
        if (set.gyro)
            odom_deskew_gyro_kernel<false><<<(unsigned)((np + 255) / 256), 256, 0, ctx->stream>>>(
                ctx->d_odom_in, nullptr, d_map_seg, st.first, st.active, a, np, ctx->d_odom_ts_map, ctx->d_gyro_ft,
                ctx->d_odom_ll + gyro_ll, ctx->d_gyro_knots, ctx->d_odom_xi, nullptr);
        else
            odom_deskew_kernel<false><<<(unsigned)((np + 255) / 256), 256, 0, ctx->stream>>>(
                ctx->d_odom_in, nullptr, d_map_seg, st.first, st.active, a, np, ctx->d_odom_ts_map, ctx->d_odom_xi,
                nullptr);
        ctx->launches++;
        CK(cudaGetLastError());
    }
    // 4. the loop: the same chunks (and CUDA graphs) at every step - the grid table keeps its pointer (the first step
    // has the most lanes, so the arena's table never regrows after it), only its entries change
    // (a step of sparse maps runs the kSparse instantiation: a plan and chunk graphs of its own)
    LoopPlan& LP = sparse ? L_sparse : L;
    bool& have_plan = sparse ? planned_sparse : planned;
    if (!have_plan) {
        S.grids = ctx->odom_maps.d_grids;
        S.sparse = sparse;
        if (lanes.n) CK(ctx->d_lane_seq.ensure(n_seqs));
        if ((rc = plan_iteration(ctx, params, src_iter, nullptr, n_seqs, dlog, dlog ? R.log_cap : 0, true, &LP, &S, lanes)))
            return rc;
        LP.b.lane_radius = set.adaptive ? ctx->d_lane_radius.p : nullptr;
        LP.b.lane_seq = lanes.n ? ctx->d_lane_seq.p : nullptr;
        have_plan = true;
    }
    if (lanes.n)            // the sequence each lane of this step runs (the lanes' settings are the sequences')
        CK(cudaMemcpyAsync(ctx->d_lane_seq, st.seq.data(), st.seq.size() * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    if ((rc = run_chunks(ctx, LP, params, dlog, dlog ? R.log_cap : 0, params->max_iterations, 16, true))) return rc;
    // 4b. (IMU) the step's frames' velocities, which the next step's priors read
    if (imu_dev.v) {
        odom_velocity_kernel<<<(unsigned)((st.active + 127) / 128), 128, 0, ctx->stream>>>(
            ctx->d_state, st.first, st.active, d_prev, n_frames, d_hist_T, imu_dev);
        ctx->launches++;
        CK(cudaGetLastError());
    }
    // 5. (adaptive) the step's frames into their sequences' threshold states, and the next step's radii
    if (set.adaptive) {
        const int* d_seq = d_prev2 + st.active;
        odom_threshold_kernel<<<(unsigned)((st.active + 127) / 128), 128, 0, ctx->stream>>>(
            ctx->d_state, ctx->d_seq_prior, st.first, st.active, d_seq, d_seq + st.active, set.threshold,
            params->search_radius, ctx->d_thr_state, ctx->d_lane_radius);
        ctx->launches++;
        CK(cudaGetLastError());
    }
    return DCREG_OK;
}

// After the steps: (sess) the next window, and (voxel map) the final update, every sequence's map with its last frame
// in it, packed by sequence (one more sync), both into the session's other buffer, so its own stays as it was until
// the push commits; then the results in the caller's frame order (after a failed step only the frames before it, and
// that step's message), the deskewed points, the commit
int OdomCall::finish() {
    int rc;
    const long long kept_points = sess ? U.keep_dst.back() : 0;
    if (sess && failed < 0 && kept_points > 0) {
        const long long* d_keep_dst = ctx->d_odom_ll + keep_ll;
        const int keep = (int)U.keep_ref.size();
        retain_points_kernel<<<(unsigned)((kept_points + 255) / 256), 256, 0, ctx->stream>>>(
            d_map_src, sess->win[sess->cur], n_frames, d_keep_dst, keep, d_keep_dst + keep + 1,
            ctx->d_odom_int + keep_int, kept_points, sess->win[1 - sess->cur]);
        ctx->launches++;
        CK(cudaGetLastError());
    }
    StepMap sm;
    bool update_failed = false;
    if (sess && set.voxel_map && failed < 0) {
        odom_plan::MapInput in;
        odom_plan::map_step(P, (int)P.steps.size(), true, MS, &in);
        if ((rc = build_map(in, nullptr, nullptr, sess->win[1 - sess->cur], &sm))) return rc;
        for (const Readback& r : sm.more) CK(cudaMemcpyAsync(r.host, r.dev, r.bytes, cudaMemcpyDeviceToHost, ctx->stream));
        if (sm.map) CK(cudaStreamSynchronize(ctx->stream));
        int b = 0;
        const std::string why = odom_plan::map_failure(in, 0, n_frames, arena_plan::kMaxPoints, sm.bad, sm.kept, {}, "", &b);
        update_failed = map_failed(in, nullptr, why, b);
    }
    const std::string err = ctx->err;
    std::vector<adaptive::State> thr;               // (sess, adaptive) the states after the push, read back with the results
    if (sess && set.adaptive && failed < 0 && !update_failed) {
        thr.resize((size_t)n_seqs);
        CK(cudaMemcpyAsync(thr.data(), ctx->d_thr_state, thr.size() * sizeof(adaptive::State), cudaMemcpyDeviceToHost,
                           ctx->stream));
    }
    std::vector<int> dev_seq;                       // (lanes) every device trial's sequence, for its log records
    if (lanes.n) {
        dev_seq.resize((size_t)n_frames);
        for (int s = 0; s < n_seqs; ++s)
            for (int k = seq_offsets[s]; k < seq_offsets[s + 1]; ++k) dev_seq[(size_t)P.dev[(size_t)k]] = s;
    }
    if ((rc = finish_call(ctx, params, n_frames, dlog, R, P.dev.data(),
                          failed >= 0 ? P.steps[(size_t)failed].first : n_frames, lanes, dev_seq.data())))
        return rc;
    if (search_radius) memcpy(search_radius, frame_radius.data(), frame_radius.size() * sizeof(double));
    if (failed >= 0 || update_failed) { ctx->err = err; return DCREG_BAD_ARG; }
    if (deskewed_xyz) {         // the frames' kept (deskewed) points, put in the caller's frame order
        const long long n_points = P.dev_off[(size_t)n_frames];
        std::vector<float4> h((size_t)std::max<long long>(n_points, 1));
        CK(cudaMemcpyAsync(h.data(), ctx->d_scan_src, (size_t)n_points * sizeof(float4), cudaMemcpyDeviceToHost,
                           ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        for (int k = 0; k < n_frames; ++k) {
            const long long d0 = P.dev_off[(size_t)P.dev[(size_t)k]];
            float* o = deskewed_xyz + (size_t)src_off[k] * 3;
            for (long long i = 0; i < src_off[k + 1] - src_off[k]; ++i) {
                const float4 p = h[(size_t)(d0 + i)];
                o[3 * i] = p.x; o[3 * i + 1] = p.y; o[3 * i + 2] = p.z;
            }
        }
    }
    if (imu_dev.v) {            // (IMU) the frames' velocities (imu_v keeps v_init without samples: anchors alone)
        CK(cudaMemcpyAsync(imu_v.data(), ctx->d_imu_v, (size_t)n_frames * 3 * sizeof(double), cudaMemcpyDeviceToHost,
                           ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
    }
    if (set.imu && gi.velocity)
        for (int k = 0; k < n_frames; ++k)
            std::copy(&imu_v[(size_t)P.dev[(size_t)k] * 3], &imu_v[(size_t)P.dev[(size_t)k] * 3] + 3, gi.velocity + (size_t)k * 3);
    if (sess) {
        commit_push(*sess, U, n_frames, seq_offsets, R.T_out, deltas);
        if (set.imu)
            for (int s = 0; s < n_seqs; ++s)
                if (seq_offsets[s + 1] > seq_offsets[s])
                    std::copy(&imu_v[(size_t)P.dev[(size_t)(seq_offsets[s + 1] - 1)] * 3],
                              &imu_v[(size_t)P.dev[(size_t)(seq_offsets[s + 1] - 1)] * 3] + 3, &sess->last_v[(size_t)s * 3]);
        if (set.voxel_map) sess->map_off.assign(sm.kept.begin(), sm.kept.end());
        if (set.adaptive) sess->thr_state.swap(thr);
        if (set.gyro)
            for (int s = 0; s < n_seqs; ++s)
                if (seq_offsets[s + 1] > seq_offsets[s]) sess->last_mid[(size_t)s] = next_mid[(size_t)s];
        if (prior) sess->dr_T.swap(next_dr);
    }
    return DCREG_OK;
}

// Every odometry entry point: the frames continue the sequences of a history (odom_plan::History), whose retained
// frames act as anchors outside the call: they are not registered and return nothing, their points come from the
// window buffer and their poses from the session, and their last increments continue the deltas.  A one-shot call
// (sess null) runs on the empty history, where every sequence starts.  A push (sess) runs on the session's: a sequence
// may have no frame, frames are named by their number in the sequence since the session opened, the retain step
// gathers the next window, and only a push that succeeds changes the session (commit_push).
static int run_odometry(dcreg_ctx* ctx, const char* name, const OdomSettings& set, dcreg_ctx::OdomSession* sess,
                        const int* seq_offsets, int n_frames, const float* xyz, const int64_t* frame_offsets, int stride,
                        const double* deltas, const float* timestamps, const Results& R, int64_t* frame_points,
                        float* deskewed_xyz, double* search_radius = nullptr, GyroInput gi = {}) {
    if (!ctx) return DCREG_BAD_ARG;
    OdomCall o{ctx, name, set, sess, seq_offsets, n_frames, xyz, frame_offsets, stride, deltas, timestamps, R,
               frame_points, deskewed_xyz, search_radius, gi};
    int rc;
    if ((rc = o.check()) || (rc = o.upload()) || (rc = o.start())) return rc;
    for (int i = o.prior ? 0 : 1; i < (int)o.P.steps.size() && o.failed < 0; ++i)
        if ((rc = o.step(i))) return rc;
    return o.finish();
}

int dcreg_icp_run_odometry(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_seqs, const int* seq_offsets,
                           int n_frames, const float* xyz, const int64_t* frame_offsets, int stride, double cell_size,
                           int map_frames, int motion, const double* T_init, const double* deltas, double* T_prior,
                           double* T_out, int* n_iterations, int* converged, int* status, double* cov,
                           dcreg_iter_log* log, int log_cap) {
    return run_odometry(ctx, "icp_run_odometry",
                        odom_settings(params, n_seqs, cell_size, map_frames, motion, 0.0, 0.0, 1, 1, T_init,
                                      ctx && ctx->lane_params),
                        nullptr,
                        seq_offsets, n_frames, xyz, frame_offsets, stride, deltas, nullptr,
                        Results{T_out, n_iterations, converged, status, log, log_cap, cov, T_prior}, nullptr, nullptr);
}

int dcreg_icp_run_odometry_voxel(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_seqs, const int* seq_offsets,
                                 int n_frames, const float* xyz, const int64_t* frame_offsets, int stride,
                                 double cell_size, int map_frames, int motion, double source_voxel, double map_voxel,
                                 const double* T_init, const double* deltas, int64_t* frame_points, double* T_prior,
                                 double* T_out, int* n_iterations, int* converged, int* status, double* cov,
                                 dcreg_iter_log* log, int log_cap) {
    return run_odometry(ctx, "icp_run_odometry_voxel",
                        with_map_input(odom_settings(params, n_seqs, cell_size, map_frames, motion, source_voxel,
                                                     map_voxel, 1, 1, T_init, ctx && ctx->lane_params),
                                       ctx),
                        nullptr, seq_offsets, n_frames, xyz, frame_offsets, stride, deltas, nullptr,
                        Results{T_out, n_iterations, converged, status, log, log_cap, cov, T_prior}, frame_points, nullptr);
}

int dcreg_icp_run_odometry_voxel_n(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_seqs, const int* seq_offsets,
                                   int n_frames, const float* xyz, const int64_t* frame_offsets, int stride,
                                   double cell_size, int map_frames, int motion, double source_voxel, double map_voxel,
                                   int source_max_points, int map_max_points, const double* T_init,
                                   const double* deltas, int64_t* frame_points, double* T_prior, double* T_out,
                                   int* n_iterations, int* converged, int* status, double* cov, dcreg_iter_log* log,
                                   int log_cap) {
    return run_odometry(ctx, "icp_run_odometry_voxel_n",
                        with_map_input(odom_settings(params, n_seqs, cell_size, map_frames, motion, source_voxel,
                                                     map_voxel, source_max_points, map_max_points, T_init,
                                                     ctx && ctx->lane_params),
                                       ctx),
                        nullptr, seq_offsets, n_frames, xyz, frame_offsets, stride, deltas, nullptr,
                        Results{T_out, n_iterations, converged, status, log, log_cap, cov, T_prior}, frame_points, nullptr);
}

int dcreg_icp_run_odometry_deskew(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_seqs, const int* seq_offsets,
                                  int n_frames, const float* xyz, const int64_t* frame_offsets, int stride,
                                  double cell_size, int map_frames, int motion, double source_voxel, double map_voxel,
                                  int source_max_points, int map_max_points, const double* T_init, const double* deltas,
                                  const float* timestamps, int64_t* frame_points, double* T_prior, double* T_out,
                                  int* n_iterations, int* converged, int* status, double* cov, float* deskewed_xyz,
                                  dcreg_iter_log* log, int log_cap) {
    return run_odometry(ctx, "icp_run_odometry_deskew",
                        with_map_input(odom_settings(params, n_seqs, cell_size, map_frames, motion, source_voxel,
                                                     map_voxel, source_max_points, map_max_points, T_init,
                                                     ctx && ctx->lane_params),
                                       ctx),
                        nullptr, seq_offsets, n_frames, xyz, frame_offsets, stride, deltas, timestamps,
                        Results{T_out, n_iterations, converged, status, log, log_cap, cov, T_prior}, frame_points,
                        deskewed_xyz);
}

// the settings of the voxel map (dcreg_icp_run_odometry_map, dcreg_odometry_open_map): no window
static OdomSettings odom_map_settings(const dcreg_icp_params* params, int n_seqs, double cell_size, int motion,
                                      double source_voxel, double map_voxel, int source_max_points, int map_max_points,
                                      double max_distance, const double* T_init, bool lanes) {
    OdomSettings set = odom_settings(params, n_seqs, cell_size, 0, motion, source_voxel, map_voxel, source_max_points,
                                     map_max_points, T_init, lanes);
    set.voxel_map = true;
    set.max_distance = max_distance;
    return set;
}

int dcreg_icp_run_odometry_map(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_seqs, const int* seq_offsets,
                               int n_frames, const float* xyz, const int64_t* frame_offsets, int stride, double cell_size,
                               int motion, double source_voxel, double map_voxel, int source_max_points,
                               int map_max_points, double max_distance, const double* T_init, const double* deltas,
                               const float* timestamps, int64_t* frame_points, double* T_prior, double* T_out,
                               int* n_iterations, int* converged, int* status, double* cov, float* deskewed_xyz,
                               dcreg_iter_log* log, int log_cap) {
    return run_odometry(ctx, "icp_run_odometry_map",
                        with_map_input(odom_map_settings(params, n_seqs, cell_size, motion, source_voxel, map_voxel,
                                                         source_max_points, map_max_points, max_distance, T_init,
                                                         ctx && ctx->lane_params),
                                       ctx),
                        nullptr, seq_offsets, n_frames, xyz, frame_offsets, stride, deltas, timestamps,
                        Results{T_out, n_iterations, converged, status, log, log_cap, cov, T_prior}, frame_points,
                        deskewed_xyz);
}

// the settings of dcreg_icp_run_odometry_adaptive / dcreg_odometry_open_adaptive: the window (map_frames >= 1) or the
// voxel map (map_frames = 0), with the adaptive threshold when `adaptive` is given
static OdomSettings odom_adaptive_settings(const dcreg_icp_params* params, int n_seqs, double cell_size, int map_frames,
                                           int motion, double source_voxel, double map_voxel, int source_max_points,
                                           int map_max_points, double max_distance,
                                           const dcreg_adaptive_threshold* adaptive, const double* T_init, bool lanes) {
    OdomSettings set = map_frames == 0 ? odom_map_settings(params, n_seqs, cell_size, motion, source_voxel, map_voxel,
                                                           source_max_points, map_max_points, max_distance, T_init, lanes)
                                       : odom_settings(params, n_seqs, cell_size, map_frames, motion, source_voxel,
                                                       map_voxel, source_max_points, map_max_points, T_init, lanes);
    if (adaptive) {
        set.adaptive = true;
        set.threshold = adaptive::Settings{adaptive->initial_threshold, adaptive->min_motion, adaptive->max_range};
    }
    return set;
}

int dcreg_icp_run_odometry_adaptive(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_seqs, const int* seq_offsets,
                                    int n_frames, const float* xyz, const int64_t* frame_offsets, int stride,
                                    double cell_size, int map_frames, int motion, double source_voxel, double map_voxel,
                                    int source_max_points, int map_max_points, double max_distance,
                                    const dcreg_adaptive_threshold* adaptive, const double* T_init, const double* deltas,
                                    const float* timestamps, int64_t* frame_points, double* T_prior, double* T_out,
                                    int* n_iterations, int* converged, int* status, double* cov, float* deskewed_xyz,
                                    double* search_radius, dcreg_iter_log* log, int log_cap) {
    return run_odometry(ctx, "icp_run_odometry_adaptive",
                        with_map_input(odom_adaptive_settings(params, n_seqs, cell_size, map_frames, motion,
                                                              source_voxel, map_voxel, source_max_points,
                                                              map_max_points, max_distance, adaptive, T_init,
                                                              ctx && ctx->lane_params),
                                       ctx),
                        nullptr, seq_offsets, n_frames, xyz, frame_offsets, stride, deltas, timestamps,
                        Results{T_out, n_iterations, converged, status, log, log_cap, cov, T_prior}, frame_points,
                        deskewed_xyz, search_radius);
}

// the settings of dcreg_icp_run_odometry_gyro / dcreg_odometry_open_gyro: the adaptive call's, with the gyro when given
static OdomSettings odom_gyro_settings(OdomSettings set, const dcreg_gyro* gyro) {
    if (gyro) {
        set.gyro = true;
        std::copy(gyro->R_sensor_imu, gyro->R_sensor_imu + 9, set.gyro_set.R_si);
        std::copy(gyro->bias, gyro->bias + 3, set.gyro_set.bias);
    }
    return set;
}

int dcreg_icp_run_odometry_gyro(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_seqs, const int* seq_offsets,
                                int n_frames, const float* xyz, const int64_t* frame_offsets, int stride,
                                double cell_size, int map_frames, int motion, double source_voxel, double map_voxel,
                                int source_max_points, int map_max_points, double max_distance,
                                const dcreg_adaptive_threshold* adaptive, const dcreg_gyro* gyro, const double* T_init,
                                const double* deltas, const float* timestamps, const double* frame_times,
                                const double* samples, const int64_t* sample_offsets, int64_t* frame_points,
                                double* T_prior, double* T_out, int* n_iterations, int* converged, int* status,
                                double* cov, float* deskewed_xyz, double* search_radius, dcreg_iter_log* log,
                                int log_cap) {
    return run_odometry(ctx, "icp_run_odometry_gyro",
                        with_map_input(odom_gyro_settings(odom_adaptive_settings(params, n_seqs, cell_size,
                                                                                 map_frames, motion, source_voxel,
                                                                                 map_voxel, source_max_points,
                                                                                 map_max_points, max_distance,
                                                                                 adaptive, T_init,
                                                                                 ctx && ctx->lane_params),
                                                          gyro),
                                       ctx),
                        nullptr, seq_offsets, n_frames, xyz, frame_offsets, stride, deltas, timestamps,
                        Results{T_out, n_iterations, converged, status, log, log_cap, cov, T_prior}, frame_points,
                        deskewed_xyz, search_radius,
                        gyro ? GyroInput{frame_times, samples, sample_offsets} : GyroInput{});
}

// the settings of dcreg_icp_run_odometry_imu / dcreg_odometry_open_imu: the gyro call's, with the gyro and the
// accelerometer when imu is given (v_init null: every sequence starts at rest)
static OdomSettings odom_imu_settings(OdomSettings set, const dcreg_imu* imu, const double* v_init) {
    if (!imu) return set;
    dcreg_gyro g;
    std::copy(imu->R_sensor_imu, imu->R_sensor_imu + 9, g.R_sensor_imu);
    std::copy(imu->gyro_bias, imu->gyro_bias + 3, g.bias);
    set = odom_gyro_settings(set, &g);
    set.imu = true;
    std::copy(imu->accel_bias, imu->accel_bias + 3, set.accel_bias);
    std::copy(imu->gravity, imu->gravity + 3, set.gravity);
    set.v_init.assign((size_t)std::max(set.n_seqs, 0) * 3, 0.0);
    if (v_init) std::copy(v_init, v_init + set.v_init.size(), set.v_init.begin());
    return set;
}

int dcreg_icp_run_odometry_imu(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_seqs, const int* seq_offsets,
                               int n_frames, const float* xyz, const int64_t* frame_offsets, int stride,
                               double cell_size, int map_frames, int motion, double source_voxel, double map_voxel,
                               int source_max_points, int map_max_points, double max_distance,
                               const dcreg_adaptive_threshold* adaptive, const dcreg_imu* imu, const double* T_init,
                               const double* v_init, const double* deltas, const float* timestamps,
                               const double* frame_times, const double* samples, const int64_t* sample_offsets,
                               int64_t* frame_points, double* T_prior, double* T_out, int* n_iterations, int* converged,
                               int* status, double* cov, float* deskewed_xyz, double* search_radius, double* velocity,
                               dcreg_iter_log* log, int log_cap) {
    return run_odometry(ctx, "icp_run_odometry_imu",
                        with_map_input(odom_imu_settings(odom_adaptive_settings(params, n_seqs, cell_size, map_frames,
                                                                                motion, source_voxel, map_voxel,
                                                                                source_max_points, map_max_points,
                                                                                max_distance, adaptive, T_init,
                                                                                ctx && ctx->lane_params),
                                                         imu, v_init),
                                       ctx),
                        nullptr, seq_offsets, n_frames, xyz, frame_offsets, stride, deltas, timestamps,
                        Results{T_out, n_iterations, converged, status, log, log_cap, cov, T_prior}, frame_points,
                        deskewed_xyz, search_radius,
                        imu ? GyroInput{frame_times, samples, sample_offsets, se3::kImuStride, velocity} : GyroInput{});
}

// Opens the context's one session with the settings `set` (dcreg_odometry_open, _open_map, _open_adaptive, _open_gyro,
// _open_imu)
static int open_session(dcreg_ctx* ctx, const char* name, const OdomSettings& set) {
    if (ctx->odom) {
        ctx->err = std::string(name) + ": a session is open already (dcreg_odometry_close it first)";
        return DCREG_BAD_ARG;
    }
    std::unique_ptr<dcreg_ctx::OdomSession> ss(new dcreg_ctx::OdomSession());
    ss->set = set;
    ss->set.sparse_maps = ctx->sparse_maps;
    ss->set.map_spacing = ctx->map_spacing;
    ss->set.map_input_voxel = ctx->map_input_voxel;
    ss->set.prior_map = ctx->prior_map;
    const int n_seqs = set.n_seqs;
    BatchCheck c{name, !ss->set.T_init.empty(), "null pointer or n_seqs <= 0",
                 "sequences are independent - give each rank its own, do not shard them", n_seqs};
    c.own_cell = true; c.cell_size = set.cell_size; c.need_target = false; c.one_iteration = true;
    if (ss->set.prior_map && set.voxel_map)
        c.own_msg = "the prior map (dcreg_set_prior_map) registers against the target: no voxel map (map_frames >= 1)";
    else if (ss->set.prior_map && ctx->comm)
        c.own_msg = "the prior map (dcreg_set_prior_map) does not run on a sharded context";
    else
        c.own_msg = odometry_settings_error(ss->set, false);
    c.lanes = (int)ss->set.lanes.size();
    const int rc = check_batch_call(ctx, ss->set.lanes.empty() ? &ss->set.params : ss->set.lanes.data(), c);
    if (rc) return rc;
    const std::string why = v_init_error(ss->set);
    if (!why.empty()) { ctx->err = std::string(name) + ": " + why; return DCREG_BAD_ARG; }
    ss->last_v = ss->set.v_init;
    ss->hist = odom_plan::History(n_seqs);
    ss->map_off.assign((size_t)n_seqs + 1, 0);
    ss->thr_state.assign((size_t)n_seqs, adaptive::State{0.0, 0});
    ss->last_mid.assign((size_t)n_seqs, NAN);
    if (ss->set.prior_map) ss->dr_T = ss->set.T_init;
    ss->last_delta.assign((size_t)n_seqs * 16, 0.0);
    for (int s = 0; s < n_seqs; ++s)
        for (int c4 = 0; c4 < 4; ++c4) ss->last_delta[(size_t)s * 16 + 5 * c4] = 1.0;
    ctx->odom = std::move(ss);
    return DCREG_OK;
}

int dcreg_odometry_open(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_seqs, double cell_size, int map_frames,
                        int motion, double source_voxel, double map_voxel, int source_max_points, int map_max_points,
                        const double* T_init) {
    if (!ctx) return DCREG_BAD_ARG;
    return open_session(ctx, "odometry_open",
                        odom_settings(params, n_seqs, cell_size, map_frames, motion, source_voxel, map_voxel,
                                      source_max_points, map_max_points, T_init, ctx && ctx->lane_params));
}

int dcreg_odometry_open_map(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_seqs, double cell_size, int motion,
                            double source_voxel, double map_voxel, int source_max_points, int map_max_points,
                            double max_distance, const double* T_init) {
    if (!ctx) return DCREG_BAD_ARG;
    return open_session(ctx, "odometry_open_map",
                        odom_map_settings(params, n_seqs, cell_size, motion, source_voxel, map_voxel, source_max_points,
                                          map_max_points, max_distance, T_init, ctx && ctx->lane_params));
}

int dcreg_odometry_open_adaptive(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_seqs, double cell_size,
                                 int map_frames, int motion, double source_voxel, double map_voxel, int source_max_points,
                                 int map_max_points, double max_distance, const dcreg_adaptive_threshold* adaptive,
                                 const double* T_init) {
    if (!ctx) return DCREG_BAD_ARG;
    return open_session(ctx, "odometry_open_adaptive",
                        odom_adaptive_settings(params, n_seqs, cell_size, map_frames, motion, source_voxel, map_voxel,
                                               source_max_points, map_max_points, max_distance, adaptive, T_init,
                                               ctx && ctx->lane_params));
}

int dcreg_odometry_open_gyro(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_seqs, double cell_size, int map_frames,
                             int motion, double source_voxel, double map_voxel, int source_max_points,
                             int map_max_points, double max_distance, const dcreg_adaptive_threshold* adaptive,
                             const dcreg_gyro* gyro, const double* T_init) {
    if (!ctx) return DCREG_BAD_ARG;
    return open_session(ctx, "odometry_open_gyro",
                        odom_gyro_settings(odom_adaptive_settings(params, n_seqs, cell_size, map_frames, motion,
                                                                  source_voxel, map_voxel, source_max_points,
                                                                  map_max_points, max_distance, adaptive, T_init,
                                                                  ctx && ctx->lane_params),
                                           gyro));
}

int dcreg_odometry_open_imu(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_seqs, double cell_size, int map_frames,
                            int motion, double source_voxel, double map_voxel, int source_max_points, int map_max_points,
                            double max_distance, const dcreg_adaptive_threshold* adaptive, const dcreg_imu* imu,
                            const double* T_init, const double* v_init) {
    if (!ctx) return DCREG_BAD_ARG;
    return open_session(ctx, "odometry_open_imu",
                        odom_imu_settings(odom_adaptive_settings(params, n_seqs, cell_size, map_frames, motion,
                                                                 source_voxel, map_voxel, source_max_points,
                                                                 map_max_points, max_distance, adaptive, T_init,
                                                                 ctx && ctx->lane_params),
                                          imu, v_init));
}

int dcreg_odometry_local_map(dcreg_ctx* ctx, int seq, float* xyz, int64_t cap, int64_t* n) {
    if (!ctx) return DCREG_BAD_ARG;
    if (!ctx->odom) { ctx->err = "odometry_local_map: no session is open (dcreg_odometry_open_map)"; return DCREG_BAD_ARG; }
    const dcreg_ctx::OdomSession& ss = *ctx->odom;
    if (ss.set.prior_map) {
        ctx->err = "odometry_local_map: the session registers against the prior map (dcreg_set_prior_map): no local map";
        return DCREG_BAD_ARG;
    }
    if (!ss.set.voxel_map) {
        ctx->err = "odometry_local_map: the session keeps a window of frames, not a voxel map (dcreg_odometry_open_map)";
        return DCREG_BAD_ARG;
    }
    if (!n || seq < 0 || seq >= ss.set.n_seqs) {
        ctx->err = "odometry_local_map: null n, or seq outside [0, n_seqs)";
        return DCREG_BAD_ARG;
    }
    const long long a = ss.map_off[(size_t)seq], m = ss.map_off[(size_t)seq + 1] - a;
    *n = m;
    if (cap < m || (m > 0 && !xyz)) {
        ctx->err = "odometry_local_map: sequence " + std::to_string(seq) + "'s map has " + std::to_string(m) +
                   " points, more than cap = " + std::to_string(cap) + " (or xyz is null)";
        return DCREG_BAD_ARG;
    }
    if (m == 0) return DCREG_OK;
    CK(cudaSetDevice(ctx->device));
    std::vector<float4> h((size_t)m);
    CK(cudaMemcpyAsync(h.data(), ss.win[ss.cur].p + a, (size_t)m * sizeof(float4), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    for (long long i = 0; i < m; ++i) {
        xyz[3 * i] = h[(size_t)i].x; xyz[3 * i + 1] = h[(size_t)i].y; xyz[3 * i + 2] = h[(size_t)i].z;
    }
    return DCREG_OK;
}

int dcreg_odometry_push(dcreg_ctx* ctx, const int* seq_offsets, int n_frames, const float* xyz,
                        const int64_t* frame_offsets, int stride, const double* deltas, int64_t* frame_points,
                        double* T_prior, double* T_out, int* n_iterations, int* converged, int* status, double* cov,
                        dcreg_iter_log* log, int log_cap) {
    if (!ctx) return DCREG_BAD_ARG;
    if (!ctx->odom) { ctx->err = "odometry_push: no session is open (dcreg_odometry_open)"; return DCREG_BAD_ARG; }
    dcreg_ctx::OdomSession& ss = *ctx->odom;
    return run_odometry(ctx, "odometry_push", ss.set, &ss, seq_offsets, n_frames, xyz, frame_offsets, stride, deltas,
                        nullptr, Results{T_out, n_iterations, converged, status, log, log_cap, cov, T_prior},
                        frame_points, nullptr);
}

int dcreg_odometry_push_deskew(dcreg_ctx* ctx, const int* seq_offsets, int n_frames, const float* xyz,
                               const int64_t* frame_offsets, int stride, const double* deltas, const float* timestamps,
                               int64_t* frame_points, double* T_prior, double* T_out, int* n_iterations, int* converged,
                               int* status, double* cov, float* deskewed_xyz, dcreg_iter_log* log, int log_cap) {
    if (!ctx) return DCREG_BAD_ARG;
    if (!ctx->odom) { ctx->err = "odometry_push_deskew: no session is open (dcreg_odometry_open)"; return DCREG_BAD_ARG; }
    dcreg_ctx::OdomSession& ss = *ctx->odom;
    return run_odometry(ctx, "odometry_push_deskew", ss.set, &ss, seq_offsets, n_frames, xyz, frame_offsets, stride,
                        deltas, timestamps, Results{T_out, n_iterations, converged, status, log, log_cap, cov, T_prior},
                        frame_points, deskewed_xyz);
}

int dcreg_odometry_push_adaptive(dcreg_ctx* ctx, const int* seq_offsets, int n_frames, const float* xyz,
                                 const int64_t* frame_offsets, int stride, const double* deltas, const float* timestamps,
                                 int64_t* frame_points, double* T_prior, double* T_out, int* n_iterations, int* converged,
                                 int* status, double* cov, float* deskewed_xyz, double* search_radius, dcreg_iter_log* log,
                                 int log_cap) {
    if (!ctx) return DCREG_BAD_ARG;
    if (!ctx->odom) { ctx->err = "odometry_push_adaptive: no session is open (dcreg_odometry_open)"; return DCREG_BAD_ARG; }
    dcreg_ctx::OdomSession& ss = *ctx->odom;
    return run_odometry(ctx, "odometry_push_adaptive", ss.set, &ss, seq_offsets, n_frames, xyz, frame_offsets, stride,
                        deltas, timestamps, Results{T_out, n_iterations, converged, status, log, log_cap, cov, T_prior},
                        frame_points, deskewed_xyz, search_radius);
}

int dcreg_odometry_push_gyro(dcreg_ctx* ctx, const int* seq_offsets, int n_frames, const float* xyz,
                             const int64_t* frame_offsets, int stride, const double* deltas, const float* timestamps,
                             const double* frame_times, const double* samples, const int64_t* sample_offsets,
                             int64_t* frame_points, double* T_prior, double* T_out, int* n_iterations, int* converged,
                             int* status, double* cov, float* deskewed_xyz, double* search_radius, dcreg_iter_log* log,
                             int log_cap) {
    if (!ctx) return DCREG_BAD_ARG;
    if (!ctx->odom) { ctx->err = "odometry_push_gyro: no session is open (dcreg_odometry_open_gyro)"; return DCREG_BAD_ARG; }
    dcreg_ctx::OdomSession& ss = *ctx->odom;
    return run_odometry(ctx, "odometry_push_gyro", ss.set, &ss, seq_offsets, n_frames, xyz, frame_offsets, stride,
                        deltas, timestamps, Results{T_out, n_iterations, converged, status, log, log_cap, cov, T_prior},
                        frame_points, deskewed_xyz, search_radius, GyroInput{frame_times, samples, sample_offsets});
}

int dcreg_odometry_push_imu(dcreg_ctx* ctx, const int* seq_offsets, int n_frames, const float* xyz,
                            const int64_t* frame_offsets, int stride, const double* deltas, const float* timestamps,
                            const double* frame_times, const double* samples, const int64_t* sample_offsets,
                            int64_t* frame_points, double* T_prior, double* T_out, int* n_iterations, int* converged,
                            int* status, double* cov, float* deskewed_xyz, double* search_radius, double* velocity,
                            dcreg_iter_log* log, int log_cap) {
    if (!ctx) return DCREG_BAD_ARG;
    if (!ctx->odom) { ctx->err = "odometry_push_imu: no session is open (dcreg_odometry_open_imu)"; return DCREG_BAD_ARG; }
    dcreg_ctx::OdomSession& ss = *ctx->odom;
    return run_odometry(ctx, "odometry_push_imu", ss.set, &ss, seq_offsets, n_frames, xyz, frame_offsets, stride,
                        deltas, timestamps, Results{T_out, n_iterations, converged, status, log, log_cap, cov, T_prior},
                        frame_points, deskewed_xyz, search_radius,
                        GyroInput{frame_times, samples, sample_offsets, se3::kImuStride, velocity});
}

// The session's buffers go with it; nothing queued may still read them
int dcreg_odometry_close(dcreg_ctx* ctx) {
    if (!ctx) return DCREG_BAD_ARG;
    if (!ctx->odom) { ctx->err = "odometry_close: no session is open (dcreg_odometry_open)"; return DCREG_BAD_ARG; }
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->odom.reset();
    return DCREG_OK;
}

int dcreg_voxel_downsample(dcreg_ctx* ctx, int n_clouds, const float* xyz, const int64_t* offsets, int stride,
                           double voxel, float* out_xyz, int64_t* out_offsets, int64_t* out_index) {
    return dcreg_voxel_downsample_n(ctx, n_clouds, xyz, offsets, stride, voxel, 1, out_xyz, out_offsets, out_index);
}

int dcreg_voxel_downsample_n(dcreg_ctx* ctx, int n_clouds, const float* xyz, const int64_t* offsets, int stride,
                             double voxel, int max_points, float* out_xyz, int64_t* out_offsets, int64_t* out_index) {
    return dcreg_voxel_downsample_spaced(ctx, n_clouds, xyz, offsets, stride, voxel, max_points, 0.0, out_xyz,
                                         out_offsets, out_index);
}

int dcreg_voxel_downsample_spaced(dcreg_ctx* ctx, int n_clouds, const float* xyz, const int64_t* offsets, int stride,
                                  double voxel, int max_points, double min_spacing, float* out_xyz, int64_t* out_offsets,
                                  int64_t* out_index) {
    if (!ctx) return DCREG_BAD_ARG;
    auto bad = [ctx](const std::string& why) { ctx->err = "voxel_downsample: " + why; return (int)DCREG_BAD_ARG; };
    if (max_points < 1) return bad("max_points must be >= 1");
    if (!(min_spacing >= 0.0 && min_spacing < INFINITY)) return bad("min_spacing must be finite and >= 0 (0: no spacing)");
    if (n_clouds <= 0 || !xyz || !offsets || !out_xyz || !out_offsets) return bad("null pointer or n_clouds <= 0");
    if (stride < 3) return bad("stride < 3");
    if (!(voxel > 0.0 && voxel < INFINITY)) return bad("voxel must be finite and > 0");
    const std::string why = arena_plan::check_offsets(n_clouds, offsets, arena_plan::kMaxPoints, "cloud");
    if (!why.empty()) return bad(why);
    CK(cudaSetDevice(ctx->device));
    std::vector<int> out_of_range((size_t)n_clouds);
    std::vector<int64_t> kept((size_t)n_clouds + 1);
    const float* h_xyz = nullptr;
    const long long* h_index = nullptr;
    int rc = voxel_filter_host(ctx, n_clouds, xyz, offsets, stride, voxel, max_points, min_spacing, out_index != nullptr,
                               true, kept.data(), out_of_range.data(), &h_xyz, &h_index);
    if (rc) return rc;
    for (int b = 0; b < n_clouds; ++b)
        if (out_of_range[(size_t)b])
            return bad("cloud " + std::to_string(b) + ": a voxel coordinate lies outside [-2^20, 2^20) (voxel too small for "
                       "the cloud's coordinates)");
    memcpy(out_offsets, kept.data(), kept.size() * sizeof(int64_t));
    const long long k = kept[(size_t)n_clouds];
    memcpy(out_xyz, h_xyz, (size_t)k * 3 * sizeof(float));
    if (out_index) memcpy(out_index, h_index, (size_t)k * sizeof(int64_t));
    return DCREG_OK;
}

int dcreg_icp_run_pairs(dcreg_ctx* ctx, const dcreg_icp_params* params, int n_pairs, const float* src_xyz,
                        const int64_t* src_offsets, const float* tgt_xyz, const int64_t* tgt_offsets, int stride,
                        double cell_size, const double* T_init, double* T_out, int* n_iterations, int* converged,
                        int* status, double* cov, double error_threshold, double* metrics, dcreg_iter_log* log,
                        int log_cap) {
    if (!ctx) return DCREG_BAD_ARG;
    BatchCheck c{"icp_run_pairs", params && n_pairs > 0 && src_xyz && src_offsets && tgt_xyz && tgt_offsets && T_init && T_out,
                 "null pointer or n_pairs <= 0", "pairs are independent - give each rank its own, do not shard them", n_pairs};
    c.offsets = src_offsets; c.item = "source"; c.stride = stride; c.own_cell = true; c.cell_size = cell_size;
    c.need_target = false;
    c.lanes = ctx->lane_params ? n_pairs : 0;
    int rc = check_batch_call(ctx, params, c);
    if (rc) return rc;
    const std::string why = arena_plan::check_offsets(n_pairs, tgt_offsets, arena_plan::kMaxPoints, "icp_run_pairs: target");
    if (!why.empty()) { ctx->err = why; return DCREG_BAD_ARG; }
    const long long n_tgt = tgt_offsets[n_pairs];
    CK(cudaSetDevice(ctx->device));
    CK(ctx->d_pair_tgt_seg.ensure(n_pairs + 1));
    CK(ctx->d_pair_T.ensure((long long)n_pairs * 16));
    CK(ctx->d_pair_tgt.ensure(n_tgt));
    CK(cudaMemcpyAsync(ctx->d_pair_tgt_seg, tgt_offsets, (size_t)(n_pairs + 1) * sizeof(long long), cudaMemcpyHostToDevice, ctx->stream));
    // the targets: packed with w = index over all targets, then every pair's dense grid in the arena
    if ((rc = upload_points(ctx, tgt_xyz, n_tgt, stride, nullptr, 1, ctx->d_pair_tgt, nullptr))) return rc;
    Batch S{n_pairs, src_xyz, stride, src_offsets};
    int sparse_at = -1;             // (sparse_maps) the targets are sparse row indexes: the first too large for a grid
    if ((rc = build_grid_arena(ctx, ctx->pair_tgt, ctx->d_pair_tgt, tgt_offsets, ctx->d_pair_tgt_seg, n_pairs, cell_size,
                               search_rings(params->search_radius, cell_size), "icp_run_pairs: target", &S.cells,
                               ctx->sparse_maps ? &sparse_at : nullptr)))
        return rc;
    S.sort = Batch::kGridTable;
    S.grid_table = true; S.grids = ctx->pair_tgt.d_grids; S.cell_off = ctx->pair_tgt.d_cell_off; S.cell_size = cell_size;
    S.sparse = sparse_at >= 0;
    if ((rc = stage_sources(ctx, S)) ||
        (rc = run_loop(ctx, params, n_pairs, T_init, Results{T_out, n_iterations, converged, status, log, log_cap, cov}, true,
                       &S, call_lanes(params, n_pairs, ctx->lane_params))))
        return rc;
    if (!metrics) return DCREG_OK;
    if (S.sparse) {                 // nn1_search expands rings over the whole box
        ctx->err = sparse_at < n_pairs
                       ? "p2p metrics: the target of pair " + std::to_string(sparse_at) +
                             " is too large for a dense grid (a sparse row index: the metrics need the dense grid)"
                       : std::string("p2p metrics: the targets of the call exceed 2^30 dense cells in total (sparse row "
                                     "indexes: the metrics need dense grids), from pair 0");
        return DCREG_BAD_ARG;
    }
    CK(cudaMemcpyAsync(ctx->d_pair_T, T_out, (size_t)n_pairs * 16 * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    return p2p_metrics(ctx, n_pairs, ctx->d_scan_src, ctx->d_scan_seg, src_offsets, ctx->d_pair_tgt, ctx->d_pair_tgt_seg,
                       tgt_offsets, ctx->pair_tgt.d_grids, ctx->d_pair_T, cell_size, error_threshold,
                       "p2p metrics: the aligned source of pair", metrics);
}

int dcreg_icp_run_host_planes(dcreg_ctx* ctx, const dcreg_icp_params* params, const double T_init[16],
                              dcreg_plane_callback cb, void* user, double T_out[16], dcreg_iter_log* log,
                              int log_cap, int* n_iterations, int* converged) {
    if (!ctx) return DCREG_BAD_ARG;
    if (!params || !T_init || !T_out || !cb) { ctx->err = "icp_run_host_planes: null pointer"; return DCREG_BAD_ARG; }
    if (!ctx->d_src || ctx->n_src <= 0) { ctx->err = "[ICP Error] Input measure cloud is null or empty."; return DCREG_BAD_ARG; }
    CK(cudaSetDevice(ctx->device));
    int status = DCREG_OK;
    const Results R{T_out, n_iterations, converged, &status, log, log_cap};
    dcreg_iter_log* dlog = nullptr;
    int rc;
    if ((rc = setup_log(ctx, R, 1, &dlog))) return rc;
    CK(ctx->d_planes64.ensure(ctx->n_src));
    CK(ctx->d_planes32.ensure(ctx->n_src));
    CK(ctx->h_pinned.ensure((long long)(sizeof(IcpState) + (size_t)ctx->n_src * sizeof(double4))));
    IcpState* hs = (IcpState*)ctx->h_pinned.p;
    double* hplanes = (double*)(ctx->h_pinned.p + sizeof(IcpState));
    if ((rc = init_state(ctx, T_init))) return rc;
    double T[16];
    memcpy(T, T_init, sizeof(T));
    for (int it = 0; it < params->max_iterations; ++it) {
        int64_t npt = -1;
        if (cb(user, T, hplanes, &npt) != 0) { ctx->err = "plane callback failed"; return DCREG_BAD_ARG; }
        CK(cudaMemcpyAsync(ctx->d_planes64, hplanes, (size_t)ctx->n_src * sizeof(double4), cudaMemcpyHostToDevice,
                           ctx->stream));
        k1::Pose P;                                   // the host holds the current pose in this mode
        for (int r = 0; r < 3; ++r) {
            for (int c = 0; c < 3; ++c) P.R[r * 3 + c] = T[r * 4 + c];
            P.t[r] = T[r * 4 + 3];
        }
        // n_corr_pt is the caller's count (5th neighbour inside the radius, BEFORE the plane gates:
        // icp_test_runner.cpp:1726-1731, 1856), not the number of non-zero planes K1 sees
        if ((rc = launch_reduce(ctx, ctx->d_src, ctx->d_planes64, true, ctx->n_src, &P, params->use_weight_derivative,
                                params->weight_slope, params->weight_gate, npt >= 0 ? (double)npt : -1.0)))
            return rc;
        if ((rc = nccl_allreduce_acc(ctx))) return rc;
        if ((rc = launch_k2(ctx, params, dlog, log_cap, kCoherentStep))) return rc;
        CK(cudaMemcpyAsync(hs, ctx->d_state, sizeof(IcpState), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        for (int r = 0; r < 3; ++r) {
            for (int c = 0; c < 3; ++c) T[r * 4 + c] = hs->R[r * 3 + c];
            T[r * 4 + 3] = hs->t[r];
        }
        if (hs->done) break;
    }
    if ((rc = finish_call(ctx, params, 1, dlog, R))) return rc;
    return status;
}

int dcreg_last_covariance(dcreg_ctx* ctx, double cov[36]) {
    if (!ctx || !cov) return DCREG_BAD_ARG;
    CK(cudaSetDevice(ctx->device));
    covariance_kernel<<<1, 32, 0, ctx->stream>>>(ctx->d_state, ctx->d_small + 256);
    ctx->launches++;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(cov, ctx->d_small + 256, 36 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return DCREG_OK;
}

int dcreg_comm_unique_id(dcreg_ctx* ctx, uint8_t id_out[128]) {
    if (!ctx || !id_out) return DCREG_BAD_ARG;
    if (!g_nccl.load(ctx->err)) return DCREG_NCCL_ERROR;
    ncclUniqueId id;
    int r = g_nccl.GetUniqueId(&id);
    if (r != 0) { ctx->err = "ncclGetUniqueId failed"; return DCREG_NCCL_ERROR; }
    memcpy(id_out, id.internal, 128);
    return DCREG_OK;
}

// Map every rank's mailbox into this process (cudaIpc handles carried by one ncclAllGather): afterwards the sum over
// ranks runs inside the reducing kernels (peer_reduce.cuh) and NCCL is not on the data path any more.  Any failure
// leaves peer_ok = false: the NCCL all-reduce fallback stays in place.
static void setup_peer_mailboxes(dcreg_ctx* ctx) {
    ctx->peer_ok = false;
    if (ctx->nranks < 2 || ctx->nranks > peer::kMaxRanks || !g_nccl.AllGather || getenv("DCREG_NO_PEER")) return;
    cudaIpcMemHandle_t mine;
    unsigned char* d_handles = nullptr;
    std::vector<cudaIpcMemHandle_t> all(ctx->nranks);
    bool ok = cudaMalloc(&ctx->d_mailbox, sizeof(peer::Mailbox)) == cudaSuccess &&
              cudaMemset(ctx->d_mailbox, 0, sizeof(peer::Mailbox)) == cudaSuccess &&
              cudaIpcGetMemHandle(&mine, ctx->d_mailbox) == cudaSuccess &&
              cudaMalloc(&d_handles, sizeof(mine) * ctx->nranks) == cudaSuccess;
    // every rank takes part in the collectives below even if its own setup failed (flag travels with the handle)
    unsigned char blob[sizeof(cudaIpcMemHandle_t)];
    memset(blob, 0, sizeof(blob));
    if (ok) memcpy(blob, &mine, sizeof(mine));
    unsigned char* d_mine = nullptr;
    if (cudaMalloc(&d_mine, sizeof(blob)) != cudaSuccess) { ok = false; }
    if (!d_handles || !d_mine) {          // cannot even run the collective coherently: give up on every rank the same way
        if (d_handles) cudaFree(d_handles);
        if (d_mine) cudaFree(d_mine);
        if (ctx->d_mailbox) { cudaFree(ctx->d_mailbox); ctx->d_mailbox = nullptr; }
        cudaGetLastError();
        return;
    }
    cudaMemcpyAsync(d_mine, blob, sizeof(blob), cudaMemcpyHostToDevice, ctx->stream);
    int r = g_nccl.AllGather(d_mine, d_handles, sizeof(blob), kNcclInt8, ctx->comm, ctx->stream);
    if (r == 0) {
        cudaMemcpyAsync(all.data(), d_handles, sizeof(mine) * ctx->nranks, cudaMemcpyDeviceToHost, ctx->stream);
        if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) r = 1;
    }
    if (r != 0) ok = false;
    peer::View v{};
    v.nranks = ctx->nranks; v.rank = ctx->rank;
    for (int q = 0; q < ctx->nranks && ok; ++q) {
        static const unsigned char zero[sizeof(cudaIpcMemHandle_t)] = {0};
        if (memcmp(&all[q], zero, sizeof(zero)) == 0) { ok = false; break; }      // that rank could not export
        if (q == ctx->rank) { v.box[q] = ctx->d_mailbox; continue; }
        void* ptr = nullptr;
        if (cudaIpcOpenMemHandle(&ptr, all[q], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { ok = false; break; }
        ctx->peer_ptr[q] = ptr;
        v.box[q] = (peer::Mailbox*)ptr;
    }
    // agree: peer mode only if EVERY rank mapped everything (one more tiny collective: min over ranks)
    double* d_flag = ctx->d_small + 700;
    const double flag = ok ? 1.0 : 0.0;
    cudaMemcpyAsync(d_flag, &flag, sizeof(double), cudaMemcpyHostToDevice, ctx->stream);
    // sum of the flags == nranks  <=>  all ok
    double total = 0.0;
    if (g_nccl.AllReduce(d_flag, d_flag, 1, kNcclFloat64, kNcclSum, ctx->comm, ctx->stream) == 0) {
        cudaMemcpyAsync(&total, d_flag, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream);
        cudaStreamSynchronize(ctx->stream);
    }
    cudaFree(d_handles); cudaFree(d_mine);
    if (total > (double)ctx->nranks - 0.5) {
        ctx->peer_view = v;
        ctx->peer_ok = true;
    } else {
        for (int q = 0; q < peer::kMaxRanks; ++q)
            if (ctx->peer_ptr[q]) { cudaIpcCloseMemHandle(ctx->peer_ptr[q]); ctx->peer_ptr[q] = nullptr; }
        if (ctx->d_mailbox) { cudaFree(ctx->d_mailbox); ctx->d_mailbox = nullptr; }
        cudaGetLastError();
    }
}

int dcreg_comm_init(dcreg_ctx* ctx, const uint8_t nccl_unique_id[128], int rank, int nranks) {
    if (!ctx || !nccl_unique_id || nranks < 1 || rank < 0 || rank >= nranks) return DCREG_BAD_ARG;
    if (!g_nccl.load(ctx->err)) return DCREG_NCCL_ERROR;
    CK(cudaSetDevice(ctx->device));
    ncclUniqueId id;
    memcpy(id.internal, nccl_unique_id, 128);
    int r = g_nccl.CommInitRank(&ctx->comm, nranks, id, rank);
    if (r != 0) {
        ctx->comm = nullptr;
        ctx->err = std::string("ncclCommInitRank: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "error");
        return DCREG_NCCL_ERROR;
    }
    ctx->rank = rank; ctx->nranks = nranks;
    setup_peer_mailboxes(ctx);
    ctx->drop_graphs();
    return DCREG_OK;
}

int dcreg_comm_mode(const dcreg_ctx* ctx) {
    if (!ctx || !ctx->comm) return 0;
    return ctx->peer_ok ? 2 : 1;
}

int dcreg_comm_destroy(dcreg_ctx* ctx) {
    if (!ctx) return DCREG_BAD_ARG;
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    for (int q = 0; q < peer::kMaxRanks; ++q)
        if (ctx->peer_ptr[q]) { cudaIpcCloseMemHandle(ctx->peer_ptr[q]); ctx->peer_ptr[q] = nullptr; }
    if (ctx->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(ctx->comm);     // (a collective: peers are still alive here)
    if (ctx->d_mailbox) { cudaFree(ctx->d_mailbox); ctx->d_mailbox = nullptr; }
    ctx->peer_ok = false; ctx->peer_view = peer::View{};
    ctx->comm = nullptr; ctx->rank = 0; ctx->nranks = 1;
    ctx->drop_graphs();
    return DCREG_OK;
}

}  // extern "C"
