// k1_stream.cuh - K1, the streaming kernel: fused point-to-plane residual / LOAM weight / gate / 6-DoF Jacobian
// row / 21 + 6 (+2) normal-equation sums over device-resident (point, plane) slots, for sm_90a.
//
// Shape of the kernel and why (tools/microbench*.cu measure the pipe costs this rests on):
//   * Cost model.  The FP64 vector ops (DFMA/DMUL/DADD), the FP64 tensor op (DMMA m8n8k4) and the 64-bit
//     conversions (F2F) all issue through one shared pipe, and their costs ADD to the cycle every other instruction
//     takes: the kernel time is (instructions + extra FP64 slots) / issue rate, independent of occupancy once latency
//     is covered.  Rewrites that only move work between those units (LDG vs TMA bulk + mbarrier ring vs cp.async
//     ring, 8..32 warps/SM, 1..4 slots per thread, vector vs DMMA accumulation, F2F vs integer conversions) did not
//     lower that sum during development (not re-measured on H100).
//   * So the kernel minimises issue slots per slot: float->double
//     is 3-4 integer instructions (IMAD.WIDE shifts the float fields into place; for the point the exponent re-bias
//     is folded into the rotation constants), the reference's float32 round trips are 4 (LEA carry trick), the 29
//     sums are plain DFMA chains (29 x 2 slots, cheaper than 8 DMMA x 16.4 + the 16 LDS/STS of a fragment
//     transpose), pose and gate constants live in the kernel-parameter constant bank, and the main loop is unrolled
//     over the 4 ring slots with no predicates: ring addresses and copy offsets are immediates.
//   * Loads: each lane copies its own 16 B point and 16 B (32 B) plane with cp.async (LDGSTS, L1 bypass) into a
//     lane-private 4-deep shared-memory ring, so the ring needs NO barrier (only cp.async.wait_group) and no
//     registers; 16 warps x 4 KB are in flight per SM.  (TMA bulk copies were tried first: a single producer
//     thread per CTA streamed less than per-lane LDGSTS/LDG in a copy-only experiment during development; not
//     re-measured on H100.)
//     A CTA streams one contiguous range of each array; its warps interleave 512 B chunks inside it.
//   * Reduction: 31-shuffle transpose-reduction per warp -> per-block partial (32 doubles) -> the last block (atomic
//     ticket) sums the partials in a fixed order with all loads in flight at once, applies the world->body
//     congruence with 42 threads and writes the 27 + stats.  Deterministic for a given grid size.
//   * Measured time on H100: bench.py's `roofline` and `reduction` entries (DESIGN.md §4).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "k1_reduce.cuh"
#include "peer_reduce.cuh"

namespace k1s {

constexpr int kWarpsPerBlock = 8;
constexpr int kThreads = kWarpsPerBlock * 32;
constexpr int kDepth = 4;                // chunks in flight per warp (a chunk = 32 slots = 1 KB, 1.5 KB with FP64 planes)
static_assert((kDepth & (kDepth - 1)) == 0, "ring depth must be a power of two");

struct Args {
    const float4* src;
    const void* plane;
    long long n;
    k1::Pose pose;
    double Rs[9];                // R * 2^896: undoes the exponent bias the raw point conversion leaves out (f32_raw)
    double slope, gate;          // LOAM weight 1 - slope |r| (0.9) and its gate (0.1): constant-bank operands
    double* partials;            // [grid][kPk]
    unsigned int* counter;
    double* acc;                 // [k2::kAcc] final, body frame
    double npt_override;         // >= 0: N_corr_pt of this rank as counted by the caller's correspondence stage (host-kd-tree
                                 // mode: the reference counts BEFORE the plane gates, icp_test_runner.cpp:1726-1731, 1856)
    peer::View peer;             // multi-GPU: sum over ranks inside the last block (nranks <= 1: none)
};

// 16-byte asynchronous global -> shared copy (LDGSTS), L1 bypassed: the data is streamed exactly once
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
    const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ---- integer-ALU conversions (the FP64 pipe is the binding resource: k1_reduce.cuh) ------------------------------
// float -> double * 2^-896 in 3 instructions (LOP3, IMAD.WIDE, LOP3): the float's exponent/mantissa bits are shifted
// into the FP64 fields without re-biasing the exponent; the missing 2^896 is folded into the rotation constants
// (Args::Rs), which is exact.  +-0 stays +-0.
__device__ __forceinline__ double f32_raw(float f) {
    const unsigned u = __float_as_uint(f);
    unsigned long long w;
    asm("mul.wide.u32 %0, %1, 0x20000000;" : "=l"(w) : "r"(u & 0x7fffffffu));
    return __hiloint2double((int)((unsigned)(w >> 32) | (u & 0x80000000u)), (int)(unsigned)w);
}
// float -> double in 4 instructions.  Exact for every normal float; +-0 and float denormals (|x| < 1.2e-38) come out
// as +-2^-127-sized values instead of 0 (an absolute perturbation of 1e-38 on a plane component), and Inf / NaN map to
// finite values (plane_to_f64 drops such a slot).
__device__ __forceinline__ double f32_f64(float f) {
    const unsigned u = __float_as_uint(f);
    unsigned long long w;
    asm("mul.wide.u32 %0, %1, 0x20000000;" : "=l"(w) : "r"(u & 0x7fffffffu));
    return __hiloint2double((int)((unsigned)(w >> 32) + ((u & 0x80000000u) | 0x38000000u)), (int)(unsigned)w);
}
// (double)(float)x, round-to-nearest-even on the FP64 bit pattern in 4 instructions: LEA (bit 29 -> carry),
// IADD3.X (+ 0x0FFFFFFF + carry), IADD3.X (carry into the high word), LOP3.  Same values as k1::round_f32.
__device__ __forceinline__ double rnd_f32(double x) {
    const unsigned lo = (unsigned)__double2loint(x), hi = (unsigned)__double2hiint(x);
    unsigned lo2, hi2;
    asm("{\n\t.reg .u32 t;\n\t"
        "shl.b32 t, %2, 2;\n\t"
        "add.cc.u32 t, t, 0x80000000;\n\t"
        "addc.cc.u32 %0, %2, 0x0FFFFFFF;\n\t"
        "addc.u32 %1, %3, 0;\n\t}"
        : "=r"(lo2), "=r"(hi2) : "r"(lo), "r"(hi));
    return __hiloint2double((int)hi2, (int)(lo2 & 0xE0000000u));
}

// Non-finite inputs.  The integer conversions above map NaN and +-Inf to finite values, so a NaN would not reach r by
// itself: with an exactly zero plane component (0 x huge = 0) r can stay small and the slot pass the gate, adding
// ~1e77 to H.  In the reference such a slot has a NaN or infinite r, hence s = max(0, .) = 0 (icp_test_runner.cpp:1776),
// and is dropped.  So `has` also requires every input of the slot to be finite: the integer max of the magnitude bits
// (the same `& 0x7fffffff` the conversions use) below the all-ones exponent, on the integer pipe.
__device__ __forceinline__ unsigned f32_mag(float f) { return __float_as_uint(f) & 0x7fffffffu; }

template <typename PlaneT>
__device__ __forceinline__ void plane_to_f64(const PlaneT& v, double& nx, double& ny, double& nz, double& d, bool& has);
template <>
__device__ __forceinline__ void plane_to_f64<float4>(const float4& v, double& nx, double& ny, double& nz, double& d,
                                                     bool& has) {
    const unsigned mn = max(max(f32_mag(v.x), f32_mag(v.y)), f32_mag(v.z));
    has = (mn - 1u) < 0x7f7fffffu && f32_mag(v.w) < 0x7f800000u;  // a non-zero, finite normal and a finite offset
    nx = f32_f64(v.x); ny = f32_f64(v.y); nz = f32_f64(v.z); d = f32_f64(v.w);
}
template <>
__device__ __forceinline__ void plane_to_f64<double4>(const double4& v, double& nx, double& ny, double& nz, double& d,
                                                      bool& has) {
    const unsigned hx = (unsigned)__double2hiint(v.x) & 0x7fffffffu, hy = (unsigned)__double2hiint(v.y) & 0x7fffffffu;
    const unsigned hz = (unsigned)__double2hiint(v.z) & 0x7fffffffu, hd = (unsigned)__double2hiint(v.w) & 0x7fffffffu;
    const unsigned lo = (unsigned)__double2loint(v.x) | (unsigned)__double2loint(v.y) | (unsigned)__double2loint(v.z);
    has = ((hx | hy | hz | lo) != 0u) && max(max(hx, hy), max(hz, hd)) < 0x7ff00000u;
    // a dropped slot's s is +0, and 0 x NaN or 0 x Inf in s n would still reach the sums: keep only the low words of
    // such a normal (a finite value below 2^-1022, like the leftovers of s and r in front)
    nx = __hiloint2double(has ? __double2hiint(v.x) : 0, __double2loint(v.x));
    ny = __hiloint2double(has ? __double2hiint(v.y) : 0, __double2loint(v.y));
    nz = __hiloint2double(has ? __double2hiint(v.z) : 0, __double2loint(v.z));
    d = v.w;
}

// Per-slot front of the streaming kernel: same arithmetic as k1::slot_front (k1_reduce.cuh), issue-slot trimmed:
// raw-scaled point conversion, 4-instruction rounding, gate constants from the constant bank, and an invalid slot is
// dropped by zeroing only the HIGH words of s and r (the leftovers are < 2^-1022, so every product that reaches an
// accumulator underflows to exactly 0).  counts: bit 0.. = slots with a plane (non-zero, finite), bit 16.. = slots
// that pass the gate (and whose point is finite).
template <bool kUseWd>
__device__ __forceinline__ void front(const Args& a, float4 p, double nx, double ny, double nz, double d, bool has,
                                      double (&c)[8], unsigned& counts) {
    const double px = f32_raw(p.x), py = f32_raw(p.y), pz = f32_raw(p.z);
    const double wx = fma(a.Rs[2], pz, fma(a.Rs[1], py, a.Rs[0] * px));   // Rp (no translation)
    const double wy = fma(a.Rs[5], pz, fma(a.Rs[4], py, a.Rs[3] * px));
    const double wz = fma(a.Rs[8], pz, fma(a.Rs[7], py, a.Rs[6] * px));
    const double qx = rnd_f32(wx + a.pose.t[0]);                  // utils.hpp:630-636 (float32 store)
    const double qy = rnd_f32(wy + a.pose.t[1]);
    const double qz = rnd_f32(wz + a.pose.t[2]);
    const double rr = fma(nx, qx, fma(ny, qy, fma(nz, qz, d)));   // icp_test_runner.cpp:1774
    const double ss = fma(fabs(rr), -a.slope, 1.0);               // :1776 (max(0, .) is implied by the gate)
    const bool finite = max(max(f32_mag(p.x), f32_mag(p.y)), f32_mag(p.z)) < 0x7f800000u;   // (plane: in `has`)
    const bool valid = has && finite && (ss > a.gate);            // :1785
    const double s = __hiloint2double(valid ? __double2hiint(ss) : 0, __double2loint(ss));
    const double r = __hiloint2double(valid ? __double2hiint(rr) : 0, __double2loint(rr));
    double ux = rnd_f32(s * nx);                                  // coeff.x/y/z (:1787-1789)
    double uy = rnd_f32(s * ny);
    double uz = rnd_f32(s * nz);
    c[6] = -rnd_f32(s * r);                                       // -coeff.intensity (:1790, 1906)
    c[7] = r;
    if (kUseWd) {                                                 // :1780-1783, 1898: row scale w/s = 2 - 1/s on 0 < s < 1
        const double sw = valid ? ss : 1.0;                       // (s == 1 gives k = 1: no derivative, as in the reference)
        const double k = 2.0 - k1::rcp_newton(sw);
        ux *= k; uy *= k; uz *= k;
    }
    c[0] = wy * uz - wz * uy;                                     // Rp x (k u')
    c[1] = wz * ux - wx * uz;
    c[2] = wx * uy - wy * ux;
    c[3] = ux; c[4] = uy; c[5] = uz;
    counts += (has ? 1u : 0u) + (valid ? 0x10000u : 0u);
}

template <typename PlaneT> struct SlotPair { float4 p; PlaneT pl; };
struct TrueT { static constexpr bool value = true; };
struct FalseT { static constexpr bool value = false; };

// packed per-block partial of the streaming kernel: 21 upper-triangular entries of the world-frame H (row-major
// over i <= j), 6 rhs, sum r^2, sum b^2, N_eff, N_pt, pad
constexpr int kPk = 32, kPkG = 21, kPkR2 = 27, kPkB2 = 28, kPkNeff = 29, kPkNpt = 30;

struct TailSmem {
    double red[kWarpsPerBlock][kPk];
    double fin[kPk];
    double acc[kPk];             // body-frame accumulators (k2::kAcc layout): input of the in-kernel solve step
    bool is_last;
};

__device__ __forceinline__ int pk_index(int a, int b) {           // packed upper-triangular index of H(a, b), 6 x 6
    const int i = a < b ? a : b, j = a < b ? b : a;
    return i * 6 - (i * (i - 1)) / 2 + (j - i);
}

// Grid reduction of the packed partials, in two steps so that the multi-GPU exchange (peer_reduce.cuh) and the solve
// step (the loop kernel) can sit between / behind them inside the same kernel.
//
// reduce_to_fin: every lane of every warp calls this with its warp's total number `lane`.  warp totals -> block
// partial (32 doubles, one coalesced 256 B row) -> atomic ticket -> the last block sums the rows in a fixed order
// (warp w: rows w, w + 8, ...; all of a lane's loads are in flight at once) into ts.fin (world frame, packed kPk
// layout).  Returns true in every thread of the last block.  Deterministic for a given grid size.
// `nblocks` = blocks that feed this ticket (gridDim.x; the loop kernel has one ticket per trial = per blockIdx.y).
__device__ __forceinline__ bool reduce_to_fin(double mine, TailSmem& ts, double* partials, unsigned int* counter,
                                              int block, int nblocks) {
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    ts.red[warp][lane] = mine;
    __syncthreads();
    if (warp == 0) {
        double s = 0.0;
#pragma unroll
        for (int w = 0; w < kWarpsPerBlock; ++w) s += ts.red[w][lane];
        partials[(size_t)block * kPk + lane] = s;
        __syncwarp();                                             // the warp's 32 stores happen-before lane 0's release
        if (lane == 0) {
            // ticket with release (this block's partial row is visible before the count) and acquire (the last block
            // sees every other block's row) semantics at GPU scope: one atomic instead of fence + atomic + fence
            unsigned int t;
            asm volatile("atom.add.acq_rel.gpu.global.u32 %0, [%1], 1;" : "=r"(t) : "l"(counter) : "memory");
            ts.is_last = (t == (unsigned)nblocks - 1u);
        }
    }
    __syncthreads();
    if (!ts.is_last) return false;
    {
        constexpr int kRows = 40;                                  // rows in flight per lane and trip
        double s = 0.0;
        for (int b0 = warp; b0 < nblocks; b0 += kWarpsPerBlock * kRows) {
            double t[kRows];
#pragma unroll
            for (int u = 0; u < kRows; ++u) {
                const int b = b0 + u * kWarpsPerBlock;
                t[u] = (b < nblocks) ? __ldcg(partials + (size_t)b * kPk + lane) : 0.0;
            }
#pragma unroll
            for (int u = 0; u < kRows; ++u) s += t[u];
        }
        ts.red[warp][lane] = s;                                   // (red[][] was last read before the ticket's barrier)
    }
    __syncthreads();
    if (warp == 0) {
        double s = 0.0;
#pragma unroll
        for (int w = 0; w < kWarpsPerBlock; ++w) s += ts.red[w][lane];
        ts.fin[lane] = s;
        if (lane == 0) *counter = 0u;                             // every block has arrived: ready for the next launch
    }
    __syncthreads();
    return true;
}

// Solver-block variant of the same reduction (the loop kernel's single-trial path, dcreg_b200.cu): no ticket; a block
// that has written its row publishes it with a per-row flag, and one dedicated block sums the rows while they land.
//
// Order rule, shared with reduce_to_fin: fin[l] = ((0 + W_0[l]) + W_1[l]) + ... + W_7[l], where W_w[l] =
// ((0 + row_w[l]) + row_{w+8}[l]) + row_{w+16}[l] + ... in increasing row order.  stream_rows_to_fin performs exactly
// these additions, only earlier: a row is added once it and every earlier row of its warp's sequence have landed, so
// the result is bit-identical to reduce_to_fin over the same rows.
//
// Flags carry `want` = epoch + 1 of the launch (a per-context counter that only grows): flags are never reset, and a
// flag left by an earlier launch holds a smaller value, so it never matches.
__device__ __forceinline__ void publish_row(double mine, TailSmem& ts, double* row, unsigned long long* flag,
                                            unsigned long long want) {
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    ts.red[warp][lane] = mine;
    __syncthreads();
    if (warp == 0) {
        double s = 0.0;
#pragma unroll
        for (int w = 0; w < kWarpsPerBlock; ++w) s += ts.red[w][lane];
        row[lane] = s;
        __syncwarp();                                             // the warp's 32 stores happen-before lane 0's release
        if (lane == 0) asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(flag), "l"(want) : "memory");
    }
}

// All threads of the solver block call this (a warp may arrive late: nothing waits for it before the final barrier).
// Warp w polls the flags of its next 32 rows (one acquire load per lane), takes the ready prefix of its sequence and
// issues all of that prefix's loads at once, so after the last row lands about one poll round and the 8-way sum remain.
// Returns false in every thread if a warp still missed a row `timeout_ns` after it first found none ready (ts.fin is
// then meaningless).
__device__ __forceinline__ bool stream_rows_to_fin(TailSmem& ts, const double* partials, const unsigned long long* flags,
                                                   unsigned long long want, int nrows, unsigned long long timeout_ns) {
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    double s = 0.0;
    bool timed_out = false;
    int k = 0;                                                    // rows warp + 8 j, j < k, are summed
    unsigned long long t0 = 0;
    while (warp + kWarpsPerBlock * k < nrows) {
        const int r = warp + kWarpsPerBlock * (k + lane);
        bool ready = true;                                        // rows past the end count as landed
        if (r < nrows) {
            unsigned long long f;
            asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(f) : "l"(flags + r) : "memory");
            ready = f == want;
        }
        const unsigned int bits = __ballot_sync(0xffffffffu, ready);
        const int n = bits == 0xffffffffu ? 32 : __ffs(~bits) - 1;    // ready prefix of the warp's sequence
        __syncwarp();                                             // the acquiring lanes' view reaches every lane
        for (int j0 = 0; j0 < n; j0 += 8) {
            double t[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int b = warp + kWarpsPerBlock * (k + j0 + u);
                t[u] = (j0 + u < n && b < nrows) ? __ldcg(partials + (size_t)b * kPk + lane) : 0.0;
            }
#pragma unroll
            for (int u = 0; u < 8; ++u)
                if (j0 + u < n && warp + kWarpsPerBlock * (k + j0 + u) < nrows) s += t[u];
        }
        k += n;
        if (n == 0) {
            unsigned long long now;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
            if (t0 == 0) t0 = now;
            else if (now - t0 > timeout_ns) { timed_out = true; break; }
        }
    }
    ts.red[warp][lane] = s;
    const bool ok = !__syncthreads_or(timed_out);
    if (warp == 0) {
        double f = 0.0;
#pragma unroll
        for (int w = 0; w < kWarpsPerBlock; ++w) f += ts.red[w][lane];
        ts.fin[lane] = f;
    }
    __syncthreads();
    return ok;
}

// world -> body: H_body = Q^T H Q, g_body = Q^T g with Q = blkdiag(R, R); one thread per output entry.  fin: packed
// world-frame totals (shared memory), out: k2::kAcc doubles (shared or global).  Called by all threads of the block.
__device__ __forceinline__ void congruence(const double* fin, const double* R, double* out) {
    const int tid = threadIdx.x;
    if (tid < 36) {
        const int i = tid / 6, j = tid % 6;
        if (j >= i) {
            const int bi = (i / 3) * 3, bj = (j / 3) * 3, ii = i % 3, jj = j % 3;
            double acc = 0.0;
#pragma unroll
            for (int k = 0; k < 3; ++k)
#pragma unroll
                for (int l = 0; l < 3; ++l) acc = fma(R[k * 3 + ii] * fin[pk_index(bi + k, bj + l)], R[l * 3 + jj], acc);
            out[pk_index(i, j)] = acc;
        }
    } else if (tid < 42) {
        const int i = tid - 36, bi = (i / 3) * 3, ii = i % 3;
        double acc = 0.0;
#pragma unroll
        for (int k = 0; k < 3; ++k) acc = fma(R[k * 3 + ii], fin[kPkG + bi + k], acc);
        out[21 + i] = acc;
    } else if (tid == 42) {
        out[k2::kAccSumR2] = fin[kPkR2];
        out[k2::kAccNeff] = fin[kPkNeff];
        out[k2::kAccNpt] = fin[kPkNpt];
        out[k2::kAccSumB2] = fin[kPkB2];
        out[k2::kAcc - 1] = 0.0;
    }
}

template <typename PlaneT>
struct Smem {
    float4 rs[kWarpsPerBlock][kDepth][32];     // lane-private ring slots: every lane copies and reads its own slot,
    PlaneT rp[kWarpsPerBlock][kDepth][32];     // so the ring needs no barrier at all, only cp.async.wait_group
    TailSmem tail;
};

template <typename PlaneT, bool kUseWd, int kTeamCtas>
__global__ void __launch_bounds__(kThreads, 2) reduce_stream_kernel(const __grid_constant__ Args a) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    Smem<PlaneT>& sm = *reinterpret_cast<Smem<PlaneT>*>(smem_raw);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const PlaneT* gplane = reinterpret_cast<const PlaneT*>(a.plane);
    const unsigned int epoch0 = peer::load_epoch(a.peer);

    double vh[21], vg[6], vr2 = 0.0, vb2 = 0.0;          // the 29 running sums of this lane's slots
#pragma unroll
    for (int i = 0; i < 21; ++i) vh[i] = 0.0;
#pragma unroll
    for (int i = 0; i < 6; ++i) vg[i] = 0.0;
    unsigned counts = 0;
    // chunk = 32 consecutive slots (one per lane).  The grid is split into teams of kTeamCtas CTAs; a team owns a
    // contiguous chunk range and its T = 8 kTeamCtas warps interleave inside it (warp i: chunks i, i + T, ...).
    // Consecutive chunks of a warp are a compile-time T chunks apart, so every copy address is the running pointer
    // plus an immediate; kTeamCtas = gridDim.x is the plain grid-stride order.
    constexpr int T = kTeamCtas * kWarpsPerBlock;
    const unsigned nchunks = (unsigned)((a.n + 31) >> 5);         // host guarantees n < 2^36
    const unsigned teams = gridDim.x / kTeamCtas, tm = blockIdx.x / kTeamCtas;
    const int wi = (int)(blockIdx.x - tm * kTeamCtas) * kWarpsPerBlock + warp;
    const unsigned per = nchunks / teams, rem = nchunks - per * teams;        // the first `rem` teams take one more
    const unsigned c_lo = tm * per + min(tm, rem);
    const unsigned c_hi = c_lo + per + (tm < rem ? 1u : 0u);
    const int cnt = (int)(c_hi - c_lo);
    const int my = (cnt > wi) ? (cnt - wi + T - 1) / T : 0;
    // only the globally last chunk can be partial; it is the last chunk of one warp of the last team
    const int last_cnt = (int)(a.n - ((long long)(nchunks - 1) << 5));
    const bool owns_last = (my > 0) && (c_hi == nchunks) && (((cnt - 1) % T) == wi);
    const int klast = (owns_last && last_cnt < 32) ? my - 1 : -1;
    constexpr int kStep = T * 32;                                 // elements between consecutive chunks of one warp
    const float4* gs = a.src + ((size_t)(c_lo + wi) << 5) + lane;   // next element to fetch (this lane)
    const PlaneT* gp = gplane + ((size_t)(c_lo + wi) << 5) + lane;
    float4* ring_s = &sm.rs[warp][0][lane];                       // + 32 per ring slot
    PlaneT* ring_p = &sm.rp[warp][0][lane];

    auto copy_chunk = [&](int slot, int ahead) {                  // chunk `ahead` past the running pointers -> ring slot
        cp_async16(ring_s + slot * 32, gs + ahead * kStep);
        cp_async16(ring_p + slot * 32, gp + ahead * kStep);
        if (sizeof(PlaneT) == 32)
            cp_async16(reinterpret_cast<char*>(ring_p + slot * 32) + 16, reinterpret_cast<const char*>(gp + ahead * kStep) + 16);
    };
#pragma unroll
    for (int j = 0; j < kDepth; ++j) {
        if (j < my && (j != klast || lane < last_cnt)) copy_chunk(j, j);
        cp_async_commit();                                        // always: uniform group count
    }
    gs += kDepth * kStep; gp += kDepth * kStep;                   // pointers now address chunk k + kDepth for k = 0

    // consume ring slot `slot` (values -> registers), then front + accumulate
    auto consume = [&](int slot, auto tail_tag) {
        constexpr bool kTail = decltype(tail_tag)::value;
        float4 p = ring_s[slot * 32];
        PlaneT pl = ring_p[slot * 32];
        if (kTail && lane >= last_cnt) {           // lanes past the end never copied anything: feed zeros, not stale bits
            p = make_float4(0.f, 0.f, 0.f, 0.f);
            pl = PlaneT{};
        }
        return SlotPair<PlaneT>{p, pl};
    };
    auto accumulate = [&](const float4& p, const PlaneT& pl) {
        double nx, ny, nz, d;
        bool has;
        plane_to_f64<PlaneT>(pl, nx, ny, nz, d, has);
        double c[8];
        front<kUseWd>(a, p, nx, ny, nz, d, has, c, counts);
        int q = 0;
#pragma unroll
        for (int i = 0; i < 6; ++i) {
#pragma unroll
            for (int j = i; j < 6; ++j) { vh[q] = fma(c[i], c[j], vh[q]); ++q; }
            vg[i] = fma(c[i], c[6], vg[i]);
        }
        vr2 = fma(c[7], c[7], vr2);
        vb2 = fma(c[6], c[6], vb2);
    };

    // main loop: chunk k is consumed and chunk k + kDepth (a certainly full chunk) refills its ring slot - no
    // predicates, ring slots and copy offsets are compile-time constants of the 4x unrolled body
    const int nfull = (klast >= 0) ? my - 1 : my;                 // chunks that are certainly full
    const int nmain = (nfull > kDepth) ? ((nfull - kDepth) & ~(kDepth - 1)) : 0;
    int k = 0;
    for (; k < nmain; k += kDepth) {
#pragma unroll
        for (int j = 0; j < kDepth; ++j) {
            cp_async_wait<kDepth - 1>();                          // chunk k + j has landed (this lane's own copies)
            const auto v = consume(j, FalseT{});
            copy_chunk(j, j);
            cp_async_commit();
            accumulate(v.p, v.pl);
        }
        gs += kDepth * kStep; gp += kDepth * kStep;
    }
    // drain: the last few chunks, with the general (predicated) refill and the peeled partial chunk
    int slot = 0;                                                 // nmain is a multiple of kDepth
    for (; k < my; ++k) {
        cp_async_wait<kDepth - 1>();
        const int kn = k + kDepth;
        const bool refill = kn < my && (kn != klast || lane < last_cnt);
        if (k != klast) {
            const auto v = consume(slot, FalseT{});
            if (refill) copy_chunk(slot, 0);
            cp_async_commit();
            accumulate(v.p, v.pl);
        } else {
            const auto v = consume(slot, TrueT{});
            cp_async_commit();
            accumulate(v.p, v.pl);
        }
        gs += kStep; gp += kStep;
        slot = (slot + 1) & (kDepth - 1);
    }
    cp_async_wait<0>();
    int neff = (int)(counts >> 16), npt = (int)(counts & 0xffffu);

    // ---- reduction tail -------------------------------------------------------------------------------------
    // warp: 5-round transpose-reduction of the 32 per-lane values (29 sums, N_eff, N_pt, pad): every round halves
    // the values a lane still carries, so 31 shuffles replace 32 x 5 butterflies and lane l ends with total l
    double v[32];
    {
        int q = 0;
#pragma unroll
        for (int i = 0; i < 6; ++i)
#pragma unroll
            for (int j = i; j < 6; ++j) { v[q] = vh[q]; ++q; }
#pragma unroll
        for (int i = 0; i < 6; ++i) v[kPkG + i] = vg[i];
        v[kPkR2] = vr2; v[kPkB2] = vb2; v[kPkNeff] = (double)neff; v[kPkNpt] = (double)npt; v[31] = 0.0;
    }
#pragma unroll
    for (int half = 16; half >= 1; half >>= 1) {
        const bool up = (lane & half) != 0;
#pragma unroll
        for (int i = 0; i < half; ++i) {
            const double send = up ? v[i] : v[i + half];
            const double keep = up ? v[i + half] : v[i];
            v[i] = keep + __shfl_xor_sync(0xffffffffu, send, half);
        }
    }
    if (!reduce_to_fin(v[0], sm.tail, a.partials, a.counter, (int)blockIdx.x, (int)gridDim.x)) return;
    if (a.peer.nranks > 1 || a.npt_override >= 0.0) {             // (uniform) host-kd-tree count, sum over ranks
        if (a.npt_override >= 0.0 && tid == 0) sm.tail.fin[kPkNpt] = a.npt_override;
        __syncthreads();
        peer::all_reduce32(a.peer, sm.tail.fin, sm.tail.red, epoch0);
    }
    congruence(sm.tail.fin, a.pose.R, a.acc);
}

}  // namespace k1s
