// k1_reduce.cuh - per-slot math of the normal equations and the loop kernel's DMMA Gram accumulation.  The loop kernel
// (dcreg_b200.cu: planes come straight out of the correspondence stage) uses it as is; the streaming kernel K1
// (k1_stream.cuh: frozen planes) has an issue-slot trimmed copy of the same arithmetic.  Both end in k1s's packed tail.
//
// Replaces, per source slot and per ICP iteration (reference file:line):
//   pointBodyToGlobal (FP64 math, float32 store)         DCReg/include/utils.hpp:630-636
//   residual + LOAM weight + gate                         DCReg/src/icp_test_runner.cpp:1774-1803
//   stream compaction of flagged slots                    icp_test_runner.cpp:1816-1840 (skipped: gated in place)
//   computePointToPlaneJacobian + row fill                DCReg/include/math_utils.hpp:102-121, icp_test_runner.cpp:1863-1907
//   H = A^T A, g = A^T b                                  icp_test_runner.cpp:1910-1919
//   SymmetricHessianComputer (21 + 6 accumulators)        DCReg/include/hessian_computer.h:62-123
//
// Formulation.  The reference's Jacobian row is (s + r ds_dr) [ -n^T R [p]x , n^T R ] with the normal rebuilt
// from the float32-stored coeff = (s n, s r) as n = coeff/s (:1786-1790, 1889, 1898, 1906).  With u' = fl32(s n)
// and w = s + r ds_dr this row equals
//       (w/s) [ (Rp x u')^T , u'^T ] blkdiag(R, R),
// so per slot only the 8 world-frame components c = [k (Rp x u'), k u', b, r] are formed (k = w/s = 1 without
// the weight derivative, 2 - 1/s with it; b = -fl32(s r)), the sums are the 8x8 Gram matrix C = sum c c^T
//       H_world = C[0:6,0:6],  g_world = C[0:6,6],  sum b^2 = C[6,6],  sum r^2 = C[7,7],
// and the constant congruence with blkdiag(R, R) is applied once, in the last block.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "k2_solve.cuh"

namespace k1 {

using k2::kAcc;

constexpr int kTRow = 36;                // padded row stride (doubles) of a warp's DMMA transpose buffer

struct Pose {            // R row-major, t
    double R[9];
    double t[3];
};

// fast full-precision reciprocal for s in (0.1, 1]: MUFU.RCP64H seed + 2 Newton steps (error < 1 ulp)
__device__ __forceinline__ double rcp_newton(double s) {
    double y;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(s));
    double e = fma(-s, y, 1.0);
    y = fma(y, e, y);
    e = fma(-s, y, 1.0);
    return fma(y, e, y);
}

// (double)(float)x without the two F2F conversions: round-to-nearest-even to 24 significant bits directly on
// the FP64 bit pattern (5 integer instructions).  Identical to the float round trip for x = 0 and for
// 2^-126 <= |x| < 2^128, i.e. whenever the float32 result is a normal number or zero.
__device__ __forceinline__ double round_f32(double x) {
    unsigned long long b = (unsigned long long)__double_as_longlong(x);
    const unsigned lsb = ((unsigned)b >> 29) & 1u;
    b += 0x0FFFFFFFull + lsb;                      // 64-bit add: the carry runs into the exponent when needed
    b &= 0xFFFFFFFFE0000000ull;
    return __longlong_as_double((long long)b);
}

// Per-slot front: residual, weight, gate, float32 round trips, Jacobian row in the world frame.
// Output c[8] = [k (Rp x u'), k u', b, r], all zeros for an invalid slot (no plane or gated out).  A non-finite point
// gives a NaN or infinite r (the point arrives through an exact conversion), so it fails the gate as in the reference;
// the row is built from Rp only when the slot is valid, since 0 x NaN would otherwise put NaN into every sum.
// slope / gate: dcreg_icp_params::weight_slope / weight_gate (0.9 / 0.1 in the reference, icp_test_runner.cpp:1776, 1785)
template <bool kUseWd>
__device__ __forceinline__ void slot_front(const Pose& P, double px, double py, double pz, double nx, double ny,
                                           double nz, double d, bool has, double (&c)[8], int& neff,
                                           double slope = 0.9, double gate = 0.1) {
    const double wx = fma(P.R[2], pz, fma(P.R[1], py, P.R[0] * px));     // Rp (no translation)
    const double wy = fma(P.R[5], pz, fma(P.R[4], py, P.R[3] * px));
    const double wz = fma(P.R[8], pz, fma(P.R[7], py, P.R[6] * px));
    const double qx = round_f32(wx + P.t[0]);                     // utils.hpp:630-636 (float32 store)
    const double qy = round_f32(wy + P.t[1]);
    const double qz = round_f32(wz + P.t[2]);
    const double rr = fma(nx, qx, fma(ny, qy, fma(nz, qz, d)));   // icp_test_runner.cpp:1774
    const double ss = 1.0 - slope * fabs(rr);                     // :1776 (max(0, .) is implied by the gate >= 0)
    const bool valid = has && (ss > gate);                        // :1785
    const double s = valid ? ss : 0.0;
    const double r = valid ? rr : 0.0;
    double ux = round_f32(s * nx);                                // coeff.x/y/z (:1787-1789)
    double uy = round_f32(s * ny);
    double uz = round_f32(s * nz);
    c[6] = -round_f32(s * r);                                     // -coeff.intensity (:1790, 1906)
    c[7] = r;
    if (kUseWd) {                                                 // :1780-1783, 1898: row scale w/s = 2 - 1/s on 0 < s < 1
        const double sw = valid ? ss : 1.0;                       // (s == 1 gives k = 1: no derivative, as in the reference)
        const double k = 2.0 - rcp_newton(sw);
        ux *= k; uy *= k; uz *= k;
    }
    const double vx = valid ? wx : 0.0, vy = valid ? wy : 0.0, vz = valid ? wz : 0.0;
    c[0] = vy * uz - vz * uy;                                     // Rp x (k u')
    c[1] = vz * ux - vx * uz;
    c[2] = vx * uy - vy * ux;
    c[3] = ux; c[4] = uy; c[5] = uz;
    neff += valid ? 1 : 0;
}

// ---- Gram accumulation with the FP64 tensor-core instruction (used by the ICP iteration kernel) -----------------
// One mma.sync.m8n8k4 (SASS: DMMA) adds c c^T for 4 slots: A = c (8 components x 4 slots), B = A^T; each lane owns
// only two entries of C (flat index 2*lane, 2*lane + 1), so no per-thread block of 29 accumulators is needed next to
// the register-hungry k-NN / plane-fit code.  The per-slot components are transposed into the fragment layout
// through a 2.3 KB per-warp shared buffer (8 STS.64 + 8 LDS.64 per 32 slots, conflict-free with the padded stride).
// (The streaming kernel uses plain DFMA chains instead: there the FP64 issue slots are the bottleneck and
// 29 DFMA take fewer FP64 issue slots than 8 DMMA.)  All 32 lanes must call this convergently.
__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                 : "+d"(c0), "+d"(c1)
                 : "d"(a), "d"(b));
}

__device__ __forceinline__ void gram_accumulate_dmma(double* tb, int lane, const double (&c)[8], double& c0, double& c1,
                                                     double& e0, double& e1) {
    const int rd_off = (lane >> 2) * kTRow + (lane & 3);   // fragment element: component lane/4 of slot lane%4
#pragma unroll
    for (int j = 0; j < 8; ++j) tb[j * kTRow + lane] = c[j];
    __syncwarp();
#pragma unroll
    for (int g = 0; g < 8; g += 2) {
        const double f0 = tb[rd_off + 4 * g], f1 = tb[rd_off + 4 * g + 4];
        dmma884(c0, c1, f0, f0);
        dmma884(e0, e1, f1, f1);                            // two accumulator pairs: halves the dependent chain
    }
    __syncwarp();
}

}  // namespace k1
