// k2_fast.cuh - the 3x3 pieces of the solve step, written for ONE dependent chain per lane.
//
// Where the time of the solve step goes (~4.4 k warp instructions executed exactly once by one warp in every ICP
// iteration): two 3x3 Jacobi eigen-decompositions (6 sweeps x 3 rotations, each with two
// IEEE divisions and a square root = ~120 dependent instructions), two 3x3 inverses through a generic full-pivot LU on
// local-memory arrays, and a PCG with two more divisions and a square root per iteration.  Nothing here is throughput:
// it is one long dependent chain, so the only way to make it faster is to make it SHORTER.  This file does that
// without changing what is computed (paper Eq. 18-21, 43-46; icp_test_runner.cpp:2418-2469):
//   * reciprocal / reciprocal square root by the hardware seed (MUFU.RCP64H / MUFU.RSQ64H) + Newton steps - <= 1-2 ulp,
//     ~1/3 of the instructions of an IEEE-rounded division; a Jacobi rotation needs one of each plus one more rsqrt;
//   * the Jacobi iteration starts from the eigenvectors of the PREVIOUS ICP iteration (kept in the loop state): the
//     Schur blocks change little from one iteration to the next, so A' = V^T S V is already nearly diagonal and 1-3
//     sweeps reach the same convergence test the cold start needs 5-6 sweeps for;
//   * the 3x3 inverse comes from a symmetric-pivoted L D L^T kept in registers (for the positive semi-definite Gram
//     blocks H_RR / H_tt full pivoting picks diagonal pivots, so its pivots ARE Eigen FullPivLU's and the
//     FullPivLU::isInvertible decision is reproduced from them), three reciprocals, no local-memory arrays.
// Results differ from the reference decomposition (small_la.cuh, used by the seams and for every log record) by
// rounding only: eigenvalues to ~1e-15 relative, far inside the 1e-8 contract (tools/test_k2_fast.cu, host-compiled,
// checks this on random / ill-conditioned / rank-deficient blocks; tests/test_gpu_configs.py checks the trajectories).
#pragma once
#include <cuda_runtime.h>
#include <math.h>

#ifndef K2F_HD
#define K2F_HD __host__ __device__ __forceinline__
#endif

namespace k2f {

// 1 / x for normal, finite x (|x| in ~[1e-300, 1e300])
K2F_HD double fast_rcp(double x) {
#ifdef __CUDA_ARCH__
    double y;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
    double e = fma(-x, y, 1.0);
    y = fma(y, e, y);
    e = fma(-x, y, 1.0);
    return fma(y, e, y);
#else
    return 1.0 / x;
#endif
}

// 1 / sqrt(x) for normal, finite x > 0
K2F_HD double fast_rsqrt(double x) {
#ifdef __CUDA_ARCH__
    double y;
    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
    // two Newton steps: y <- y (1.5 - 0.5 x y^2)
    const double hx = 0.5 * x;
    double t = fma(-hx * y, y, 0.5);      // 0.5 - 0.5 x y^2
    y = fma(y, t, y);
    t = fma(-hx * y, y, 0.5);
    return fma(y, t, y);
#else
    return 1.0 / sqrt(x);
#endif
}

// a / b with one residual correction (last-bit accurate in all but rare cases)
K2F_HD double fast_div(double a, double b) {
    const double y = fast_rcp(b);
    const double q = a * y;
    return fma(fma(-b, q, a), y, q);
}

// ---- 3x3 symmetric positive semi-definite inverse ---------------------------------------------------------------
// A row-major (read as a symmetric matrix: A[i][j] for i <= j).  Symmetric-pivoted L D L^T: for a PSD Gram block
// full pivoting picks diagonal pivots, so d1, d2, d3 ARE Eigen FullPivLU's pivots and the return value is
// FullPivLU::isInvertible's decision (a pivot is zero when |p| <= eps * 3 * |largest pivot|, as
// dla::fullpiv_inverse<3>).  The inverse is assembled from the factors, A^-1 = sum_k u_k u_k^T / d_k with u_k the rows
// of L^-1 (as backward stable as the pivoted LU; an adjugate / determinant formula is NOT: it loses cond(A) more
// digits, and the translation block of a corridor has cond ~1e6).  inv may live in shared memory (indexed dynamically).
K2F_HD bool spd_inverse3(const double* A, double* inv) {
    const double a00 = A[0], a01 = A[1], a02 = A[2], a11 = A[4], a12 = A[5], a22 = A[8];
    double p1 = a00; int i1 = 0;
    if (a11 > p1) { p1 = a11; i1 = 1; }
    if (a22 > p1) { p1 = a22; i1 = 2; }
    // (j, k) = the other two indices, ascending; c_j, c_k = their couplings to the pivot, d_j, d_k their diagonals, o = a_jk
    const int j = i1 == 0 ? 1 : 0, k = i1 == 2 ? 1 : 2;
    const double dj = i1 == 0 ? a11 : a00, dk = i1 == 2 ? a11 : a22;
    const double cj = i1 == 2 ? a02 : a01;
    const double ck = i1 == 0 ? a02 : a12;
    const double o = i1 == 0 ? a12 : (i1 == 1 ? a02 : a01);
    if (!(p1 > 0.0)) return false;                                // also NaN
    const double r1 = fast_rcp(p1);
    const double fj = cj * r1, fk = ck * r1;
    const double sj = dj - fj * cj, sk = dk - fk * ck, so = o - fj * ck;
    const bool jfirst = !(sk > sj);                               // first maximum in scan order
    const double p2 = jfirst ? sj : sk, rest = jfirst ? sk : sj;
    if (!(fabs(p2) > 0.0)) return false;
    const double r2 = fast_rcp(p2);
    const double l21 = so * r2;
    const double p3 = rest - l21 * so;
    const double mx = fmax(fabs(p1), fmax(fabs(p2), fabs(p3)));
    const double thr = 2.220446049250313e-16 * 3.0 * mx;
    if (!(fabs(p1) > thr && fabs(p2) > thr && fabs(p3) > thr)) return false;
    const double r3 = fast_rcp(p3);
    // permuted order (pi0, pi1, pi2) = (i1, first of the complement, the other)
    const int q1 = jfirst ? j : k, q2 = jfirst ? k : j;
    const double l10 = jfirst ? fj : fk, l20 = jfirst ? fk : fj;
    // rows of L^-1: u0 = (1, 0, 0), u1 = (-l10, 1, 0), u2 = (l10 l21 - l20, -l21, 1)
    const double u20 = l10 * l21 - l20;
    const double m00 = r1 + l10 * l10 * r2 + u20 * u20 * r3;
    const double m01 = -l10 * r2 - u20 * l21 * r3;
    const double m02 = u20 * r3;
    const double m11 = r2 + l21 * l21 * r3;
    const double m12 = -l21 * r3;
    const double m22 = r3;
    inv[i1 * 3 + i1] = m00;
    inv[i1 * 3 + q1] = m01; inv[q1 * 3 + i1] = m01;
    inv[i1 * 3 + q2] = m02; inv[q2 * 3 + i1] = m02;
    inv[q1 * 3 + q1] = m11;
    inv[q1 * 3 + q2] = m12; inv[q2 * 3 + q1] = m12;
    inv[q2 * 3 + q2] = m22;
    return true;
}

// ---- 3x3 symmetric eigen-decomposition, cyclic Jacobi with a warm start --------------------------------------------
// S row-major symmetric.  Vw: orthonormal starting basis in columns (the previous iteration's eigenvectors), or
// nullptr for a cold start.  On return w ascending, V eigenvectors in columns (same conventions as dla::jacobi_eigh3).
// Same convergence test as dla::jacobi_eigh3 (off^2 <= 1e-34 diag^2).  Returns the number of sweeps used.
K2F_HD int jacobi_eigh3_warm(const double* S, const double* Vw, double* w, double* V) {
    double a[3][3], v[3][3];
    if (Vw) {
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) v[i][j] = Vw[i * 3 + j];
        double t[3][3];                                            // T = S V
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) t[i][j] = S[i * 3 + 0] * v[0][j] + S[i * 3 + 1] * v[1][j] + S[i * 3 + 2] * v[2][j];
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = i; j < 3; ++j) {                          // A' = V^T T, upper triangle mirrored
                const double s = v[0][i] * t[0][j] + v[1][i] * t[1][j] + v[2][i] * t[2][j];
                a[i][j] = s; a[j][i] = s;
            }
    } else {
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) { a[i][j] = S[i * 3 + j]; v[i][j] = (i == j) ? 1.0 : 0.0; }
    }
    int sweeps = 0;
#pragma unroll 1
    for (int sweep = 0; sweep < 40; ++sweep) {
        const double off = a[0][1] * a[0][1] + a[0][2] * a[0][2] + a[1][2] * a[1][2];
        const double diag = a[0][0] * a[0][0] + a[1][1] * a[1][1] + a[2][2] * a[2][2];
        if (off <= 1e-34 * diag || off == 0.0) break;
        ++sweeps;
#pragma unroll
        for (int p = 0; p < 2; ++p) {
#pragma unroll
            for (int q = p + 1; q < 3; ++q) {
                const double apq = a[p][q];
                if (fabs(apq) < 1e-300) { a[p][q] = a[q][p] = 0.0; continue; }
                const double app = a[p][p], aqq = a[q][q];
                // t = sgn(theta) / (|theta| + sqrt(theta^2 + 1)), theta = d / h: t = +-|h| / (|d| + sqrt(d^2 + h^2))
                const double d = aqq - app, h = 2.0 * apq;
                const double n2 = d * d + h * h;
                const double den = fabs(d) + n2 * fast_rsqrt(n2);
                const double tt = copysign(fabs(h), d * h >= 0.0 ? 1.0 : -1.0) * fast_rcp(den);
                const double c = fast_rsqrt(tt * tt + 1.0), sn = tt * c;
                a[p][p] = app - tt * apq;
                a[q][q] = aqq + tt * apq;
                a[p][q] = a[q][p] = 0.0;
                const int k = 3 - p - q;                           // the one remaining index
                const double akp = a[k][p], akq = a[k][q];
                const double nkp = c * akp - sn * akq, nkq = sn * akp + c * akq;
                a[k][p] = a[p][k] = nkp;
                a[k][q] = a[q][k] = nkq;
#pragma unroll
                for (int r = 0; r < 3; ++r) {
                    const double vrp = v[r][p], vrq = v[r][q];
                    v[r][p] = c * vrp - sn * vrq;
                    v[r][q] = sn * vrp + c * vrq;
                }
            }
        }
    }
    double l0 = a[0][0], l1 = a[1][1], l2 = a[2][2];
#define K2F_SWAP3(x, y, cx, cy)                                               \
    if (y < x) {                                                              \
        const double t_ = x; x = y; y = t_;                                   \
        _Pragma("unroll") for (int r = 0; r < 3; ++r) { const double u_ = v[r][cx]; v[r][cx] = v[r][cy]; v[r][cy] = u_; } \
    }
    K2F_SWAP3(l0, l1, 0, 1)
    K2F_SWAP3(l1, l2, 1, 2)
    K2F_SWAP3(l0, l1, 0, 1)
#undef K2F_SWAP3
    w[0] = l0; w[1] = l1; w[2] = l2;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) V[i * 3 + j] = v[i][j];
    return sweeps;
}

}  // namespace k2f
