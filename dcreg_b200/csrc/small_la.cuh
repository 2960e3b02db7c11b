// small_la.cuh - fixed-size FP64 dense linear algebra for the device side of the solve kernel.
//
// The reference leans on Eigen 3.3.7 for these (SelfAdjointEigenSolver, JacobiSVD,
// colPivHouseholderQr, FullPivLU; call sites dcreg.hpp:62-83,182,190,197,201,224 and
// icp_test_runner.cpp:1747,2016-2028,2422-2449).  Eigen is not available here, and nothing in it
// runs on a GPU anyway; these are independent implementations of the same mathematical
// operations, written for registers / local arrays of one CUDA thread (or one lane group).
#pragma once
#include <cuda_runtime.h>
#include <math.h>

namespace dla {

#define DLA_FN __device__ __forceinline__

// ---------------------------------------------------------------------------------------------
// Symmetric eigen-decomposition by cyclic Jacobi rotations.  A (row-major N*N, symmetric) is
// destroyed; on return w[] holds the eigenvalues in ASCENDING order and V (row-major) the
// matching eigenvectors in its COLUMNS (same convention as Eigen's SelfAdjointEigenSolver).
// Jacobi is used instead of a closed form because the 3x3 Schur blocks reach condition numbers
// of 1e3..1e6 and the contract is 1e-8 relative on every eigenvalue (SURVEY.md §7 hard parts).
// ---------------------------------------------------------------------------------------------
template <int N>
__device__ __noinline__ void jacobi_eigh(double* A, double* w, double* V) {
#pragma unroll
    for (int i = 0; i < N; ++i)
#pragma unroll
        for (int j = 0; j < N; ++j) V[i * N + j] = (i == j) ? 1.0 : 0.0;

    for (int sweep = 0; sweep < 40; ++sweep) {
        double off = 0.0, diag = 0.0;
#pragma unroll
        for (int i = 0; i < N; ++i) {
            diag += A[i * N + i] * A[i * N + i];
#pragma unroll
            for (int j = i + 1; j < N; ++j) off += A[i * N + j] * A[i * N + j];
        }
        if (off <= 1e-34 * diag || off == 0.0) break;
        for (int p = 0; p < N - 1; ++p) {
            for (int q = p + 1; q < N; ++q) {
                const double apq = A[p * N + q];
                if (apq == 0.0) continue;
                const double app = A[p * N + p], aqq = A[q * N + q];
                // skip rotations that cannot change the diagonal any more
                if (fabs(apq) < 1e-300) { A[p * N + q] = A[q * N + p] = 0.0; continue; }
                const double theta = (aqq - app) / (2.0 * apq);
                const double tt = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(tt * tt + 1.0), s = tt * c;
                const double tau = s / (1.0 + c);
                A[p * N + p] = app - tt * apq;
                A[q * N + q] = aqq + tt * apq;
                A[p * N + q] = A[q * N + p] = 0.0;
#pragma unroll
                for (int k = 0; k < N; ++k) {
                    if (k != p && k != q) {
                        const double akp = A[k * N + p], akq = A[k * N + q];
                        const double nkp = akp - s * (akq + tau * akp);
                        const double nkq = akq + s * (akp - tau * akq);
                        A[k * N + p] = A[p * N + k] = nkp;
                        A[k * N + q] = A[q * N + k] = nkq;
                    }
                }
#pragma unroll
                for (int k = 0; k < N; ++k) {
                    const double vkp = V[k * N + p], vkq = V[k * N + q];
                    V[k * N + p] = vkp - s * (vkq + tau * vkp);
                    V[k * N + q] = vkq + s * (vkp - tau * vkq);
                }
            }
        }
    }
#pragma unroll
    for (int i = 0; i < N; ++i) w[i] = A[i * N + i];
    // selection sort, ascending, permuting columns of V
    for (int i = 0; i < N - 1; ++i) {
        int m = i;
        for (int j = i + 1; j < N; ++j)
            if (w[j] < w[m]) m = j;
        if (m != i) {
            const double tw = w[i]; w[i] = w[m]; w[m] = tw;
            for (int k = 0; k < N; ++k) {
                const double tv = V[k * N + i]; V[k * N + i] = V[k * N + m]; V[k * N + m] = tv;
            }
        }
    }
}

// 3x3 specialisation kept entirely in registers (all indices static after unrolling): this one sits on the
// critical path of every ICP iteration (two Schur blocks), the generic version above spills to local memory.
__device__ __noinline__ void jacobi_eigh3(const double* Ain, double* w, double* V) {
    double a[3][3], v[3][3];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) { a[i][j] = Ain[i * 3 + j]; v[i][j] = (i == j) ? 1.0 : 0.0; }
    for (int sweep = 0; sweep < 40; ++sweep) {
        const double off = a[0][1] * a[0][1] + a[0][2] * a[0][2] + a[1][2] * a[1][2];
        const double diag = a[0][0] * a[0][0] + a[1][1] * a[1][1] + a[2][2] * a[2][2];
        if (off <= 1e-34 * diag || off == 0.0) break;
#pragma unroll
        for (int p = 0; p < 2; ++p) {
#pragma unroll
            for (int q = p + 1; q < 3; ++q) {
                const double apq = a[p][q];
                if (fabs(apq) < 1e-300) { a[p][q] = a[q][p] = 0.0; continue; }
                const double app = a[p][p], aqq = a[q][q];
                // t = sgn(theta) / (|theta| + sqrt(theta^2 + 1)) with theta = d / h, written without forming theta:
                // one division and one square root instead of two divisions and a square root
                const double d = aqq - app, h = 2.0 * apq;
                const double tt = copysign(fabs(h), d * h >= 0.0 ? 1.0 : -1.0) / (fabs(d) + sqrt(d * d + h * h));
                const double c = rsqrt(tt * tt + 1.0), sn = tt * c;
                const double tau = sn / (1.0 + c);
                a[p][p] = app - tt * apq;
                a[q][q] = aqq + tt * apq;
                a[p][q] = a[q][p] = 0.0;
                const int k = 3 - p - q;                    // the one remaining index
                const double akp = a[k][p], akq = a[k][q];
                a[k][p] = a[p][k] = akp - sn * (akq + tau * akp);
                a[k][q] = a[q][k] = akq + sn * (akp - tau * akq);
#pragma unroll
                for (int r = 0; r < 3; ++r) {
                    const double vrp = v[r][p], vrq = v[r][q];
                    v[r][p] = vrp - sn * (vrq + tau * vrp);
                    v[r][q] = vrq + sn * (vrp - tau * vrq);
                }
            }
        }
    }
    double l0 = a[0][0], l1 = a[1][1], l2 = a[2][2];
    // sort ascending with column swaps (3-element network)
#define DLA_SWAP3(x, y, cx, cy)                                              \
    if (y < x) {                                                              \
        const double t_ = x; x = y; y = t_;                                   \
        _Pragma("unroll") for (int r = 0; r < 3; ++r) { const double u_ = v[r][cx]; v[r][cx] = v[r][cy]; v[r][cy] = u_; } \
    }
    DLA_SWAP3(l0, l1, 0, 1)
    DLA_SWAP3(l1, l2, 1, 2)
    DLA_SWAP3(l0, l1, 0, 1)
#undef DLA_SWAP3
    w[0] = l0; w[1] = l1; w[2] = l2;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) V[i * 3 + j] = v[i][j];
}

// ---------------------------------------------------------------------------------------------
// Least-squares / linear solve by Householder QR with column pivoting, M x N (M >= N), one rhs.
// Same structure as a rank-revealing pivoted QR solve: columns whose remaining norm falls below
// (eps * max column norm)^2 / M * (M - k) are treated as exactly dependent and their solution
// component is set to zero (this is what makes an all-zero coordinate column - e.g. the z = 0
// floor of the cylinder scene - give a zero normal component instead of NaN).
// A is row-major M*N and is destroyed; b (M) is destroyed; x (N) receives the solution.
// Replaces matA0.colPivHouseholderQr().solve(matB0) (icp_test_runner.cpp:1747) and
// H.colPivHouseholderQr().solve(g) (dcreg.hpp:182,190,197).
// ---------------------------------------------------------------------------------------------
template <int M, int N>
__host__ __device__ __noinline__ void colpiv_qr_solve(double* A, double* b, double* x) {
    const double eps = 2.220446049250313e-16;
    double normU[N], normD[N];
    int perm[N];
    double maxn = 0.0;
#pragma unroll
    for (int j = 0; j < N; ++j) {
        double s = 0.0;
#pragma unroll
        for (int i = 0; i < M; ++i) s += A[i * N + j] * A[i * N + j];
        normU[j] = normD[j] = sqrt(s);
        perm[j] = j;
        if (normU[j] > maxn) maxn = normU[j];
    }
    const double thr_helper = (maxn * eps) * (maxn * eps) / (double)M;
    const double downdate_thr = 1.4901161193847656e-08;  // sqrt(eps)
    int nz = N;
    for (int k = 0; k < N; ++k) {
        int big = k;
        double bign = normU[k];
        for (int j = k + 1; j < N; ++j)
            if (normU[j] > bign) { bign = normU[j]; big = j; }
        if (nz == N && bign * bign < thr_helper * (double)(M - k)) nz = k;
        if (big != k) {
            for (int i = 0; i < M; ++i) {
                const double tmp = A[i * N + k]; A[i * N + k] = A[i * N + big]; A[i * N + big] = tmp;
            }
            double tn = normU[k]; normU[k] = normU[big]; normU[big] = tn;
            tn = normD[k]; normD[k] = normD[big]; normD[big] = tn;
            const int tp = perm[k]; perm[k] = perm[big]; perm[big] = tp;
        }
        // Householder reflector for column k, rows k..M-1:  H = I - tau v v^T, v = (1, ess)
        double tail = 0.0;
        for (int i = k + 1; i < M; ++i) tail += A[i * N + k] * A[i * N + k];
        const double c0 = A[k * N + k];
        double tau, beta;
        if (tail <= 2.2250738585072014e-308) {
            tau = 0.0; beta = c0;
            for (int i = k + 1; i < M; ++i) A[i * N + k] = 0.0;
        } else {
            beta = sqrt(c0 * c0 + tail);
            if (c0 >= 0.0) beta = -beta;
            const double inv = 1.0 / (c0 - beta);
            for (int i = k + 1; i < M; ++i) A[i * N + k] *= inv;
            tau = (beta - c0) / beta;
        }
        A[k * N + k] = beta;
        // apply to the remaining columns and to b
        for (int j = k + 1; j < N; ++j) {
            double tmp = A[k * N + j];
            for (int i = k + 1; i < M; ++i) tmp += A[i * N + k] * A[i * N + j];
            A[k * N + j] -= tau * tmp;
            for (int i = k + 1; i < M; ++i) A[i * N + j] -= tau * A[i * N + k] * tmp;
        }
        if (k < nz) {
            double tmp = b[k];
            for (int i = k + 1; i < M; ++i) tmp += A[i * N + k] * b[i];
            b[k] -= tau * tmp;
            for (int i = k + 1; i < M; ++i) b[i] -= tau * A[i * N + k] * tmp;
        }
        // norm down-dating (LAPACK working note 176 style)
        for (int j = k + 1; j < N; ++j) {
            if (normU[j] != 0.0) {
                double t = fabs(A[k * N + j]) / normU[j];
                t = (1.0 + t) * (1.0 - t);
                if (t < 0.0) t = 0.0;
                const double r = normU[j] / normD[j];
                const double t2 = t * r * r;
                if (t2 <= downdate_thr) {
                    double s = 0.0;
                    for (int i = k + 1; i < M; ++i) s += A[i * N + j] * A[i * N + j];
                    normD[j] = normU[j] = sqrt(s);
                } else {
                    normU[j] *= sqrt(t);
                }
            }
        }
    }
    // back substitution on the leading nz x nz triangle
    double c[N];
#pragma unroll
    for (int i = 0; i < N; ++i) c[i] = 0.0;
    for (int i = nz - 1; i >= 0; --i) {
        double s = b[i];
        for (int j = i + 1; j < nz; ++j) s -= A[i * N + j] * c[j];
        c[i] = s / A[i * N + i];
    }
#pragma unroll
    for (int i = 0; i < N; ++i) x[i] = 0.0;
    for (int i = 0; i < nz; ++i) x[perm[i]] = c[i];
}

// Plain IEEE `/` and `sqrt`: the arithmetic of colpiv_qr_solve_reg unless the caller passes another with the same
// members (the loop's plane fit passes correctly rounded primitives with a deferred range test, corr.cuh).  rcp and
// div_by split a division whose divisor is shared: div_by(a, b, rcp(b)) is a / b.
struct PlainArith {
    __host__ __device__ __forceinline__ double div(double a, double b) const { return a / b; }
    __host__ __device__ __forceinline__ double rcp(double) const { return 0.0; }
    __host__ __device__ __forceinline__ double div_by(double a, double b, double) const { return a / b; }
    __host__ __device__ __forceinline__ double sqrt(double a) const { return ::sqrt(a); }
};

// Same algorithm, same operations in the same order (bit-identical results, tools/test_qr_reg.cu), but every array
// index is a compile-time constant after unrolling: the pivot column is brought to position k with conditional
// swaps against each later column and the rank cut `nz` becomes a predicate, so A, b and the norms stay in registers
// instead of local memory.  Used for the 5x3 plane fit, which runs once per source slot.  Every division and square
// root goes through `ar`; with PlainArith they are the `/` and `sqrt` of colpiv_qr_solve.
template <int M, int N, class Ar = PlainArith>
__host__ __device__ __forceinline__ void colpiv_qr_solve_reg(double (&A)[M][N], double (&b)[M], double (&x)[N], Ar ar = Ar()) {
    const double eps = 2.220446049250313e-16;
    double normU[N], normD[N];
    int perm[N];
    double maxn = 0.0;
#pragma unroll
    for (int j = 0; j < N; ++j) {
        double s = 0.0;
#pragma unroll
        for (int i = 0; i < M; ++i) s += A[i][j] * A[i][j];
        normU[j] = normD[j] = ar.sqrt(s);
        perm[j] = j;
        if (normU[j] > maxn) maxn = normU[j];
    }
    const double thr_helper = (maxn * eps) * (maxn * eps) / (double)M;
    const double downdate_thr = 1.4901161193847656e-08;  // sqrt(eps)
    int nz = N;
#pragma unroll
    for (int k = 0; k < N; ++k) {
        int big = k;
        double bign = normU[k];
#pragma unroll
        for (int j = k + 1; j < N; ++j)
            if (normU[j] > bign) { bign = normU[j]; big = j; }
        if (nz == N && bign * bign < thr_helper * (double)(M - k)) nz = k;
#pragma unroll
        for (int j = k + 1; j < N; ++j) {
            if (big == j) {
#pragma unroll
                for (int i = 0; i < M; ++i) { const double tmp = A[i][k]; A[i][k] = A[i][j]; A[i][j] = tmp; }
                double tn = normU[k]; normU[k] = normU[j]; normU[j] = tn;
                tn = normD[k]; normD[k] = normD[j]; normD[j] = tn;
                const int tp = perm[k]; perm[k] = perm[j]; perm[j] = tp;
            }
        }
        // Householder reflector for column k, rows k..M-1:  H = I - tau v v^T, v = (1, ess)
        double tail = 0.0;
#pragma unroll
        for (int i = k + 1; i < M; ++i) tail += A[i][k] * A[i][k];
        const double c0 = A[k][k];
        double tau, beta;
        if (tail <= 2.2250738585072014e-308) {
            tau = 0.0; beta = c0;
#pragma unroll
            for (int i = k + 1; i < M; ++i) A[i][k] = 0.0;
        } else {
            beta = ar.sqrt(c0 * c0 + tail);
            if (c0 >= 0.0) beta = -beta;
            const double inv = ar.div(1.0, c0 - beta);
#pragma unroll
            for (int i = k + 1; i < M; ++i) A[i][k] *= inv;
            tau = ar.div(beta - c0, beta);
        }
        A[k][k] = beta;
        // apply to the remaining columns and to b
#pragma unroll
        for (int j = k + 1; j < N; ++j) {
            double tmp = A[k][j];
#pragma unroll
            for (int i = k + 1; i < M; ++i) tmp += A[i][k] * A[i][j];
            A[k][j] -= tau * tmp;
#pragma unroll
            for (int i = k + 1; i < M; ++i) A[i][j] -= tau * A[i][k] * tmp;
        }
        if (k < nz) {
            double tmp = b[k];
#pragma unroll
            for (int i = k + 1; i < M; ++i) tmp += A[i][k] * b[i];
            b[k] -= tau * tmp;
#pragma unroll
            for (int i = k + 1; i < M; ++i) b[i] -= tau * A[i][k] * tmp;
        }
        // norm down-dating (LAPACK working note 176 style)
#pragma unroll
        for (int j = k + 1; j < N; ++j) {
            if (normU[j] != 0.0) {
                double t = ar.div(fabs(A[k][j]), normU[j]);
                t = (1.0 + t) * (1.0 - t);
                if (t < 0.0) t = 0.0;
                const double r = ar.div(normU[j], normD[j]);
                const double t2 = t * r * r;
                if (t2 <= downdate_thr) {
                    double s = 0.0;
#pragma unroll
                    for (int i = k + 1; i < M; ++i) s += A[i][j] * A[i][j];
                    normD[j] = normU[j] = ar.sqrt(s);
                } else {
                    normU[j] *= ar.sqrt(t);
                }
            }
        }
    }
    // back substitution on the leading nz x nz triangle
    double c[N];
#pragma unroll
    for (int i = 0; i < N; ++i) c[i] = 0.0;
#pragma unroll
    for (int i = N - 1; i >= 0; --i) {
        if (i < nz) {
            double s = b[i];
#pragma unroll
            for (int j = i + 1; j < N; ++j)
                if (j < nz) s -= A[i][j] * c[j];
            c[i] = ar.div(s, A[i][i]);
        }
    }
#pragma unroll
    for (int i = 0; i < N; ++i) x[i] = 0.0;
#pragma unroll
    for (int i = 0; i < N; ++i)
        if (i < nz) {
#pragma unroll
            for (int t = 0; t < N; ++t)
                if (perm[i] == t) x[t] = c[i];
        }
}

// ---------------------------------------------------------------------------------------------
// N x N inverse by LU with full pivoting.  Returns false when the matrix is numerically singular
// (a pivot below eps * N * |largest pivot|), mirroring FullPivLU::isInvertible as used by the
// released Schur block (icp_test_runner.cpp:2422-2423, 2442) and the covariance step (2016-2018).
// A row-major, destroyed; Ainv row-major.
// ---------------------------------------------------------------------------------------------
template <int N>
__device__ __noinline__ bool fullpiv_inverse(double* A, double* Ainv) {
    int prow[N], pcol[N];
    double maxpivot = 0.0;
    bool singular = false;
    for (int k = 0; k < N; ++k) {
        int br = k, bc = k;
        double bv = -1.0;
        for (int i = k; i < N; ++i)
            for (int j = k; j < N; ++j) {
                const double v = fabs(A[i * N + j]);
                if (v > bv) { bv = v; br = i; bc = j; }
            }
        prow[k] = br; pcol[k] = bc;
        if (bv > maxpivot) maxpivot = bv;
        if (bv == 0.0) { singular = true; for (int kk = k; kk < N; ++kk) { prow[kk] = kk; pcol[kk] = kk; } break; }
        if (br != k)
            for (int j = 0; j < N; ++j) { const double t = A[k * N + j]; A[k * N + j] = A[br * N + j]; A[br * N + j] = t; }
        if (bc != k)
            for (int i = 0; i < N; ++i) { const double t = A[i * N + k]; A[i * N + k] = A[i * N + bc]; A[i * N + bc] = t; }
        const double piv = A[k * N + k];
        for (int i = k + 1; i < N; ++i) {
            const double f = A[i * N + k] / piv;
            A[i * N + k] = f;
            for (int j = k + 1; j < N; ++j) A[i * N + j] -= f * A[k * N + j];
        }
    }
    if (singular) return false;
    const double thr = 2.220446049250313e-16 * (double)N * maxpivot;
    for (int k = 0; k < N; ++k)
        if (fabs(A[k * N + k]) <= thr) return false;
    // Solve P A Q = L U  =>  A^-1 = Q U^-1 L^-1 P.  Column by column (N reciprocals instead of N^2 divisions).
    double rd[N];
    for (int i = 0; i < N; ++i) rd[i] = 1.0 / A[i * N + i];
    for (int col = 0; col < N; ++col) {
        double y[N];
        // rhs = P e_col : apply the row swaps in order to the unit vector
        for (int i = 0; i < N; ++i) y[i] = (i == col) ? 1.0 : 0.0;
        for (int k = 0; k < N; ++k)
            if (prow[k] != k) { const double t = y[k]; y[k] = y[prow[k]]; y[prow[k]] = t; }
        for (int i = 0; i < N; ++i)
            for (int j = 0; j < i; ++j) y[i] -= A[i * N + j] * y[j];
        for (int i = N - 1; i >= 0; --i) {
            for (int j = i + 1; j < N; ++j) y[i] -= A[i * N + j] * y[j];
            y[i] *= rd[i];
        }
        // undo the column swaps (reverse order)
        for (int k = N - 1; k >= 0; --k)
            if (pcol[k] != k) { const double t = y[k]; y[k] = y[pcol[k]]; y[pcol[k]] = t; }
        for (int i = 0; i < N; ++i) Ainv[i * N + col] = y[i];
    }
    return true;
}

DLA_FN void mat3_mul(const double* A, const double* B, double* C) {
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            C[i * 3 + j] = A[i * 3 + 0] * B[0 * 3 + j] + A[i * 3 + 1] * B[1 * 3 + j] + A[i * 3 + 2] * B[2 * 3 + j];
}

DLA_FN void mat6_vec(const double* A, const double* x, double* y) {
#pragma unroll
    for (int i = 0; i < 6; ++i) {
        double s = 0.0;
#pragma unroll
        for (int j = 0; j < 6; ++j) s += A[i * 6 + j] * x[j];
        y[i] = s;
    }
}

}  // namespace dla
