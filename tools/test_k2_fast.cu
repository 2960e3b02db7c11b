// Check of dcreg_b200/csrc/k2_fast.cuh: the warm-started Jacobi and the L D L^T inverse with the FullPivLU
// invertibility decision, on random / ill-conditioned / rank-deficient 3x3 Gram blocks.
//   host build   (nvcc -O2, no GPU): the algorithms, with exact 1/x and 1/sqrt(x) in place of the MUFU seeds;
//   device build (-DK2F_DEVICE_TEST, nvcc -gencode arch=compute_90a,code=sm_90a --fmad=true, as the library): the same
//                generator and checks in a kernel, one chunk per thread, with the device arithmetic the solve step runs,
//                plus a sweep of fast_rcp / fast_div against __drcp_rn / __ddiv_rn over [1e-300, 1e300] (powers of
//                two, all-ones mantissas, the ends, log-uniform samples); fast_rsqrt's sample goes to argv[1] for an
//                mpmath comparison (tests/test_host_la.py).
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include "../dcreg_b200/csrc/k2_fast.cuh"

#ifdef K2F_DEVICE_TEST
#define HD __host__ __device__
#else
#define HD
#endif

struct Rng {
    unsigned long long s;
    HD double operator()() {
        s ^= s << 13; s ^= s >> 7; s ^= s << 17;
        return (double)(s >> 11) * (1.0 / 9007199254740992.0);
    }
};

// Gram block sum_k s_k n_k n_k^T with `rank` independent directions and a spread of scales
HD static void make_block(Rng& urand, int rank, double spread, double* A) {
    for (int e = 0; e < 9; ++e) A[e] = 0.0;
    double basis[3][3];
    for (int k = 0; k < 3; ++k) for (int i = 0; i < 3; ++i) basis[k][i] = urand() * 2.0 - 1.0;
    const int terms = rank == 3 ? 40 : rank;
    for (int t = 0; t < terms; ++t) {
        double n[3] = {0, 0, 0};
        if (rank == 3) {
            for (int k = 0; k < 3; ++k) { const double c = (urand() * 2.0 - 1.0) * pow(spread, -(double)k); for (int i = 0; i < 3; ++i) n[i] += c * basis[k][i]; }
        } else {
            for (int i = 0; i < 3; ++i) n[i] = basis[t][i];
        }
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) A[i * 3 + j] += n[i] * n[j];
    }
}

// reference: full-pivot LU decision exactly as dla::fullpiv_inverse<3> (small_la.cuh), host loops
// ratio: the smallest |pivot| over the largest (FullPivLU calls a block singular at <= 3 eps)
HD static bool ref_invertible(const double* Ain, double* ratio) {
    double A[9];
    for (int e = 0; e < 9; ++e) A[e] = Ain[e];
    double maxpivot = 0.0;
    for (int k = 0; k < 3; ++k) {
        int br = k, bc = k; double bv = -1.0;
        for (int i = k; i < 3; ++i) for (int j = k; j < 3; ++j) { const double v = fabs(A[i * 3 + j]); if (v > bv) { bv = v; br = i; bc = j; } }
        if (bv > maxpivot) maxpivot = bv;
        if (bv == 0.0) { *ratio = 0.0; return false; }
        if (br != k) for (int j = 0; j < 3; ++j) { const double t = A[k * 3 + j]; A[k * 3 + j] = A[br * 3 + j]; A[br * 3 + j] = t; }
        if (bc != k) for (int i = 0; i < 3; ++i) { const double t = A[i * 3 + k]; A[i * 3 + k] = A[i * 3 + bc]; A[i * 3 + bc] = t; }
        const double piv = A[k * 3 + k];
        for (int i = k + 1; i < 3; ++i) { const double f = A[i * 3 + k] / piv; A[i * 3 + k] = f; for (int j = k + 1; j < 3; ++j) A[i * 3 + j] -= f * A[k * 3 + j]; }
    }
    const double thr = 2.220446049250313e-16 * 3.0 * maxpivot;
    *ratio = fmin(fabs(A[0]), fmin(fabs(A[4]), fabs(A[8]))) / maxpivot;
    for (int k = 0; k < 3; ++k) if (fabs(A[k * 3 + k]) <= thr) return false;
    return true;
}

struct Stats {
    int bad, n_sys, n_sing, decisions_differ;
    double disagree_ratio;          // largest pivot ratio of a block whose decision differs from the plain LU's
    double worst_eig, worst_res, worst_orth, worst_inv, worst_warm;
    long long sweeps_cold, sweeps_warm;
};

HD static void run_chunk(unsigned long long seed, int count, Stats& S) {
    Rng urand{seed};
    int& bad = S.bad; int& n_sys = S.n_sys; int& n_sing = S.n_sing; int& decisions_differ = S.decisions_differ;
    double& worst_eig = S.worst_eig; double& worst_res = S.worst_res; double& worst_orth = S.worst_orth;
    double& worst_inv = S.worst_inv; double& worst_warm = S.worst_warm;
    long long& sweeps_cold = S.sweeps_cold; long long& sweeps_warm = S.sweeps_warm;
    for (int it = 0; it < count; ++it) {
        const int rank = (it % 10 == 0) ? 1 + (it / 10) % 2 : 3;
        const double spread = pow(10.0, urand() * 1.5);                  // eigenvalue ratios up to spread^4 = 1e6
        double A[9], w[3], V[9];
        make_block(urand, rank, spread, A);
        ++n_sys;
        const int sc = k2f::jacobi_eigh3_warm(A, nullptr, w, V);
        sweeps_cold += sc;
        const double scale = fabs(w[2]) > 0 ? fabs(w[2]) : 1.0;
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) {
            double r = 0, o = 0;
            for (int k = 0; k < 3; ++k) { r += A[i * 3 + k] * V[k * 3 + j]; o += V[k * 3 + i] * V[k * 3 + j]; }
            worst_res = fmax(worst_res, fabs(r - w[j] * V[i * 3 + j]) / scale);
            worst_orth = fmax(worst_orth, fabs(o - (i == j ? 1.0 : 0.0)));
        }
        if (!(w[0] <= w[1] && w[1] <= w[2])) ++bad;
        // perturb the block a little (the next ICP iteration) and restart warm from V
        double B[9], w2[3], V2[9], w3[3], V3[9], P[9];
        make_block(urand, 3, spread, P);
        for (int e = 0; e < 9; ++e) B[e] = A[e] + 1e-3 * P[e] * (A[0] + A[4] + A[8]) / (P[0] + P[4] + P[8] + 1e-300);
        const int sw = k2f::jacobi_eigh3_warm(B, V, w2, V2);
        k2f::jacobi_eigh3_warm(B, nullptr, w3, V3);
        sweeps_warm += sw;
        for (int k = 0; k < 3; ++k) worst_warm = fmax(worst_warm, fabs(w2[k] - w3[k]) / fmax(fabs(w3[2]), 1e-300));
        // relative error of every eigenvalue, in units of the condition number (the warm start forms V^T S V in floating point)
        if (rank == 3) for (int k = 0; k < 3; ++k) worst_eig = fmax(worst_eig, fabs(w2[k] - w3[k]) / fmax(fabs(w3[k]), 1e-300) / (w3[2] / fmax(w3[0], 1e-300)));
        // inverse + decision
        double inv[9];
        double ratio = 0.0;
        const bool ok = k2f::spd_inverse3(A, inv), ok_ref = ref_invertible(A, &ratio);
        if (ok != ok_ref) { ++decisions_differ; S.disagree_ratio = fmax(S.disagree_ratio, ratio); }
        if (!ok_ref) ++n_sing;
        if (ok && rank == 3) {
            const double cond = w[2] / fmax(w[0], 1e-300);
            for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) {
                double s = 0;
                for (int k = 0; k < 3; ++k) s += A[i * 3 + k] * inv[k * 3 + j];
                worst_inv = fmax(worst_inv, fabs(s - (i == j ? 1.0 : 0.0)) / cond);
            }
        }
    }
}

#ifdef K2F_DEVICE_TEST
constexpr int kChunks = 256;
__global__ void checks_kernel(Stats* out) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= kChunks) return;
    Stats S{};
    run_chunk(0x9E3779B97F4A7C15ull + 0x632BE59BD9B4E019ull * (unsigned long long)c, 200000 / kChunks, S);
    out[c] = S;
}

__device__ long long ulp_diff(double a, double b) {
    if (a == b) return 0;
    if (!isfinite(a) || !isfinite(b) || (a < 0) != (b < 0)) return 1LL << 62;
    const long long d = __double_as_longlong(a) - __double_as_longlong(b);
    return d < 0 ? -d : d;
}

// x_k over [1e-300, 1e300]: k < 1993: 2^(k - 996), then the all-ones mantissas just below those powers, the two ends, then
// log-uniform samples (both signs for the divisions)
constexpr int kPow = 1993, kSweep = 2 * kPow + 2 + (1 << 20);
__device__ double sweep_x(int k) {
    if (k < kPow) return ldexp(1.0, k - 996);
    if (k < 2 * kPow) return ldexp(2.0 - ldexp(1.0, -52), k - kPow - 997);   // 2^-996 (1 - 2^-53) .. 2^996 (1 - 2^-53)
    if (k == 2 * kPow) return 1e-300;
    if (k == 2 * kPow + 1) return 1e300;
    Rng r{0xD1B54A32D192ED03ull ^ (unsigned long long)k * 0x9E3779B97F4A7C15ull};
    r(); r();
    return pow(10.0, -300.0 + 600.0 * r());
}

__global__ void ulp_kernel(unsigned long long* worst, double* rsq) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= kSweep) return;
    const double x = sweep_x(k);
    atomicMax(&worst[0], (unsigned long long)ulp_diff(k2f::fast_rcp(x), __drcp_rn(x)));
    atomicMax(&worst[0], (unsigned long long)ulp_diff(k2f::fast_rcp(-x), __drcp_rn(-x)));
    // a / b with a, b and a / b in the domain: a = x, b from the mirrored index, kept when the quotient stays inside
    const double b = sweep_x(kSweep - 1 - k);
    const double q = __ddiv_rn(x, b);
    if (fabs(q) >= 1e-300 && fabs(q) <= 1e300) {
        atomicMax(&worst[1], (unsigned long long)ulp_diff(k2f::fast_div(x, b), q));
        atomicMax(&worst[1], (unsigned long long)ulp_diff(k2f::fast_div(-x, b), -q));
    }
    const double y = k2f::fast_rsqrt(x);
    if (k < 2 * kPow + 2 || (k & 63) == 0) {                  // every structured point and 1 / 64 of the samples
        const int j = k < 2 * kPow + 2 ? k : 2 * kPow + 2 + ((k - 2 * kPow - 2) >> 6);
        rsq[2 * j] = x; rsq[2 * j + 1] = y;
    }
}
constexpr int kRsq = 2 * kPow + 2 + ((kSweep - 2 * kPow - 2 + 63) >> 6);

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); return 2; } } while (0)
#endif

int main(int argc, char** argv) {
    Stats S{};
#ifdef K2F_DEVICE_TEST
    Stats* d_st; unsigned long long* d_worst; double* d_rsq;
    CK(cudaMalloc(&d_st, kChunks * sizeof(Stats)));
    CK(cudaMalloc(&d_worst, 2 * sizeof(unsigned long long)));
    CK(cudaMalloc(&d_rsq, 2 * (size_t)kRsq * sizeof(double)));
    CK(cudaMemset(d_worst, 0, 2 * sizeof(unsigned long long)));
    checks_kernel<<<kChunks / 32, 32>>>(d_st);
    ulp_kernel<<<(kSweep + 255) / 256, 256>>>(d_worst, d_rsq);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    Stats h[kChunks];
    unsigned long long worst_ulp[2];
    CK(cudaMemcpy(h, d_st, sizeof(h), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(worst_ulp, d_worst, sizeof(worst_ulp), cudaMemcpyDeviceToHost));
    double* rsq = (double*)malloc(2 * (size_t)kRsq * sizeof(double));
    CK(cudaMemcpy(rsq, d_rsq, 2 * (size_t)kRsq * sizeof(double), cudaMemcpyDeviceToHost));
    for (int c = 0; c < kChunks; ++c) {
        S.bad += h[c].bad; S.n_sys += h[c].n_sys; S.n_sing += h[c].n_sing; S.decisions_differ += h[c].decisions_differ;
        S.disagree_ratio = fmax(S.disagree_ratio, h[c].disagree_ratio);
        S.worst_eig = fmax(S.worst_eig, h[c].worst_eig); S.worst_res = fmax(S.worst_res, h[c].worst_res);
        S.worst_orth = fmax(S.worst_orth, h[c].worst_orth); S.worst_inv = fmax(S.worst_inv, h[c].worst_inv);
        S.worst_warm = fmax(S.worst_warm, h[c].worst_warm);
        S.sweeps_cold += h[c].sweeps_cold; S.sweeps_warm += h[c].sweeps_warm;
    }
    printf("device: fast_rcp max %llu ulp from __drcp_rn, fast_div max %llu ulp from __ddiv_rn over %d points\n",
           worst_ulp[0], worst_ulp[1], kSweep);
    if (argc > 1) {
        FILE* f = fopen(argv[1], "wb");
        if (!f) { printf("cannot write %s\n", argv[1]); return 2; }
        fwrite(rsq, sizeof(double), 2 * (size_t)kRsq, f);
        fclose(f);
    }
    free(rsq);
    cudaFree(d_st); cudaFree(d_worst); cudaFree(d_rsq);
    const bool ulp_ok = worst_ulp[0] <= 2 && worst_ulp[1] <= 2;        // k2_fast.cuh: <= 1-2 ulp
#else
    run_chunk(0x9E3779B97F4A7C15ull, 200000, S);
    const bool ulp_ok = true;
#endif
    printf("%d systems (%d singular), decisions differing from FullPivLU: %d (largest pivot ratio among them %.2f eps), "
           "order errors: %d\n", S.n_sys, S.n_sing, S.decisions_differ, S.disagree_ratio / 2.220446049250313e-16, S.bad);
    printf("residual %.2e orthogonality %.2e warm-vs-cold eigenvalue (abs/lmax) %.2e (rel/cond, full rank) %.2e inverse/cond %.2e\n",
           S.worst_res, S.worst_orth, S.worst_warm, S.worst_eig, S.worst_inv);
    printf("mean sweeps cold %.2f warm %.2f\n", (double)S.sweeps_cold / S.n_sys, (double)S.sweeps_warm / S.n_sys);
    // decisions that differ from the plain LU: 2 of 200 000 on the host, 1 of 199 936 on sm_90a; each must sit at the
    // threshold, a pivot ratio within a few eps of FullPivLU's 3 eps (16 eps: dcreg_oracle_mp.PIVOT_CLEAR)
    const bool pass = ulp_ok && S.bad == 0 && S.decisions_differ <= S.n_sys / 40000 &&
                      S.disagree_ratio < 16.0 * 2.220446049250313e-16 && S.n_sing > 1000 && S.worst_res < 1e-14 &&
                      S.worst_orth < 1e-14 && S.worst_warm < 1e-14 && S.worst_eig < 1e-14 && S.worst_inv < 1e-14 &&
                      S.sweeps_warm < S.sweeps_cold;
    printf(pass ? "K2_FAST_OK\n" : "K2_FAST_FAIL\n");
    return pass ? 0 : 1;
}
