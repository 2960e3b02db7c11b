// Device check of the loop's plane fit (tests/test_gpu_fit_plane.py), built for sm_90a with the library's flags:
// corr::fit_plane_reg (correctly rounded primitives, plain fallback) against the fit as it was before them, kept
// below as ref_fit with its pivoted QR (plain `/` and `sqrt`).  ok, nx, ny, nz and d must be bit-identical, under the
// default gates (1e-6, 0.2) and loose ones (0, 1e30) that let every fit reach the normalisation and the gate.
//   usage: test_fit_plane [points.f32 keys.i32]   (float4 points and rows of five int32 positions, e.g. C2 and corridor
//          neighbourhoods written by the test), after the built-in sets:
//   * the 400 000 systems of tools/test_qr_reg.cu (random, wide, z = 0 floor, dependent columns, duplicate rows,
//     collinear lattices, thin, all zero);
//   * exact collinear and coplanar lattices and pivot ties (equal column norms, permuted axes);
//   * all 120 row orders of 64 five-point sets;
//   * neighbourhoods scaled past float range (infinite or NaN coordinates), where the fallback must run;
//   * finite neighbourhoods of extreme scale (float subnormals beside 2^100-2^126), where the fallback must run and
//     return finite planes.
// Prints, per set, systems, mismatches and fallbacks; FIT_PLANE_OK on success.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "../dcreg_b200/csrc/corr.cuh"

// ---- the fit before the correctly rounded primitives, verbatim (plain / and sqrt) ----
template <int M, int N>
__device__ __forceinline__ void ref_qr(double (&A)[M][N], double (&b)[M], double (&x)[N]) {
    const double eps = 2.220446049250313e-16;
    double normU[N], normD[N];
    int perm[N];
    double maxn = 0.0;
#pragma unroll
    for (int j = 0; j < N; ++j) {
        double s = 0.0;
#pragma unroll
        for (int i = 0; i < M; ++i) s += A[i][j] * A[i][j];
        normU[j] = normD[j] = sqrt(s);
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
            beta = sqrt(c0 * c0 + tail);
            if (c0 >= 0.0) beta = -beta;
            const double inv = 1.0 / (c0 - beta);
#pragma unroll
            for (int i = k + 1; i < M; ++i) A[i][k] *= inv;
            tau = (beta - c0) / beta;
        }
        A[k][k] = beta;
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
#pragma unroll
        for (int j = k + 1; j < N; ++j) {
            if (normU[j] != 0.0) {
                double t = fabs(A[k][j]) / normU[j];
                t = (1.0 + t) * (1.0 - t);
                if (t < 0.0) t = 0.0;
                const double r = normU[j] / normD[j];
                const double t2 = t * r * r;
                if (t2 <= downdate_thr) {
                    double s = 0.0;
#pragma unroll
                    for (int i = k + 1; i < M; ++i) s += A[i][j] * A[i][j];
                    normD[j] = normU[j] = sqrt(s);
                } else {
                    normU[j] *= sqrt(t);
                }
            }
        }
    }
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
            c[i] = s / A[i][i];
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

__device__ __forceinline__ bool ref_fit(const corr::Grid& g, const int* kpos, double min_norm, double thickness,
                                        double& nx, double& ny, double& nz, double& d) {
    double A[5][3], b[5], x[3];
#pragma unroll
    for (int j = 0; j < 5; ++j) {
        const float4 p = __ldg(&g.pts[kpos[j]]);
        A[j][0] = (double)p.x;
        A[j][1] = (double)p.y;
        A[j][2] = (double)p.z;
        b[j] = -1.0;
    }
    ref_qr<5, 3>(A, b, x);
    const double ps = sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
    if (!(ps >= min_norm)) return false;
    nx = x[0] / ps; ny = x[1] / ps; nz = x[2] / ps; d = 1.0 / ps;
    double worst = 0.0;
#pragma unroll
    for (int j = 0; j < 5; ++j) {
        const float4 p = __ldg(&g.pts[kpos[j]]);
        double e = nx * (double)p.x + ny * (double)p.y + nz * (double)p.z + d;
        e *= e;
        worst = fmax(worst, e);
    }
    return worst < thickness * thickness;
}

// out[10 * i ..]: new ok, n, d | reference ok, n, d (as doubles; untouched outputs keep the sentinel) ; fell[i]: the
// fast fit set its range flag, so fit_plane_reg ran the fallback
__global__ void fits(corr::Grid g, const int* keys, int n, double min_norm, double thickness, double* out, int* fell) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int* kp = keys + 5 * i;
    const double s = -12345.0;
    double a[4] = {s, s, s, s}, r[4] = {s, s, s, s}, f[4] = {s, s, s, s};
    const bool ok = corr::fit_plane_reg(g, kp, min_norm, thickness, a[0], a[1], a[2], a[3]);
    const bool rok = ref_fit(g, kp, min_norm, thickness, r[0], r[1], r[2], r[3]);
    bool bad = false;
    corr::fit_plane_ar(g.pts, kp, min_norm, thickness, f[0], f[1], f[2], f[3], corr::CrArith{bad});
    double* o = out + 10 * i;
    o[0] = ok; o[5] = rok;
    for (int k = 0; k < 4; ++k) { o[1 + k] = a[k]; o[6 + k] = r[k]; }
    fell[i] = bad;
}

static unsigned long long st = 88172645463325252ull;
static double rnd() { st ^= st << 13; st ^= st >> 7; st ^= st << 17; return (double)(st >> 11) / 9007199254740992.0; }

struct Set {
    const char* name;
    std::vector<float4> pts;
    std::vector<int> keys;
    bool need_fallback = false, need_finite_fallback = false;
    void add5(const float P[5][3]) {
        for (int i = 0; i < 5; ++i) { keys.push_back((int)pts.size()); pts.push_back(make_float4(P[i][0], P[i][1], P[i][2], 0.f)); }
    }
};

static bool run(const Set& s) {
    const int n = (int)s.keys.size() / 5;
    float4* dp; int* dk; double* dout; int* dfell;
    cudaMalloc(&dp, s.pts.size() * sizeof(float4)); cudaMalloc(&dk, s.keys.size() * sizeof(int));
    cudaMalloc(&dout, (size_t)n * 10 * sizeof(double)); cudaMalloc(&dfell, (size_t)n * sizeof(int));
    cudaMemcpy(dp, s.pts.data(), s.pts.size() * sizeof(float4), cudaMemcpyHostToDevice);
    cudaMemcpy(dk, s.keys.data(), s.keys.size() * sizeof(int), cudaMemcpyHostToDevice);
    corr::Grid g;
    memset(&g, 0, sizeof(g));
    g.pts = dp;
    g.n = (int)s.pts.size();
    std::vector<double> out((size_t)n * 10);
    std::vector<int> fell(n);
    const double gates[2][2] = {{1e-6, 0.2}, {0.0, 1e30}};
    long bad = 0, fallbacks = 0, finite_fallbacks = 0, valid = 0;
    for (const auto& gt : gates) {
        fits<<<(n + 127) / 128, 128>>>(g, dk, n, gt[0], gt[1], dout, dfell);
        if (cudaMemcpy(out.data(), dout, out.size() * sizeof(double), cudaMemcpyDeviceToHost) != cudaSuccess) {
            printf("CUDA error: %s\n", cudaGetErrorString(cudaGetLastError()));
            exit(1);
        }
        cudaMemcpy(fell.data(), dfell, fell.size() * sizeof(int), cudaMemcpyDeviceToHost);
        for (int i = 0; i < n; ++i) {
            const double* o = &out[(size_t)10 * i];
            valid += o[0] != 0.0;
            fallbacks += fell[i];
            bool finite = true;   // the reference wrote a finite (n, d)
            for (int k = 6; k < 10; ++k) finite = finite && std::isfinite(o[k]) && o[k] != -12345.0;
            finite_fallbacks += fell[i] && finite;
            if (memcmp(o, o + 5, 5 * sizeof(double)) != 0) {
                if (bad < 5) printf("  %s #%d: ok %g n %a %a %a d %a vs ok %g n %a %a %a d %a\n", s.name, i, o[0], o[1], o[2], o[3], o[4], o[5], o[6], o[7], o[8], o[9]);
                ++bad;
            }
        }
    }
    printf("%s: %d systems x 2 gates, %ld mismatches, %ld valid planes, %ld fallbacks (%ld with a finite plane)\n", s.name, n, bad,
           valid, fallbacks, finite_fallbacks);
    cudaFree(dp); cudaFree(dk); cudaFree(dout); cudaFree(dfell);
    return bad == 0 && (!s.need_fallback || fallbacks > 0) && (!s.need_finite_fallback || finite_fallbacks > 0);
}

int main(int argc, char** argv) {
    bool ok = true;
    {   // tools/test_qr_reg.cu's generator
        Set s; s.name = "qr_reg systems";
        for (int trial = 0; trial < 400000; ++trial) {
            float P[5][3];
            const int kind = trial % 8;
            for (int i = 0; i < 5; ++i)
                for (int j = 0; j < 3; ++j) P[i][j] = (float)((rnd() - 0.5) * (kind == 1 ? 80.0 : 2.0));
            if (kind == 2) for (int i = 0; i < 5; ++i) P[i][2] = 0.0f;
            if (kind == 3) for (int i = 0; i < 5; ++i) P[i][1] = (float)(2.0 * P[i][0]);
            if (kind == 4) { for (int j = 0; j < 3; ++j) { P[1][j] = P[0][j]; P[3][j] = P[2][j]; } }
            if (kind == 5) for (int i = 0; i < 5; ++i) for (int j = 0; j < 3; ++j) P[i][j] = (float)(i * (j + 1) * 0.25);
            if (kind == 6) for (int i = 0; i < 5; ++i) P[i][2] = (float)(1e-6 * (rnd() - 0.5));
            if (kind == 7) for (int i = 0; i < 5; ++i) for (int j = 0; j < 3; ++j) P[i][j] = 0.0f;
            s.add5(P);
        }
        ok = run(s) && ok;
    }
    {   // exact lattices and pivot ties
        Set s; s.name = "lattices and ties";
        for (int t = 0; t < 20000; ++t) {
            float P[5][3];
            const int kind = t % 5, ax = (t / 5) % 3;
            const float h = (float)(0.05 * (1 + t % 13)), o[3] = {(float)(int)(rnd() * 80 - 40), (float)(int)(rnd() * 80 - 40), (float)(int)(rnd() * 20)};
            for (int i = 0; i < 5; ++i) {
                float v[3];
                if (kind == 0) { v[0] = i * h; v[1] = 2 * i * h; v[2] = 3 * i * h; }                     // collinear
                else if (kind == 1) { v[0] = (i % 3) * h; v[1] = (i / 3) * h; v[2] = 0.f; }              // coplanar lattice
                else if (kind == 2) { v[0] = (i % 2) * h; v[1] = ((i + 1) % 2) * h; v[2] = (i / 2) * h; } // equal norms
                else if (kind == 3) { v[0] = v[1] = v[2] = (i + 1) * h; }                                 // three-way tie
                else { v[0] = (i % 3 - 1) * h; v[1] = (i % 2) * h; v[2] = (i / 4) * h; }
                for (int j = 0; j < 3; ++j) P[i][(j + ax) % 3] = v[j] + (t % 2 ? o[j] : 0.f);
            }
            s.add5(P);
        }
        ok = run(s) && ok;
    }
    {   // all 120 row orders of 64 sets: 16 random, 16 on a lattice, 16 floor (z = 0), 16 on a wall of radius 40
        Set s; s.name = "row orders";
        for (int set = 0; set < 64; ++set) {
            float Q[5][3];
            for (int i = 0; i < 5; ++i) {
                const double u = rnd(), v = rnd();
                if (set < 16) { for (int j = 0; j < 3; ++j) Q[i][j] = (float)(rnd() - 0.5); }
                else if (set < 32) { Q[i][0] = (float)(0.25 * (i % 3)); Q[i][1] = (float)(0.25 * (i / 3)); Q[i][2] = (float)(0.25 * ((i * 7) % 2)); }
                else if (set < 48) { Q[i][0] = (float)(10 + u); Q[i][1] = (float)(-5 + v); Q[i][2] = 0.f; }
                else { const double th = 0.3 + 0.02 * u; Q[i][0] = (float)(40 * cos(th)); Q[i][1] = (float)(40 * sin(th)); Q[i][2] = (float)(5 + v); }
            }
            int p[5] = {0, 1, 2, 3, 4};
            do {
                float P[5][3];
                for (int i = 0; i < 5; ++i) for (int j = 0; j < 3; ++j) P[i][j] = Q[p[i]][j];
                s.add5(P);
            } while (std::next_permutation(p, p + 5));
        }
        ok = run(s) && ok;
    }
    {   // past float range: the primitives' range is left, so the fallback must run
        Set s; s.name = "non-finite neighbourhoods"; s.need_fallback = true;
        for (int t = 0; t < 4000; ++t) {
            float P[5][3];
            for (int i = 0; i < 5; ++i) for (int j = 0; j < 3; ++j) P[i][j] = (float)((rnd() - 0.5) * 2.0);
            const int i = t % 5, j = (t / 5) % 3;
            P[i][j] = (t / 15) % 3 == 0 ? P[i][j] * 1e38f * 1e38f : ((t / 15) % 3 == 1 ? NAN : -INFINITY);
            s.add5(P);
        }
        ok = run(s) && ok;
    }
    {   // finite but extreme scales: three nearly identical rows of float subnormals beside coordinates near 2^100-2^126
        // drive QR operands (column norms, downdates) below the primitives' range while n and d stay finite, so the
        // fallback must run and return the plain fit's finite plane
        Set s; s.name = "extreme-scale neighbourhoods"; s.need_fallback = true; s.need_finite_fallback = true;
        for (int t = 0; t < 40000; ++t) {
            const int ax = t % 3, kind = (t / 3) % 3, k = 2 + (int)(rnd() * 60);
            float v[5][3] = {}, P[5][3];
            v[0][1] = v[1][1] = ldexpf((float)k, -149); v[2][1] = ldexpf((float)(k + 1), -149);
            v[3][0] = (rnd() < 0.5 ? -1 : 1) * ldexpf(1.0f + (float)rnd(), 100 + (int)(rnd() * 27));
            v[3][1] = (rnd() < 0.5 ? -1 : 1) * ldexpf(1.0f + (float)rnd(), 90 + (int)(rnd() * 30));
            v[3][2] = ldexpf((float)(1 + (int)(rnd() * 8)), -149);
            v[4][1] = (rnd() < 0.5 ? -1 : 1) * ldexpf(1.0f + (float)rnd(), 100 + (int)(rnd() * 27));
            if (kind == 1) v[4][2] = ldexpf(1.0f + (float)rnd(), -140 + (int)(rnd() * 20));
            if (kind == 2) v[3][2] = ldexpf(1.0f + (float)rnd(), -100 + (int)(rnd() * 60));
            for (int r = 0; r < 5; ++r) for (int c = 0; c < 3; ++c) P[r][(c + ax) % 3] = v[r][c];
            s.add5(P);
        }
        ok = run(s) && ok;
    }
    if (argc >= 3) {   // neighbourhoods of real clouds
        Set s; s.name = argv[1];
        FILE* f = fopen(argv[1], "rb");
        FILE* k = fopen(argv[2], "rb");
        if (!f || !k) { printf("cannot open %s / %s\n", argv[1], argv[2]); return 1; }
        float4 p;
        while (fread(&p, sizeof(p), 1, f) == 1) s.pts.push_back(p);
        int key;
        while (fread(&key, sizeof(key), 1, k) == 1) s.keys.push_back(key);
        fclose(f); fclose(k);
        if (s.keys.empty() || s.keys.size() % 5) { printf("bad key file\n"); return 1; }
        ok = run(s) && ok;
    }
    if (ok) printf("FIT_PLANE_OK\n");
    return ok ? 0 : 1;
}
