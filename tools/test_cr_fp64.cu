// Device check of dcreg_b200/csrc/cr_fp64.cuh (tests/test_gpu_fit_plane.py), built for sm_90a with the library's flags:
//   * crf::div and crf::sqrt against __ddiv_rn / __dsqrt_rn, bit for bit wherever their flag is clear, over 2^27
//     operand pairs and 2^27 radicands.  Operand classes (index mod 8): random bit patterns (every exponent, so
//     log-uniform magnitudes plus zeros, subnormals, infinities and NaN), all-ones / all-zeros mantissas, operands next
//     to each range bound, results near powers of two, exact quotients and squares, quotients next to the quotient
//     bounds, the fit's magnitudes (1e-3 .. 1e3) and signed zeros;
//   * the flag is set on zero, subnormal, huge, infinite and NaN divisors, on subnormal, tiny, infinite and NaN
//     dividends, on quotients outside the range, and on negative, subnormal, huge, infinite and NaN radicands; signed
//     zero dividends and radicands are exact with the flag clear.
// Prints CR_FP64_OK on success.
#include <cstdio>
#include <cstring>
#include "../dcreg_b200/csrc/cr_fp64.cuh"

__device__ __forceinline__ unsigned long long mix(unsigned long long z) {
    z += 0x9e3779b97f4a7c15ull;
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}
__device__ __forceinline__ double from_bits(unsigned long long u) { return __longlong_as_double((long long)u); }
__device__ __forceinline__ unsigned long long bits(double v) { return (unsigned long long)__double_as_longlong(v); }
// sign s, biased exponent e (0 .. 2047), mantissa m
__device__ __forceinline__ double make(unsigned long long s, long long e, unsigned long long m) {
    e = e < 0 ? 0 : (e > 2047 ? 2047 : e);
    return from_bits((s << 63) | ((unsigned long long)e << 52) | (m & 0xfffffffffffffull));
}
// a mantissa that is all zeros, all ones, or one of those with a few random low or high bits changed
__device__ __forceinline__ unsigned long long edge_mantissa(unsigned long long r) {
    const unsigned long long all = (r & 1) ? 0xfffffffffffffull : 0ull;
    switch ((r >> 1) & 3) {
        case 0: return all;
        case 1: return all ^ ((r >> 8) & 0xf);
        case 2: return all ^ (((r >> 8) & 0xf) << 48);
        default: return all ^ (1ull << ((r >> 8) % 52));
    }
}
__device__ __forceinline__ long long near(unsigned long long r, long long e) { return e + (long long)(r % 7) - 3; }

__device__ void div_operands(unsigned long long i, double& a, double& b) {
    const unsigned long long r0 = mix(2 * i), r1 = mix(2 * i + 1), r2 = mix(r0 ^ r1);
    const unsigned long long sa = r2 & 1, sb = (r2 >> 1) & 1;
    switch (i & 7) {
        case 0: a = from_bits(r0); b = from_bits(r1); break;                                       // every pattern
        case 1: a = make(sa, 1 + r0 % 2046, edge_mantissa(r1)); b = make(sb, 1 + r1 % 2046, edge_mantissa(r0)); break;
        case 2: {                                                                                  // next to a bound
            const long long eb[4] = {0x001, 0x7f8, 0x3ff, 0x002};
            const long long ea[4] = {0x038, 0x7fe, 0x3ff, 0x037};
            a = make(sa, near(r0 >> 20, ea[r2 >> 8 & 3]), (r2 >> 12 & 1) ? edge_mantissa(r0) : r0);
            b = make(sb, near(r1 >> 20, eb[r2 >> 10 & 3]), (r2 >> 13 & 1) ? edge_mantissa(r1) : r1);
            break;
        }
        case 3: {                                                                                  // q near 2^k
            b = make(sb, 0x3ff - 500 + (long long)(r0 % 1000), r1);
            const double q = make(sa, 0x3ff - 400 + (long long)(r1 % 800), (r2 >> 8 & 1) ? (r2 >> 12) % 5 : 0xfffffffffffffull - (r2 >> 12) % 5);
            a = __dmul_rn(q, b);
            break;
        }
        case 4: {                                                                                  // exact quotient
            b = make(sb, 0x3ff - 300 + (long long)(r0 % 600), r1 & 0xffffffe000000ull);            // 27 significant bits
            const double m = (double)(1 + (r2 >> 8) % (1ull << 26));
            a = sa ? -__dmul_rn(b, m) : __dmul_rn(b, m);
            break;
        }
        case 5: {                                                                                  // q next to 2^-1022 or 2^1017
            b = make(sb, 0x3ff - 200 + (long long)(r0 % 400), r1);
            const long long eq = near(r0 >> 32, (r2 >> 8 & 1) ? 0x001 : 0x7f8);
            const double q = make(sa, eq, (r2 >> 9 & 1) ? edge_mantissa(r2 >> 10) : r2 >> 10);
            a = __dmul_rn(q, b);
            break;
        }
        case 6: a = make(sa, 0x3ff - 10 + (long long)(r0 % 20), r1); b = make(sb, 0x3ff - 10 + (long long)(r1 % 20), r0); break;
        default: a = sa ? -0.0 : 0.0; b = make(sb, r0 % 2048, r1); break;                         // signed zero dividend
    }
}

__device__ double sqrt_operand(unsigned long long i) {
    const unsigned long long r0 = mix(~i), r1 = mix(r0 + 7), r2 = mix(r0 ^ r1);
    switch (i & 7) {
        case 0: return from_bits(r0);
        case 1: return make(r2 & 1, 1 + r0 % 2046, edge_mantissa(r1));
        case 2: { const long long e[4] = {0x035, 0x7f8, 0x001, 0x3ff}; return make(0, near(r0 >> 20, e[r2 >> 8 & 3]), (r2 >> 12 & 1) ? edge_mantissa(r1) : r1); }
        case 3: {                                                                                  // sqrt near 2^k
            const double s = make(0, 0x3ff - 480 + (long long)(r0 % 960), (r2 >> 8 & 1) ? (r2 >> 12) % 5 : 0xfffffffffffffull - (r2 >> 12) % 5);
            return __dmul_rn(s, s);
        }
        case 4: {                                                                                  // exact square
            const double m = (double)(1 + (r1 >> 8) % (1ull << 26));
            const double s = make(0, 0x3ff - 450 + (long long)(r0 % 900), 0);
            return __dmul_rn(__dmul_rn(m, m), __dmul_rn(s, s));
        }
        case 5: return make(0, 0x3ff - 600 + (long long)(r0 % 1200), r1);
        case 6: return make(0, 0x3ff - 20 + (long long)(r0 % 40), r1);
        default: return (r0 & 1) ? -0.0 : 0.0;
    }
}

// counts: [0] div compared, [1] div mismatches, [2] sqrt compared, [3] sqrt mismatches, [4 + c] div compared in class
// c, [12 + c] sqrt compared in class c
__global__ void sweep(unsigned long long n, unsigned long long* counts) {
    unsigned long long dc = 0, dm = 0, sc = 0, sm = 0;
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
        double a, b;
        div_operands(i, a, b);
        bool bad = false;
        const double q = crf::div(a, b, bad);
        if (!bad) {
            ++dc;
            atomicAdd(&counts[4 + (i & 7)], 1ull);
            if (bits(q) != bits(__ddiv_rn(a, b))) {
                if (atomicAdd(&counts[1], 1ull) < 5) printf("div mismatch %a / %a: %a vs %a\n", a, b, q, __ddiv_rn(a, b));
                ++dm;
            }
        }
        const double x = sqrt_operand(i);
        bad = false;
        const double s = crf::sqrt(x, bad);
        if (!bad) {
            ++sc;
            atomicAdd(&counts[12 + (i & 7)], 1ull);
            if (bits(s) != bits(__dsqrt_rn(x))) {
                if (atomicAdd(&counts[3], 1ull) < 5) printf("sqrt mismatch %a: %a vs %a\n", x, s, __dsqrt_rn(x));
                ++sm;
            }
        }
    }
    atomicAdd(&counts[0], dc); atomicAdd(&counts[2], sc);
    (void)dm; (void)sm;
}

// one operation per thread: op 0 = a / b, 1 = sqrt(a); out = value, flag
__global__ void single(int n, const int* op, const double* a, const double* b, double* out, int* flag) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    bool bad = false;
    out[i] = op[i] == 0 ? crf::div(a[i], b[i], bad) : crf::sqrt(a[i], bad);
    flag[i] = bad;
}

static double dbits(unsigned long long u) { double d; memcpy(&d, &u, 8); return d; }

int main() {
    const unsigned long long n = 1ull << 27;
    unsigned long long* dcounts;
    cudaMalloc(&dcounts, 20 * sizeof(unsigned long long));
    cudaMemset(dcounts, 0, 20 * sizeof(unsigned long long));
    sweep<<<132 * 16, 256>>>(n, dcounts);
    unsigned long long c[20];
    if (cudaMemcpy(c, dcounts, sizeof(c), cudaMemcpyDeviceToHost) != cudaSuccess) { printf("CUDA error\n"); return 1; }
    printf("div: %llu of %llu compared, %llu mismatches; per class", c[0], n, c[1]);
    for (int k = 0; k < 8; ++k) printf(" %llu", c[4 + k]);
    printf("\nsqrt: %llu of %llu compared, %llu mismatches; per class", c[2], n, c[3]);
    for (int k = 0; k < 8; ++k) printf(" %llu", c[12 + k]);
    printf("\n");
    bool ok = c[1] == 0 && c[3] == 0 && c[0] + c[2] >= 100000000ull;
    for (int k = 0; k < 8; ++k) ok = ok && c[4 + k] > n / 64 && c[12 + k] > n / 64;

    // operands the flag must catch (expect = 1) and signed zeros it must pass exactly (expect = 0)
    const double inf = dbits(0x7ff0000000000000ull), nan = dbits(0x7ff8000000000000ull), dmax = dbits(0x7fefffffffffffffull);
    const double sub = dbits(0x000fffffffffffffull), tiny = dbits(1ull), huge = dbits(0x7f80000000000000ull);
    const double justbelow = dbits(0x037fffffffffffffull);   // largest dividend below 2^-967
    struct Case { int op; double a, b; int expect; const char* what; };
    const Case cases[] = {
        {0, 1.5, 0.0, 1, "zero divisor"}, {0, 1.5, -0.0, 1, "-zero divisor"}, {0, 1.5, sub, 1, "subnormal divisor"},
        {0, 1.5, -tiny, 1, "smallest subnormal divisor"}, {0, 1.5, huge, 1, "divisor 2^1017"}, {0, 1.5, dmax, 1, "huge divisor"},
        {0, 1.5, inf, 1, "infinite divisor"}, {0, 1.5, -inf, 1, "-infinite divisor"}, {0, 1.5, nan, 1, "NaN divisor"},
        {0, sub, 1.5, 1, "subnormal dividend"}, {0, justbelow, 1.0, 1, "dividend below 2^-967"}, {0, inf, 1.5, 1, "infinite dividend"},
        {0, nan, 1.5, 1, "NaN dividend"}, {0, dmax, 0.5, 1, "overflowing quotient"}, {0, 1e300, 1e-10, 1, "huge quotient"},
        {0, 1e-300, 1e10, 1, "subnormal quotient"}, {0, 0.0, inf, 1, "zero over infinity"}, {0, 0.0, 0.0, 1, "zero over zero"},
        {1, -1.0, 0.0, 1, "negative radicand"}, {1, -inf, 0.0, 1, "-infinite radicand"}, {1, sub, 0.0, 1, "subnormal radicand"},
        {1, tiny, 0.0, 1, "smallest subnormal radicand"}, {1, huge, 0.0, 1, "radicand 2^1017"}, {1, dmax, 0.0, 1, "huge radicand"},
        {1, inf, 0.0, 1, "infinite radicand"}, {1, nan, 0.0, 1, "NaN radicand"},
        {0, 0.0, 3.0, 0, "+0 / 3"}, {0, -0.0, 3.0, 0, "-0 / 3"}, {0, 0.0, -3.0, 0, "+0 / -3"}, {0, -0.0, -3.0, 0, "-0 / -3"},
        {1, 0.0, 0.0, 0, "sqrt(+0)"}, {1, -0.0, 0.0, 0, "sqrt(-0)"}, {0, 1.0, 3.0, 0, "1 / 3"}, {1, 2.0, 0.0, 0, "sqrt(2)"},
    };
    const int m = sizeof(cases) / sizeof(cases[0]);
    int op[64], flag[64];
    double a[64], b[64], out[64];
    for (int i = 0; i < m; ++i) { op[i] = cases[i].op; a[i] = cases[i].a; b[i] = cases[i].b; }
    int *dop, *dflag;
    double *da, *db, *dout;
    cudaMalloc(&dop, sizeof(op)); cudaMalloc(&dflag, sizeof(flag)); cudaMalloc(&da, sizeof(a)); cudaMalloc(&db, sizeof(b)); cudaMalloc(&dout, sizeof(out));
    cudaMemcpy(dop, op, sizeof(op), cudaMemcpyHostToDevice);
    cudaMemcpy(da, a, sizeof(a), cudaMemcpyHostToDevice);
    cudaMemcpy(db, b, sizeof(b), cudaMemcpyHostToDevice);
    single<<<1, 64>>>(m, dop, da, db, dout, dflag);
    if (cudaMemcpy(flag, dflag, sizeof(flag), cudaMemcpyDeviceToHost) != cudaSuccess) { printf("CUDA error\n"); return 1; }
    cudaMemcpy(out, dout, sizeof(out), cudaMemcpyDeviceToHost);
    for (int i = 0; i < m; ++i) {
        bool good = flag[i] == cases[i].expect;
        if (cases[i].expect == 0) {   // exact: compare with the host's IEEE result, sign of zero included
            const double ref = cases[i].op == 0 ? cases[i].a / cases[i].b : sqrt(cases[i].a);
            good = good && memcmp(&ref, &out[i], 8) == 0;
        }
        if (!good) { printf("%s: flag %d (expected %d), value %a\n", cases[i].what, flag[i], cases[i].expect, out[i]); ok = false; }
    }
    printf("%d special operands checked\n", m);
    if (ok) printf("CR_FP64_OK\n");
    return ok ? 0 : 1;
}
