// Pipe-rate microbenchmarks for sm_90a (H100): FP64 FMA, F2F conversions, INT ALU, mixed.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/microbench tools/microbench.cu
#include <cstdio>
#include <cuda_runtime.h>
#define ITERS 2048
template <int MODE>
__global__ void kern(double* out, double a, double b, int n) {
    double x[8];
    for (int i = 0; i < 8; ++i) x[i] = a + i + threadIdx.x * 1e-3;
    unsigned u[8];
    for (int i = 0; i < 8; ++i) u[i] = threadIdx.x + i;
    for (int it = 0; it < n; ++it) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            if (MODE == 0) x[i] = fma(x[i], a, b);                       // DFMA
            if (MODE == 1) x[i] = (double)(float)x[i] + 1e-3;            // 2x F2F + DADD
            if (MODE == 2) { x[i] = fma(x[i], a, b); u[i] = u[i] * 1664525u + 1013904223u; }   // DFMA + IMAD
            if (MODE == 3) { float f = __int_as_float(0x3f800000 | (u[i] & 0x7fffff)); x[i] += (double)f; u[i] += 7; }  // F2F.F64.F32 + DADD
            if (MODE == 4) x[i] = x[i] * a;                              // DMUL
            if (MODE == 5) { x[i] = fma(x[i], a, b); x[i] = (double)(float)x[i]; }  // DFMA + 2 F2F dependent
        }
    }
    double s = 0; for (int i = 0; i < 8; ++i) s += x[i] + u[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
template <int MODE>
void run(const char* name, double ops_per_iter_per_thread, int blocks_per_sm, int threads) {
    int sms = 132; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    int clk = 0; cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
    double* out; cudaMalloc(&out, sizeof(double) * sms * blocks_per_sm * threads);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    kern<MODE><<<sms * blocks_per_sm, threads>>>(out, 1.0000001, 1e-9, 64);
    cudaEventRecord(e0);
    kern<MODE><<<sms * blocks_per_sm, threads>>>(out, 1.0000001, 1e-9, ITERS);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    double total = ops_per_iter_per_thread * ITERS * (double)sms * blocks_per_sm * threads;
    double per_clk_sm = total / (ms * 1e-3) / (clk * 1e3) / sms;
    printf("%-34s blocks/SM %d thr %4d : %8.3f ms  %7.2f ops/clk/SM (at %d MHz)\n", name, blocks_per_sm, threads, ms, per_clk_sm, clk / 1000);
    cudaFree(out);
}
int main() {
    for (int b : {1, 2, 4}) {
        run<0>("DFMA", 8, b, 256);
        run<4>("DMUL", 8, b, 256);
        run<1>("F2F round trip (2 F2F + DADD)", 8, b, 256);
        run<3>("F2F.F64.F32 + DADD", 8, b, 256);
        run<2>("DFMA + IMAD (count DFMA)", 8, b, 256);
        run<5>("DFMA + 2 F2F dep (count DFMA)", 8, b, 256);
    }
    return 0;
}
