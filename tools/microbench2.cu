// FP64 tensor-core (mma.sync m8n8k4 f64) rate on sm_90a, alone and mixed with DFMA / F2F.
#include <cstdio>
#include <cuda_runtime.h>
#define ITERS 2048
__device__ __forceinline__ void dmma(double& d0, double& d1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                 : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}
template <int MODE, int NACC>
__global__ void kern(double* out, double a, double b, int n) {
    double c0[NACC], c1[NACC], x[4];
    for (int i = 0; i < NACC; ++i) { c0[i] = i; c1[i] = -i; }
    for (int i = 0; i < 4; ++i) x[i] = a + i + threadIdx.x * 1e-3;
    double av = a + threadIdx.x * 1e-6, bv = b + threadIdx.x * 1e-7;
    for (int it = 0; it < n; ++it) {
#pragma unroll
        for (int i = 0; i < NACC; ++i) {
            dmma(c0[i], c1[i], av, bv);
            if (MODE == 1) { x[i & 3] = fma(x[i & 3], a, b); x[(i + 1) & 3] = fma(x[(i + 1) & 3], a, b); }   // + 2 DFMA per DMMA
            if (MODE == 2) { x[i & 3] = fma(x[i & 3], a, b); x[(i+1)&3] = fma(x[(i+1)&3], a, b); x[(i+2)&3] = fma(x[(i+2)&3], a, b); x[(i+3)&3] = fma(x[(i+3)&3], a, b); }
        }
    }
    double s = 0; for (int i = 0; i < NACC; ++i) s += c0[i] + c1[i];
    for (int i = 0; i < 4; ++i) s += x[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
template <int MODE, int NACC>
void run(const char* name, int blocks_per_sm, int threads) {
    int sms = 132; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    int clk = 0; cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
    double* out; cudaMalloc(&out, sizeof(double) * sms * blocks_per_sm * threads);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    kern<MODE, NACC><<<sms * blocks_per_sm, threads>>>(out, 1.0000001, 1e-9, 64);
    cudaEventRecord(e0);
    kern<MODE, NACC><<<sms * blocks_per_sm, threads>>>(out, 1.0000001, 1e-9, ITERS);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    double warps = (double)sms * blocks_per_sm * threads / 32;
    double dmmas = warps * NACC * ITERS;
    double fma_per_clk_sm = dmmas * 256 / (ms * 1e-3) / (clk * 1e3) / sms;
    double cyc_per_dmma_smsp = (ms * 1e-3) * (clk * 1e3) / (dmmas / (sms * 4.0));
    printf("%-28s NACC %d blocks/SM %d thr %4d : %8.3f ms  %7.2f DMMA-FMA/clk/SM  %6.2f cyc/DMMA/SMSP\n", name, NACC, blocks_per_sm, threads, ms,
           fma_per_clk_sm, cyc_per_dmma_smsp);
    cudaFree(out);
}
int main() {
    for (int b : {1, 2, 4}) {
        run<0, 1>("DMMA only", b, 256);
        run<0, 4>("DMMA only", b, 256);
        run<0, 8>("DMMA only", b, 256);
        run<1, 4>("DMMA + 2 DFMA each", b, 256);
        run<2, 4>("DMMA + 4 DFMA each", b, 256);
    }
    return 0;
}
