// Read-only streaming bandwidth on H100: how fast can a kernel READ two 160 MB arrays (no writes)?
#include <cstdio>
#include <cuda_runtime.h>
template <int U>
__global__ void rd(const float4* __restrict__ a, const float4* __restrict__ b, long long n, float* out) {
    float s = 0.f;
    const long long stride = (long long)gridDim.x * blockDim.x;
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (; i + (U - 1) * stride < n; i += U * stride) {
        float4 x[U], y[U];
#pragma unroll
        for (int u = 0; u < U; ++u) x[u] = __ldcs(&a[i + u * stride]);
#pragma unroll
        for (int u = 0; u < U; ++u) y[u] = __ldcs(&b[i + u * stride]);
#pragma unroll
        for (int u = 0; u < U; ++u) s += x[u].x + x[u].y + x[u].z + x[u].w + y[u].x + y[u].y + y[u].z + y[u].w;
    }
    for (; i < n; i += stride) { float4 x = a[i], y = b[i]; s += x.x + y.x; }
    if (s == 123.456f) out[0] = s;
}
__global__ void cp(const float4* __restrict__ a, float4* __restrict__ b, long long n) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) b[i] = a[i];
}
int main() {
    const long long n = 10'000'000;
    int sms = 132; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    float4 *a, *b; float* out;
    cudaMalloc(&a, n * 16); cudaMalloc(&b, n * 16); cudaMalloc(&out, 4);
    cudaMemset(a, 1, n * 16); cudaMemset(b, 2, n * 16);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    auto time = [&](auto launch, const char* name, double bytes) {
        launch(); launch();
        cudaEventRecord(e0);
        for (int r = 0; r < 20; ++r) launch();
        cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1); ms /= 20;
        printf("%-40s %8.3f us  %8.1f GB/s\n", name, ms * 1e3, bytes / (ms * 1e-3) / 1e9);
    };
    for (int bps : {2, 4, 8, 16}) {
        char nm[64];
        snprintf(nm, 64, "read 2x160MB U=1 blocks/SM=%d", bps); time([&] { rd<1><<<sms * bps, 256>>>(a, b, n, out); }, nm, 2.0 * n * 16);
        snprintf(nm, 64, "read 2x160MB U=2 blocks/SM=%d", bps); time([&] { rd<2><<<sms * bps, 256>>>(a, b, n, out); }, nm, 2.0 * n * 16);
        snprintf(nm, 64, "read 2x160MB U=4 blocks/SM=%d", bps); time([&] { rd<4><<<sms * bps, 256>>>(a, b, n, out); }, nm, 2.0 * n * 16);
    }
    time([&] { cp<<<sms * 8, 256>>>(a, b, n); }, "copy 160MB->160MB (r+w bytes)", 2.0 * n * 16);
    // bigger buffers
    float4 *c, *d; const long long m = 64'000'000;
    cudaMalloc(&c, m * 16); cudaMalloc(&d, m * 16); cudaMemset(c, 1, m * 16); cudaMemset(d, 2, m * 16);
    time([&] { rd<4><<<sms * 8, 256>>>(c, d, m, out); }, "read 2x1GB U=4 blocks/SM=8", 2.0 * m * 16);
    time([&] { cp<<<sms * 8, 256>>>(c, d, m); }, "copy 1GB->1GB (r+w bytes)", 2.0 * m * 16);
    return 0;
}
