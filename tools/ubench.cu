// tools/ubench.cu -- latency / throughput microbenchmarks of the fp64 building blocks of the solve kernel on sm_90a.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/ubench tools/ubench.cu ; prints cycles per operation.
#include <cstdio>
#include <cuda_runtime.h>
#define DMMA(d0, d1, a, b, c0, c1) asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%4,%5};" : "=d"(d0), "=d"(d1) : "d"(a), "d"(b), "d"(c0), "d"(c1))
__global__ void k_lat(double *out, long long *cyc, double seed) {
    __shared__ double sm[1024];
    const int lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) sm[i] = seed + i * 1e-9;
    __syncthreads();
    double x = seed + lane * 1e-3, y = 1.0000001, z = 0.5;
    long long t0, t1; int idx = 0;
    // 0: dependent DFMA chain
    t0 = clock64();
#pragma unroll
    for (int i = 0; i < 256; i++) x = fma(x, y, z);
    t1 = clock64(); if (threadIdx.x == 0) cyc[idx] = t1 - t0; idx++;
    // 1: 4 independent DFMA chains (per-op cost)
    double a0 = x, a1 = x + 1, a2 = x + 2, a3 = x + 3;
    t0 = clock64();
#pragma unroll
    for (int i = 0; i < 64; i++) { a0 = fma(a0, y, z); a1 = fma(a1, y, z); a2 = fma(a2, y, z); a3 = fma(a3, y, z); }
    t1 = clock64(); if (threadIdx.x == 0) cyc[idx] = t1 - t0; idx++;
    x = a0 + a1 + a2 + a3;
    // 2: dependent shfl (64-bit)
    t0 = clock64();
#pragma unroll
    for (int i = 0; i < 256; i++) x = __shfl_sync(0xffffffffu, x, (lane + 1) & 31);
    t1 = clock64(); if (threadIdx.x == 0) cyc[idx] = t1 - t0; idx++;
    // 3: dependent rsqrt
    x = fabs(x) + 1.5;
    t0 = clock64();
#pragma unroll
    for (int i = 0; i < 64; i++) x = rsqrt(x) + 1.5;
    t1 = clock64(); if (threadIdx.x == 0) cyc[idx] = t1 - t0; idx++;
    // 4: dependent 1/sqrt
    t0 = clock64();
#pragma unroll
    for (int i = 0; i < 64; i++) x = 1.0 / sqrt(x) + 1.5;
    t1 = clock64(); if (threadIdx.x == 0) cyc[idx] = t1 - t0; idx++;
    // 5: dependent division
    t0 = clock64();
#pragma unroll
    for (int i = 0; i < 64; i++) x = 1.0 / x + 1.5;
    t1 = clock64(); if (threadIdx.x == 0) cyc[idx] = t1 - t0; idx++;
    // 6: dependent LDS (pointer chase through doubles)
    int p = lane;
    t0 = clock64();
#pragma unroll
    for (int i = 0; i < 256; i++) p = ((int)sm[p] + p + 33) & 1023;
    t1 = clock64(); if (threadIdx.x == 0) cyc[idx] = t1 - t0; idx++;
    x += p;
    // 7: dependent DMMA chain
    double c0 = x, c1 = x;
    t0 = clock64();
#pragma unroll
    for (int i = 0; i < 256; i++) DMMA(c0, c1, y, z, c0, c1);
    t1 = clock64(); if (threadIdx.x == 0) cyc[idx] = t1 - t0; idx++;
    // 8: 8 independent DMMA chains (throughput, one warp)
    double e[8][2];
    for (int k = 0; k < 8; k++) { e[k][0] = x + k; e[k][1] = x - k; }
    t0 = clock64();
#pragma unroll
    for (int i = 0; i < 32; i++)
#pragma unroll
        for (int k = 0; k < 8; k++) DMMA(e[k][0], e[k][1], y, z, e[k][0], e[k][1]);
    t1 = clock64(); if (threadIdx.x == 0) cyc[idx] = t1 - t0; idx++;
    for (int k = 0; k < 8; k++) x += e[k][0] + e[k][1];
    // 9: __syncthreads cost
    t0 = clock64();
#pragma unroll
    for (int i = 0; i < 64; i++) __syncthreads();
    t1 = clock64(); if (threadIdx.x == 0) cyc[idx] = t1 - t0; idx++;
    // 10: __syncwarp cost
    t0 = clock64();
#pragma unroll
    for (int i = 0; i < 64; i++) { sm[lane] = x; __syncwarp(); x += sm[(lane + 1) & 31]; __syncwarp(); }
    t1 = clock64(); if (threadIdx.x == 0) cyc[idx] = t1 - t0; idx++;
    // 11: 8 independent DFMA chains
    double b[8]; for (int k = 0; k < 8; k++) b[k] = x + k;
    t0 = clock64();
#pragma unroll
    for (int i = 0; i < 32; i++)
#pragma unroll
        for (int k = 0; k < 8; k++) b[k] = fma(b[k], y, z);
    t1 = clock64(); if (threadIdx.x == 0) cyc[idx] = t1 - t0; idx++;
    for (int k = 0; k < 8; k++) x += b[k];
    // 12: dependent DMUL+DADD via sqrt
    t0 = clock64();
#pragma unroll
    for (int i = 0; i < 64; i++) x = sqrt(x) + 1.5;
    t1 = clock64(); if (threadIdx.x == 0) cyc[idx] = t1 - t0; idx++;
    out[blockIdx.x * blockDim.x + threadIdx.x] = x + c0 + c1;
}
int main() {
    const char *names[] = {"DFMA dependent (256)", "DFMA 4 chains (256 ops)", "SHFL.64 dependent (256)", "rsqrt dependent (64)", "1/sqrt dependent (64)", "1/x dependent (64)",
                           "LDS.64 dependent (256)", "DMMA dependent (256)", "DMMA 8 chains (256 ops)", "__syncthreads (64)", "STS+syncwarp+LDS+syncwarp (64)", "DFMA 8 chains (256 ops)", "sqrt dependent (64)"};
    const int nops[] = {256, 256, 256, 64, 64, 64, 256, 256, 256, 64, 64, 256, 64};
    double *out; long long *cyc; cudaMalloc(&out, 1 << 20); cudaMalloc(&cyc, 64 * 8);
    for (int threads : {32, 128, 256, 512}) {
        for (int rep = 0; rep < 2; rep++) k_lat<<<1, threads>>>(out, cyc, 1.25);
        cudaDeviceSynchronize();
        long long h[16]; cudaMemcpy(h, cyc, sizeof(h), cudaMemcpyDeviceToHost);
        printf("--- %d threads in the CTA (every warp runs the same sequence; cycles seen by warp 0) ---\n", threads);
        for (int i = 0; i < 13; i++) printf("  %-36s %8lld cyc  %7.2f cyc/op\n", names[i], h[i], (double)h[i] / nops[i]);
    }
    printf("%s\n", cudaGetErrorString(cudaGetLastError()));
    return 0;
}
