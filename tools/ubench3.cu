// tools/ubench3.cu -- do the fp64 tensor pipe (DMMA) and the DFMA pipe co-issue from the same SM sub-partition (scheduler)?
// One CTA of 256 threads per SM (8 warps, two per scheduler, like vilo_solve_kernel).  Each warp runs either a DMMA stream (8 independent
// accumulator chains) or an "evaluation-like" DFMA stream (4 independent chains of dependent FMAs + shared-memory loads); the time of each
// role is reported for: all warps DFMA, all warps DMMA, one DMMA + one DFMA warp per scheduler, DMMA on schedulers 0-1 / DFMA on 2-3.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/ubench3 tools/ubench3.cu
#include <cstdio>
#include <cuda_runtime.h>
#define DMMA(d0, d1, a, b, c0, c1) asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%4,%5};" : "=d"(d0), "=d"(d1) : "d"(a), "d"(b), "d"(c0), "d"(c1))
__global__ void k(double *out, long long *cyc, unsigned dmma_mask, int n_dmma, int n_fma) {
    __shared__ double sm[1024];
    const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) sm[i] = 1.0 + i * 1e-9;
    __syncthreads();
    double acc = 0.0;
    const long long t0 = clock64();
    if ((dmma_mask >> wid) & 1) {
        double e[8][2];
        for (int q = 0; q < 8; q++) { e[q][0] = lane; e[q][1] = q; }
        const double a = 1.0000001, b = 0.9999999;
        for (int i = 0; i < n_dmma; i++) {
#pragma unroll
            for (int q = 0; q < 8; q++) DMMA(e[q][0], e[q][1], a, b, e[q][0], e[q][1]);
        }
        for (int q = 0; q < 8; q++) acc += e[q][0] + e[q][1];
    } else {
        double a0 = lane, a1 = lane + 1, a2 = lane + 2, a3 = lane + 3;
        const double y = 1.0000001;
        for (int i = 0; i < n_fma; i++) {
            const double z0 = sm[(lane + 4 * i) & 1023], z1 = sm[(lane + 4 * i + 1) & 1023];
#pragma unroll
            for (int u = 0; u < 4; u++) { a0 = fma(a0, y, z0); a1 = fma(a1, y, z1); a2 = fma(a2, y, z0); a3 = fma(a3, y, z1); }
        }
        acc = a0 + a1 + a2 + a3;
    }
    const long long t1 = clock64();
    if (lane == 0 && blockIdx.x == 0) cyc[wid] = t1 - t0;
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
}
int main() {
    double *out; long long *cyc; cudaMalloc(&out, 132 * 256 * 8); cudaMalloc(&cyc, 64);
    const int ND = 512, NF = 512;      // per warp: 4096 DMMA or 8192 DFMA (+ 1024 LDS.64)
    struct { const char *name; unsigned mask; } cases[] = {
        {"all 8 warps DFMA stream", 0x00}, {"all 8 warps DMMA stream", 0xff},
        {"warps 0-3 DMMA, 4-7 DFMA (one of each per scheduler)", 0x0f}, {"warps 0,1,4,5 DMMA (schedulers 0,1), 2,3,6,7 DFMA (schedulers 2,3)", 0x33},
        {"warp 0 DMMA only, 1-7 DFMA", 0x01}, {"warps 0-3 DMMA, 4-7 idle-ish (DFMA n=1)", 0x0f}};
    for (int c = 0; c < 6; c++) {
        long long h[8];
        for (int rep = 0; rep < 2; rep++) { k<<<132, 256>>>(out, cyc, cases[c].mask, ND, c == 5 ? 1 : NF); cudaDeviceSynchronize(); }
        cudaMemcpy(h, cyc, 64, cudaMemcpyDeviceToHost);
        printf("%-75s cycles per warp:", cases[c].name);
        for (int w = 0; w < 8; w++) printf(" %6lld%c", h[w], ((cases[c].mask >> w) & 1) ? 'T' : 'F');
        printf("\n");
    }
    printf("(T: DMMA warp, %d DMMA each; F: DFMA warp, %d DFMA + %d LDS.64 each)\n", ND * 8, NF * 16, NF * 2);
    return 0;
}
