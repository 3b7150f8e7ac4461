// DMMA (mma.sync m8n8k4 f64) latency / throughput probe (sm_90a), next to the DFMA rate of tools/fp64_probe.cu.
#include <cstdio>
#include <cuda_runtime.h>
__device__ __forceinline__ void dmma(double& c0, double& c1, double a, double b)
{
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
__global__ void k_lat(double* out, long long* cyc, int n)
{
    double a = out[threadIdx.x & 7], b = out[8 + (threadIdx.x & 7)], c0 = 0, c1 = 0;
    long long t0 = clock64();
    for (int i = 0; i < n; i++) { dmma(c0, c1, a, b); dmma(c0, c1, a, b); dmma(c0, c1, a, b); dmma(c0, c1, a, b); }
    long long t1 = clock64();
    if (threadIdx.x == 0) cyc[0] = t1 - t0;
    out[32 + threadIdx.x % 32] = c0 + c1;
}
template <int NACC>
__global__ void k_tput(double* out, long long* cyc, int n)
{
    double a = out[threadIdx.x & 7], b = out[8 + (threadIdx.x & 7)];
    double c[NACC][2];
#pragma unroll
    for (int k = 0; k < NACC; k++) c[k][0] = c[k][1] = 0.0;
    __syncthreads();
    long long t0 = clock64();
    for (int i = 0; i < n; i++) {
#pragma unroll
        for (int k = 0; k < NACC; k++) dmma(c[k][0], c[k][1], a, b);
    }
    __syncthreads();
    long long t1 = clock64();
    if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
    double s = 0;
#pragma unroll
    for (int k = 0; k < NACC; k++) s += c[k][0] + c[k][1];
    out[64 + (threadIdx.x & 31)] = s;
}
// DFMA warps and DMMA warps at the same time: do the FP64 CUDA-core pipe and the DMMA tensor sub-pipe add up?
__global__ void k_mixed(double* out, long long* cyc, int n, int dmma_warps)
{
    const int w = threadIdx.x >> 5;
    double a = out[threadIdx.x & 7], b = out[8 + (threadIdx.x & 7)];
    double c[8][2];
#pragma unroll
    for (int k = 0; k < 8; k++) { c[k][0] = a + k; c[k][1] = b + k; }
    __syncthreads();
    long long t0 = clock64();
    if (w < dmma_warps) {
        for (int i = 0; i < n; i++) {
#pragma unroll
            for (int k = 0; k < 8; k++) dmma(c[k][0], c[k][1], a, b);
        }
    } else {
        for (int i = 0; i < n; i++) {
#pragma unroll
            for (int k = 0; k < 8; k++) { c[k][0] = fma(c[k][0], a, b); c[k][1] = fma(c[k][1], a, b); }
        }
    }
    long long t1 = clock64();
    cyc[w] = t1 - t0;
    double s = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) s += c[k][0] + c[k][1];
    out[64 + (threadIdx.x & 31)] = s;
}
// barrier cost with many warps + named barrier subsets
__global__ void k_bar(long long* cyc, int n)
{
    __syncthreads();
    long long t0 = clock64();
    for (int i = 0; i < n; i++) __syncthreads();
    long long t1 = clock64();
    if (threadIdx.x == 0) { cyc[0] = t1 - t0; }
}
__global__ void k_bar64(long long* cyc, int n)
{
    long long t0 = clock64();
    if (threadIdx.x < 64) for (int i = 0; i < n; i++) asm volatile("bar.sync 1, 64;" ::: "memory");
    long long t1 = clock64();
    if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
// shared-memory flag handoff between two warps (volatile spin), round-trip
__global__ void k_flag(long long* cyc, int n)
{
    __shared__ volatile int f0, f1;
    if (threadIdx.x == 0) { f0 = 0; f1 = 0; }
    __syncthreads();
    long long t0 = clock64();
    if (threadIdx.x == 0) for (int i = 1; i <= n; i++) { f0 = i; while (f1 != i) {} }
    if (threadIdx.x == 32) for (int i = 1; i <= n; i++) { while (f0 != i) {} f1 = i; }
    long long t1 = clock64();
    if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
int main()
{
    double* d; long long* c; cudaMalloc(&d, 4096); cudaMalloc(&c, 4096);
    double h[16]; for (int i = 0; i < 16; i++) h[i] = 1.0 + 1e-9 * i; cudaMemcpy(d, h, sizeof(h), cudaMemcpyHostToDevice);
    long long hc[8];
    const int n = 4096;
    k_lat<<<1, 32>>>(d, c, n); cudaMemcpy(hc, c, 8, cudaMemcpyDeviceToHost);
    printf("DMMA.8x8x4 dependent-accumulator latency: %.1f cycles\n", hc[0] / (4.0 * n));
    for (int thr : {32, 128, 256, 512, 1024}) {
        k_tput<4><<<1, thr>>>(d, c, n); cudaMemcpy(hc, c, 8, cudaMemcpyDeviceToHost);
        printf("DMMA throughput 1 CTA x %4d thr, 4 acc: %.2f FMA/clk/SM (%.2f DMMA/clk)\n", thr, 256.0 * 4 * n * (thr / 32) / (double)hc[0], 4.0 * n * (thr / 32) / (double)hc[0]);
        k_tput<8><<<1, thr>>>(d, c, n); cudaMemcpy(hc, c, 8, cudaMemcpyDeviceToHost);
        printf("DMMA throughput 1 CTA x %4d thr, 8 acc: %.2f FMA/clk/SM\n", thr, 256.0 * 8 * n * (thr / 32) / (double)hc[0]);
    }
    int n_sm = 0;
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, 0);
    k_tput<8><<<n_sm, 512>>>(d, c, n); cudaMemcpy(hc, c, 8, cudaMemcpyDeviceToHost);
    printf("DMMA throughput %d CTAs x 512 thr, 8 acc: %.2f FMA/clk/SM (CTA 0)\n", n_sm, 256.0 * 8 * n * 16 / (double)hc[0]);
    for (int thr : {64, 256, 512, 1024}) {
        k_bar<<<1, thr>>>(c, 2048); cudaMemcpy(hc, c, 16, cudaMemcpyDeviceToHost);
        printf("%4d thr: __syncthreads %.1f cycles\n", thr, hc[0] / 2048.0);
        k_bar64<<<1, thr>>>(c, 2048); cudaMemcpy(hc, c, 8, cudaMemcpyDeviceToHost);
        printf("%4d thr: named barrier of 2 warps %.1f cycles\n", thr, hc[0] / 2048.0);
    }
    for (int dw : {0, 4, 8}) {
        k_mixed<<<1, 256>>>(d, c, n, dw); cudaMemcpy(hc, c, 64, cudaMemcpyDeviceToHost);
        long long mx = 0; for (int i = 0; i < 8; i++) mx = hc[i] > mx ? hc[i] : mx;
        printf("8 warps, %d DMMA + %d DFMA warps: %.1f FMA/clk/SM in total (slowest warp)\n", dw, 8 - dw, (dw * 8.0 * n * 256 + (8 - dw) * 16.0 * n * 32) / (double)mx);
    }
    k_flag<<<1, 64>>>(c, 2048); cudaMemcpy(hc, c, 8, cudaMemcpyDeviceToHost);
    printf("shared-memory flag round trip between two warps: %.1f cycles\n", hc[0] / 2048.0);
    printf("%s\n", cudaGetErrorString(cudaDeviceSynchronize()));
    return 0;
}
