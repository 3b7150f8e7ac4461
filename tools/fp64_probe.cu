// FP64 / shared-memory latency + throughput probe (sm_90a).
#include <cstdio>
#include <cuda_runtime.h>
__global__ void k_lat(double* out, long long* cyc, int n) {
    double a = out[0], b = out[1], c = out[2];
    long long t0 = clock64();
    for (int i = 0; i < n; i++) { a = fma(a, b, c); a = fma(a, b, c); a = fma(a, b, c); a = fma(a, b, c); }
    long long t1 = clock64();
    float fa = (float)out[0], fb = (float)out[1], fc = (float)out[2];
    for (int i = 0; i < n; i++) { fa = fmaf(fa, fb, fc); fa = fmaf(fa, fb, fc); fa = fmaf(fa, fb, fc); fa = fmaf(fa, fb, fc); }
    long long t2 = clock64();
    double r = out[3];
    for (int i = 0; i < n; i++) { r = rsqrt(r) + 1.0; }
    long long t3 = clock64();
    double q = out[3];
    for (int i = 0; i < n; i++) { q = 1.0 / q + 1.5; }
    long long t4 = clock64();
    if (threadIdx.x == 0 && blockIdx.x == 0) { cyc[0] = t1 - t0; cyc[1] = t2 - t1; cyc[2] = t3 - t2; cyc[3] = t4 - t3; }
    out[4 + threadIdx.x % 4] = a + fa + r + q;
}
__global__ void k_tput(double* out, long long* cyc, int n) {
    double a0 = out[0] + threadIdx.x, a1 = a0 + 1, a2 = a0 + 2, a3 = a0 + 3, a4 = a0 + 4, a5 = a0 + 5, a6 = a0 + 6, a7 = a0 + 7;
    const double b = out[1], c = out[2];
    __syncthreads();
    long long t0 = clock64();
    for (int i = 0; i < n; i++) {
        a0 = fma(a0, b, c); a1 = fma(a1, b, c); a2 = fma(a2, b, c); a3 = fma(a3, b, c);
        a4 = fma(a4, b, c); a5 = fma(a5, b, c); a6 = fma(a6, b, c); a7 = fma(a7, b, c);
    }
    __syncthreads();
    long long t1 = clock64();
    if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
    out[8 + (threadIdx.x & 7)] = a0 + a1 + a2 + a3 + a4 + a5 + a6 + a7;
}
__global__ void k_smem(double* out, long long* cyc, int n) {
    extern __shared__ double sm[];
    for (int i = threadIdx.x; i < 16384; i += blockDim.x) sm[i] = i * 1e-3;
    __syncthreads();
    int idx = threadIdx.x;
    long long t0 = clock64();
    double acc = 0;
    for (int i = 0; i < n; i++) { double v = sm[idx]; idx = ((int)v + idx * 7 + 1) & 16383; acc += v; }   // dependent LDS.64 chain
    long long t1 = clock64();
    for (int i = 0; i < n; i++) { __syncthreads(); }
    long long t2 = clock64();
    if (threadIdx.x == 0) { cyc[0] = t1 - t0; cyc[1] = t2 - t1; }
    out[16 + (threadIdx.x & 3)] = acc;
}
int main() {
    double* d; long long* c; cudaMalloc(&d, 4096); cudaMalloc(&c, 4096);
    double h[8] = {1.0000001, 0.9999999, 1e-9, 2.0, 0, 0, 0, 0}; cudaMemcpy(d, h, sizeof(h), cudaMemcpyHostToDevice);
    long long hc[64];
    const int n = 4096;
    k_lat<<<1, 32>>>(d, c, n); cudaMemcpy(hc, c, 32, cudaMemcpyDeviceToHost);
    printf("latency (cycles/op, 1 warp): DFMA %.1f  FFMA %.1f  rsqrt(double)+add %.1f  1/x(double)+add %.1f\n", hc[0] / (4.0 * n), hc[1] / (4.0 * n), hc[2] / (double)n, hc[3] / (double)n);
    for (int thr : {32, 128, 256, 512, 1024}) {
        k_tput<<<1, thr>>>(d, c, n); cudaMemcpy(hc, c, 8, cudaMemcpyDeviceToHost);
        printf("throughput 1 CTA x %4d thr: %.2f DFMA/clk/SM\n", thr, 8.0 * n * thr / (double)hc[0]);
    }
    cudaFuncSetAttribute(k_smem, cudaFuncAttributeMaxDynamicSharedMemorySize, 180 * 1024);
    for (int thr : {32, 512, 1024}) {
        k_smem<<<1, thr, 16384 * 8>>>(d, c, 2048); cudaMemcpy(hc, c, 16, cudaMemcpyDeviceToHost);
        printf("%4d thr, 128 KB dyn smem: dependent LDS.64 %.1f cycles, __syncthreads %.1f cycles\n", thr, hc[0] / 2048.0, hc[1] / 2048.0);
        k_smem<<<1, thr, 180 * 1024>>>(d, c, 2048); cudaMemcpy(hc, c, 16, cudaMemcpyDeviceToHost);
        printf("%4d thr, 180 KB dyn smem: dependent LDS.64 %.1f cycles, __syncthreads %.1f cycles\n", thr, hc[0] / 2048.0, hc[1] / 2048.0);
    }
    printf("%s\n", cudaGetErrorString(cudaDeviceSynchronize()));
    return 0;
}
