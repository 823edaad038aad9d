// Latency/throughput microbenchmarks for the fp64 path (single warp / multi warp).
#include <cstdio>
#include <cuda_runtime.h>
__global__ void k_dfma(double* out, long long* cyc, int n) {
  double a = out[0], b = 1.0000001, c = 1e-9;
  long long t0 = clock64();
  for (int i = 0; i < n; ++i) { a = fma(a, b, c); a = fma(a, b, c); a = fma(a, b, c); a = fma(a, b, c); }
  long long t1 = clock64();
  out[threadIdx.x] = a; if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
__global__ void k_dfma_ilp(double* out, long long* cyc, int n) {
  double a0 = out[0], a1 = a0 + 1, a2 = a0 + 2, a3 = a0 + 3, a4 = a0 + 4, a5 = a0 + 5, a6 = a0 + 6, a7 = a0 + 7, b = 1.0000001, c = 1e-9;
  long long t0 = clock64();
  for (int i = 0; i < n; ++i) { a0 = fma(a0, b, c); a1 = fma(a1, b, c); a2 = fma(a2, b, c); a3 = fma(a3, b, c);
    a4 = fma(a4, b, c); a5 = fma(a5, b, c); a6 = fma(a6, b, c); a7 = fma(a7, b, c); }
  long long t1 = clock64();
  out[threadIdx.x] = a0 + a1 + a2 + a3 + a4 + a5 + a6 + a7; if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}
__global__ void k_shfl(double* out, long long* cyc, int n) {
  double a = out[threadIdx.x & 31];
  long long t0 = clock64();
  for (int i = 0; i < n; ++i) { a = __shfl_sync(0xffffffffu, a, (threadIdx.x + 1) & 31); a = __shfl_sync(0xffffffffu, a, (threadIdx.x + 3) & 31);
    a = __shfl_sync(0xffffffffu, a, (threadIdx.x + 5) & 31); a = __shfl_sync(0xffffffffu, a, (threadIdx.x + 7) & 31); }
  long long t1 = clock64();
  out[threadIdx.x] = a; if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
__global__ void k_lds(double* out, long long* cyc, int n) {
  __shared__ int idx[1024];
  for (int i = threadIdx.x; i < 1024; i += blockDim.x) idx[i] = (i * 37 + 11) & 1023;
  __syncthreads();
  int p = threadIdx.x;
  long long t0 = clock64();
  for (int i = 0; i < n; ++i) { p = idx[p]; p = idx[p]; p = idx[p]; p = idx[p]; }
  long long t1 = clock64();
  out[threadIdx.x] = p; if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
__global__ void k_ldg(const int* __restrict__ idx, double* out, long long* cyc, int n) {
  int p = threadIdx.x;
  long long t0 = clock64();
  for (int i = 0; i < n; ++i) { p = idx[p]; p = idx[p]; p = idx[p]; p = idx[p]; }
  long long t1 = clock64();
  out[threadIdx.x] = p; if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
__device__ __forceinline__ double fast_rsqrt(double d) {
  double r = (double)rsqrtf((float)d); const double h = 0.5 * d;
  r = r * (1.5 - h * r * r); r = r * (1.5 - h * r * r); return r; }
__global__ void k_rsqrt(double* out, long long* cyc, int n, int mode) {
  double a = out[0] + 2.0;
  long long t0 = clock64();
  for (int i = 0; i < n; ++i) { if (mode == 0) { a = rsqrt(a) + 1.5; a = rsqrt(a) + 1.5; } else if (mode == 1) { a = fast_rsqrt(a) + 1.5; a = fast_rsqrt(a) + 1.5; }
    else if (mode == 2) { a = sqrt(a) + 1.5; a = sqrt(a) + 1.5; } else { a = 1.0 / a + 1.5; a = 1.0 / a + 1.5; } }
  long long t1 = clock64();
  out[threadIdx.x] = a; if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
__global__ void k_sync(double* out, long long* cyc, int n) {
  long long t0 = clock64();
  for (int i = 0; i < n; ++i) { __syncthreads(); __syncthreads(); __syncthreads(); __syncthreads(); }
  long long t1 = clock64();
  if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
int main() {
  double* out; long long* cyc; int* idx;
  cudaMalloc(&out, 8 * 4096); cudaMalloc(&cyc, 8 * 1024); cudaMalloc(&idx, 4 << 20);
  cudaMemset(out, 0, 8 * 4096);
  int* h = new int[1 << 20]; for (int i = 0; i < (1 << 20); ++i) h[i] = (int)(((long long)i * 7919 + 13) & ((1 << 20) - 1));
  cudaMemcpy(idx, h, 4 << 20, cudaMemcpyHostToDevice);
  long long c; const int n = 2000;
  auto get = [&]() { cudaDeviceSynchronize(); cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost); return (double)c; };
  k_dfma<<<1, 32>>>(out, cyc, n); printf("DFMA dependent latency      : %.1f cyc\n", get() / (4.0 * n));
  k_dfma_ilp<<<1, 32>>>(out, cyc, n); printf("DFMA 1 warp, 8 indep chains : %.2f cyc/instr\n", get() / (8.0 * n));
  k_dfma_ilp<<<1, 256>>>(out, cyc, n); printf("DFMA 8 warps x 8 chains     : %.2f cyc/warp-instr/SM (-> %.1f FMA/clk/SM)\n", get() / (64.0 * n), 32.0 * 64.0 * n / get());
  k_dfma_ilp<<<1, 1024>>>(out, cyc, n); printf("DFMA 32 warps x 8 chains    : %.2f cyc/warp-instr/SM (-> %.1f FMA/clk/SM)\n", get() / (256.0 * n), 32.0 * 256.0 * n / get());
  k_shfl<<<1, 32>>>(out, cyc, n); printf("double shuffle dependent    : %.1f cyc\n", get() / (4.0 * n));
  k_lds<<<1, 32>>>(out, cyc, n); printf("LDS dependent latency       : %.1f cyc\n", get() / (4.0 * n));
  k_ldg<<<1, 32>>>(idx, out, cyc, n); printf("LDG dependent (L2/L1 hit)   : %.1f cyc\n", get() / (4.0 * n));
  for (int m = 0; m < 4; ++m) { k_rsqrt<<<1, 32>>>(out, cyc, n, m); printf("%s + add dependent : %.1f cyc\n", m == 0 ? "rsqrt(double)" : m == 1 ? "fast_rsqrt   " : m == 2 ? "sqrt(double) " : "1.0/x        ", get() / (2.0 * n)); }
  k_sync<<<1, 256>>>(out, cyc, n); printf("__syncthreads (256 thr)     : %.1f cyc\n", get() / (4.0 * n));
  return 0;
}
