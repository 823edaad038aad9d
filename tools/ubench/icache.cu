// Instruction-cache capacity: a loop over a straight-line body of S KB of independent integer
// instructions (eight IMAD chains on runtime operands, nothing the compiler can fold), for S from
// 8 to 224 KB.  Cycles per warp instruction from clock64, with one block of 128 threads per SM and
// with four, the four blocks of an SM started a quarter of a body apart so that they walk the code
// at different points, as the sparse solver's blocks do.  While the body fits a cache level the
// cost per instruction is the issue rate; past a level's capacity an LRU cache misses on every line
// of the walk and the cost steps up.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o icache icache.cu && ./icache
#include <cstdio>
#include <cuda_runtime.h>

#define NT 128
#define REPS 64

template <int KB>
__global__ void __launch_bounds__(NT) k_body(const unsigned* __restrict__ in, unsigned* out, long long* cyc,
                                            int* sm_slots, int blocks_per_sm) {
  constexpr int NI = KB * 1024 / 16 / 8;       // 16-byte instructions, eight per step
  unsigned a0 = in[0] + threadIdx.x, a1 = in[1], a2 = in[2], a3 = in[3], a4 = in[4], a5 = in[5], a6 = in[6], a7 = in[7];
  const unsigned m0 = in[8], m1 = in[9], c0 = in[10], c1 = in[11];
  __shared__ int slot;
  if (threadIdx.x == 0) {
    unsigned smid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    slot = atomicAdd(sm_slots + smid, 1) % blocks_per_sm;
  }
  __syncthreads();
  // stagger: block k of an SM starts k/4 of a body later (at least 2 cycles per instruction)
  const long long delay = (long long)slot * (KB * 1024 / 16) * 2 / 4;
  const long long ts = clock64();
  while (clock64() - ts < delay) {}
  const long long t0 = clock64();
  for (int r = 0; r < REPS; ++r) {
#pragma unroll
    for (int o = 0; o < NI / 64; ++o) {      // (one flat loop of more than 1024 steps is not unrolled)
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        const unsigned m = (i & 1) ? m1 : m0, c = (i & 2) ? c1 : c0;
        a0 = a0 * m + c; a1 = a1 * m + c; a2 = a2 * m + c; a3 = a3 * m + c;
        a4 = a4 * m + c; a5 = a5 * m + c; a6 = a6 * m + c; a7 = a7 * m + c;
      }
    }
    asm volatile("" : "+r"(a0), "+r"(a1), "+r"(a2), "+r"(a3), "+r"(a4), "+r"(a5), "+r"(a6), "+r"(a7));
  }
  const long long t1 = clock64();
  out[blockIdx.x * NT + threadIdx.x] = a0 ^ a1 ^ a2 ^ a3 ^ a4 ^ a5 ^ a6 ^ a7;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

template <int KB>
static void run(int n_sm, unsigned* in, unsigned* out, long long* cyc, int* slots) {
  double cpi[2];
  for (int v = 0; v < 2; ++v) {
    const int bps = v ? 4 : 1, nb = n_sm * bps;
    for (int w = 0; w < 2; ++w) {            // the first launch loads the module
      cudaMemset(slots, 0, 4 * 1024);
      k_body<KB><<<nb, NT>>>(in, out, cyc, slots, bps);
    }
    cudaDeviceSynchronize();
    static long long h[4 * 1024];
    cudaMemcpy(h, cyc, 8 * nb, cudaMemcpyDeviceToHost);
    double s = 0.0;
    for (int b = 0; b < nb; ++b) s += (double)h[b];
    cpi[v] = s / nb / ((double)REPS * (KB * 1024 / 16));
  }
  printf("%4d KB   %7.3f   %7.3f\n", KB, cpi[0], cpi[1]);
}

int main() {
  int dev = 0, n_sm = 0;
  cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, dev);
  unsigned *in, *out; long long* cyc; int* slots;
  cudaMalloc(&in, 64); cudaMalloc(&out, 4 * 4 * 1024 * NT); cudaMalloc(&cyc, 8 * 4 * 1024); cudaMalloc(&slots, 4 * 1024);
  const unsigned h_in[12] = {1u, 2u, 3u, 4u, 5u, 6u, 7u, 8u, 0x9e3779b1u, 0x85ebca6bu, 0x165667b1u, 0x27d4eb2fu};
  cudaMemcpy(in, h_in, sizeof(h_in), cudaMemcpyHostToDevice);
  printf("%s, %d SMs; cycles per warp instruction (mean over blocks), %d threads per block\n", prop.name, n_sm, NT);
  printf("body    1 blk/SM  4 blk/SM\n");
  run<8>(n_sm, in, out, cyc, slots);
  run<16>(n_sm, in, out, cyc, slots);
  run<32>(n_sm, in, out, cyc, slots);
  run<48>(n_sm, in, out, cyc, slots);
  run<64>(n_sm, in, out, cyc, slots);
  run<80>(n_sm, in, out, cyc, slots);
  run<96>(n_sm, in, out, cyc, slots);
  run<112>(n_sm, in, out, cyc, slots);
  run<128>(n_sm, in, out, cyc, slots);
  run<144>(n_sm, in, out, cyc, slots);
  run<160>(n_sm, in, out, cyc, slots);
  run<192>(n_sm, in, out, cyc, slots);
  run<224>(n_sm, in, out, cyc, slots);
  const cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { printf("CUDA error: %s\n", cudaGetErrorString(e)); return 1; }
  return 0;
}
