// TEST INFRASTRUCTURE -- not product code, never loaded by omg_tools_b200.
//
// Stand-in for <cuda_runtime.h> that lets omg_tools_b200/csrc/omg_b200.cu compile with g++
// as a *functional CPU emulation* of the CUDA kernels (tools/cpu_emu/README.md): every
// thread of a block is a fiber with its own stack; __syncthreads() and the warp shuffles
// are barriers between fibers, scheduled round-robin on one OS thread (deterministic).
// Device memory is host memory, streams are synchronous.  The point is to execute the
// real kernel source -- table decoding, shared-memory layout, barrier placement, the
// factorisation, the interior-point logic -- in this GPU-less container before spending
// GPU minutes; it says nothing about performance and cannot find data races.
#pragma once
#define OMG_CPU_EMU 1
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <functional>

struct uint3 { unsigned x, y, z; };
struct dim3 { unsigned x, y, z; dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {} };
struct alignas(16) double2 { double x, y; };
struct alignas(8) int2 { int x, y; };
struct alignas(16) int4 { int x, y, z, w; };
struct alignas(16) uint4 { unsigned x, y, z, w; };
struct alignas(8) uint2 { unsigned x, y; };
static inline uint2 make_uint2(unsigned x, unsigned y) { uint2 r; r.x = x; r.y = y; return r; }
static inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { uint4 r; r.x = x; r.y = y; r.z = z; r.w = w; return r; }
static inline double2 make_double2(double x, double y) { double2 r; r.x = x; r.y = y; return r; }
static inline int2 make_int2(int x, int y) { int2 r; r.x = x; r.y = y; return r; }
static inline int4 make_int4(int x, int y, int z, int w) { int4 r; r.x = x; r.y = y; r.z = z; r.w = w; return r; }

// set by the fiber scheduler before a fiber resumes
extern uint3 threadIdx, blockIdx;
extern dim3 blockDim, gridDim;
extern double omg_emu_smem[];      // the running block's dynamic shared memory

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __shared__ static          // blocks run one after the other
#define __align__(n) alignas(n)

#define OMG_DYN_SHARED(name) static double* const name = omg_emu_smem
#define OMG_LAUNCH(kern, grid, block, smem, stream, ...) \
  omg_emu_launch((const void*)(kern), (grid), (block), (size_t)(smem), [&]() { kern(__VA_ARGS__); })

// As on the device, a launch with more than 48 KB of dynamic shared memory fails (the kernel does
// not run, cudaGetLastError reports it) unless cudaFuncSetAttribute(kern,
// cudaFuncAttributeMaxDynamicSharedMemorySize, >= smem) was called for that kernel.
void omg_emu_launch(const void* kern, int grid, int block, size_t smem_bytes, const std::function<void()>& body);
void __syncthreads();
static inline void __threadfence() {}
double __shfl_down_sync(unsigned mask, double v, int delta);
double __shfl_sync(unsigned mask, double v, int src_lane);
double __shfl_xor_sync(unsigned mask, double v, int lane_mask);
long long clock64();
static inline double rsqrt(double x) { return 1.0 / sqrt(x); }
static inline int atomicAdd(int* p, int v) { int o = *p; *p = o + v; return o; }   // one OS thread
template <typename T> static inline T __ldg(const T* p) { return *p; }
static inline double __hiloint2double(int hi, int lo) {
  const uint64_t u = ((uint64_t)(uint32_t)hi << 32) | (uint32_t)lo; double d; memcpy(&d, &u, 8); return d; }
static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }

// ---- runtime API subset used by the host side of omg_b200.cu ----------------------
typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorEmu = 1, cudaErrorInvalidValue = 2 };
typedef void* cudaStream_t;
typedef struct omg_emu_event { double t; }* cudaEvent_t;
enum cudaMemcpyKind { cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice, cudaMemcpyDefault };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize };
struct cudaDeviceProp { int multiProcessorCount; size_t sharedMemPerBlockOptin, sharedMemPerMultiprocessor; };
struct cudaFuncAttributes { size_t sharedSizeBytes; int numRegs; };

template <typename T> static inline cudaError_t cudaMalloc(T** p, size_t n) {
  *p = static_cast<T*>(aligned_alloc(256, ((n ? n : 1) + 255) / 256 * 256)); return *p ? cudaSuccess : cudaErrorEmu; }
static inline cudaError_t cudaFree(void* p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { memcpy(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { memcpy(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemset(void* d, int v, size_t n) { memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t = nullptr) { memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
static inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
static inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp* p, int) {
  // H100 (sm_90a): 227 KB opt-in shared memory per block, 228 KB per SM -- the layout
  // decisions of omg_problem_create (kernel variant, blocks per SM) are the GPU's
  p->multiProcessorCount = 2; p->sharedMemPerBlockOptin = 232448; p->sharedMemPerMultiprocessor = 233472;
  return cudaSuccess; }
static inline cudaError_t cudaFuncGetAttributes(cudaFuncAttributes* a, const void*) { a->sharedSizeBytes = 1024; a->numRegs = 0; return cudaSuccess; }
cudaError_t cudaFuncSetAttribute(const void* kern, cudaFuncAttribute, int value);
static inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int* occ, const void*, int nt, size_t smem) {
  int o = (int)((233472 - 1024) / (smem + 1024)); const int by_threads = 2048 / (nt > 0 ? nt : 1);
  if (o > by_threads) o = by_threads; *occ = o; return cudaSuccess; }
cudaError_t cudaEventCreate(cudaEvent_t* e);
cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t = nullptr);
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t a, cudaEvent_t b);
cudaError_t cudaEventDestroy(cudaEvent_t e);
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
cudaError_t cudaGetLastError();
static inline const char* cudaGetErrorString(cudaError_t e) {
  return e == cudaSuccess ? "no error" : e == cudaErrorInvalidValue ? "invalid argument" : "emulation error"; }
