// TEST INFRASTRUCTURE -- fiber scheduler behind tools/cpu_emu/cuda_runtime.h.
// One OS thread; the threads of a block are fibers run round-robin until they block at a
// barrier (__syncthreads, or the two warp barriers inside a shuffle) or finish.  Blocks of a
// grid run one after the other.  A barrier that can never complete aborts with a message.
#include "cuda_runtime.h"
#include <stdio.h>
#include <sys/mman.h>
#include <time.h>
#include <map>
#include <vector>

uint3 threadIdx, blockIdx;
dim3 blockDim, gridDim;
alignas(128) double omg_emu_smem[32768];     // 256 KB

extern "C" void omg_emu_switch(void** save_sp, void* load_sp);
asm(R"(
.text
.globl omg_emu_switch
.type omg_emu_switch,@function
omg_emu_switch:
  pushq %rbp
  pushq %rbx
  pushq %r12
  pushq %r13
  pushq %r14
  pushq %r15
  movq %rsp, (%rdi)
  movq %rsi, %rsp
  popq %r15
  popq %r14
  popq %r13
  popq %r12
  popq %rbx
  popq %rbp
  ret
.size omg_emu_switch,.-omg_emu_switch
)");

namespace {
enum { RUN = 0, WAIT_BLOCK, WAIT_WARP, DONE };
struct Fiber { void* sp; int state; };
const size_t kStack = 512 * 1024;
const int kMaxThreads = 1024;
std::vector<Fiber> fibers;
char* stacks = nullptr;
void* sched_sp = nullptr;
int cur = 0, n_threads = 0, alive = 0, arrived = 0;
int warp_alive[kMaxThreads / 32], warp_arrived[kMaxThreads / 32];
double shfl_slot[kMaxThreads];
const std::function<void()>* body = nullptr;
std::map<const void*, int> max_dyn_smem;     // cudaFuncAttributeMaxDynamicSharedMemorySize per kernel
cudaError_t last_error = cudaSuccess;
const size_t kDefaultDynSmem = 48 * 1024, kOptinDynSmem = 232448;   // H100: 48 KB default, 227 KB opt-in

void yield_to_scheduler() { omg_emu_switch(&fibers[cur].sp, sched_sp); }

void release_block() {
  for (int i = 0; i < n_threads; ++i) if (fibers[i].state == WAIT_BLOCK) fibers[i].state = RUN;
  arrived = 0;
}
void release_warp(int w) {
  for (int i = 32 * w; i < 32 * w + 32 && i < n_threads; ++i) if (fibers[i].state == WAIT_WARP) fibers[i].state = RUN;
  warp_arrived[w] = 0;
}
void warp_barrier() {
  const int w = cur >> 5;
  fibers[cur].state = WAIT_WARP;
  if (++warp_arrived[w] == warp_alive[w]) release_warp(w);
  if (fibers[cur].state != RUN) yield_to_scheduler();
}
void trampoline() {
  (*body)();
  const int w = cur >> 5;
  fibers[cur].state = DONE;
  --alive; --warp_alive[w];
  if (alive > 0 && arrived == alive) release_block();            // exited threads leave the barrier
  if (warp_alive[w] > 0 && warp_arrived[w] == warp_alive[w]) release_warp(w);
  yield_to_scheduler();
  abort();   // a finished fiber is never resumed
}
}  // namespace

void __syncthreads() {
  fibers[cur].state = WAIT_BLOCK;
  if (++arrived == alive) release_block();
  if (fibers[cur].state != RUN) yield_to_scheduler();
}

double __shfl_down_sync(unsigned, double v, int delta) {
  const int me = cur, lane = me & 31;
  shfl_slot[me] = v;
  warp_barrier();
  const double r = (lane + delta < 32 && me + delta < n_threads) ? shfl_slot[me + delta] : v;
  warp_barrier();
  return r;
}

double __shfl_sync(unsigned, double v, int src_lane) {
  const int me = cur, base = me & ~31;
  shfl_slot[me] = v;
  warp_barrier();
  const int src = base + (src_lane & 31);
  const double r = (src < n_threads) ? shfl_slot[src] : v;
  warp_barrier();
  return r;
}

double __shfl_xor_sync(unsigned, double v, int lane_mask) {
  const int me = cur, base = me & ~31;
  shfl_slot[me] = v;
  warp_barrier();
  const int src = base + ((me ^ lane_mask) & 31);
  const double r = (src < n_threads) ? shfl_slot[src] : v;
  warp_barrier();
  return r;
}

long long clock64() {
  timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts);
  return (long long)ts.tv_sec * 1000000000LL + ts.tv_nsec;
}

cudaError_t cudaFuncSetAttribute(const void* kern, cudaFuncAttribute, int value) {
  if (value < 0 || (size_t)value > kOptinDynSmem) return last_error = cudaErrorInvalidValue;
  max_dyn_smem[kern] = value;
  return cudaSuccess;
}

cudaError_t cudaGetLastError() { const cudaError_t e = last_error; last_error = cudaSuccess; return e; }

void omg_emu_launch(const void* kern, int grid, int block, size_t smem_bytes, const std::function<void()>& fn) {
  if (block <= 0 || block > kMaxThreads || (block & 31)) {
    fprintf(stderr, "omg_emu_launch: unsupported launch (block %d, smem %zu)\n", block, smem_bytes); abort(); }
  if (smem_bytes > kDefaultDynSmem) {
    const auto it = max_dyn_smem.find(kern);
    if (it == max_dyn_smem.end() || (size_t)it->second < smem_bytes) { last_error = cudaErrorInvalidValue; return; }
  }
  if (!stacks) {
    stacks = static_cast<char*>(mmap(nullptr, kStack * kMaxThreads, PROT_READ | PROT_WRITE,
                                     MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0));
    if (stacks == MAP_FAILED) { perror("mmap"); abort(); }
  }
  body = &fn; n_threads = block;
  gridDim = dim3(grid); blockDim = dim3(block);
  fibers.assign(block, Fiber{nullptr, RUN});
  for (int b = 0; b < grid; ++b) {
    blockIdx = uint3{(unsigned)b, 0, 0};
    // uninitialised shared memory on the GPU is arbitrary: poison it so that a read before
    // write shows up as NaN instead of a lucky zero
    memset(omg_emu_smem, 0xff, smem_bytes);
    alive = block; arrived = 0;
    for (int w = 0; w < block / 32; ++w) { warp_alive[w] = 32; warp_arrived[w] = 0; }
    for (int i = 0; i < block; ++i) {
      char* top = stacks + kStack * (size_t)(i + 1);           // 16-byte aligned
      void** sp = reinterpret_cast<void**>(top);
      *--sp = nullptr;                                          // fake return address of trampoline
      *--sp = reinterpret_cast<void*>(&trampoline);             // 'ret' target of the first switch
      for (int r = 0; r < 6; ++r) *--sp = nullptr;              // rbp rbx r12 r13 r14 r15
      fibers[i].sp = sp; fibers[i].state = RUN;
    }
    // Schedule: the order in which runnable fibers are resumed between barriers.  A kernel
    // without data races gives bit-identical results for every order; OMG_EMU_SCHED=reverse
    // or =random:<seed> (tests/test_kernel_emulation.py) turns a read that is not separated
    // from the write of another thread by a barrier into a different result.
    std::vector<int> order(block);
    for (int i = 0; i < block; ++i) order[i] = i;
    const char* sched = getenv("OMG_EMU_SCHED");
    const bool reverse = sched && strncmp(sched, "reverse", 7) == 0;
    const bool shuffle = sched && strncmp(sched, "random", 6) == 0;
    unsigned long long rng = 88172645463325252ULL;
    if (shuffle && strchr(sched, ':')) rng ^= strtoull(strchr(sched, ':') + 1, nullptr, 10) * 2654435761ULL + (unsigned)b;
    if (reverse) for (int i = 0; i < block; ++i) order[i] = block - 1 - i;
    while (alive > 0) {
      bool progress = false;
      if (shuffle)
        for (int i = block - 1; i > 0; --i) {
          rng ^= rng << 13; rng ^= rng >> 7; rng ^= rng << 17;
          const int j = (int)(rng % (unsigned long long)(i + 1));
          const int t = order[i]; order[i] = order[j]; order[j] = t;
        }
      for (int oi = 0; oi < block; ++oi) {
        const int i = order[oi];
        if (fibers[i].state != RUN) continue;
        cur = i; threadIdx = uint3{(unsigned)i, 0, 0};
        omg_emu_switch(&sched_sp, fibers[i].sp);
        progress = true;
      }
      if (!progress) {
        fprintf(stderr, "omg_emu: deadlock in block %d: %d threads alive, %d at __syncthreads\n", b, alive, arrived);
        abort();
      }
    }
  }
  body = nullptr;
}

cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = new omg_emu_event{0.0}; return cudaSuccess; }
cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t) { e->t = (double)clock64() * 1e-6; return cudaSuccess; }
cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t a, cudaEvent_t b) { *ms = (float)(b->t - a->t); return cudaSuccess; }
cudaError_t cudaEventDestroy(cudaEvent_t e) { delete e; return cudaSuccess; }
