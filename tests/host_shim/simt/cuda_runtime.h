// SIMT EMULATOR for tests — <cuda_runtime.h> stand-in that lets g++ compile the product's .cu / .cuh sources unchanged and RUN
// them on the host: tests/build_emulated.py turns every `kernel<<<grid, block, smem, stream>>>(args)` of oxcull.cu into
// simt::Launch(grid, block, smem).go(kernel, args), and this header supplies
//   * the execution model: every CUDA thread of a block is a fiber (ucontext) of one OS thread; fibers run until they reach a
//     block barrier or a warp collective, where they wait for the other participants (cooperative round-robin scheduling, so a
//     warp's lanes exchange values exactly as __shfl_sync / __ballot_sync / __match_any_sync / __reduce_*_sync define); blocks of
//     a grid are distributed over a few OS threads; __shared__ variables are thread_local statics of the block's OS thread;
//     atomics are real atomics;
//   * the runtime API the library calls (cudaMalloc = aligned_alloc, streams and events are no-ops because every operation
//     completes before the call returns, graph capture reports "not supported" so hosts fall back to eager launches, a
//     2-"SM" device so persistent grids stay small).
// Floating point: each __f*_rn intrinsic is one IEEE binary32 operation under -ffp-contract=off (see ../cuda_runtime.h).
// What it is NOT: a model of GPU scheduling, memory ordering or performance — it checks the kernels' LOGIC AND ARITHMETIC in the
// CPU tier; races and hardware behaviour stay with compute-sanitizer and the GPU parity suite.  TEST INFRASTRUCTURE ONLY: the
// product never builds or loads an emulated library (oxylus_b200/ has no reference to it).
#pragma once
#include <ucontext.h>

#include <atomic>
#include <chrono>
#include <climits>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <functional>
#include <thread>
#include <type_traits>
#include <vector>

#include "../cuda_runtime.h"

// ------------------------------------------------------------------------------------------------ execution model
struct dim3 {
  unsigned int x, y, z;
  constexpr dim3(unsigned int x_ = 1, unsigned int y_ = 1, unsigned int z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct uint3 { unsigned int x, y, z; };

namespace simt {

struct Fiber {
  ucontext_t ctx;
  char* stack = nullptr;
  uint3 tid{0, 0, 0};
  unsigned lane = 0, warp = 0;
  bool done = true;
};
struct WarpState {
  unsigned long long slot[32];
  unsigned arrived = 0, read = 0, live = 0, gen = 0;
};
struct BlockState {
  std::vector<Fiber> fibers;
  std::vector<WarpState> warps;
  ucontext_t sched;
  Fiber* cur = nullptr;
  uint3 bid{0, 0, 0};
  dim3 bdim, gdim;
  unsigned live_threads = 0, sync_arrived = 0, sync_gen = 0;
  bool progress = false;
  std::function<void()> body;
};
inline thread_local BlockState* g_block = nullptr;
constexpr size_t FIBER_STACK = 256 * 1024;

inline void yield() { swapcontext(&g_block->cur->ctx, &g_block->sched); }
inline void wait_until(const std::function<bool()>& ready) {
  while (!ready()) yield();
  g_block->progress = true;
}

inline void fiber_entry() {
  BlockState* b = g_block;
  b->body();
  Fiber* f = b->cur;
  f->done = true;
  b->warps[f->warp].live &= ~(1u << f->lane);
  b->live_threads--;
  b->progress = true;
  swapcontext(&f->ctx, &b->sched);
}

inline void run_block(BlockState& b, unsigned n_threads) {
  g_block = &b;
  if (b.fibers.size() < n_threads) b.fibers.resize(n_threads);
  b.warps.assign((n_threads + 31) / 32, WarpState());
  b.live_threads = n_threads; b.sync_arrived = 0; b.sync_gen = 0;
  for (unsigned t = 0; t < n_threads; t++) {
    Fiber& f = b.fibers[t];
    if (!f.stack) f.stack = static_cast<char*>(std::malloc(FIBER_STACK));
    f.tid = uint3{t % b.bdim.x, (t / b.bdim.x) % b.bdim.y, t / (b.bdim.x * b.bdim.y)};
    f.lane = t & 31; f.warp = t >> 5; f.done = false;
    b.warps[f.warp].live |= 1u << f.lane;
    getcontext(&f.ctx);
    f.ctx.uc_stack.ss_sp = f.stack; f.ctx.uc_stack.ss_size = FIBER_STACK; f.ctx.uc_link = nullptr;
    makecontext(&f.ctx, reinterpret_cast<void (*)()>(fiber_entry), 0);
  }
  // OXC_SIMT_ORDER=reverse|shuffle: resume the fibers in another order.  Each fiber runs until it has to wait, so lanes of a warp
  // are as far from lockstep as they can be; changing the order changes who gets ahead of whom.  A kernel that leans on implicit
  // warp-synchronous execution (a shared-memory hand-off without __syncwarp) gives different results under different orders.
  static const int order_mode = [] { const char* e = std::getenv("OXC_SIMT_ORDER"); return !e ? 0 : (e[0] == 'r' ? 1 : 2); }();
  unsigned idle_rounds = 0, round = 0;
  while (b.live_threads) {
    b.progress = false;
    round++;
    for (unsigned i = 0; i < n_threads; i++) {
      unsigned t = i;
      if (order_mode == 1) t = n_threads - 1 - i;
      else if (order_mode == 2) t = (unsigned)(((unsigned long long)i * 2654435761ull + round * 40503ull) % n_threads); // not a permutation every round: fine, it only picks who runs next
      Fiber& f = b.fibers[t];
      if (f.done) continue;
      b.cur = &f;
      swapcontext(&b.sched, &f.ctx);
    }
    idle_rounds = b.progress ? 0 : idle_rounds + 1;
    if (idle_rounds > 4) {
      std::fprintf(stderr, "simt: deadlock in block (%u,%u,%u): %u threads wait for participants that never arrive\n", b.bid.x, b.bid.y, b.bid.z, b.live_threads);
      std::abort();
    }
  }
  b.cur = nullptr;
}

struct Launch {
  dim3 grid, block;
  Launch(dim3 g, dim3 b, size_t /*dynamic shared memory: a fixed thread_local buffer here*/ = 0) : grid(g), block(b) {}
  template <typename K, typename... A>
  void go(K kernel, A... args) const {
    const unsigned n_blocks = grid.x * grid.y * grid.z, n_threads = block.x * block.y * block.z;
    if (!n_blocks || !n_threads) return;
    static const bool trace = std::getenv("OXC_SIMT_TRACE") != nullptr;
    if (trace) std::fprintf(stderr, "simt: launch %p grid (%u,%u,%u) block (%u,%u,%u)\n", (void*)kernel, grid.x, grid.y, grid.z, block.x, block.y, block.z);
    std::atomic<unsigned> next{0};
    auto worker = [&]() {
      static thread_local BlockState state; // fiber stacks are reused by the launches this OS thread serves
      for (unsigned i = next.fetch_add(1); i < n_blocks; i = next.fetch_add(1)) {
        state.bid = uint3{i % grid.x, (i / grid.x) % grid.y, i / (grid.x * grid.y)};
        state.bdim = block; state.gdim = grid;
        state.body = [&]() { kernel(args...); };
        run_block(state, n_threads);
      }
    };
    static const unsigned hw = [] { const char* e = std::getenv("OXC_SIMT_THREADS"); const unsigned n = e ? (unsigned)std::atoi(e) : std::thread::hardware_concurrency(); return n ? n : 1u; }();
    const unsigned n_workers = n_blocks < hw ? n_blocks : hw;
    if (n_workers <= 1) { worker(); return; }
    std::vector<std::thread> pool;
    for (unsigned w = 1; w < n_workers; w++) pool.emplace_back(worker);
    worker();
    for (std::thread& t : pool) t.join();
  }
};

// ---- warp collectives: publish, wait for the participants, combine, wait until everybody has read ----
template <typename F>
inline auto collective(unsigned mask, unsigned long long mine, F combine) {
  BlockState* b = g_block;
  Fiber* f = b->cur;
  WarpState& w = b->warps[f->warp];
  // a partial mask means several groups of the warp run the same collective side by side (__reduce_*_sync(peers, ..) after
  // __match_any_sync): every live lane takes part in the rendezvous, the result only looks at the lane's own group
  const bool partial = mask != 0xffffffffu;
  auto expected = [&]() { return partial ? w.live : (mask & w.live); };
  w.slot[f->lane] = mine;
  w.arrived |= 1u << f->lane;
  wait_until([&]() { return (w.arrived & expected()) == expected(); });
  auto r = combine(w.slot, mask & w.live);
  w.read |= 1u << f->lane;
  if ((w.read & expected()) == expected()) { w.arrived &= ~w.read; w.read = 0; w.gen++; b->progress = true; }
  else { const unsigned g = w.gen; wait_until([&]() { return w.gen != g; }); }
  return r;
}
template <typename T>
inline unsigned long long to_bits(T v) { static_assert(sizeof(T) <= 8, "shuffle payload"); unsigned long long u = 0; memcpy(&u, &v, sizeof(T)); return u; }
template <typename T>
inline T from_bits(unsigned long long u) { T v; memcpy(&v, &u, sizeof(T)); return v; }
inline unsigned lane_id() { return g_block->cur->lane; }

} // namespace simt

#define threadIdx (simt::g_block->cur->tid)
#define blockIdx (simt::g_block->bid)
#define blockDim (simt::g_block->bdim)
#define gridDim (simt::g_block->gdim)

#undef __global__
#define __global__ static __attribute__((unused))
#define __shared__ thread_local /* block-scope thread_local = one instance per OS thread = per running block */

static inline void __syncthreads() {
  simt::BlockState* b = simt::g_block;
  const unsigned g = b->sync_gen;
  if (++b->sync_arrived >= b->live_threads) { b->sync_arrived = 0; b->sync_gen++; b->progress = true; return; }
  simt::wait_until([&]() { return b->sync_gen != g || b->sync_arrived >= b->live_threads; });
  if (b->sync_gen == g) { b->sync_arrived = 0; b->sync_gen++; } // the missing participants exited instead of arriving
}
static inline void __syncwarp(unsigned mask = 0xffffffffu) { simt::collective(mask, 0ull, [](const unsigned long long*, unsigned) { return 0; }); }
template <typename T>
static inline T __shfl_sync(unsigned mask, T v, int src, int width = 32) {
  const unsigned lane = simt::lane_id();
  const unsigned s = (lane & ~(unsigned)(width - 1)) | ((unsigned)src & (unsigned)(width - 1));
  return simt::from_bits<T>(simt::collective(mask, simt::to_bits(v), [s](const unsigned long long* slot, unsigned) { return slot[s]; }));
}
template <typename T>
static inline T __shfl_xor_sync(unsigned mask, T v, int lane_mask, int = 32) {
  const unsigned s = simt::lane_id() ^ (unsigned)lane_mask;
  return simt::from_bits<T>(simt::collective(mask, simt::to_bits(v), [s](const unsigned long long* slot, unsigned) { return slot[s & 31]; }));
}
template <typename T>
static inline T __shfl_up_sync(unsigned mask, T v, unsigned delta, int = 32) {
  const unsigned lane = simt::lane_id();
  return simt::from_bits<T>(simt::collective(mask, simt::to_bits(v), [lane, delta](const unsigned long long* slot, unsigned) { return lane >= delta ? slot[lane - delta] : slot[lane]; }));
}
template <typename T>
static inline T __shfl_down_sync(unsigned mask, T v, unsigned delta, int = 32) {
  const unsigned lane = simt::lane_id();
  return simt::from_bits<T>(simt::collective(mask, simt::to_bits(v), [lane, delta](const unsigned long long* slot, unsigned) { return lane + delta < 32 ? slot[lane + delta] : slot[lane]; }));
}
static inline unsigned __ballot_sync(unsigned mask, bool pred) {
  return simt::collective(mask, pred ? 1ull : 0ull, [](const unsigned long long* slot, unsigned m) { unsigned r = 0; for (int i = 0; i < 32; i++) if ((m >> i & 1) && slot[i]) r |= 1u << i; return r; });
}
static inline bool __any_sync(unsigned mask, bool pred) { return __ballot_sync(mask, pred) != 0; }
static inline bool __all_sync(unsigned mask, bool pred) { return __ballot_sync(mask, !pred) == 0; }
template <typename T>
static inline unsigned __match_any_sync(unsigned mask, T v) {
  const unsigned long long mine = simt::to_bits(v);
  return simt::collective(mask, mine, [mine](const unsigned long long* slot, unsigned m) { unsigned r = 0; for (int i = 0; i < 32; i++) if ((m >> i & 1) && slot[i] == mine) r |= 1u << i; return r; });
}
#define OXC_SIMT_REDUCE(name, init, op)                                                                                     \
  static inline unsigned name(unsigned mask, unsigned v) {                                                                  \
    return simt::collective(mask, (unsigned long long)v, [](const unsigned long long* slot, unsigned m) {                   \
      unsigned r = init;                                                                                                    \
      for (int i = 0; i < 32; i++) if (m >> i & 1) { const unsigned x = (unsigned)slot[i]; r = op; }                        \
      return r; });                                                                                                         \
  }
OXC_SIMT_REDUCE(__reduce_or_sync, 0u, (r | x))
OXC_SIMT_REDUCE(__reduce_add_sync, 0u, (r + x))
OXC_SIMT_REDUCE(__reduce_max_sync, 0u, (r > x ? r : x))
OXC_SIMT_REDUCE(__reduce_min_sync, 0xffffffffu, (r < x ? r : x))
#undef OXC_SIMT_REDUCE
static inline unsigned __activemask() { return simt::g_block->warps[simt::g_block->cur->warp].live; }
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
static inline int __ffs(int v) { return __builtin_ffs(v); }
// a polling loop waits for ANOTHER block / rank (a different OS thread): let that thread run, and do not count the round as a deadlock
static inline void __nanosleep(unsigned) { simt::g_block->progress = true; std::this_thread::yield(); simt::yield(); }
static inline void __threadfence() { std::atomic_thread_fence(std::memory_order_seq_cst); }
static inline void __threadfence_system() { std::atomic_thread_fence(std::memory_order_seq_cst); }
static inline size_t __cvta_generic_to_shared(const void* p) { return (size_t)p; }
static inline unsigned int min(unsigned int a, unsigned int b) { return a < b ? a : b; }
static inline unsigned int max(unsigned int a, unsigned int b) { return a > b ? a : b; }
static inline unsigned long long min(unsigned long long a, unsigned long long b) { return a < b ? a : b; }
static inline unsigned long long max(unsigned long long a, unsigned long long b) { return a > b ? a : b; }
static inline long long min(long long a, long long b) { return a < b ? a : b; }
static inline long long max(long long a, long long b) { return a > b ? a : b; }

// ---- atomics (blocks run on several OS threads) ----
template <typename T>
static inline T atomicAdd(T* p, T v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
template <typename T>
static inline T atomicSub(T* p, T v) { return __atomic_fetch_sub(p, v, __ATOMIC_RELAXED); }
template <typename T>
static inline T atomicOr(T* p, T v) { return __atomic_fetch_or(p, v, __ATOMIC_RELAXED); }
template <typename T>
static inline T atomicXor(T* p, T v) { return __atomic_fetch_xor(p, v, __ATOMIC_RELAXED); }
template <typename T>
static inline T atomicAnd(T* p, T v) { return __atomic_fetch_and(p, v, __ATOMIC_RELAXED); }
template <typename T>
static inline T atomicExch(T* p, T v) { return __atomic_exchange_n(p, v, __ATOMIC_RELAXED); }
template <typename T>
static inline T atomicCAS(T* p, T c, T v) { __atomic_compare_exchange_n(p, &c, v, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED); return c; }
template <typename T>
static inline T atomicMax(T* p, T v) {
  T o = __atomic_load_n(p, __ATOMIC_RELAXED);
  while (o < v && !__atomic_compare_exchange_n(p, &o, v, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
  return o;
}
template <typename T>
static inline T atomicMin(T* p, T v) {
  T o = __atomic_load_n(p, __ATOMIC_RELAXED);
  while (o > v && !__atomic_compare_exchange_n(p, &o, v, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
  return o;
}

// ------------------------------------------------------------------------------------------------ runtime API
typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorMemoryAllocation = 2, cudaErrorNotSupported = 801, cudaErrorInvalidValue = 1 };
typedef struct SimtStream* cudaStream_t;
typedef struct SimtEvent { std::chrono::steady_clock::time_point t; }* cudaEvent_t;
typedef struct SimtGraph* cudaGraph_t;
typedef struct SimtGraphExec* cudaGraphExec_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3, cudaMemcpyDefault = 4 };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2, cudaStreamCaptureModeThreadLocal = 1, cudaIpcMemLazyEnablePeerAccess = 1 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
struct cudaIpcMemHandle_t { char reserved[64]; };
struct cudaDeviceProp { char name[256]; int multiProcessorCount; int major, minor; size_t totalGlobalMem; size_t sharedMemPerBlockOptin; };

static inline const char* cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : e == cudaErrorNotSupported ? "not supported by the SIMT emulator" : "error (SIMT emulator)"; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
static inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp* p, int) {
  memset(p, 0, sizeof *p);
  snprintf(p->name, sizeof p->name, "SIMT emulator (host)");
  p->multiProcessorCount = 2; p->major = 9; p->minor = 0; p->totalGlobalMem = (size_t)8 << 30; p->sharedMemPerBlockOptin = 227 * 1024;
  return cudaSuccess;
}
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
static inline cudaError_t cudaMalloc(void** p, size_t n) { *p = aligned_alloc(256, (n + 255) / 256 * 256 + 256); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
template <typename T>
static inline cudaError_t cudaMalloc(T** p, size_t n) { return cudaMalloc(reinterpret_cast<void**>(p), n); }
static inline cudaError_t cudaFree(void* p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMallocHost(void** p, size_t n) { return cudaMalloc(p, n); }
template <typename T>
static inline cudaError_t cudaMallocHost(T** p, size_t n) { return cudaMalloc(reinterpret_cast<void**>(p), n); }
static inline cudaError_t cudaFreeHost(void* p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { if (n) memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { if (n) memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemset(void* d, int v, size_t n) { if (n) memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t = nullptr) { if (n) memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = reinterpret_cast<cudaStream_t>(new int(0)); return cudaSuccess; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t s) { delete reinterpret_cast<int*>(s); return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
static inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = new SimtEvent(); return cudaSuccess; }
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { return cudaEventCreate(e); }
static inline cudaError_t cudaEventDestroy(cudaEvent_t e) { delete e; return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t = nullptr) { e->t = std::chrono::steady_clock::now(); return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t a, cudaEvent_t b) { *ms = std::chrono::duration<float, std::milli>(b->t - a->t).count(); return cudaSuccess; }
template <typename K>
static inline cudaError_t cudaFuncSetAttribute(K, cudaFuncAttribute, int) { return cudaSuccess; }
template <typename K>
static inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int* n, K, int, size_t) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaStreamBeginCapture(cudaStream_t, int) { return cudaErrorNotSupported; }
static inline cudaError_t cudaStreamEndCapture(cudaStream_t, cudaGraph_t* g) { *g = nullptr; return cudaErrorNotSupported; }
static inline cudaError_t cudaGraphInstantiate(cudaGraphExec_t* e, cudaGraph_t, unsigned long long) { *e = nullptr; return cudaErrorNotSupported; }
static inline cudaError_t cudaGraphDestroy(cudaGraph_t) { return cudaSuccess; }
static inline cudaError_t cudaGraphExecDestroy(cudaGraphExec_t) { return cudaSuccess; }
static inline cudaError_t cudaGraphLaunch(cudaGraphExec_t, cudaStream_t) { return cudaErrorNotSupported; }
// "peer memory": ranks of an emulated multi-GPU run are threads of one process, so a handle is just the address
static inline cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t* h, void* p) { memset(h, 0, sizeof *h); memcpy(h->reserved, &p, sizeof p); return cudaSuccess; }
static inline cudaError_t cudaIpcOpenMemHandle(void** p, cudaIpcMemHandle_t h, unsigned) { memcpy(p, h.reserved, sizeof *p); return cudaSuccess; }
static inline cudaError_t cudaIpcCloseMemHandle(void*) { return cudaSuccess; }
