// Minimal SIMT emulation of the CUDA constructs used by the integer / byte kernels of log_b200 (lgr_bin.cu,
// lgr_shard.cu), so that `-m "not gpu"` tests can execute the REAL kernel source on the CPU.  Test infrastructure only:
// nothing in the product links against this.
//
// Model: one fiber (ucontext) per CUDA thread, CTAs run one after the other on a single OS thread.  A fiber runs until
// it reaches a barrier (__syncthreads / any *_sync warp collective) or returns; barriers release when every LIVE
// thread of the scope has arrived (threads that returned no longer count, as on the GPU).  A barrier nobody can
// complete is reported as a deadlock -- i.e. divergent-barrier bugs fail loudly here.  Scheduling is deterministic;
// atomics are plain read-modify-writes.  Not modelled: memory-model races, warp-synchronous timing, performance.
#pragma once
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <ucontext.h>

#include <functional>
#include <type_traits>
#include <vector>

// ---- optional ThreadSanitizer build (EMU_TSAN): every WARP is a TSan fiber (TSan tracks at most ~250 live threads, fewer than
// the CUDA threads of one CTA, so lanes of a warp share an identity), barriers / kernel boundaries are the only
// happens-before edges, atomics are real atomics -> TSan reports data races between the warps of a CTA (shared AND global
// memory), i.e. a CPU stand-in for compute-sanitizer racecheck (minus intra-warp hazards).  Fiber switches are "no-sync".
#ifdef EMU_TSAN
extern "C" {
void* __tsan_get_current_fiber(void);
void* __tsan_create_fiber(unsigned flags);
void __tsan_destroy_fiber(void* fiber);
void __tsan_switch_to_fiber(void* fiber, unsigned flags);
void __tsan_acquire(void* addr);
void __tsan_release(void* addr);
}
#define EMU_NOTSAN __attribute__((no_sanitize("thread")))
#define EMU_TSAN_ACQUIRE(p) __tsan_acquire((void*)(p))
#define EMU_TSAN_RELEASE(p) __tsan_release((void*)(p))
#else
#define EMU_NOTSAN
#define EMU_TSAN_ACQUIRE(p) ((void)0)
#define EMU_TSAN_RELEASE(p) ((void)0)
#endif

#define __global__
#define __device__
#define __host__
#define __constant__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)
#define __shared__ static
#define __align__(n) __attribute__((aligned(n)))

struct dim3 {
  unsigned x, y, z;
  dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct alignas(8) float2 { float x, y; };
struct alignas(16) float4 { float x, y, z, w; };
struct alignas(16) int4 { int x, y, z, w; };
inline int4 make_int4(int x, int y, int z, int w) { return int4{x, y, z, w}; }
inline float2 make_float2(float x, float y) { return float2{x, y}; }
inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }

typedef void* cudaStream_t;
typedef void* cudaEvent_t;
typedef int cudaError_t;
enum { cudaSuccess = 0 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
inline cudaError_t cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t) { memset(p, v, n); return cudaSuccess; }
template <class F> inline cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute, int) { return cudaSuccess; }
inline cudaError_t cudaEventCreate(cudaEvent_t*) { return cudaSuccess; }
inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t, cudaEvent_t) { *ms = 0.f; return cudaSuccess; }

namespace emu {

enum State { READY = 0, WAIT_CTA, WAIT_WARP, DONE };

struct Fiber {
  ucontext_t ctx;
  char* stack = nullptr;
  dim3 tid;
  int state = READY;
  void* tsan = nullptr;
};

struct Cta {
  Fiber* fibers = nullptr;
  int nthreads = 0, alive = 0, cta_waiting = 0;
  int warp_alive[32], warp_waiting[32];
  struct Slot { unsigned long long u[4]; };
  Slot scratch[32][32];                 // [warp][lane] exchange slots of the warp collectives (up to 32 bytes per lane)
  int cta_acc = 0;                       // __syncthreads_or / _and / _count accumulator
  int cta_gen = 0, warp_gen[32];         // barrier generations (TSan: alternating sync objects)
  char cta_sync[2], warp_sync[32][2], launch_sync, done_sync;
  void* sched_tsan = nullptr;
  void* warp_tsan[32];
  int cta_result = 0;
  std::function<void()> body;
  dim3 block_idx, block_dim, grid_dim;
  char* dyn = nullptr;
};

inline Cta*& cta() { static Cta* c = nullptr; return c; }
inline Fiber*& cur() { static Fiber* f = nullptr; return f; }
inline ucontext_t& sched_ctx() { static ucontext_t c; return c; }
inline void* dyn_smem() { return cta()->dyn; }

EMU_NOTSAN inline void yield() {
#ifdef EMU_TSAN
  __tsan_switch_to_fiber(cta()->sched_tsan, 1);
#endif
  swapcontext(&cur()->ctx, &sched_ctx());
}

EMU_NOTSAN inline void release_cta(Cta* c) {
  for (int t = 0; t < c->nthreads; t++) if (c->fibers[t].state == WAIT_CTA) c->fibers[t].state = READY;
  c->cta_waiting = 0;
}
EMU_NOTSAN inline void release_warp(Cta* c, int w) {
  for (int l = 0; l < 32 && w * 32 + l < c->nthreads; l++)
    if (c->fibers[w * 32 + l].state == WAIT_WARP) c->fibers[w * 32 + l].state = READY;
  c->warp_waiting[w] = 0;
}

EMU_NOTSAN inline void barrier_cta() {
  Cta* c = cta();
  char* sync = &c->cta_sync[c->cta_gen & 1];
  EMU_TSAN_RELEASE(sync);
  if (++c->cta_waiting == c->alive) { c->cta_gen++; release_cta(c); EMU_TSAN_ACQUIRE(sync); return; }
  cur()->state = WAIT_CTA;
  yield();
  EMU_TSAN_ACQUIRE(sync);
}
EMU_NOTSAN inline void barrier_warp() {
  Cta* c = cta();
  const int w = cur()->tid.x >> 5;
  char* sync = &c->warp_sync[w][c->warp_gen[w] & 1];
  EMU_TSAN_RELEASE(sync);
  if (++c->warp_waiting[w] == c->warp_alive[w]) { c->warp_gen[w]++; release_warp(c, w); EMU_TSAN_ACQUIRE(sync); return; }
  cur()->state = WAIT_WARP;
  yield();
  EMU_TSAN_ACQUIRE(sync);
}

EMU_NOTSAN inline void fiber_entry() {
  Cta* c = cta();
  EMU_TSAN_ACQUIRE(&c->launch_sync);
  c->body();
  EMU_TSAN_RELEASE(&c->done_sync);
  Fiber* f = cur();
  f->state = DONE;
  const int w = f->tid.x >> 5;
  c->alive--; c->warp_alive[w]--;
  if (c->cta_waiting > 0 && c->cta_waiting == c->alive) { c->cta_gen++; release_cta(c); }
  if (c->warp_waiting[w] > 0 && c->warp_waiting[w] == c->warp_alive[w]) { c->warp_gen[w]++; release_warp(c, w); }
#ifdef EMU_TSAN
  __tsan_switch_to_fiber(c->sched_tsan, 1);
#endif
  swapcontext(&f->ctx, &sched_ctx());
}

constexpr size_t STACK = 192 * 1024;

template <class F>
EMU_NOTSAN inline void launch(dim3 grid, dim3 block, size_t smem, F fn) {
  if (grid.y != 1 || grid.z != 1 || block.y != 1 || block.z != 1) { fprintf(stderr, "emu: 1-D launches only\n"); abort(); }
  Cta c;
  c.nthreads = (int)block.x;
  std::vector<Fiber> storage(c.nthreads);
  c.fibers = storage.data();
  for (int t = 0; t < c.nthreads; t++) c.fibers[t].stack = (char*)malloc(STACK);
  std::vector<char> dyn(smem + 64);
  c.dyn = (char*)(((uintptr_t)dyn.data() + 63) & ~(uintptr_t)63);
  c.block_dim = block; c.grid_dim = grid;
  c.body = fn;
  cta() = &c;
#ifdef EMU_TSAN
  c.sched_tsan = __tsan_get_current_fiber();
#endif
  EMU_TSAN_RELEASE(&c.launch_sync);
  for (unsigned b = 0; b < grid.x; b++) {
    c.block_idx = dim3(b);
    c.alive = c.nthreads; c.cta_waiting = 0; c.cta_acc = 0; c.cta_gen = 0;
    for (int w = 0; w < 32; w++) { c.warp_waiting[w] = 0; c.warp_alive[w] = 0; c.warp_gen[w] = 0; }
    for (int t = 0; t < c.nthreads; t++) {
      Fiber& f = c.fibers[t];
      f.tid = dim3((unsigned)t); f.state = READY;
      c.warp_alive[t >> 5]++;
      getcontext(&f.ctx);
      f.ctx.uc_stack.ss_sp = f.stack; f.ctx.uc_stack.ss_size = STACK; f.ctx.uc_link = nullptr;
      makecontext(&f.ctx, (void (*)())fiber_entry, 0);
    }
#ifdef EMU_TSAN
    for (int w = 0; w * 32 < c.nthreads; w++) c.warp_tsan[w] = __tsan_create_fiber(0);
    for (int t = 0; t < c.nthreads; t++) c.fibers[t].tsan = c.warp_tsan[t >> 5];
#endif
    while (c.alive > 0) {
      bool ran = false;
      // EMU_SCHED_SEED=<n> in the environment: visit the runnable threads in a different pseudo-random order on every pass
      // (default: ascending thread id).  Results must not depend on it beyond floating-point summation order.
      static const char* seed_env = getenv("EMU_SCHED_SEED");
      static unsigned long long rng = seed_env ? 0x9E3779B97F4A7C15ull * (1 + strtoull(seed_env, nullptr, 10)) : 0;
      unsigned start = 0, stride = 1;
      if (seed_env) {
        rng ^= rng << 13; rng ^= rng >> 7; rng ^= rng << 17;
        start = (unsigned)(rng % (unsigned)c.nthreads);
        stride = 1 + 2 * (unsigned)((rng >> 32) % 64);                 // odd stride: a permutation of a power-of-two thread count
        if (c.nthreads & (c.nthreads - 1)) stride = 1;                 // not a power of two: just rotate
      }
      for (int k = 0; k < c.nthreads; k++) {
        const int t = (int)((start + (unsigned long long)k * stride) % (unsigned)c.nthreads);
        Fiber& f = c.fibers[t];
        if (f.state != READY) continue;
        ran = true;
        cur() = &f;
#ifdef EMU_TSAN
        __tsan_switch_to_fiber(f.tsan, 1);
#endif
        swapcontext(&sched_ctx(), &f.ctx);
      }
      if (!ran) {
        fprintf(stderr, "emu: DEADLOCK in block %u: %d threads alive, %d at __syncthreads", b, c.alive, c.cta_waiting);
        for (int w = 0; w < 32; w++) if (c.warp_waiting[w]) fprintf(stderr, "; warp %d: %d of %d at a warp collective", w, c.warp_waiting[w], c.warp_alive[w]);
        fprintf(stderr, "\n");
        abort();
      }
    }
#ifdef EMU_TSAN
    for (int w = 0; w * 32 < c.nthreads; w++) __tsan_destroy_fiber(c.warp_tsan[w]);
    // The next CTA reuses the same __shared__ storage, so by default it is ordered after this one; races BETWEEN CTAs on
    // global memory are then not reported (compute-sanitizer racecheck does not look at global memory either).
    // EMU_TSAN_UNORDERED_CTAS leaves the CTAs of a launch concurrent: global-memory races between CTAs are reported, and so
    // is every reuse of the emulated shared storage -- filter those reports by location (tests/emu/README.md).
#ifndef EMU_TSAN_UNORDERED_CTAS
    EMU_TSAN_ACQUIRE(&c.done_sync);
    EMU_TSAN_RELEASE(&c.launch_sync);
#endif
#endif
  }
  EMU_TSAN_ACQUIRE(&c.done_sync);
  for (int t = 0; t < c.nthreads; t++) free(c.fibers[t].stack);
  cta() = nullptr; cur() = nullptr;
}

// ---- warp collectives -------------------------------------------------------------------------------------------
EMU_NOTSAN inline int lane_id() { return cur()->tid.x & 31; }
EMU_NOTSAN inline int warp_id() { return cur()->tid.x >> 5; }
EMU_NOTSAN inline bool lane_alive(int l) {
  Cta* c = cta();
  const int t = warp_id() * 32 + l;
  return t < c->nthreads && c->fibers[t].state != DONE;
}
template <class T> EMU_NOTSAN inline void publish(T v) {
  static_assert(sizeof(T) <= sizeof(Cta::Slot), "collective payload");
  Cta::Slot u = {{0, 0, 0, 0}}; memcpy(&u, &v, sizeof(T));
  cta()->scratch[warp_id()][lane_id()] = u;
  barrier_warp();
}
template <class T> EMU_NOTSAN inline T peek(int l) { T v; memcpy(&v, &cta()->scratch[warp_id()][l], sizeof(T)); return v; }
}  // namespace emu

#define threadIdx (emu::cur()->tid)
#define blockIdx (emu::cta()->block_idx)
#define blockDim (emu::cta()->block_dim)
#define gridDim (emu::cta()->grid_dim)

inline void __syncthreads() { emu::barrier_cta(); }
inline void __syncwarp(unsigned = 0xffffffffu) { emu::barrier_warp(); }
inline void __trap() { fprintf(stderr, "emu: __trap()\n"); abort(); }

// LGR_ON_LSD_FALLBACK() in lgr_bin.cu (defined by build_emu.py): lists whose MSD work stack overflowed, so that a test can
// prove it reached the LSD sort
inline long long& emu_lsd_fallbacks() { static long long n = 0; return n; }
inline void emu_count_lsd_fallback() { if (threadIdx.x == 0) emu_lsd_fallbacks()++; }

EMU_NOTSAN inline int __syncthreads_reduce(int pred, int mode) {   // 0 or, 1 and, 2 count
  emu::Cta* c = emu::cta();
  // phase 1: everybody contributes
  if (c->cta_waiting == 0) c->cta_acc = (mode == 1) ? 1 : 0;
  if (mode == 0) c->cta_acc |= (pred != 0); else if (mode == 1) c->cta_acc &= (pred != 0); else c->cta_acc += (pred != 0);
  emu::barrier_cta();
  const int r = c->cta_acc;
  emu::barrier_cta();          // nobody starts the next reduction before everyone has read this one
  return r;
}
inline int __syncthreads_or(int p) { return __syncthreads_reduce(p, 0); }
inline int __syncthreads_and(int p) { return __syncthreads_reduce(p, 1); }
inline int __syncthreads_count(int p) { return __syncthreads_reduce(p, 2); }

inline unsigned __ballot_sync(unsigned, int pred) {
  emu::publish<unsigned>(pred ? 1u : 0u);
  unsigned r = 0;
  for (int l = 0; l < 32; l++) if (emu::lane_alive(l) && emu::peek<unsigned>(l)) r |= 1u << l;
  emu::barrier_warp();
  return r;
}
inline int __all_sync(unsigned m, int pred) {
  emu::publish<unsigned>(pred ? 1u : 0u);
  int r = 1;
  for (int l = 0; l < 32; l++) if (emu::lane_alive(l) && !emu::peek<unsigned>(l)) r = 0;
  emu::barrier_warp();
  return r;
}
inline int __any_sync(unsigned m, int pred) { return __ballot_sync(m, pred) != 0; }
template <class T> inline T __shfl_sync(unsigned, T v, int src) {
  emu::publish<T>(v);
  const T r = emu::peek<T>(src & 31);
  emu::barrier_warp();
  return r;
}
template <class T> inline T __shfl_up_sync(unsigned, T v, unsigned d) {
  emu::publish<T>(v);
  const int l = emu::lane_id();
  const T r = l >= (int)d ? emu::peek<T>(l - (int)d) : v;
  emu::barrier_warp();
  return r;
}
template <class T> inline T __shfl_down_sync(unsigned, T v, unsigned d) {
  emu::publish<T>(v);
  const int l = emu::lane_id();
  const T r = l + (int)d < 32 ? emu::peek<T>(l + (int)d) : v;
  emu::barrier_warp();
  return r;
}
template <class T> inline T __shfl_xor_sync(unsigned, T v, int m) {
  emu::publish<T>(v);
  const T r = emu::peek<T>((emu::lane_id() ^ m) & 31);
  emu::barrier_warp();
  return r;
}
inline unsigned __match_any_sync(unsigned, unsigned v) {
  emu::publish<unsigned>(v);
  unsigned r = 0;
  for (int l = 0; l < 32; l++) if (emu::lane_alive(l) && emu::peek<unsigned>(l) == v) r |= 1u << l;
  emu::barrier_warp();
  return r;
}
template <class T> inline T emu_reduce(T v, int op) {
  emu::publish<T>(v);
  T r = v; bool first = true;
  for (int l = 0; l < 32; l++) if (emu::lane_alive(l)) {
    const T x = emu::peek<T>(l);
    if (first) { r = x; first = false; } else r = op == 0 ? (T)(r + x) : (x > r ? x : r);
  }
  emu::barrier_warp();
  return r;
}
inline unsigned __reduce_add_sync(unsigned, unsigned v) { return emu_reduce<unsigned>(v, 0); }
inline int __reduce_add_sync(unsigned, int v) { return emu_reduce<int>(v, 0); }
inline unsigned __reduce_max_sync(unsigned, unsigned v) { return emu_reduce<unsigned>(v, 1); }
inline int __reduce_max_sync(unsigned, int v) { return emu_reduce<int>(v, 1); }

// ---- scalar intrinsics ------------------------------------------------------------------------------------------
inline int __popc(unsigned x) { return __builtin_popcount(x); }
inline int __ffs(int x) { return __builtin_ffs(x); }
inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
inline int __clzll(long long x) { return x ? __builtin_clzll((unsigned long long)x) : 64; }
inline float __int_as_float(int i) { float f; memcpy(&f, &i, 4); return f; }
inline int __float_as_int(float f) { int i; memcpy(&i, &f, 4); return i; }
inline unsigned __float_as_uint(float f) { unsigned i; memcpy(&i, &f, 4); return i; }
inline float __uint_as_float(unsigned i) { float f; memcpy(&f, &i, 4); return f; }
inline float __fdividef(float a, float b) { return a / b; }
template <class T> inline T __ldg(const T* p) { return *p; }

// relaxed atomics, like the device's: no ordering of other data
template <class T> inline T atomicAdd(T* p, T v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
inline float atomicAdd(float* p, float v) {
  uint32_t* u = reinterpret_cast<uint32_t*>(p);
  uint32_t o = __atomic_load_n(u, __ATOMIC_RELAXED), n;
  float f;
  do { memcpy(&f, &o, 4); f += v; memcpy(&n, &f, 4); } while (!__atomic_compare_exchange_n(u, &o, n, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED));
  memcpy(&f, &o, 4);
  return f;
}
inline int atomicAdd(int* p, unsigned v) { return __atomic_fetch_add(p, (int)v, __ATOMIC_RELAXED); }
template <class T> inline T atomicOr(T* p, T v) { return __atomic_fetch_or(p, v, __ATOMIC_RELAXED); }
template <class T> inline T atomicMax(T* p, T v) {
  T o = __atomic_load_n(p, __ATOMIC_RELAXED);
  while (v > o && !__atomic_compare_exchange_n(p, &o, v, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
  return o;
}

#define EMU_MINMAX(T)                                   \
  inline T min(T a, T b) { return b < a ? b : a; }      \
  inline T max(T a, T b) { return a < b ? b : a; }
EMU_MINMAX(int)
EMU_MINMAX(unsigned)
EMU_MINMAX(long long)
EMU_MINMAX(unsigned long long)
EMU_MINMAX(long)
EMU_MINMAX(unsigned long)
EMU_MINMAX(float)
#undef EMU_MINMAX
inline long long min(long long a, int b) { return a < b ? a : b; }
inline long long min(int a, long long b) { return a < b ? a : b; }
inline long min(long a, int b) { return a < b ? a : b; }
inline long min(int a, long b) { return a < b ? a : b; }
inline long long max(long long a, int b) { return a < b ? (long long)b : a; }
inline long max(long a, int b) { return a < b ? (long)b : a; }

// ---- float intrinsics (correctly rounded on the host as on the device) --------------------------------------------
inline float __fmul_rn(float a, float b) { return a * b; }
inline float __fadd_rn(float a, float b) { return a + b; }
inline float __fsub_rn(float a, float b) { return a - b; }
inline float __fdiv_rn(float a, float b) { return a / b; }
inline float __fsqrt_rn(float a) { return sqrtf(a); }
inline float __fmaf_rn(float a, float b, float c) { return fmaf(a, b, c); }
inline float4 atomicAdd(float4* p, float4 v) {
  float4 o;
  o.x = atomicAdd(&p->x, v.x); o.y = atomicAdd(&p->y, v.y); o.z = atomicAdd(&p->z, v.z); o.w = atomicAdd(&p->w, v.w);
  return o;
}
