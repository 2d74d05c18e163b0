// tests/emu/cuda_runtime.h -- CPU interpreter for the slice of CUDA that mesh_navigation_b200/csrc uses.
//
// TEST INFRASTRUCTURE ONLY.  This header lets g++ compile the *unchanged* kernel sources (meshnav.cu,
// band_engine.cuh, problems.cuh) into tests/emu/libmeshnav_emu.so so that the `-m "not gpu"` test-suite can run the
// kernels' control flow -- the band engine, the sub-warp replay, the in-round sweeps, the warp-parallel back-tracking --
// against the oracle on small meshes without a GPU.  It is never linked into libmeshnav_b200.so, never loaded by the
// mesh_navigation_b200 package, and is not a fallback: it is 1000x slower than the device and exists to catch logic
// regressions before GPU time is spent.
//
// Execution model
//   * one CUDA thread = one fiber (hand-rolled x86-64 context switch); fibers of a CTA are scheduled cooperatively in
//     one OS process and switch only at warp collectives and barriers, so a warp behaves like 32 lock-step lanes at
//     exactly the points where CUDA requires convergence (full-mask *_sync intrinsics, __syncthreads);
//   * `__shared__` = function-local static: one instance per process;
//   * kernels that need inter-CTA synchronisation (cooperative launch / clusters) run one forked PROCESS per CTA;
//     "device memory" is a MAP_SHARED arena, global atomics are real atomics, grid / cluster barriers are
//     sense-reversing barriers in the arena.  Other launches run their CTAs one after the other in the caller;
//   * memory-ordering bugs (missing fences) are NOT modelled: x86 is TSO and fibers are sequential inside a CTA.
#pragma once
#ifndef __x86_64__
#error "tests/emu needs x86-64 (hand-written context switch)"
#endif
#include <sched.h>
#include <signal.h>
#include <sys/mman.h>
#include <sys/prctl.h>
#include <sys/wait.h>
#include <unistd.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <numeric>
#include <stdexcept>
#include <string>
#include <tuple>
#include <unordered_map>
#include <utility>
#include <vector>
#include <emmintrin.h>
#include <x86intrin.h>

#define MNB_EMU_ACTIVE 1

// ---- qualifiers ----------------------------------------------------------------------------------------------------
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline __attribute__((always_inline))
#define __noinline__ __attribute__((noinline))
#define __launch_bounds__(...)
#define __align__(n) __attribute__((aligned(n)))
#define __shared__ static

// ---- vector types --------------------------------------------------------------------------------------------------
struct __attribute__((aligned(8))) uint2 { unsigned int x, y; };
struct __attribute__((aligned(16))) uint4 { unsigned int x, y, z, w; };
struct __attribute__((aligned(8))) int2 { int x, y; };
struct __attribute__((aligned(16))) int4 { int x, y, z, w; };
struct __attribute__((aligned(8))) float2 { float x, y; };
struct float3 { float x, y, z; };
struct __attribute__((aligned(16))) float4 { float x, y, z, w; };
struct __attribute__((aligned(16))) double2 { double x, y; };
struct __attribute__((aligned(16))) double4 { double x, y, z, w; };
struct uint3 { unsigned int x, y, z; };
static inline uint2 make_uint2(unsigned x, unsigned y) { return uint2{x, y}; }
static inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { return uint4{x, y, z, w}; }
static inline int4 make_int4(int x, int y, int z, int w) { return int4{x, y, z, w}; }
static inline float2 make_float2(float x, float y) { return float2{x, y}; }
static inline float3 make_float3(float x, float y, float z) { return float3{x, y, z}; }
static inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
static inline double2 make_double2(double x, double y) { return double2{x, y}; }
static inline double4 make_double4(double x, double y, double z, double w) { return double4{x, y, z, w}; }
struct dim3 {
  unsigned int x, y, z;
  dim3(unsigned int x_ = 1, unsigned int y_ = 1, unsigned int z_ = 1) : x(x_), y(y_), z(z_) {}
};

// built-in coordinates: plain globals, rewritten by the scheduler whenever a fiber / CTA is switched in
inline uint3 threadIdx{0, 0, 0}, blockIdx{0, 0, 0}, blockDim{1, 1, 1}, gridDim{1, 1, 1};

// ---- scalar helpers --------------------------------------------------------------------------------------------------
using std::isfinite;
using std::isinf;
using std::isnan;
static inline unsigned int __float_as_uint(float f) { unsigned int u; std::memcpy(&u, &f, 4); return u; }
static inline float __uint_as_float(unsigned int u) { float f; std::memcpy(&f, &u, 4); return f; }
static inline int __float_as_int(float f) { int u; std::memcpy(&u, &f, 4); return u; }
static inline float __int_as_float(int u) { float f; std::memcpy(&f, &u, 4); return f; }
static inline float __fadd_rn(float a, float b) { volatile float r = a + b; return r; }
static inline float __fmul_rn(float a, float b) { volatile float r = a * b; return r; }
static inline int __popc(unsigned int x) { return __builtin_popcount(x); }
static inline int __ffs(int x) { return __builtin_ffs(x); }
static inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
static inline int __clzll(long long x) { return x ? __builtin_clzll((unsigned long long)x) : 64; }
static inline long long clock64() { return (long long)__rdtsc(); }
static inline int min(int a, int b) { return a < b ? a : b; }
static inline unsigned int min(unsigned int a, unsigned int b) { return a < b ? a : b; }
static inline long long min(long long a, long long b) { return a < b ? a : b; }
static inline unsigned long long min(unsigned long long a, unsigned long long b) { return a < b ? a : b; }
static inline unsigned long min(unsigned long a, unsigned long b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }
static inline unsigned int max(unsigned int a, unsigned int b) { return a > b ? a : b; }
static inline long long max(long long a, long long b) { return a > b ? a : b; }
static inline unsigned long long max(unsigned long long a, unsigned long long b) { return a > b ? a : b; }
static inline unsigned long max(unsigned long a, unsigned long b) { return a > b ? a : b; }

// ---- memory access intrinsics: device memory is ordinary (shared) memory; 16-byte words move as one SSE access ----------
namespace emu {
template <class T> struct is16 : std::integral_constant<bool, sizeof(T) == 16 && alignof(T) >= 16> {};
template <class T>
static inline T load_once(const T* p) {
  if constexpr (is16<T>::value) {
    __m128i v = _mm_load_si128(reinterpret_cast<const __m128i*>(p));
    T r; std::memcpy(&r, &v, 16); return r;
  } else if constexpr (sizeof(T) == 4) {
    uint32_t v = __atomic_load_n(reinterpret_cast<const uint32_t*>(p), __ATOMIC_RELAXED); T r; std::memcpy(&r, &v, 4); return r;
  } else if constexpr (sizeof(T) == 8) {
    uint64_t v = __atomic_load_n(reinterpret_cast<const uint64_t*>(p), __ATOMIC_RELAXED); T r; std::memcpy(&r, &v, 8); return r;
  } else {
    return *reinterpret_cast<const volatile T*>(p);
  }
}
template <class T>
static inline void store_once(T* p, const T& v) {
  if constexpr (is16<T>::value) {
    __m128i x; std::memcpy(&x, &v, 16); _mm_store_si128(reinterpret_cast<__m128i*>(p), x);
  } else if constexpr (sizeof(T) == 4) {
    uint32_t x; std::memcpy(&x, &v, 4); __atomic_store_n(reinterpret_cast<uint32_t*>(p), x, __ATOMIC_RELAXED);
  } else if constexpr (sizeof(T) == 8) {
    uint64_t x; std::memcpy(&x, &v, 8); __atomic_store_n(reinterpret_cast<uint64_t*>(p), x, __ATOMIC_RELAXED);
  } else {
    *reinterpret_cast<volatile T*>(p) = v;
  }
}
}  // namespace emu
template <class T> static inline T __ldg(const T* p) { return emu::load_once(p); }
template <class T> static inline T __ldcg(const T* p) { return emu::load_once(p); }
template <class T> static inline T __ldca(const T* p) { return emu::load_once(p); }
template <class T> static inline T __ldcs(const T* p) { return emu::load_once(p); }
template <class T> static inline void __stcg(T* p, const T& v) { emu::store_once(p, v); }
template <class T> static inline void __stcs(T* p, const T& v) { emu::store_once(p, v); }
static inline void __threadfence() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
static inline void __threadfence_block() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }

// ---- atomics -------------------------------------------------------------------------------------------------------
template <class T> static inline T atomicAdd(T* p, T v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline float atomicAdd(float* p, float v) {
  uint32_t* u = reinterpret_cast<uint32_t*>(p); uint32_t old = __atomic_load_n(u, __ATOMIC_RELAXED);
  for (;;) { const uint32_t nw = __float_as_uint(__uint_as_float(old) + v); if (__atomic_compare_exchange_n(u, &old, nw, false, __ATOMIC_SEQ_CST, __ATOMIC_RELAXED)) return __uint_as_float(old); }
}
static inline double atomicAdd(double* p, double v) {
  uint64_t* u = reinterpret_cast<uint64_t*>(p); uint64_t old = __atomic_load_n(u, __ATOMIC_RELAXED);
  for (;;) { double o; __builtin_memcpy(&o, &old, 8); const double nv = o + v; uint64_t nw; __builtin_memcpy(&nw, &nv, 8);
             if (__atomic_compare_exchange_n(u, &old, nw, false, __ATOMIC_SEQ_CST, __ATOMIC_RELAXED)) return o; }
}
template <class T> static inline T atomicSub(T* p, T v) { return __atomic_fetch_sub(p, v, __ATOMIC_SEQ_CST); }
template <class T> static inline T atomicOr(T* p, T v) { return __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST); }
template <class T> static inline T atomicAnd(T* p, T v) { return __atomic_fetch_and(p, v, __ATOMIC_SEQ_CST); }
template <class T> static inline T atomicExch(T* p, T v) { return __atomic_exchange_n(p, v, __ATOMIC_SEQ_CST); }
template <class T> static inline T atomicCAS(T* p, T cmp, T v) { __atomic_compare_exchange_n(p, &cmp, v, false, __ATOMIC_SEQ_CST, __ATOMIC_RELAXED); return cmp; }
template <class T> static inline T atomicMin(T* p, T v) {
  T old = __atomic_load_n(p, __ATOMIC_RELAXED);
  while (v < old && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_SEQ_CST, __ATOMIC_RELAXED)) {}
  return old;
}
template <class T> static inline T atomicMax(T* p, T v) {
  T old = __atomic_load_n(p, __ATOMIC_RELAXED);
  while (v > old && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_SEQ_CST, __ATOMIC_RELAXED)) {}
  return old;
}

// ====================================================================================================================
// fibers, warps, CTAs
// ====================================================================================================================
extern "C" void mnb_emu_switch(void** save_sp, void* load_sp);
asm(R"ASM(
.text
.globl mnb_emu_switch
.type mnb_emu_switch,@function
mnb_emu_switch:
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
.size mnb_emu_switch,.-mnb_emu_switch
)ASM");

namespace emu {

constexpr int MAX_THREADS = 1024;
constexpr size_t STACK_BYTES = 256 * 1024;
enum { F_RUNNABLE = 0, F_WAIT_WARP = 1, F_WAIT_CTA = 2, F_DONE = 3 };

struct Fiber { void* sp; int tid; int state; unsigned wait_gen; };
struct Warp { unsigned arrived, gen, alive; unsigned part[2]; uint64_t slot[2][32]; };   // part: lanes that took part in the collective of that buffer
struct ProcBarrier { unsigned count, gen, n, pad; };
struct LaunchCtl {                 // lives in the shared arena, one per forked launch
  ProcBarrier grid;
  ProcBarrier cluster[64];
  int abort_flag;
};
struct Cta {
  int nthreads, alive;
  unsigned bar_arrived, bar_gen;
  Warp warps[MAX_THREADS / 32];
  Fiber fibers[MAX_THREADS];
  void* sched_sp;
  Fiber* cur;
  void (*invoke)(void*);
  void* invoke_ctx;
  unsigned char* dyn_smem;
  LaunchCtl* lc;                   // null for sequential launches
  unsigned cluster_size, cluster_id;
};
inline Cta g_cta;
inline char* g_stacks = nullptr;   // MAX_THREADS stacks, mapped once (children inherit them copy-on-write)
inline unsigned char* g_dyn_smem = nullptr;
constexpr size_t DYN_SMEM_BYTES = 256 * 1024;

[[noreturn]] static inline void die(const char* msg) {
  fprintf(stderr, "[mnb-emu] fatal: %s (block %u thread %u)\n", msg, blockIdx.x, threadIdx.x);
  fflush(stderr);
  _exit(97);
}

static inline void yield_to_scheduler() { mnb_emu_switch(&g_cta.cur->sp, g_cta.sched_sp); }

static inline void warp_complete(Warp& w) { w.part[w.gen & 1u] = w.alive; w.arrived = 0; w.gen++; }

// All lanes named by `mask` (minus lanes that already returned from the kernel) must call the same collective.
// Returns the slot array holding every lane's contribution; *part receives the lanes that took part (a lane may be resumed
// long after the collective completed, when other lanes have already left the kernel: the live mask of THAT moment is the
// wrong one to reduce over).
static inline const uint64_t* warp_exchange(unsigned mask, uint64_t mine, unsigned* part = nullptr) {
  Fiber* f = g_cta.cur;
  const int lane = f->tid & 31;
  Warp& w = g_cta.warps[f->tid >> 5];
  if ((mask & w.alive) != w.alive) die("warp collective with a partial mask: the emulator only models full-warp convergence");
  const unsigned buf = w.gen & 1u;
  w.slot[buf][lane] = mine;
  w.arrived |= 1u << lane;
  if ((w.arrived & w.alive) == w.alive) {
    warp_complete(w);
  } else {
    f->state = F_WAIT_WARP; f->wait_gen = w.gen;
    yield_to_scheduler();
  }
  if (part) *part = w.part[buf];
  return w.slot[buf];
}

static inline void cta_barrier() {
  Cta& c = g_cta;
  Fiber* f = c.cur;
  c.bar_arrived++;
  if ((int)c.bar_arrived == c.alive) { c.bar_arrived = 0; c.bar_gen++; }
  else { f->state = F_WAIT_CTA; f->wait_gen = c.bar_gen; yield_to_scheduler(); }
}

static inline void proc_barrier(ProcBarrier* b, LaunchCtl* lc) {
  const unsigned g = __atomic_load_n(&b->gen, __ATOMIC_ACQUIRE);
  if (__atomic_add_fetch(&b->count, 1u, __ATOMIC_ACQ_REL) == b->n) {
    __atomic_store_n(&b->count, 0u, __ATOMIC_RELAXED);
    __atomic_add_fetch(&b->gen, 1u, __ATOMIC_ACQ_REL);
    return;
  }
  unsigned long spins = 0;
  while (__atomic_load_n(&b->gen, __ATOMIC_ACQUIRE) == g) {
    if (__atomic_load_n(&lc->abort_flag, __ATOMIC_RELAXED)) _exit(98);
    if (++spins > 64) sched_yield();
  }
}

static inline void grid_barrier() {
  cta_barrier();
  if (g_cta.lc && g_cta.cur->tid == 0) proc_barrier(&g_cta.lc->grid, g_cta.lc);
  cta_barrier();
}
static inline void cluster_barrier() {
  cta_barrier();
  if (g_cta.lc && g_cta.cluster_size > 1 && g_cta.cur->tid == 0) proc_barrier(&g_cta.lc->cluster[g_cta.cluster_id], g_cta.lc);
  cta_barrier();
}

static void fiber_entry() {
  Cta& c = g_cta;
  c.invoke(c.invoke_ctx);
  // the thread returned from the kernel: it no longer takes part in collectives / barriers
  Fiber* f = c.cur;
  f->state = F_DONE;
  Warp& w = c.warps[f->tid >> 5];
  w.alive &= ~(1u << (f->tid & 31));
  if (w.alive && w.arrived && (w.arrived & w.alive) == w.alive) warp_complete(w);
  c.alive--;
  if (c.alive > 0 && (int)c.bar_arrived == c.alive) { c.bar_arrived = 0; c.bar_gen++; }
  yield_to_scheduler();
  die("resumed a finished fiber");
}

static inline void ensure_stacks() {
  if (g_stacks) return;
  g_stacks = (char*)mmap(nullptr, (size_t)MAX_THREADS * STACK_BYTES, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
  g_dyn_smem = (unsigned char*)mmap(nullptr, DYN_SMEM_BYTES, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
  if (g_stacks == MAP_FAILED || g_dyn_smem == MAP_FAILED) { fprintf(stderr, "[mnb-emu] cannot map fiber stacks\n"); abort(); }
}

// run one CTA to completion in the calling process
static inline void run_cta(unsigned bx, unsigned nblocks, unsigned nthreads, void (*invoke)(void*), void* ictx, LaunchCtl* lc,
                           unsigned cluster_size) {
  ensure_stacks();
  Cta& c = g_cta;
  if (nthreads > (unsigned)MAX_THREADS) { fprintf(stderr, "[mnb-emu] block of %u threads\n", nthreads); abort(); }
  c.nthreads = (int)nthreads; c.alive = (int)nthreads; c.bar_arrived = 0; c.bar_gen = 0;
  c.invoke = invoke; c.invoke_ctx = ictx; c.dyn_smem = g_dyn_smem; c.lc = lc;
  c.cluster_size = cluster_size ? cluster_size : 1; c.cluster_id = bx / c.cluster_size;
  blockIdx = uint3{bx, 0, 0}; gridDim = uint3{nblocks, 1, 1}; blockDim = uint3{nthreads, 1, 1};
  const int nwarps = ((int)nthreads + 31) / 32;
  for (int w = 0; w < nwarps; ++w) {
    const int lanes = std::min(32, (int)nthreads - 32 * w);
    c.warps[w].arrived = 0; c.warps[w].gen = 0; c.warps[w].alive = lanes == 32 ? 0xffffffffu : ((1u << lanes) - 1u);
  }
  for (unsigned t = 0; t < nthreads; ++t) {
    Fiber& f = c.fibers[t];
    f.tid = (int)t; f.state = F_RUNNABLE; f.wait_gen = 0;
    char* top = g_stacks + (size_t)(t + 1) * STACK_BYTES;      // 16-byte aligned
    void** sp = reinterpret_cast<void**>(top);
    *--sp = nullptr;                                           // fake return address of fiber_entry (never used)
    *--sp = reinterpret_cast<void*>(&fiber_entry);             // `ret` target of the first switch
    for (int k = 0; k < 6; ++k) *--sp = nullptr;               // rbp rbx r12 r13 r14 r15
    f.sp = sp;
  }
  // MNB_EMU_SHUFFLE=<seed>: the warps of a CTA are visited in a pseudo-random order that changes on every scheduler pass
  // and a warp is preempted after a random number of lane activations: exposes code that silently depends on "warp 0 runs
  // first" or on a warp running from barrier to barrier undisturbed (a missing __syncthreads shows up as a parity failure)
  static const char* shuffle_env = getenv("MNB_EMU_SHUFFLE");
  uint64_t rng = shuffle_env ? (0x9E3779B97F4A7C15ull * (uint64_t)(atoll(shuffle_env) + 1) + bx) : 0;
  auto next_rand = [&]() { rng ^= rng << 13; rng ^= rng >> 7; rng ^= rng << 17; return rng; };
  int order[MAX_THREADS / 32];
  for (int w = 0; w < nwarps; ++w) order[w] = w;
  int remaining = (int)nthreads;
  while (remaining > 0) {
    bool progress = false;
    if (rng) for (int w = nwarps - 1; w > 0; --w) { const int k = (int)(next_rand() % (uint64_t)(w + 1)); std::swap(order[w], order[k]); }
    for (int wi = 0; wi < nwarps; ++wi) {
      const int w = order[wi];
      int budget = rng ? 1 + (int)(next_rand() % 3) : 1 << 30;       // passes over the warp before it is preempted
      bool ran;
      do {
        ran = false;
        const int t0 = 32 * w, t1 = std::min((int)nthreads, t0 + 32);
        for (int t = t0; t < t1; ++t) {
          Fiber& f = c.fibers[t];
          if (f.state == F_DONE) continue;
          if (f.state == F_WAIT_WARP && c.warps[w].gen == f.wait_gen) continue;
          if (f.state == F_WAIT_CTA && c.bar_gen == f.wait_gen) continue;
          f.state = F_RUNNABLE;
          c.cur = &f; threadIdx = uint3{(unsigned)t, 0, 0};
          mnb_emu_switch(&c.sched_sp, f.sp);
          ran = true; progress = true;
          if (f.state == F_DONE) remaining--;
        }
      } while (ran && --budget > 0);
    }
    if (!progress) {
      fprintf(stderr, "[mnb-emu] deadlock in block %u: %d threads left, barrier %u/%d arrived\n", bx, remaining, c.bar_arrived, c.alive);
      for (int w = 0; w < nwarps; ++w) if (c.warps[w].arrived) fprintf(stderr, "  warp %d: arrived %08x alive %08x\n", w, c.warps[w].arrived, c.warps[w].alive);
      fflush(stderr);
      _exit(96);
    }
  }
}

}  // namespace emu

// ---- warp / block intrinsics ---------------------------------------------------------------------------------------
static inline void __syncthreads() { emu::cta_barrier(); }
static inline void __syncwarp(unsigned mask = 0xffffffffu) { emu::warp_exchange(mask, 0); }
namespace emu {
template <class T> static inline uint64_t to_u64(T v) { static_assert(sizeof(T) <= 8, "shuffle payload"); uint64_t u = 0; std::memcpy(&u, &v, sizeof(T)); return u; }
template <class T> static inline T from_u64(uint64_t u) { T v; std::memcpy(&v, &u, sizeof(T)); return v; }
static inline int my_lane() { return g_cta.cur->tid & 31; }
}  // namespace emu
template <class T> static inline T __shfl_sync(unsigned mask, T v, int src, int width = 32) {
  const uint64_t* s = emu::warp_exchange(mask, emu::to_u64(v));
  const int lane = emu::my_lane();
  return emu::from_u64<T>(s[(lane & ~(width - 1)) | (src & (width - 1))]);
}
template <class T> static inline T __shfl_xor_sync(unsigned mask, T v, int lane_mask, int width = 32) {
  const uint64_t* s = emu::warp_exchange(mask, emu::to_u64(v));
  const int lane = emu::my_lane(), src = lane ^ lane_mask;
  const int seg_end = (lane & ~(width - 1)) + width;
  return emu::from_u64<T>(s[src < seg_end ? src : lane]);
}
template <class T> static inline T __shfl_up_sync(unsigned mask, T v, unsigned delta, int width = 32) {
  const uint64_t* s = emu::warp_exchange(mask, emu::to_u64(v));
  const int lane = emu::my_lane(), src = lane - (int)delta;
  return emu::from_u64<T>(s[src >= (lane & ~(width - 1)) ? src : lane]);
}
template <class T> static inline T __shfl_down_sync(unsigned mask, T v, unsigned delta, int width = 32) {
  const uint64_t* s = emu::warp_exchange(mask, emu::to_u64(v));
  const int lane = emu::my_lane(), src = lane + (int)delta;
  return emu::from_u64<T>(s[src < (lane & ~(width - 1)) + width ? src : lane]);
}
static inline unsigned __ballot_sync(unsigned mask, int pred) {
  unsigned alive = 0;                                                        // lanes that returned before the vote contribute 0
  const uint64_t* s = emu::warp_exchange(mask, pred ? 1u : 0u, &alive);
  unsigned r = 0;
  for (int l = 0; l < 32; ++l) if (((alive >> l) & 1u) && s[l]) r |= 1u << l;
  return r & mask;
}
static inline int __any_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) != 0; }
static inline int __all_sync(unsigned mask, int pred) {
  unsigned alive = 0;
  const uint64_t* s = emu::warp_exchange(mask, pred ? 1u : 0u, &alive);
  for (int l = 0; l < 32; ++l) if (((alive >> l) & 1u) && !s[l]) return 0;
  return 1;
}
static inline unsigned __reduce_min_sync(unsigned mask, unsigned v) {
  unsigned alive = 0;
  const uint64_t* s = emu::warp_exchange(mask, v, &alive);
  unsigned r = 0xffffffffu;
  for (int l = 0; l < 32; ++l) if ((alive >> l) & 1u) r = std::min(r, (unsigned)s[l]);
  return r;
}
static inline unsigned __reduce_max_sync(unsigned mask, unsigned v) {
  unsigned alive = 0;
  const uint64_t* s = emu::warp_exchange(mask, v, &alive);
  unsigned r = 0;
  for (int l = 0; l < 32; ++l) if ((alive >> l) & 1u) r = std::max(r, (unsigned)s[l]);
  return r;
}
static inline unsigned __reduce_add_sync(unsigned mask, unsigned v) {
  unsigned alive = 0;
  const uint64_t* s = emu::warp_exchange(mask, v, &alive);
  unsigned r = 0;
  for (int l = 0; l < 32; ++l) if ((alive >> l) & 1u) r += (unsigned)s[l];
  return r;
}
static inline unsigned __activemask() { return emu::g_cta.warps[emu::g_cta.cur->tid >> 5].alive; }

// ====================================================================================================================
// runtime API
// ====================================================================================================================
typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorMemoryAllocation = 2, cudaErrorInvalidValue = 1, cudaErrorLaunchFailure = 719 };
typedef struct EmuStream* cudaStream_t;
struct EmuEvent { double t_ms; };
typedef EmuEvent* cudaEvent_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3, cudaMemcpyDefault = 4 };
enum { cudaStreamNonBlocking = 1, cudaHostAllocMapped = 2 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8, cudaFuncAttributeNonPortableClusterSizeAllowed = 10 };
struct cudaDeviceProp { int major, minor, multiProcessorCount; char name[64]; size_t totalGlobalMem; };
enum cudaLaunchAttributeID { cudaLaunchAttributeClusterDimension = 4 };
struct cudaLaunchAttributeValue { struct { unsigned x, y, z; } clusterDim; };
struct cudaLaunchAttribute { cudaLaunchAttributeID id; cudaLaunchAttributeValue val; };
struct cudaLaunchConfig_t { dim3 gridDim, blockDim; size_t dynamicSmemBytes = 0; cudaStream_t stream = nullptr; cudaLaunchAttribute* attrs = nullptr; unsigned numAttrs = 0; };

namespace emu {
inline cudaError_t g_last_error = cudaSuccess;
constexpr size_t ARENA_BYTES = 48ull << 30;
inline char* g_arena = nullptr;
inline size_t g_arena_top = 0;
inline std::multimap<size_t, void*>* g_free = nullptr;
inline std::unordered_map<void*, size_t>* g_sizes = nullptr;

static inline void ensure_arena() {
  if (g_arena) return;
  g_arena = (char*)mmap(nullptr, ARENA_BYTES, PROT_READ | PROT_WRITE, MAP_SHARED | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
  if (g_arena == MAP_FAILED) { fprintf(stderr, "[mnb-emu] cannot reserve the device arena\n"); abort(); }
  g_free = new std::multimap<size_t, void*>(); g_sizes = new std::unordered_map<void*, size_t>();
}
static inline void* arena_alloc(size_t n) {
  ensure_arena();
  n = (n + 4095) & ~(size_t)4095;
  auto it = g_free->find(n);
  if (it != g_free->end()) { void* p = it->second; g_free->erase(it); (*g_sizes)[p] = n; return p; }
  if (g_arena_top + n > ARENA_BYTES) return nullptr;
  void* p = g_arena + g_arena_top; g_arena_top += n; (*g_sizes)[p] = n;
  return p;
}
static inline void arena_free(void* p) {
  if (!p) return;
  auto it = g_sizes->find(p);
  if (it == g_sizes->end()) return;
  const size_t n = it->second; g_sizes->erase(it);
  if (n >= (1u << 20)) madvise(p, n, MADV_REMOVE);   // give the pages back; contents are undefined after cudaMalloc anyway
  g_free->emplace(n, p);
}
static inline int sm_count() { const char* e = getenv("MNB_EMU_SMS"); const int n = e ? atoi(e) : 4; return n < 1 ? 1 : (n > 32 ? 32 : n); }
static inline double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// launch: sequential CTAs in the caller unless the kernel synchronises across CTAs (cooperative / cluster launch)
template <class Tuple, class Kern, size_t... I>
static inline void call_kernel(Kern k, Tuple& t, std::index_sequence<I...>) { k(std::get<I>(t)...); }
template <class Kern, class... Args>
static inline cudaError_t launch(Kern kern, unsigned grid, unsigned block, size_t smem, unsigned cluster, bool cooperative, Args... args) {
  if (grid == 0 || block == 0 || block > (unsigned)MAX_THREADS || smem > DYN_SMEM_BYTES) { g_last_error = cudaErrorInvalidValue; return g_last_error; }
  auto tup = std::make_tuple(args...);
  struct Ctx { Kern k; decltype(tup)* t; } ictx{kern, &tup};
  auto invoke = +[](void* p) { Ctx* c = static_cast<Ctx*>(p); call_kernel(c->k, *c->t, std::index_sequence_for<Args...>{}); };
  const bool needs_procs = grid > 1 && (cooperative || cluster > 1);
  if (!needs_procs) {
    for (unsigned bx = 0; bx < grid; ++bx) run_cta(bx, grid, block, invoke, &ictx, nullptr, 1);
    return cudaSuccess;
  }
  if (grid > 64 || (cluster > 1 && grid % cluster != 0)) { g_last_error = cudaErrorInvalidValue; return g_last_error; }
  ensure_stacks();
  LaunchCtl* lc = static_cast<LaunchCtl*>(arena_alloc(sizeof(LaunchCtl)));
  std::memset(lc, 0, sizeof(LaunchCtl));
  lc->grid.n = grid;
  for (unsigned k = 0; k < 64; ++k) lc->cluster[k].n = cluster > 1 ? cluster : 1;
  fflush(stdout); fflush(stderr);
  std::vector<pid_t> pids(grid, -1);
  bool failed = false;
  for (unsigned bx = 0; bx < grid && !failed; ++bx) {
    const pid_t pid = fork();
    if (pid == 0) {
      prctl(PR_SET_PDEATHSIG, SIGKILL);          // a CTA process must not outlive (and spin without) the test process
      run_cta(bx, grid, block, invoke, &ictx, lc, cluster > 1 ? cluster : 1);
      _exit(0);
    }
    if (pid < 0) failed = true; else pids[bx] = pid;
  }
  if (failed) __atomic_store_n(&lc->abort_flag, 1, __ATOMIC_RELAXED);
  unsigned left = 0; for (pid_t p : pids) if (p > 0) left++;
  while (left > 0) {
    int status = 0;
    const pid_t p = waitpid(-1, &status, 0);
    if (p < 0) { if (errno == EINTR) continue; break; }
    bool ours = false; for (pid_t q : pids) if (q == p) ours = true;
    if (!ours) continue;
    left--;
    if (!(WIFEXITED(status) && WEXITSTATUS(status) == 0)) {
      if (!failed) fprintf(stderr, "[mnb-emu] kernel process %d ended abnormally (status 0x%x)\n", (int)p, status);
      failed = true; __atomic_store_n(&lc->abort_flag, 1, __ATOMIC_RELAXED);
    }
  }
  arena_free(lc);
  if (failed) { g_last_error = cudaErrorLaunchFailure; return g_last_error; }
  return cudaSuccess;
}
}  // namespace emu

static inline const char* cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : (e == cudaErrorLaunchFailure ? "emulated kernel failed" : "emulated CUDA error"); }
static inline cudaError_t cudaGetLastError() { const cudaError_t e = emu::g_last_error; emu::g_last_error = cudaSuccess; return e; }
static inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp* p, int) {
  std::memset(p, 0, sizeof(*p)); p->major = 9; p->minor = 0; p->multiProcessorCount = emu::sm_count();
  std::snprintf(p->name, sizeof(p->name), "mnb-emu (CPU interpreter, test only)"); p->totalGlobalMem = emu::ARENA_BYTES;
  return cudaSuccess;
}
static inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = reinterpret_cast<cudaStream_t>(new int(0)); return cudaSuccess; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t s) { delete reinterpret_cast<int*>(s); return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
static inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = new EmuEvent{0.0}; return cudaSuccess; }
static inline cudaError_t cudaEventDestroy(cudaEvent_t e) { delete e; return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t = nullptr) { e->t_ms = emu::now_ms(); return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t a, cudaEvent_t b) { *ms = (float)(b->t_ms - a->t_ms); return cudaSuccess; }
// MNB_EMU_MALLOC_LIMIT=<bytes> (read at every call): a single request above it fails, as on a device that cannot hold it --
// tests/test_emu_host_memory.py drives the host code's allocation-failure paths with it
static inline cudaError_t cudaMalloc(void** p, size_t n) {
  const char* limit = getenv("MNB_EMU_MALLOC_LIMIT");
  *p = (limit && n > strtoull(limit, nullptr, 10)) ? nullptr : emu::arena_alloc(n ? n : 1);
  return *p ? cudaSuccess : cudaErrorMemoryAllocation;
}
// bytes allocated from the arena and not freed (whole 4096-byte pages per allocation): the leak probe of the same tests
extern "C" __attribute__((used, visibility("default"))) inline size_t mnb_emu_allocated_bytes() {
  size_t sum = 0;
  if (emu::g_sizes) for (const auto& kv : *emu::g_sizes) sum += kv.second;
  return sum;
}
static inline cudaError_t cudaFree(void* p) { emu::arena_free(p); return cudaSuccess; }
static inline cudaError_t cudaHostAlloc(void** p, size_t n, unsigned) { return cudaMalloc(p, n); }
static inline cudaError_t cudaFreeHost(void* p) { return cudaFree(p); }
static inline cudaError_t cudaHostGetDevicePointer(void** d, void* h, unsigned) { *d = h; return cudaSuccess; }
static inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { std::memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { std::memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t = nullptr) { std::memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemset(void* d, int v, size_t n) { std::memset(d, v, n); return cudaSuccess; }
template <class F> static inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int* n, F, int, size_t) { *n = 2; return cudaSuccess; }
template <class F> static inline cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute, int) { return cudaSuccess; }
template <class... KArgs, class... Args>
static inline cudaError_t cudaLaunchKernelEx(const cudaLaunchConfig_t* cfg, void (*kern)(KArgs...), Args&&... args) {
  unsigned cluster = 1;
  for (unsigned i = 0; i < cfg->numAttrs; ++i) if (cfg->attrs[i].id == cudaLaunchAttributeClusterDimension) cluster = cfg->attrs[i].val.clusterDim.x;
  return emu::launch(kern, cfg->gridDim.x, cfg->blockDim.x, cfg->dynamicSmemBytes, cluster, false, std::decay_t<KArgs>(args)...);
}
