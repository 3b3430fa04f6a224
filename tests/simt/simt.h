// simt.h — TEST INFRASTRUCTURE.  A single-OS-thread SIMT emulator that runs the product's CUDA sources on the host, so
// that kernels written while no GPU is available can be executed against the oracle before they ever see a GPU
// (tests/simt/README.md).  It is NOT a CPU path of the product: liblsdreg.so never contains it; tests build a separate
// liblsdreg_emu.so from translated copies of the sources (tests/simt/build_emu.py) and load it explicitly.
//
// Model: a kernel launch runs block after block; the threads of a block are fibers (own stacks, hand-written context
// switch) scheduled round-robin by one OS thread.  A fiber runs until it reaches a barrier or a warp collective, where it
// yields until every live thread of the block / warp has arrived.  Consequences: atomics are trivially atomic; there is no
// real concurrency, so data races do not show — but wrong indices, wrong capacities, wrong phase structure, missing
// participants of a collective (reported as a deadlock) and plain arithmetic do.  Launches are synchronous; streams and
// events are no-ops; "device" memory is host memory (filled with 0xA5 on allocation to expose reads of uninitialised data).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <functional>
#include <type_traits>
#include <vector>

#define LSD_SIMT_EMU 1
#define __launch_bounds__(...)
#undef __shared__
#define __shared__ static
#undef __constant__
#define __constant__

namespace simt {

struct Dim3 { unsigned x = 1, y = 1, z = 1; Dim3() {} Dim3(unsigned a, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {} Dim3(dim3 d) : x(d.x), y(d.y), z(d.z) {} };

struct Ctx { void* rsp = nullptr; };
extern "C" void simt_switch(Ctx* from, Ctx* to);
asm(R"(
.text
.globl simt_switch
.type simt_switch,@function
simt_switch:
  pushq %rbp
  pushq %rbx
  pushq %r12
  pushq %r13
  pushq %r14
  pushq %r15
  movq %rsp, (%rdi)
  movq (%rsi), %rsp
  popq %r15
  popq %r14
  popq %r13
  popq %r12
  popq %rbx
  popq %rbp
  ret
.size simt_switch,.-simt_switch
)");

constexpr size_t kStack = 192 * 1024;

struct WarpState {
  int gen = 0, arrived = 0, live = 0;
  unsigned live_mask = 0;
  unsigned long long slot[32];
  unsigned long long res[2][32];
  unsigned res_live[2];
};

struct Fiber {
  Ctx ctx;
  char* stack = nullptr;
  unsigned tid = 0;
  Dim3 tid3;
  bool done = true;
};

struct State {
  std::vector<Fiber> fibers;
  std::vector<WarpState> warps;
  Ctx sched;
  Fiber* cur = nullptr;
  const std::function<void()>* body = nullptr;
  Dim3 block_idx, block_dim, grid_dim;
  int n_threads = 0, alive = 0;
  int bar_gen = 0, bar_arrived = 0;
  unsigned long long progress = 0;
  std::vector<char> dyn_smem;
  long long launches = 0, collectives = 0;
};
inline State& S() { static State s; return s; }

inline void yield() { State& s = S(); simt_switch(&s.cur->ctx, &s.sched); }

inline void release_warp(WarpState& w) {
  const int g = w.gen;
  memcpy(w.res[g & 1], w.slot, sizeof(w.slot));
  w.res_live[g & 1] = w.live_mask;
  w.arrived = 0;
  w.gen++;
  S().progress++;
}

// every live lane of the calling warp deposits v and gets the 32 deposited values back
inline const unsigned long long* xchg(unsigned long long v, unsigned* live_out = nullptr) {
  State& s = S();
  const unsigned tid = s.cur->tid;
  WarpState& w = s.warps[tid >> 5];
  const int lane = tid & 31, g = w.gen;
  s.collectives++;
  w.slot[lane] = v;
  w.arrived++;
  if (w.arrived == w.live) release_warp(w);
  else while (w.gen == g) yield();
  if (live_out) *live_out = w.res_live[g & 1];
  return w.res[g & 1];
}

inline void syncthreads() {
  State& s = S();
  const int g = s.bar_gen;
  s.bar_arrived++;
  if (s.bar_arrived == s.alive) { s.bar_arrived = 0; s.bar_gen++; s.progress++; }
  else while (s.bar_gen == g) yield();
}

inline void fiber_exit() {  // the calling fiber's kernel body returned
  State& s = S();
  Fiber* f = s.cur;
  f->done = true;
  s.alive--;
  s.progress++;
  WarpState& w = s.warps[f->tid >> 5];
  w.live--;
  w.live_mask &= ~(1u << (f->tid & 31));
  if (w.live > 0 && w.arrived == w.live) release_warp(w);             // the others were waiting for this lane only
  if (s.alive > 0 && s.bar_arrived == s.alive) { s.bar_arrived = 0; s.bar_gen++; }
  simt_switch(&f->ctx, &s.sched);
  abort();  // a finished fiber is never resumed
}

extern "C" inline void simt_fiber_entry() {
  (*S().body)();
  fiber_exit();
}

inline void run_block(const std::function<void()>& body) {
  State& s = S();
  const int n = s.n_threads;
  if ((int)s.fibers.size() < n) {
    const size_t old = s.fibers.size();
    s.fibers.resize(n);
    for (size_t i = old; i < (size_t)n; i++) s.fibers[i].stack = (char*)aligned_alloc(64, kStack);
  }
  s.warps.assign((n + 31) / 32, WarpState());
  s.body = &body;
  s.alive = n; s.bar_gen = 0; s.bar_arrived = 0;
  for (int t = 0; t < n; t++) {
    Fiber& f = s.fibers[t];
    f.tid = (unsigned)t;
    f.tid3.x = t % s.block_dim.x; f.tid3.y = (t / s.block_dim.x) % s.block_dim.y; f.tid3.z = t / (s.block_dim.x * s.block_dim.y);
    f.done = false;
    WarpState& w = s.warps[t >> 5];
    w.live++; w.live_mask |= 1u << (t & 31);
    // initial frame: six callee-saved registers, the entry address, a fake return address; at entry rsp = top - 8
    uintptr_t top = ((uintptr_t)f.stack + kStack) & ~(uintptr_t)15;
    void** sp = (void**)top;
    *--sp = nullptr;
    *--sp = (void*)&simt_fiber_entry;
    for (int r = 0; r < 6; r++) *--sp = nullptr;
    f.ctx.rsp = sp;
  }
  unsigned long long last = ~0ull;
  while (s.alive > 0) {
    if (s.progress == last) {
      fprintf(stderr, "simt: DEADLOCK in block (%u,%u): %d threads alive, none can proceed (a barrier or warp collective is missing participants)\n",
              s.block_idx.x, s.block_idx.y, s.alive);
      for (size_t wi = 0; wi < s.warps.size(); wi++)
        if (s.warps[wi].arrived) fprintf(stderr, "  warp %zu: %d of %d live lanes arrived at a collective\n", wi, s.warps[wi].arrived, s.warps[wi].live);
      fprintf(stderr, "  block barrier: %d of %d arrived\n", s.bar_arrived, s.alive);
      abort();
    }
    last = s.progress;
    for (int t = 0; t < n; t++) {
      Fiber& f = s.fibers[t];
      if (f.done) continue;
      s.cur = &f;
      simt_switch(&s.sched, &f.ctx);
    }
  }
  s.cur = nullptr;
}

inline void launch(Dim3 grid, Dim3 block, size_t smem, const std::function<void()>& body) {
  State& s = S();
  s.launches++;
  s.grid_dim = grid; s.block_dim = block;
  s.n_threads = (int)(block.x * block.y * block.z);
  if (s.n_threads <= 0 || s.n_threads > 1024) { fprintf(stderr, "simt: bad block size %d\n", s.n_threads); abort(); }
  s.dyn_smem.assign(smem + 16, 0);
  for (unsigned bz = 0; bz < grid.z; bz++)
    for (unsigned by = 0; by < grid.y; by++)
      for (unsigned bx = 0; bx < grid.x; bx++) {
        s.block_idx = Dim3(bx, by, bz);
        run_block(body);
      }
}

inline Dim3 to_dim3(dim3 d) { return Dim3(d); }
template <class T, class = typename std::enable_if<std::is_arithmetic<T>::value>::type> inline Dim3 to_dim3(T v) { return Dim3((unsigned)v); }
inline void* dyn_smem() { return S().dyn_smem.data(); }
inline const Dim3& tid3() { return S().cur->tid3; }
inline int lane_id() { return (int)(S().cur->tid & 31); }

// ---------------------------------------------------------------- "device" memory and the runtime API
inline cudaError_t rt_malloc(void** p, size_t n) { *p = malloc(n ? n : 1); if (!*p) return cudaErrorMemoryAllocation; memset(*p, 0xA5, n); return cudaSuccess; }
inline cudaError_t rt_free(void* p) { free(p); return cudaSuccess; }
inline cudaError_t rt_memcpy(void* d, const void* s, size_t n) { if (n) memmove(d, s, n); return cudaSuccess; }
inline cudaError_t rt_memset(void* d, int v, size_t n) { if (n) memset(d, v, n); return cudaSuccess; }
inline cudaError_t rt_ok() { return cudaSuccess; }
template <class T> inline cudaError_t rt_set(T* p, T v) { *p = v; return cudaSuccess; }

}  // namespace simt

// counters device code may bump under #ifdef LSD_SIMT_EMU (tuning aids: list occupancies, fallback rates); read through
// the extra export simt_stats() of liblsdreg_emu.so
namespace simt { inline long long* stats() { static long long v[32]; return v; } }
#define SIMT_STAT_ADD(i, v) (simt::stats()[(i)] += (long long)(v))
#define SIMT_STAT_MAX(i, v) (simt::stats()[(i)] = std::max(simt::stats()[(i)], (long long)(v)))
extern "C" inline long long* simt_stats() { return simt::stats(); }
extern "C" inline long long simt_collectives() { return simt::S().collectives; }

// ---------------------------------------------------------------- CUDA built-in variables and functions
#define threadIdx (simt::tid3())
#define blockIdx (simt::S().block_idx)
#define blockDim (simt::S().block_dim)
#define gridDim (simt::S().grid_dim)

inline void __syncthreads() { simt::syncthreads(); }
inline void __syncwarp(unsigned = 0xffffffffu) { simt::xchg(0); }
inline void __threadfence() {}
inline void __threadfence_system() {}
inline void __threadfence_block() {}

inline unsigned __ballot_sync(unsigned, int pred) {
  unsigned live;
  const unsigned long long* r = simt::xchg(pred ? 1ull : 0ull, &live);
  unsigned m = 0;
  for (int i = 0; i < 32; i++) if ((live >> i & 1u) && r[i]) m |= 1u << i;
  return m;
}
inline int __any_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) != 0; }
inline int __all_sync(unsigned mask, int pred) { unsigned live; const unsigned long long* r = simt::xchg(pred ? 1ull : 0ull, &live); for (int i = 0; i < 32; i++) if ((live >> i & 1u) && !r[i]) return 0; return 1; }

template <class T> inline unsigned long long simt_bits(T v) { unsigned long long b = 0; static_assert(sizeof(T) <= 8, "shuffle payload"); memcpy(&b, &v, sizeof(T)); return b; }
template <class T> inline T simt_unbits(unsigned long long b) { T v; memcpy(&v, &b, sizeof(T)); return v; }
template <class T> inline T __shfl_sync(unsigned, T v, int src) { const unsigned long long* r = simt::xchg(simt_bits(v)); return simt_unbits<T>(r[src & 31]); }
template <class T> inline T __shfl_xor_sync(unsigned, T v, int o) { const int lane = simt::lane_id(); const unsigned long long* r = simt::xchg(simt_bits(v)); return simt_unbits<T>(r[(lane ^ o) & 31]); }
template <class T> inline T __shfl_up_sync(unsigned, T v, unsigned o) { const int lane = simt::lane_id(); const unsigned long long* r = simt::xchg(simt_bits(v)); return lane >= (int)o ? simt_unbits<T>(r[lane - o]) : v; }
template <class T> inline T __shfl_down_sync(unsigned, T v, unsigned o) { const int lane = simt::lane_id(); const unsigned long long* r = simt::xchg(simt_bits(v)); return lane + (int)o < 32 ? simt_unbits<T>(r[lane + o]) : v; }
inline unsigned __reduce_min_sync(unsigned, unsigned v) { unsigned live; const unsigned long long* r = simt::xchg(v, &live); unsigned m = 0xffffffffu; for (int i = 0; i < 32; i++) if (live >> i & 1u) m = std::min(m, (unsigned)r[i]); return m; }
inline int __reduce_min_sync(unsigned, int v) { unsigned live; const unsigned long long* r = simt::xchg((unsigned long long)(long long)v, &live); int m = 0x7fffffff; for (int i = 0; i < 32; i++) if (live >> i & 1u) m = std::min(m, (int)(long long)r[i]); return m; }
inline unsigned __reduce_max_sync(unsigned, unsigned v) { unsigned live; const unsigned long long* r = simt::xchg(v, &live); unsigned m = 0; for (int i = 0; i < 32; i++) if (live >> i & 1u) m = std::max(m, (unsigned)r[i]); return m; }
inline unsigned simt_lanemask_lt() { return (1u << simt::lane_id()) - 1u; }

template <class T> inline T __ldg(const T* p) { return *p; }
template <class T> inline T __ldcg(const T* p) { return *p; }
template <class T> inline T __ldcs(const T* p) { return *p; }

// atomics: one OS thread, so a plain read-modify-write is atomic
template <class T> inline T atomicAdd(T* p, T v) { T o = *p; *p = o + v; return o; }
inline unsigned atomicAdd(unsigned* p, int v) { unsigned o = *p; *p = o + (unsigned)v; return o; }
inline int atomicAdd(int* p, unsigned v) { int o = *p; *p = o + (int)v; return o; }
template <class T> inline T atomicMax(T* p, T v) { T o = *p; if (v > o) *p = v; return o; }
template <class T> inline T atomicMin(T* p, T v) { T o = *p; if (v < o) *p = v; return o; }
template <class T> inline T atomicOr(T* p, T v) { T o = *p; *p = o | v; return o; }
template <class T> inline T atomicAnd(T* p, T v) { T o = *p; *p = o & v; return o; }
template <class T> inline T atomicExch(T* p, T v) { T o = *p; *p = v; return o; }
template <class T> inline T atomicCAS(T* p, T cmp, T v) { T o = *p; if (o == cmp) *p = v; return o; }

inline long long clock64() { return 0; }   // no cycle counter in the emulator: timings read 0
inline int __popc(unsigned v) { return __builtin_popcount(v); }
inline int __popcll(unsigned long long v) { return __builtin_popcountll(v); }
inline int __ffs(int v) { return __builtin_ffs(v); }
inline int __ffsll(long long v) { return __builtin_ffsll(v); }
inline int __clz(int v) { return v ? __builtin_clz((unsigned)v) : 32; }
inline int __float_as_int(float f) { int i; memcpy(&i, &f, 4); return i; }
inline float __int_as_float(int i) { float f; memcpy(&f, &i, 4); return f; }
inline unsigned __float_as_uint(float f) { unsigned i; memcpy(&i, &f, 4); return i; }
inline float __uint_as_float(unsigned i) { float f; memcpy(&f, &i, 4); return f; }
inline long long __double_as_longlong(double d) { long long i; memcpy(&i, &d, 8); return i; }
inline double __longlong_as_double(long long i) { double d; memcpy(&d, &i, 8); return d; }
// build with -ffp-contract=off: these are then exactly the round-to-nearest single operations
inline float __fadd_rn(float a, float b) { volatile float r = a + b; return r; }
inline float __fmul_rn(float a, float b) { volatile float r = a * b; return r; }
inline float __fsub_rn(float a, float b) { volatile float r = a - b; return r; }
inline float __fmaf_rn(float a, float b, float c) { return fmaf(a, b, c); }
inline double __fma_rn(double a, double b, double c) { return fma(a, b, c); }
inline long long __double2ll_rn(double d) { return llrint(d); }
inline int __double2int_rn(double d) { return (int)lrint(d); }
inline int __float2int_rn(float f) { return (int)lrintf(f); }
inline int __float2int_rd(float f) { return (int)floorf(f); }
inline float rsqrtf(float x) { return 1.0f / sqrtf(x); }

#define SIMT_MINMAX(T) inline T min(T a, T b) { return a < b ? a : b; } inline T max(T a, T b) { return a > b ? a : b; }
SIMT_MINMAX(int) SIMT_MINMAX(unsigned) SIMT_MINMAX(long) SIMT_MINMAX(unsigned long) SIMT_MINMAX(long long) SIMT_MINMAX(unsigned long long)
SIMT_MINMAX(float) SIMT_MINMAX(double)
inline unsigned min(unsigned a, int b) { return min(a, (unsigned)b); }
inline unsigned min(int a, unsigned b) { return min((unsigned)a, b); }
inline unsigned max(unsigned a, int b) { return max(a, (unsigned)b); }
inline unsigned max(int a, unsigned b) { return max((unsigned)a, b); }
inline long long min(long long a, int b) { return min(a, (long long)b); }
inline long long min(int a, long long b) { return min((long long)a, b); }
inline unsigned long long min(unsigned long long a, unsigned b) { return min(a, (unsigned long long)b); }
inline double min(double a, float b) { return min(a, (double)b); }
inline double min(float a, double b) { return min((double)a, b); }
inline double max(double a, float b) { return max(a, (double)b); }
inline double max(float a, double b) { return max((double)a, b); }

// ---------------------------------------------------------------- the runtime API the sources call (no libcudart behind it)
#define cudaMalloc(p, n) simt::rt_malloc((void**)(p), (n))
#define cudaMallocHost(p, n) simt::rt_malloc((void**)(p), (n))
#define cudaHostAlloc(p, n, f) simt::rt_malloc((void**)(p), (n))
#define cudaHostGetDevicePointer(dp, hp, f) simt::rt_set((void**)(dp), (void*)(hp))
#define cudaFree(p) simt::rt_free((void*)(p))
#define cudaFreeHost(p) simt::rt_free((void*)(p))
#define cudaMemcpy(d, s, n, k) simt::rt_memcpy((d), (s), (n))
#define cudaMemcpyAsync(d, s, n, k, st) simt::rt_memcpy((d), (s), (n))
#define cudaMemset(d, v, n) simt::rt_memset((d), (v), (n))
#define cudaMemsetAsync(d, v, n, st) simt::rt_memset((d), (v), (n))
#define cudaMemcpyToSymbol(sym, src, n) simt::rt_memcpy((void*)&(sym), (src), (n))
#define cudaSetDevice(d) simt::rt_ok()
#define cudaGetDevice(p) simt::rt_set((p), 0)
#define cudaGetDeviceCount(p) simt::rt_set((p), 1)
#define cudaGetLastError() simt::rt_ok()
#define cudaPeekAtLastError() simt::rt_ok()
#define cudaDeviceSynchronize() simt::rt_ok()
#define cudaDeviceSetLimit(a, b) simt::rt_ok()
#define cudaDeviceGetAttribute(p, a, d) simt::rt_set((p), 1)
#define cudaStreamCreateWithFlags(p, f) simt::rt_set((p), (cudaStream_t)0x10)
#define cudaStreamCreate(p) simt::rt_set((p), (cudaStream_t)0x10)
#define cudaStreamDestroy(s) simt::rt_ok()
#define cudaStreamSynchronize(s) simt::rt_ok()
#define cudaStreamQuery(s) simt::rt_ok()
#define cudaStreamWaitEvent(s, e, f) simt::rt_ok()
#define cudaEventCreate(p) simt::rt_set((p), (cudaEvent_t)0x20)
#define cudaEventCreateWithFlags(p, f) simt::rt_set((p), (cudaEvent_t)0x20)
#define cudaEventDestroy(e) simt::rt_ok()
#define cudaEventRecord(e, s) simt::rt_ok()
#define cudaEventSynchronize(e) simt::rt_ok()
#define cudaEventElapsedTime(ms, a, b) simt::rt_set((ms), 0.001f)
#define cudaGetErrorString(e) "simt emulator"
#define cudaIpcGetMemHandle(h, p) cudaErrorNotSupported
#define cudaIpcOpenMemHandle(p, h, f) cudaErrorNotSupported
#define cudaIpcCloseMemHandle(p) cudaErrorNotSupported
#define cudaDeviceEnablePeerAccess(d, f) simt::rt_ok()
#define cudaPointerGetAttributes(a, p) cudaErrorNotSupported
