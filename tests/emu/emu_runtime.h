// SPDX: test infrastructure only.
//
// A tiny single-OS-thread, fiber-based emulator of the CUDA SIMT execution model, used ONLY by the
// `-m "not gpu"` unit tests to run the kernel *logic* of off-policy_b200/csrc/*.cu on a CPU (the build
// container has no GPU, and every GPU round-trip costs minutes of a small budget).  It is NOT a product
// fallback: the product loader (off-policy_b200/offpolicy/_b200/capi.py) only ever loads the nvcc-built
// libmarl_b200.so and raises when there is no CUDA device.  Nothing here is shipped or timed.
//
// Model: blocks run one after another; the threads of a block are fibers (own stacks, cooperative switch) scheduled round-robin
// (or in reverse / pseudo-random order, EMU_ORDER=reverse|random, to shake out missing barriers);
// __syncthreads / warp collectives are cooperative barriers.  `__shared__` becomes `static` (valid
// because blocks are sequential).  wgmma and mbarrier are restated in csrc/mx_tc.cuh's MX_EMU half; TMA and clusters are not emulated.
#pragma once
#include <ucontext.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <vector>

struct uint3 { unsigned x, y, z; };
struct dim3 {
  unsigned x, y, z;
  dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct float2 { float x, y; };
struct alignas(16) float4 { float x, y, z, w; };
struct int2 { int x, y; };
struct alignas(16) int4 { int x, y, z, w; };
struct alignas(16) uint4 { unsigned x, y, z, w; };
struct alignas(16) double2 { double x, y; };
static inline float2 make_float2(float x, float y) { return float2{x, y}; }
static inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
static inline int4 make_int4(int x, int y, int z, int w) { return int4{x, y, z, w}; }
static inline double2 make_double2(double x, double y) { return double2{x, y}; }

typedef void* cudaStream_t;
typedef int cudaError_t;
#define cudaSuccess 0
enum cudaMemcpyKind { cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3, cudaMemcpyDefault = 4 };
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t) { memcpy(d, s, n); return 0; }
static inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t) { memset(d, v, n); return 0; }
static inline cudaError_t cudaGetLastError() { return 0; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return 0; }
static inline const char* cudaGetErrorString(cudaError_t) { return "emu"; }

namespace emu {

// Context switch: on x86-64 a hand-written register swap (callee-saved registers + stack pointer, ~15 instructions); swapcontext()
// makes two rt_sigprocmask system calls per switch, which dominated the emulated test time.  Elsewhere: ucontext.
#if defined(__x86_64__)
#define EMU_FAST_SWITCH 1
#else
#define EMU_FAST_SWITCH 0
#endif

struct Fiber {
  ucontext_t ctx;
  void* sp;                // EMU_FAST_SWITCH: saved stack pointer
  uint3 tid;
  int lin, lane, warp;
  bool done;
  char* stack;
};
struct Warp {
  int arrived, gen, nlanes;
  uint64_t slot[32];
  unsigned ballot;
};
struct Globals {
  uint3 block;
  dim3 bdim, gdim;
  int nthreads, alive, arrived, gen;
  long progress;
  ucontext_t sched;
  void* sched_sp;
  std::vector<Fiber> fibers;
  std::vector<Warp> warps;
  std::vector<char> dynsmem;
  const std::function<void()>* body;
  int num_sms;
};
extern Globals g;
extern Fiber* cur;

void yield();
void syncthreads();
void warp_barrier();
void launch(dim3 grid, dim3 block, size_t smem, const std::function<void()>& body);
inline void* dyn_smem() { return g.dynsmem.data(); }

template <class T>
inline T shfl_from(T v, int src) {
  static_assert(sizeof(T) <= 8, "shfl type");
  Warp& w = g.warps[cur->warp];
  uint64_t bits = 0;
  memcpy(&bits, &v, sizeof(T));
  w.slot[cur->lane] = bits;
  warp_barrier();
  T r = v;
  if (src >= 0 && src < w.nlanes) memcpy(&r, &w.slot[src], sizeof(T));
  warp_barrier();
  return r;
}
inline unsigned ballot(int pred) {
  Warp& w = g.warps[cur->warp];
  w.slot[cur->lane] = pred ? 1 : 0;
  warp_barrier();
  unsigned m = 0;
  for (int i = 0; i < w.nlanes; ++i) m |= (w.slot[i] ? 1u : 0u) << i;
  warp_barrier();
  return m;
}
}  // namespace emu

#define threadIdx (emu::cur->tid)
#define blockIdx (emu::g.block)
#define blockDim (emu::g.bdim)
#define gridDim (emu::g.gdim)
#define warpSize 32

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __shared__ static
#define __align__(n) __attribute__((aligned(n)))
#define __syncthreads() emu::syncthreads()
#define __syncwarp(...) emu::warp_barrier()
#define __threadfence() ((void)0)
#define __threadfence_block() ((void)0)
#define __threadfence_system() ((void)0)

template <class T> inline T __shfl_sync(unsigned, T v, int src, int width = 32) {
  int base = (emu::cur->lane / width) * width;
  return emu::shfl_from(v, base + (src % width));
}
template <class T> inline T __shfl_xor_sync(unsigned, T v, int m, int width = 32) {
  int l = emu::cur->lane, src = l ^ m;
  if (src / width != l / width) src = l;
  return emu::shfl_from(v, src);
}
template <class T> inline T __shfl_down_sync(unsigned, T v, unsigned d, int width = 32) {
  int l = emu::cur->lane, src = l + (int)d;
  if (src / width != l / width) src = l;
  return emu::shfl_from(v, src);
}
template <class T> inline T __shfl_up_sync(unsigned, T v, unsigned d, int width = 32) {
  int l = emu::cur->lane, src = l - (int)d;
  if (src < 0 || src / width != l / width) src = l;
  return emu::shfl_from(v, src);
}
inline unsigned __ballot_sync(unsigned, int p) { return emu::ballot(p); }
inline int __any_sync(unsigned, int p) { return emu::ballot(p) != 0; }
inline int __all_sync(unsigned, int p) { unsigned b = emu::ballot(p); return b == ((emu::g.warps[emu::cur->warp].nlanes >= 32) ? 0xffffffffu : ((1u << emu::g.warps[emu::cur->warp].nlanes) - 1)); }
inline unsigned __activemask() { return 0xffffffffu; }

template <class T> inline T atomicAdd(T* p, T v) { T o = *p; *p = o + v; return o; }
inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { auto o = *p; *p = o + v; return o; }
template <class T> inline T atomicMax(T* p, T v) { T o = *p; if (v > o) *p = v; return o; }
template <class T> inline T atomicMin(T* p, T v) { T o = *p; if (v < o) *p = v; return o; }
template <class T> inline T atomicExch(T* p, T v) { T o = *p; *p = v; return o; }
template <class T> inline T atomicCAS(T* p, T c, T v) { T o = *p; if (o == c) *p = v; return o; }

template <class T> inline T __ldg(const T* p) { return *p; }
template <class T> inline T __ldcg(const T* p) { return *p; }
inline float __expf(float x) { return expf(x); }
inline float __logf(float x) { return logf(x); }
inline float __fdividef(float a, float b) { return a / b; }
inline float __frcp_rn(float a) { return 1.0f / a; }
inline float rsqrtf(float a) { return 1.0f / sqrtf(a); }
inline float __fmaf_rn(float a, float b, float c) { return fmaf(a, b, c); }
inline unsigned __float_as_uint(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
inline float __uint_as_float(unsigned u) { float f; memcpy(&f, &u, 4); return f; }
inline int __float_as_int(float f) { int u; memcpy(&u, &f, 4); return u; }
inline float __int_as_float(int u) { float f; memcpy(&f, &u, 4); return f; }
inline int __popc(unsigned x) { return __builtin_popcount(x); }
inline int __ffs(int x) { return __builtin_ffs(x); }
inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
using std::max;
using std::min;

#define MX_LAUNCH(kern, grid, block, smem, stream, ...) \
  emu::launch((grid), (block), (smem), [&]() { kern(__VA_ARGS__); })
