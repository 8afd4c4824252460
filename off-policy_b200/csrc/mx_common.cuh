// Common device/host helpers for the H100 (sm_90a) off-policy MARL update engine.
//
// Build modes:
//   * product:  nvcc -gencode arch=compute_90a,code=sm_90a  (the only thing shipped / loaded / timed)
//   * MARL_EMU: g++ with tests/emu/emu_runtime.h -- CPU fiber emulation of the SIMT kernels, used by the
//               `-m "not gpu"` unit tests only (kernel-logic checks in a container without a GPU).
#pragma once
#include <stdint.h>

#ifdef MARL_EMU
#include "emu_runtime.h"
#define MX_EMU 1
#define MX_PDL_WAIT() ((void)0)
#define MX_PDL_THETA_WRITTEN() ((void)0)
#else
#include <cuda_runtime.h>
#define MX_EMU 0
#define MX_LAUNCH(kern, grid, block, smem, stream, ...) kern<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)

// Programmatic dependent launch (mx_launch in mx_internal.h says which launches may overlap their predecessor).
// MX_PDL_WAIT() = griddepcontrol.wait (returns at once in a plain launch) followed by launch_dependents, i.e. a dependent may
// start as soon as every CTA of this grid is past its own wait -- never before this grid's predecessor has completed.
extern int g_mx_pdl, g_mx_pdl_auto, g_mx_pdl_rows;      // option pdl: -1 automatic (per learner step, by size), 0 off, 1 on
extern int g_mx_pdl_skip_next;
#define MX_PDL_THETA_WRITTEN() (g_mx_pdl_skip_next = 1)
#define MX_PDL_WAIT()                                                     \
  do {                                                                    \
    asm volatile("griddepcontrol.wait;" ::: "memory");                    \
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");       \
  } while (0)
extern int g_mx_smem_carveout;
#endif

#define MX_H 64          // hidden size the kernels are specialised for (reference default, config.py:63)
#define MX_G (3 * MX_H)  // GRU gate rows [r; z; n]

#define MX_DEVINL __device__ __forceinline__
#if MX_EMU
#define MX_NOINLINE
#else
#define MX_NOINLINE __noinline__
#endif

// dynamic shared memory base
#if MX_EMU
#define MX_DYN_SMEM(name) float* name = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(emu::dyn_smem()) + 15) & ~uintptr_t(15))
#else
#define MX_DYN_SMEM(name)                                    \
  extern __shared__ __align__(16) unsigned char _mx_smem[]; \
  float* name = reinterpret_cast<float*>(_mx_smem)
#endif

MX_DEVINL int mx_imin(int a, int b) { return a < b ? a : b; }
MX_DEVINL int mx_imax(int a, int b) { return a > b ? a : b; }
__host__ __device__ static inline int mx_ceil_div(int a, int b) { return (a + b - 1) / b; }
__host__ __device__ static inline int mx_round_up(int a, int b) { return (a + b - 1) / b * b; }
__host__ __device__ static inline int64_t mx_round_up64(int64_t a, int64_t b) { return (a + b - 1) / b * b; }

MX_DEVINL float mx_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
MX_DEVINL double mx_warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
MX_DEVINL float mx_warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

MX_DEVINL float mx_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

MX_DEVINL float4 mx_ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
MX_DEVINL void mx_st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

// streaming 16-byte global load/store (read-once data: bypass L1 allocation)
MX_DEVINL float4 mx_ld4_stream(const float* p) {
#if MX_EMU
  return *reinterpret_cast<const float4*>(p);
#else
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
#endif
}
MX_DEVINL void mx_st4_stream(float* p, float4 v) {
#if MX_EMU
  *reinterpret_cast<float4*>(p) = v;
#else
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
#endif
}

// ---- asynchronous global -> shared copies (LDGSTS): all of a thread's copies are in flight at once ----
MX_DEVINL void mx_cp16(float* sdst, const float* gsrc) {
#if MX_EMU
  *reinterpret_cast<float4*>(sdst) = *reinterpret_cast<const float4*>(gsrc);
#else
  unsigned sa = (unsigned)__cvta_generic_to_shared(sdst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sa), "l"(gsrc) : "memory");
#endif
}
// 16-byte copy that reads only `nbytes` (0 or 16) from global memory and zero-fills the rest: a branch-free "copy or clear"
MX_DEVINL void mx_cp16z(float* sdst, const float* gsrc, int nbytes) {
#if MX_EMU
  if (nbytes) *reinterpret_cast<float4*>(sdst) = *reinterpret_cast<const float4*>(gsrc);
  else *reinterpret_cast<float4*>(sdst) = float4{0.f, 0.f, 0.f, 0.f};
#else
  unsigned sa = (unsigned)__cvta_generic_to_shared(sdst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(sa), "l"(gsrc), "r"(nbytes) : "memory");
#endif
}
MX_DEVINL void mx_cp4(float* sdst, const float* gsrc) {
#if MX_EMU
  *sdst = *gsrc;
#else
  unsigned sa = (unsigned)__cvta_generic_to_shared(sdst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(sa), "l"(gsrc) : "memory");
#endif
}
MX_DEVINL void mx_cp_commit() {
#if !MX_EMU
  asm volatile("cp.async.commit_group;" ::: "memory");
#endif
}
template <int N>
MX_DEVINL void mx_cp_wait() {   // wait until at most N of this thread's committed groups are still pending
#if !MX_EMU
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
#endif
}

// fast transcendental forms for the recurrences (absolute error ~2e-7): ex2.approx.ftz + rcp.approx.ftz, no range fix-ups -- the
// saturated cases fall out of IEEE inf / 0 arithmetic (ex2 -> +inf gives rcp -> 0; ex2 -> 0 gives rcp(1) = 1)
MX_DEVINL float mx_ex2(float x) {
#if MX_EMU
  return exp2f(x);
#else
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
#endif
}
MX_DEVINL float mx_rcp(float x) {
#if MX_EMU
  return 1.0f / x;
#else
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
#endif
}
MX_DEVINL float mx_sigmoid_fast(float x) { return mx_rcp(1.0f + mx_ex2(-1.4426950408889634f * x)); }
MX_DEVINL float mx_tanh_fast(float x) { return fmaf(2.0f, mx_rcp(1.0f + mx_ex2(-2.8853900817779268f * x)), -1.0f); }   // 2*sigmoid(2x) - 1

// two-lane fp32 FMA / add on float2 (sm_90 has no packed FFMA2: two FFMAs, the same rounding per lane)
MX_DEVINL float2 mx_ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
MX_DEVINL float2 mx_fadd2(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }

// LayerNorm statistics the way ATen's CPU/CUDA kernels define them: biased variance, eps inside the sqrt.
#define MX_LN_EPS 1e-5f
