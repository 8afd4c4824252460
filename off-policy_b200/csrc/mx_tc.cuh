// wgmma / mbarrier building blocks (namespace tc) used by the tensor-core kernels (tc_linear.cu, tc_bwd.cu, mixer_wide.cu).
//
// A layer is D[128][N] (+)= A[128][K] . B[N][K]^T with both operands K-major in shared memory (no swizzle, core matrices of 8 rows x
// 16 bytes; LBO = stride between core matrices adjacent in K, SBO = stride between 8-row groups).  tc::mma runs it as
// wgmma.mma_async m64nNk8 (kind tf32): every warpgroup of the CTA takes a share of the (64-row half, column chunk) tiles, waits for its
// own wgmma group and stores the register fragments into the CTA's accumulator `acc`, an fp32 [column][128 rows] array.  `acc` is the
// CTA's slice of a region the caller owns (tc::cta_slice of the learner's workspace, sized by mx_tc_acc_floats; it stays in L2) or a
// shared-memory array.  Each thread then arrives on the layer's mbarrier (tc::arrive, count = blockDim.x) and, after the wait, reads
// its row back with tc::ld_row (32 consecutive rows of a column are one coalesced 128-byte line), so that bias, activation and
// LayerNorm run on registers with no cross-thread traffic.  The wgmma fragment layout spreads a row over four lanes: the accumulator
// keeps the epilogues row-local at the price of one L2 round trip per layer.
//
// CPU-emulated unit-test build (MX_EMU, tests/emu): only the instruction-level primitives are restated on plain memory.  The emulated
// wgmma decodes the two shared-memory descriptors with the convention above, truncates the operands to TF32 the way the tensor core
// reads them and adds into the calling thread's own fragment registers, synchronously; mbarriers count their arrivals.  Everything
// built on those primitives (tile dealing, fragment placement, accumulator slices, arrivals) is the code the GPU runs.  The emulation
// cannot see async-proxy hazards, which fence_async_smem covers and only the GPU tests can confirm.
#pragma once
#include "mx_common.cuh"

#define MX_TC_ACC_SLOTS (264 * 256)     // the most accumulator columns (CTAs x columns per CTA) one launch uses: two CTAs per SM on a
                                        // 132-SM H100 at 256 columns each

#if !MX_EMU
#include <cuda.h>
#define MX_DYN_SMEM_RAW(name) extern __shared__ __align__(1024) unsigned char name[]
namespace tc {

typedef unsigned long long Bar;      // mbarrier storage: `__shared__ __align__(8) tc::Bar bar_s;`
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint32_t op_addr(const void* p) { return smem_u32(p); }      // operand tile address for make_desc
__device__ __forceinline__ uint32_t bar_addr(Bar* b) { return smem_u32(b); }
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit_wait() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
}
// D[64][64] += A[64][8] . B[64][8]^T
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t ad, uint64_t bd) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
      "%32, %33, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]),
        "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]),
        "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(ad), "l"(bd), "r"(1));
}
// D[64][16] += A[64][8] . B[16][8]^T
__device__ __forceinline__ void wgmma_n16(float (&d)[8], uint64_t ad, uint64_t bd) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(ad), "l"(bd), "r"(1));
}

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
// every thread of the CTA arrives once its accumulator stores are done (release: the stores are visible to threads past the wait)
__device__ __forceinline__ void arrive(uint32_t bar) {
  __threadfence_block();
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}\n" ::"r"(bar) : "memory");
}
// Bounded wait: a barrier that is never completed (a lost arrival) traps after ~2 s instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  long long t0 = 0;
  for (uint32_t it = 0; !done; ++it) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (!done && (it & 1023u) == 1023u) {
      const long long now = clock64();
      if (t0 == 0) t0 = now;
      else if (now - t0 > 4000000000LL) __trap();
    }
  }
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ float to_tf32(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}

}  // namespace tc
#else
#include <cassert>
#define MX_DYN_SMEM_RAW(name) unsigned char* name = reinterpret_cast<unsigned char*>(tc::emu_base())
namespace tc {

struct Bar { int phase, count, pending, pad; };
inline Bar* g_bars[64];
inline int g_nbars = 0;
inline char* emu_base() { return reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(emu::dyn_smem()) + 15) & ~uintptr_t(15)); }

inline uint32_t op_addr(const void* p) {
  const ptrdiff_t o = reinterpret_cast<const char*>(p) - emu_base();
  assert(o >= 0 && o < (1 << 18) && (o & 15) == 0 && "operand tiles live in dynamic shared memory, 16-byte aligned");
  return (uint32_t)o;
}
inline uint32_t bar_addr(Bar* b) {
  for (int i = 0; i < g_nbars; ++i) if (g_bars[i] == b) return (uint32_t)i;
  assert(g_nbars < 64);
  g_bars[g_nbars] = b;
  return (uint32_t)g_nbars++;
}
inline void mbar_init_fence() {}

// the emulated instructions are synchronous: nothing to fence, commit or wait for
inline void wg_fence() {}
inline void wg_commit_wait() {}
inline float tf32_read(float x) { uint32_t u; memcpy(&u, &x, 4); u &= 0xFFFFE000u; memcpy(&x, &u, 4); return x; }      // the tensor core ignores the low 13 mantissa bits
// element (r, k) of a K-major no-swizzle operand from its descriptor: start, LBO (K direction) and SBO (8-row groups), 16-byte units
inline float desc_elem(uint64_t desc, int r, int k) {
  const uint32_t start = (uint32_t)(desc & 0x3FFF) << 4, lbo = (uint32_t)((desc >> 16) & 0x3FFF) << 4, sbo = (uint32_t)((desc >> 32) & 0x3FFF) << 4;
  return tf32_read(*reinterpret_cast<const float*>(emu_base() + start + (r >> 3) * sbo + (k >> 2) * lbo + (r & 7) * 16 + (k & 3) * 4));
}
// wgmma.mma_async m64nNk8 f32.tf32.tf32 for the calling thread.  Accumulator fragment (PTX ISA, "wgmma .m64nNk8 register fragment
// layout for accumulator matrix D"): warp w of the warpgroup holds rows 16 w .. 16 w + 15; in it, with groupID = laneid / 4 and
// threadID_in_group = laneid % 4, register d[i] is element (groupID + 8 * ((i % 4) / 2), 8 * (i / 4) + 2 * threadID_in_group + (i % 2)).
// Exact products, one rounding per instruction (the tensor core adds the K = 8 products in a wide adder).
template <int N>
inline void wgmma_emu(float (&d)[N / 2], uint64_t ad, uint64_t bd) {
  const int w = emu::cur->warp % 4, group_id = emu::cur->lane / 4, tig = emu::cur->lane % 4;
  for (int i = 0; i < N / 2; ++i) {
    const int row = 16 * w + group_id + 8 * ((i % 4) / 2), col = 8 * (i / 4) + 2 * tig + (i % 2);
    double s = d[i];
    for (int k = 0; k < 8; ++k) s += (double)desc_elem(ad, row, k) * (double)desc_elem(bd, col, k);
    d[i] = (float)s;
  }
}
inline void wgmma_n64(float (&d)[32], uint64_t ad, uint64_t bd) { wgmma_emu<64>(d, ad, bd); }
inline void wgmma_n16(float (&d)[8], uint64_t ad, uint64_t bd) { wgmma_emu<16>(d, ad, bd); }

inline void mbar_init(uint32_t bar, uint32_t count) { Bar* b = g_bars[bar]; b->phase = 0; b->count = (int)count; b->pending = 0; }
// the phase completes with the count-th arrival: a kernel that loses one stops at the emulator's deadlock check
inline void arrive(uint32_t bar) {
  Bar* b = g_bars[bar];
  if (++b->pending == b->count) { b->pending = 0; b->phase ^= 1; }
  emu::g.progress++;
}
inline void mbar_wait(uint32_t bar, uint32_t parity) { Bar* b = g_bars[bar]; while ((uint32_t)b->phase == parity) emu::yield(); }
inline void fence_async_smem() {}
inline float to_tf32(float x) {      // cvt.rna.tf32.f32: round to nearest, ties away from zero, 10 mantissa bits
  uint32_t u; memcpy(&u, &x, 4); u += 0x1000u; u &= 0xFFFFE000u; memcpy(&x, &u, 4); return x;
}

}  // namespace tc
#endif

namespace tc {

// K-major, no swizzle: element (r, k) of a [rows][K] fp32/tf32 operand.  Core matrix = 8 rows x 4 elements (16 B per row).
// Physical arrangement used here: the K/4 core matrices of one 8-row group are contiguous (128 B apart), 8-row groups
// follow each other ((K/4)*128 B apart).
__device__ __forceinline__ uint32_t core_off_bytes(int r, int k, int K) {
  return (uint32_t)((r >> 3) * (K >> 2) * 128 + (k >> 2) * 128 + (r & 7) * 16 + (k & 3) * 4);
}

// wgmma shared-memory matrix descriptor (sm_90): start>>4 [0,14) | LBO>>4 [16,30) | SBO>>4 [32,46) | base offset 0 | layout [62,64) = 0
// (no swizzle: interleaved core matrices)
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  return d;
}

// write one element into the hi / lo operand tiles
__device__ __forceinline__ void put_split(char* hi, char* lo, int r, int k, int K, float x) {
  const float h = to_tf32(x);
  const uint32_t o = core_off_bytes(r, k, K);
  *reinterpret_cast<float*>(hi + o) = h;
  *reinterpret_cast<float*>(lo + o) = x - h;
}

// CTA (blockIdx.x, blockIdx.y)'s accumulator: its slice of a caller-owned region of gridDim.x * gridDim.y * ncols * 128 floats
__device__ __forceinline__ float* cta_slice(float* base, int ncols) {
  return base + (size_t)(blockIdx.y * gridDim.x + blockIdx.x) * ncols * 128;
}

// One (64-row half, NC-column chunk) tile of D = A . B^T over `passes` hi / lo products, issued by the calling warpgroup and
// written (accumulate = 0) or added (accumulate = 1) into the accumulator.  Fragment of m64nNk8 (w = warp in the warpgroup,
// g = lane / 4, t = lane % 4): d[4j + i] = D[16w + g + 8 (i >> 1)][8j + 2t + (i & 1)].
template <int NC>
__device__ __forceinline__ void mma_tile(float* acc, int col0, int half, int n0, const char* a_hi, const char* a_lo, const char* b_hi,
                                         const char* b_lo, int K, int passes, uint32_t lbo, uint32_t sbo, uint32_t accumulate) {
  float d[NC / 2];
#pragma unroll
  for (int i = 0; i < NC / 2; ++i) d[i] = 0.f;
  const uint32_t grp = (uint32_t)(K >> 2) * 128;      // bytes per 8-row group
  wg_fence();
  for (int p = 0; p < passes; ++p) {
    const char* a = (p == 1) ? a_lo : a_hi;      // hi*hi, lo*hi, hi*lo
    const char* b = (p == 2) ? b_lo : b_hi;
    const uint32_t ab = op_addr(a) + (uint32_t)(8 * half) * grp, bb = op_addr(b) + (uint32_t)(n0 >> 3) * grp;
    for (int k8 = 0; k8 < K / 8; ++k8) {
      const uint64_t ad = make_desc(ab + k8 * 256, lbo, sbo), bd = make_desc(bb + k8 * 256, lbo, sbo);
      if constexpr (NC == 64) wgmma_n64(d, ad, bd); else wgmma_n16(d, ad, bd);
    }
  }
  wg_commit_wait();
  const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
  const int row = 64 * half + 16 * w + (lane >> 2), c = col0 + n0 + 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < NC / 8; ++j)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float* o = acc + (size_t)(c + 8 * j + (i & 1)) * 128 + row + 8 * (i >> 1);
      *o = accumulate ? *o + d[4 * j + i] : d[4 * j + i];
    }
}

// The MMAs of one layer: D[128][N] = A[128][K] . B[N][K]^T (accumulate = 0) or += (accumulate = 1, a K dimension fed in chunks) into
// accumulator columns [col0, col0 + N), with `passes` = 1 (plain TF32) or 3 (3xTF32).  Called by EVERY thread of the CTA: the work
// items (two 64-row halves x the 64- and 16-column chunks of N) are dealt round-robin to the CTA's warpgroups.  N % 16 == 0, K % 8 == 0.
// The caller arrives on the layer's mbarrier afterwards (one arrival may cover several calls).  swap_ls puts the K-direction stride in
// SBO instead of LBO: only the probe of the descriptor convention (mx_tc_linear_probe) sets it.
__device__ __forceinline__ void mma(float* acc, int col0, const char* a_hi, const char* a_lo, const char* b_hi, const char* b_lo, int N, int K,
                                    int passes, uint32_t accumulate, int swap_ls = 0) {
  const uint32_t kstride = 128, mstride = (uint32_t)(K >> 2) * 128;
  const uint32_t lbo = swap_ls ? mstride : kstride, sbo = swap_ls ? kstride : mstride;
  const int wg = threadIdx.x >> 7, nwg = blockDim.x >> 7;
  const int n64 = N >> 6, n16 = (N & 63) >> 4, nitems = 2 * (n64 + n16);
  for (int it = wg; it < nitems; it += nwg) {      // warpgroup-uniform
    const int half = it & 1, c = it >> 1;
    if (c < n64) mma_tile<64>(acc, col0, half, 64 * c, a_hi, a_lo, b_hi, b_lo, K, passes, lbo, sbo, accumulate);
    else mma_tile<16>(acc, col0, half, 64 * n64 + 16 * (c - n64), a_hi, a_lo, b_hi, b_lo, K, passes, lbo, sbo, accumulate);
  }
}

// columns [col0, col0 + NV) of accumulator row `row` (after the layer's mbarrier wait)
template <int NV>
__device__ __forceinline__ void ld_row(const float* acc, int col0, int row, float (&v)[NV]) {
  const float* p = acc + (size_t)col0 * 128 + row;
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = p[(size_t)i * 128];
}

}  // namespace tc
