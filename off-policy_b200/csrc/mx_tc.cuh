// wgmma / mbarrier building blocks (namespace tc) used by the tensor-core kernels (tc_linear.cu, tc_bwd.cu).
//
// The kernels are written against a "tensor memory" model: a [128 rows][columns] fp32 accumulator per CTA, filled by the MMAs of a
// layer and read back one row per thread (tmem_ld32 / tmem_ld64), so that bias, activation and LayerNorm run on registers with no
// cross-thread traffic.  On sm_90a the MMAs are wgmma.mma_async (m64nNk8, kind tf32, both operands K-major in shared memory, no
// swizzle): every warpgroup of the CTA takes a share of the (64-row half, column chunk) tiles, waits for its own wgmma group and
// writes the register fragments into the CTA's accumulator ([column][128 rows]: a tmem_ld of 32 consecutive rows is one coalesced
// 128-byte line).  The accumulator is the CTA's slice of a region the caller owns (the learner's workspace, sized by
// mx_tc_acc_floats; it stays in L2) or a shared-memory array; each thread then arrives on the layer's mbarrier (count = blockDim.x)
// and tmem_ld reads its row back after the wait.  Hopper has no tensor memory, and the wgmma fragment layout spreads a row over four
// lanes: the accumulator keeps the epilogues row-local at the price of one L2 round trip per layer.
//
// CPU-emulated unit-test build (MX_EMU, tests/emu): the same API restated on plain memory -- shared-memory descriptors are decoded
// with the no-swizzle K-major convention (LBO = stride between core matrices adjacent in K, SBO = stride between 8-row groups),
// operands are truncated to TF32 the way the tensor core reads them, the accumulator lives in a [128 lanes][512 columns] array, and
// thread 0 runs the MMAs synchronously and completes the mbarrier phase at once.  The emulation checks INDEXING and data flow
// (operand tiles, descriptors, accumulator rows / columns, barrier phases); it cannot see async-proxy hazards, which the fences in the
// kernels cover and only the GPU tests can confirm.
#pragma once
#include "mx_common.cuh"

#define MX_TC_ACC_SLOTS (264 * 256)     // the most accumulator columns (CTAs x columns per CTA) one launch uses: two CTAs per SM on a
                                        // 132-SM H100 at 256 columns each

#if !MX_EMU
#include <cuda.h>
namespace tc {

// the calling CTA's accumulator (set by tmem_alloc)
__device__ __forceinline__ float*& acc_ref() {
  __shared__ float* acc_s;
  return acc_s;
}
__device__ __forceinline__ float* acc_cta() { return acc_ref(); }
// CTA (blockIdx.x, blockIdx.y)'s slice of a caller-owned region of gridDim.x * gridDim.y * ncols * 128 floats
__device__ __forceinline__ float* cta_slice(float* base, int ncols) {
  return base + (size_t)(blockIdx.y * gridDim.x + blockIdx.x) * ncols * 128;
}

typedef unsigned long long Bar;      // mbarrier storage: `__shared__ __align__(8) tc::Bar bar_s;`
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint32_t op_addr(const void* p) { return smem_u32(p); }      // operand tile address for make_desc
__device__ __forceinline__ uint32_t bar_addr(Bar* b) { return smem_u32(b); }
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

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

// One (64-row half, NC-column chunk) tile of D = A . B^T over `passes` hi / lo products, issued by the calling warpgroup and
// written (acc = 0) or added (acc = 1) into the accumulator array.  Fragment of m64nNk8 (w = warp in the warpgroup, g = lane / 4,
// t = lane % 4): d[4j + i] = D[16w + g + 8 (i >> 1)][8j + 2t + (i & 1)].
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

// D[128][N] (+)= A[128][K] . B[N][K]^T into accumulator columns [col0, col0 + N), called by EVERY thread of the CTA: the work items
// (two 64-row halves x the 64- and 16-column chunks of N) are dealt round-robin to the CTA's warpgroups.  N % 16 == 0, K % 8 == 0.
__device__ __forceinline__ void mma_rows(uint32_t tmem_d, const char* a_hi, const char* a_lo, const char* b_hi, const char* b_lo, int N, int K,
                                         int passes, int swap_ls, uint32_t accumulate) {
  const uint32_t kstride = 128, mstride = (uint32_t)(K >> 2) * 128;
  const uint32_t lbo = swap_ls ? mstride : kstride, sbo = swap_ls ? kstride : mstride;
  float* acc = acc_cta();
  const int col0 = (int)(tmem_d & 0xFFFF);
  const int wg = threadIdx.x >> 7, nwg = blockDim.x >> 7;
  const int n64 = N >> 6, n16 = (N & 63) >> 4, nitems = 2 * (n64 + n16);
  for (int it = wg; it < nitems; it += nwg) {      // warpgroup-uniform
    const int half = it & 1, c = it >> 1;
    if (c < n64) mma_tile<64>(acc, col0, half, 64 * c, a_hi, a_lo, b_hi, b_lo, K, passes, lbo, sbo, accumulate);
    else mma_tile<16>(acc, col0, half, 64 * n64 + 16 * (c - n64), a_hi, a_lo, b_hi, b_lo, K, passes, lbo, sbo, accumulate);
  }
}

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
// every thread of the CTA arrives once its accumulator stores are done (release: the stores are visible to threads past the wait)
__device__ __forceinline__ void commit(uint32_t bar) {
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
// (ordering points of the accumulator around thread barriers: its reads and writes are ordinary loads and stores on sm_90a)
__device__ __forceinline__ void fence_before() {}
__device__ __forceinline__ void fence_after() {}

// Called by one warp before the CTA's first barrier: *slot (shared memory) receives the accumulator address (row 0, column 0) and
// `acc` (NCOLS x 128 floats, global or shared memory) becomes the CTA's accumulator.
template <int NCOLS>
__device__ __forceinline__ void tmem_alloc(uint32_t* slot, float* acc) {
  if ((threadIdx.x & 31) == 0) { *slot = 0; acc_ref() = acc; }
}
template <int NCOLS>
__device__ __forceinline__ void tmem_dealloc(uint32_t) {}
// address = (row << 16) | column; the calling thread reads row (address >> 16) + lane
__device__ __forceinline__ void tmem_ld32(uint32_t taddr, float (&v)[32]) {
  const float* p = acc_cta() + (size_t)(taddr & 0xFFFF) * 128 + (taddr >> 16) + (threadIdx.x & 31);
#pragma unroll
  for (int i = 0; i < 32; ++i) v[i] = p[(size_t)i * 128];
}
__device__ __forceinline__ void tmem_ld64(uint32_t taddr, float (&v)[64]) {
  const float* p = acc_cta() + (size_t)(taddr & 0xFFFF) * 128 + (taddr >> 16) + (threadIdx.x & 31);
#pragma unroll
  for (int i = 0; i < 64; ++i) v[i] = p[(size_t)i * 128];
}

__device__ __forceinline__ float to_tf32(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}

// write one element into the hi / lo operand tiles
__device__ __forceinline__ void put_split(char* hi, char* lo, int r, int k, int K, float x) {
  const float h = to_tf32(x);
  const uint32_t o = core_off_bytes(r, k, K);
  *reinterpret_cast<float*>(hi + o) = h;
  *reinterpret_cast<float*>(lo + o) = x - h;
}

// The MMAs of one layer: D[128][N] = A[128][K] . B[N][K]^T with `passes` = 1 (plain TF32) or 3 (3xTF32).  Called by every thread.
// swap_ls: which descriptor field carries the K-direction stride (probe of the no-swizzle convention).
__device__ __forceinline__ void issue_layer(uint32_t tmem_d, const char* a_hi, const char* a_lo, const char* b_hi, const char* b_lo, int N, int K,
                                            int passes, int swap_ls, uint32_t bar) {
  mma_rows(tmem_d, a_hi, a_lo, b_hi, b_lo, N, K, passes, swap_ls, 0u);
  commit(bar);
}

// Same, for a layer whose K dimension is fed in chunks (the operand tiles are refilled between calls): acc0 = 0 starts the
// accumulator, acc0 = 1 adds this chunk's products to what the previous calls left there.  The caller waits on `bar` after each call.
__device__ __forceinline__ void issue_layer_acc(uint32_t tmem_d, const char* a_hi, const char* a_lo, const char* b_hi, const char* b_lo, int N, int K,
                                                int swap_ls, uint32_t acc0, uint32_t bar, bool do_commit = true) {
  mma_rows(tmem_d, a_hi, a_lo, b_hi, b_lo, N, K, 3, swap_ls, acc0);
  if (do_commit) commit(bar);      // (one arrival may cover several groups of MMAs issued back to back)
}

}  // namespace tc

namespace tc {
#define MX_DYN_SMEM_RAW(name) extern __shared__ __align__(1024) unsigned char name[]
}
#else
#include <cassert>
namespace tc {

struct Bar { int phase, count, pending, pad; };
inline float g_tmem[128][512];
inline Bar* g_bars[64];
inline int g_nbars = 0;
inline char* emu_base() { return reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(emu::dyn_smem()) + 15) & ~uintptr_t(15)); }
#define MX_DYN_SMEM_RAW(name) unsigned char* name = reinterpret_cast<unsigned char*>(tc::emu_base())

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
inline uint32_t core_off_bytes(int r, int k, int K) { return (uint32_t)((r >> 3) * (K >> 2) * 128 + (k >> 2) * 128 + (r & 7) * 16 + (k & 3) * 4); }
inline uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  assert((saddr & 15) == 0 && (lbo_bytes & 15) == 0 && (sbo_bytes & 15) == 0 && (lbo_bytes >> 4) < 0x4000 && (sbo_bytes >> 4) < 0x4000);
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 46;
  return d;
}
inline uint32_t make_idesc_tf32(int M, int N) {
  assert(M == 128 && N % 16 == 0 && N >= 16 && N <= 256);
  uint32_t i = 0;
  i |= 1u << 4; i |= 2u << 7; i |= 2u << 10;
  i |= (uint32_t)(N >> 3) << 17;
  i |= (uint32_t)(M >> 4) << 24;
  return i;
}
inline float tf32_read(float x) { uint32_t u; memcpy(&u, &x, 4); u &= 0xFFFFE000u; memcpy(&x, &u, 4); return x; }      // the tensor core ignores the low 13 mantissa bits
inline void mma_tf32(uint32_t tmem_d, uint64_t adesc, uint64_t bdesc, uint32_t idesc, uint32_t accumulate) {
  const int N = (int)((idesc >> 17) & 0x3F) << 3, M = (int)((idesc >> 24) & 0x1F) << 4;
  const uint32_t sa = (uint32_t)(adesc & 0x3FFF) << 4, la = (uint32_t)((adesc >> 16) & 0x3FFF) << 4, ba = (uint32_t)((adesc >> 32) & 0x3FFF) << 4;
  const uint32_t sb = (uint32_t)(bdesc & 0x3FFF) << 4, lb = (uint32_t)((bdesc >> 16) & 0x3FFF) << 4, bb = (uint32_t)((bdesc >> 32) & 0x3FFF) << 4;
  const char* base = emu_base();
  const int lane0 = (int)(tmem_d >> 16), col0 = (int)(tmem_d & 0xFFFF);
  assert(lane0 == 0 && col0 + N <= 512 && M == 128);
  for (int r = 0; r < M; ++r)
    for (int n = 0; n < N; ++n) {
      double acc = accumulate ? (double)g_tmem[r][col0 + n] : 0.0;      // exact products, one rounding per instruction (the tensor core adds the K = 8 products in a wide adder)
      for (int k = 0; k < 8; ++k) {
        const float av = tf32_read(*reinterpret_cast<const float*>(base + sa + (r >> 3) * ba + (k >> 2) * la + (r & 7) * 16 + (k & 3) * 4));
        const float bv = tf32_read(*reinterpret_cast<const float*>(base + sb + (n >> 3) * bb + (k >> 2) * lb + (n & 7) * 16 + (k & 3) * 4));
        acc += (double)av * (double)bv;
      }
      g_tmem[r][col0 + n] = (float)acc;
    }
}
inline void commit(uint32_t bar) { Bar* b = g_bars[bar]; b->phase ^= 1; emu::g.progress++; }      // MMAs ran synchronously: the phase completes at once
inline void mbar_init(uint32_t bar, uint32_t count) { Bar* b = g_bars[bar]; b->phase = 0; b->count = (int)count; b->pending = 0; }
inline void mbar_wait(uint32_t bar, uint32_t parity) { Bar* b = g_bars[bar]; while ((uint32_t)b->phase == parity) emu::yield(); }
inline void fence_async_smem() {}
inline void fence_before() {}
inline void fence_after() {}
template <int NCOLS> inline void tmem_alloc(uint32_t* slot, float*) { *slot = 0; }      // (the emulated accumulator is g_tmem)
inline float* cta_slice(float* base, int) { return base; }
template <int NCOLS> inline void tmem_dealloc(uint32_t) {}
inline void tmem_check(uint32_t taddr, int ncols) {
  assert((int)(taddr >> 16) == 32 * (emu::cur->warp & 3) && "a warp reads the 32 accumulator rows of its quadrant");
  assert((int)(taddr & 0xFFFF) + ncols <= 512);
}
inline void tmem_ld32(uint32_t taddr, float (&v)[32]) {
  tmem_check(taddr, 32);
  const int row = (int)(taddr >> 16) + emu::cur->lane, c0 = (int)(taddr & 0xFFFF);
  for (int i = 0; i < 32; ++i) v[i] = g_tmem[row][c0 + i];
}
inline void tmem_ld64(uint32_t taddr, float (&v)[64]) {
  tmem_check(taddr, 64);
  const int row = (int)(taddr >> 16) + emu::cur->lane, c0 = (int)(taddr & 0xFFFF);
  for (int i = 0; i < 64; ++i) v[i] = g_tmem[row][c0 + i];
}
inline float to_tf32(float x) {      // cvt.rna.tf32.f32: round to nearest, ties away from zero, 10 mantissa bits
  uint32_t u; memcpy(&u, &x, 4); u += 0x1000u; u &= 0xFFFFE000u; memcpy(&x, &u, 4); return x;
}
inline void put_split(char* hi, char* lo, int r, int k, int K, float x) {
  const float h = to_tf32(x);
  const uint32_t o = core_off_bytes(r, k, K);
  *reinterpret_cast<float*>(hi + o) = h;
  *reinterpret_cast<float*>(lo + o) = x - h;
}
inline void issue_layer(uint32_t tmem_d, const char* a_hi, const char* a_lo, const char* b_hi, const char* b_lo, int N, int K, int passes, int swap_ls,
                        uint32_t bar) {
  if (threadIdx.x != 0) return;      // every thread calls; thread 0 runs the MMAs
  const uint32_t kstride = 128, mstride = (uint32_t)(K >> 2) * 128;
  const uint32_t lbo = swap_ls ? mstride : kstride, sbo = swap_ls ? kstride : mstride;
  const uint32_t idesc = make_idesc_tf32(128, N);
  uint32_t acc = 0;
  for (int p = 0; p < passes; ++p) {
    const char* a = (p == 1) ? a_lo : a_hi;
    const char* b = (p == 2) ? b_lo : b_hi;
    for (int k8 = 0; k8 < K / 8; ++k8) {
      mma_tf32(tmem_d, make_desc(op_addr(a) + k8 * 256, lbo, sbo), make_desc(op_addr(b) + k8 * 256, lbo, sbo), idesc, acc);
      acc = 1;
    }
  }
  commit(bar);
}

// Same, for a layer whose K dimension is fed in chunks (the operand tiles are refilled between calls): acc0 = 0 starts the
// accumulator, acc0 = 1 adds this chunk's products to what the previous calls left in the accumulator.  The caller waits on `bar` after each call.
inline void issue_layer_acc(uint32_t tmem_d, const char* a_hi, const char* a_lo, const char* b_hi, const char* b_lo, int N, int K,
                                                int swap_ls, uint32_t acc0, uint32_t bar, bool do_commit = true) {
  if (threadIdx.x != 0) return;
  const uint32_t kstride = 128, mstride = (uint32_t)(K >> 2) * 128;
  const uint32_t lbo = swap_ls ? mstride : kstride, sbo = swap_ls ? kstride : mstride;
  const uint32_t idesc = make_idesc_tf32(128, N);
  uint32_t acc = acc0;
  for (int p = 0; p < 3; ++p) {
    const char* a = (p == 1) ? a_lo : a_hi;      // hi*hi, lo*hi, hi*lo
    const char* b = (p == 2) ? b_lo : b_hi;
    for (int k8 = 0; k8 < K / 8; ++k8) {
      mma_tf32(tmem_d, make_desc(op_addr(a) + k8 * 256, lbo, sbo), make_desc(op_addr(b) + k8 * 256, lbo, sbo), idesc, acc);
      acc = 1;
    }
  }
  if (do_commit) commit(bar);      // (one commit may cover several groups of MMAs issued back to back)
}

}  // namespace tc
#endif
