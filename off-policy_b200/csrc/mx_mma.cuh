// Warp-level tensor-core tiles for the FP32-accurate backward GEMMs: mma.sync.m16n8k8 TF32 with the 3xTF32 split
// (hi = cvt.rna.tf32(x), lo = x - hi; D += lo*hi + hi*lo + hi*hi, fp32 accumulate in registers: relative error ~2^-21, the same
// accuracy class as the wgmma forward).  The FFMA micro-kernels of mx_tile.cuh are bound by the shared-memory pipe (one 16-byte
// load per 6-8 FFMAs, and a wide load occupies the LSU for four cycles); a fragment loaded once here feeds 3 x 1024 MACs.
//
// Fragment layout of mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 (g = lane >> 2, t = lane & 3):
//   A (16 x 8): a0 = A[g][t]      a1 = A[g + 8][t]      a2 = A[g][t + 4]      a3 = A[g + 8][t + 4]
//   B (8 x 8):  b0 = B[t][g]      b1 = B[t + 4][g]
//   C (16 x 8): c0 = C[g][2t]     c1 = C[g][2t + 1]     c2 = C[g + 8][2t]     c3 = C[g + 8][2t + 1]
//
// CPU-emulated build: the same fragments, the product computed from a per-warp scratch (operands truncated to TF32 the way the
// tensor core reads them, exact products, one rounding per instruction).
#pragma once
#include "mx_common.cuh"

struct MxFragA { float hi[4], lo[4]; };
struct MxFragB { float hi[2], lo[2]; };

#if !MX_EMU
MX_DEVINL float mx_tf32_rna(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}
MX_DEVINL void mx_mma_1688(float (&c)[4], const float (&a)[4], const float (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(__float_as_uint(a[0])), "r"(__float_as_uint(a[1])), "r"(__float_as_uint(a[2])), "r"(__float_as_uint(a[3])),
                 "r"(__float_as_uint(b[0])), "r"(__float_as_uint(b[1])));
}
#else
#include <string.h>
inline float mx_tf32_rna(float x) { uint32_t u; memcpy(&u, &x, 4); u += 0x1000u; u &= 0xFFFFE000u; memcpy(&x, &u, 4); return x; }
inline float mx_tf32_trunc(float x) { uint32_t u; memcpy(&u, &x, 4); u &= 0xFFFFE000u; memcpy(&x, &u, 4); return x; }
inline void mx_mma_1688(float (&c)[4], const float (&a)[4], const float (&b)[2]) {
  static float sa[64][32][4], sb[64][32][2];      // [warp][lane][reg]: one CTA runs at a time in the emulator
  const int w = emu::cur->warp, lane = emu::cur->lane, g = lane >> 2, t = lane & 3;
  for (int i = 0; i < 4; ++i) sa[w][lane][i] = mx_tf32_trunc(a[i]);
  for (int i = 0; i < 2; ++i) sb[w][lane][i] = mx_tf32_trunc(b[i]);
  emu::warp_barrier();
  auto A = [&](int r, int k) { return sa[w][4 * (r & 7) + (k & 3)][(r >> 3) + 2 * (k >> 2)]; };
  auto B = [&](int k, int n) { return sb[w][4 * n + (k & 3)][k >> 2]; };
  const int rows[4] = {g, g, g + 8, g + 8}, cols[4] = {2 * t, 2 * t + 1, 2 * t, 2 * t + 1};
  for (int o = 0; o < 4; ++o) {
    double acc = (double)c[o];
    for (int k = 0; k < 8; ++k) acc += (double)A(rows[o], k) * (double)B(k, cols[o]);
    c[o] = (float)acc;
  }
  emu::warp_barrier();
}
#endif

MX_DEVINL void mx_split_a(MxFragA& f, float a0, float a1, float a2, float a3) {
  const float v[4] = {a0, a1, a2, a3};
#pragma unroll
  for (int i = 0; i < 4; ++i) { f.hi[i] = mx_tf32_rna(v[i]); f.lo[i] = v[i] - f.hi[i]; }
}
MX_DEVINL void mx_split_b(MxFragB& f, float b0, float b1) {
  f.hi[0] = mx_tf32_rna(b0); f.lo[0] = b0 - f.hi[0];
  f.hi[1] = mx_tf32_rna(b1); f.lo[1] = b1 - f.hi[1];
}
// C += A . B with fp32-level accuracy (small terms first)
MX_DEVINL void mx_mma3(float (&c)[4], const MxFragA& a, const MxFragB& b) {
  mx_mma_1688(c, a.lo, b.hi);
  mx_mma_1688(c, a.hi, b.lo);
  mx_mma_1688(c, a.hi, b.hi);
}

// ---- data gradient: C[r][8w + ..] += sum_{n < 64} dY_s[r][n] * Wc[n][kcol0 + 8w + ..] for the MT 16-row tiles of the CTA tile; warp w (0..7)
// owns the 8 output columns [8w, 8w + 8).  Accumulates into c[MT][4] (C-fragment layout) so that several weight chunks can be summed.
template <int MT>
MX_DEVINL void mx_mma_dgrad_acc(float (&c)[MT][4], const float* __restrict__ dY_s, int ldy, const float* __restrict__ Wc, int ldw) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
#pragma unroll 2
  for (int ks = 0; ks < 8; ++ks) {
    MxFragB b;
    mx_split_b(b, Wc[(8 * ks + t) * ldw + 8 * w + g], Wc[(8 * ks + t + 4) * ldw + 8 * w + g]);
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      const float* d = dY_s + (16 * mt + g) * ldy + 8 * ks + t;
      MxFragA a;
      mx_split_a(a, d[0], d[8 * ldy], d[4], d[8 * ldy + 4]);
      mx_mma3(c[mt], a, b);
    }
  }
}
// C fragments -> out_s[r][8w + ..] (row-major tile in shared memory, 8-byte stores)
template <int MT>
MX_DEVINL void mx_mma_store(const float (&c)[MT][4], float* __restrict__ out_s, int ldo) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int mt = 0; mt < MT; ++mt) {
    float* o = out_s + (16 * mt + g) * ldo + 8 * w + 2 * t;
    o[0] = c[mt][0]; o[1] = c[mt][1];
    o[8 * ldo] = c[mt][2]; o[8 * ldo + 1] = c[mt][3];
  }
}

// ---- weight gradient of one 64(n) x 64(k) output block over the TM rows of the tile (TM % 8 == 0):
//   dW[nb + n][kb + k] (+)= sum_r dY_s[r][n] * X_s[r][k]     (caller offsets dY_s to column nb and X_s to column kb)
// The contraction runs over the tile ROWS, so both operands are read "transposed" from their row-major tiles; warp w owns the 8 output
// columns k in [8w, 8w + 8) for all four 16-row (n) tiles.
MX_DEVINL void mx_mma_wgrad_block(const float* __restrict__ dY_s, int ldy, const float* __restrict__ X_s, int ldx, int TM, float* __restrict__ dW,
                                  int N, int K, int nb, int kb, bool accumulate) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
  if (kb + 8 * w >= K) return;        // this warp's columns are all outside (warp-uniform; no barriers inside)
  float c[4][4];
#pragma unroll
  for (int mt = 0; mt < 4; ++mt)
#pragma unroll
    for (int i = 0; i < 4; ++i) c[mt][i] = 0.f;
  for (int ks = 0; ks < TM / 8; ++ks) {
    const float* xr = X_s + (8 * ks + t) * ldx + 8 * w + g;
    MxFragB b;
    mx_split_b(b, xr[0], xr[4 * ldx]);
    const float* dr = dY_s + (8 * ks + t) * ldy + g;
#pragma unroll
    for (int mt = 0; mt < 4; ++mt) {
      MxFragA a;
      mx_split_a(a, dr[16 * mt], dr[16 * mt + 8], dr[4 * ldy + 16 * mt], dr[4 * ldy + 16 * mt + 8]);
      mx_mma3(c[mt], a, b);
    }
  }
#pragma unroll
  for (int mt = 0; mt < 4; ++mt)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int n = nb + 16 * mt + g + ((i >> 1) ? 8 : 0), k = kb + 8 * w + 2 * t + (i & 1);
      if (n < N && k < K) {
        float* p = dW + (size_t)n * K + k;
        *p = accumulate ? (*p + c[mt][i]) : c[mt][i];
      }
    }
}
