// Tensor-core (wgmma) dense layers with fp32-level accuracy: Y[M][N] = X[M][K] . W[N][K]^T (+ bias)
//
// Operands are split on the fly into TF32 hi / lo parts (hi = cvt.rna.tf32, lo = x - hi) and three MMAs accumulate
// hi*hi + lo*hi + hi*lo in fp32 ("3xTF32": relative error ~2^-21, inside the 1e-4 gradient parity budget that rules single-pass
// TF32/BF16 out).  One CTA = one 128-row tile:
//   all threads : fill A (and W) hi/lo tiles in shared memory in the canonical K-major no-swizzle core-matrix layout
//                 (8 rows x 16 bytes per core matrix), fence.proxy.async, barrier
//   warpgroups  : wgmma.mma_async m64nNk8 kind tf32 over their share of the tile (mx_tc.cuh), fragments -> the CTA's accumulator,
//                 mbarrier arrival
//   all threads : mbarrier wait, read the accumulator row (thread = row), epilogue, global stores
// This file holds the front-layer kernels and a probe entry point (mx_tc_linear_probe) used by the GPU tests to pin the
// descriptor conventions against an fp64 reference.
#include "mx_internal.h"

#include "mx_tc.cuh"
#include <string.h>

// =====================================================================================================
// front forward on the tensor cores: LN -> fc1 -> ReLU -> LN -> fc2 -> ReLU -> LN -> W_ih for a 128-row tile per CTA.
// Thread r owns accumulator row r: after tc::ld_row a whole 64-wide layer output sits in that thread's
// registers, so bias / ReLU / LayerNorm need no cross-thread traffic at all; the normalised row is split into TF32
// hi/lo and written straight back into the A operand tiles for the next layer.
// =====================================================================================================
#include "mx_kernels.h"

struct FrontTcSmem { int o_ahi, o_alo, o_w1h, o_w1l, o_w2h, o_w2l, o_wih, o_wil, total; };
static FrontTcSmem front_tc_smem(int Kp) {
  FrontTcSmem s;
  int o = 0;
  s.o_ahi = o; o += 128 * 64 * 4;
  s.o_alo = o; o += 128 * 64 * 4;
  s.o_w1h = o; o += 64 * Kp * 4;
  s.o_w1l = o; o += 64 * Kp * 4;
  s.o_w2h = o; o += 64 * 64 * 4;
  s.o_w2l = o; o += 64 * 64 * 4;
  s.o_wih = o; o += 192 * 64 * 4;
  s.o_wil = o; o += 192 * 64 * 4;
  s.total = o;
  return s;
}

__device__ __forceinline__ void tc_stage_weight(char* hi, char* lo, const float* __restrict__ W, int N, int K, int Kp) {
  for (int idx = threadIdx.x; idx < N * Kp; idx += blockDim.x) {
    const int n = idx / Kp, k = idx - n * Kp;
    tc::put_split(hi, lo, n, k, Kp, k < K ? W[(size_t)n * K + k] : 0.f);
  }
}

// Weight images: [w1 hi | w1 lo | w2 hi | w2 lo | w_ih hi | w_ih lo], each already in the wgmma core-matrix layout, so a CTA
// stages all three layers with straight 16-byte cp.async copies (no per-CTA conversion).  Rebuilt once per step.
struct TcPrepArgs { const float* th[2]; float* img[2]; };
// fc1 image: in_dim <= 64: one [64][Kp] tile.  64 < in_dim <= 128 ("wide"): K is fed in chunks of 64 columns, each chunk its own
// [64][Kc] hi | lo tile pair (Kc = 64, then round_up(in_dim - 64, 8)); the floats add up to 64 * Kp either way.
__device__ __forceinline__ void tc_w1_image_slot(int n, int k, int Kp, char* base, char** hi, char** lo, int* kk, int* Kd) {
  if (Kp <= 64) { *hi = base; *lo = base + 64 * Kp * 4; *kk = k; *Kd = Kp; return; }
  const int c = k >> 6, Kc = c == 0 ? 64 : Kp - 64;
  char* chunk = base + (c == 0 ? 0 : 2 * 64 * 64 * 4);
  *hi = chunk; *lo = chunk + 64 * Kc * 4; *kk = k & 63; *Kd = Kc;
  (void)n;
}
__global__ void __launch_bounds__(256) k_tc_prep_weights(TcPrepArgs p, MxNetLayout L) {
  const float* __restrict__ th = p.th[blockIdx.y];
  const int I = L.in_dim, Kp = (I + 7) & ~7;
  const int n1 = MX_H * Kp, n2 = MX_H * MX_H, n3 = MX_G * MX_H;
  char* base = reinterpret_cast<char*>(p.img[blockIdx.y]);
  MX_PDL_WAIT();
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < n1 + n2 + n3; idx += gridDim.x * blockDim.x) {
    int n, k, K, Kd;
    const float* W;
    char *hi, *lo;
    if (idx < n1) {
      n = idx / Kp; k = idx - n * Kp; K = I; W = th + L.w1;
      const float x = k < K ? W[(size_t)n * K + k] : 0.f;
      int kk;
      tc_w1_image_slot(n, k, Kp, base, &hi, &lo, &kk, &Kd);
      tc::put_split(hi, lo, n, kk, Kd, x);
      continue;
    }
    else if (idx < n1 + n2) { const int j = idx - n1; n = j / MX_H; k = j % MX_H; K = MX_H; Kd = MX_H; W = th + L.w2; hi = base + 2 * n1 * 4; lo = hi + n2 * 4; }
    else { const int j = idx - n1 - n2; n = j / MX_H; k = j % MX_H; K = MX_H; Kd = MX_H; W = th + L.wih; hi = base + (2 * n1 + 2 * n2) * 4; lo = hi + n3 * 4; }
    tc::put_split(hi, lo, n, k, Kd, k < K ? W[(size_t)n * K + k] : 0.f);
  }
}

size_t mx_tc_acc_floats(int64_t M) {
  // the widest user is k_wgrad_tc: 512 columns per CTA, at most one CTA per 64-row chunk (the forward: 2 nets x 256 per 128-row tile)
  const int64_t need = (M > 0 ? (M + 63) / 64 : 1) * 512;
  return (size_t)(need < MX_TC_ACC_SLOTS ? need : MX_TC_ACC_SLOTS) * 128;
}
size_t mx_tc_image_floats(int in_dim) {
  const int Kp = mx_round_up(in_dim, 8);
  return (size_t)2 * (MX_H * Kp + MX_H * MX_H + MX_G * MX_H);
}
// one launch for `nets` parameter vectors (live, target)
int mx_launch_tc_prep_weights(const float* const theta[2], const MxNetLayout& L, float* const img[2], int nets, cudaStream_t s) {
  const int n = MX_H * mx_round_up(L.in_dim, 8) + MX_H * MX_H + MX_G * MX_H;
  TcPrepArgs p;
  for (int k = 0; k < 2; ++k) { p.th[k] = theta[k < nets ? k : 0]; p.img[k] = img[k < nets ? k : 0]; }
  return mx_launch("k_tc_prep_weights", k_tc_prep_weights, dim3((n + 255) / 256, nets), dim3(256), 0, s, MX_STEP, p, L);
}

// 64-term sums on 8 independent chains (a thread owns a whole row: no other warp hides FADD latency for it)
__device__ __forceinline__ float tc_sum64(const float (&v)[64]) {
  float p[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) p[i] = v[i];
#pragma unroll
  for (int c = 8; c < 64; c += 8)
#pragma unroll
    for (int i = 0; i < 8; ++i) p[i] += v[c + i];
  return ((p[0] + p[1]) + (p[2] + p[3])) + ((p[4] + p[5]) + (p[6] + p[7]));
}
__device__ __forceinline__ float tc_sumsq64(const float (&v)[64], float mean, int n_valid) {
  float p[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) p[i] = 0.f;
#pragma unroll
  for (int c = 0; c < 64; c += 8)
#pragma unroll
    for (int i = 0; i < 8; ++i) { const float d = (c + i < n_valid) ? v[c + i] - mean : 0.f; p[i] = fmaf(d, d, p[i]); }
  return ((p[0] + p[1]) + (p[2] + p[3])) + ((p[4] + p[5]) + (p[6] + p[7]));
}

// write this thread's row (64 values) into the A tiles, 16 bytes at a time
__device__ __forceinline__ void tc_put_row64(char* hi, char* lo, int r, const float (&x)[64]) {
#pragma unroll
  for (int k4 = 0; k4 < 16; ++k4) {
    float4 h, l;
    h.x = tc::to_tf32(x[4 * k4]); h.y = tc::to_tf32(x[4 * k4 + 1]); h.z = tc::to_tf32(x[4 * k4 + 2]); h.w = tc::to_tf32(x[4 * k4 + 3]);
    l.x = x[4 * k4] - h.x; l.y = x[4 * k4 + 1] - h.y; l.z = x[4 * k4 + 2] - h.z; l.w = x[4 * k4 + 3] - h.w;
    const uint32_t o = tc::core_off_bytes(r, 4 * k4, 64);
    *reinterpret_cast<float4*>(hi + o) = h;
    *reinterpret_cast<float4*>(lo + o) = l;
  }
}

__global__ void __launch_bounds__(128, 1) k_front_fwd_tc(FrontFwdArgs a, FrontTcSmem sm) {
  MX_DYN_SMEM_RAW(smem_raw);
  __shared__ __align__(8) tc::Bar bar_s;
  __shared__ float par_s[6 * MX_H + MX_G + 2 * 64];      // b1,g1,be1,b2,g2,be2 | b_ih | fn_g, fn_b
  const int tid = threadIdx.x;
  const int net = blockIdx.y;
  const float* __restrict__ th = a.theta[net];
  const MxNetLayout L = a.L;
  const bool live = (net == 0);
  const int I = L.in_dim, Kp = (I + 7) & ~7;
  char* base = reinterpret_cast<char*>(smem_raw);
  char *a_hi = base + sm.o_ahi, *a_lo = base + sm.o_alo;
  char *w1h = base + sm.o_w1h, *w1l = base + sm.o_w1l, *w2h = base + sm.o_w2h, *w2l = base + sm.o_w2l, *wih = base + sm.o_wih, *wil = base + sm.o_wil;
  const uint32_t bar = tc::bar_addr(&bar_s);
  if (tid == 0) {
    tc::mbar_init(bar, blockDim.x);
    tc::mbar_init_fence();
  }
  for (int i = tid; i < MX_H; i += blockDim.x) {
    par_s[i] = th[L.b1 + i]; par_s[MX_H + i] = th[L.ln1_g + i]; par_s[2 * MX_H + i] = th[L.ln1_b + i];
    par_s[3 * MX_H + i] = th[L.b2 + i]; par_s[4 * MX_H + i] = th[L.ln2_g + i]; par_s[5 * MX_H + i] = th[L.ln2_b + i];
    par_s[6 * MX_H + MX_G + i] = i < I ? th[L.fn_g + i] : 0.f; par_s[6 * MX_H + MX_G + 64 + i] = i < I ? th[L.fn_b + i] : 0.f;
  }
  for (int i = tid; i < MX_G; i += blockDim.x) par_s[6 * MX_H + i] = th[L.bih + i];
  MX_PDL_WAIT();        // the mbarrier and the parameter rows are private / parameter data; the images and inputs are not
  if (a.tc_img[net]) {
    // the image is byte-identical to the shared-memory weight region: straight 16-byte async copies
    // two groups: fc1+fc2 first, W_ih (two thirds of the bytes) lands while the first two layers run
    const int nvec = (sm.total - sm.o_w1h) >> 4, nvec12 = (sm.o_wih - sm.o_w1h) >> 4;
    const float* src = a.tc_img[net];
    float* dst = reinterpret_cast<float*>(w1h);
    for (int v = tid; v < nvec12; v += blockDim.x) mx_cp16(dst + 4 * v, src + 4 * v);
    mx_cp_commit();
    for (int v = nvec12 + tid; v < nvec; v += blockDim.x) mx_cp16(dst + 4 * v, src + 4 * v);
    mx_cp_commit();
  } else {
    tc_stage_weight(w1h, w1l, th + L.w1, MX_H, I, Kp);
    tc_stage_weight(w2h, w2l, th + L.w2, MX_H, MX_H, MX_H);
    tc_stage_weight(wih, wil, th + L.wih, MX_G, MX_H, MX_H);
  }
  const float* bih_s = par_s + 6 * MX_H;
  const float* fng_s = par_s + 6 * MX_H + MX_G;
  const float* fnb_s = fng_s + 64;
  __syncthreads();        // parameters and the mbarrier are visible; the weight copies are still in flight
  uint32_t phase = 0;
  const int ntiles = (a.M + 127) / 128;
  const int I4 = (I + 3) >> 2;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    float* acc = tc::cta_slice(a.tc_acc, 256);      // (per tile: a pointer held across the loop costs registers)
    const int m = tile * 128 + tid;
    const bool ok = m < a.M;
    // ---- input row (thread per row, 16-byte loads): LayerNorm over I features, split, write the layer-1 A tile (K = Kp) ----
    {
      float x[64];
#pragma unroll
      for (int c4 = 0; c4 < 16; ++c4) {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (ok && c4 < I4) v = *reinterpret_cast<const float4*>(a.X + (size_t)m * a.ldx + 4 * c4);
        x[4 * c4] = v.x; x[4 * c4 + 1] = v.y; x[4 * c4 + 2] = v.z; x[4 * c4 + 3] = v.w;
      }
#pragma unroll
      for (int c = 0; c < 64; ++c) if (c >= I) x[c] = 0.f;
      const float mean = tc_sum64(x) / (float)I;
      const float rstd = rsqrtf(tc_sumsq64(x, mean, I) / (float)I + MX_LN_EPS);
      if (live && ok && a.st0) { a.st0[2 * (size_t)m] = mean; a.st0[2 * (size_t)m + 1] = rstd; }
#pragma unroll
      for (int c4 = 0; c4 < 16; ++c4)
        if (4 * c4 < Kp) {
          float4 h, l;
          float v[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int c = 4 * c4 + j;
            v[j] = c < I ? (a.feature_norm ? ((x[c] - mean) * rstd * fng_s[c] + fnb_s[c]) : x[c]) : 0.f;
          }
          h.x = tc::to_tf32(v[0]); h.y = tc::to_tf32(v[1]); h.z = tc::to_tf32(v[2]); h.w = tc::to_tf32(v[3]);
          l.x = v[0] - h.x; l.y = v[1] - h.y; l.z = v[2] - h.z; l.w = v[3] - h.w;
          const uint32_t o = tc::core_off_bytes(tid, 4 * c4, Kp);
          *reinterpret_cast<float4*>(a_hi + o) = h;
          *reinterpret_cast<float4*>(a_lo + o) = l;
        }
    }
    // ---- fc1, fc2 ----
    for (int layer = 0; layer < 2; ++layer) {
      mx_cp_wait<1>();
      tc::fence_async_smem();
      __syncthreads();
      tc::mma(acc, 0, a_hi, a_lo, layer == 0 ? w1h : w2h, layer == 0 ? w1l : w2l, MX_H, layer == 0 ? Kp : MX_H, 3, 0);
      tc::arrive(bar);
      tc::mbar_wait(bar, phase);
      phase ^= 1;
      float v[64];
      tc::ld_row(acc, 0, tid, v);
      const float* bs = par_s + layer * 3 * MX_H;
#pragma unroll
      for (int c = 0; c < 64; ++c) { const float z = v[c] + bs[c]; v[c] = a.act_tanh ? tanhf(z) : fmaxf(z, 0.f); }
      const float mean = tc_sum64(v) * (1.f / 64.f);
      const float rstd = rsqrtf(tc_sumsq64(v, mean, 64) * (1.f / 64.f) + MX_LN_EPS);
      float* u_out = layer == 0 ? a.u1 : a.u2;
      float* st_out = layer == 0 ? a.st1 : a.st2;
      if (live && ok && u_out) {
#pragma unroll
        for (int c4 = 0; c4 < 16; ++c4) *reinterpret_cast<float4*>(u_out + (size_t)m * MX_H + 4 * c4) = make_float4(v[4 * c4], v[4 * c4 + 1], v[4 * c4 + 2], v[4 * c4 + 3]);
        if (st_out) { st_out[2 * (size_t)m] = mean; st_out[2 * (size_t)m + 1] = rstd; }
      }
#pragma unroll
      for (int c = 0; c < 64; ++c) v[c] = (v[c] - mean) * rstd * bs[MX_H + c] + bs[2 * MX_H + c];
      tc_put_row64(a_hi, a_lo, tid, v);      // the MMAs that read the previous A tile have completed (mbarrier)
    }
    // ---- gi = x2 . W_ih^T + b_ih ----
    mx_cp_wait<0>();
    tc::fence_async_smem();
    __syncthreads();
    tc::mma(acc, 0, a_hi, a_lo, wih, wil, MX_G, MX_H, 3, 0);
    tc::arrive(bar);
    tc::mbar_wait(bar, phase);
    phase ^= 1;
    float* gi = a.gi[net];
#pragma unroll 1
    for (int c0 = 0; c0 < MX_G; c0 += 64) {
      float t0[64];
      tc::ld_row(acc, c0, tid, t0);
      if (ok) {
#pragma unroll
        for (int c4 = 0; c4 < 16; ++c4)
          *reinterpret_cast<float4*>(gi + (size_t)m * MX_G + c0 + 4 * c4) =
              make_float4(t0[4 * c4] + bih_s[c0 + 4 * c4], t0[4 * c4 + 1] + bih_s[c0 + 4 * c4 + 1], t0[4 * c4 + 2] + bih_s[c0 + 4 * c4 + 2],
                          t0[4 * c4 + 3] + bih_s[c0 + 4 * c4 + 3]);
      }
    }
    __syncthreads();     // every thread has drained its accumulator reads before the next tile's MMAs overwrite the accumulator
  }
}


// ---- 256-thread variant: TWO threads per accumulator row ------------------------------------------------------------------------------------
// Warps w and w + 4 share accumulator row quadrant w & 3, so thread (r, half) reads columns [32 half, 32 half + 32) of row r: every epilogue
// (bias, activation, LayerNorm, TF32 split, operand write-back, activation stores) is half as long per thread, eight warps instead of four
// hide each other's latencies, and the unrolled code a warp walks through is half as large (the 128-thread kernel spends ~30 % of its
// time on instruction-cache misses).  LayerNorm statistics cross the pair through shared memory (four values per layer).
__device__ __forceinline__ float tc_pair_sum(float v, float (*ex)[2][128], int& buf, int half, int r) {
  ex[buf][half][r] = v;
  __syncthreads();
  const float o = ex[buf][half ^ 1][r];
  buf ^= 1;          // the next exchange uses the other buffer: this one is rewritten only after another barrier
  return half ? o + v : v + o;      // same operand order in both threads of the pair
}
__device__ __forceinline__ float tc_sum32(const float (&v)[32]) {
  float p[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) p[i] = v[i];
#pragma unroll
  for (int c = 8; c < 32; c += 8)
#pragma unroll
    for (int i = 0; i < 8; ++i) p[i] += v[c + i];
  return ((p[0] + p[1]) + (p[2] + p[3])) + ((p[4] + p[5]) + (p[6] + p[7]));
}
__device__ __forceinline__ float tc_sumsq32(const float (&v)[32], float mean, int c0, int n_valid) {
  float p[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) p[i] = 0.f;
#pragma unroll
  for (int c = 0; c < 32; c += 8)
#pragma unroll
    for (int i = 0; i < 8; ++i) { const float d = (c0 + c + i < n_valid) ? v[c + i] - mean : 0.f; p[i] = fmaf(d, d, p[i]); }
  return ((p[0] + p[1]) + (p[2] + p[3])) + ((p[4] + p[5]) + (p[6] + p[7]));
}
// this thread's 32 columns [c0, c0 + 32) of row r into the A tiles (K = 64), 16 bytes at a time
__device__ __forceinline__ void tc_put_row32(char* hi, char* lo, int r, int c0, const float (&x)[32]) {
#pragma unroll
  for (int k4 = 0; k4 < 8; ++k4) {
    float4 h, l;
    h.x = tc::to_tf32(x[4 * k4]); h.y = tc::to_tf32(x[4 * k4 + 1]); h.z = tc::to_tf32(x[4 * k4 + 2]); h.w = tc::to_tf32(x[4 * k4 + 3]);
    l.x = x[4 * k4] - h.x; l.y = x[4 * k4 + 1] - h.y; l.z = x[4 * k4 + 2] - h.z; l.w = x[4 * k4 + 3] - h.w;
    const uint32_t o = tc::core_off_bytes(r, c0 + 4 * k4, 64);
    *reinterpret_cast<float4*>(hi + o) = h;
    *reinterpret_cast<float4*>(lo + o) = l;
  }
}

__global__ void __launch_bounds__(256, 1) k_front_fwd_tc2(FrontFwdArgs a, FrontTcSmem sm) {
  MX_DYN_SMEM_RAW(smem_raw);
  __shared__ __align__(8) tc::Bar bar_s;
  __shared__ float par_s[6 * MX_H + MX_G + 2 * 64];      // b1,g1,be1,b2,g2,be2 | b_ih | fn_g, fn_b
  __shared__ float ex_s[2][2][128];                        // pair exchange of LayerNorm partial sums
  const int tid = threadIdx.x;
  const int r = tid & 127, half = tid >> 7, c0 = 32 * half;
  const int net = blockIdx.y;
  const float* __restrict__ th = a.theta[net];
  const MxNetLayout L = a.L;
  const bool live = (net == 0);
  const int I = L.in_dim, Kp = (I + 7) & ~7;
  char* base = reinterpret_cast<char*>(smem_raw);
  char *a_hi = base + sm.o_ahi, *a_lo = base + sm.o_alo;
  char *w1h = base + sm.o_w1h, *w1l = base + sm.o_w1l, *w2h = base + sm.o_w2h, *w2l = base + sm.o_w2l, *wih = base + sm.o_wih, *wil = base + sm.o_wil;
  const uint32_t bar = tc::bar_addr(&bar_s);
  float* acc = tc::cta_slice(a.tc_acc, 256);
  if (tid == 0) {
    tc::mbar_init(bar, blockDim.x);
    tc::mbar_init_fence();
  }
  for (int i = tid; i < MX_H; i += blockDim.x) {
    par_s[i] = th[L.b1 + i]; par_s[MX_H + i] = th[L.ln1_g + i]; par_s[2 * MX_H + i] = th[L.ln1_b + i];
    par_s[3 * MX_H + i] = th[L.b2 + i]; par_s[4 * MX_H + i] = th[L.ln2_g + i]; par_s[5 * MX_H + i] = th[L.ln2_b + i];
    par_s[6 * MX_H + MX_G + i] = i < I ? th[L.fn_g + i] : 0.f; par_s[6 * MX_H + MX_G + 64 + i] = i < I ? th[L.fn_b + i] : 0.f;
  }
  for (int i = tid; i < MX_G; i += blockDim.x) par_s[6 * MX_H + i] = th[L.bih + i];
  MX_PDL_WAIT();
  if (a.tc_img[net]) {
    const int nvec = (sm.total - sm.o_w1h) >> 4, nvec12 = (sm.o_wih - sm.o_w1h) >> 4;
    const float* src = a.tc_img[net];
    float* dst = reinterpret_cast<float*>(w1h);
    for (int v = tid; v < nvec12; v += blockDim.x) mx_cp16(dst + 4 * v, src + 4 * v);
    mx_cp_commit();
    for (int v = nvec12 + tid; v < nvec; v += blockDim.x) mx_cp16(dst + 4 * v, src + 4 * v);
    mx_cp_commit();
  } else {
    tc_stage_weight(w1h, w1l, th + L.w1, MX_H, I, Kp);
    tc_stage_weight(w2h, w2l, th + L.w2, MX_H, MX_H, MX_H);
    tc_stage_weight(wih, wil, th + L.wih, MX_G, MX_H, MX_H);
  }
  const float* bih_s = par_s + 6 * MX_H;
  const float* fng_s = par_s + 6 * MX_H + MX_G;
  const float* fnb_s = fng_s + 64;
  __syncthreads();
  uint32_t phase = 0;
  int xb = 0;
  const int ntiles = (a.M + 127) / 128;
  const int I4 = (I + 3) >> 2;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int m = tile * 128 + r;
    const bool ok = m < a.M;
    // ---- input row, columns [c0, c0 + 32): LayerNorm over I features (pair-wise statistics), split, layer-1 A tile (K = Kp) ----
    {
      float x[32];
#pragma unroll
      for (int c4 = 0; c4 < 8; ++c4) {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (ok && 8 * half + c4 < I4) v = *reinterpret_cast<const float4*>(a.X + (size_t)m * a.ldx + c0 + 4 * c4);
        x[4 * c4] = v.x; x[4 * c4 + 1] = v.y; x[4 * c4 + 2] = v.z; x[4 * c4 + 3] = v.w;
      }
#pragma unroll
      for (int c = 0; c < 32; ++c) if (c0 + c >= I) x[c] = 0.f;
      const float mean = tc_pair_sum(tc_sum32(x), ex_s, xb, half, r) / (float)I;
      const float rstd = rsqrtf(tc_pair_sum(tc_sumsq32(x, mean, c0, I), ex_s, xb, half, r) / (float)I + MX_LN_EPS);
      if (live && ok && a.st0 && half == 0) { a.st0[2 * (size_t)m] = mean; a.st0[2 * (size_t)m + 1] = rstd; }
#pragma unroll
      for (int c4 = 0; c4 < 8; ++c4)
        if (c0 + 4 * c4 < Kp) {
          float4 h, l;
          float v[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int c = c0 + 4 * c4 + j;
            v[j] = c < I ? (a.feature_norm ? ((x[4 * c4 + j] - mean) * rstd * fng_s[c] + fnb_s[c]) : x[4 * c4 + j]) : 0.f;
          }
          h.x = tc::to_tf32(v[0]); h.y = tc::to_tf32(v[1]); h.z = tc::to_tf32(v[2]); h.w = tc::to_tf32(v[3]);
          l.x = v[0] - h.x; l.y = v[1] - h.y; l.z = v[2] - h.z; l.w = v[3] - h.w;
          const uint32_t o = tc::core_off_bytes(r, c0 + 4 * c4, Kp);
          *reinterpret_cast<float4*>(a_hi + o) = h;
          *reinterpret_cast<float4*>(a_lo + o) = l;
        }
    }
    // ---- fc1, fc2 ----
    for (int layer = 0; layer < 2; ++layer) {
      mx_cp_wait<1>();
      tc::fence_async_smem();
      __syncthreads();
      tc::mma(acc, 0, a_hi, a_lo, layer == 0 ? w1h : w2h, layer == 0 ? w1l : w2l, MX_H, layer == 0 ? Kp : MX_H, 3, 0);
      tc::arrive(bar);
      tc::mbar_wait(bar, phase);
      phase ^= 1;
      float v[32];
      tc::ld_row(acc, c0, r, v);
      const float* bs = par_s + layer * 3 * MX_H;
#pragma unroll
      for (int c = 0; c < 32; ++c) { const float z = v[c] + bs[c0 + c]; v[c] = a.act_tanh ? tanhf(z) : fmaxf(z, 0.f); }
      const float mean = tc_pair_sum(tc_sum32(v), ex_s, xb, half, r) * (1.f / 64.f);
      const float rstd = rsqrtf(tc_pair_sum(tc_sumsq32(v, mean, c0, 64), ex_s, xb, half, r) * (1.f / 64.f) + MX_LN_EPS);
      float* u_out = layer == 0 ? a.u1 : a.u2;
      float* st_out = layer == 0 ? a.st1 : a.st2;
      if (live && ok && u_out) {
#pragma unroll
        for (int c4 = 0; c4 < 8; ++c4) *reinterpret_cast<float4*>(u_out + (size_t)m * MX_H + c0 + 4 * c4) = make_float4(v[4 * c4], v[4 * c4 + 1], v[4 * c4 + 2], v[4 * c4 + 3]);
        if (st_out && half == 0) { st_out[2 * (size_t)m] = mean; st_out[2 * (size_t)m + 1] = rstd; }
      }
#pragma unroll
      for (int c = 0; c < 32; ++c) v[c] = (v[c] - mean) * rstd * bs[MX_H + c0 + c] + bs[2 * MX_H + c0 + c];
      tc_put_row32(a_hi, a_lo, r, c0, v);      // the MMAs that read the previous A tile have completed (mbarrier)
    }
    // ---- gi = x2 . W_ih^T + b_ih: columns [96 half, 96 half + 96) ----
    mx_cp_wait<0>();
    tc::fence_async_smem();
    __syncthreads();
    tc::mma(acc, 0, a_hi, a_lo, wih, wil, MX_G, MX_H, 3, 0);
    tc::arrive(bar);
    tc::mbar_wait(bar, phase);
    phase ^= 1;
    float* gi = a.gi[net];
#pragma unroll 1
    for (int g0 = 96 * half; g0 < 96 * half + 96; g0 += 32) {
      float t0[32];
      tc::ld_row(acc, g0, r, t0);
      if (ok) {
#pragma unroll
        for (int c4 = 0; c4 < 8; ++c4)
          *reinterpret_cast<float4*>(gi + (size_t)m * MX_G + g0 + 4 * c4) =
              make_float4(t0[4 * c4] + bih_s[g0 + 4 * c4], t0[4 * c4 + 1] + bih_s[g0 + 4 * c4 + 1], t0[4 * c4 + 2] + bih_s[g0 + 4 * c4 + 2],
                          t0[4 * c4 + 3] + bih_s[g0 + 4 * c4 + 3]);
      }
    }
    __syncthreads();
  }
}


// =====================================================================================================
// Wide inputs (64 < in_dim <= 128: SMAC 8m / 2s3z observations): fc1's K dimension is fed in chunks of 64 columns that accumulate in the
// accumulator, and EVERY weight operand is streamed through one 32 KB chunk buffer (fc1 chunk 0, fc1 chunk 1, fc2, W_ih gate r, z, n -- six
// [64][K] hi | lo pairs per tile, copied from the L2-resident image with cp.async), so a CTA needs 96 KB of shared memory and 256
// accumulator columns and TWO CTAs share an SM: while one waits for an MMA, a copy or its row loads, the other runs its epilogue (with
// fc2 and W_ih resident, 224 KB and one CTA per SM, ncu at 8m showed 4 warps per SM, issue-active 11 %, long-scoreboard 5 warps per issue).  The copy
// of chunk i + 1 is issued as soon as the MMAs of chunk i have completed, i.e. it flies during the epilogue between them; the three gate
// blocks of gi accumulate in their own accumulator columns, so the epilogue of gate g overlaps the copy of gate g + 1.
// =====================================================================================================
struct WideTcSmem { int o_ahi, o_alo, o_wc, total; };
static WideTcSmem wide_tc_smem() {
  WideTcSmem s;
  s.o_ahi = 0; s.o_alo = 128 * 64 * 4; s.o_wc = 2 * 128 * 64 * 4; s.total = s.o_wc + 2 * 64 * 64 * 4;
  return s;
}
__device__ __forceinline__ void tcw_stage(char* dst, const float* __restrict__ src, int nbytes) {
  float* d = reinterpret_cast<float*>(dst);
  for (int v = threadIdx.x; v < (nbytes >> 4); v += blockDim.x) mx_cp16(d + 4 * v, src + 4 * v);
}
__global__ void __launch_bounds__(128, 2) k_front_fwd_tc_wide2(FrontFwdArgs a, WideTcSmem sm) {
  MX_DYN_SMEM_RAW(smem_raw);
  __shared__ __align__(8) tc::Bar bar_s;
  __shared__ float par_s[6 * MX_H + MX_G + 2 * 128];      // b1,g1,be1,b2,g2,be2 | b_ih | feature-norm gain, bias
  const int tid = threadIdx.x;
  const int net = blockIdx.y;
  const float* __restrict__ th = a.theta[net];
  const MxNetLayout L = a.L;
  const bool live = (net == 0);
  const int I = L.in_dim, Kp = (I + 7) & ~7, Kc1 = Kp - 64;
  char* base = reinterpret_cast<char*>(smem_raw);
  char *a_hi = base + sm.o_ahi, *a_lo = base + sm.o_alo, *wc = base + sm.o_wc;
  const uint32_t bar = tc::bar_addr(&bar_s);
  float* acc = tc::cta_slice(a.tc_acc, 256);
  if (tid == 0) {
    tc::mbar_init(bar, blockDim.x);
    tc::mbar_init_fence();
  }
  float* bih_s = par_s + 6 * MX_H;
  float* fng = bih_s + MX_G;
  float* fnb = fng + 128;
  for (int i = tid; i < MX_H; i += blockDim.x) {
    par_s[i] = th[L.b1 + i]; par_s[MX_H + i] = th[L.ln1_g + i]; par_s[2 * MX_H + i] = th[L.ln1_b + i];
    par_s[3 * MX_H + i] = th[L.b2 + i]; par_s[4 * MX_H + i] = th[L.ln2_g + i]; par_s[5 * MX_H + i] = th[L.ln2_b + i];
  }
  for (int i = tid; i < MX_G; i += blockDim.x) bih_s[i] = th[L.bih + i];
  for (int i = tid; i < 128; i += blockDim.x) { fng[i] = (i < I && a.feature_norm) ? th[L.fn_g + i] : 1.f; fnb[i] = (i < I && a.feature_norm) ? th[L.fn_b + i] : 0.f; }
  MX_PDL_WAIT();
  // image: [fc1 chunk 0 hi|lo][fc1 chunk 1 hi|lo][fc2 hi|lo][W_ih hi (192 rows)][W_ih lo]
  const float* img = a.tc_img[net];
  const float* img_c1 = img + 2 * 64 * 64;
  const float* img_w2 = img + 2 * 64 * Kp;
  const float* img_wih = img_w2 + 2 * 4096;
  __syncthreads();
  uint32_t phase = 0;
  const int ntiles = (a.M + 127) / 128;
  const int I4 = (I + 3) >> 2;
  if ((int)blockIdx.x < ntiles) { tcw_stage(wc, img, 2 * 64 * 64 * 4); mx_cp_commit(); }      // first tile's fc1 chunk 0
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int m = tile * 128 + tid;
    const bool ok = m < a.M;
    const float* xrow = a.X + (size_t)(ok ? m : 0) * a.ldx;
    float mean = 0.f, rstd = 1.f;
    {
      float p[4] = {0.f, 0.f, 0.f, 0.f};
      for (int cb = 0; cb < I4; cb += 8) {
        float4 q8[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) q8[i] = (ok && cb + i < I4) ? *reinterpret_cast<const float4*>(xrow + 4 * (cb + i)) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int c = 4 * (cb + i);
          p[0] += (c < I) ? q8[i].x : 0.f; p[1] += (c + 1 < I) ? q8[i].y : 0.f; p[2] += (c + 2 < I) ? q8[i].z : 0.f; p[3] += (c + 3 < I) ? q8[i].w : 0.f;
        }
      }
      mean = ((p[0] + p[1]) + (p[2] + p[3])) / (float)I;
      float q[4] = {0.f, 0.f, 0.f, 0.f};
      for (int cb = 0; cb < I4; cb += 8) {
        float4 q8[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) q8[i] = (ok && cb + i < I4) ? *reinterpret_cast<const float4*>(xrow + 4 * (cb + i)) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int c = 4 * (cb + i);
          const float d0 = (c < I) ? q8[i].x - mean : 0.f, d1 = (c + 1 < I) ? q8[i].y - mean : 0.f, d2 = (c + 2 < I) ? q8[i].z - mean : 0.f,
                      d3 = (c + 3 < I) ? q8[i].w - mean : 0.f;
          q[0] = fmaf(d0, d0, q[0]); q[1] = fmaf(d1, d1, q[1]); q[2] = fmaf(d2, d2, q[2]); q[3] = fmaf(d3, d3, q[3]);
        }
      }
      rstd = rsqrtf(((q[0] + q[1]) + (q[2] + q[3])) / (float)I + MX_LN_EPS);
      if (live && ok && a.st0) { a.st0[2 * (size_t)m] = mean; a.st0[2 * (size_t)m + 1] = rstd; }
      if (!a.feature_norm) { mean = 0.f; rstd = 1.f; }      // (gain 1 / bias 0 in shared memory): the raw input goes through unchanged
    }
    // ---- fc1 in two K chunks ----
    for (int ch = 0; ch < 2; ++ch) {
      const int Kc = ch == 0 ? 64 : Kc1;
      for (int cb = 0; 4 * cb < Kc; cb += 8) {
        float4 q8[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int c0 = 64 * ch + 4 * (cb + i);
          q8[i] = (ok && 4 * (cb + i) < Kc && c0 < I) ? *reinterpret_cast<const float4*>(xrow + c0) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int c4 = cb + i;
          if (4 * c4 >= Kc) continue;
          const int c0 = 64 * ch + 4 * c4;
          float x[4] = {q8[i].x, q8[i].y, q8[i].z, q8[i].w};
          float4 h, l;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int c = c0 + j;
            x[j] = (ok && c < I) ? ((x[j] - mean) * rstd * fng[c] + fnb[c]) : 0.f;
          }
          h.x = tc::to_tf32(x[0]); h.y = tc::to_tf32(x[1]); h.z = tc::to_tf32(x[2]); h.w = tc::to_tf32(x[3]);
          l.x = x[0] - h.x; l.y = x[1] - h.y; l.z = x[2] - h.z; l.w = x[3] - h.w;
          const uint32_t o = tc::core_off_bytes(tid, 4 * c4, Kc);
          *reinterpret_cast<float4*>(a_hi + o) = h;
          *reinterpret_cast<float4*>(a_lo + o) = l;
        }
      }
      mx_cp_wait<0>();
      tc::fence_async_smem();
      __syncthreads();
      tc::mma(acc, 0, a_hi, a_lo, wc, wc + 64 * Kc * 4, MX_H, Kc, 3, ch > 0 ? 1u : 0u);
      tc::arrive(bar);
      tc::mbar_wait(bar, phase);        // the MMAs have read the A tile and the chunk buffer: both may be refilled
      phase ^= 1;
      if (ch == 0) tcw_stage(wc, img_c1, 2 * 64 * Kc1 * 4); else tcw_stage(wc, img_w2, 2 * 4096 * 4);
      mx_cp_commit();
    }
    // ---- fc1 epilogue, fc2, fc2 epilogue ----
    for (int layer = 0; layer < 2; ++layer) {
      if (layer == 1) {
        mx_cp_wait<0>();
        tc::fence_async_smem();
        __syncthreads();
        tc::mma(acc, 0, a_hi, a_lo, wc, wc + 4096 * 4, MX_H, MX_H, 3, 0);
        tc::arrive(bar);
        tc::mbar_wait(bar, phase);
        phase ^= 1;
        tcw_stage(wc, img_wih, 4096 * 4); tcw_stage(wc + 4096 * 4, img_wih + 3 * 4096, 4096 * 4);      // gate r: hi | lo
        mx_cp_commit();
      }
      float v[64];
      tc::ld_row(acc, 0, tid, v);
      const float* bs = par_s + layer * 3 * MX_H;
#pragma unroll
      for (int c = 0; c < 64; ++c) { const float z = v[c] + bs[c]; v[c] = a.act_tanh ? tanhf(z) : fmaxf(z, 0.f); }
      const float mu = tc_sum64(v) * (1.f / 64.f);
      const float rs = rsqrtf(tc_sumsq64(v, mu, 64) * (1.f / 64.f) + MX_LN_EPS);
      float* u_out = layer == 0 ? a.u1 : a.u2;
      float* st_out = layer == 0 ? a.st1 : a.st2;
      if (live && ok && u_out) {
#pragma unroll
        for (int c4 = 0; c4 < 16; ++c4) *reinterpret_cast<float4*>(u_out + (size_t)m * MX_H + 4 * c4) = make_float4(v[4 * c4], v[4 * c4 + 1], v[4 * c4 + 2], v[4 * c4 + 3]);
        if (st_out) { st_out[2 * (size_t)m] = mu; st_out[2 * (size_t)m + 1] = rs; }
      }
#pragma unroll
      for (int c = 0; c < 64; ++c) v[c] = (v[c] - mu) * rs * bs[MX_H + c] + bs[2 * MX_H + c];
      __syncthreads();          // every thread has drained its accumulator reads before the next layer's MMAs overwrite the accumulator
      tc_put_row64(a_hi, a_lo, tid, v);
    }
    // ---- gi = x2 . W_ih^T + b_ih, one gate block (64 columns) at a time into accumulator columns 64 + 64 g ----
    float* gi = a.gi[net];
#pragma unroll 1
    for (int g = 0; g < 3; ++g) {
      mx_cp_wait<0>();
      tc::fence_async_smem();
      __syncthreads();
      tc::mma(acc, 64 + 64 * g, a_hi, a_lo, wc, wc + 4096 * 4, MX_H, MX_H, 3, 0);
      tc::arrive(bar);
      tc::mbar_wait(bar, phase);
      phase ^= 1;
      if (g < 2) {
        tcw_stage(wc, img_wih + (g + 1) * 4096, 4096 * 4); tcw_stage(wc + 4096 * 4, img_wih + (3 + g + 1) * 4096, 4096 * 4);
        mx_cp_commit();
      } else if (tile + (int)gridDim.x < ntiles) {
        tcw_stage(wc, img, 2 * 64 * 64 * 4);       // the next tile's fc1 chunk 0
        mx_cp_commit();
      }
      float t0[64];
      tc::ld_row(acc, 64 + 64 * g, tid, t0);
      if (ok) {
        const int c0 = 64 * g;
#pragma unroll
        for (int c4 = 0; c4 < 16; ++c4)
          *reinterpret_cast<float4*>(gi + (size_t)m * MX_G + c0 + 4 * c4) =
              make_float4(t0[4 * c4] + bih_s[c0 + 4 * c4], t0[4 * c4 + 1] + bih_s[c0 + 4 * c4 + 1], t0[4 * c4 + 2] + bih_s[c0 + 4 * c4 + 2],
                          t0[4 * c4 + 3] + bih_s[c0 + 4 * c4 + 3]);
      }
    }
    __syncthreads();     // accumulator reads drained; the A tile is free for the next tile
  }
  mx_cp_wait<0>();
}

int g_mx_front_tc = 1;        // 1: tensor-core 3xTF32 kernels (default), 0: FFMA kernel (mx_set_option("front_tc", 0))
extern int g_mx_wgrad_tc;      // tc_bwd.cu

bool mx_front_tc_usable(int in_dim, bool have_image) {
  if (!g_mx_front_tc) return false;
  return in_dim <= 64 || (in_dim <= 128 && have_image);
}

int mx_launch_front_fwd_tc(const FrontFwdArgs& a, int nets, cudaStream_t s) {
  const int ntiles = mx_ceil_div(a.M, 128);
  if (!a.tc_acc || a.tc_acc_cols < 256 * nets) { mx_set_error("front_fwd_tc: accumulator region missing or too small"); return 1; }
  if (a.L.in_dim > 64) {
    if (!a.tc_img[0] || (nets > 1 && !a.tc_img[1])) { mx_set_error("front_fwd_tc_wide: weight images missing"); return 1; }
    WideTcSmem s2 = wide_tc_smem();
    int g2 = 2 * mx_num_sms() / nets;
    if (g2 > ntiles) g2 = ntiles;
    if (g2 * nets * 256 > a.tc_acc_cols) g2 = a.tc_acc_cols / (256 * nets);
    if (g2 < 1) g2 = 1;
    return mx_launch("k_front_fwd_tc_wide", k_front_fwd_tc_wide2, dim3(g2, nets), dim3(128), (size_t)s2.total, s, MX_STEP, a, s2);
  }
  FrontTcSmem sm = front_tc_smem(mx_round_up(a.L.in_dim, 8));
  const size_t smem = (size_t)sm.total;
  int gx = mx_num_sms() / nets;
  if (gx > ntiles) gx = ntiles;
  if (gx * nets * 256 > a.tc_acc_cols) gx = a.tc_acc_cols / (256 * nets);      // 256 accumulator columns per CTA
  if (gx < 1) gx = 1;
  // (inputs of 57..64 columns fill the 227 KB with operand tiles: the pair-exchange buffer of the 256-thread kernel no longer fits beside them)
  if (smem + 5 * 1024 + 256 <= MX_SMEM_OPTIN_MAX)
    return mx_launch("k_front_fwd_tc", k_front_fwd_tc2, dim3(gx, nets), dim3(256), smem, s, MX_STEP, a, sm);
  // (its own name: tests pin which of the two variants ran)
  return mx_launch("k_front_fwd_tc1", k_front_fwd_tc, dim3(gx, nets), dim3(128), smem, s, MX_STEP, a, sm);
}

extern "C" int mx_set_option(const char* name, int32_t value) {
  if (mx_set_option_common(name, value) == 0) return 0;
  if (!strcmp(name, "front_tc")) { g_mx_front_tc = value; return 0; }
  if (!strcmp(name, "wgrad_tc")) { g_mx_wgrad_tc = value; return 0; }
#if !MX_EMU
  if (!strcmp(name, "pdl")) { g_mx_pdl = value; return 0; }
  if (!strcmp(name, "pdl_rows")) { g_mx_pdl_rows = value; return 0; }
#endif
  mx_set_error("mx_set_option: unknown option %s", name);
  return 1;
}

struct TcProbeArgs {
  const float *X, *W;
  float* Y;
  int M, N, K, passes, swap_ls;
};

// N is taken in blocks of up to 64 columns: the B block and the block's accumulator live in shared memory beside the A tile
__global__ void __launch_bounds__(128) k_tc_linear_probe(TcProbeArgs a) {
  MX_DYN_SMEM_RAW(smem_raw);
  __shared__ __align__(8) tc::Bar bar_s;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int K = a.K, N = a.N;
  char* a_hi = reinterpret_cast<char*>(smem_raw);
  char* a_lo = a_hi + 128 * K * 4;
  char* b_hi = a_lo + 128 * K * 4;
  char* b_lo = b_hi + 64 * K * 4;
  float* acc = reinterpret_cast<float*>(b_lo + 64 * K * 4);      // [64 columns][128 rows]
  const int m0 = blockIdx.x * 128;
  const uint32_t bar = tc::bar_addr(&bar_s);
  if (tid == 0) {
    tc::mbar_init(bar, blockDim.x);
    tc::mbar_init_fence();
  }
  // A tile (zero rows beyond M)
  for (int idx = tid; idx < 128 * K; idx += 128) {
    const int r = idx / K, k = idx % K;
    const float x = (m0 + r < a.M) ? a.X[(size_t)(m0 + r) * K + k] : 0.f;
    tc::put_split(a_hi, a_lo, r, k, K, x);
  }
  const int row = m0 + warp * 32 + lane;
  uint32_t phase = 0;
  for (int n0 = 0; n0 < N; n0 += 64) {
    const int nc = N - n0 < 64 ? N - n0 : 64;
    for (int idx = tid; idx < nc * K; idx += 128) {
      const int r = idx / K, k = idx % K;
      tc::put_split(b_hi, b_lo, r, k, K, a.W[(size_t)(n0 + r) * K + k]);
    }
    tc::fence_async_smem();
    __syncthreads();
    tc::mma(acc, 0, a_hi, a_lo, b_hi, b_lo, nc, K, a.passes, 0, a.swap_ls);
    tc::arrive(bar);
    tc::mbar_wait(bar, phase);
    phase ^= 1;
    for (int c0 = 0; c0 < nc; c0 += 32) {
      float v[32];
      tc::ld_row(acc, c0, tid, v);
      if (row < a.M)
        for (int c = 0; c < 32 && c0 + c < nc; ++c) a.Y[(size_t)row * N + n0 + c0 + c] = v[c];
    }
    __syncthreads();      // accumulator reads done before the next block's MMAs overwrite it; B block free
  }
}

extern "C" int mx_tc_linear_probe(const float* X, const float* W, float* Y, int32_t M, int32_t N, int32_t K, int32_t passes, int32_t swap_ls,
                                  void* stream) {
  if (N % 16 || N < 16 || N > 256 || K % 8 || K < 8 || K > 64 || M < 1) { mx_set_error("tc probe: M >= 1, N %% 16, N <= 256, K %% 8, K <= 64 required"); return 1; }
  TcProbeArgs a{X, W, Y, M, N, K, passes, swap_ls};
  const size_t smem = (size_t)(2 * 128 + 2 * 64) * K * 4 + 64 * 128 * 4;
  return mx_launch("k_tc_linear_probe", k_tc_linear_probe, dim3((M + 127) / 128), dim3(128), smem, (cudaStream_t)stream, MX_PLAIN, a);
}
