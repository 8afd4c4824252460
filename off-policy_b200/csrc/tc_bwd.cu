// Weight gradients of the agent network's time-batched layers on the wgmma tensor cores (3xTF32): k_wgrad_tc.
//
//   dW_ih = dgi^T x2     dW_hh = [dgi_r, dgi_z, dgi_n * r]^T h_{t-1}     dW2 = da2^T x1     dW1 = da1^T x0     + every bias gradient
//
// These are reductions over the ROWS of the step (K = rows), so both MMA operands are the row-major activations read TRANSPOSED:
// A[feature][row] and B[feature][row], K-major.  A thread stages (feature, 4 consecutive rows) pairs: four scalar loads from the
// L2-resident activations, TF32 hi / lo split, two 16-byte stores into the core-matrix layout; within a warp the 32 pairs are
// (8 features) x (4 row quads), which is 512 contiguous bytes of the tile -- no bank conflicts, every store a full wavefront.
// Normalised activations (x2, x1, x0) are recomputed from the saved pre-norm rows and statistics while staging; bias gradients fall out
// of a column of ones appended to B.  Three accumulators live in the CTA's accumulator (mx_tc.cuh) for the whole CTA (rows are split over CTAs in chunks of 64):
//   D1[128][144] = [dgi_r | dgi_z]^T     . [x2 | h_prev | 1]   -> dW_ih[0:128], dW_hh[0:128], db_ih[0:128] (= db_hh[0:128])
//   D2[128][144] = [dgi_n | dgi_n * r]^T . [x2 | h_prev | 1]   -> dW_ih[128:192] (rows 0-63, cols 0-63), dW_hh[128:192] (rows 64-127, cols 64-127)
//   D3[128][..]  = [da2   | da1]^T       . [x1 | x0]           -> dW2 (rows 0-63, cols 0-63), dW1 (rows 64-127, cols 64..)
//   D4[128][16]  = [da2   | da1]^T       . [1 | 0..]           -> db2, db1 (a 16-column accumulator in D1's padding; same A tile, same arrival)
// The off-diagonal blocks of D2 / D3 are products nobody needs (half of two of the three MMAs): the tensor core is not the limit here.
// Each CTA writes its sums as ONE gradient partial (its row of gpart), like k_front_bwd does for the LayerNorm parameters it keeps.
#include "mx_internal.h"
#include "mx_kernels.h"
#include "mx_tc.cuh"

#include <string.h>

int g_mx_wgrad_tc = -1;       // -1 (default): by input width -- inputs <= 64 (3m, MPE) on the FFMA backward, wider inputs (8m / 2s3z, obs 80) on
                              // k_front_bwd_tc + k_wgrad_tc (split not yet measured on the H100); 0 / 1 / 2 force a mode
static inline int wgrad_mode(int in_dim) { return g_mx_wgrad_tc >= 0 ? g_mx_wgrad_tc : (in_dim > 64 ? 2 : 0); }

#define WG_ROWS 64            // rows per MMA group (the K extent of one staged tile)
#define WG_DSTRIDE 160        // accumulator column stride between the three accumulators

#define WG_MAX_IN 128          // input widths up to here: D3 = [x1 | x0] is 64 + round_up(I, 16) <= 192 columns, the rest of the 512 accumulator columns
#define WG_ONES_COL 144        // db2 / db1 = [da2 | da1]^T . 1: a 16-column accumulator in the padding between D1 (144 wide) and D2 (at 160)
struct WgradSmem { int o_ahi, o_alo, o_bhi, o_blo, o_ones, total; };
static WgradSmem wgrad_smem(int n3) {
  const int nb = n3 > 144 ? n3 : 144;
  WgradSmem s;
  int o = 0;
  s.o_ahi = o; o += 128 * WG_ROWS * 4;
  s.o_alo = o; o += 128 * WG_ROWS * 4;
  s.o_bhi = o; o += nb * WG_ROWS * 4;
  s.o_blo = o; o += nb * WG_ROWS * 4;
  s.o_ones = o; o += 2 * 16 * WG_ROWS * 4;      // [16][64] hi | lo: feature 0 = 1 for the chunk's valid rows
  s.total = o;
  return s;
}

// one (feature, row quad) pair -> hi / lo tiles
__device__ __forceinline__ void wg_put(char* hi, char* lo, int feat, int kq, const float (&x)[4]) {
  float4 h, l;
  h.x = tc::to_tf32(x[0]); h.y = tc::to_tf32(x[1]); h.z = tc::to_tf32(x[2]); h.w = tc::to_tf32(x[3]);
  l.x = x[0] - h.x; l.y = x[1] - h.y; l.z = x[2] - h.z; l.w = x[3] - h.w;
  const uint32_t o = tc::core_off_bytes(feat, 4 * kq, WG_ROWS);
  *reinterpret_cast<float4*>(hi + o) = h;
  *reinterpret_cast<float4*>(lo + o) = l;
}
// pair index -> (feature, row quad): lanes of a warp cover 8 consecutive features x 4 consecutive row quads
__device__ __forceinline__ void wg_pair(int p, int* feat, int* kq) {
  const int fr = p & 7, kl = (p >> 3) & 3, rest = p >> 5;
  *feat = (rest >> 2) * 8 + fr;
  *kq = (rest & 3) * 4 + kl;
}

struct WgradArgs {
  FrontBwdArgs f;
  int nchunks, Kp16;
  int ln_zero_from;      // CTAs from this index on also zero the LayerNorm ranges of their partial (k_front_bwd_tc ran fewer CTAs); -1: none
  int ln_parts;          // > 0: k_front_bwd_tc left its LayerNorm sums in f.ln_part[ln_parts][512] (streamed mode) instead of the partial rows
};

#define WG_THREADS 512        // staging is load-latency bound: 16 warps keep enough loads in flight; warps 0-3 own the accumulator rows in the epilogue
__global__ void __launch_bounds__(WG_THREADS, 1) k_wgrad_tc(WgradArgs w, WgradSmem sm) {
  MX_DYN_SMEM_RAW(smem_raw);
  __shared__ __align__(8) tc::Bar bar_s;
  __shared__ float par_s[4 * 64 + 2 * 128];  // ln2 g,b | ln1 g,b | fn g (128), fn b (128)
  __shared__ float st_s[3 * 2 * WG_ROWS];    // (mean, rstd) of the chunk's rows for LN2 | LN1 | the feature LayerNorm
  const FrontBwdArgs& a = w.f;
  const MxNetLayout L = a.L;
  const float* __restrict__ th = a.theta;
  const int tid = threadIdx.x, warp = tid >> 5;
  const int I = L.in_dim, N = a.N, T1 = a.T1 > 0 ? a.T1 : a.T + 1;
  const int Kp16 = w.Kp16, N3 = 64 + Kp16;
  char* base = reinterpret_cast<char*>(smem_raw);
  char *a_hi = base + sm.o_ahi, *a_lo = base + sm.o_alo, *b_hi = base + sm.o_bhi, *b_lo = base + sm.o_blo;
  char *o_hi = base + sm.o_ones, *o_lo = o_hi + 16 * WG_ROWS * 4;
  const uint32_t bar = tc::bar_addr(&bar_s);
  float* acc = tc::cta_slice(a.tc_acc, 512);
  if (tid == 0) {
    tc::mbar_init(bar, blockDim.x);
    tc::mbar_init_fence();
  }
  for (int i = tid; i < 64; i += blockDim.x) {
    par_s[i] = th[L.ln2_g + i]; par_s[64 + i] = th[L.ln2_b + i]; par_s[128 + i] = th[L.ln1_g + i]; par_s[192 + i] = th[L.ln1_b + i];
  }
  for (int i = tid; i < 128; i += blockDim.x) { par_s[256 + i] = i < I ? th[L.fn_g + i] : 0.f; par_s[384 + i] = i < I ? th[L.fn_b + i] : 0.f; }
  MX_PDL_WAIT();
  __syncthreads();
  uint32_t phase = 0;
  int iter = 0;
  for (int chunk = blockIdx.x; chunk < w.nchunks; chunk += gridDim.x, ++iter) {
    const int row0 = chunk * WG_ROWS;
    const uint32_t acc0 = iter > 0 ? 1u : 0u;
    for (int i = tid; i < 3 * 2 * WG_ROWS; i += blockDim.x) {      // (the previous chunk's readers are past their last MMA wait)
      const int which = i / (2 * WG_ROWS), rr = (i % (2 * WG_ROWS)) >> 1, comp = i & 1;
      const int m = row0 + rr;
      const float* src = which == 0 ? a.st2 : (which == 1 ? a.st1 : a.st0);
      st_s[i] = (m < a.M && (which < 2 || a.feature_norm)) ? src[2 * (size_t)m + comp] : 0.f;
    }
    __syncthreads();
    // ---- B = [x2 | h_prev | 1 | 0..]  (144 features) ----
    // Every staging phase below is two loops: all global loads of the phase first (independent, all in flight together), then the
    // LayerNorm / TF32 split / shared-memory stores -- one memory round trip per phase instead of one per loop iteration.
    {
      constexpr int NIT = (144 * 16 + WG_THREADS - 1) / WG_THREADS;
      float raw[NIT][4];
#pragma unroll
      for (int it = 0; it < NIT; ++it) {
        const int p = tid + it * WG_THREADS;
        int n, kq;
        wg_pair(p, &n, &kq);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int m = row0 + 4 * kq + j;
          float v = 0.f;
          if (p < 144 * 16 && m < a.M) {
            if (n < 64) v = a.u2[(size_t)m * MX_H + n];
            else if (n < 128) {
              if (a.no_gru) v = 0.f;                     // MLP variant: no recurrent matrix
              else if (((m / N) % T1) > 0) v = a.hall[(size_t)(m - N) * MX_H + (n - 64)];
              else if (a.h0) v = a.h0[(size_t)m * MX_H + (n - 64)];
            } else if (n == 128) v = 1.f;
          }
          raw[it][j] = v;
        }
      }
#pragma unroll
      for (int it = 0; it < NIT; ++it) {
        const int p = tid + it * WG_THREADS;
        if (p >= 144 * 16) break;
        int n, kq;
        wg_pair(p, &n, &kq);
        float x[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int rr = 4 * kq + j;
          x[j] = (n < 64 && row0 + rr < a.M) ? (raw[it][j] - st_s[2 * rr]) * st_s[2 * rr + 1] * par_s[n] + par_s[64 + n] : raw[it][j];
        }
        wg_put(b_hi, b_lo, n, kq, x);
      }
    }
    // ---- A = [dgi_r | dgi_z] -> D1 ; then A = [dgi_n | dgi_n * r] -> D2 (same B) ----
    for (int pass = 0; pass < 2; ++pass) {
      {
        constexpr int NIT = 128 * 16 / WG_THREADS;
        static_assert(NIT * WG_THREADS == 128 * 16, "A tile pairs must divide over the CTA");
        float raw[NIT][4], rg[NIT][4];
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
          int f, kq;
          wg_pair(tid + it * WG_THREADS, &f, &kq);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int m = row0 + 4 * kq + j;
            float v = 0.f, g = 1.f;
            if (m < a.M) {
              if (pass == 0) v = a.dgi[(size_t)m * MX_G + f];
              else {
                v = a.dgi[(size_t)m * MX_G + 2 * MX_H + (f & 63)];
                if (f >= 64) g = a.no_gru ? 0.f : a.gates[(size_t)m * MX_G + (f - 64)];
              }
            }
            raw[it][j] = v; rg[it][j] = g;
          }
        }
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
          int f, kq;
          wg_pair(tid + it * WG_THREADS, &f, &kq);
          float x[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) x[j] = (pass == 1 && f >= 64) ? raw[it][j] * rg[it][j] : raw[it][j];
          wg_put(a_hi, a_lo, f, kq, x);
        }
      }
      tc::fence_async_smem();
      __syncthreads();
      tc::mma(acc, pass * WG_DSTRIDE, a_hi, a_lo, b_hi, b_lo, 144, WG_ROWS, 3, acc0);
      tc::arrive(bar);
      tc::mbar_wait(bar, phase);      // the MMAs have read the tiles: A (and after the second pass B) may be refilled
      phase ^= 1;
    }
    // ---- A = [da2 | da1], B = [x1 | x0 | 1] -> D3 ----
    {
      constexpr int NA = 128 * 16 / WG_THREADS;
      constexpr int NB = ((64 + WG_MAX_IN) * 16 + WG_THREADS - 1) / WG_THREADS;
      float ra[NA][4], rb[NB][4];
#pragma unroll
      for (int it = 0; it < NA; ++it) {
        int f, kq;
        wg_pair(tid + it * WG_THREADS, &f, &kq);
        const float* src = f < 64 ? a.da2_out : a.da1_out;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int m = row0 + 4 * kq + j;
          ra[it][j] = m < a.M ? src[(size_t)m * MX_H + (f & 63)] : 0.f;
        }
      }
#pragma unroll
      for (int it = 0; it < NB; ++it) {
        const int p = tid + it * WG_THREADS;
        int n, kq;
        wg_pair(p, &n, &kq);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int m = row0 + 4 * kq + j;
          float v = 0.f;
          if (p < N3 * 16 && m < a.M) {
            if (n < 64) v = a.u1[(size_t)m * MX_H + n];
            else if (n < 64 + I) v = a.X[(size_t)m * a.ldx + (n - 64)];
          }
          rb[it][j] = v;
        }
      }
#pragma unroll
      for (int it = 0; it < NA; ++it) {
        int f, kq;
        wg_pair(tid + it * WG_THREADS, &f, &kq);
        wg_put(a_hi, a_lo, f, kq, ra[it]);
      }
#pragma unroll
      for (int it = 0; it < NB; ++it) {
        const int p = tid + it * WG_THREADS;
        if (p >= N3 * 16) break;
        int n, kq;
        wg_pair(p, &n, &kq);
        float x[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int rr = 4 * kq + j;
          float v = rb[it][j];
          if (row0 + rr < a.M) {
            if (n < 64) v = (v - st_s[2 * WG_ROWS + 2 * rr]) * st_s[2 * WG_ROWS + 2 * rr + 1] * par_s[128 + n] + par_s[192 + n];
            else if (n < 64 + I && a.feature_norm) {
              const int c = n - 64;
              v = (v - st_s[4 * WG_ROWS + 2 * rr]) * st_s[4 * WG_ROWS + 2 * rr + 1] * par_s[256 + c] + par_s[384 + c];
            }
          }
          x[j] = v;
        }
        wg_put(b_hi, b_lo, n, kq, x);
      }
    }
    for (int p = tid; p < 16 * 16; p += blockDim.x) {      // the ones block: feature 0 = 1 for valid rows (lo part: zeros)
      int n, kq;
      wg_pair(p, &n, &kq);
      float x[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) x[j] = (n == 0 && row0 + 4 * kq + j < a.M) ? 1.f : 0.f;
      wg_put(o_hi, o_lo, n, kq, x);
    }
    tc::fence_async_smem();
    __syncthreads();
    tc::mma(acc, 2 * WG_DSTRIDE, a_hi, a_lo, b_hi, b_lo, N3, WG_ROWS, 3, acc0);
    tc::mma(acc, WG_ONES_COL, a_hi, a_lo, o_hi, o_lo, 16, WG_ROWS, 3, acc0);
    tc::arrive(bar);      // one arrival for both
    tc::mbar_wait(bar, phase);
    phase ^= 1;
  }
  // ---- epilogue: thread r (warps 0-3) = accumulator row r -> this CTA's gradient partial ----
  float* gp = a.gpart + (size_t)blockIdx.x * a.P;
  if (warp < 4) {
  const bool any = iter > 0;      // a CTA without rows writes zeros (its accumulator was never written)
  const int r = tid;
  float v[64];
  float t[32];
  // D1: gates r, z
  if (any) tc::ld_row(acc, 0, r, v);
#pragma unroll
  for (int c4 = 0; c4 < 16; ++c4)
    *reinterpret_cast<float4*>(gp + L.wih + (size_t)r * MX_H + 4 * c4) = any ? make_float4(v[4 * c4], v[4 * c4 + 1], v[4 * c4 + 2], v[4 * c4 + 3]) : make_float4(0.f, 0.f, 0.f, 0.f);
  const bool gru = !a.no_gru;       // MLP variant: the recurrent slots of the partial are never written (they stay at their initial zeros)
  if (any) tc::ld_row(acc, 64, r, v);
  if (gru) {
#pragma unroll
    for (int c4 = 0; c4 < 16; ++c4)
      *reinterpret_cast<float4*>(gp + L.whh + (size_t)r * MX_H + 4 * c4) = any ? make_float4(v[4 * c4], v[4 * c4 + 1], v[4 * c4 + 2], v[4 * c4 + 3]) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (any) tc::ld_row(acc, 128, r, t);      // column 128: D1's ones column; column 144 (= t[16]): [da2 | da1]^T . 1
  gp[L.bih + r] = any ? t[0] : 0.f;
  if (gru) gp[L.bhh + r] = any ? t[0] : 0.f;
  gp[(r < 64 ? L.b2 : L.b1) + (r & 63)] = any ? t[16] : 0.f;
  // D2: n gate.  rows 0-63: dW_ih[128 + r] = cols 0-63, db_ih ; rows 64-127: dW_hh[128 + r - 64] = cols 64-127, db_hh
  if (any) tc::ld_row(acc, WG_DSTRIDE + (r < 64 ? 0 : 64), r, v);
  if (r < 64 || gru) {
    float* dst = gp + (r < 64 ? L.wih : L.whh) + (size_t)(128 + (r & 63)) * MX_H;
#pragma unroll
    for (int c4 = 0; c4 < 16; ++c4)
      *reinterpret_cast<float4*>(dst + 4 * c4) = any ? make_float4(v[4 * c4], v[4 * c4 + 1], v[4 * c4 + 2], v[4 * c4 + 3]) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (any) tc::ld_row(acc, WG_DSTRIDE + 128, r, t);
  if (r < 64 || gru) gp[(r < 64 ? L.bih : L.bhh) + 128 + (r & 63)] = any ? t[0] : 0.f;
  // D3: rows 0-63: dW2[r] = cols 0-63, db2 ; rows 64-127: dW1[r - 64][0:I] = cols 64.., db1
  if (any) tc::ld_row(acc, 2 * WG_DSTRIDE + (r < 64 ? 0 : 64), r, v);
  if (r < 64) {
#pragma unroll
    for (int c4 = 0; c4 < 16; ++c4)
      *reinterpret_cast<float4*>(gp + L.w2 + (size_t)r * MX_H + 4 * c4) = any ? make_float4(v[4 * c4], v[4 * c4 + 1], v[4 * c4 + 2], v[4 * c4 + 3]) : make_float4(0.f, 0.f, 0.f, 0.f);
  } else {
    float* dst = gp + L.w1 + (size_t)(r - 64) * I;
#pragma unroll
    for (int c = 0; c < 64; ++c)
      if (c < I) dst[c] = any ? v[c] : 0.f;
    if (I > 64) {                                 // wide inputs: the second 64-column block of x0 (CTA-uniform branch)
      float v2[64];
      if (any) tc::ld_row(acc, 2 * WG_DSTRIDE + 128, r, v2);
#pragma unroll
      for (int c = 0; c < 64; ++c)
        if (64 + c < I) dst[64 + c] = any ? v2[c] : 0.f;
    }
  }
  }
  if (w.ln_parts > 0) {      // LayerNorm sums of k_front_bwd_tc's CTAs blockIdx.x, + gridDim.x, ... (fixed order) -> this partial row
    for (int c = tid; c < 512; c += blockDim.x) {
      float sum = 0.f;
      for (int r = blockIdx.x; r < w.ln_parts; r += gridDim.x) sum += a.ln_part[(size_t)r * 512 + c];
      const int which = c >> 6;      // 0 ln2_g, 1 ln2_b, 2 ln1_g, 3 ln1_b, 4-5 fn_g, 6-7 fn_b
      if (which < 4) gp[(which == 0 ? L.ln2_g : which == 1 ? L.ln2_b : which == 2 ? L.ln1_g : L.ln1_b) + (c & 63)] = sum;
      else { const int cc = (c - 256) & 127; if (cc < I) gp[(c < 384 ? L.fn_g : L.fn_b) + cc] = sum; }
    }
  } else
  if (w.ln_zero_from >= 0 && (int)blockIdx.x >= w.ln_zero_from) {
    for (int c = tid; c < MX_H; c += blockDim.x) { gp[L.ln2_g + c] = 0.f; gp[L.ln2_b + c] = 0.f; gp[L.ln1_g + c] = 0.f; gp[L.ln1_b + c] = 0.f; }
    for (int c = tid; c < I; c += blockDim.x) { gp[L.fn_g + c] = 0.f; gp[L.fn_b + c] = 0.f; }
  }
}

bool mx_wgrad_tc_usable(const FrontBwdArgs& a) {
  return wgrad_mode(a.L.in_dim) && a.da2_out && a.da1_out && !a.skip_wgrad && a.L.in_dim <= WG_MAX_IN && a.M >= 1;
}

static int launch_wgrad_tc(const FrontBwdArgs& a, int nparts, int ln_zero_from, cudaStream_t s, int ln_parts = 0);
int mx_launch_wgrad_tc(const FrontBwdArgs& a, int nparts, cudaStream_t s) { return launch_wgrad_tc(a, nparts, -1, s); }
static int launch_wgrad_tc(const FrontBwdArgs& a, int nparts, int ln_zero_from, cudaStream_t s, int ln_parts) {
  {   // CTAs beyond the last 64-row chunk have no rows and never touch their accumulator
    const int busy = nparts < mx_ceil_div(a.M, WG_ROWS) ? nparts : mx_ceil_div(a.M, WG_ROWS);
    if (!a.tc_acc || (int64_t)busy * 512 > a.tc_acc_cols) { mx_set_error("wgrad_tc: accumulator region missing or too small"); return 1; }
  }
  WgradArgs w;
  w.f = a;
  w.ln_zero_from = ln_zero_from;
  w.ln_parts = ln_parts;
  w.nchunks = mx_ceil_div(a.M, WG_ROWS);
  w.Kp16 = mx_round_up(a.L.in_dim, 16);
  WgradSmem sm = wgrad_smem(64 + w.Kp16);
  return mx_launch("k_wgrad_tc", k_wgrad_tc, dim3(nparts), dim3(WG_THREADS), (size_t)sm.total, s, MX_STEP, w, sm);
}


// =====================================================================================================
// k_front_bwd_tc: the data-gradient chain of the front layers on wgmma (option wgrad_tc = 2; with k_wgrad_tc it replaces
// k_front_bwd for input widths <= 64).  Mirror image of k_front_fwd_tc: a 128-row tile per CTA, thread r owns row r, so the three
// LayerNorm backward passes and ReLU masks run on registers after the accumulator row is read:
//   dx2 = dgi . W_ih (K = 192 fed as three gate chunks that accumulate) -> LN2' , ReLU' -> da2
//   dx1 = da2 . W2 -> LN1', ReLU' -> da1 ;  dx0 = da1 . W1 -> the feature LayerNorm's gain / bias gradients
// B operands are TRANSPOSED weight images (k_tc_prep_weights_T).  da2 / da1 go to global memory for k_wgrad_tc.  LayerNorm gain / bias
// gradients are column sums over rows = over threads: each tile writes [dy * xhat | dy] through an XOR-swizzled scratch (the A
// tile's shared memory, free between MMAs) and threads 0-63 / 64-127 keep running sums of one column each.
// =====================================================================================================
struct BwdTcSmem { int o_ahi, o_alo, o_wih, o_w2, o_w1, total; };
static BwdTcSmem bwd_tc_smem(int Kp16, bool stream = false) {
  BwdTcSmem s;
  int o = 0;
  s.o_ahi = o; o += 128 * 64 * 4;
  s.o_alo = o; o += 128 * 64 * 4;
  if (stream) {      // gate chunks, W2^T and W1^T take turns in one region (copied from the image while the previous operand's epilogue runs)
    s.o_wih = s.o_w2 = s.o_w1 = o;
    o += 2 * (Kp16 > 64 ? Kp16 : 64) * 64 * 4;
    s.total = o;
    return s;
  }
  s.o_wih = o; o += 3 * 2 * 64 * 64 * 4;      // three gate chunks, each [64][64] hi | lo
  s.o_w2 = o;
  if (Kp16 <= 64) {                           // everything resident: 224 KB at obs 64
    o += 2 * 64 * 64 * 4;
    s.o_w1 = o; o += 2 * Kp16 * 64 * 4;
  } else {                                    // wide inputs: W2^T and W1^T take turns in one region, restaged per tile from the image
    s.o_w1 = o; o += 2 * Kp16 * 64 * 4;
  }
  s.total = o;
  return s;
}
size_t mx_tc_imageT_floats(int in_dim) { return (size_t)2 * (3 * 64 * 64 + 64 * 64 + mx_round_up(in_dim, 16) * 64); }

// transposed images: B[n][k] with n = the layer's INPUT feature, k = its output feature (what the data gradient contracts over)
__global__ void __launch_bounds__(256) k_tc_prep_weights_T(const float* __restrict__ th, MxNetLayout L, float* img) {
  const int I = L.in_dim, Kp16 = (I + 15) & ~15;
  const int n_ih = 3 * 64 * 64, n_2 = 64 * 64, n_1 = Kp16 * 64;
  char* base = reinterpret_cast<char*>(img);
  MX_PDL_WAIT();
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < n_ih + n_2 + n_1; idx += gridDim.x * blockDim.x) {
    if (idx < n_ih) {
      const int c = idx / 4096, j = idx - c * 4096, n = j >> 6, k = j & 63;          // chunk c: gates 64c .. 64c+63
      char* hi = base + (size_t)c * 2 * 4096 * 4;
      tc::put_split(hi, hi + 4096 * 4, n, k, 64, th[L.wih + (size_t)(64 * c + k) * MX_H + n]);
    } else if (idx < n_ih + n_2) {
      const int j = idx - n_ih, n = j >> 6, k = j & 63;
      char* hi = base + (size_t)2 * n_ih * 4;
      tc::put_split(hi, hi + 4096 * 4, n, k, 64, th[L.w2 + (size_t)k * MX_H + n]);
    } else {
      const int j = idx - n_ih - n_2, n = j >> 6, k = j & 63;
      char* hi = base + (size_t)2 * (n_ih + n_2) * 4;
      tc::put_split(hi, hi + (size_t)n_1 * 4, n, k, 64, n < I ? th[L.w1 + (size_t)k * I + n] : 0.f);
    }
  }
}

__device__ __forceinline__ void bt_put_row64(char* hi, char* lo, int r, const float (&x)[64]) {
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
// Column sums over the tile's 128 rows of two [128][64] arrays, one row per thread.  The rows are written into two 32 KB scratch
// arrays (element (r, c) at r * 64 + (c ^ (r & 31)): conflict-free for the row writes and for the column reads); then threads 0-63
// add column t of the first array to their running sum, threads 64-127 column t - 64 of the second.
#define BT_SC(r, c) ((r) * 64 + ((c) ^ ((r) & 31)))
__device__ __forceinline__ void bt_colsum_read(const float* sc0, const float* sc1, int tid, float* acc) {
  __syncthreads();
  const float* sc = tid < 64 ? sc0 : sc1;
  const int col = tid & 63;
  float s = 0.f;
#pragma unroll 8
  for (int r = 0; r < 128; ++r) s += sc[BT_SC(r, col)];
  *acc += s;
  __syncthreads();
}
// LayerNorm backward + ReLU mask for one row held in registers: dy -> da (in place); the products for the gain / bias gradients go
// straight into the scratch rows (sc0: dy * xhat, sc1: dy)
__device__ __forceinline__ void bt_ln_bwd_relu(bool act_tanh, float (&dy)[64], const float* __restrict__ urow, bool ok, float mean, float rstd, const float* gamma_s,
                                               float* sc0, float* sc1, int tid) {
  float u[64];
#pragma unroll
  for (int c4 = 0; c4 < 16; ++c4) {
    const float4 q = ok ? *reinterpret_cast<const float4*>(urow + 4 * c4) : make_float4(0.f, 0.f, 0.f, 0.f);
    u[4 * c4] = q.x; u[4 * c4 + 1] = q.y; u[4 * c4 + 2] = q.z; u[4 * c4 + 3] = q.w;
  }
  float p1[8], p2[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { p1[i] = 0.f; p2[i] = 0.f; }
#pragma unroll
  for (int c = 0; c < 64; ++c) {
    const float xh = ok ? (u[c] - mean) * rstd : 0.f;
    sc0[BT_SC(tid, c)] = dy[c] * xh;
    sc1[BT_SC(tid, c)] = dy[c];
    const float dxh = dy[c] * gamma_s[c];
    dy[c] = dxh;
    p1[c & 7] += dxh;
    p2[c & 7] = fmaf(dxh, xh, p2[c & 7]);
  }
  const float s1 = (((p1[0] + p1[1]) + (p1[2] + p1[3])) + ((p1[4] + p1[5]) + (p1[6] + p1[7]))) * (1.f / 64.f);
  const float s2 = (((p2[0] + p2[1]) + (p2[2] + p2[3])) + ((p2[4] + p2[5]) + (p2[6] + p2[7]))) * (1.f / 64.f);
#pragma unroll
  for (int c = 0; c < 64; ++c) {
    const float xh = ok ? (u[c] - mean) * rstd : 0.f;
    const float du = rstd * (dy[c] - s1 - xh * s2);
    dy[c] = act_tanh ? du * (1.f - u[c] * u[c]) : (u[c] > 0.f ? du : 0.f);
  }
}

__global__ void __launch_bounds__(128, 2) k_front_bwd_tc(FrontBwdArgs a, BwdTcSmem sm) {
  MX_DYN_SMEM_RAW(smem_raw);
  __shared__ __align__(8) tc::Bar bar_s;
  __shared__ float par_s[2 * 64];            // gains: ln2 | ln1
  const MxNetLayout L = a.L;
  const float* __restrict__ th = a.theta;
  const int tid = threadIdx.x;
  const int I = L.in_dim, Kp16 = (I + 15) & ~15;
  char* base = reinterpret_cast<char*>(smem_raw);
  char *a_hi = base + sm.o_ahi, *a_lo = base + sm.o_alo, *wih = base + sm.o_wih, *w2 = base + sm.o_w2, *w1 = base + sm.o_w1;
  float* sc0 = reinterpret_cast<float*>(a_hi);
  float* sc1 = reinterpret_cast<float*>(a_lo);
  const uint32_t bar = tc::bar_addr(&bar_s);
  const bool stream = sm.o_wih == sm.o_w2;              // one chunk buffer for every weight operand (two CTAs per SM)
  const bool restage = !stream && sm.o_w1 == sm.o_w2;
  const float* img_w2 = a.tc_imgT + 2 * 3 * 4096;
  const float* img_w1 = img_w2 + 2 * 4096;
  float* acc = tc::cta_slice(a.tc_acc, 128);
  if (tid == 0) {
    tc::mbar_init(bar, blockDim.x);
    tc::mbar_init_fence();
  }
  for (int i = tid; i < 64; i += blockDim.x) { par_s[i] = th[L.ln2_g + i]; par_s[64 + i] = th[L.ln1_g + i]; }
  MX_PDL_WAIT();
  {   // the transposed weight images are byte-identical to the shared-memory weight region (resident part)
    const float* src = a.tc_imgT;
    float* dst = reinterpret_cast<float*>(wih);
    const int nvec = stream ? (2 * 4096 * 4) >> 4 : ((restage ? sm.o_w2 : sm.total) - sm.o_wih) >> 4;      // streamed: the first gate chunk only
    for (int v = tid; v < nvec; v += blockDim.x) mx_cp16(dst + 4 * v, src + 4 * v);
    mx_cp_commit();
  }
  auto stage_chunk = [&](const float* src, int nbytes) {      // streamed mode: the chunk buffer is free once the MMAs that read it have completed
    float* dst = reinterpret_cast<float*>(wih);
    for (int v = tid; v < (nbytes >> 4); v += blockDim.x) mx_cp16(dst + 4 * v, src + 4 * v);
    mx_cp_commit();
  };
  __syncthreads();
  uint32_t phase = 0;
  float acc2 = 0.f, acc1 = 0.f, acc0a = 0.f, acc0b = 0.f;      // running column sums: threads 0-63 gain gradients, 64-127 bias gradients
  const int ntiles = (a.M + 127) / 128;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int m = tile * 128 + tid;
    const bool ok = m < a.M;
    const size_t mm = ok ? (size_t)m : 0;
    // ---- dx2 = dgi . W_ih : three gate chunks ----
    for (int ch = 0; ch < 3; ++ch) {
      float x[64];
#pragma unroll
      for (int c4 = 0; c4 < 16; ++c4) {
        const float4 q = ok ? *reinterpret_cast<const float4*>(a.dgi + mm * MX_G + 64 * ch + 4 * c4) : make_float4(0.f, 0.f, 0.f, 0.f);
        x[4 * c4] = q.x; x[4 * c4 + 1] = q.y; x[4 * c4 + 2] = q.z; x[4 * c4 + 3] = q.w;
      }
      bt_put_row64(a_hi, a_lo, tid, x);
      mx_cp_wait<0>();
      tc::fence_async_smem();
      __syncthreads();
      const char* wch = stream ? wih : wih + ch * 2 * 4096 * 4;
      tc::mma(acc, 0, a_hi, a_lo, wch, wch + 4096 * 4, 64, 64, 3, ch > 0 ? 1u : 0u);
      tc::arrive(bar);
      tc::mbar_wait(bar, phase);
      phase ^= 1;
      if (stream) stage_chunk(ch < 2 ? a.tc_imgT + (ch + 1) * 2 * 4096 : img_w2, 2 * 4096 * 4);      // next gate chunk, then W2^T: in flight during the loads / epilogue
    }
    // ---- LN2', ReLU' -> da2 ; then fc2 and LN1', ReLU' -> da1 ----
    for (int layer = 0; layer < 2; ++layer) {
      float v[64];
      tc::ld_row(acc, 0, tid, v);
      const float* st = layer == 0 ? a.st2 : a.st1;
      const float* uu = layer == 0 ? a.u2 : a.u1;
      // (the MMAs that read the A tile have completed: its shared memory is the scratch until the next operand is written)
      bt_ln_bwd_relu(a.act_tanh != 0, v, uu + mm * MX_H, ok, ok ? st[2 * mm] : 0.f, ok ? st[2 * mm + 1] : 0.f, par_s + 64 * layer, sc0, sc1, tid);
      bt_colsum_read(sc0, sc1, tid, layer == 0 ? &acc2 : &acc1);
      float* da_out = layer == 0 ? a.da2_out : a.da1_out;
      if (ok) {
#pragma unroll
        for (int c4 = 0; c4 < 16; ++c4) *reinterpret_cast<float4*>(da_out + mm * MX_H + 4 * c4) = make_float4(v[4 * c4], v[4 * c4 + 1], v[4 * c4 + 2], v[4 * c4 + 3]);
      }
      bt_put_row64(a_hi, a_lo, tid, v);
      if (stream) mx_cp_wait<0>();
      else if (restage) {      // the previous MMAs that read this region have completed (every issue is waited for)
        const float* src = layer == 0 ? img_w2 : img_w1;
        float* dst = reinterpret_cast<float*>(w2);
        const int nvec = (layer == 0 ? 2 * 4096 * 4 : 2 * Kp16 * 64 * 4) >> 4;
        for (int q = tid; q < nvec; q += blockDim.x) mx_cp16(dst + 4 * q, src + 4 * q);
        mx_cp_commit();
        mx_cp_wait<0>();
      }
      tc::fence_async_smem();
      __syncthreads();
      if (layer == 0) tc::mma(acc, 0, a_hi, a_lo, w2, w2 + 4096 * 4, 64, 64, 3, 0);
      else tc::mma(acc, 0, a_hi, a_lo, w1, w1 + Kp16 * 64 * 4, Kp16, 64, 3, 0);
      tc::arrive(bar);
      tc::mbar_wait(bar, phase);
      phase ^= 1;
      if (stream) {
        if (layer == 0) stage_chunk(img_w1, 2 * Kp16 * 64 * 4);
        else if (tile + (int)gridDim.x < ntiles) stage_chunk(a.tc_imgT, 2 * 4096 * 4);      // the next tile's first gate chunk
      }
    }
    // ---- dx0 -> gain / bias gradients of the feature LayerNorm (64 input columns per round) ----
    {
      const float mean = (ok && a.feature_norm) ? a.st0[2 * mm] : 0.f, rstd = (ok && a.feature_norm) ? a.st0[2 * mm + 1] : 0.f;
      for (int cb = 0; 64 * cb < I; ++cb) {
        float v[64];
        tc::ld_row(acc, 64 * cb, tid, v);         // columns >= Kp16 hold leftovers of the previous layer: masked below
#pragma unroll
        for (int c4 = 0; c4 < 16; ++c4) {
          float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
          if (ok && 64 * cb + 4 * c4 < I) q = *reinterpret_cast<const float4*>(a.X + mm * a.ldx + 64 * cb + 4 * c4);
          const float xr[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int c = 4 * c4 + j;
            const float d = (ok && 64 * cb + c < I) ? v[c] : 0.f;
            sc0[BT_SC(tid, c)] = d * (xr[j] - mean) * rstd;
            sc1[BT_SC(tid, c)] = d;
          }
        }
        float part = 0.f;
        bt_colsum_read(sc0, sc1, tid, &part);
        if (cb == 0) acc0a += part; else acc0b += part;
      }
    }
    __syncthreads();     // accumulator reads drained before the next tile's MMAs
  }
  // ---- this CTA's partial of the LayerNorm gain / bias gradients ----
  const int col = tid & 63;
  if (a.ln_part) {      // two CTAs per SM = more CTAs than gradient partial rows: the sums go to a side array [CTA][512] that k_wgrad_tc folds in
    float* lp = a.ln_part + (size_t)blockIdx.x * 512;      // ln2_g | ln2_b | ln1_g | ln1_b | fn_g[128] | fn_b[128]
    const int half = tid < 64 ? 0 : 1;
    lp[64 * half + col] = acc2; lp[128 + 64 * half + col] = acc1;
    lp[256 + 128 * half + col] = (col < I && a.feature_norm) ? acc0a : 0.f;
    lp[256 + 128 * half + 64 + col] = (64 + col < I && a.feature_norm) ? acc0b : 0.f;
  } else {
  float* gp = a.gpart + (size_t)blockIdx.x * a.P;
  if (tid < 64) {
    gp[L.ln2_g + col] = acc2; gp[L.ln1_g + col] = acc1;
    if (col < I) gp[L.fn_g + col] = a.feature_norm ? acc0a : 0.f;
    if (64 + col < I) gp[L.fn_g + 64 + col] = a.feature_norm ? acc0b : 0.f;
  } else {
    gp[L.ln2_b + col] = acc2; gp[L.ln1_b + col] = acc1;
    if (col < I) gp[L.fn_b + col] = a.feature_norm ? acc0a : 0.f;
    if (64 + col < I) gp[L.fn_b + 64 + col] = a.feature_norm ? acc0b : 0.f;
  }
  }
  mx_cp_wait<0>();
}

bool mx_front_bwd_tc_usable(const FrontBwdArgs& a) {
  return wgrad_mode(a.L.in_dim) >= 2 && mx_wgrad_tc_usable(a) && a.tc_imgT && !a.dX && !a.h0 && (a.ldx & 3) == 0;
}

// k_tc_prep_weights_T -> k_front_bwd_tc -> k_wgrad_tc ; *nparts_used = the number of gradient partials written
bool mx_tc_prep_T_wanted(int in_dim) { return wgrad_mode(in_dim) >= 2 && in_dim <= WG_MAX_IN; }
int mx_launch_tc_prep_weights_T(const float* theta, const MxNetLayout& L, float* imgT, cudaStream_t s) {
  const int n = 3 * 4096 + 4096 + mx_round_up(L.in_dim, 16) * 64;
  return mx_launch("k_tc_prep_weights_T", k_tc_prep_weights_T, dim3((n + 255) / 256), dim3(256), 0, s, MX_STEP, theta, L, imgT);
}

int mx_launch_front_bwd_tc(const FrontBwdArgs& a, int* nparts_used, cudaStream_t s) {
  const int Kp16 = mx_round_up(a.L.in_dim, 16);
  if (!a.tc_imgT_ready && mx_launch_tc_prep_weights_T(a.theta, a.L, a.tc_imgT, s)) return 1;
  // streamed (every weight operand through ONE chunk buffer, two CTAs per SM) when the caller gives the side array for the LayerNorm sums
  const bool stream = a.ln_part != nullptr;
  BwdTcSmem sm = bwd_tc_smem(Kp16, stream);
  const int ntiles = mx_ceil_div(a.M, 128), nchunks = mx_ceil_div(a.M, WG_ROWS);
  int ga = mx_num_sms(), gb = mx_num_sms();
  if (stream && 2 * (sm.total + 2048) <= (int)MX_SMEM_OPTIN_MAX) ga = 2 * mx_num_sms();      // two CTAs per SM fit
  if (ga > ntiles) ga = ntiles;
  if (gb > nchunks) gb = nchunks;
  if (!a.tc_acc || a.tc_acc_cols < 512) { mx_set_error("front_bwd_tc: accumulator region missing or too small"); return 1; }
  if (ga * 128 > a.tc_acc_cols) ga = a.tc_acc_cols / 128;      // accumulator columns per CTA: 128 here, 512 in k_wgrad_tc
  if (gb * 512 > a.tc_acc_cols) gb = a.tc_acc_cols / 512;
  FrontBwdArgs b = a;
  b.wgrad_external = 1;
  if (ga > a.ln_part_rows && stream) ga = a.ln_part_rows;
  if (const int rc = mx_launch("k_front_bwd_tc", k_front_bwd_tc, dim3(ga), dim3(128), (size_t)sm.total, s, MX_STEP, b, sm)) return rc;
  *nparts_used = gb;
  if (stream) return launch_wgrad_tc(b, gb, -1, s, ga);
  return launch_wgrad_tc(b, gb, ga < gb ? ga : -1, s);
}
