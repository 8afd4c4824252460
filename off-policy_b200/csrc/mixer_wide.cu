// Wide-state QMIX mixer: the hypernetworks' state-reading first layers as tensor-core GEMMs (wgmma, 3xTF32).
//
// With SMAC's global-all-local state (every agent's observation appended to the global state, e.g. 2 374 floats on 3s5z_vs_3s6z) a
// tile of state rows no longer fits beside the hypernet tiles in shared memory (mixer.cu).  Such a learner (mx_mix_wide_state) runs the
// four state-reading layers -- hyper_w1 and hyper_w2 (first layers, or the only layers with 1-layer hypernets), hyper_b1 and hyper_b2's
// first layer -- as the stacked columns of one GEMM, and the hypernet kernels work from its outputs:
//
//   k_mixw_prep   : weights of the live and the target net -> row-major TF32 hi / lo images [net][Cp][Sp] + bias [net][Cp]
//   k_mixw_fwd    : pre[net][row][c] = sum_k share[row][k] W_net[c][k] + b_net[c] over every state row of the batch (row = b (T+1) + t);
//                   the live net uses rows t < T, the target net rows t >= 1, so the state is read once for both
//   k_mixw_wgrad  : dW[c][k] = sum_e d_pre[e][c] share[row(e)][k], db[c] = sum_e d_pre[e][c] over the E = B T live elements.  Every CTA
//                   owns a (128 columns x 64 state features) tile and reduces over all elements itself: the result is gradient
//                   partial 0 of the state layers and the optimiser reads that one partial (no per-CTA partial rows over ~S x C floats)
//
// Both GEMMs are D[128][N] += A[128][32] . B[N][32]^T chunks on tc::mma (mx_tc.cuh) with the accumulator in shared memory;
// operands are split into TF32 hi / lo on the way into shared memory (state rows, d_pre) or copied pre-split (the weight images).  The next
// chunk's weight tile is in flight (cp.async) and the next chunk's state values in registers while the tensor cores run the current one.
#include "mx_internal.h"
#include "mx_kernels.h"
#include "mx_tc.cuh"

#define MXW_KC 32           // K chunk (state features in the forward, elements in the weight gradient)
#define MXW_NB 128          // forward: output columns per CTA
#define MXW_NS 64           // weight gradient: state features per CTA

size_t mx_mixw_image_floats(const MxMixWide& w) { return (size_t)2 * ((size_t)2 * w.Cp * w.Sp + w.Cp); }

struct MixwRow { int j, r, w, b; };      // block of a stacked column (-1: padding), its row in the block, weight / bias offsets
MX_DEVINL MixwRow mixw_row(const MxMixWide& w, int c) {
  MixwRow o{-1, 0, 0, 0};
#pragma unroll
  for (int j = 0; j < 4; ++j)
    if (c >= w.col[j] && c < w.col[j] + w.rows[j]) { o.j = j; o.r = c - w.col[j]; o.w = w.w[j]; o.b = w.b[j]; }
  return o;
}

__global__ void __launch_bounds__(256) k_mixw_prep(const float* __restrict__ th0, const float* __restrict__ th1, MxMixWide w, int S, float* img) {
  const int net = blockIdx.y;
  const float* __restrict__ th = net ? th1 : th0;
  float* hi = img + (size_t)net * (2 * (size_t)w.Cp * w.Sp + w.Cp);
  float* lo = hi + (size_t)w.Cp * w.Sp;
  float* bias = lo + (size_t)w.Cp * w.Sp;
  const size_t n = (size_t)w.Cp * w.Sp;
  MX_PDL_WAIT();
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < n + w.Cp; idx += (size_t)gridDim.x * blockDim.x) {
    if (idx >= n) {
      const MixwRow o = mixw_row(w, (int)(idx - n));
      bias[idx - n] = o.j >= 0 ? th[o.b + o.r] : 0.f;
      continue;
    }
    const int c = (int)(idx / w.Sp), k = (int)(idx - (size_t)c * w.Sp);
    const MixwRow o = mixw_row(w, c);
    const float x = (o.j >= 0 && k < S) ? th[o.w + (size_t)o.r * S + k] : 0.f;
    const float h = tc::to_tf32(x);
    hi[idx] = h;
    lo[idx] = x - h;
  }
}

// ---- forward -------------------------------------------------------------------------------------------------------------------
struct MixwFwdSmem { int o_ahi, o_alo, o_bhi, o_blo, o_acc, total; };     // bytes; B tiles double-buffered
static MixwFwdSmem mixw_fwd_smem() {
  MixwFwdSmem m;
  int o = 0;
  m.o_ahi = o; o += 128 * MXW_KC * 4;
  m.o_alo = o; o += 128 * MXW_KC * 4;
  m.o_bhi = o; o += 2 * MXW_NB * MXW_KC * 4;
  m.o_blo = o; o += 2 * MXW_NB * MXW_KC * 4;
  m.o_acc = o; o += MXW_NB * 128 * 4;
  m.total = o;
  return m;
}

// weight rows [c0, c0 + nb) x K chunk kc of one net's image -> core-matrix tiles (16-byte async copies: 4 features of one row each)
MX_DEVINL void mixw_stage_w(char* hi, char* lo, const float* img_hi, const float* img_lo, int Sp, int c0, int nb, int kc) {
  for (int idx = threadIdx.x; idx < nb * (MXW_KC / 4); idx += blockDim.x) {
    const int r = idx / (MXW_KC / 4), k4 = idx - r * (MXW_KC / 4);
    const size_t g = (size_t)(c0 + r) * Sp + (size_t)kc * MXW_KC + 4 * k4;
    const uint32_t o = tc::core_off_bytes(r, 4 * k4, MXW_KC);
    mx_cp16(reinterpret_cast<float*>(hi + o), img_hi + g);
    mx_cp16(reinterpret_cast<float*>(lo + o), img_lo + g);
  }
}
// the thread's 8 float4 of a [128 rows][32] state chunk: zeros past the rows and past column S (the row's pad columns are not read)
MX_DEVINL void mixw_load_x(float4 (&v)[8], const float* __restrict__ X, int ld, int S, int R, int m0, int kc) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int idx = threadIdx.x + 128 * i, r = idx >> 3, k = kc * MXW_KC + 4 * (idx & 7);
    float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
    if (m0 + r < R && k < S) {
      const float* p = X + (size_t)(m0 + r) * ld + k;
      if (k + 4 <= S) x = mx_ld4(p);
      else { x.x = p[0]; if (k + 1 < S) x.y = p[1]; if (k + 2 < S) x.z = p[2]; }
    }
    v[i] = x;
  }
}
MX_DEVINL void mixw_put4(char* hi, char* lo, int r, int k, float4 x) {
  const uint32_t o = tc::core_off_bytes(r, k, MXW_KC);
  const float4 h = make_float4(tc::to_tf32(x.x), tc::to_tf32(x.y), tc::to_tf32(x.z), tc::to_tf32(x.w));
  mx_st4(reinterpret_cast<float*>(hi + o), h);
  mx_st4(reinterpret_cast<float*>(lo + o), make_float4(x.x - h.x, x.y - h.y, x.z - h.z, x.w - h.w));
}

// grid (row tiles of 128, 2 nets x column blocks of MXW_NB); thread r owns accumulator row r in the epilogue
__global__ void __launch_bounds__(128, 1) k_mixw_fwd(MixerArgs a, MixwFwdSmem sm) {
  MX_DYN_SMEM_RAW(smem_raw);
  __shared__ __align__(8) tc::Bar bar_s;
  const MxMixWide w = a.wl;
  const int tid = threadIdx.x;
  const int ncb = (w.Cp + MXW_NB - 1) / MXW_NB;
  const int net = blockIdx.y / ncb, c0 = (blockIdx.y - net * ncb) * MXW_NB;
  const int nb = w.Cp - c0 < MXW_NB ? w.Cp - c0 : MXW_NB;      // multiple of 16
  const int R = a.B * (a.T + 1), m0 = blockIdx.x * 128;
  const float* img_hi = a.wimg + (size_t)net * (2 * (size_t)w.Cp * w.Sp + w.Cp);
  const float* img_lo = img_hi + (size_t)w.Cp * w.Sp;
  const float* bias = img_lo + (size_t)w.Cp * w.Sp;
  char* a_hi = reinterpret_cast<char*>(smem_raw) + sm.o_ahi;
  char* a_lo = reinterpret_cast<char*>(smem_raw) + sm.o_alo;
  char* b_hi = reinterpret_cast<char*>(smem_raw) + sm.o_bhi;
  char* b_lo = reinterpret_cast<char*>(smem_raw) + sm.o_blo;
  const uint32_t bar = tc::bar_addr(&bar_s);
  float* acc = reinterpret_cast<float*>(smem_raw + sm.o_acc);
  if (tid == 0) {
    tc::mbar_init(bar, blockDim.x);
    tc::mbar_init_fence();
  }
  MX_PDL_WAIT();
  const int nk = w.Sp / MXW_KC;
  const int bstride = MXW_NB * MXW_KC * 4;
  float4 xv[8];
  mixw_load_x(xv, a.share, a.share_ld, a.L.S, R, m0, 0);
  mixw_stage_w(b_hi, b_lo, img_hi, img_lo, w.Sp, c0, nb, 0);
  mx_cp_commit();
  uint32_t phase = 0;
  for (int kc = 0; kc < nk; ++kc) {
    const int buf = kc & 1;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int idx = tid + 128 * i;
      mixw_put4(a_hi, a_lo, idx >> 3, 4 * (idx & 7), xv[i]);
    }
    if (kc + 1 < nk) {
      mixw_stage_w(b_hi + (buf ^ 1) * bstride, b_lo + (buf ^ 1) * bstride, img_hi, img_lo, w.Sp, c0, nb, kc + 1);
      mx_cp_commit();
      mx_cp_wait<1>();
    } else {
      mx_cp_wait<0>();
    }
    tc::fence_async_smem();
    __syncthreads();
    if (kc + 1 < nk) mixw_load_x(xv, a.share, a.share_ld, a.L.S, R, m0, kc + 1);      // in flight during the MMAs
    tc::mma(acc, 0, a_hi, a_lo, b_hi + buf * bstride, b_lo + buf * bstride, nb, MXW_KC, 3, kc > 0 ? 1u : 0u);
    tc::arrive(bar);
    tc::mbar_wait(bar, phase);
    phase ^= 1;
    __syncthreads();      // operand tiles free for the next chunk
  }
  const int m = m0 + tid;
  float* out = a.pre + ((size_t)net * R + m) * w.Cp + c0;
  for (int cc = 0; cc < nb; cc += 32) {
    float v[32];
    tc::ld_row(acc, cc, tid, v);
    if (m < R)
#pragma unroll
      for (int c = 0; c < 32; c += 4)
        if (cc + c < nb)
          mx_st4(out + cc + c, make_float4(v[c] + bias[c0 + cc + c], v[c + 1] + bias[c0 + cc + c + 1], v[c + 2] + bias[c0 + cc + c + 2],
                                           v[c + 3] + bias[c0 + cc + c + 3]));
  }
}

int mx_launch_mixw_state_fwd(const MixerArgs& a, cudaStream_t s) {
  const MxMixWide& w = a.wl;
  if (!a.wimg || !a.pre || a.share_ld % 4) { mx_set_error("mixer (wide state): workspace regions missing or share_ld not a multiple of 4"); return 1; }
  {
    const size_t n = (size_t)w.Cp * w.Sp + w.Cp;
    int grid = (int)((n + 255) / 256);
    if (grid > 4 * mx_num_sms()) grid = 4 * mx_num_sms();
    if (const int rc = mx_launch("k_mixw_prep", k_mixw_prep, dim3(grid, 2), dim3(256), 0, s, MX_STEP, a.theta, a.theta_tgt, w, a.L.S, a.wimg))
      return rc;
  }
  const MixwFwdSmem sm = mixw_fwd_smem();
  const int R = a.B * (a.T + 1);
  const dim3 grid(mx_ceil_div(R, 128), 2 * mx_ceil_div(w.Cp, MXW_NB));
  return mx_launch("k_mixw_fwd", k_mixw_fwd, grid, dim3(128), (size_t)sm.total, s, MX_STEP, a, sm);
}

// ---- weight gradient -----------------------------------------------------------------------------------------------------------
// A[c][e] = d_pre[e][c0 + c] (128 columns), B[n][e] = share[row(e)][k0 + n] (64 features) and, on the first feature tile, a row of
// ones (n = 64, padded to 80) whose accumulator column is the bias gradient
struct MixwGradSmem { int o_ahi, o_alo, o_bhi, o_blo, o_acc, total; };
static MixwGradSmem mixw_grad_smem() {
  MixwGradSmem m;
  int o = 0;
  m.o_ahi = o; o += 128 * MXW_KC * 4;
  m.o_alo = o; o += 128 * MXW_KC * 4;
  m.o_bhi = o; o += (MXW_NS + 16) * MXW_KC * 4;
  m.o_blo = o; o += (MXW_NS + 16) * MXW_KC * 4;
  m.o_acc = o; o += (MXW_NS + 16) * 128 * 4;
  m.total = o;
  return m;
}

// the thread's element quads of chunk kc: A (column c = idx & 127, elements 4 (idx >> 7) ..) and B (feature n = idx & 63, ..)
MX_DEVINL void mixw_load_g(float4 (&av)[8], float4 (&bv)[4], const MixerArgs& a, int c0, int k0, int E, int kc) {
  const int S = a.L.S, Cp = a.wl.Cp;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int idx = threadIdx.x + 128 * i, c = c0 + (idx & 127), e = kc * MXW_KC + 4 * (idx >> 7);
    float x[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) x[j] = (c < Cp && e + j < E) ? a.d_pre[(size_t)(e + j) * Cp + c] : 0.f;
    av[i] = make_float4(x[0], x[1], x[2], x[3]);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = threadIdx.x + 128 * i, k = k0 + (idx & 63), e = kc * MXW_KC + 4 * (idx >> 6);
    float x[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      x[j] = 0.f;
      if (k < S && e + j < E) {
        const int b = (e + j) / a.T, t = (e + j) - b * a.T;
        x[j] = a.share[((size_t)b * (a.T + 1) + t) * a.share_ld + k];
      }
    }
    bv[i] = make_float4(x[0], x[1], x[2], x[3]);
  }
}

// grid (feature tiles of MXW_NS, column tiles of 128)
__global__ void __launch_bounds__(128, 2) k_mixw_wgrad(MixerArgs a, MixwGradSmem sm) {
  MX_DYN_SMEM_RAW(smem_raw);
  __shared__ __align__(8) tc::Bar bar_s;
  const MxMixWide w = a.wl;
  const int tid = threadIdx.x;
  const int S = a.L.S, E = a.B * a.T;
  const int k0 = blockIdx.x * MXW_NS, c0 = blockIdx.y * 128;
  const bool with_bias = blockIdx.x == 0;
  const int nb = with_bias ? MXW_NS + 16 : MXW_NS;
  char* a_hi = reinterpret_cast<char*>(smem_raw) + sm.o_ahi;
  char* a_lo = reinterpret_cast<char*>(smem_raw) + sm.o_alo;
  char* b_hi = reinterpret_cast<char*>(smem_raw) + sm.o_bhi;
  char* b_lo = reinterpret_cast<char*>(smem_raw) + sm.o_blo;
  const uint32_t bar = tc::bar_addr(&bar_s);
  float* acc = reinterpret_cast<float*>(smem_raw + sm.o_acc);
  if (tid == 0) {
    tc::mbar_init(bar, blockDim.x);
    tc::mbar_init_fence();
  }
  MX_PDL_WAIT();
  const int nk = mx_ceil_div(E, MXW_KC);
  float4 av[8], bv[4];
  mixw_load_g(av, bv, a, c0, k0, E, 0);
  uint32_t phase = 0;
  for (int kc = 0; kc < nk; ++kc) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int idx = tid + 128 * i;
      mixw_put4(a_hi, a_lo, idx & 127, 4 * (idx >> 7), av[i]);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int idx = tid + 128 * i;
      mixw_put4(b_hi, b_lo, idx & 63, 4 * (idx >> 6), bv[i]);
    }
    if (with_bias)       // ones row (valid elements) + 15 zero rows
      for (int idx = tid; idx < 16 * (MXW_KC / 4); idx += 128) {
        const int n = idx / (MXW_KC / 4), q = idx - n * (MXW_KC / 4), e = kc * MXW_KC + 4 * q;
        float x[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) x[j] = (n == 0 && e + j < E) ? 1.f : 0.f;
        mixw_put4(b_hi, b_lo, MXW_NS + n, 4 * q, make_float4(x[0], x[1], x[2], x[3]));
      }
    tc::fence_async_smem();
    __syncthreads();
    if (kc + 1 < nk) mixw_load_g(av, bv, a, c0, k0, E, kc + 1);      // in flight during the MMAs
    tc::mma(acc, 0, a_hi, a_lo, b_hi, b_lo, nb, MXW_KC, 3, kc > 0 ? 1u : 0u);
    tc::arrive(bar);
    tc::mbar_wait(bar, phase);
    phase ^= 1;
    __syncthreads();
  }
  // row c of the accumulator = stacked column c0 + tid: gradient partial 0 of its weight row (and bias)
  const MixwRow o = mixw_row(w, c0 + tid);
  float v[32];
  for (int cc = 0; cc < MXW_NS; cc += 32) {
    tc::ld_row(acc, cc, tid, v);
    if (o.j >= 0)
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if (k0 + cc + i < S) a.gpart[o.w + (size_t)o.r * S + k0 + cc + i] = v[i];
  }
  if (with_bias) {      // accumulator column MXW_NS, read as element 16 of the 32 columns ending at nb = MXW_NS + 16
    tc::ld_row(acc, MXW_NS - 16, tid, v);
    if (o.j >= 0) a.gpart[o.b + o.r] = v[16];
  }
}

int mx_launch_mixw_state_wgrad(const MixerArgs& a, cudaStream_t s) {
  if (!a.d_pre) { mx_set_error("mixer (wide state): d_pre region missing"); return 1; }
  const MixwGradSmem sm = mixw_grad_smem();
  const dim3 grid(mx_ceil_div(a.L.S, MXW_NS), mx_ceil_div(a.wl.Cp, 128));
  return mx_launch("k_mixw_wgrad", k_mixw_wgrad, grid, dim3(128), (size_t)sm.total, s, MX_STEP, a, sm);
}
