// Forward kernels of the recurrent agent network (RNNBase + Linear head), live and target nets in one launch.
//
//   k_front_fwd   time-batched front: LN(x) -> fc1 -> ReLU -> LN -> fc2 -> ReLU -> LN -> W_ih (all T+1 steps at once)
//                 reference: algorithms/utils/mlp.py:25-29,76-87 + the input half of nn.GRU (rnn.py:21)
//   k_gru_fwd     the serial recurrence h_t = GRU(gi_t, h_{t-1}), W_hh resident in registers, h in shared memory
//                 reference: nn.GRU called from algorithms/utils/rnn.py:19-23 (gate order r,z,n; h_0 = 0)
//   k_qhead       LN(h_t) -> Linear(H,A), taken-action gather, avail-masked greedy argmax (double-Q), target gather
//                 reference: rnn.py:22, act.py:32, QMixPolicy.py:69-93,102-174, utils/util.py:297-302, qmix.py:134-148
//
// Row order: row-step m = (b*(T+1) + t)*N + n (episode-major, exactly the sampled batch's memory order), so the
// front kernels see one dense [M][ld] matrix; the reference stacks agents on the batch axis instead (qmix.py:108).
#include "mx_internal.h"
#include "mx_kernels.h"
#include "mx_tile.cuh"

// =====================================================================================================
// front forward
// =====================================================================================================
template <int RM>
__global__ void __launch_bounds__(MX_TILE_THREADS) k_front_fwd(FrontFwdArgs a) {
  constexpr int TM = 16 * RM;
  MX_DYN_SMEM(smem);
  const int net = blockIdx.y;
  const float* __restrict__ th = a.theta[net];
  const MxNetLayout L = a.L;
  const int I = L.in_dim, Ipad = (I + 3) & ~3;
  const int lda = mx_ld_dev(Ipad > MX_H ? Ipad : MX_H);
  const int ldw = lda;
  float* A_s = smem;                 // [TM][lda]
  float* Wc = A_s + TM * lda;        // [64][ldw]
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4, lane = tid & 31, warp = tid >> 5;
  const bool live = (net == 0);
  const int ntiles = (a.M + TM - 1) / TM;
  MX_PDL_WAIT();

  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int m0 = tile * TM;
    // ---- load the input rows (all loads of a warp's rows issued before any use), LayerNorm over the I features ----
    if (I <= 128) {
      constexpr int RW = TM / (MX_TILE_THREADS / 32);       // rows per warp
      float xv[RW][4];
#pragma unroll
      for (int q = 0; q < RW; ++q) {
        const int m = m0 + warp + q * (MX_TILE_THREADS / 32);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int c = lane + 32 * u;
          xv[q][u] = (m < a.M && c < I) ? a.X[(size_t)m * a.ldx + c] : 0.f;
        }
      }
#pragma unroll
      for (int q = 0; q < RW; ++q) {
        const int r = warp + q * (MX_TILE_THREADS / 32), m = m0 + r;
        float* row = A_s + r * lda;
        const float mean = mx_warp_sum(xv[q][0] + xv[q][1] + xv[q][2] + xv[q][3]) / (float)I;
        float qq = 0.f;
#pragma unroll
        for (int u = 0; u < 4; ++u) { const float d = (lane + 32 * u < I) ? xv[q][u] - mean : 0.f; qq += d * d; }
        const float rstd = rsqrtf(mx_warp_sum(qq) / (float)I + MX_LN_EPS);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int c = lane + 32 * u;
          if (c < Ipad) {
            float v = 0.f;
            if (c < I && m < a.M) v = a.feature_norm ? ((xv[q][u] - mean) * rstd * th[L.fn_g + c] + th[L.fn_b + c]) : xv[q][u];
            row[c] = v;
          }
        }
        if (live && lane == 0 && a.st0 && m < a.M) { a.st0[2 * (size_t)m] = mean; a.st0[2 * (size_t)m + 1] = rstd; }
      }
    } else
    for (int r = warp; r < TM; r += MX_TILE_THREADS / 32) {
      const int m = m0 + r;
      float* row = A_s + r * lda;
      if (m < a.M) {
        const float* x = a.X + (size_t)m * a.ldx;
        float s = 0.f;
        for (int c = lane; c < I; c += 32) s += x[c];
        const float mean = mx_warp_sum(s) / (float)I;
        float q = 0.f;
        for (int c = lane; c < I; c += 32) { float d = x[c] - mean; q += d * d; }
        const float rstd = rsqrtf(mx_warp_sum(q) / (float)I + MX_LN_EPS);
        for (int c = lane; c < Ipad; c += 32) {
          float v = 0.f;
          if (c < I) v = a.feature_norm ? ((x[c] - mean) * rstd * th[L.fn_g + c] + th[L.fn_b + c]) : x[c];
          row[c] = v;
        }
        if (live && lane == 0 && a.st0) { a.st0[2 * (size_t)m] = mean; a.st0[2 * (size_t)m + 1] = rstd; }
      } else {
        for (int c = lane; c < Ipad; c += 32) row[c] = 0.f;
      }
    }
    // ---- fc1 and fc2: Linear -> ReLU -> LayerNorm, output becomes the next layer's A operand ----
    for (int layer = 0; layer < 2; ++layer) {
      const int K = layer == 0 ? I : MX_H, Kpad = (K + 3) & ~3;
      const int w_off = layer == 0 ? L.w1 : L.w2, b_off = layer == 0 ? L.b1 : L.b2;
      const int g_off = layer == 0 ? L.ln1_g : L.ln2_g, be_off = layer == 0 ? L.ln1_b : L.ln2_b;
      mx_stage_weight(Wc, ldw, th + w_off, MX_H, K, K, 0, 0, Kpad);
      __syncthreads();
      float acc[RM][4];
#pragma unroll
      for (int i = 0; i < RM; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
      mx_mm_nt<RM>(A_s, lda, Wc, ldw, Kpad, acc);
#pragma unroll
      for (int i = 0; i < RM; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) { const float z = acc[i][j] + th[b_off + tx + 16 * j]; acc[i][j] = a.act_tanh ? tanhf(z) : fmaxf(z, 0.f); }
      float mean[RM], rstd[RM];
      mx_row_stats64<RM>(acc, mean, rstd);
      float* u_out = layer == 0 ? a.u1 : a.u2;
      float* st_out = layer == 0 ? a.st1 : a.st2;
      __syncthreads();   // every thread is done reading A_s / Wc
#pragma unroll
      for (int i = 0; i < RM; ++i) {
        const int r = ty * RM + i, m = m0 + r;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int c = tx + 16 * j;
          A_s[r * lda + c] = (acc[i][j] - mean[i]) * rstd[i] * th[g_off + c] + th[be_off + c];
          if (live && m < a.M && u_out) u_out[(size_t)m * MX_H + c] = acc[i][j];
        }
        if (live && m < a.M && tx == 0 && st_out) { st_out[2 * (size_t)m] = mean[i]; st_out[2 * (size_t)m + 1] = rstd[i]; }
      }
      // (the next mx_stage_weight writes Wc, which nobody reads any more; A_s is published by the barrier below)
    }
    // ---- gi = x2 . W_ih^T + b_ih, three 64-row chunks (r, z, n) ----
    float* gi = a.gi[net];
    for (int c3 = 0; c3 < 3; ++c3) {
      mx_stage_weight(Wc, ldw, th + L.wih, MX_G, MX_H, MX_H, 64 * c3, 0, MX_H);
      __syncthreads();
      float acc[RM][4];
#pragma unroll
      for (int i = 0; i < RM; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
      mx_mm_nt<RM>(A_s, lda, Wc, ldw, MX_H, acc);
#pragma unroll
      for (int i = 0; i < RM; ++i) {
        const int m = m0 + ty * RM + i;
        if (m < a.M) {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int c = 64 * c3 + tx + 16 * j;
            gi[(size_t)m * MX_G + c] = acc[i][j] + th[L.bih + c];
          }
        }
      }
      __syncthreads();   // Wc is restaged next; A_s is rewritten by the next tile
    }
  }
}

// =====================================================================================================
// GRU recurrence
// =====================================================================================================
#define GRU_PF 5                 // gi rows are prefetched this many steps ahead (L2 latency ~ 2-3 step times)
#define GRU_RING 8               // power of two: slot = t & 7;  GRU_PF + 2 <= GRU_RING (a slot is rewritten two barriers after its last read)
#define GRU_THREADS 256

template <int RPC>
__global__ void __launch_bounds__(GRU_THREADS, 1) k_gru_fwd(GruFwdArgs a) {
  // K-split quad layout: thread = 4*i + q owns, for unit i, the r/z/n rows of W_hh restricted to the interleaved
  // k-slice {16m + 4q + c : m,c < 4} (3 x 16 weights in registers, packed in pairs).  Per step a thread reads only ITS 16 h values
  // (4 LDS.128, the quad's four slices are 64 contiguous bytes -> one wavefront per warp instruction), runs 24 packed FFMA2
  // (two 4-deep chains per gate), and the quad completes the dot products with two xor-shuffles.  Every lane of the quad then
  // holds the full pre-activations, so the gates need no shared-memory exchange; h is double-buffered -> ONE barrier per step.
  // gi_t is streamed GRU_PF steps ahead with cp.async into a shared-memory ring.  The per-step instruction stream is what bounds
  // this kernel (a dependent chain, two warps per scheduler): stores are lane-uniform (lane q of a quad writes ONE of h / r / z / n
  // through a per-lane pointer, no divergent branches), the step loop is unrolled by two so the h buffers are compile-time.
  __shared__ __align__(16) float h_s[2][RPC][MX_H];
  __shared__ __align__(16) float gi_s[GRU_RING][RPC][MX_G];
  const int net = blockIdx.y;
  const float* __restrict__ th = a.theta[net];
  const int tid = threadIdx.x;
  const int i = tid >> 2, q = tid & 3;
  const int row0 = blockIdx.x * RPC;
  const bool live = (net == 0) && a.gates != nullptr;     // only the live net keeps gate activations for the backward pass
  float2 wr[8], wz[8], wn[8];
#pragma unroll
  for (int m = 0; m < 4; ++m)
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const int k = 16 * m + 4 * q + 2 * c;
      wr[2 * m + c] = make_float2(th[a.whh + i * MX_H + k], th[a.whh + i * MX_H + k + 1]);
      wz[2 * m + c] = make_float2(th[a.whh + (MX_H + i) * MX_H + k], th[a.whh + (MX_H + i) * MX_H + k + 1]);
      wn[2 * m + c] = make_float2(th[a.whh + (2 * MX_H + i) * MX_H + k], th[a.whh + (2 * MX_H + i) * MX_H + k + 1]);
    }
  const float br = th[a.bhh + i], bz = th[a.bhh + MX_H + i], bn = th[a.bhh + 2 * MX_H + i];
  MX_PDL_WAIT();        // the W_hh slice above is parameter data; everything below reads the predecessor's outputs
  for (int idx = tid; idx < 2 * RPC * MX_H; idx += GRU_THREADS) {                               // h_0 = 0 (QMixPolicy.py:193-196) or given
    const int r = (idx / MX_H) % RPC, c = idx % MX_H;
    (&h_s[0][0][0])[idx] = (a.h0 && row0 + r < a.R) ? a.h0[(size_t)(row0 + r) * MX_H + c] : 0.f;
  }
  for (int idx = tid; idx < GRU_RING * RPC * MX_G; idx += GRU_THREADS) (&gi_s[0][0][0])[idx] = 0.f;   // rows past R stay zero

  const float* gi = a.gi[net];
  const int T1 = a.T + 1, N = a.N;
  // lane-uniform stores: lane q of a quad writes value q of (h, r, z, n) of its unit; lane 0 also writes W_hn h + b_hn
  float* stp[RPC];
  float* hnp[RPC];
  bool st_on[RPC], hn_on[RPC];
  const size_t st_stride = (size_t)N * (q == 0 ? MX_H : MX_G), hn_stride = (size_t)N * MX_H;
#pragma unroll
  for (int r = 0; r < RPC; ++r) {
    const int row = row0 + r;
    const bool valid = row < a.R;
    const int b = valid ? row / N : 0, n = valid ? row % N : 0;
    const size_t m0 = ((size_t)b * T1) * N + n;      // + t*N per step
    stp[r] = (q == 0) ? a.hall[net] + m0 * MX_H + i : (live ? a.gates + m0 * MX_G + (q - 1) * MX_H + i : nullptr);
    hnp[r] = live ? a.hn + m0 * MX_H + i : nullptr;
    st_on[r] = valid && (q == 0 || live);
    hn_on[r] = valid && live && q == 0;
  }
  // prefetch assignment: RPC*48 16-byte pieces per step, at most one per thread (RPC <= 4)
  const int pf_r = tid / (MX_G / 4), pf_q = tid % (MX_G / 4);
  const bool pf_on = tid < RPC * (MX_G / 4) && (row0 + pf_r) < a.R;
  const float* pf_src = gi;
  float* pf_dst = &gi_s[0][0][0];
  if (pf_on) {
    const int row = row0 + pf_r;
    pf_src = gi + (((size_t)(row / N) * T1) * N + (row % N)) * MX_G + 4 * pf_q;
    pf_dst = &gi_s[0][pf_r][4 * pf_q];
  }
  const size_t pf_stride = (size_t)N * MX_G;
  auto prefetch = [&](int t) {          // called with t = 0, 1, 2, ... in order: the source pointer just advances
    if (pf_on && t < T1) { mx_cp16(pf_dst + (t & (GRU_RING - 1)) * (RPC * MX_G), pf_src); pf_src += pf_stride; }
    mx_cp_commit();
  };
  __syncthreads();          // the zero fill above precedes the first asynchronous copies into the ring
#pragma unroll
  for (int t = 0; t < GRU_PF; ++t) prefetch(t);
  mx_cp_wait<GRU_PF - 1>();
  __syncthreads();

  auto step = [&](const int t, const int cur) {
    const int nxt = cur ^ 1;
    prefetch(t + GRU_PF);               // slot (t+GRU_PF) & 7: last read at step t+GRU_PF-8 <= t-3, at least two barriers ago
    const float* gs = &gi_s[t & (GRU_RING - 1)][0][0];
#pragma unroll
    for (int r = 0; r < RPC; ++r) {
      const float* hrow = &h_s[cur][r][0];
      const float* g = gs + r * MX_G;
      float4 hv[4];
#pragma unroll
      for (int m = 0; m < 4; ++m) hv[m] = mx_ld4(hrow + 16 * m + 4 * q);
      const float gr = g[i] + br, gz = g[MX_H + i] + bz, gn = g[2 * MX_H + i], hp = hrow[i];      // off the dependent chain
      float2 r0 = make_float2(0.f, 0.f), r1 = r0, z0 = r0, z1 = r0, n0 = r0, n1 = r0;
#pragma unroll
      for (int m = 0; m < 4; ++m) {
        const float2 lo = make_float2(hv[m].x, hv[m].y), hi = make_float2(hv[m].z, hv[m].w);
        r0 = mx_ffma2(wr[2 * m], lo, r0); z0 = mx_ffma2(wz[2 * m], lo, z0); n0 = mx_ffma2(wn[2 * m], lo, n0);
        r1 = mx_ffma2(wr[2 * m + 1], hi, r1); z1 = mx_ffma2(wz[2 * m + 1], hi, z1); n1 = mx_ffma2(wn[2 * m + 1], hi, n1);
      }
      r0 = mx_fadd2(r0, r1); z0 = mx_fadd2(z0, z1); n0 = mx_fadd2(n0, n1);
      float pr = r0.x + r0.y, pz = z0.x + z0.y, pn = n0.x + n0.y;
      pr += __shfl_xor_sync(0xffffffffu, pr, 1); pn += __shfl_xor_sync(0xffffffffu, pn, 1); pz += __shfl_xor_sync(0xffffffffu, pz, 1);
      pr += __shfl_xor_sync(0xffffffffu, pr, 2); pn += __shfl_xor_sync(0xffffffffu, pn, 2); pz += __shfl_xor_sync(0xffffffffu, pz, 2);
      const float rg = mx_sigmoid_fast(pr + gr);
      const float hn = pn + bn;
      const float ng = mx_tanh_fast(fmaf(rg, hn, gn));
      const float zg = mx_sigmoid_fast(pz + gz);
      const float hnew = fmaf(zg, hp - ng, ng);             // (1-z)*n + z*h
      h_s[nxt][r][i] = hnew;              // all four lanes of the quad store the same value: keeps every lane on ONE path (a q == 0
                                          // guard lets the compiler specialise the other lanes and the warp then runs both paths)
      const float v = q == 0 ? hnew : (q == 1 ? rg : (q == 2 ? zg : ng));
      if (st_on[r]) *stp[r] = v;
      if (hn_on[r]) *hnp[r] = hn;
      stp[r] += st_stride; hnp[r] += hn_stride;
    }
    mx_cp_wait<GRU_PF - 1>();           // gi of step t+1 has landed (this thread's copies); the barrier publishes it
    __syncthreads();
  };
  int t = 0;
  for (; t + 1 < T1; t += 2) { step(t, 0); step(t + 1, 1); }
  if (t < T1) step(t, 0);
  mx_cp_wait<0>();
}

// ---- 128-thread variant (one row per CTA): K split over TWO lanes ---------------------------------------------------------------------------
// thread = 2*i + q owns, for unit i, the r/z/n rows of W_hh restricted to the interleaved k-slice {8m + 4q + c : m < 8, c < 4} (3 x 32
// weights in registers).  Half the warps of k_gru_fwd per row: on an SM that hosts two rows (192 row-CTAs on 148 SMs at the 3m shapes)
// every scheduler sees two warps instead of four, and on the others one -- the step is a dependent chain, fewer co-resident warps means
// less issue and LSU contention; one xor-shuffle level instead of two.
#define GRU2_THREADS 128
// Only ROWS = 1 is launched.  The parameter stays because the single-row rewrite of this source compiles to a different register
// allocation and schedule that measured up to 0.3 % slower at SMAC 8m (H100 80GB HBM3, 700 W power limit).
template <int ROWS>
__global__ void __launch_bounds__(GRU2_THREADS, 2) k_gru_fwd2(GruFwdArgs a) {
  __shared__ __align__(16) float h_s[2][ROWS][MX_H];
  __shared__ __align__(16) float gi_s[GRU_RING][ROWS][MX_G];
  const int net = blockIdx.y;
  const float* __restrict__ th = net ? a.theta[1] : a.theta[0];
  const int tid = threadIdx.x;
  const int i = tid >> 1, q = tid & 1;
  const bool live = (net == 0) && a.gates != nullptr;
  float2 wr[16], wz[16], wn[16];
#pragma unroll
  for (int m = 0; m < 8; ++m)
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const int k = 8 * m + 4 * q + 2 * c;
      wr[2 * m + c] = make_float2(th[a.whh + i * MX_H + k], th[a.whh + i * MX_H + k + 1]);
      wz[2 * m + c] = make_float2(th[a.whh + (MX_H + i) * MX_H + k], th[a.whh + (MX_H + i) * MX_H + k + 1]);
      wn[2 * m + c] = make_float2(th[a.whh + (2 * MX_H + i) * MX_H + k], th[a.whh + (2 * MX_H + i) * MX_H + k + 1]);
    }
  const float br = th[a.bhh + i], bz = th[a.bhh + MX_H + i], bn = th[a.bhh + 2 * MX_H + i];
  MX_PDL_WAIT();
  const float* gi = net ? a.gi[1] : a.gi[0];
  float* hall = net ? a.hall[1] : a.hall[0];
  const int T1 = a.T + 1, N = a.N;
  // lane-uniform stores: lane 0 of a pair writes h, r, W_hn h + b_hn; lane 1 writes z, n
  float *p1[ROWS], *p2[ROWS], *p3[ROWS];
  bool rok[ROWS];
  const float* pf_src[ROWS];
  const bool pf_on = tid < MX_G / 4;
#pragma unroll
  for (int r = 0; r < ROWS; ++r) {
    const int row = blockIdx.x * ROWS + r;
    rok[r] = row < a.R;
    const int rr = rok[r] ? row : 0;
    for (int idx = tid; idx < 2 * MX_H; idx += GRU2_THREADS) (&h_s[0][0][0])[(idx >> 6) * ROWS * MX_H + r * MX_H + (idx & 63)] = (a.h0 && idx < MX_H && rok[r]) ? a.h0[(size_t)rr * MX_H + idx] : 0.f;
    const int b = rr / N, n = rr % N;
    const size_t m0 = ((size_t)b * T1) * N + n;
    p1[r] = q == 0 ? hall + m0 * MX_H + i : (live ? a.gates + m0 * MX_G + MX_H + i : hall);
    p2[r] = live ? a.gates + m0 * MX_G + (q == 0 ? 0 : 2 * MX_H) + i : hall;
    p3[r] = live ? a.hn + m0 * MX_H + i : hall;
    pf_src[r] = gi + m0 * MX_G + 4 * (pf_on ? tid : 0);
  }
  const bool on1 = q == 0 || live, on2 = live, on3 = live && q == 0;
  const size_t s1 = (size_t)N * ((q == 0) ? MX_H : MX_G), s2 = (size_t)N * MX_G, s3 = (size_t)N * MX_H;
  float* pf_dst = &gi_s[0][0][4 * (pf_on ? tid : 0)];
  const size_t pf_stride = (size_t)N * MX_G;
  auto prefetch = [&](int t) {
    if (pf_on && t < T1) {
#pragma unroll
      for (int r = 0; r < ROWS; ++r) {
        if (rok[r]) mx_cp16(pf_dst + ((t & (GRU_RING - 1)) * ROWS + r) * MX_G, pf_src[r]);
        pf_src[r] += pf_stride;
      }
    }
    mx_cp_commit();
  };
#pragma unroll
  for (int t = 0; t < GRU_PF; ++t) prefetch(t);
  mx_cp_wait<GRU_PF - 1>();
  __syncthreads();

  auto step = [&](const int t, const int cur) {
    const int nxt = cur ^ 1;
    prefetch(t + GRU_PF);
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
      const float* g = &gi_s[t & (GRU_RING - 1)][r][0];
      const float* hrow = &h_s[cur][r][0];
      float4 hv[8];
#pragma unroll
      for (int m = 0; m < 8; ++m) hv[m] = mx_ld4(hrow + 8 * m + 4 * q);
      const float gr = g[i] + br, gz = g[MX_H + i] + bz, gn = g[2 * MX_H + i], hp = hrow[i];
      float2 r0 = make_float2(0.f, 0.f), r1 = r0, z0 = r0, z1 = r0, n0 = r0, n1 = r0;
#pragma unroll
      for (int m = 0; m < 8; ++m) {
        const float2 lo = make_float2(hv[m].x, hv[m].y), hi = make_float2(hv[m].z, hv[m].w);
        r0 = mx_ffma2(wr[2 * m], lo, r0); n0 = mx_ffma2(wn[2 * m], lo, n0); z0 = mx_ffma2(wz[2 * m], lo, z0);
        r1 = mx_ffma2(wr[2 * m + 1], hi, r1); n1 = mx_ffma2(wn[2 * m + 1], hi, n1); z1 = mx_ffma2(wz[2 * m + 1], hi, z1);
      }
      r0 = mx_fadd2(r0, r1); n0 = mx_fadd2(n0, n1); z0 = mx_fadd2(z0, z1);
      float pr = r0.x + r0.y, pn = n0.x + n0.y, pz = z0.x + z0.y;
      pr += __shfl_xor_sync(0xffffffffu, pr, 1); pn += __shfl_xor_sync(0xffffffffu, pn, 1); pz += __shfl_xor_sync(0xffffffffu, pz, 1);
      const float rg = mx_sigmoid_fast(pr + gr);
      const float hn = pn + bn;
      const float ng = mx_tanh_fast(fmaf(rg, hn, gn));
      const float zg = mx_sigmoid_fast(pz + gz);
      const float hnew = fmaf(zg, hp - ng, ng);
      h_s[nxt][r][i] = hnew;                  // both lanes of the pair store the same value: one code path for every lane
      if (rok[r]) {
        if (on1) *p1[r] = q == 0 ? hnew : zg;
        if (on2) *p2[r] = q == 0 ? rg : ng;
        if (on3) *p3[r] = hn;
      }
      p1[r] += s1; p2[r] += s2; p3[r] += s3;
    }
    mx_cp_wait<GRU_PF - 1>();
    __syncthreads();
  };
  int t = 0;
  for (; t + 1 < T1; t += 2) { step(t, 0); step(t + 1, 1); }
  if (t < T1) step(t, 0);
  mx_cp_wait<0>();
}

// =====================================================================================================
// Q head + action selection (one warp per row-step).  APL: availability bits per lane (1: A <= 32, 2: A <= 64, lane l holds
// actions l and l + 32)
// =====================================================================================================
template <int APL>
__global__ void __launch_bounds__(256) k_qhead(QHeadArgs a) {
  __shared__ float wq_s[2][32 * APL * MX_H];   // A <= 32 * APL
  __shared__ float bq_s[2][32 * APL];
  __shared__ float lg_s[2][MX_H], lb_s[2][MX_H];
  const int tid = threadIdx.x, lane = tid & 31;
  const int A = a.A;
  for (int net = 0; net < 2; ++net) {
    const float* th = a.theta[net];
    for (int i = tid; i < A * MX_H; i += blockDim.x) wq_s[net][i] = th[a.wq + i];
    for (int i = tid; i < A; i += blockDim.x) bq_s[net][i] = th[a.bq + i];
    for (int i = tid; i < MX_H; i += blockDim.x) { lg_s[net][i] = th[a.lno_g + i]; lb_s[net][i] = th[a.lno_b + i]; }
  }
  MX_PDL_WAIT();
  __syncthreads();
  const int wglobal = blockIdx.x * (blockDim.x >> 5) + (tid >> 5);
  const int wtotal = gridDim.x * (blockDim.x >> 5);
  const int T1 = a.T + 1, N = a.N;
  for (int m = wglobal; m < a.M; m += wtotal) {
    const int n = m % N;
    const int bt = m / N;
    const int t = bt % T1, b = bt / T1;
    float q_live_at_act = 0.f, tq_sel = 0.f;
    int greedy = 0;
    // all global operands of this row-step first (one round trip), then the arithmetic
    const float* hl = a.hall[0] + (size_t)m * MX_H;
    const float* ht = a.hall[1] + (size_t)m * MX_H;
    const float hl0 = hl[lane], hl1 = hl[lane + 32], ht0 = ht[lane], ht1 = ht[lane + 32];
    const int act = (t < a.T) ? a.act_idx[(size_t)b * a.ld_tn + (size_t)t * N + n] : 0;
    float av = 1.f;
    if (a.avail && lane < A) av = a.avail[(size_t)m * a.act_ld + lane];
    const unsigned avail_mask = __ballot_sync(0xffffffffu, av != 0.f);
    unsigned avail_hi = 0u;                                                      // actions 32..63
    if constexpr (APL == 2) {
      float av2 = 1.f;
      if (a.avail && lane + 32 < A) av2 = a.avail[(size_t)m * a.act_ld + lane + 32];
      avail_hi = __ballot_sync(0xffffffffu, av2 != 0.f);
    }
    // ---------------- live ----------------
    {
      const float mean = mx_warp_sum(hl0 + hl1) * (1.f / MX_H);
      const float d0 = hl0 - mean, d1 = hl1 - mean;
      const float rstd = rsqrtf(mx_warp_sum(d0 * d0 + d1 * d1) * (1.f / MX_H) + MX_LN_EPS);
      if (lane == 0) { a.sto[2 * (size_t)m] = mean; a.sto[2 * (size_t)m + 1] = rstd; }
      const float y0 = d0 * rstd * lg_s[0][lane] + lb_s[0][lane];
      const float y1 = d1 * rstd * lg_s[0][lane + 32] + lb_s[0][lane + 32];
      float best = 0.f;
      for (int k = 0; k < A; ++k) {
        float q = mx_warp_sum(y0 * wq_s[0][k * MX_H + lane] + y1 * wq_s[0][k * MX_H + lane + 32]) + bq_s[0][k];
        if (a.qall0 && lane == 0) a.qall0[(size_t)m * A + k] = q;
        if (k == act) q_live_at_act = q;
        unsigned on;
        if constexpr (APL == 1) on = (avail_mask >> k) & 1u;
        else on = ((k < 32 ? avail_mask : avail_hi) >> (k & 31)) & 1u;
        const float qm = on ? q : -1e10f;                                        // util.py:297-302
        if (k == 0 || qm > best) { best = qm; greedy = k; }                     // first maximum wins
      }
    }
    // ---------------- target ----------------
    {
      const float mean = mx_warp_sum(ht0 + ht1) * (1.f / MX_H);
      const float d0 = ht0 - mean, d1 = ht1 - mean;
      const float rstd = rsqrtf(mx_warp_sum(d0 * d0 + d1 * d1) * (1.f / MX_H) + MX_LN_EPS);
      const float y0 = d0 * rstd * lg_s[1][lane] + lb_s[1][lane];
      const float y1 = d1 * rstd * lg_s[1][lane + 32] + lb_s[1][lane + 32];
      float tbest = 0.f;
      for (int k = 0; k < A; ++k) {
        float q = mx_warp_sum(y0 * wq_s[1][k * MX_H + lane] + y1 * wq_s[1][k * MX_H + lane + 32]) + bq_s[1][k];
        if (a.qall1 && lane == 0) a.qall1[(size_t)m * A + k] = q;
        if (a.double_q) { if (k == greedy) tq_sel = q; }
        else if (k == 0 || q > tbest) { tbest = q; tq_sel = q; }                 // plain max, no avail mask (qmix.py:144)
      }
    }
    if (lane == 0) {
      if (a.greedy) a.greedy[m] = greedy;
      if (t < a.T) a.q_taken[((size_t)b * a.T + t) * N + n] = q_live_at_act;
      if (t >= 1) a.q_next[((size_t)b * a.T + (t - 1)) * N + n] = tq_sel;
    }
  }
}

// =====================================================================================================
// MLP variant (M_QMix, mqmix.py:101-176): Q values are columns [0, A) of the "gi" rows; one thread per (b, n):
// taken-action Q at step 0, greedy action of the LIVE net at step 1 under next_avail (first maximum), target Q there (double-Q),
// or the target net's own masked maximum.
// =====================================================================================================
__global__ void __launch_bounds__(256) k_mlp_qselect(MlpQSelArgs a) {
  const int total = a.B * a.N;
  MX_PDL_WAIT();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int n = i % a.N, b = i / a.N;
    const size_t m0 = ((size_t)b * 2) * a.N + n, m1 = m0 + a.N;
    const float* q0 = a.gi[0] + m0 * MX_G;
    const float* q1 = a.gi[0] + m1 * MX_G;
    const float* t1 = a.gi[1] + m1 * MX_G;
    const int act = a.act_idx[(size_t)b * a.ld_tn + n];
    int greedy = 0;
    float best = 0.f, tbest = 0.f;
    for (int k = 0; k < a.A; ++k) {
      const bool off = a.avail && a.avail[m1 * a.act_ld + k] == 0.f;
      const float qm = off ? -1e10f : q1[k];                                                // mqmix.py:147-149
      if (k == 0 || qm > best) { best = qm; greedy = k; }
      const float tm = off ? -1e10f : t1[k];               // not double-Q: target_policy.get_actions masks too (mqmix.py:155-160)
      if (k == 0 || tm > tbest) tbest = tm;
    }
    a.q_taken[i] = q0[act];
    a.q_next[i] = a.double_q ? t1[greedy] : tbest;
    if (a.greedy) { a.greedy[m0] = 0; a.greedy[m1] = greedy; }
    if (a.qall0)
      for (int k = 0; k < a.A; ++k) {
        a.qall0[m0 * a.A + k] = q0[k]; a.qall0[m1 * a.A + k] = q1[k];
        a.qall1[m0 * a.A + k] = a.gi[1][m0 * MX_G + k]; a.qall1[m1 * a.A + k] = t1[k];
      }
  }
}
int mx_launch_mlp_qselect(const MlpQSelArgs& a, cudaStream_t s) {
  int grid = mx_ceil_div(a.B * a.N, 256);
  if (grid > mx_num_sms() * 4) grid = mx_num_sms() * 4;
  return mx_launch("k_mlp_qselect", k_mlp_qselect, dim3(grid), dim3(256), 0, s, MX_STEP, a);
}

// =====================================================================================================
// --prev_act_inp: network input rows [obs | previous one-hot action]
// =====================================================================================================
__global__ void __launch_bounds__(256) k_pack_prev_act(const float* __restrict__ obs, int obs_ld, const float* __restrict__ acts, int act_ld,
                                                       float* __restrict__ X, int ldx, int B, int T, int N, int O, int A) {
  const long long total = (long long)B * (T + 1) * N * ldx;
  MX_PDL_WAIT();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % ldx);
    const long long m = i / ldx;
    const int n = (int)(m % N);
    const long long bt = m / N;
    const int t = (int)(bt % (T + 1));
    const long long b = bt / (T + 1);
    float v = 0.f;
    if (c < O) v = obs[m * obs_ld + c];
    else if (c < O + A && t > 0) v = acts[((b * T + (t - 1)) * N + n) * act_ld + (c - O)];     // zeros at t = 0 (qmix.py:122)
    X[i] = v;
  }
}

int mx_launch_pack_prev_act(const float* obs, int obs_ld, const float* acts, int act_ld, float* X, int ldx, int B, int T, int N, int O, int A,
                            cudaStream_t s) {
  const long long total = (long long)B * (T + 1) * N * ldx;
  int grid = (int)((total + 255) / 256);
  const int cap = mx_num_sms() * 8;
  if (grid > cap) grid = cap;
  return mx_launch("k_pack_prev_act", k_pack_prev_act, dim3(grid), dim3(256), 0, s, MX_STEP, obs, obs_ld, acts, act_ld, X, ldx, B, T, N, O, A);
}

// =====================================================================================================
// launchers
// =====================================================================================================
size_t mx_front_fwd_smem(int in_dim, int RM) {
  const int Ipad = mx_round_up(in_dim, 4);
  const int lda = mx_ld(Ipad > MX_H ? Ipad : MX_H);
  return (size_t)(16 * RM + 64) * lda * sizeof(float);
}

extern int g_mx_front_tc;
int mx_launch_front_fwd_tc(const FrontFwdArgs& a, int nets, cudaStream_t s);
bool mx_front_tc_usable(int in_dim, bool have_image);

int mx_launch_front_fwd(const FrontFwdArgs& a, int nets, cudaStream_t s) {
  if (mx_front_tc_usable(a.L.in_dim, a.tc_img[0] != nullptr) && (a.ldx & 3) == 0) return mx_launch_front_fwd_tc(a, nets, s);
  const int RM = 2;
  const int ntiles = mx_ceil_div(a.M, 16 * RM);
  int gx = mx_num_sms() / nets;
  if (gx < 1) gx = 1;
  if (gx > ntiles) gx = ntiles;
  const size_t smem = mx_front_fwd_smem(a.L.in_dim, RM);
  return mx_launch("k_front_fwd", k_front_fwd<RM>, dim3(gx, nets), dim3(MX_TILE_THREADS), smem, s, MX_STEP, a);
}

int mx_launch_gru_fwd(const GruFwdArgs& a, int nets, cudaStream_t s) {
  const int sms = mx_num_sms();
  int rpc = 1;     // one resident CTA per SM (the kernel is register heavy): grow rows-per-CTA until the grid fits one wave
  while (rpc < 4 && mx_ceil_div(a.R, rpc) * nets > 2 * sms) rpc *= 2;   // two CTAs fit per SM (<= 128 registers): co-resident CTAs hide each other's latencies
  // sequences: the 128-thread kernel, one row per CTA (r02 sweeps: 3m 174 vs 188 us, 2s3z 555 vs 619, 8m 1408 vs 1494).  The one-step
  // "branch" calls of R-MADDPG keep the multi-row CTAs: a CTA per row would spend its time loading W_hh
  if (a.T + 1 >= 8) return mx_launch("k_gru_fwd", k_gru_fwd2<1>, dim3(a.R, nets), dim3(GRU2_THREADS), 0, s, MX_STEP, a);
  auto kern = rpc == 1 ? k_gru_fwd<1> : rpc == 2 ? k_gru_fwd<2> : k_gru_fwd<4>;
  return mx_launch("k_gru_fwd", kern, dim3(mx_ceil_div(a.R, rpc), nets), dim3(GRU_THREADS), 0, s, MX_STEP, a);
}

int mx_launch_qhead(const QHeadArgs& a, cudaStream_t s) {
  if (a.A > 64) { mx_set_error("qhead: act_dim %d > 64 unsupported", a.A); return 1; }
  int grid = mx_ceil_div(a.M, 8);
  const int cap = mx_num_sms() * 4;
  if (grid > cap) grid = cap;
  return mx_launch("k_qhead", a.A > 32 ? k_qhead<2> : k_qhead<1>, dim3(grid), dim3(256), 0, s, MX_STEP, a);
}
