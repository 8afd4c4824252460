// Backward kernels of the recurrent agent network (BPTT through the GRU over the full episode).
//
//   k_qhead_bwd   d(q_taken) -> Linear head grads, post-GRU LayerNorm backward -> dL/dh_t (row-parallel)
//   k_gru_bwd     serial reverse recurrence: gate derivatives + dh_{t-1} = z*dh + W_hh^T dgh  (W_hh^T slices in registers)
//   k_front_bwd   time-batched: dW_ih/db_ih, dW_hh/db_hh, then back through LN2/fc2/LN1/fc1/LN0 with all
//                 weight gradients reduced per CTA into its gradient partial
//
// reference: autograd of nn.GRU / nn.LayerNorm / nn.Linear invoked by loss.backward() at qmix.py:191 for the
// module stack in algorithms/utils/{mlp,rnn,act}.py.  Gradients are numerators (see mixer.cu).
#include "mx_internal.h"
#include "mx_kernels.h"
#include "mx_tile.cuh"

// =====================================================================================================
// Q head backward (one warp per row-step)
// =====================================================================================================
// Shared memory: wq[A][64] | per-warp private accumulators dW[8][A][64], db[8][32 APL], dgamma[8][64], dbeta[8][64] (APL: 1 for
// A <= 32, 2 for A <= 64).  Only the owning warp touches its slice while rows are processed (no atomics); the CTA's partial is the
// sum over the 8 warps in fixed order, so the step is run-to-run deterministic.
static inline size_t qhead_bwd_smem(int A, int APL) { return (size_t)(A * MX_H * 9 + 8 * 32 * APL + 2 * 8 * MX_H + 2 * MX_H) * sizeof(float); }

template <int APL>
__global__ void __launch_bounds__(256) k_qhead_bwd(QHeadBwdArgs a) {
  constexpr int AR = 32 * APL;
  MX_DYN_SMEM(smem);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int A = a.A, AW = A * MX_H;
  float* wq_s = smem;
  float* dw_w = wq_s + AW;               // [8][A*64]
  float* db_w = dw_w + 8 * AW;           // [8][32 APL]
  float* dg_w = db_w + 8 * AR;           // [8][64]
  float* dbt_w = dg_w + 8 * MX_H;        // [8][64]
  float* lg_s = dbt_w + 8 * MX_H;
  float* lb_s = lg_s + MX_H;
  for (int i = tid; i < AW; i += blockDim.x) wq_s[i] = a.theta[a.wq + i];
  for (int i = tid; i < 8 * AW + 8 * AR; i += blockDim.x) dw_w[i] = 0.f;      // dw_w and db_w are contiguous
  for (int i = tid; i < MX_H; i += blockDim.x) { lg_s[i] = a.theta[a.lno_g + i]; lb_s[i] = a.theta[a.lno_b + i]; }
  MX_PDL_WAIT();
  __syncthreads();
  const int wglobal = blockIdx.x * (blockDim.x >> 5) + warp;
  const int wtotal = gridDim.x * (blockDim.x >> 5);
  const int T1 = a.T + 1, N = a.N;
  float dg0 = 0.f, dg1 = 0.f, db0 = 0.f, db1 = 0.f;
  float* my_dw = dw_w + warp * AW;
  for (int m = wglobal; m < a.M; m += wtotal) {
    const int n = m % N;
    const int bt = m / N;
    const int t = bt % T1, b = bt / T1;
    float* out = a.dh_out + (size_t)m * MX_H;
    if (t >= a.T) {                       // Q at the bootstrap step only feeds the (detached) target
      out[lane] = 0.f; out[lane + 32] = 0.f;
      continue;
    }
    const size_t e = (size_t)b * a.T + t;
    const int act = a.act_idx[(size_t)b * a.ld_tn + (size_t)t * N + n];
    const float dqv = a.dq_taken[e * N + n];
    const float* h = a.hall + (size_t)m * MX_H;
    const float mean = a.sto[2 * (size_t)m], rstd = a.sto[2 * (size_t)m + 1];
    const float xh0 = (h[lane] - mean) * rstd, xh1 = (h[lane + 32] - mean) * rstd;
    const float y0 = xh0 * lg_s[lane] + lb_s[lane], y1 = xh1 * lg_s[lane + 32] + lb_s[lane + 32];
    const float dy0 = dqv * wq_s[act * MX_H + lane], dy1 = dqv * wq_s[act * MX_H + lane + 32];
    my_dw[act * MX_H + lane] += dqv * y0;
    my_dw[act * MX_H + lane + 32] += dqv * y1;
    if (lane == 0) db_w[warp * AR + act] += dqv;
    dg0 += dy0 * xh0; dg1 += dy1 * xh1; db0 += dy0; db1 += dy1;
    // LayerNorm backward
    const float dx0 = dy0 * lg_s[lane], dx1 = dy1 * lg_s[lane + 32];
    const float c1 = mx_warp_sum(dx0 + dx1) * (1.f / MX_H);
    const float c2 = mx_warp_sum(dx0 * xh0 + dx1 * xh1) * (1.f / MX_H);
    out[lane] = rstd * (dx0 - c1 - xh0 * c2);
    out[lane + 32] = rstd * (dx1 - c1 - xh1 * c2);
  }
  dg_w[warp * MX_H + lane] = dg0; dg_w[warp * MX_H + lane + 32] = dg1;
  dbt_w[warp * MX_H + lane] = db0; dbt_w[warp * MX_H + lane + 32] = db1;
  __syncthreads();
  float* gp = a.gpart + (size_t)blockIdx.x * a.P;
  for (int i = tid; i < AW; i += blockDim.x) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) v += dw_w[w * AW + i];
    gp[a.wq + i] = v;
  }
  for (int i = tid; i < A; i += blockDim.x) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) v += db_w[w * AR + i];
    gp[a.bq + i] = v;
  }
  for (int i = tid; i < MX_H; i += blockDim.x) {
    float g = 0.f, bb = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) { g += dg_w[w * MX_H + i]; bb += dbt_w[w * MX_H + i]; }
    gp[a.lno_g + i] = g; gp[a.lno_b + i] = bb;
  }
}

// =====================================================================================================
// GRU backward through time
// =====================================================================================================
#define BWD_THREADS 256

template <int RPC>
__global__ void __launch_bounds__(BWD_THREADS, 1) k_gru_bwd(GruBwdArgs a) {
  // dh_{t-1}[k] = z*dh + sum_{j<192} W_hh[j][k] dgh[j].  Thread = 4*k + s owns column k restricted to the interleaved j-slice
  // {16m + 4s + c : m < 12, c < 4} (48 weights in registers, packed in pairs along j): 12 LDS.128 per step (the quad's four slices
  // are 64 contiguous bytes -> one wavefront per warp instruction), 24 packed FFMA2 in three 8-deep chains, then a two-level
  // xor-shuffle.  All four lanes of a quad carry dh[k] and do the (cheap) gate derivatives of unit k redundantly, so no lane
  // diverges; lane s publishes ONE of d(gh)_r / d(gh)_z / d(gh)_n into the buffer of this step's parity -> ONE barrier per step.
  // Operands of step t (r, z, n, hn, h_{t-1}, dL/dh_t) are streamed PF steps ahead by cp.async into a power-of-two ring.
  constexpr int RING = RPC <= 2 ? 8 : 4;
  constexpr int PF = RING - 2;
  __shared__ __align__(16) float ops_s[RING][RPC][6][MX_H];
  __shared__ __align__(16) float dgh_s[2][RPC][MX_G];
  const int tid = threadIdx.x;
  const int k = tid >> 2, s = tid & 3;
  const int row0 = blockIdx.x * RPC;
  float2 w[24];
#pragma unroll
  for (int m = 0; m < 12; ++m)
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const int j = 16 * m + 4 * s + 2 * c;
      w[2 * m + c] = make_float2(a.theta[a.whh + j * MX_H + k], a.theta[a.whh + (j + 1) * MX_H + k]);
    }
  const int T1 = a.T1 > 0 ? a.T1 : a.T + 1, N = a.N;
  MX_PDL_WAIT();        // W_hh columns above are parameter data; the operand streams below are the predecessor's outputs

  // prefetch assignment: RPC*96 16-byte pieces per step, up to two per thread; sources walk backwards in time
  constexpr int NPIECE = (RPC * 96 + BWD_THREADS - 1) / BWD_THREADS;
  const float* pf_src[NPIECE];      // source of the NEXT step to prefetch (h_{t-1} pieces: already one step earlier)
  size_t pf_stride[NPIECE];
  int pf_dst[NPIECE];               // float offset inside one ring slot, -1: no piece / row past R (slot stays zero)
  bool pf_hprev[NPIECE];
  const float* pf_h0[NPIECE];
  const int t_first = a.T - 1;
#pragma unroll
  for (int u = 0; u < NPIECE; ++u) {
    const int c = tid + u * BWD_THREADS;
    pf_dst[u] = -1; pf_src[u] = a.hall; pf_stride[u] = 0; pf_hprev[u] = false; pf_h0[u] = nullptr;
    if (c < RPC * 96) {
      const int r = c / 96, rem = c % 96, op = rem / 16, q4 = rem % 16;
      const int row = row0 + r;
      if (row < a.R) {
        pf_dst[u] = (r * 6 + op) * MX_H + 4 * q4;
        const size_t m0 = ((size_t)(row / N) * T1) * N + (row % N);
        const float* base;
        if (op < 3) { base = a.gates + m0 * MX_G + op * MX_H + 4 * q4; pf_stride[u] = (size_t)N * MX_G; }
        else if (op == 3) { base = a.hn + m0 * MX_H + 4 * q4; pf_stride[u] = (size_t)N * MX_H; }
        else if (op == 4) { base = a.hall + m0 * MX_H + 4 * q4; pf_stride[u] = (size_t)N * MX_H; pf_hprev[u] = true;
                            if (a.h0) pf_h0[u] = a.h0 + (size_t)row * MX_H + 4 * q4; }
        else { base = a.dh_out + m0 * MX_H + 4 * q4; pf_stride[u] = (size_t)N * MX_H; }
        pf_src[u] = base + (ptrdiff_t)(pf_hprev[u] ? t_first - 1 : t_first) * (ptrdiff_t)pf_stride[u];
      }
    }
  }
  auto prefetch = [&](int t) {        // called with t = T-1, T-2, ... in order
    if (t >= 0) {
#pragma unroll
      for (int u = 0; u < NPIECE; ++u) {
        if (pf_dst[u] >= 0) {
          float* dst = &ops_s[t & (RING - 1)][0][0][0] + pf_dst[u];
          const bool first = pf_hprev[u] && t == 0;             // h_{-1} = h0, or zeros (zero-fill form of the copy: no branch)
          mx_cp16z(dst, first ? (pf_h0[u] ? pf_h0[u] : a.hall) : pf_src[u], (first && !pf_h0[u]) ? 0 : 16);
          pf_src[u] -= pf_stride[u];
        }
      }
    }
    mx_cp_commit();
  };

  for (int idx = tid; idx < RING * RPC * 6 * MX_H; idx += BWD_THREADS) (&ops_s[0][0][0][0])[idx] = 0.f;     // rows past R stay zero
  // zero the rows of dgi that receive no gradient (t >= TB; for QMIX: the bootstrap step t == T)
  for (int tz = a.T; tz < T1; ++tz)
    for (int idx = tid; idx < RPC * MX_G; idx += BWD_THREADS) {
      const int r = idx / MX_G, c = idx % MX_G;
      const int row = row0 + r;
      if (row < a.R) {
        const size_t mm = (((size_t)(row / N) * T1) + tz) * N + (row % N);
        a.dgi[mm * MX_G + c] = 0.f;
      }
    }
  // lane s of a quad writes d(gi)_s of unit k (s = 0, 1, 2: r, z, n) and publishes d(gh)_s (lane 3 repeats lane 2's shared store)
  float* dgp[RPC];
  bool dg_on[RPC];
  float carry[RPC];
  const size_t dg_stride = (size_t)N * MX_G;
  const int sq = s < 3 ? s : 2;
#pragma unroll
  for (int r = 0; r < RPC; ++r) {
    const int row = row0 + r;
    const bool valid = row < a.R;
    const size_t m0 = valid ? ((size_t)(row / N) * T1) * N + (row % N) : 0;
    dgp[r] = a.dgi + (m0 + (size_t)t_first * N) * MX_G + sq * MX_H + k;
    dg_on[r] = valid && s < 3;
    carry[r] = 0.f;
  }
  __syncthreads();          // the zero fill precedes the first asynchronous copies into the ring
#pragma unroll
  for (int d = 0; d < PF; ++d) prefetch(t_first - d);
  mx_cp_wait<PF - 1>();
  __syncthreads();

  auto step = [&](const int t, const int cur) {
    prefetch(t - PF);                  // slot (t-PF) & (RING-1) == (t+2) & (RING-1): last read two barriers ago
    const float* os = &ops_s[t & (RING - 1)][0][0][0];
    float cz[RPC];
#pragma unroll
    for (int r = 0; r < RPC; ++r) {
      const float* o = os + r * 6 * MX_H;
      const float rg = o[k], zg = o[MX_H + k], ng = o[2 * MX_H + k], hn = o[3 * MX_H + k], hp = o[4 * MX_H + k];
      const float dh = o[5 * MX_H + k] + carry[r];
      const float d_n = dh * (1.f - zg) * (1.f - ng * ng);     // d pre-activation of n
      const float d_z = dh * (hp - ng) * zg * (1.f - zg);
      const float d_r = d_n * hn * rg * (1.f - rg);
      const float vg = s == 0 ? d_r : (s == 1 ? d_z : d_n);
      const float vs = s == 0 ? d_r : (s == 1 ? d_z : d_n * rg);                  // the n row reaches W_hn h + b_hn through r
      dgh_s[cur][r][sq * MX_H + k] = vs;
      if (dg_on[r]) *dgp[r] = vg;
      dgp[r] -= dg_stride;
      cz[r] = dh * zg;
    }
    mx_cp_wait<PF - 1>();       // operands of step t-1 have landed (the newer groups may still be in flight)
    __syncthreads();            // publishes dgh_s[cur] and the ring slot of step t-1
#pragma unroll
    for (int r = 0; r < RPC; ++r) {
      float2 p0 = make_float2(0.f, 0.f), p1 = p0, p2 = p0;
#pragma unroll
      for (int m = 0; m < 12; m += 3) {
        const float4 d0 = mx_ld4(&dgh_s[cur][r][16 * m + 4 * s]);
        const float4 d1 = mx_ld4(&dgh_s[cur][r][16 * (m + 1) + 4 * s]);
        const float4 d2 = mx_ld4(&dgh_s[cur][r][16 * (m + 2) + 4 * s]);
        p0 = mx_ffma2(w[2 * m], make_float2(d0.x, d0.y), p0); p0 = mx_ffma2(w[2 * m + 1], make_float2(d0.z, d0.w), p0);
        p1 = mx_ffma2(w[2 * m + 2], make_float2(d1.x, d1.y), p1); p1 = mx_ffma2(w[2 * m + 3], make_float2(d1.z, d1.w), p1);
        p2 = mx_ffma2(w[2 * m + 4], make_float2(d2.x, d2.y), p2); p2 = mx_ffma2(w[2 * m + 5], make_float2(d2.z, d2.w), p2);
      }
      p0 = mx_fadd2(mx_fadd2(p0, p1), p2);
      float p = p0.x + p0.y;
      p += __shfl_xor_sync(0xffffffffu, p, 1);
      p += __shfl_xor_sync(0xffffffffu, p, 2);
      carry[r] = cz[r] + p;     // dh_{t-1}[k] = z*dh + W_hh^T dgh
    }
    // the next step writes dgh_s[cur ^ 1]; readers of dgh_s[cur] are separated from its next writer by the next barrier
  };
  int t = t_first;
  for (; t >= 1; t -= 2) { step(t, 0); step(t - 1, 1); }
  if (t == 0) step(0, 0);
  mx_cp_wait<0>();
}

// ---- 128-thread variant (one row per CTA) -----------------------------------------------------------------------------------------------
// thread = 4*kp + s owns the column PAIR (2kp, 2kp+1) restricted to the interleaved j-slice {16m + 4s + c : m < 12, c < 4}: the 12
// LDS.128 of a step feed both columns, so the shared-memory traffic per row-step is half of k_gru_bwd's (the wide loads cost four
// LSU cycles each whatever the broadcast, and that pipe is what bounds the 256-thread kernel: 96 LDS.128 per row-step there, 48 here);
// 48 packed FFMA2 per thread in four 12-deep chains, two xor-shuffle levels for the two column sums.  Lanes s = 0, 1 (and their
// duplicates 2, 3) own unit 2kp + (s & 1) for the gate derivatives; the stores of a unit are split between the two duplicates.
#define BWD2_THREADS 128
// Only ROWS = 1 is launched (see k_gru_fwd2).
template <int ROWS>
__global__ void __launch_bounds__(BWD2_THREADS, 2) k_gru_bwd2(GruBwdArgs a) {
  constexpr int RING = 8, PF = 6;
  __shared__ __align__(16) float ops_s[RING][ROWS][6][MX_H];
  __shared__ __align__(16) float dgh_s[2][ROWS][MX_G];
  const int tid = threadIdx.x;
  const int kp = tid >> 2, s = tid & 3;
  float2 w0[24], w1[24];
#pragma unroll
  for (int m = 0; m < 12; ++m)
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const int j = 16 * m + 4 * s + 2 * c;
      w0[2 * m + c] = make_float2(a.theta[a.whh + j * MX_H + 2 * kp], a.theta[a.whh + (j + 1) * MX_H + 2 * kp]);
      w1[2 * m + c] = make_float2(a.theta[a.whh + j * MX_H + 2 * kp + 1], a.theta[a.whh + (j + 1) * MX_H + 2 * kp + 1]);
    }
  const int T1 = a.T1 > 0 ? a.T1 : a.T + 1, N = a.N;
  MX_PDL_WAIT();
  const int t_first = a.T - 1;
  // prefetch: 96 16-byte pieces per row-step, one per thread (threads < 96)
  const bool pf_on = tid < 96;
  const int op = pf_on ? tid / 16 : 0, q4 = tid % 16;
  const bool pf_hprev = op == 4;
  const size_t pf_stride = (size_t)N * (op < 3 ? MX_G : MX_H);
  const int ku = 2 * kp + (s & 1);          // unit of this lane; the lane and its duplicate (s ^ 2) split the unit's stores
  const int half = s >> 1;
  const size_t dg_stride = (size_t)N * MX_G;
  bool rok[ROWS];
  const float* pf_src[ROWS];
  const float* pf_h0[ROWS];
  float* dgp[ROWS];
  float carry[ROWS];
#pragma unroll
  for (int r = 0; r < ROWS; ++r) {
    const int row = blockIdx.x * ROWS + r;
    rok[r] = row < a.R;
    const int rr = rok[r] ? row : 0;
    const size_t m0 = ((size_t)(rr / N) * T1) * N + (rr % N);
    const float* base = op < 3 ? a.gates + m0 * MX_G + op * MX_H + 4 * q4 : (op == 3 ? a.hn : (op == 4 ? a.hall : a.dh_out)) + m0 * MX_H + 4 * q4;
    pf_src[r] = base + (ptrdiff_t)(pf_hprev ? t_first - 1 : t_first) * (ptrdiff_t)pf_stride;
    pf_h0[r] = (pf_hprev && a.h0) ? a.h0 + (size_t)rr * MX_H + 4 * q4 : nullptr;
    if (rok[r])
      for (int tz = a.T; tz < T1; ++tz)       // rows of dgi that receive no gradient (t >= TB; for QMIX: the bootstrap step t == T)
        for (int c = tid; c < MX_G; c += BWD2_THREADS) a.dgi[(m0 + (size_t)tz * N) * MX_G + c] = 0.f;
    dgp[r] = a.dgi + (m0 + (size_t)t_first * N) * MX_G + ku;
    carry[r] = 0.f;
  }
  float* pf_dst = &ops_s[0][0][op][4 * q4];
  auto prefetch = [&](int t) {        // called with t = T-1, T-2, ... in order
    if (t >= 0 && pf_on) {
      const bool first = pf_hprev && t == 0;             // h_{-1} = h0, or zeros (zero-fill form of the copy: no branch)
#pragma unroll
      for (int r = 0; r < ROWS; ++r) {
        if (rok[r]) mx_cp16z(pf_dst + ((t & (RING - 1)) * ROWS + r) * (6 * MX_H), first ? (pf_h0[r] ? pf_h0[r] : a.hall) : pf_src[r], (first && !pf_h0[r]) ? 0 : 16);
        pf_src[r] -= pf_stride;
      }
    }
    mx_cp_commit();
  };
  if (ROWS > 1) {      // a row slot without a row (odd R): its operands stay zero, nothing of it is stored
    for (int idx = tid; idx < RING * ROWS * 6 * MX_H; idx += BWD2_THREADS) (&ops_s[0][0][0][0])[idx] = 0.f;
    __syncthreads();
  }
#pragma unroll
  for (int d = 0; d < PF; ++d) prefetch(t_first - d);
  mx_cp_wait<PF - 1>();
  __syncthreads();

  auto step = [&](const int t, const int cur) {
    prefetch(t - PF);
    float cz[ROWS];
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
      const float* o = &ops_s[t & (RING - 1)][r][0][0];
      const float rg = o[ku], zg = o[MX_H + ku], ng = o[2 * MX_H + ku], hn = o[3 * MX_H + ku], hp = o[4 * MX_H + ku];
      const float dh = o[5 * MX_H + ku] + carry[r];
      const float d_n = dh * (1.f - zg) * (1.f - ng * ng);
      const float d_z = dh * (hp - ng) * zg * (1.f - zg);
      const float d_r = d_n * hn * rg * (1.f - rg);
      // half 0: r (and z); half 1: n
      dgh_s[cur][r][(half ? 2 * MX_H : 0) + ku] = half ? d_n * rg : d_r;
      if (!half) dgh_s[cur][r][MX_H + ku] = d_z;
      if (rok[r]) {
        dgp[r][half ? 2 * MX_H : 0] = half ? d_n : d_r;
        if (!half) dgp[r][MX_H] = d_z;
      }
      dgp[r] -= dg_stride;
      cz[r] = dh * zg;
    }
    mx_cp_wait<PF - 1>();
    __syncthreads();
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
      float2 a0 = make_float2(0.f, 0.f), a1 = a0, b0 = a0, b1 = a0;
#pragma unroll
      for (int m = 0; m < 12; ++m) {
        const float4 d = mx_ld4(&dgh_s[cur][r][16 * m + 4 * s]);
        const float2 lo = make_float2(d.x, d.y), hi = make_float2(d.z, d.w);
        a0 = mx_ffma2(w0[2 * m], lo, a0); b0 = mx_ffma2(w1[2 * m], lo, b0);
        a1 = mx_ffma2(w0[2 * m + 1], hi, a1); b1 = mx_ffma2(w1[2 * m + 1], hi, b1);
      }
      a0 = mx_fadd2(a0, a1); b0 = mx_fadd2(b0, b1);
      float p0 = a0.x + a0.y, p1 = b0.x + b0.y;
      p0 += __shfl_xor_sync(0xffffffffu, p0, 1); p1 += __shfl_xor_sync(0xffffffffu, p1, 1);
      p0 += __shfl_xor_sync(0xffffffffu, p0, 2); p1 += __shfl_xor_sync(0xffffffffu, p1, 2);
      carry[r] = cz[r] + ((s & 1) ? p1 : p0);     // dh_{t-1}[ku] = z*dh + W_hh^T dgh
    }
  };
  int t = t_first;
  for (; t >= 1; t -= 2) { step(t, 0); step(t - 1, 1); }
  if (t == 0) step(0, 0);
  mx_cp_wait<0>();
}

// =====================================================================================================
// front backward (time-batched)
// =====================================================================================================
struct FrontBwdSmem {
  int ldi, ld64, ldg;
  int o_dgi, o_dgn, o_x, o_hp, o_u, o_da, o_x0, o_xh0, o_dx0, o_wc, o_col, o_stat, o_lnp, total;
};
static FrontBwdSmem front_bwd_smem(int in_dim, int TM, bool gru_ext = false) {     // gru_ext: k_gru_wgrad owns dW_ih / dW_hh (no h_{t-1}, dgi_n * r tiles here)
  FrontBwdSmem s;
  const int I64 = mx_round_up(in_dim, 64);
  s.ldi = mx_ld(I64); s.ld64 = mx_ld(64); s.ldg = mx_ld(MX_G);
  int o = 0;
  s.o_dgi = o; o += TM * s.ldg;     // dgi tile (r,z,n)
  s.o_dgn = o; o += gru_ext ? 0 : TM * s.ld64;    // dgi_n * r  (gradient reaching W_hn h)
  s.o_x = o; o += TM * s.ld64;      // r gate (staging), then x2, later x1
  s.o_hp = o; o += gru_ext ? 0 : TM * s.ld64;     // h_{t-1}
  s.o_u = o; o += TM * s.ld64;      // u2, later u1 (post-ReLU, pre-LN)
  s.o_da = o; o += TM * s.ld64;     // gradient w.r.t. the Linear output (after ReLU mask)
  s.o_x0 = o; o += TM * s.ldi;      // raw input rows, then LN0 output (fc1 input)
  s.o_xh0 = o; o += TM * s.ldi;     // normalised input before the affine
  s.o_dx0 = o; o += TM * s.ldi;     // gradient w.r.t. the LN0 output (only when the input gradient is requested)
  s.o_wc = o; o += 64 * s.ld64;
  s.o_col = o; o += 2 * I64 + 4 * 64;   // column accumulators for LayerNorm gains/biases
  s.o_stat = o; o += 3 * TM * 2;        // (mean, rstd) of LN0 / LN1 / LN2 for the tile rows
  s.o_lnp = o; o += 4 * 64;             // ln1_g, ln1_b, ln2_g, ln2_b
  s.total = o;
  return s;
}

// LayerNorm backward on a 64-wide row spread over a half-warp; v = upstream grad w.r.t. LN output (cols 4tx+j),
// u = LN input.  Returns grad w.r.t. LN input, masked by ReLU (u > 0); dgamma/dbeta partials accumulate in registers.
template <int RM>
MX_DEVINL void ln64_bwd_relu(bool act_tanh, float (&v)[RM][4], const float* u_s, int ld, const float* stat /*[TM][2]*/, const float* gamma_s,
                             float (&dg)[4], float (&db)[4]) {
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
#pragma unroll
  for (int i = 0; i < RM; ++i) {
    const int r = ty * RM + i;
    const float mean = stat[2 * r], rstd = stat[2 * r + 1];
    const float4 u4 = mx_ld4(u_s + r * ld + 4 * tx);
    const float uu[4] = {u4.x, u4.y, u4.z, u4.w};
    float xh[4], dx[4], s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      xh[j] = (uu[j] - mean) * rstd;
      dg[j] = fmaf(v[i][j], xh[j], dg[j]);
      db[j] += v[i][j];
      dx[j] = v[i][j] * gamma_s[4 * tx + j];
      s1 += dx[j]; s2 += dx[j] * xh[j];
    }
    s1 = mx_row16_sum(s1) * (1.f / 64.f);
    s2 = mx_row16_sum(s2) * (1.f / 64.f);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float du = rstd * (dx[j] - s1 - xh[j] * s2);
      v[i][j] = act_tanh ? du * (1.f - uu[j] * uu[j]) : (uu[j] > 0.f ? du : 0.f);
    }
  }
}

template <int RM>
__global__ void __launch_bounds__(MX_TILE_THREADS) k_front_bwd(FrontBwdArgs a, FrontBwdSmem sm) {
  constexpr int TM = 16 * RM;
  MX_DYN_SMEM(smem);
  const MxNetLayout L = a.L;
  const float* __restrict__ th = a.theta;
  const int I = L.in_dim, I64 = mx_round_up(I, 64);
  float* dgi_s = smem + sm.o_dgi; float* dgn_s = smem + sm.o_dgn; float* x_s = smem + sm.o_x; float* hp_s = smem + sm.o_hp;
  float* u_s = smem + sm.o_u; float* da_s = smem + sm.o_da; float* x0_s = smem + sm.o_x0; float* xh0_s = smem + sm.o_xh0;
  float* Wc = smem + sm.o_wc;
  float* col0g = smem + sm.o_col; float* col0b = col0g + I64;          // LN0 gain / bias grads   [I64] each
  float* col1g = col0b + I64; float* col1b = col1g + 64;               // LN1
  float* col2g = col1b + 64; float* col2b = col2g + 64;                // LN2
  float* st0_s = smem + sm.o_stat; float* st1_s = st0_s + 2 * TM; float* st2_s = st1_s + 2 * TM;
  float* ln1g_s = smem + sm.o_lnp; float* ln1b_s = ln1g_s + 64; float* ln2g_s = ln1b_s + 64; float* ln2b_s = ln2g_s + 64;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int ntiles = (a.M + TM - 1) / TM;
  const int T1 = a.T1 > 0 ? a.T1 : a.T + 1, N = a.N;
  const bool ldx_vec = (a.ldx & 3) == 0;
  const bool wg = !a.skip_wgrad;
  const bool wgemm = wg && !a.wgrad_external;      // the weight-gradient GEMMs and bias column sums run here (else: k_wgrad_tc)
  const bool gru_here = !a.gru_wgrad_ext;          // else k_gru_wgrad (beside this kernel) produces dW_ih / dW_hh / db_ih / db_hh
  float* dx0_s = smem + sm.o_dx0;
  float* gp = a.gpart + (size_t)blockIdx.x * a.P;
  for (int i = tid; i < 2 * I64 + 4 * 64; i += MX_TILE_THREADS) col0g[i] = 0.f;
  if (tid < 64) { ln1g_s[tid] = th[L.ln1_g + tid]; ln1b_s[tid] = th[L.ln1_b + tid]; ln2g_s[tid] = th[L.ln2_g + tid]; ln2b_s[tid] = th[L.ln2_b + tid]; }
  float dg1[4] = {0.f, 0.f, 0.f, 0.f}, db1[4] = {0.f, 0.f, 0.f, 0.f}, dg2[4] = {0.f, 0.f, 0.f, 0.f}, db2[4] = {0.f, 0.f, 0.f, 0.f};
  int iter = 0;
  MX_PDL_WAIT();
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++iter) {
    const int m0 = tile * TM;
    const bool accum = iter > 0;
    __syncthreads();
    // ---- stage the tile's raw operands with cp.async: dgi, r gate, u2, u1?, h_{t-1}, the input rows, LN statistics ----
    mx_stage_rows(dgi_s, sm.ldg, a.dgi, MX_G, m0, a.M, TM, MX_G);
    if (!gru_here) {}
    else if (!a.no_gru) mx_stage_rows(x_s, sm.ld64, a.gates, MX_G, m0, a.M, TM, MX_H);          // r gate = first 64 columns of the gates row
    else for (int i = tid; i < TM * sm.ld64; i += MX_TILE_THREADS) x_s[i] = 0.f;
    mx_stage_rows(u_s, sm.ld64, a.u2, MX_H, m0, a.M, TM, MX_H);
    for (int r = tid >> 4; gru_here && r < TM; r += MX_TILE_THREADS / 16) {
      const int m = m0 + r;
      const bool has = !a.no_gru && m < a.M && ((m / N) % T1) > 0;
      float* d = hp_s + r * sm.ld64 + 4 * tx;
      if (has) mx_cp16(d, a.hall + (size_t)(m - N) * MX_H + 4 * tx);
      else if (m < a.M && a.h0) mx_cp16(d, a.h0 + (size_t)m * MX_H + 4 * tx);
      else mx_st4(d, make_float4(0.f, 0.f, 0.f, 0.f));
    }
    if (ldx_vec) mx_stage_rows(x0_s, sm.ldi, a.X, a.ldx, m0, a.M, TM, mx_round_up(I, 4));
    mx_cp_commit();
    for (int i = tid; i < 3 * TM * 2; i += MX_TILE_THREADS) {
      const int which = i / (2 * TM), rr = (i % (2 * TM)) >> 1, comp = i & 1;
      const int m = m0 + rr;
      const float* src = which == 0 ? a.st0 : (which == 1 ? a.st1 : a.st2);
      st0_s[i] = (m < a.M && (which > 0 || a.feature_norm)) ? src[2 * (size_t)m + comp] : 0.f;
    }
    mx_cp_wait<0>();
    __syncthreads();
    for (int idx = tid; gru_here && idx < TM * MX_H; idx += MX_TILE_THREADS) {
      const int r = idx >> 6, c = idx & 63;
      const int o = r * sm.ld64 + c;
      dgn_s[o] = dgi_s[r * sm.ldg + 2 * MX_H + c] * x_s[o];                                // dgi_n * r
      x_s[o] = (m0 + r < a.M) ? (u_s[o] - st2_s[2 * r]) * st2_s[2 * r + 1] * ln2g_s[c] + ln2b_s[c] : 0.f;   // x2 = LN2(u2)
    }
    __syncthreads();
    // ---- GRU weight gradients: dW_ih = dgi^T x2 ; dW_hh = [dgi_r, dgi_z, dgi_n*r]^T h_{t-1} ----
    if (wgemm && gru_here) {
      for (int nb = 0; nb < 3; ++nb) {
        mx_wgrad_block(dgi_s + nb * 64, sm.ldg, x_s, sm.ld64, TM, gp + L.wih, MX_G, MX_H, nb * 64, 0, accum);
        if (a.no_gru) continue;
        const float* dgh = nb < 2 ? dgi_s + nb * 64 : dgn_s;
        const int ldd = nb < 2 ? sm.ldg : sm.ld64;
        mx_wgrad_block(dgh, ldd, hp_s, sm.ld64, TM, gp + L.whh + nb * 64 * MX_H, 64, MX_H, 0, 0, accum);
      }
      mx_colsum(dgi_s, sm.ldg, TM, MX_G, gp + L.bih, accum);
      if (!a.no_gru) {
        mx_colsum(dgi_s, sm.ldg, TM, 2 * MX_H, gp + L.bhh, accum);
        mx_colsum(dgn_s, sm.ld64, TM, MX_H, gp + L.bhh + 2 * MX_H, accum);
      }
    }
    // ---- dx2 = dgi . W_ih  (three 64-row chunks) ----
    float v[RM][4];
#pragma unroll
    for (int i = 0; i < RM; ++i)
#pragma unroll
      for (int jx = 0; jx < 4; ++jx) v[i][jx] = 0.f;
    for (int nc = 0; nc < 3; ++nc) {
      __syncthreads();
      mx_stage_weight(Wc, sm.ld64, th + L.wih, MX_G, MX_H, MX_H, nc * 64, 0, 64);
      __syncthreads();
      mx_mm_nn<RM>(dgi_s + nc * 64, sm.ldg, Wc, sm.ld64, v);
    }
    // ---- LN2 backward + ReLU mask -> da2 ----
    ln64_bwd_relu<RM>(a.act_tanh != 0, v, u_s, sm.ld64, st2_s, ln2g_s, dg2, db2);
    __syncthreads();     // x_s (x2), u_s (u2) no longer needed by anyone
#pragma unroll
    for (int i = 0; i < RM; ++i) mx_st4(da_s + (ty * RM + i) * sm.ld64 + 4 * tx, make_float4(v[i][0], v[i][1], v[i][2], v[i][3]));
    if (a.wgrad_external) {
#pragma unroll
      for (int i = 0; i < RM; ++i) {
        const int m = m0 + ty * RM + i;
        if (m < a.M) mx_st4(a.da2_out + (size_t)m * MX_H + 4 * tx, make_float4(v[i][0], v[i][1], v[i][2], v[i][3]));
      }
    }
    mx_stage_rows(u_s, sm.ld64, a.u1, MX_H, m0, a.M, TM, MX_H);
    mx_cp_commit();
    mx_cp_wait<0>();
    __syncthreads();
    for (int idx = tid; idx < TM * MX_H; idx += MX_TILE_THREADS) {
      const int r = idx >> 6, c = idx & 63;
      const int o = r * sm.ld64 + c;
      x_s[o] = (m0 + r < a.M) ? (u_s[o] - st1_s[2 * r]) * st1_s[2 * r + 1] * ln1g_s[c] + ln1b_s[c] : 0.f;   // x1 = LN1(u1)
    }
    __syncthreads();
    // ---- fc2: dW2 = da2^T x1, db2 ; dx1 = da2 . W2 ----
    if (wgemm) {
      mx_wgrad_block(da_s, sm.ld64, x_s, sm.ld64, TM, gp + L.w2, MX_H, MX_H, 0, 0, accum);
      mx_colsum(da_s, sm.ld64, TM, MX_H, gp + L.b2, accum);
    }
    mx_stage_weight(Wc, sm.ld64, th + L.w2, MX_H, MX_H, MX_H, 0, 0, 64);
    __syncthreads();      // W2 staged; every warp is past the fc2 weight gradient that read x_s (x1)
#pragma unroll
    for (int i = 0; i < RM; ++i)
#pragma unroll
      for (int jx = 0; jx < 4; ++jx) v[i][jx] = 0.f;
    mx_mm_nn<RM>(da_s, sm.ld64, Wc, sm.ld64, v);
    ln64_bwd_relu<RM>(a.act_tanh != 0, v, u_s, sm.ld64, st1_s, ln1g_s, dg1, db1);
    __syncthreads();     // da_s (da2) consumed by everyone
#pragma unroll
    for (int i = 0; i < RM; ++i) mx_st4(da_s + (ty * RM + i) * sm.ld64 + 4 * tx, make_float4(v[i][0], v[i][1], v[i][2], v[i][3]));
    if (a.wgrad_external) {
#pragma unroll
      for (int i = 0; i < RM; ++i) {
        const int m = m0 + ty * RM + i;
        if (m < a.M) mx_st4(a.da1_out + (size_t)m * MX_H + 4 * tx, make_float4(v[i][0], v[i][1], v[i][2], v[i][3]));
      }
    }
    // x0 = LN0(x) and the normalised input, in place over the staged raw rows
    for (int idx = tid; idx < TM * I64; idx += MX_TILE_THREADS) {
      const int r = idx / I64, c = idx - r * I64, m = m0 + r;
      float xh = 0.f, x0 = 0.f;
      if (m < a.M && c < I) {
        const float x = ldx_vec ? x0_s[r * sm.ldi + c] : a.X[(size_t)m * a.ldx + c];
        if (a.feature_norm) {
          xh = (x - st0_s[2 * r]) * st0_s[2 * r + 1];
          x0 = xh * th[L.fn_g + c] + th[L.fn_b + c];
        } else x0 = x;
      }
      x0_s[r * sm.ldi + c] = x0; xh0_s[r * sm.ldi + c] = xh;
    }
    __syncthreads();
    // ---- fc1: dW1 = da1^T x0, db1 ; dx0 = da1 . W1 (only for the LN0 gain/bias) ----
    if (wgemm) {
      for (int kb = 0; kb * 64 < I; ++kb) {
        mx_wgrad_block(da_s, sm.ld64, x0_s + kb * 64, sm.ldi, TM, gp + L.w1, MX_H, I, 0, kb * 64, accum);
      }
      mx_colsum(da_s, sm.ld64, TM, MX_H, gp + L.b1, accum);
    }
    if (a.feature_norm || a.dX) {
      for (int kb = 0; kb * 64 < I; ++kb) {
        __syncthreads();
        mx_stage_weight(Wc, sm.ld64, th + L.w1, MX_H, I, I, 0, kb * 64, 64);
        __syncthreads();
#pragma unroll
        for (int i = 0; i < RM; ++i)
#pragma unroll
          for (int jx = 0; jx < 4; ++jx) v[i][jx] = 0.f;
        mx_mm_nn<RM>(da_s, sm.ld64, Wc, sm.ld64, v);
        float cg[4] = {0.f, 0.f, 0.f, 0.f}, cb[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int jx = 0; jx < 4; ++jx) {
          const int c = kb * 64 + 4 * tx + jx;
          if (c < I) {
            float sg = 0.f, sb = 0.f;
#pragma unroll
            for (int i = 0; i < RM; ++i) {
              sg = fmaf(v[i][jx], xh0_s[(ty * RM + i) * sm.ldi + c], sg); sb += v[i][jx];
              if (a.dX) dx0_s[(ty * RM + i) * sm.ldi + c] = v[i][jx];
            }
            cg[jx] = sg; cb[jx] = sb;
          }
        }
        if (wg && a.feature_norm) {       // the 16 row groups add their column partials one after the other (deterministic)
          for (int g = 0; g < MX_TILE_THREADS / 16; ++g) {
            if (ty == g) {
#pragma unroll
              for (int jx = 0; jx < 4; ++jx) {
                const int c = kb * 64 + 4 * tx + jx;
                if (c < I) { col0g[c] += cg[jx]; col0b[c] += cb[jx]; }
              }
            }
            __syncthreads();
          }
        }
      }
      if (a.dX) {
        // gradient w.r.t. the raw input rows: backward of the feature LayerNorm (warp per row)
        __syncthreads();
        const int lane = tid & 31, warp = tid >> 5;
        for (int r = warp; r < TM; r += MX_TILE_THREADS / 32) {
          const int m = m0 + r;
          if (m >= a.M) continue;
          float s1 = 0.f, s2 = 0.f;
          for (int c = lane; c < I; c += 32) {
            const float dxh = dx0_s[r * sm.ldi + c] * (a.feature_norm ? th[L.fn_g + c] : 1.f);
            s1 += dxh; s2 += dxh * xh0_s[r * sm.ldi + c];
          }
          s1 = mx_warp_sum(s1) / (float)I; s2 = mx_warp_sum(s2) / (float)I;
          const float rstd = st0_s[2 * r + 1];
          for (int c = lane; c < I; c += 32) {
            const float d0 = dx0_s[r * sm.ldi + c];
            a.dX[(size_t)m * a.ldx + c] = a.feature_norm ? rstd * (d0 * th[L.fn_g + c] - s1 - xh0_s[r * sm.ldi + c] * s2) : d0;
          }
        }
      }
    }
  }
  // ---- LayerNorm gain / bias gradients: per-thread partials -> per-CTA column sums -> this CTA's gradient partial ----
  for (int g = 0; g < MX_TILE_THREADS / 16; ++g) {       // row groups in turn: fixed summation order, no shared atomics
    if (ty == g) {
#pragma unroll
      for (int jx = 0; jx < 4; ++jx) {
        const int c = 4 * tx + jx;
        col1g[c] += dg1[jx]; col1b[c] += db1[jx];
        col2g[c] += dg2[jx]; col2b[c] += db2[jx];
      }
    }
    __syncthreads();
  }
  if (wg) {
    for (int c = tid; c < MX_H; c += MX_TILE_THREADS) {
      gp[L.ln2_g + c] = col2g[c]; gp[L.ln2_b + c] = col2b[c];
      gp[L.ln1_g + c] = col1g[c]; gp[L.ln1_b + c] = col1b[c];
    }
    for (int c = tid; c < I; c += MX_TILE_THREADS) { gp[L.fn_g + c] = col0g[c]; gp[L.fn_b + c] = col0b[c]; }
  }
}


// =====================================================================================================
// k_gru_wgrad: the GRU weight gradients of the time-batched backward as their own kernel,
//   dW_ih = dgi^T x2, db_ih ;  dW_hh = [dgi_r, dgi_z, dgi_n * r]^T h_{t-1}, db_hh
// They depend only on what k_gru_bwd left (dgi) and on saved forward rows, not on k_front_bwd's data-gradient chain, so the QMIX
// step launches this on the forked branch BESIDE k_front_bwd: same tiles, same grid, CTA b of both kernels
// fills disjoint columns of gradient partial b; the two CTAs fit one SM together (shared memory ~77 + ~134 KB at 3m).
// 256 threads at <= 128 registers so that a CTA of each kernel is resident together.  Two passes per tile (W_ih, then W_hh); thread
// (tn, tk) owns rows {64 g + 2 tn, + 1 : g = 0..2} x columns 8 tk .. + 7 of the pass's matrix: per tile row 3 LDS.64 + 2 LDS.128 feed
// 24 FFMA2 (pairs along the gate-row dimension, the x / h value duplicated).
// =====================================================================================================
struct GruWgradSmem { int ld64, ldg, o_dgi, o_dgn, o_x, o_hp, o_stat, o_lnp, total; };
static GruWgradSmem gru_wgrad_smem(int TM) {
  GruWgradSmem s;
  s.ld64 = mx_ld(64); s.ldg = mx_ld(MX_G);
  int o = 0;
  s.o_dgi = o; o += TM * s.ldg;
  s.o_dgn = o; o += TM * s.ld64;     // r gate, then dgi_n * r in place
  s.o_x = o; o += TM * s.ld64;       // u2, then x2 = LN2(u2) in place
  s.o_hp = o; o += TM * s.ld64;      // h_{t-1}
  s.o_stat = o; o += 2 * TM;
  s.o_lnp = o; o += 2 * 64;
  s.total = o;
  return s;
}

template <int RM>
__global__ void __launch_bounds__(MX_TILE_THREADS, 2) k_gru_wgrad(FrontBwdArgs a, GruWgradSmem sm) {
  constexpr int TM = 16 * RM;
  MX_DYN_SMEM(smem);
  const MxNetLayout L = a.L;
  const float* __restrict__ th = a.theta;
  float* dgi_s = smem + sm.o_dgi; float* dgn_s = smem + sm.o_dgn; float* x_s = smem + sm.o_x; float* hp_s = smem + sm.o_hp;
  float* st2_s = smem + sm.o_stat; float* ln2g_s = smem + sm.o_lnp; float* ln2b_s = ln2g_s + 64;
  const int tid = threadIdx.x, tx = tid & 15;
  const int tk = tid & 7, tn = tid >> 3;
  const int ntiles = (a.M + TM - 1) / TM;
  const int T1 = a.T1 > 0 ? a.T1 : a.T + 1, N = a.N;
  float* gp = a.gpart + (size_t)blockIdx.x * a.P;
  if (tid < 64) { ln2g_s[tid] = th[L.ln2_g + tid]; ln2b_s[tid] = th[L.ln2_b + tid]; }
  int iter = 0;
  MX_PDL_WAIT();
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++iter) {
    const int m0 = tile * TM;
    __syncthreads();
    mx_stage_rows(dgi_s, sm.ldg, a.dgi, MX_G, m0, a.M, TM, MX_G);
    mx_stage_rows(dgn_s, sm.ld64, a.gates, MX_G, m0, a.M, TM, MX_H);          // r gate = first 64 columns of the gates row
    mx_stage_rows(x_s, sm.ld64, a.u2, MX_H, m0, a.M, TM, MX_H);
    for (int r = tid >> 4; r < TM; r += MX_TILE_THREADS / 16) {
      const int m = m0 + r;
      const bool has = m < a.M && ((m / N) % T1) > 0;
      float* d = hp_s + r * sm.ld64 + 4 * tx;
      if (has) mx_cp16(d, a.hall + (size_t)(m - N) * MX_H + 4 * tx);
      else if (m < a.M && a.h0) mx_cp16(d, a.h0 + (size_t)m * MX_H + 4 * tx);
      else mx_st4(d, make_float4(0.f, 0.f, 0.f, 0.f));
    }
    mx_cp_commit();
    for (int i = tid; i < 2 * TM; i += MX_TILE_THREADS) {
      const int m = m0 + (i >> 1);
      st2_s[i] = m < a.M ? a.st2[2 * (size_t)m + (i & 1)] : 0.f;
    }
    mx_cp_wait<0>();
    __syncthreads();
    for (int idx = tid; idx < TM * MX_H; idx += MX_TILE_THREADS) {
      const int r = idx >> 6, c = idx & 63;
      const int o = r * sm.ld64 + c;
      dgn_s[o] = dgi_s[r * sm.ldg + 2 * MX_H + c] * dgn_s[o];                              // dgi_n * r
      x_s[o] = (m0 + r < a.M) ? (x_s[o] - st2_s[2 * r]) * st2_s[2 * r + 1] * ln2g_s[c] + ln2b_s[c] : 0.f;   // x2 = LN2(u2)
    }
    __syncthreads();
    const bool accum = iter > 0;
#pragma unroll 1
    for (int pass = 0; pass < 2; ++pass) {
      const float* X_s = pass ? hp_s : x_s;
      const float* D2_s = pass ? dgn_s + 2 * tn : dgi_s + 2 * MX_H + 2 * tn;      // the n-gate rows: dgi_n for W_in, dgi_n * r for W_hn
      const int ld2 = pass ? sm.ld64 : sm.ldg;
      float2 acc[3][8];
#pragma unroll
      for (int g = 0; g < 3; ++g)
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[g][k] = make_float2(0.f, 0.f);
#pragma unroll 2
      for (int r = 0; r < TM; ++r) {
        const float4 x0 = mx_ld4(X_s + r * sm.ld64 + 8 * tk), x1 = mx_ld4(X_s + r * sm.ld64 + 8 * tk + 4);
        const float xs[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
        const float2 d0 = *reinterpret_cast<const float2*>(dgi_s + r * sm.ldg + 2 * tn);
        const float2 d1 = *reinterpret_cast<const float2*>(dgi_s + r * sm.ldg + MX_H + 2 * tn);
        const float2 d2 = *reinterpret_cast<const float2*>(D2_s + r * ld2);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float2 xx = make_float2(xs[k], xs[k]);
          acc[0][k] = mx_ffma2(d0, xx, acc[0][k]);
          acc[1][k] = mx_ffma2(d1, xx, acc[1][k]);
          acc[2][k] = mx_ffma2(d2, xx, acc[2][k]);
        }
      }
      float* W = gp + (pass ? L.whh : L.wih);
#pragma unroll
      for (int g = 0; g < 3; ++g)
#pragma unroll
        for (int h = 0; h < 2; ++h) {          // the two rows of the pair
          float* w = W + (size_t)(64 * g + 2 * tn + h) * MX_H + 8 * tk;
          float4 lo = make_float4(h ? acc[g][0].y : acc[g][0].x, h ? acc[g][1].y : acc[g][1].x, h ? acc[g][2].y : acc[g][2].x, h ? acc[g][3].y : acc[g][3].x);
          float4 hi = make_float4(h ? acc[g][4].y : acc[g][4].x, h ? acc[g][5].y : acc[g][5].x, h ? acc[g][6].y : acc[g][6].x, h ? acc[g][7].y : acc[g][7].x);
          if (accum) {
            const float4 p0 = mx_ld4(w), p1 = mx_ld4(w + 4);
            lo.x += p0.x; lo.y += p0.y; lo.z += p0.z; lo.w += p0.w; hi.x += p1.x; hi.y += p1.y; hi.z += p1.z; hi.w += p1.w;
          }
          mx_st4(w, lo); mx_st4(w + 4, hi);
        }
    }
    mx_colsum(dgi_s, sm.ldg, TM, MX_G, gp + L.bih, accum);
    mx_colsum(dgi_s, sm.ldg, TM, 2 * MX_H, gp + L.bhh, accum);
    mx_colsum(dgn_s, sm.ld64, TM, MX_H, gp + L.bhh + 2 * MX_H, accum);
  }
}

// =====================================================================================================
// launchers
// =====================================================================================================
int mx_launch_qhead_bwd(const QHeadBwdArgs& a, int* nparts_used, cudaStream_t s) {
  if (a.A > 64) { mx_set_error("qhead_bwd: act_dim %d > 64 unsupported", a.A); return 1; }
  int grid = mx_ceil_div(a.M, 8 * 4);   // ~4 rows per warp
  const int cap = mx_num_sms();
  if (grid > cap) grid = cap;
  if (grid < 1) grid = 1;
  const int apl = a.A > 32 ? 2 : 1;
  *nparts_used = grid;
  return mx_launch("k_qhead_bwd", apl == 2 ? k_qhead_bwd<2> : k_qhead_bwd<1>, dim3(grid), dim3(256), qhead_bwd_smem(a.A, apl), s, MX_STEP, a);
}

// MLP variant: gradient w.r.t. the "gi" rows = the Q-head outputs: only the taken action of the step-0 rows receives dL/dq
__global__ void __launch_bounds__(256) k_mlp_dgi(const float* __restrict__ dq_taken, const int32_t* __restrict__ act_idx, int ld_tn,
                                                 float* __restrict__ dgi, int B, int N) {
  const long long total = (long long)B * 2 * N * MX_G;
  MX_PDL_WAIT();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % MX_G);
    const long long m = i / MX_G;
    const int n = (int)(m % N);
    const long long bt = m / N;
    const int t = (int)(bt & 1);
    const long long b = bt >> 1;
    float v = 0.f;
    if (t == 0 && c == act_idx[b * ld_tn + n]) v = dq_taken[b * N + n];
    dgi[i] = v;
  }
}
int mx_launch_mlp_dgi(const float* dq_taken, const int32_t* act_idx, int ld_tn, float* dgi, int B, int N, cudaStream_t s) {
  const long long total = (long long)B * 2 * N * MX_G;
  int grid = (int)((total + 255) / 256);
  const int cap = mx_num_sms() * 8;
  if (grid > cap) grid = cap;
  return mx_launch("k_mlp_dgi", k_mlp_dgi, dim3(grid), dim3(256), 0, s, MX_STEP, dq_taken, act_idx, ld_tn, dgi, B, N);
}

int mx_launch_gru_bwd(const GruBwdArgs& a, cudaStream_t s) {
  const int sms = mx_num_sms();
  int rpc = 1;
  while (rpc < 4 && mx_ceil_div(a.R, rpc) > 2 * sms) rpc *= 2;
  // sequences: the 128-thread kernel, one row per CTA (r02 sweeps)
  if (a.T >= 8) return mx_launch("k_gru_bwd", k_gru_bwd2<1>, dim3(a.R), dim3(BWD2_THREADS), 0, s, MX_STEP, a);
  auto kern = rpc == 1 ? k_gru_bwd<1> : rpc == 2 ? k_gru_bwd<2> : k_gru_bwd<4>;
  return mx_launch("k_gru_bwd", kern, dim3(mx_ceil_div(a.R, rpc)), dim3(BWD_THREADS), 0, s, MX_STEP, a);
}

// Tile height: the grid is one persistent CTA per SM, so the kernel takes `waves` tile-times; pick the 16*RM rows per tile that
// minimise waves * (fixed per-tile cost + RM) -- e.g. 3m: 5856 rows = 183 tiles of 32 (2 waves) but 122 tiles of 48 (1 wave).
static int front_bwd_pick_rm(int M, int in_dim, int sms, bool gru_ext) {
  int best = 2;
  double best_cost = 1e30;
  for (int rm = 2; rm <= 4; ++rm) {
    FrontBwdSmem sm = front_bwd_smem(in_dim, 16 * rm, gru_ext);
    if ((size_t)sm.total * sizeof(float) + 16 > MX_SMEM_OPTIN_MAX) continue;
    const int tiles = mx_ceil_div(M, 16 * rm);
    const double cost = (double)mx_ceil_div(tiles, sms) * (1.0 + rm);
    if (cost < best_cost - 1e-9) { best_cost = cost; best = rm; }
  }
  return best;
}

// The 32-row tile (RM 2, front_bwd_pick_rm's fallback) must fit; its input tiles are round_up(in_dim, 64) wide.
int mx_front_bwd_max_in_dim(bool gru_ext) {
  int w = 0;
  while ((size_t)front_bwd_smem(w + 64, 32, gru_ext).total * sizeof(float) + 16 <= MX_SMEM_OPTIN_MAX) w += 64;
  return w;
}

static int front_bwd_launch(const FrontBwdArgs& a, int rm, int* nparts_used, cudaStream_t s) {
  const int TM = 16 * rm;
  FrontBwdSmem sm = front_bwd_smem(a.L.in_dim, TM, a.gru_wgrad_ext != 0);
  const size_t smem = (size_t)sm.total * sizeof(float) + 16;
  const int ntiles = mx_ceil_div(a.M, TM);
  int grid = mx_num_sms();
  if (grid > ntiles) grid = ntiles;
#if !MX_EMU
  if (smem > MX_SMEM_OPTIN_MAX) { mx_set_error("front_bwd: %zu bytes of shared memory needed (obs_dim too large)", smem); return 1; }
#endif
  auto kern = rm == 3 ? k_front_bwd<3> : rm == 4 ? k_front_bwd<4> : k_front_bwd<2>;
  *nparts_used = grid;
  return mx_launch("k_front_bwd", kern, dim3(grid), dim3(MX_TILE_THREADS), smem, s, MX_STEP, a, sm);
}

bool mx_front_bwd_tc_usable(const FrontBwdArgs& a);
int mx_launch_front_bwd_tc(const FrontBwdArgs& a, int* nparts_used, cudaStream_t s);
int mx_launch_front_bwd(const FrontBwdArgs& a_in, int* nparts_used, cudaStream_t s) {
  if (mx_front_bwd_tc_usable(a_in)) return mx_launch_front_bwd_tc(a_in, nparts_used, s);
  FrontBwdArgs a = a_in;
  a.wgrad_external = mx_wgrad_tc_usable(a) ? 1 : 0;
  const int rm = front_bwd_pick_rm(a.M, a.L.in_dim, mx_num_sms(), a.gru_wgrad_ext != 0);
  const int rc = front_bwd_launch(a, rm, nparts_used, s);
  if (rc || !a.wgrad_external) return rc;
  return mx_launch_wgrad_tc(a, *nparts_used, s);      // one gradient partial per k_front_bwd CTA: the same rows of gpart
}

// ---- k_gru_wgrad beside k_front_bwd ----
bool mx_wgrad_tc_usable(const FrontBwdArgs& a);
bool mx_gru_wgrad_split_usable(const FrontBwdArgs& a) {
  if (a.no_gru || a.skip_wgrad) return false;
  return !mx_front_bwd_tc_usable(a) && !mx_wgrad_tc_usable(a);
}
// `a` must be the arguments the following mx_launch_front_bwd call gets (gru_wgrad_ext = 1): same tile height, same grid, so CTA b
// of both kernels writes gradient partial b
int mx_launch_gru_wgrad(const FrontBwdArgs& a, cudaStream_t s) {
  const int rm = front_bwd_pick_rm(a.M, a.L.in_dim, mx_num_sms(), true);
  const int TM = 16 * rm;
  GruWgradSmem sm = gru_wgrad_smem(TM);
  const size_t smem = (size_t)sm.total * sizeof(float) + 16;
  const int ntiles = mx_ceil_div(a.M, TM);
  int grid = mx_num_sms();
  if (grid > ntiles) grid = ntiles;
  auto kern = rm == 3 ? k_gru_wgrad<3> : rm == 4 ? k_gru_wgrad<4> : k_gru_wgrad<2>;
  return mx_launch("k_gru_wgrad", kern, dim3(grid), dim3(MX_TILE_THREADS), smem, s, MX_STEP, a, sm);
}
