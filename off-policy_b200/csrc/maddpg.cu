// Recurrent MADDPG / MATD3 learner (shared centralised observation, continuous actions): actor + centralised critic
// with K Q heads, target nets, two Adam groups.  Built from the same agent-net kernels as QMIX (front / GRU / LayerNorm
// building blocks) plus: critic-input packing, dense heads, "branch" GRU steps (one step from a stored hidden state,
// all (b,t) in parallel instead of the reference's Python loop of 2T single-step calls), TD / actor losses.
//
// reference: offpolicy/algorithms/r_maddpg/r_maddpg.py:114-331, r_maddpg/algorithm/{rMADDPGPolicy,r_actor_critic}.py,
// r_matd3/* (K = 2 heads, actor every 2nd update, Gaussian target noise handed in by the host from torch's CPU RNG).
//
// cfg.mlp: the transition-level MADDPG / MATD3 (algorithms/maddpg/maddpg.py:90-249, maddpg/algorithm/actor_critic.py) on the same
// kernels, see maddpg_step_mlp.
#include <string.h>

#include <vector>

#include "mx_internal.h"
#include "mx_kernels.h"

// =====================================================================================================
// small kernels
// =====================================================================================================
struct PackArgs {
  int mode;                 // 0: buffer actions (b,t) ; 1: next-step (share[t+1], target-actor actions[t+1]) ; 2: agent-replaced copies (i,b,t)
  int B, T, N, S, Ac;
  const float* share;       // [B][T+1][share_ld]
  int share_ld;
  const float* acts;        // [B][T][N][act_ld]
  int act_ld;
  const float* actor_out;   // [B*(T+1)*N][Ac]   (mode 1: target actor (+noise); mode 2: live actor)
  float* x;                 // [rows][ldx]
  int ldx;
  const float* hseq;        // mode 2: live critic states [B*T][H] -> h0 rows
  float* h0;                // mode 2: [rows][H]
  // several policies (share_policy = False): the critic sees the actions of ALL agents; this policy's N agents occupy columns
  // [off, off + N*Ac) of the CA-wide centralised action vector, the other policies' slices come from the assembled buffers
  int CA, off, ca_ld;
  const float* cent_acts;   // [B][T][ca_ld] buffer actions of every agent (mx_maddpg_cent_contribute), or null: single shared policy
  const float* cent_nacts;  // [B][T][ca_ld] target-actor actions at t+1 of every agent
};

__global__ void __launch_bounds__(256) k_pack_critic_in(PackArgs a) {
  const int IC = a.S + (a.cent_acts ? a.CA : a.N * a.Ac);
  const long long rows = (long long)(a.mode == 2 ? a.N : 1) * a.B * a.T;
  const long long total = rows * a.ldx;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const long long row = idx / a.ldx;
    const int c = (int)(idx - row * a.ldx);
    int i = 0;
    long long bt = row;
    if (a.mode == 2) { i = (int)(row / ((long long)a.B * a.T)); bt = row - (long long)i * a.B * a.T; }
    const int b = (int)(bt / a.T), t = (int)(bt % a.T);
    float v = 0.f;
    if (c < a.S) {
      v = a.share[((size_t)b * (a.T + 1) + t + (a.mode == 1 ? 1 : 0)) * a.share_ld + c];
    } else if (c < IC && a.cent_acts) {
      const int j = c - a.S;                                           // column of the centralised action vector
      const size_t cj = ((size_t)b * a.T + t) * a.ca_ld + j;
      if (a.mode == 0) v = a.cent_acts[cj];
      else if (a.mode == 1) v = a.cent_nacts[cj];
      else {
        const int jo = j - a.off;                                      // own agent i's slot is replaced by the live actor's action
        v = (jo >= i * a.Ac && jo < (i + 1) * a.Ac) ? a.actor_out[(((size_t)b * (a.T + 1) + t) * a.N + i) * a.Ac + (jo - i * a.Ac)] : a.cent_acts[cj];
      }
    } else if (c < IC) {
      const int n = (c - a.S) / a.Ac, k = (c - a.S) % a.Ac;
      if (a.mode == 0) v = a.acts[(((size_t)b * a.T + t) * a.N + n) * a.act_ld + k];
      else if (a.mode == 1) v = a.actor_out[(((size_t)b * (a.T + 1) + t + 1) * a.N + n) * a.Ac + k];
      else v = (n == i) ? a.actor_out[(((size_t)b * (a.T + 1) + t) * a.N + n) * a.Ac + k] : a.acts[(((size_t)b * a.T + t) * a.N + n) * a.act_ld + k];
    }
    a.x[idx] = v;
  }
  if (a.mode == 2 && a.h0) {
    const long long th = rows * MX_H;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < th; idx += (long long)gridDim.x * blockDim.x) {
      const long long row = idx / MX_H;
      const int c = (int)(idx % MX_H);
      const long long bt = row % ((long long)a.B * a.T);
      const int t = (int)(bt % a.T);
      a.h0[idx] = t > 0 ? a.hseq[(size_t)(bt - 1) * MX_H + c] : 0.f;      // critic state BEFORE step t
    }
  }
}

struct HeadArgs {
  const float* theta;
  int lno_g, lno_b, w, b;   // LayerNorm + Linear(H, OD): rows of W contiguous (q_outs.k are adjacent: [k][H] then biases [k])
  int OD;
  int b_stride;             // distance between consecutive biases in the flat vector (1 for a Linear(H,OD); 4 for K separate Linear(H,1))
  int w_stride;             // distance between consecutive weight rows
  const float* h;           // [M][H]
  int M;
  float* sto;               // (mean, rstd) [M][2] or null
  const float* noise;       // [M][OD] added to the output, or null
  float* out;               // [M][OD]
  float* out_min;           // [M] min over the OD outputs, or null
};

__global__ void __launch_bounds__(256) k_head_fwd(HeadArgs a) {
  __shared__ float w_s[8 * MX_H];
  __shared__ float lg_s[MX_H], lb_s[MX_H], b_s[8];
  const int tid = threadIdx.x, lane = tid & 31;
  for (int i = tid; i < a.OD * MX_H; i += blockDim.x) w_s[i] = a.theta[a.w + (i / MX_H) * a.w_stride + (i % MX_H)];
  for (int i = tid; i < a.OD; i += blockDim.x) b_s[i] = a.theta[a.b + i * a.b_stride];
  for (int i = tid; i < MX_H; i += blockDim.x) { lg_s[i] = a.theta[a.lno_g + i]; lb_s[i] = a.theta[a.lno_b + i]; }
  __syncthreads();
  const int wglobal = blockIdx.x * (blockDim.x >> 5) + (tid >> 5), wtotal = gridDim.x * (blockDim.x >> 5);
  for (int m = wglobal; m < a.M; m += wtotal) {
    const float* h = a.h + (size_t)m * MX_H;
    const float h0 = h[lane], h1 = h[lane + 32];
    const float mean = mx_warp_sum(h0 + h1) * (1.f / MX_H);
    const float d0 = h0 - mean, d1 = h1 - mean;
    const float rstd = rsqrtf(mx_warp_sum(d0 * d0 + d1 * d1) * (1.f / MX_H) + MX_LN_EPS);
    if (a.sto && lane == 0) { a.sto[2 * (size_t)m] = mean; a.sto[2 * (size_t)m + 1] = rstd; }
    const float y0 = d0 * rstd * lg_s[lane] + lb_s[lane], y1 = d1 * rstd * lg_s[lane + 32] + lb_s[lane + 32];
    float mn = 0.f;
    for (int o = 0; o < a.OD; ++o) {
      float q = mx_warp_sum(y0 * w_s[o * MX_H + lane] + y1 * w_s[o * MX_H + lane + 32]) + b_s[o];
      if (a.noise) q += a.noise[(size_t)m * a.OD + o];
      if (lane == 0) a.out[(size_t)m * a.OD + o] = q;
      mn = (o == 0 || q < mn) ? q : mn;
    }
    if (a.out_min && lane == 0) a.out_min[m] = mn;
  }
}

struct HeadBwdArgs {
  const float* theta;
  int lno_g, lno_b, w, b, OD, b_stride, w_stride;
  const float* h;           // [M][H]
  const float* sto;         // [M][2]
  const float* dout;        // [M][OD]
  int M;
  float* dh_out;            // [M][H]
  float* gpart;             // per-CTA partial or null (frozen head)
  long long P;
};

__global__ void __launch_bounds__(256) k_head_bwd(HeadBwdArgs a) {
  __shared__ float w_s[8 * MX_H], dw_s[8 * MX_H];
  __shared__ float db_s[8], dg_s[MX_H], dbb_s[MX_H], lg_s[MX_H], lb_s[MX_H];
  const int tid = threadIdx.x, lane = tid & 31;
  for (int i = tid; i < a.OD * MX_H; i += blockDim.x) { w_s[i] = a.theta[a.w + (i / MX_H) * a.w_stride + (i % MX_H)]; dw_s[i] = 0.f; }
  for (int i = tid; i < 8; i += blockDim.x) db_s[i] = 0.f;
  for (int i = tid; i < MX_H; i += blockDim.x) { dg_s[i] = 0.f; dbb_s[i] = 0.f; lg_s[i] = a.theta[a.lno_g + i]; lb_s[i] = a.theta[a.lno_b + i]; }
  __syncthreads();
  const int wglobal = blockIdx.x * (blockDim.x >> 5) + (tid >> 5), wtotal = gridDim.x * (blockDim.x >> 5);
  float dg0 = 0.f, dg1 = 0.f, db0 = 0.f, db1 = 0.f;
  float dw0[8], dw1[8], dbo[8];      // this warp's head-weight gradient in registers: summed over warps in a fixed order below
#pragma unroll
  for (int o = 0; o < 8; ++o) { dw0[o] = 0.f; dw1[o] = 0.f; dbo[o] = 0.f; }
  for (int m = wglobal; m < a.M; m += wtotal) {
    const float* h = a.h + (size_t)m * MX_H;
    const float mean = a.sto[2 * (size_t)m], rstd = a.sto[2 * (size_t)m + 1];
    const float xh0 = (h[lane] - mean) * rstd, xh1 = (h[lane + 32] - mean) * rstd;
    const float y0 = xh0 * lg_s[lane] + lb_s[lane], y1 = xh1 * lg_s[lane + 32] + lb_s[lane + 32];
    float dy0 = 0.f, dy1 = 0.f;
#pragma unroll
    for (int o = 0; o < 8; ++o)
      if (o < a.OD) {
        const float d = a.dout[(size_t)m * a.OD + o];
        dy0 = fmaf(d, w_s[o * MX_H + lane], dy0);
        dy1 = fmaf(d, w_s[o * MX_H + lane + 32], dy1);
        dw0[o] = fmaf(d, y0, dw0[o]); dw1[o] = fmaf(d, y1, dw1[o]); dbo[o] += d;
      }
    dg0 += dy0 * xh0; dg1 += dy1 * xh1; db0 += dy0; db1 += dy1;
    const float dx0 = dy0 * lg_s[lane], dx1 = dy1 * lg_s[lane + 32];
    const float c1 = mx_warp_sum(dx0 + dx1) * (1.f / MX_H);
    const float c2 = mx_warp_sum(dx0 * xh0 + dx1 * xh1) * (1.f / MX_H);
    a.dh_out[(size_t)m * MX_H + lane] = rstd * (dx0 - c1 - xh0 * c2);
    a.dh_out[(size_t)m * MX_H + lane + 32] = rstd * (dx1 - c1 - xh1 * c2);
  }
  if (!a.gpart) return;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) {       // warps in turn: deterministic, no shared atomics
    if ((tid >> 5) == w) {
#pragma unroll
      for (int o = 0; o < 8; ++o)
        if (o < a.OD) {
          dw_s[o * MX_H + lane] += dw0[o]; dw_s[o * MX_H + lane + 32] += dw1[o];
          if (lane == 0) db_s[o] += dbo[o];
        }
      dg_s[lane] += dg0; dg_s[lane + 32] += dg1;
      dbb_s[lane] += db0; dbb_s[lane + 32] += db1;
    }
    __syncthreads();
  }
  float* gp = a.gpart + (size_t)blockIdx.x * a.P;
  for (int i = tid; i < a.OD * MX_H; i += blockDim.x) gp[a.w + (i / MX_H) * a.w_stride + (i % MX_H)] = dw_s[i];
  for (int i = tid; i < a.OD; i += blockDim.x) gp[a.b + i * a.b_stride] = db_s[i];
  for (int i = tid; i < MX_H; i += blockDim.x) { gp[a.lno_g + i] = dg_s[i]; gp[a.lno_b + i] = dbb_s[i]; }
}

struct CriticLossArgs {
  int B, T, N, K;
  int ld_tn, ld_t;          // floats between consecutive episodes of rewards (>= T*N) and dones_env (>= T)
  const float* qpred;       // [B*T][K]
  const float* qnext_min;   // [B*T]
  const float* rewards;     // [B][T][N]
  const float* dones_env;   // [B][T]
  const float* weights;     // [B] or null
  float gamma, huber_delta, per_nu, per_eps;
  int use_huber;
  int prio_mean_k;          // 1: priority = mean_k |err_k| + per_eps (T = 1, maddpg.py:144); 0: the recurrent formula below
  float* dq;                // [B*T][K]
  float* err;               // [K][B*T]
  float* scal;              // [4]: sum(1-bad), loss numerator, -, elements
  float* prio;              // [B] or null
};

__global__ void __launch_bounds__(256) k_critic_loss(CriticLossArgs a) {   // ONE CTA (B*T is small); deterministic sums
  __shared__ float red[2][256];
  const int E = a.B * a.T, tid = threadIdx.x;
  float den = 0.f, ls = 0.f;
  for (int e = tid; e < E; e += blockDim.x) {
    const int b = e / a.T, t = e % a.T;
    const float rew = a.rewards[(size_t)b * a.ld_tn + (size_t)t * a.N];
    const float de = a.dones_env[(size_t)b * a.ld_t + t];
    const float bad = t > 0 ? a.dones_env[(size_t)b * a.ld_t + t - 1] : 0.f;
    const float keep = 1.f - bad;
    const float y = rew + a.gamma * (1.f - de) * a.qnext_min[e];
    const float w = a.weights ? a.weights[b] : 1.f;
    den += keep;
    for (int k = 0; k < a.K; ++k) {
      const float err = (a.qpred[(size_t)e * a.K + k] - y) * keep;
      float le, dle;
      if (a.use_huber) {
        const float ae = fabsf(err);
        if (ae <= a.huber_delta) { le = 0.5f * err * err; dle = err; }
        else { le = a.huber_delta * (ae - 0.5f * a.huber_delta); dle = err > 0.f ? a.huber_delta : -a.huber_delta; }
      } else { le = err * err; dle = 2.f * err; }
      a.dq[(size_t)e * a.K + k] = dle * keep * w;
      a.err[(size_t)k * E + e] = err;
      ls += le * w;
    }
  }
  red[0][tid] = den; red[1][tid] = ls;
  __syncthreads();
  if (tid == 0) {
    float s0 = 0.f, s1 = 0.f;
    for (int i = 0; i < (int)blockDim.x; ++i) { s0 += red[0][i]; s1 += red[1][i]; }
    a.scal[0] = s0; a.scal[1] = s1; a.scal[2] = 0.f; a.scal[3] = (float)E;
  }
  if (a.prio) {
    __syncthreads();
    for (int b = tid; b < a.B; b += blockDim.x) {
      if (a.prio_mean_k) {
        float sm = 0.f;
        for (int k = 0; k < a.K; ++k) sm += fabsf(a.err[(size_t)k * E + b]);
        a.prio[b] = sm / (float)a.K + a.per_eps;
        continue;
      }
      float acc = 0.f;
      for (int k = 0; k < a.K; ++k) {
        float mx = 0.f, sm = 0.f;
        for (int t = 0; t < a.T; ++t) { const float e = fabsf(a.err[(size_t)k * E + b * a.T + t]); sm += e; mx = fmaxf(mx, e); }
        acc += (1.f - a.per_nu) * (sm / (float)a.T) + a.per_nu * mx + a.per_eps;
      }
      a.prio[b] = acc / (float)a.K + a.per_eps;          // r_maddpg.py:216-217 adds per_eps twice
    }
  }
}

struct ActorLossArgs {
  int B, T, N, K;
  int ld_tn;                // floats between consecutive episodes of dones (>= T*N)
  const float* qa;          // [N*B*T][K] critic outputs on the agent-replaced copies (head 0 is used)
  const float* dones;       // [B][T][N]
  const float* valid;       // T = 1 (cfg.mlp): valid_transition [rows][N] read at row valid_idx[b] (b when null), maddpg.py:197-232; or null
  const int64_t* valid_idx;
  float* dout;              // [N*B*T][K]
  float* scal;              // [4]: sum(1-done_mask), loss numerator = -sum Q (1-done_mask)
};

__global__ void __launch_bounds__(256) k_actor_loss(ActorLossArgs a) {   // ONE CTA
  __shared__ float red[2][256];
  const int rows = a.N * a.B * a.T, tid = threadIdx.x;
  float den = 0.f, ls = 0.f;
  for (int row = tid; row < rows; row += blockDim.x) {
    const int i = row / (a.B * a.T), bt = row % (a.B * a.T);
    const int b = bt / a.T, t = bt % a.T;
    const float dm = t > 0 ? a.dones[(size_t)b * a.ld_tn + (size_t)(t - 1) * a.N + i] : 0.f;    // r_maddpg.py:268-272
    const float keep = a.valid ? a.valid[(size_t)(a.valid_idx ? a.valid_idx[b] : b) * a.N + i] : 1.f - dm;
    den += keep;
    ls -= a.qa[(size_t)row * a.K] * keep;
    for (int k = 0; k < a.K; ++k) a.dout[(size_t)row * a.K + k] = k == 0 ? -keep : 0.f;
  }
  red[0][tid] = den; red[1][tid] = ls;
  __syncthreads();
  if (tid == 0) {
    float s0 = 0.f, s1 = 0.f;
    for (int i = 0; i < (int)blockDim.x; ++i) { s0 += red[0][i]; s1 += red[1][i]; }
    a.scal[0] = s0; a.scal[1] = s1; a.scal[2] = 0.f; a.scal[3] = (float)rows;
  }
}

// The action of one agent as one-hot blocks (MultiDiscrete: one per sub-space, act.py:15-17; Box / Discrete: one block of Ac).
#define MX_MAX_ACT 32       // widest action the kernels below hold in registers (cfg.mlp; the recurrent learner keeps Ac <= 8)
struct ActSegs {
  int n;                    // number of blocks, >= 1
  int len[MX_MAX_ACT_SEG];  // their widths, summing to Ac
};

// d(actor action of agent i at (b,t)) = dX[(i,b,t)][S + i*Ac + k]   ->   dense head gradient of the actor [M_a][Ac].
// Discrete actors (soft != null): the action is the straight-through hard Gumbel-softmax sample, so the gradient reaches the
// logits through the soft sample y = softmax(logits + g) of its block:  dlogit_k = y_k (d_k - sum_{j in block(k)} d_j y_j)   (util.py:160-165)
// dact rows have dact_ld >= Ac columns, the ones past Ac are zero-filled (cfg.mlp: the actor's "gi" gradient rows, dact_ld = 3H).
__global__ void __launch_bounds__(256) k_scatter_actor_grad(const float* dX, int ldx, int B, int T, int N, int S, int Ac, const float* soft, float* dact, int off,
                                                            int dact_ld, ActSegs sg) {
  const long long rows = (long long)B * (T + 1) * N;
  for (long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x; m < rows; m += (long long)gridDim.x * blockDim.x) {
    const int n = (int)(m % N);
    const long long bt1 = m / N;
    const int t = (int)(bt1 % (T + 1)), b = (int)(bt1 / (T + 1));
    float d[MX_MAX_ACT];      // fully unrolled below: held in registers
#pragma unroll
    for (int k = 0; k < MX_MAX_ACT; ++k) d[k] = (k < Ac && t < T) ? dX[(((size_t)n * B + b) * T + t) * ldx + S + off + n * Ac + k] : 0.f;
    if (soft) {
      float y[MX_MAX_ACT];
#pragma unroll
      for (int k = 0; k < MX_MAX_ACT; ++k) y[k] = k < Ac ? soft[m * Ac + k] : 0.f;
      int k0 = 0;
#pragma unroll
      for (int s = 0; s < MX_MAX_ACT_SEG; ++s) {
        if (s >= sg.n) break;
        const int k1 = k0 + sg.len[s];
        float dot = 0.f;
#pragma unroll
        for (int k = 0; k < MX_MAX_ACT; ++k)
          if (k >= k0 && k < k1) dot += d[k] * y[k];
#pragma unroll
        for (int k = 0; k < MX_MAX_ACT; ++k)
          if (k >= k0 && k < k1) d[k] = y[k] * (d[k] - dot);
        k0 = k1;
      }
    }
#pragma unroll
    for (int k = 0; k < MX_MAX_ACT; ++k)
      if (k < Ac) dact[m * dact_ld + k] = d[k];
    for (int k = Ac; k < dact_ld; ++k) dact[m * dact_ld + k] = 0.f;
  }
}

// Discrete action heads (Ac <= MX_MAX_ACT, one thread per row), each block of sg on its own.  mode 0: `onehot_from_logits` = every
// maximal logit of the block is hot (util.py:106-118);  mode 1: hard Gumbel-softmax, value (y_hard - y) + y with y = softmax(logits + g)
// over the block and y_hard the one-hot of the block's maxima of y (util.py:133-166, temperature 1).  Unavailable actions are forced to
// -1e10 first (util.py:115, 141); MultiDiscrete heads ignore the mask (MADDPGPolicy.py:73-89), so the caller passes none.
struct ActXformArgs {
  int M, Ac, mode;
  const float* logits;      // [M][Ac]  (already includes the Gumbel draw when gumbel == null)
  const float* gumbel;      // [M][Ac] or null
  const float* avail;       // [M][avail_ld] or null
  int avail_ld;
  float* out;               // [M][Ac]
  float* soft;              // [M][Ac] soft sample (mode 1) or null
  ActSegs sg;
};
__global__ void __launch_bounds__(256) k_act_transform(ActXformArgs a) {
  for (long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x; m < a.M; m += (long long)gridDim.x * blockDim.x) {
    float v[MX_MAX_ACT];      // fully unrolled below: held in registers
#pragma unroll
    for (int k = 0; k < MX_MAX_ACT; ++k) {
      float x = 0.f;
      if (k < a.Ac) {
        x = a.logits[m * a.Ac + k];
        if (a.gumbel) x += a.gumbel[m * a.Ac + k];
        if (a.avail && a.avail[m * a.avail_ld + k] == 0.f) x = -1e10f;
      }
      v[k] = x;
    }
    int k0 = 0;
#pragma unroll
    for (int s = 0; s < MX_MAX_ACT_SEG; ++s) {
      if (s >= a.sg.n) break;
      const int k1 = k0 + a.sg.len[s];
      float mx = -INFINITY;
#pragma unroll
      for (int k = 0; k < MX_MAX_ACT; ++k)
        if (k >= k0 && k < k1) mx = fmaxf(mx, v[k]);
      if (a.mode == 0) {
#pragma unroll
        for (int k = 0; k < MX_MAX_ACT; ++k)
          if (k >= k0 && k < k1) a.out[m * a.Ac + k] = v[k] == mx ? 1.f : 0.f;
        k0 = k1;
        continue;
      }
      float sum = 0.f;
#pragma unroll
      for (int k = 0; k < MX_MAX_ACT; ++k)
        if (k >= k0 && k < k1) { v[k] = expf(v[k] - mx); sum += v[k]; }
      float ymax = 0.f;
#pragma unroll
      for (int k = 0; k < MX_MAX_ACT; ++k)
        if (k >= k0 && k < k1) { v[k] = v[k] / sum; ymax = fmaxf(ymax, v[k]); }
#pragma unroll
      for (int k = 0; k < MX_MAX_ACT; ++k)
        if (k >= k0 && k < k1) {
          const float hard = v[k] == ymax ? 1.f : 0.f;
          a.out[m * a.Ac + k] = (hard - v[k]) + v[k];
          if (a.soft) a.soft[m * a.Ac + k] = v[k];
        }
      k0 = k1;
    }
  }
}

// ---- cfg.mlp: the heads sit in the weight_ih slot, so the front kernel's "gi" rows [M][3H] carry the head outputs in columns [0, K) ----
// out[m][k] = gi[m][k] (+ noise[m][k]), out_min[m] = min_k of the same values; either output may be null
__global__ void __launch_bounds__(256) k_mlp_head_cols(const float* __restrict__ gi, int M, int K, const float* __restrict__ noise,
                                                       float* __restrict__ out, float* __restrict__ out_min) {
  for (long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x; m < M; m += (long long)gridDim.x * blockDim.x) {
    float mn = 0.f;
    for (int k = 0; k < K; ++k) {
      float v = gi[m * MX_G + k];
      if (noise) v += noise[m * K + k];
      if (out) out[m * K + k] = v;
      mn = (k == 0 || v < mn) ? v : mn;      // torch.min over the heads (maddpg.py:117)
    }
    if (out_min) out_min[m] = mn;
  }
}

// dgi[m][j] = j < K ? src[m][j] : 0 over [M][3H]: the gradient at the head outputs as the "gi" gradient rows k_front_bwd reads
__global__ void __launch_bounds__(256) k_mlp_dgi_cols(const float* __restrict__ src, int K, int M, float* __restrict__ dgi) {
  const long long total = (long long)M * MX_G;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long m = i / MX_G;
    const int j = (int)(i - m * MX_G);
    dgi[i] = j < K ? src[m * K + j] : 0.f;
  }
}

// =====================================================================================================
// handle
// =====================================================================================================
// The regions of one pass of a network over its rows (offsets in floats into the workspace).  Slot k of gi / h / out belongs to copy k
// of the network (0: live, 1: target); a pass that runs one copy only has that copy's slot.
struct MxPassWs {
  int64_t x;                // critic passes: the packed input rows [M][ldc]
  int64_t gi[2], h[2];      // [M][3H] GRU input rows (cfg.mlp: the head outputs in columns [0, OD)), [M][H] hidden states
  int64_t u1, u2, st0, st1, st2, sto, gates, hn;      // the live copy's activations, kept for the backward
  int64_t out[2];           // head outputs [M][OD]
  int64_t dout, dh, dgi;    // gradients at the head outputs, the hidden states and the GRU input rows
};

struct MxMaddpgWs {
  struct : MxPassWs { int64_t act, soft; } a;   // actor rows Ma = B*(T+1)*N; out[1]: target actions; act / soft: the live actor's Gumbel sample
  struct : MxPassWs { int64_t err; } c;         // critic over the buffer sequences, rows Mc = B*T; err: TD errors [K][Mc]
  struct : MxPassWs { int64_t qmin; } t;        // target branch, rows Mc (target slots); qmin: min over the target heads
  struct : MxPassWs { int64_t h0, dx; } r;      // agent-replaced copies, rows Mr = N*B*T (live slots); h0: critic state before the step,
                                                // dx: gradient at the input rows
  int64_t gpart_a, gpart_c, grad_a, grad_c, spart, info, prio, adam_ta, adam_tc, scal_c, scal_a;
  int64_t p2p_abort;        // data parallel: the sticky abort word of both exchanges (-1 after a peer time-out: no update is applied)
  int64_t tc_da2, tc_da1, tc_imgT, tc_acc, tc_acc_cols;      // scratch of the tensor-core backward (option wgrad_tc), shared by the critic and actor updates
  int64_t cent_acts, cent_nacts;        // [B*T][ca_ld] centralised action vectors assembled from all policies (cent_act_dim > 0)
  int64_t total;
};

struct mx_maddpg {
  mx_maddpg_cfg cfg;
  MxNetLayout actor, critic;
  int64_t Pa, Pc;
  int npart;
  float *th_a, *th_a_tgt, *m_a, *v_a, *th_c, *th_c_tgt, *m_c, *v_c;
  float* ws;
  MxMaddpgWs W;
  int64_t num_updates;
  const float* valid = nullptr;     // cfg.mlp: valid_transition store [rows][n_agents] (mx_maddpg_set_valid)
  int force_update_actor = -1;      // graph capture: -1 = decide from num_updates, 0 / 1 = record this variant
  MxP2pPeers p2p[2];                // data parallel (mx_maddpg_set_peers): the peers of the actor's [0] and the critic's [1] exchange
  int phase_next = 0;               // mx_maddpg_step_phase: the phase the update in progress expects next (0: none in progress)
  bool phase_actor = false;         //   and whether that update trains the actor
};

static inline int mx_imin_host(int a, int b) { return a < b ? a : b; }
static int cent_act_width(const mx_maddpg_cfg* c) { return c->cent_act_dim > 0 ? c->cent_act_dim : c->n_agents * c->act_dim; }
static int critic_in_dim(const mx_maddpg_cfg* c) { return c->state_dim + cent_act_width(c); }
// the one-hot blocks of one agent's action: cfg.act_seg, or one block of act_dim when n_act_seg = 0
static ActSegs act_segs(const mx_maddpg_cfg* c) {
  ActSegs sg;
  memset(&sg, 0, sizeof(sg));
  if (c->n_act_seg <= 0) { sg.n = 1; sg.len[0] = c->act_dim; return sg; }
  sg.n = c->n_act_seg;
  for (int i = 0; i < c->n_act_seg; ++i) sg.len[i] = c->act_seg[i];
  return sg;
}
static int maddpg_check(const mx_maddpg_cfg* c) {
  if (!c) { mx_set_error("null cfg"); return 1; }
  if (c->hidden != MX_H) { mx_set_error("hidden_size %d unsupported: kernels are specialised for %d", c->hidden, MX_H); return 1; }
  if (c->n_agents <= 0 || c->obs_dim <= 0 || c->act_dim <= 0 || c->state_dim <= 0 || c->episode_len <= 0 || c->max_batch <= 0) { mx_set_error("mx_maddpg: non-positive dimension"); return 1; }
  if (c->num_q < 1 || c->num_q > 4) { mx_set_error("mx_maddpg: num_q must be 1..4"); return 1; }
  if (c->act_dim > (c->mlp ? MX_MAX_ACT : 8)) {
    mx_set_error("mx_maddpg: act_dim %d > %d (the %s learner's limit)", c->act_dim, c->mlp ? MX_MAX_ACT : 8, c->mlp ? "MLP" : "recurrent"); return 1;
  }
  if (c->n_act_seg < 0 || c->n_act_seg > MX_MAX_ACT_SEG) { mx_set_error("mx_maddpg: n_act_seg %d outside [0, %d]", c->n_act_seg, MX_MAX_ACT_SEG); return 1; }
  if (c->n_act_seg > 0) {
    if (!c->discrete) { mx_set_error("mx_maddpg: action segments (MultiDiscrete) need discrete = 1"); return 1; }
    if (!c->mlp) {      // n_act_seg > 0 means MultiDiscrete (per-block transforms, no mask): built for the MLP learner only
      mx_set_error("mx_maddpg: the recurrent learner takes no action segments (n_act_seg = %d); MultiDiscrete is built for the MLP learner only", c->n_act_seg);
      return 1;
    }
    int sum = 0;
    for (int i = 0; i < c->n_act_seg; ++i) {
      if (c->act_seg[i] < 1) { mx_set_error("mx_maddpg: action segment %d has width %d < 1", i, c->act_seg[i]); return 1; }
      sum += c->act_seg[i];
    }
    if (sum != c->act_dim) { mx_set_error("mx_maddpg: action segments sum to %d, act_dim is %d", sum, c->act_dim); return 1; }
  }
  if (c->max_batch * c->episode_len > 65536) { mx_set_error("mx_maddpg: B*T too large"); return 1; }
  if (c->cent_act_dim < 0 || c->act_offset < 0 || (c->cent_act_dim > 0 && c->act_offset + c->n_agents * c->act_dim > c->cent_act_dim)) {
    mx_set_error("mx_maddpg: act_offset %d + n_agents*act_dim %d exceeds cent_act_dim %d", c->act_offset, c->n_agents * c->act_dim, c->cent_act_dim); return 1;
  }
  if (c->cent_act_dim == 0 && c->act_offset != 0) { mx_set_error("mx_maddpg: act_offset needs cent_act_dim"); return 1; }
  if (c->mlp && c->episode_len != 1) {
    mx_set_error("mx_maddpg: the MLP (transition-level) variant takes transitions as episodes of length 1"); return 1;
  }
  {     // every net's backward (and the critic's data gradient) runs k_front_bwd without k_gru_wgrad beside it
    const int lim = mx_front_bwd_max_in_dim(false);
    if (c->obs_dim > lim) { mx_set_error("mx_maddpg: actor input width %d (obs_dim) exceeds %d, the widest k_front_bwd's shared memory holds", c->obs_dim, lim); return 1; }
    if (critic_in_dim(c) > lim) {
      mx_set_error("mx_maddpg: critic input width %d (state_dim %d + %d action columns) exceeds %d, the widest k_front_bwd's shared memory holds",
                   critic_in_dim(c), c->state_dim, cent_act_width(c), lim);
      return 1;
    }
  }
  return 0;
}

// critic: q_outs.k are K separate Linear(H,1): weights [K][H] contiguous, then K biases (each padded to 4 floats)
// cfg.mlp: both nets keep their head in the first rows of the weight_ih slot (the actor's trained head; the critic's K frozen heads,
// whose live and target copies are the tails of the two critic vectors past the trunk [0, wih))
static void maddpg_layouts(const mx_maddpg_cfg* c, MxNetLayout* A, MxNetLayout* Cr) {
  mx_net_layout(c->obs_dim, c->act_dim, 0, A);
  if (c->mlp) { mx_net_layout(critic_in_dim(c), c->num_q, 0, Cr); return; }
  // critic head: out_dim = K rows of H, but each q_outs.k is its own tensor -> lay out as (w0, b0, w1, b1, ...)
  mx_net_layout(critic_in_dim(c), 1, 0, Cr);
  // mx_net_layout put wq (1 x H) and bq (1, padded to 4); extend for K heads: stride between heads = H + 4
  Cr->out_dim = c->num_q;
  Cr->size = Cr->wq + c->num_q * (MX_H + 4);
}

extern "C" int mx_maddpg_param_layout(const mx_maddpg_cfg* c, int32_t which, mx_param_entry* out, int32_t max_entries, int64_t* total_floats) {
  if (maddpg_check(c)) return -1;
  MxNetLayout A, Cr;
  maddpg_layouts(c, &A, &Cr);
  const MxNetLayout& L = which == 0 ? A : Cr;
  if (which < 0 || which > 2 || (which == 2 && !c->mlp)) { mx_set_error("mx_maddpg_param_layout: which = %d", which); return -1; }
  std::vector<mx_param_entry> v;
  auto add = [&](const char* name, int off, int rows, int cols) {
    mx_param_entry e;
    memset(&e, 0, sizeof(e));
    snprintf(e.name, MX_MAX_NAME, "%s", name);
    e.offset = off; e.rows = rows; e.cols = cols;
    v.push_back(e);
  };
  const int H = MX_H, I = L.in_dim;
  if (c->mlp) {      // MADDPG_Actor / MADDPG_Critic: MLPBase (mlp.py:52-89) + ACTLayer (act.py) / q_outs (actor_critic.py:67)
    if (which == 2) {
      for (int k = 0; k < c->num_q; ++k) {
        char nm[64];
        snprintf(nm, sizeof(nm), "q_outs.%d.weight", k); add(nm, L.wih + k * H, 1, H);
        snprintf(nm, sizeof(nm), "q_outs.%d.bias", k); add(nm, L.bih + k, 1, 0);
      }
    } else {
      if (!c->no_feature_norm) { add("mlp.feature_norm.weight", L.fn_g, I, 0); add("mlp.feature_norm.bias", L.fn_b, I, 0); }
      add("mlp.mlp.fc1.0.weight", L.w1, H, I); add("mlp.mlp.fc1.0.bias", L.b1, H, 0);
      add("mlp.mlp.fc1.2.weight", L.ln1_g, H, 0); add("mlp.mlp.fc1.2.bias", L.ln1_b, H, 0);
      add("mlp.mlp.fc_h.0.weight", L.wh, H, H); add("mlp.mlp.fc_h.0.bias", L.bh, H, 0);
      add("mlp.mlp.fc_h.2.weight", L.lnh_g, H, 0); add("mlp.mlp.fc_h.2.bias", L.lnh_b, H, 0);
      add("mlp.mlp.fc2.0.0.weight", L.w2, H, H); add("mlp.mlp.fc2.0.0.bias", L.b2, H, 0);
      add("mlp.mlp.fc2.0.2.weight", L.ln2_g, H, 0); add("mlp.mlp.fc2.0.2.bias", L.ln2_b, H, 0);
      if (which == 0 && c->n_act_seg > 0) {      // ACTLayer.action_outs (act.py:15-17): consecutive row blocks of the one head
        int r = 0;
        for (int i = 0; i < c->n_act_seg; ++i) {
          char nm[64];
          snprintf(nm, sizeof(nm), "act.action_outs.%d.weight", i); add(nm, L.wih + H * r, c->act_seg[i], H);
          snprintf(nm, sizeof(nm), "act.action_outs.%d.bias", i); add(nm, L.bih + r, c->act_seg[i], 0);
          r += c->act_seg[i];
        }
      } else if (which == 0) {
        add("act.action_out.weight", L.wih, c->act_dim, H); add("act.action_out.bias", L.bih, c->act_dim, 0);
      }
    }
    if (total_floats) *total_floats = L.size;
    const int n = (int)v.size();
    if (out) for (int i = 0; i < n && i < max_entries; ++i) out[i] = v[i];
    return n;
  }
  if (!c->no_feature_norm) { add("rnn.feature_norm.weight", L.fn_g, I, 0); add("rnn.feature_norm.bias", L.fn_b, I, 0); }
  add("rnn.mlp.fc1.0.weight", L.w1, H, I); add("rnn.mlp.fc1.0.bias", L.b1, H, 0);
  add("rnn.mlp.fc1.2.weight", L.ln1_g, H, 0); add("rnn.mlp.fc1.2.bias", L.ln1_b, H, 0);
  add("rnn.mlp.fc_h.0.weight", L.wh, H, H); add("rnn.mlp.fc_h.0.bias", L.bh, H, 0);
  add("rnn.mlp.fc_h.2.weight", L.lnh_g, H, 0); add("rnn.mlp.fc_h.2.bias", L.lnh_b, H, 0);
  add("rnn.mlp.fc2.0.0.weight", L.w2, H, H); add("rnn.mlp.fc2.0.0.bias", L.b2, H, 0);
  add("rnn.mlp.fc2.0.2.weight", L.ln2_g, H, 0); add("rnn.mlp.fc2.0.2.bias", L.ln2_b, H, 0);
  add("rnn.rnn.rnn.weight_ih_l0", L.wih, 3 * H, H); add("rnn.rnn.rnn.weight_hh_l0", L.whh, 3 * H, H);
  add("rnn.rnn.rnn.bias_ih_l0", L.bih, 3 * H, 0); add("rnn.rnn.rnn.bias_hh_l0", L.bhh, 3 * H, 0);
  add("rnn.rnn.norm.weight", L.lno_g, H, 0); add("rnn.rnn.norm.bias", L.lno_b, H, 0);
  if (which == 0) {
    add("act.action_out.weight", L.wq, c->act_dim, H); add("act.action_out.bias", L.bq, c->act_dim, 0);
  } else {
    for (int k = 0; k < c->num_q; ++k) {
      char nm[64];
      snprintf(nm, sizeof(nm), "q_outs.%d.weight", k); add(nm, L.wq + k * (H + 4), 1, H);
      snprintf(nm, sizeof(nm), "q_outs.%d.bias", k); add(nm, L.wq + k * (H + 4) + H, 1, 0);
    }
  }
  if (total_floats) *total_floats = L.size;
  const int n = (int)v.size();
  if (out) for (int i = 0; i < n && i < max_entries; ++i) out[i] = v[i];
  return n;
}

static int64_t maddpg_ws_layout(const mx_maddpg_cfg* c, int64_t Pa, int64_t Pc, int npart, MxMaddpgWs* W) {
  const int64_t B = c->max_batch, T = c->episode_len, N = c->n_agents, K = c->num_q, Ac = c->act_dim;
  const int64_t Ma = B * (T + 1) * N, Mc = B * T, Mr = N * B * T;
  const int64_t ldc = mx_round_up(critic_in_dim(c), 4);
  int64_t o = 0;
  auto tk = [&](int64_t n) { int64_t r = o; o += (n + 63) / 64 * 64; return r; };
  auto acts = [&](MxPassWs& p, int64_t M) {
    p.u1 = tk(M * MX_H); p.u2 = tk(M * MX_H); p.st0 = tk(M * 2); p.st1 = tk(M * 2); p.st2 = tk(M * 2); p.sto = tk(M * 2);
    p.gates = tk(M * MX_G); p.hn = tk(M * MX_H);
  };
  for (int k = 0; k < 2; ++k) { W->a.gi[k] = tk(Ma * MX_G); W->a.h[k] = tk(Ma * MX_H); }
  acts(W->a, Ma);
  W->a.out[0] = tk(Ma * Ac); W->a.out[1] = tk(Ma * Ac); W->a.dout = tk(Ma * Ac);
  W->a.dh = tk(Ma * MX_H); W->a.dgi = tk(Ma * MX_G); W->a.act = tk(Ma * Ac); W->a.soft = tk(Ma * Ac);
  W->c.x = tk(Mc * ldc);
  for (int k = 0; k < 2; ++k) { W->c.gi[k] = tk(Mc * MX_G); W->c.h[k] = tk(Mc * MX_H); }
  acts(W->c, Mc);
  W->c.out[0] = tk(Mc * K); W->c.dout = tk(Mc * K); W->c.dh = tk(Mc * MX_H); W->c.dgi = tk(Mc * MX_G);
  W->c.err = tk(Mc * K);
  W->t.x = tk(Mc * ldc); W->t.gi[1] = tk(Mc * MX_G); W->t.h[1] = tk(Mc * MX_H); W->t.out[1] = tk(Mc * K); W->t.qmin = tk(Mc);
  W->r.x = tk(Mr * ldc); W->r.h0 = tk(Mr * MX_H); W->r.gi[0] = tk(Mr * MX_G); W->r.h[0] = tk(Mr * MX_H);
  acts(W->r, Mr);
  W->r.out[0] = tk(Mr * K); W->r.dout = tk(Mr * K); W->r.dh = tk(Mr * MX_H); W->r.dgi = tk(Mr * MX_G); W->r.dx = tk(Mr * ldc);
  W->gpart_a = tk((int64_t)npart * Pa); W->gpart_c = tk((int64_t)npart * Pc); W->grad_a = tk(Pa + 8); W->grad_c = tk(Pc + 8);
  W->spart = tk(16); W->info = tk(8); W->prio = tk(B); W->adam_ta = tk(8); W->adam_tc = tk(8); W->scal_c = tk(8); W->scal_a = tk(8);
  W->p2p_abort = tk(8);
  {
    const int64_t Mx = Ma > Mc ? Ma : Mc;
    const size_t ia = mx_tc_imageT_floats(c->obs_dim), ic = mx_tc_imageT_floats(critic_in_dim(c));
    W->tc_da2 = tk(Mx * MX_H); W->tc_da1 = tk(Mx * MX_H); W->tc_imgT = tk((int64_t)(ia > ic ? ia : ic));
    W->tc_acc = tk((int64_t)mx_tc_acc_floats(Mx)); W->tc_acc_cols = (int64_t)mx_tc_acc_floats(Mx) / 128;
  }
  {
    const int64_t ca_ld = c->cent_act_dim > 0 ? mx_round_up(c->cent_act_dim, 4) : 0;
    W->cent_acts = tk(Mc * ca_ld); W->cent_nacts = tk(Mc * ca_ld);
  }
  W->total = o;
  return o * 4;
}

extern "C" int64_t mx_maddpg_workspace_bytes(const mx_maddpg_cfg* c) {
  if (maddpg_check(c)) return -1;
  MxNetLayout A, Cr;
  maddpg_layouts(c, &A, &Cr);
  MxMaddpgWs W;
  return maddpg_ws_layout(c, A.size, Cr.size, mx_num_sms(), &W);
}

extern "C" int mx_maddpg_create(const mx_maddpg_cfg* c, float* const actor_vecs[4], float* const critic_vecs[4], void* workspace,
                                int64_t workspace_bytes, mx_maddpg** out) {
  if (maddpg_check(c)) return 1;
  mx_maddpg* h = new mx_maddpg();
  h->cfg = *c;
  maddpg_layouts(c, &h->actor, &h->critic);
  h->Pa = h->actor.size; h->Pc = h->critic.size;
  h->npart = mx_num_sms();
  const int64_t need = maddpg_ws_layout(c, h->Pa, h->Pc, h->npart, &h->W);
  if (workspace_bytes < need) { mx_set_error("mx_maddpg_create: workspace %lld < %lld bytes", (long long)workspace_bytes, (long long)need); delete h; return 1; }
  h->th_a = actor_vecs[0]; h->th_a_tgt = actor_vecs[1]; h->m_a = actor_vecs[2]; h->v_a = actor_vecs[3];
  h->th_c = critic_vecs[0]; h->th_c_tgt = critic_vecs[1]; h->m_c = critic_vecs[2]; h->v_c = critic_vecs[3];
  h->ws = (float*)workspace;
  h->num_updates = 0;
  *out = h;
  return 0;
}
extern "C" void mx_maddpg_destroy(mx_maddpg* h) { delete h; }
extern "C" int mx_maddpg_set_valid(mx_maddpg* h, const float* valid_dev) {
  if (!h) { mx_set_error("mx_maddpg_set_valid: null handle"); return 1; }
  h->valid = valid_dev;
  return 0;
}
extern "C" const float* mx_maddpg_info(mx_maddpg* h) { return h->ws + h->W.info; }
extern "C" const float* mx_maddpg_priorities(mx_maddpg* h) { return h->ws + h->W.prio; }
extern "C" int mx_maddpg_grad_views(mx_maddpg* h, int64_t* actor_off_bytes, int64_t* critic_off_bytes) {
  *actor_off_bytes = h->W.grad_a * 4; *critic_off_bytes = h->W.grad_c * 4;
  return 0;
}

// =====================================================================================================
// step
// =====================================================================================================
static int launch1d(long long work) {
  long long g = (work + 255) / 256;
  const int cap = mx_num_sms() * 4;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

// kernel that only publishes the two loss scalars in the layout k_adam expects: grad[P+0] = denominator, [P+1] = loss numerator
__global__ void k_set_scalars(float* grad_tail, const float* scal) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    grad_tail[0] = scal[0]; grad_tail[1] = scal[1]; grad_tail[2] = 0.f; grad_tail[3] = scal[3];
  }
}

// The optimiser of one network in two halves around the data-parallel exchange: reduce_grads leaves the exchange payload grad[P+4]
// (k_grad_reduce: numerators, Adam step count bumped; k_set_scalars: the loss scalars behind them), apply_grads clips by the norm of that
// buffer and applies Adam (k_adam; normpart stays null, so the norm is always computed from the buffer, summed over the ranks or not).
// front_parts / head_parts: the gradient partials k_front_bwd and k_head_bwd wrote
static OptimArgs optim_args(mx_maddpg* h, bool actor, int front_parts, int head_parts) {
  const mx_maddpg_cfg& c = h->cfg;
  const MxNetLayout& L = actor ? h->actor : h->critic;
  const int64_t P = actor ? h->Pa : h->Pc;
  float* ws = h->ws;
  OptimArgs o;
  memset(&o, 0, sizeof(o));
  o.theta = actor ? h->th_a : h->th_c; o.theta_tgt = actor ? h->th_a_tgt : h->th_c_tgt;
  o.adam_m = actor ? h->m_a : h->m_c; o.adam_v = actor ? h->v_a : h->v_c;
  o.gpart = ws + (actor ? h->W.gpart_a : h->W.gpart_c); o.grad = ws + (actor ? h->W.grad_a : h->W.grad_c); o.P = P;
  o.nseg = 2;
  o.seg_begin[0] = 0; o.seg_end[0] = L.lno_g; o.seg_parts[0] = front_parts;
  o.seg_begin[1] = L.lno_g; o.seg_end[1] = (int)P; o.seg_parts[1] = head_parts;
  if (c.mlp) {        // every gradient comes from k_front_bwd; the critic's trained range stops at its trunk (the frozen heads follow it)
    o.nseg = 1;
    if (!actor) { o.P = L.wih; o.gpart_ld = P; o.seg_end[0] = L.wih; }
  }
  o.spart = ws + h->W.spart; o.spart_n = 0;
  o.info = ws + h->W.info + (actor ? 4 : 0);
  o.abort = ws + h->W.p2p_abort;
  o.adam_t = reinterpret_cast<double*>(ws + (actor ? h->W.adam_ta : h->W.adam_tc));
  o.err = nullptr; o.B = 0; o.T = 0; o.prio = nullptr;
  o.lr = c.lr; o.beta1 = c.adam_beta1; o.beta2 = c.adam_beta2; o.eps = c.adam_eps; o.max_grad_norm = c.max_grad_norm; o.tau = c.tau;
  o.weight_decay = c.weight_decay;
  return o;
}

static int reduce_grads(mx_maddpg* h, bool actor, int front_parts, int head_parts, cudaStream_t s) {
  const OptimArgs o = optim_args(h, actor, front_parts, head_parts);
  if (mx_launch_grad_reduce(o, s)) return 1;     // (its scalar block bumps the Adam step count; the loss scalars come from the loss kernel)
  return mx_launch("k_set_scalars", k_set_scalars, dim3(1), dim3(32), 0, s, MX_PLAIN, o.grad + o.P,
                   (const float*)(h->ws + (actor ? h->W.scal_a : h->W.scal_c)));
}

static int apply_grads(mx_maddpg* h, bool actor, cudaStream_t s) { return mx_launch_adam(optim_args(h, actor, 0, 0), s); }

// one network's exchange payload: what k_grad_reduce + k_set_scalars left, keyed to that network's own Adam step count
static MxP2pPayload p2p_payload(mx_maddpg* h, bool actor) {
  const OptimArgs o = optim_args(h, actor, 0, 0);
  MxP2pPayload pl;
  pl.grad = o.grad; pl.P = o.P; pl.adam_t = o.adam_t; pl.abort = h->ws + h->W.p2p_abort;
  return pl;
}

// with peers set (mx_maddpg_set_peers): push this rank's payload to every peer, then sum the world's in rank order; a no-op on one GPU
static int exchange(mx_maddpg* h, bool actor, cudaStream_t s) {
  const MxP2pPeers& peers = h->p2p[actor ? 0 : 1];
  if (peers.world < 2) return 0;
  const MxP2pPayload pl = p2p_payload(h, actor);
  if (mx_p2p_publish(peers, pl, MX_P2P_MAX_WORLD, s)) return 1;
  return mx_p2p_reduce(peers, pl, MX_P2P_MAX_WORLD, s);
}

// ---- the launches of one update: each builder fills its arguments from (network, pass) and the learner-wide settings; the phase lists
// below state only what differs between launches (copies of the network, row counts, h0, a data-gradient target, noise)
enum Net { ACTOR, CRITIC };
enum { LIVE = 1, TARGET = 2, BOTH = 3 };      // the copies of a network a forward runs; copy k uses slot k of the pass's regions

struct NetRef {             // one network of the learner
  const MxNetLayout& L;
  float* th[2];             // live, target parameters
  float* gpart;             // its gradient partials
  int64_t P;
};

struct Step {               // one call of learner h over batch b on stream s
  mx_maddpg* h;
  const mx_batch* b;
  cudaStream_t s;
  const mx_maddpg_cfg& c;
  const MxMaddpgWs& W;
  float* ws;
  Step(mx_maddpg* h_, const mx_batch* b_, cudaStream_t s_) : h(h_), b(b_), s(s_), c(h_->cfg), W(h_->W), ws(h_->ws) {}

  NetRef net(Net n) const {
    if (n == ACTOR) return {h->actor, {h->th_a, h->th_a_tgt}, ws + W.gpart_a, h->Pa};
    return {h->critic, {h->th_c, h->th_c_tgt}, ws + W.gpart_c, h->Pc};
  }
  int ldc() const { return mx_round_up(critic_in_dim(&c), 4); }
  int Ma() const { return b->B * (c.episode_len + 1) * c.n_agents; }      // actor rows

  // every front-layer launch of net n over pass p: input rows (actor: the batch's observations; critic: the pass's packed rows) and settings
  template <class Args> void front_common(Args& a, Net n, const MxPassWs& p) const {
    if (n == ACTOR) { a.X = b->obs; a.ldx = b->obs_ld; }
    else { a.X = ws + p.x; a.ldx = ldc(); }
    a.feature_norm = c.no_feature_norm ? 0 : 1; a.act_tanh = c.use_tanh;
    a.L = net(n).L;
  }

  // front layers of the copies `sel` of net n over the M rows of pass p; keep: also the live copy's activations, for a backward
  int front_fwd(Net n, const MxPassWs& p, int M, int sel, bool keep) const {
    const NetRef nr = net(n);
    FrontFwdArgs a;
    memset(&a, 0, sizeof(a));
    front_common(a, n, p);
    a.M = M;
    const int first = sel == TARGET ? 1 : 0, nets = sel == BOTH ? 2 : 1;
    for (int k = 0; k < nets; ++k) { a.theta[k] = nr.th[first + k]; a.gi[k] = ws + p.gi[first + k]; }
    if (keep) { a.u1 = ws + p.u1; a.u2 = ws + p.u2; a.st0 = ws + p.st0; a.st1 = ws + p.st1; a.st2 = ws + p.st2; }
    a.tc_acc = ws + W.tc_acc; a.tc_acc_cols = (int)W.tc_acc_cols;
    return mx_launch_front_fwd(a, nets, s);
  }

  // GRU of the copies `sel` of net n over pass p: R sequences of T+1 steps, N interleaved per step, starting from h0 (null: zeros)
  int gru_fwd(Net n, const MxPassWs& p, int sel, int R, int T, int N, const float* h0) const {
    const NetRef nr = net(n);
    GruFwdArgs a;
    memset(&a, 0, sizeof(a));
    const int first = sel == TARGET ? 1 : 0, nets = sel == BOTH ? 2 : 1;
    for (int k = 0; k < nets; ++k) { a.theta[k] = nr.th[first + k]; a.gi[k] = ws + p.gi[first + k]; a.hall[k] = ws + p.h[first + k]; }
    if (sel & LIVE) { a.gates = ws + p.gates; a.hn = ws + p.hn; }
    a.whh = nr.L.whh; a.bhh = nr.L.bhh; a.R = R; a.T = T; a.N = N; a.h0 = h0;
    return mx_launch_gru_fwd(a, nets, s);
  }

  // the head rows of net n: the actor's Linear(H, Ac) is contiguous; the critic's K Linear(H, 1) are (w_k, b_k) at stride H + 4 (maddpg_layouts)
  template <class Args> void head_rows(Args& a, Net n) const {
    const MxNetLayout& L = net(n).L;
    a.lno_g = L.lno_g; a.lno_b = L.lno_b; a.w = L.wq;
    if (n == ACTOR) { a.b = L.bq; a.OD = c.act_dim; a.b_stride = 1; a.w_stride = MX_H; }
    else { a.b = L.wq + MX_H; a.OD = c.num_q; a.b_stride = MX_H + 4; a.w_stride = MX_H + 4; }
  }

  // head of copy `sel` (LIVE or TARGET) of net n over the M rows of pass p (+ noise) into its out slot and / or the minimum into out_min
  int head_fwd(Net n, const MxPassWs& p, int sel, int M, const float* noise, float* out_min) const {
    const int k = sel == TARGET ? 1 : 0;
    HeadArgs a;
    memset(&a, 0, sizeof(a));
    head_rows(a, n);
    a.theta = net(n).th[k]; a.h = ws + p.h[k]; a.M = M;
    if (k == 0) a.sto = ws + p.sto;
    a.noise = noise; a.out = ws + p.out[k]; a.out_min = out_min;
    return mx_launch("k_head_fwd", k_head_fwd, dim3(launch1d((long long)M * 32)), dim3(256), 0, s, MX_PLAIN, a);
  }

  // back through the live head of net n over pass p, p.dout -> p.dh; parts: the gradient partials written, or null for a frozen head
  int head_bwd(Net n, const MxPassWs& p, int M, int* parts) const {
    const NetRef nr = net(n);
    const int grid = mx_imin_host(mx_num_sms(), mx_ceil_div(M, 32));
    HeadBwdArgs a;
    memset(&a, 0, sizeof(a));
    head_rows(a, n);
    a.theta = nr.th[0]; a.h = ws + p.h[0]; a.sto = ws + p.sto; a.dout = ws + p.dout; a.M = M; a.dh_out = ws + p.dh;
    a.gpart = parts ? nr.gpart : nullptr; a.P = nr.P;
    if (parts) *parts = grid;
    return mx_launch("k_head_bwd", k_head_bwd, dim3(grid), dim3(256), 0, s, MX_PLAIN, a);
  }

  // back through the live GRU of net n over pass p, p.dh -> p.dgi (R, T, N, T1, h0 as GruBwdArgs)
  int gru_bwd(Net n, const MxPassWs& p, int R, int T, int N, int T1, const float* h0) const {
    const NetRef nr = net(n);
    GruBwdArgs a;
    memset(&a, 0, sizeof(a));
    a.theta = nr.th[0]; a.whh = nr.L.whh; a.hall = ws + p.h[0]; a.gates = ws + p.gates; a.hn = ws + p.hn; a.dh_out = ws + p.dh;
    a.dgi = ws + p.dgi; a.R = R; a.T = T; a.N = N; a.T1 = T1; a.h0 = h0;
    return mx_launch_gru_bwd(a, s);
  }

  // back through the front layers (and GRU input weights) of the live net n over pass p from p.dgi.  dX null: a weight-gradient launch,
  // with the tensor-core scratch.  dX set: the frozen critic's data gradient only, which takes no tensor-core scratch (neither
  // tensor-core kernel computes a data gradient)
  int front_bwd(Net n, const MxPassWs& p, int M, int T, int N, int T1, const float* h0, float* dX, int* parts) const {
    const NetRef nr = net(n);
    FrontBwdArgs a;
    memset(&a, 0, sizeof(a));
    front_common(a, n, p);
    a.M = M; a.T = T; a.N = N; a.T1 = T1; a.h0 = h0; a.theta = nr.th[0];
    a.u1 = ws + p.u1; a.u2 = ws + p.u2; a.st0 = ws + p.st0; a.st1 = ws + p.st1; a.st2 = ws + p.st2; a.dgi = ws + p.dgi;
    if (c.mlp) a.no_gru = 1;
    else { a.gates = ws + p.gates; a.hall = ws + p.h[0]; }
    a.gpart = nr.gpart; a.P = nr.P;
    if (dX) {
      a.dX = dX; a.skip_wgrad = 1;
    } else {
      a.da2_out = ws + W.tc_da2; a.da1_out = ws + W.tc_da1; a.tc_imgT = ws + W.tc_imgT;
      a.tc_acc = ws + W.tc_acc; a.tc_acc_cols = (int)W.tc_acc_cols;
    }
    int unused = 0;
    return mx_launch_front_bwd(a, parts ? parts : &unused, s);
  }

  // the critic's input rows [s | actions] of one pass: mode 0 the buffer actions into c.x, 1 the target actions at the next step into
  // t.x, 2 the agent-replaced copies into r.x (the recurrent learner: with the critic state before each step)
  int pack_critic_in(int mode) const {
    PackArgs pk;
    memset(&pk, 0, sizeof(pk));
    pk.mode = mode; pk.B = b->B; pk.T = c.episode_len; pk.N = c.n_agents; pk.S = c.state_dim; pk.Ac = c.act_dim;
    pk.share = b->share; pk.share_ld = b->share_ld; pk.acts = b->acts; pk.act_ld = b->act_ld; pk.ldx = ldc();
    if (c.cent_act_dim > 0) {
      pk.CA = c.cent_act_dim; pk.off = c.act_offset; pk.ca_ld = mx_round_up(c.cent_act_dim, 4); pk.cent_acts = ws + W.cent_acts; pk.cent_nacts = ws + W.cent_nacts;
    }
    long long rows = (long long)b->B * c.episode_len;
    if (mode == 0) {
      pk.x = ws + W.c.x;
    } else if (mode == 1) {
      pk.x = ws + W.t.x; pk.actor_out = ws + W.a.out[1];
    } else {
      pk.x = ws + W.r.x; pk.actor_out = ws + (c.discrete ? W.a.act : W.a.out[0]);
      if (!c.mlp) { pk.hseq = ws + W.c.h[0]; pk.h0 = ws + W.r.h0; }
      rows *= c.n_agents;
    }
    return mx_launch("k_pack_critic_in", k_pack_critic_in, dim3(launch1d(rows * pk.ldx)), dim3(256), 0, s, MX_PLAIN, pk);
  }

  // Discrete actions of the actor rows: mode 0 arg-max one-hot, 1 hard Gumbel-softmax of logits (+ gumbel).  MultiDiscrete (n_act_seg
  // > 0, one segment included) takes no available-action mask (MADDPGPolicy.py:73-89); maddpg_check allows it on the MLP learner only
  int act_transform(int mode, const float* logits, const float* gumbel, float* out, float* soft) const {
    ActXformArgs ax;
    memset(&ax, 0, sizeof(ax));
    ax.M = Ma(); ax.Ac = c.act_dim; ax.mode = mode; ax.sg = act_segs(&c);
    ax.avail = c.n_act_seg > 0 ? nullptr : b->avail; ax.avail_ld = b->act_ld;
    ax.logits = logits; ax.gumbel = gumbel; ax.out = out; ax.soft = soft;
    return mx_launch("k_act_transform", k_act_transform, dim3(launch1d(Ma())), dim3(256), 0, s, MX_PLAIN, ax);
  }

  // d(critic input) of the agent-replaced copies -> the actor's head outputs: a.dout, or the MLP actor's "gi" gradient rows a.dgi
  int scatter_actor_grad() const {
    return mx_launch("k_scatter_actor_grad", k_scatter_actor_grad, dim3(launch1d(Ma())), dim3(256), 0, s, MX_PLAIN, (const float*)(ws + W.r.dx),
                     ldc(), b->B, c.episode_len, c.n_agents, c.state_dim, c.act_dim, (const float*)(c.discrete ? ws + W.a.soft : nullptr), ws + (c.mlp ? W.a.dgi : W.a.dout), c.act_offset,
           c.mlp ? (int)MX_G : c.act_dim, act_segs(&c));
  }

  // cfg.mlp: the head outputs in columns [0, OD) of the "gi" rows at offset gi (+ noise) into out and / or their minimum into out_min
  int mlp_head_cols(int64_t gi, int M, int OD, const float* noise, float* out, float* out_min) const {
    return mx_launch("k_mlp_head_cols", k_mlp_head_cols, dim3(launch1d(M)), dim3(256), 0, s, MX_PLAIN, (const float*)(ws + gi), M, OD, noise, out,
                     out_min);
  }

  // cfg.mlp: the gradient at the critic's head outputs p.dout as the "gi" gradient rows p.dgi that k_front_bwd reads
  int mlp_dgi_cols(const MxPassWs& p, int M) const {
    return mx_launch("k_mlp_dgi_cols", k_mlp_dgi_cols, dim3(launch1d((long long)M * MX_G)), dim3(256), 0, s, MX_PLAIN, (const float*)(ws + p.dout),
                     c.num_q, M, ws + p.dgi);
  }

  // TD target, critic loss, PER priorities: per sequence (recurrent) or the mean over the heads (MLP, maddpg.py:144: no per_nu)
  int critic_loss() const {
    const int T = c.episode_len, N = c.n_agents;
    CriticLossArgs cl;
    memset(&cl, 0, sizeof(cl));
    cl.B = b->B; cl.T = T; cl.N = N; cl.K = c.num_q; cl.ld_tn = b->ep_tn_ld > 0 ? b->ep_tn_ld : T * N; cl.ld_t = b->ep_t_ld > 0 ? b->ep_t_ld : T;
    cl.qpred = ws + W.c.out[0]; cl.qnext_min = ws + W.t.qmin; cl.rewards = b->rewards; cl.dones_env = b->dones_env;
    cl.weights = c.use_per ? b->weights : nullptr; cl.gamma = c.gamma; cl.huber_delta = c.huber_delta; cl.per_eps = c.per_eps;
    if (c.mlp) cl.prio_mean_k = 1;
    else cl.per_nu = c.per_nu;
    cl.use_huber = c.use_huber; cl.dq = ws + W.c.dout; cl.err = ws + W.c.err; cl.scal = ws + W.scal_c; cl.prio = c.use_per ? ws + W.prio : nullptr;
    return mx_launch("k_critic_loss", k_critic_loss, dim3(1), dim3(256), 0, s, MX_PLAIN, cl);
  }

  // actor loss through critic head 0 on the agent-replaced copies, masked by the agents' dones or (MLP) by valid_transition
  int actor_loss() const {
    const int T = c.episode_len, N = c.n_agents;
    ActorLossArgs al;
    memset(&al, 0, sizeof(al));
    al.B = b->B; al.T = T; al.N = N; al.K = c.num_q; al.ld_tn = b->ep_tn_ld > 0 ? b->ep_tn_ld : T * N; al.qa = ws + W.r.out[0]; al.dones = b->dones;
    if (c.mlp) { al.valid = h->valid; al.valid_idx = b->idx; }
    al.dout = ws + W.r.dout; al.scal = ws + W.scal_a;
    return mx_launch("k_actor_loss", k_actor_loss, dim3(1), dim3(256), 0, s, MX_PLAIN, al);
  }

  // The actor's copies `sel` over its rows Ma = B*(T+1)*N; the target copy's head (+ MATD3 noise) gives the target actions a.out[1],
  // for Discrete actions arg-max one-hot with the next-avail mask (MADDPG) / a hard Gumbel-softmax sample (MATD3; the head added the
  // draw).  The MLP actor's live head runs in its step's actor phase.
  int actor_fwd(int sel, const float* target_noise_dev) const {
    const int B = b->B, T = c.episode_len, N = c.n_agents;
    if (front_fwd(ACTOR, W.a, Ma(), sel, (sel & LIVE) != 0)) return 1;
    if (!c.mlp) {
      if (gru_fwd(ACTOR, W.a, sel, B * N, T, N, nullptr)) return 1;
      if ((sel & LIVE) && head_fwd(ACTOR, W.a, LIVE, Ma(), nullptr, nullptr)) return 1;
    }
    if (!(sel & TARGET)) return 0;
    const float* noise = c.target_noise > 0.f ? target_noise_dev : nullptr;
    // cfg.mlp (maddpg.py:64-74): the head sits in the weight_ih slot; the noise rows are the step-1 (next-observation) rows [b][2][N][Ac]
    if (c.mlp ? mlp_head_cols(W.a.gi[1], Ma(), c.act_dim, noise, ws + W.a.out[1], nullptr) : head_fwd(ACTOR, W.a, TARGET, Ma(), noise, nullptr))
      return 1;
    if (c.discrete) return act_transform(c.target_noise > 0.f ? 1 : 0, ws + W.a.out[1], nullptr, ws + W.a.out[1], nullptr);
    return 0;
  }
};
// ---- recurrent learner: shared_train_policy_on_batch (r_maddpg.py:114-331) ------------------------------------------------------------
// Several policies (cent_act_dim > 0): the centralised action vectors were assembled by mx_maddpg_cent_contribute.
// Two halves around the critic's Adam step: critic_grads_rnn (A-E) leaves the critic's exchange payload, actor_grads_rnn (F) reads the
// critic after that step and leaves the actor's.
static int critic_grads_rnn(const Step& st, const float* target_noise_dev) {
  const MxMaddpgWs& W = st.W;
  float* ws = st.ws;
  const int B = st.b->B, T = st.c.episode_len, Mc = B * T;

  // ---------- A. actor: live + target over the T+1 steps ----------
  if (st.actor_fwd(BOTH, target_noise_dev)) return 1;

  // ---------- B. critic over the buffer sequence (live + target) ----------
  if (st.pack_critic_in(0)) return 1;
  if (st.front_fwd(CRITIC, W.c, Mc, BOTH, true)) return 1;
  if (st.gru_fwd(CRITIC, W.c, BOTH, B, T - 1, 1, nullptr)) return 1;
  if (st.head_fwd(CRITIC, W.c, LIVE, Mc, nullptr, nullptr)) return 1;

  // ---------- C. target Q: one branch step per (b,t) from the target critic's buffer state ----------
  if (st.pack_critic_in(1)) return 1;
  if (st.front_fwd(CRITIC, W.t, Mc, TARGET, false)) return 1;
  if (st.gru_fwd(CRITIC, W.t, TARGET, Mc, 0, 1, ws + W.c.h[1])) return 1;
  if (st.head_fwd(CRITIC, W.t, TARGET, Mc, nullptr, ws + W.t.qmin)) return 1;

  // ---------- D. TD target, critic loss ----------
  if (st.critic_loss()) return 1;

  // ---------- E. critic backward + Adam ----------
  int head_parts = 0, parts = 0;
  if (st.head_bwd(CRITIC, W.c, Mc, &head_parts)) return 1;
  if (st.gru_bwd(CRITIC, W.c, B, T, 1, T, nullptr)) return 1;
  if (st.front_bwd(CRITIC, W.c, Mc, T, 1, T, nullptr, nullptr, &parts)) return 1;
  return reduce_grads(st.h, false, parts, head_parts, st.s);
}

static int actor_grads_rnn(const Step& st, const float* actor_noise_dev) {
  const MxMaddpgWs& W = st.W;
  float* ws = st.ws;
  const int B = st.b->B, T = st.c.episode_len, N = st.c.n_agents;
  const int Ma = B * (T + 1) * N, Mc = B * T, Mr = N * B * T;

  // ---------- F. actor update with the UPDATED critic ----------
  // live critic recurrence over the buffer sequence again (its parameters just changed)
  if (st.front_fwd(CRITIC, W.c, Mc, LIVE, false)) return 1;
  if (st.gru_fwd(CRITIC, W.c, LIVE, B, T - 1, 1, nullptr)) return 1;
  // the live actor's hard Gumbel-softmax sample (straight-through), r_maddpg.py:277
  if (st.c.discrete && st.act_transform(1, ws + W.a.out[0], actor_noise_dev, ws + W.a.act, ws + W.a.soft)) return 1;
  if (st.pack_critic_in(2)) return 1;
  if (st.front_fwd(CRITIC, W.r, Mr, LIVE, true)) return 1;
  if (st.gru_fwd(CRITIC, W.r, LIVE, Mr, 0, 1, ws + W.r.h0)) return 1;
  if (st.head_fwd(CRITIC, W.r, LIVE, Mr, nullptr, nullptr)) return 1;
  if (st.actor_loss()) return 1;
  // back through the (frozen) critic to its action inputs
  if (st.head_bwd(CRITIC, W.r, Mr, nullptr)) return 1;
  if (st.gru_bwd(CRITIC, W.r, Mr, 1, 1, 1, ws + W.r.h0)) return 1;
  if (st.front_bwd(CRITIC, W.r, Mr, 0, 1, 1, ws + W.r.h0, ws + W.r.dx, nullptr)) return 1;
  if (st.scatter_actor_grad()) return 1;
  // actor backward + Adam
  int ahead_parts = 0, aparts = 0;
  if (st.head_bwd(ACTOR, W.a, Ma, &ahead_parts)) return 1;
  if (st.gru_bwd(ACTOR, W.a, B * N, T, N, T + 1, nullptr)) return 1;
  if (st.front_bwd(ACTOR, W.a, Ma, T, N, 0, nullptr, nullptr, &aparts)) return 1;
  return reduce_grads(st.h, true, aparts, ahead_parts, st.s);
}

// ---- cfg.mlp: shared_train_policy_on_batch of the transition-level trainer (maddpg.py:90-249) ---------------------------------------
// A batch is B transitions stored as episodes of length 1: obs rows m = (b*2 + t)*N + n with t = 0 the observation and t = 1 the next
// observation, so the recurrent path's critic-input packing serves unchanged (mode 0: (s, a), mode 1: (s', a'), mode 2: the N
// agent-replaced copies).  No recurrence: every net is the front kernel with its head in the weight_ih slot, and k_front_bwd runs
// with no_gru.  The critic's heads are frozen (not in the reference's parameters()): the live heads give Q(s, a) and, in the actor
// phase, the gradient path into the actor; the target heads give Q'(s', a').
// Several policies (cent_act_dim > 0): the centralised action vectors were assembled by mx_maddpg_cent_contribute, so the step runs
// only the live actor and never reads its own target actions; the batch is this policy's (rewards, dones_env, shared observation,
// PER weights, maddpg.py:103-107) and the valid_transition store is this policy's [rows][n_agents].
static int critic_grads_mlp(const Step& st, const float* target_noise_dev) {
  const MxMaddpgWs& W = st.W;
  float* ws = st.ws;
  const int Mc = st.b->B, K = st.c.num_q;

  // ---------- A. live + target actor on obs and next_obs; target actions a' from the next_obs rows (maddpg.py:64-74) ----------
  if (st.actor_fwd(st.c.cent_act_dim > 0 ? LIVE : BOTH, target_noise_dev)) return 1;

  // ---------- B. live critic on (s, a), target critic on (s', a'); TD target, loss, priorities (maddpg.py:112-151) ----------
  if (st.pack_critic_in(0)) return 1;
  if (st.pack_critic_in(1)) return 1;
  if (st.front_fwd(CRITIC, W.c, Mc, LIVE, true)) return 1;
  if (st.front_fwd(CRITIC, W.t, Mc, TARGET, false)) return 1;
  if (st.mlp_head_cols(W.c.gi[0], Mc, K, nullptr, ws + W.c.out[0], nullptr)) return 1;
  if (st.mlp_head_cols(W.t.gi[1], Mc, K, nullptr, nullptr, ws + W.t.qmin)) return 1;
  if (st.critic_loss()) return 1;

  // ---------- C. critic backward through the frozen live heads into the trunk; clip + Adam over the trunk ----------
  if (st.mlp_dgi_cols(W.c, Mc)) return 1;
  int parts = 0;
  if (st.front_bwd(CRITIC, W.c, Mc, 1, 1, 0, nullptr, nullptr, &parts)) return 1;
  return reduce_grads(st.h, false, parts, 0, st.s);
}

static int actor_grads_mlp(const Step& st, const float* actor_noise_dev) {
  const MxMaddpgWs& W = st.W;
  float* ws = st.ws;
  const int B = st.b->B, N = st.c.n_agents, K = st.c.num_q, Ac = st.c.act_dim;
  const int Ma = B * 2 * N, Mr = N * B;

  // ---------- D. actor loss through head 0 of the UPDATED critic on the agent-replaced copies, masked by valid_transition ----------
  if (st.mlp_head_cols(W.a.gi[0], Ma, Ac, nullptr, ws + W.a.out[0], nullptr)) return 1;
  // get_actions(obs, avail, use_gumbel=True): hard Gumbel-softmax, straight-through (maddpg.py:209)
  if (st.c.discrete && st.act_transform(1, ws + W.a.out[0], actor_noise_dev, ws + W.a.act, ws + W.a.soft)) return 1;
  if (st.pack_critic_in(2)) return 1;
  if (st.front_fwd(CRITIC, W.r, Mr, LIVE, true)) return 1;
  if (st.mlp_head_cols(W.r.gi[0], Mr, K, nullptr, ws + W.r.out[0], nullptr)) return 1;
  if (st.actor_loss()) return 1;
  // back through the frozen critic (trunk and live head 0) to its action inputs, then into the actor's head rows
  if (st.mlp_dgi_cols(W.r, Mr)) return 1;
  if (st.front_bwd(CRITIC, W.r, Mr, 1, 1, 0, nullptr, ws + W.r.dx, nullptr)) return 1;
  if (st.scatter_actor_grad()) return 1;
  int aparts = 0;
  if (st.front_bwd(ACTOR, W.a, Ma, 1, N, 0, nullptr, nullptr, &aparts)) return 1;
  return reduce_grads(st.h, true, aparts, 0, st.s);
}

extern "C" int mx_maddpg_step(mx_maddpg* h, const mx_batch* b, const float* target_noise_dev, int32_t* update_actor_out, void* stream) {
  return mx_maddpg_step_ex(h, b, target_noise_dev, nullptr, update_actor_out, stream);
}

// the checks every update makes before its first launch, and whether it trains the actor
static int check_step(mx_maddpg* h, const mx_batch* b, const float* target_noise_dev, const float* actor_noise_dev, bool* update_actor) {
  const mx_maddpg_cfg& c = h->cfg;
  if (!b || b->B <= 0 || b->B > c.max_batch) { mx_set_error("maddpg step: batch size outside [1, max_batch=%d]", c.max_batch); return 1; }
  if (!b->obs || !b->share || !b->acts || !b->rewards || !b->dones || !b->dones_env) { mx_set_error("maddpg step: missing batch field"); return 1; }
  if (c.use_per && !b->weights) { mx_set_error("maddpg step: use_per set but batch has no importance weights"); return 1; }
  if (c.target_noise > 0.f && !target_noise_dev) { mx_set_error("maddpg step: MATD3 target noise expected"); return 1; }
  *update_actor = h->force_update_actor >= 0 ? h->force_update_actor != 0
                                             : (h->num_updates % (c.actor_update_interval > 0 ? c.actor_update_interval : 1)) == 0;
  if (c.discrete && *update_actor && !actor_noise_dev) { mx_set_error("maddpg step: discrete actor update needs the Gumbel draws (actor_noise_dev)"); return 1; }
  if (h->phase_next) { mx_set_error("maddpg step: a phased update (mx_maddpg_step_phase) is in progress, next phase %d", h->phase_next); return 1; }
  return 0;
}

static int critic_grads(const Step& st, const float* target_noise_dev) {
  return (st.c.mlp ? critic_grads_mlp : critic_grads_rnn)(st, target_noise_dev);
}
static int actor_grads(const Step& st, const float* actor_noise_dev) {
  return (st.c.mlp ? actor_grads_mlp : actor_grads_rnn)(st, actor_noise_dev);
}

// critic grads -> [exchange] -> critic Adam -> actor grads (through the updated critic) -> [exchange] -> actor Adam; the exchanges run
// only with peers set, so one GPU launches exactly the kernels of the undivided update
extern "C" int mx_maddpg_step_ex(mx_maddpg* h, const mx_batch* b, const float* target_noise_dev, const float* actor_noise_dev,
                                 int32_t* update_actor_out, void* stream) {
#if !MX_EMU
  g_mx_pdl_auto = 1;      // ~40 small dependent launches per update: programmatic dependent launch measured 491 -> 469 us (R-MADDPG), 372 -> 355 us (R-MATD3)
#endif
  bool update_actor = false;
  if (check_step(h, b, target_noise_dev, actor_noise_dev, &update_actor)) return 1;
  const Step st(h, b, (cudaStream_t)stream);
  if (critic_grads(st, target_noise_dev) || exchange(h, false, st.s) || apply_grads(h, false, st.s)) return 1;
  if (update_actor && (actor_grads(st, actor_noise_dev) || exchange(h, true, st.s) || apply_grads(h, true, st.s))) return 1;
  if (update_actor_out) *update_actor_out = update_actor ? 1 : 0;
  if (h->force_update_actor < 0) h->num_updates += 1;      // (graph replays count in mx_graph_launch)
  return 0;
}

// One update as four calls, the exchanges left to the caller between them (an all-reduce of mx_maddpg_grad_buffer, or
// mx_maddpg_p2p_publish / _reduce): MX_MADDPG_CRITIC_GRADS decides whether the update trains the actor; MX_MADDPG_CRITIC_APPLY ends an
// update that does not; MX_MADDPG_ACTOR_GRADS / _APPLY follow otherwise.  Same launches as mx_maddpg_step_ex without its exchanges.
extern "C" int mx_maddpg_step_phase(mx_maddpg* h, int32_t phase, const mx_batch* b, const float* target_noise_dev, const float* actor_noise_dev,
                                    int32_t* update_actor_out, void* stream) {
  if (!h) { mx_set_error("mx_maddpg_step_phase: null handle"); return 1; }
  if (phase < MX_MADDPG_CRITIC_GRADS || phase > MX_MADDPG_ACTOR_APPLY) { mx_set_error("mx_maddpg_step_phase: phase %d outside [0, 3]", phase); return 1; }
  if (phase != h->phase_next) {
    mx_set_error("mx_maddpg_step_phase: phase %d out of order, the update in progress expects phase %d", phase, h->phase_next); return 1;
  }
#if !MX_EMU
  g_mx_pdl_auto = 1;
#endif
  const cudaStream_t s = (cudaStream_t)stream;
  bool done = false;
  if (phase == MX_MADDPG_CRITIC_GRADS) {
    bool update_actor = false;
    if (check_step(h, b, target_noise_dev, actor_noise_dev, &update_actor)) return 1;
    if (critic_grads(Step(h, b, s), target_noise_dev)) return 1;
    h->phase_actor = update_actor;
    h->phase_next = MX_MADDPG_CRITIC_APPLY;
  } else if (phase == MX_MADDPG_CRITIC_APPLY) {
    if (apply_grads(h, false, s)) return 1;
    h->phase_next = h->phase_actor ? MX_MADDPG_ACTOR_GRADS : 0;
    done = !h->phase_actor;
  } else if (phase == MX_MADDPG_ACTOR_GRADS) {
    if (!b || b->B <= 0 || b->B > h->cfg.max_batch) { mx_set_error("mx_maddpg_step_phase: the actor phase needs the update's batch"); return 1; }
    if (actor_grads(Step(h, b, s), actor_noise_dev)) return 1;
    h->phase_next = MX_MADDPG_ACTOR_APPLY;
  } else {
    if (apply_grads(h, true, s)) return 1;
    h->phase_next = 0;
    done = true;
  }
  if (update_actor_out) *update_actor_out = h->phase_actor ? 1 : 0;
  if (done && h->force_update_actor < 0) h->num_updates += 1;
  return 0;
}

// ---- data parallel: the two exchange payloads over peer memory (p2p.cu) -------------------------------------------------------------
static bool net_ok(const char* who, const mx_maddpg* h, int32_t net) {
  if (!h) { mx_set_error("%s: null handle", who); return false; }
  if (net != MX_MADDPG_ACTOR && net != MX_MADDPG_CRITIC) { mx_set_error("%s: net %d is neither MX_MADDPG_ACTOR (0) nor MX_MADDPG_CRITIC (1)", who, net); return false; }
  return true;
}
extern "C" int64_t mx_maddpg_p2p_block_bytes(mx_maddpg* h, int32_t net) {
  if (!net_ok("mx_maddpg_p2p_block_bytes", h, net)) return -1;
  return mx_p2p_block_floats(p2p_payload(h, net == MX_MADDPG_ACTOR).P, MX_P2P_MAX_WORLD) * 4;
}
extern "C" int mx_maddpg_set_peers(mx_maddpg* h, int32_t net, int32_t rank, int32_t world, void* const* peer_blocks, uint32_t* counter_dev) {
  if (!net_ok("mx_maddpg_set_peers", h, net)) return 1;
  MxP2pPeers peers;
  if (mx_p2p_set_peers("mx_maddpg_set_peers", &peers, rank, world, peer_blocks, counter_dev)) return 1;
  const MxP2pPeers& other = h->p2p[net == MX_MADDPG_ACTOR ? 1 : 0];
  if (other.world && (other.world != world || other.rank != rank)) {
    mx_set_error("mx_maddpg_set_peers: rank %d / world %d differ from the other network's %d / %d", rank, world, other.rank, other.world);
    return 1;
  }
  for (int p = 0; p < world; ++p)
    if (peers.blocks[p] == other.blocks[p] || (p > 0 && peers.blocks[p] == peers.blocks[0])) {
      mx_set_error("mx_maddpg_set_peers: block %d is shared with another network or rank; each network of each rank needs its own", p); return 1;
    }
  if (counter_dev == other.counter) { mx_set_error("mx_maddpg_set_peers: each network needs its own arrival counter"); return 1; }
  h->p2p[net == MX_MADDPG_ACTOR ? 0 : 1] = peers;
  return 0;
}
static int p2p_call(const char* who, mx_maddpg* h, int32_t net, void* stream, bool publish) {
  if (!net_ok(who, h, net)) return 1;
  const bool actor = net == MX_MADDPG_ACTOR;
  const MxP2pPeers& peers = h->p2p[actor ? 0 : 1];
  if (!peers.world) { mx_set_error("%s: mx_maddpg_set_peers was not called for net %d", who, net); return 1; }
  const MxP2pPayload pl = p2p_payload(h, actor);
  return (publish ? mx_p2p_publish : mx_p2p_reduce)(peers, pl, MX_P2P_MAX_WORLD, (cudaStream_t)stream);
}
extern "C" int mx_maddpg_p2p_publish(mx_maddpg* h, int32_t net, void* stream) { return p2p_call("mx_maddpg_p2p_publish", h, net, stream, true); }
extern "C" int mx_maddpg_p2p_reduce(mx_maddpg* h, int32_t net, void* stream) { return p2p_call("mx_maddpg_p2p_reduce", h, net, stream, false); }
extern "C" float* mx_maddpg_grad_buffer(mx_maddpg* h, int32_t net, int64_t* n_floats) {
  if (!net_ok("mx_maddpg_grad_buffer", h, net)) return nullptr;
  const MxP2pPayload pl = p2p_payload(h, net == MX_MADDPG_ACTOR);
  if (n_floats) *n_floats = pl.P + 4;
  return pl.grad;
}

// ---- several policies (share_policy = False, scripts/train_mpe_rmaddpg.sh:14 -> train/train_mpe.py:139-150) ------------------------------
// The reference's update of policy p (r_maddpg.py:114-331) calls get_update_info (r_maddpg.py:40-105), which walks over EVERY policy q:
// buffer actions of q's agents, and next actions from q's TARGET actor on q's own observation sequence; concatenated over all agents
// they form the centralised action vectors the critic of p consumes.  Here every policy owns one mx_maddpg (its agents, its obs /
// action widths, the shared centralised observation) with cfg.cent_act_dim = total action width and cfg.act_offset = where its agents sit.
// mx_maddpg_cent_contribute(src, src_batch, noise, dst): src's target actor over src_batch (T+1 steps, Gaussian / Gumbel noise and the
// Discrete transforms exactly as in the single-policy step), then src's slices of the two assembled vectors are written into dst's
// workspace.  Call it for every policy (dst = the policy about to be updated, itself included), then mx_maddpg_step_ex(dst, ...).
__global__ void __launch_bounds__(256) k_cent_scatter(const float* __restrict__ nact, const float* __restrict__ acts, int act_ld, int B, int T, int N, int Ac,
                                                      float* __restrict__ cent_acts, float* __restrict__ cent_nacts, int ca_ld, int off) {
  const long long total = (long long)B * T * N * Ac;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(idx % Ac);
    const long long r = idx / Ac;
    const int n = (int)(r % N);
    const long long bt = r / N;
    const int t = (int)(bt % T), b = (int)(bt / T);
    const size_t dst = ((size_t)b * T + t) * ca_ld + off + n * Ac + k;
    cent_acts[dst] = acts[(((size_t)b * T + t) * N + n) * act_ld + k];
    cent_nacts[dst] = nact[(((size_t)b * (T + 1) + t + 1) * N + n) * Ac + k];          // the target actor's action at the NEXT step
  }
}

extern "C" int mx_maddpg_cent_contribute(mx_maddpg* src, const mx_batch* b, const float* target_noise_dev, mx_maddpg* dst, void* stream) {
  if (!src || !dst || !b) { mx_set_error("mx_maddpg_cent_contribute: null argument"); return 1; }
  const mx_maddpg_cfg& c = src->cfg;
  const mx_maddpg_cfg& d = dst->cfg;
  if (c.cent_act_dim <= 0 || d.cent_act_dim != c.cent_act_dim || d.episode_len != c.episode_len || d.mlp != c.mlp) {
    mx_set_error("mx_maddpg_cent_contribute: both learners need the same cent_act_dim > 0, episode length and mlp flag"); return 1;
  }
  if (b->B <= 0 || b->B > c.max_batch || b->B > d.max_batch) { mx_set_error("mx_maddpg_cent_contribute: batch size outside [1, max_batch]"); return 1; }
  if (!b->obs || !b->acts) { mx_set_error("mx_maddpg_cent_contribute: missing batch field"); return 1; }
  if (c.target_noise > 0.f && !target_noise_dev) { mx_set_error("mx_maddpg_cent_contribute: MATD3 target noise expected"); return 1; }
  cudaStream_t s = (cudaStream_t)stream;
  if (Step(src, b, s).actor_fwd(TARGET, target_noise_dev)) return 1;
  // cfg.mlp: k_cent_scatter's row (b*(T+1)+t+1)*N+n with T = 1, t = 0 is the next-observation step the target actor ran on
  const int B = b->B, T = c.episode_len, N = c.n_agents, Ac = c.act_dim;
  return mx_launch("k_cent_scatter", k_cent_scatter, dim3(launch1d((long long)B * T * N * Ac)), dim3(256), 0, s, MX_PLAIN,
                   (const float*)(src->ws + src->W.a.out[1]), b->acts, b->act_ld, B, T, N, Ac, dst->ws + dst->W.cent_acts, dst->ws + dst->W.cent_nacts,
                   mx_round_up(d.cent_act_dim, 4), c.act_offset);
}

// The noise fills a capture puts in its graph: refused before the capture rather than half-way through it.
static int check_fills(const char* who, const uint32_t* state_dev, const mx_trng_draw* fills, int32_t n_fills, const uint32_t* scratch_dev,
                       int64_t scratch_words) {
  if (n_fills < 0 || (n_fills > 0 && (!fills || !state_dev || !scratch_dev))) {
    mx_set_error("%s: %d fills need the fills, the generator state and the scratch", who, n_fills); return 1;
  }
  for (int32_t i = 0; i < n_fills; ++i) {
    const int64_t w = mx_trng_words(&fills[i]);
    if (w < 0) return 1;
    if (w > scratch_words) { mx_set_error("%s: scratch of %lld words, fill %d consumes %lld", who, (long long)scratch_words, i, (long long)w); return 1; }
  }
  return 0;
}

// [sample ->] shared_train_policy_on_batch [-> PER write-back] [-> soft update] as one CUDA graph.  The actor is updated only
// every actor_update_interval-th call, so the caller records one graph per variant (update_actor = 1 / 0) and replays the one
// the update counter asks for; the noise buffers are fixed device buffers the caller refills before each launch.
extern "C" int mx_maddpg_graph_capture(mx_replay* r, mx_maddpg* h, int32_t B, double beta, uint32_t flags, const float* target_noise_dev,
                                       const float* actor_noise_dev, int32_t update_actor, void* stream, mx_graph** out) {
  return mx_maddpg_graph_capture_ex(r, h, B, beta, flags, target_noise_dev, actor_noise_dev, update_actor, nullptr, nullptr, 0, nullptr, 0,
                                    stream, out);
}
// The same graph headed by the update's noise fills (torch_rng.cu): no host draw and no copy per replay.
extern "C" int mx_maddpg_graph_capture_ex(mx_replay* r, mx_maddpg* h, int32_t B, double beta, uint32_t flags, const float* target_noise_dev,
                                          const float* actor_noise_dev, int32_t update_actor, uint32_t* state_dev, const mx_trng_draw* fills,
                                          int32_t n_fills, uint32_t* scratch_dev, int64_t scratch_words, void* stream, mx_graph** out) {
  if (!r || !h || !out) { mx_set_error("mx_maddpg_graph_capture: null argument"); return 1; }
  if (h->cfg.cent_act_dim > 0) {      // the graph would replay the step without the other policies' contributions
    mx_set_error("mx_maddpg_graph_capture: a learner of several policies (cent_act_dim > 0) cannot be captured alone: its step needs "
                 "mx_maddpg_cent_contribute from every policy first; capture the whole batch_train with mx_maddpg_batch_graph_capture");
    return 1;
  }
  if (check_fills("mx_maddpg_graph_capture_ex", state_dev, fills, n_fills, scratch_dev, scratch_words)) return 1;
  std::vector<mx_trng_draw> fl(fills, fills + n_fills);
  if ((flags & 2u) && mx_replay_set_beta(r, beta, stream)) return 1;
  auto seq = [=](void* st) -> int {
    for (const mx_trng_draw& f : fl)
      if (mx_trng_fill(state_dev, &f, scratch_dev, scratch_words, st)) return 1;
    if (flags & 1u) { if (mx_replay_sample_uniform(r, B, st)) return 1; }
    else if (flags & 2u) { if (mx_replay_sample_per_state_beta(r, B, st)) return 1; }      // exponent: device scalar (mx_replay_set_beta)
    mx_batch b;
    if (mx_replay_batch(r, B, &b)) return 1;
    h->force_update_actor = update_actor ? 1 : 0;
    const int rc = mx_maddpg_step_ex(h, &b, target_noise_dev, actor_noise_dev, nullptr, st);
    h->force_update_actor = -1;
    if (rc) return 1;
    if (flags & 8u) { if (mx_replay_update_priorities(r, b.idx, mx_maddpg_priorities(h), nullptr, nullptr, B, st)) return 1; }
    if ((flags & 4u) && update_actor) { if (mx_maddpg_soft_update(h, st)) return 1; }      // base_runner.py:250-252
    return 0;
  };
  return mx_graph_capture_seq(seq, [h]() { h->num_updates += 1; }, stream, out);
}

// Several policies: one batch_train of the runner (runner/{rnn,mlp}/base_runner.py batch_train) as one CUDA graph.  Per policy p in id
// order: p's noise fills; the sample (uniform: one draw on stores[uniform_store], PER: p's tree) gathered into every other store;
// mx_maddpg_cent_contribute of every policy q into p; the step of p; the write-back to p's tree.  Then, when the actor was updated,
// the soft updates of all P policies.  The eager trainer does the same launches in the same order (MaddpgTrainer
// .shared_train_policy_on_batch), so a replay computes what an eager batch_train computes, bit for bit.
extern "C" int mx_maddpg_batch_graph_capture(mx_replay* const* stores, mx_maddpg* const* learners, int32_t P, int32_t uniform_store, int32_t B,
                                             double beta, uint32_t flags, const float* const* target_noise_dev,
                                             const float* const* actor_noise_dev, int32_t update_actor, uint32_t* state_dev,
                                             const mx_trng_draw* fills, const int32_t* fill_counts, uint32_t* scratch_dev,
                                             int64_t scratch_words, void* stream, mx_graph** out) {
  static const char* who = "mx_maddpg_batch_graph_capture";
  if (!stores || !learners || !target_noise_dev || !actor_noise_dev || !out) { mx_set_error("%s: null argument", who); return 1; }
  if (P < 2) { mx_set_error("%s: %d policies; one shared policy is captured by mx_maddpg_graph_capture_ex", who, P); return 1; }
  if ((flags & 1u) && (uniform_store < 0 || uniform_store >= P)) { mx_set_error("%s: uniform_store %d outside [0, %d)", who, uniform_store, P); return 1; }
  for (int32_t p = 0; p < P; ++p)
    if (!stores[p] || !learners[p]) { mx_set_error("%s: store or learner %d is null", who, p); return 1; }
  // the learners form one policy set: same centralised action width, episode length and kind, act_offsets tiling cent_act_dim in order
  const mx_maddpg_cfg& c0 = learners[0]->cfg;
  int32_t off = 0;
  for (int32_t p = 0; p < P; ++p) {
    const mx_maddpg_cfg& c = learners[p]->cfg;
    if (c.cent_act_dim <= 0 || c.cent_act_dim != c0.cent_act_dim || c.episode_len != c0.episode_len || c.mlp != c0.mlp) {
      mx_set_error("%s: learner %d (cent_act_dim %d, episode length %d, mlp %d) is not of one policy set with learner 0 (%d, %d, %d; "
                   "cent_act_dim > 0)", who, p, c.cent_act_dim, c.episode_len, c.mlp, c0.cent_act_dim, c0.episode_len, c0.mlp);
      return 1;
    }
    if (B <= 0 || B > c.max_batch) { mx_set_error("%s: batch size %d outside [1, max_batch=%d] of learner %d", who, B, c.max_batch, p); return 1; }
    if (c.act_offset != off) {
      mx_set_error("%s: learner %d has act_offset %d, expected %d: the learners are not in policy-id order or not one policy set", who, p,
                   c.act_offset, off);
      return 1;
    }
    off += c.n_agents * c.act_dim;
    const mx_replay_cfg& r = stores[p]->cfg;
    if (r.n_agents != c.n_agents || r.obs_dim != c.obs_dim || r.act_dim != c.act_dim || r.share_dim != c.state_dim || r.episode_len != c.episode_len) {
      mx_set_error("%s: store %d (agents %d, obs %d, act %d, share %d, episode %d) does not hold the batches of learner %d (%d, %d, %d, %d, %d)",
                   who, p, r.n_agents, r.obs_dim, r.act_dim, r.share_dim, r.episode_len, p, c.n_agents, c.obs_dim, c.act_dim, c.state_dim,
                   c.episode_len);
      return 1;
    }
    if (B > r.max_batch) { mx_set_error("%s: batch size %d > max_batch=%d of store %d", who, B, r.max_batch, p); return 1; }
    if ((flags & 2u) && (!r.use_per || !c.use_per)) { mx_set_error("%s: PER sampling needs use_per in store and learner %d", who, p); return 1; }
  }
  if (off != c0.cent_act_dim) { mx_set_error("%s: the %d learners' action widths sum to %d, cent_act_dim is %d", who, P, off, c0.cent_act_dim); return 1; }
  std::vector<std::vector<mx_trng_draw>> fl(P);
  for (int32_t p = 0, first = 0; p < P; first += fl[p].size(), ++p) {
    const int32_t n = fill_counts ? fill_counts[p] : 0;
    if (check_fills(who, state_dev, fills + first, n, scratch_dev, scratch_words)) return 1;
    fl[p].assign(fills + first, fills + first + n);
  }
  const std::vector<mx_replay*> R(stores, stores + P);
  const std::vector<mx_maddpg*> H(learners, learners + P);
  const std::vector<const float*> tn(target_noise_dev, target_noise_dev + (size_t)P * P), an(actor_noise_dev, actor_noise_dev + P);
  if (flags & 2u)
    for (mx_replay* r : R)
      if (mx_replay_set_beta(r, beta, stream)) return 1;
  auto seq = [=](void* st) -> int {
    std::vector<mx_batch> b(P);
    for (int32_t p = 0; p < P; ++p) {
      for (const mx_trng_draw& f : fl[p])
        if (mx_trng_fill(state_dev, &f, scratch_dev, scratch_words, st)) return 1;
      if (flags & 3u) {      // one index set for every store (rec_buffer.py:76-80,291-299, mlp_buffer.py:100-106,288-296)
        mx_replay* src = (flags & 1u) ? R[uniform_store] : R[p];
        if ((flags & 1u) ? mx_replay_sample_uniform(src, B, st) : mx_replay_sample_per_state_beta(src, B, st)) return 1;
        mx_batch sb;
        if (mx_replay_batch(src, B, &sb)) return 1;
        for (mx_replay* r : R)
          if (r != src && mx_replay_gather(r, sb.idx, B, st)) return 1;
      }
      for (int32_t q = 0; q < P; ++q)
        if (mx_replay_batch(R[q], B, &b[q])) return 1;
      for (int32_t q = 0; q < P; ++q)
        if (mx_maddpg_cent_contribute(H[q], &b[q], tn[(size_t)p * P + q], H[p], st)) return 1;
      H[p]->force_update_actor = update_actor ? 1 : 0;
      const int rc = mx_maddpg_step_ex(H[p], &b[p], tn[(size_t)p * P + p], an[p], nullptr, st);
      H[p]->force_update_actor = -1;
      if (rc) return 1;
      if (flags & 8u) { if (mx_replay_update_priorities(R[p], b[p].idx, mx_maddpg_priorities(H[p]), nullptr, nullptr, B, st)) return 1; }
    }
    if ((flags & 4u) && update_actor)       // base_runner.py batch_train: after the P updates
      for (mx_maddpg* h : H)
        if (mx_maddpg_soft_update(h, st)) return 1;
    return 0;
  };
  return mx_graph_capture_seq(seq, [H]() { for (mx_maddpg* h : H) h->num_updates += 1; }, stream, out);
}
extern "C" int64_t mx_maddpg_num_updates(const mx_maddpg* h) { return h->num_updates; }
extern "C" int mx_maddpg_set_num_updates(mx_maddpg* h, int64_t n) {
  if (!h) { mx_set_error("mx_maddpg_set_num_updates: null handle"); return 1; }
  if (n < 0) { mx_set_error("mx_maddpg_set_num_updates: update count %lld < 0", (long long)n); return 1; }
  h->num_updates = n;
  return 0;
}

// named regions of the workspace, length in 4-byte words (as mx_qmix_ws_lookup): the actor / critic Adam step counters (fp64 words),
// the resumable state a checkpoint must carry besides the parameter vectors
extern "C" int mx_maddpg_ws_lookup(const mx_maddpg* h, const char* name, int64_t* byte_offset, int64_t* n_elems) {
  if (!h || !name) { mx_set_error("mx_maddpg_ws_lookup: null argument"); return 1; }
  struct Ent { const char* n; int64_t off, cnt; };
  const Ent tab[] = {{"adam_ta", h->W.adam_ta, 8}, {"adam_tc", h->W.adam_tc, 8}, {"p2p_abort", h->W.p2p_abort, 1}};
  for (const Ent& e : tab)
    if (!strcmp(e.n, name)) { *byte_offset = e.off * 4; *n_elems = e.cnt; return 0; }
  mx_set_error("mx_maddpg_ws_lookup: unknown region '%s'", name);
  return 1;
}

// cfg.mlp: the critic's target update stops at its trunk -- the target heads stay the target critic's own initialisation
static int64_t critic_tracked(const mx_maddpg* h) { return h->cfg.mlp ? (int64_t)h->critic.wih : h->Pc; }
extern "C" int mx_maddpg_soft_update(mx_maddpg* h, void* stream) {
  if (mx_launch_polyak(h->th_c_tgt, h->th_c, critic_tracked(h), h->cfg.tau, (cudaStream_t)stream)) return 1;
  return mx_launch_polyak(h->th_a_tgt, h->th_a, h->Pa, h->cfg.tau, (cudaStream_t)stream);
}
extern "C" int mx_maddpg_hard_update(mx_maddpg* h, void* stream) {
  cudaMemcpyAsync(h->th_c_tgt, h->th_c, (size_t)critic_tracked(h) * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream);
  cudaMemcpyAsync(h->th_a_tgt, h->th_a, (size_t)h->Pa * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream);
  return 0;
}
