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
struct MxMaddpgWs {
  // actor (rows Ma = B*(T+1)*N)
  int64_t a_gi[2], a_h[2], a_u1, a_u2, a_st0, a_st1, a_st2, a_sto, a_gates, a_hn, a_out, a_nact, a_dout, a_dh, a_dgi, a_act, a_soft;
  // critic sequences (rows Mc = B*T)
  int64_t c_x, c_gi[2], c_h[2], c_u1, c_u2, c_st0, c_st1, c_st2, c_sto, c_gates, c_hn, c_q, c_dq, c_dh, c_dgi, c_err;
  // target branch (rows Mc)
  int64_t t_x, t_gi, t_h, t_q, t_qmin;
  // actor-phase branch (rows Mr = N*B*T)
  int64_t r_x, r_h0, r_gi, r_h, r_u1, r_u2, r_st0, r_st1, r_st2, r_sto, r_gates, r_hn, r_q, r_dout, r_dh, r_dgi, r_dx;
  int64_t gpart_a, gpart_c, grad_a, grad_c, spart, info, prio, adam_ta, adam_tc, scal_c, scal_a;
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
// k_act_transform arguments for the M actor rows of cfg c.  n_act_seg > 0 is a MultiDiscrete action (one segment included), which takes
// no available-action mask (MADDPGPolicy.py:73-89); maddpg_check allows it on the MLP learner only
static ActXformArgs act_xform_args(const mx_maddpg_cfg* c, int M, int mode, const float* avail, int avail_ld) {
  ActXformArgs ax;
  memset(&ax, 0, sizeof(ax));
  ax.M = M; ax.Ac = c->act_dim; ax.mode = mode; ax.sg = act_segs(c);
  ax.avail = c->n_act_seg > 0 ? nullptr : avail; ax.avail_ld = avail_ld;
  return ax;
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
  for (int k = 0; k < 2; ++k) { W->a_gi[k] = tk(Ma * MX_G); W->a_h[k] = tk(Ma * MX_H); }
  W->a_u1 = tk(Ma * MX_H); W->a_u2 = tk(Ma * MX_H); W->a_st0 = tk(Ma * 2); W->a_st1 = tk(Ma * 2); W->a_st2 = tk(Ma * 2); W->a_sto = tk(Ma * 2);
  W->a_gates = tk(Ma * MX_G); W->a_hn = tk(Ma * MX_H); W->a_out = tk(Ma * Ac); W->a_nact = tk(Ma * Ac); W->a_dout = tk(Ma * Ac);
  W->a_dh = tk(Ma * MX_H); W->a_dgi = tk(Ma * MX_G); W->a_act = tk(Ma * Ac); W->a_soft = tk(Ma * Ac);
  W->c_x = tk(Mc * ldc);
  for (int k = 0; k < 2; ++k) { W->c_gi[k] = tk(Mc * MX_G); W->c_h[k] = tk(Mc * MX_H); }
  W->c_u1 = tk(Mc * MX_H); W->c_u2 = tk(Mc * MX_H); W->c_st0 = tk(Mc * 2); W->c_st1 = tk(Mc * 2); W->c_st2 = tk(Mc * 2); W->c_sto = tk(Mc * 2);
  W->c_gates = tk(Mc * MX_G); W->c_hn = tk(Mc * MX_H); W->c_q = tk(Mc * K); W->c_dq = tk(Mc * K); W->c_dh = tk(Mc * MX_H); W->c_dgi = tk(Mc * MX_G);
  W->c_err = tk(Mc * K);
  W->t_x = tk(Mc * ldc); W->t_gi = tk(Mc * MX_G); W->t_h = tk(Mc * MX_H); W->t_q = tk(Mc * K); W->t_qmin = tk(Mc);
  W->r_x = tk(Mr * ldc); W->r_h0 = tk(Mr * MX_H); W->r_gi = tk(Mr * MX_G); W->r_h = tk(Mr * MX_H); W->r_u1 = tk(Mr * MX_H); W->r_u2 = tk(Mr * MX_H);
  W->r_st0 = tk(Mr * 2); W->r_st1 = tk(Mr * 2); W->r_st2 = tk(Mr * 2); W->r_sto = tk(Mr * 2); W->r_gates = tk(Mr * MX_G); W->r_hn = tk(Mr * MX_H);
  W->r_q = tk(Mr * K); W->r_dout = tk(Mr * K); W->r_dh = tk(Mr * MX_H); W->r_dgi = tk(Mr * MX_G); W->r_dx = tk(Mr * ldc);
  W->gpart_a = tk((int64_t)npart * Pa); W->gpart_c = tk((int64_t)npart * Pc); W->grad_a = tk(Pa + 8); W->grad_c = tk(Pc + 8);
  W->spart = tk(16); W->info = tk(8); W->prio = tk(B); W->adam_ta = tk(8); W->adam_tc = tk(8); W->scal_c = tk(8); W->scal_a = tk(8);
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

static int optimise(mx_maddpg* h, bool actor, const int parts[2], int head_parts, cudaStream_t s) {
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
  o.seg_begin[0] = 0; o.seg_end[0] = L.lno_g; o.seg_parts[0] = parts[0];
  o.seg_begin[1] = L.lno_g; o.seg_end[1] = (int)P; o.seg_parts[1] = head_parts;
  if (c.mlp) {        // every gradient comes from k_front_bwd; the critic's trained range stops at its trunk (the frozen heads follow it)
    o.nseg = 1;
    if (!actor) { o.P = L.wih; o.gpart_ld = P; o.seg_end[0] = L.wih; }
  }
  o.spart = ws + h->W.spart; o.spart_n = 0;
  o.info = ws + h->W.info + (actor ? 4 : 0);
  o.adam_t = reinterpret_cast<double*>(ws + (actor ? h->W.adam_ta : h->W.adam_tc));
  o.err = nullptr; o.B = 0; o.T = 0; o.prio = nullptr;
  o.lr = c.lr; o.beta1 = c.adam_beta1; o.beta2 = c.adam_beta2; o.eps = c.adam_eps; o.max_grad_norm = c.max_grad_norm; o.tau = c.tau;
  o.weight_decay = c.weight_decay;
  if (mx_launch_grad_reduce(o, s)) return 1;     // (its scalar block bumps the Adam step count; the loss scalars come from the loss kernel)
  MX_LAUNCH(k_set_scalars, dim3(1), dim3(32), 0, s, o.grad + o.P, (const float*)(ws + (actor ? h->W.scal_a : h->W.scal_c)));
  MX_COUNT();
  MX_MARK("k_set_scalars", s);
  return mx_launch_adam(o, s);
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
static int maddpg_step_mlp(mx_maddpg* h, const mx_batch* b, const float* target_noise_dev, const float* actor_noise_dev, bool update_actor,
                           cudaStream_t s) {
  const mx_maddpg_cfg& c = h->cfg;
  float* ws = h->ws;
  const MxMaddpgWs& W = h->W;
  const int B = b->B, N = c.n_agents, K = c.num_q, Ac = c.act_dim, S = c.state_dim;
  const int Ma = B * 2 * N, Mc = B, Mr = N * B;
  const int ldc = mx_round_up(critic_in_dim(&c), 4);
  const MxNetLayout& LA = h->actor;
  const MxNetLayout& LC = h->critic;
  const int fnorm = c.no_feature_norm ? 0 : 1;
  const bool multi = c.cent_act_dim > 0;

  // ---------- A. live + target actor on obs and next_obs; target actions a' from the next_obs rows (maddpg.py:64-74) ----------
  FrontFwdArgs ff;
  memset(&ff, 0, sizeof(ff));
  ff.tc_acc = ws + W.tc_acc; ff.tc_acc_cols = (int)W.tc_acc_cols;
  ff.X = b->obs; ff.ldx = b->obs_ld; ff.M = Ma; ff.feature_norm = fnorm; ff.act_tanh = c.use_tanh;
  ff.theta[0] = h->th_a; ff.theta[1] = h->th_a_tgt; ff.L = LA;
  ff.gi[0] = ws + W.a_gi[0]; ff.gi[1] = ws + W.a_gi[1];
  ff.u1 = ws + W.a_u1; ff.u2 = ws + W.a_u2; ff.st0 = ws + W.a_st0; ff.st1 = ws + W.a_st1; ff.st2 = ws + W.a_st2;
  if (mx_launch_front_fwd(ff, multi ? 1 : 2, s)) return 1;      // several policies: the target actions come from cent_nacts
  if (!multi) {
    MX_LAUNCH(k_mlp_head_cols, dim3(launch1d(Ma)), dim3(256), 0, s, (const float*)ff.gi[1], Ma, Ac, c.target_noise > 0.f ? target_noise_dev : nullptr,
              ws + W.a_nact, nullptr);
    MX_COUNT(); MX_MARK("k_mlp_head_cols", s);
  }
  if (c.discrete && !multi) {      // onehot_from_logits with the next-avail mask (MADDPG) / hard Gumbel-softmax, the draw already added (MATD3)
    ActXformArgs ax = act_xform_args(&c, Ma, c.target_noise > 0.f ? 1 : 0, b->avail, b->act_ld);
    ax.logits = ws + W.a_nact; ax.out = ws + W.a_nact;
    MX_LAUNCH(k_act_transform, dim3(launch1d(Ma)), dim3(256), 0, s, ax); MX_COUNT(); MX_MARK("k_act_transform", s);
  }

  // ---------- B. live critic on (s, a), target critic on (s', a'); TD target, loss, priorities (maddpg.py:112-151) ----------
  PackArgs pk;
  memset(&pk, 0, sizeof(pk));
  pk.B = B; pk.T = 1; pk.N = N; pk.S = S; pk.Ac = Ac; pk.share = b->share; pk.share_ld = b->share_ld; pk.acts = b->acts; pk.act_ld = b->act_ld;
  pk.ldx = ldc;
  if (multi) { pk.CA = c.cent_act_dim; pk.off = c.act_offset; pk.ca_ld = mx_round_up(c.cent_act_dim, 4); pk.cent_acts = ws + W.cent_acts; pk.cent_nacts = ws + W.cent_nacts; }
  pk.mode = 0; pk.x = ws + W.c_x;
  MX_LAUNCH(k_pack_critic_in, dim3(launch1d((long long)Mc * ldc)), dim3(256), 0, s, pk); MX_COUNT(); MX_MARK("k_pack_critic_in", s);
  pk.mode = 1; pk.x = ws + W.t_x; pk.actor_out = ws + W.a_nact;
  MX_LAUNCH(k_pack_critic_in, dim3(launch1d((long long)Mc * ldc)), dim3(256), 0, s, pk); MX_COUNT(); MX_MARK("k_pack_critic_in", s);
  FrontFwdArgs fc;
  memset(&fc, 0, sizeof(fc));
  fc.tc_acc = ws + W.tc_acc; fc.tc_acc_cols = (int)W.tc_acc_cols;
  fc.X = ws + W.c_x; fc.ldx = ldc; fc.M = Mc; fc.feature_norm = fnorm; fc.act_tanh = c.use_tanh; fc.theta[0] = h->th_c; fc.L = LC;
  fc.gi[0] = ws + W.c_gi[0];
  fc.u1 = ws + W.c_u1; fc.u2 = ws + W.c_u2; fc.st0 = ws + W.c_st0; fc.st1 = ws + W.c_st1; fc.st2 = ws + W.c_st2;
  if (mx_launch_front_fwd(fc, 1, s)) return 1;
  FrontFwdArgs ft;
  memset(&ft, 0, sizeof(ft));
  ft.tc_acc = ws + W.tc_acc; ft.tc_acc_cols = (int)W.tc_acc_cols;
  ft.X = ws + W.t_x; ft.ldx = ldc; ft.M = Mc; ft.feature_norm = fnorm; ft.act_tanh = c.use_tanh; ft.theta[0] = h->th_c_tgt; ft.L = LC; ft.gi[0] = ws + W.t_gi;
  if (mx_launch_front_fwd(ft, 1, s)) return 1;
  MX_LAUNCH(k_mlp_head_cols, dim3(launch1d(Mc)), dim3(256), 0, s, (const float*)fc.gi[0], Mc, K, (const float*)nullptr, ws + W.c_q, nullptr);
  MX_COUNT(); MX_MARK("k_mlp_head_cols", s);
  MX_LAUNCH(k_mlp_head_cols, dim3(launch1d(Mc)), dim3(256), 0, s, (const float*)ft.gi[0], Mc, K, (const float*)nullptr, nullptr, ws + W.t_qmin);
  MX_COUNT(); MX_MARK("k_mlp_head_cols", s);
  CriticLossArgs cl;
  memset(&cl, 0, sizeof(cl));
  cl.B = B; cl.T = 1; cl.N = N; cl.K = K; cl.ld_tn = b->ep_tn_ld > 0 ? b->ep_tn_ld : N; cl.ld_t = b->ep_t_ld > 0 ? b->ep_t_ld : 1;
  cl.qpred = ws + W.c_q; cl.qnext_min = ws + W.t_qmin; cl.rewards = b->rewards; cl.dones_env = b->dones_env;
  cl.weights = c.use_per ? b->weights : nullptr; cl.gamma = c.gamma; cl.huber_delta = c.huber_delta; cl.per_eps = c.per_eps;
  cl.use_huber = c.use_huber; cl.prio_mean_k = 1; cl.dq = ws + W.c_dq; cl.err = ws + W.c_err; cl.scal = ws + W.scal_c; cl.prio = c.use_per ? ws + W.prio : nullptr;
  MX_LAUNCH(k_critic_loss, dim3(1), dim3(256), 0, s, cl); MX_COUNT(); MX_MARK("k_critic_loss", s);

  // ---------- C. critic backward through the frozen live heads into the trunk; clip + Adam over the trunk ----------
  MX_LAUNCH(k_mlp_dgi_cols, dim3(launch1d((long long)Mc * MX_G)), dim3(256), 0, s, (const float*)(ws + W.c_dq), K, Mc, ws + W.c_dgi);
  MX_COUNT(); MX_MARK("k_mlp_dgi_cols", s);
  int parts[2] = {0, 0};
  FrontBwdArgs fb;
  memset(&fb, 0, sizeof(fb));
  fb.X = ws + W.c_x; fb.ldx = ldc; fb.M = Mc; fb.T = 1; fb.N = 1; fb.feature_norm = fnorm; fb.act_tanh = c.use_tanh; fb.no_gru = 1;
  fb.theta = h->th_c; fb.L = LC; fb.u1 = fc.u1; fb.u2 = fc.u2; fb.st0 = fc.st0; fb.st1 = fc.st1; fb.st2 = fc.st2; fb.dgi = ws + W.c_dgi;
  fb.gpart = ws + W.gpart_c; fb.P = h->Pc;
  fb.da2_out = ws + W.tc_da2; fb.da1_out = ws + W.tc_da1; fb.tc_imgT = ws + W.tc_imgT;      // (option wgrad_tc)
  fb.tc_acc = ws + W.tc_acc; fb.tc_acc_cols = (int)W.tc_acc_cols;
  if (mx_launch_front_bwd(fb, &parts[0], s)) return 1;
  if (optimise(h, false, parts, 0, s)) return 1;
  if (!update_actor) return 0;

  // ---------- D. actor loss through head 0 of the UPDATED critic on the agent-replaced copies, masked by valid_transition ----------
  MX_LAUNCH(k_mlp_head_cols, dim3(launch1d(Ma)), dim3(256), 0, s, (const float*)ff.gi[0], Ma, Ac, (const float*)nullptr, ws + W.a_out, nullptr);
  MX_COUNT(); MX_MARK("k_mlp_head_cols", s);
  if (c.discrete) {    // get_actions(obs, avail, use_gumbel=True): hard Gumbel-softmax, straight-through (maddpg.py:209)
    ActXformArgs ax = act_xform_args(&c, Ma, 1, b->avail, b->act_ld);
    ax.logits = ws + W.a_out; ax.gumbel = actor_noise_dev; ax.out = ws + W.a_act; ax.soft = ws + W.a_soft;
    MX_LAUNCH(k_act_transform, dim3(launch1d(Ma)), dim3(256), 0, s, ax); MX_COUNT(); MX_MARK("k_act_transform", s);
  }
  pk.mode = 2; pk.x = ws + W.r_x; pk.actor_out = ws + (c.discrete ? W.a_act : W.a_out);
  MX_LAUNCH(k_pack_critic_in, dim3(launch1d((long long)Mr * ldc)), dim3(256), 0, s, pk); MX_COUNT(); MX_MARK("k_pack_critic_in", s);
  FrontFwdArgs fr;
  memset(&fr, 0, sizeof(fr));
  fr.tc_acc = ws + W.tc_acc; fr.tc_acc_cols = (int)W.tc_acc_cols;
  fr.X = ws + W.r_x; fr.ldx = ldc; fr.M = Mr; fr.feature_norm = fnorm; fr.act_tanh = c.use_tanh; fr.theta[0] = h->th_c; fr.L = LC; fr.gi[0] = ws + W.r_gi;
  fr.u1 = ws + W.r_u1; fr.u2 = ws + W.r_u2; fr.st0 = ws + W.r_st0; fr.st1 = ws + W.r_st1; fr.st2 = ws + W.r_st2;
  if (mx_launch_front_fwd(fr, 1, s)) return 1;
  MX_LAUNCH(k_mlp_head_cols, dim3(launch1d(Mr)), dim3(256), 0, s, (const float*)fr.gi[0], Mr, K, (const float*)nullptr, ws + W.r_q, nullptr);
  MX_COUNT(); MX_MARK("k_mlp_head_cols", s);
  ActorLossArgs al;
  memset(&al, 0, sizeof(al));
  al.B = B; al.T = 1; al.N = N; al.K = K; al.ld_tn = b->ep_tn_ld > 0 ? b->ep_tn_ld : N; al.qa = ws + W.r_q; al.dones = b->dones;
  al.valid = h->valid; al.valid_idx = b->idx; al.dout = ws + W.r_dout; al.scal = ws + W.scal_a;
  MX_LAUNCH(k_actor_loss, dim3(1), dim3(256), 0, s, al); MX_COUNT(); MX_MARK("k_actor_loss", s);
  // back through the frozen critic (trunk and live head 0) to its action inputs, then into the actor's head rows
  MX_LAUNCH(k_mlp_dgi_cols, dim3(launch1d((long long)Mr * MX_G)), dim3(256), 0, s, (const float*)(ws + W.r_dout), K, Mr, ws + W.r_dgi);
  MX_COUNT(); MX_MARK("k_mlp_dgi_cols", s);
  FrontBwdArgs fbr;
  memset(&fbr, 0, sizeof(fbr));
  fbr.X = ws + W.r_x; fbr.ldx = ldc; fbr.M = Mr; fbr.T = 1; fbr.N = 1; fbr.feature_norm = fnorm; fbr.act_tanh = c.use_tanh; fbr.no_gru = 1;
  fbr.theta = h->th_c; fbr.L = LC; fbr.u1 = fr.u1; fbr.u2 = fr.u2; fbr.st0 = fr.st0; fbr.st1 = fr.st1; fbr.st2 = fr.st2; fbr.dgi = ws + W.r_dgi;
  fbr.gpart = ws + W.gpart_c; fbr.P = h->Pc; fbr.dX = ws + W.r_dx; fbr.skip_wgrad = 1;
  int dummy = 0;
  if (mx_launch_front_bwd(fbr, &dummy, s)) return 1;
  MX_LAUNCH(k_scatter_actor_grad, dim3(launch1d(Ma)), dim3(256), 0, s, (const float*)(ws + W.r_dx), ldc, B, 1, N, S, Ac,
            (const float*)(c.discrete ? ws + W.a_soft : nullptr), ws + W.a_dgi, c.act_offset, (int)MX_G, act_segs(&c));
  MX_COUNT(); MX_MARK("k_scatter_actor_grad", s);
  FrontBwdArgs fba;
  memset(&fba, 0, sizeof(fba));
  fba.X = b->obs; fba.ldx = b->obs_ld; fba.M = Ma; fba.T = 1; fba.N = N; fba.feature_norm = fnorm; fba.act_tanh = c.use_tanh; fba.no_gru = 1;
  fba.theta = h->th_a; fba.L = LA; fba.u1 = ff.u1; fba.u2 = ff.u2; fba.st0 = ff.st0; fba.st1 = ff.st1; fba.st2 = ff.st2; fba.dgi = ws + W.a_dgi;
  fba.gpart = ws + W.gpart_a; fba.P = h->Pa;
  fba.da2_out = ws + W.tc_da2; fba.da1_out = ws + W.tc_da1; fba.tc_imgT = ws + W.tc_imgT;
  fba.tc_acc = ws + W.tc_acc; fba.tc_acc_cols = (int)W.tc_acc_cols;
  int aparts[2] = {0, 0};
  if (mx_launch_front_bwd(fba, &aparts[0], s)) return 1;
  return optimise(h, true, aparts, 0, s);
}

extern "C" int mx_maddpg_step(mx_maddpg* h, const mx_batch* b, const float* target_noise_dev, int32_t* update_actor_out, void* stream) {
  return mx_maddpg_step_ex(h, b, target_noise_dev, nullptr, update_actor_out, stream);
}

extern "C" int mx_maddpg_step_ex(mx_maddpg* h, const mx_batch* b, const float* target_noise_dev, const float* actor_noise_dev,
                                 int32_t* update_actor_out, void* stream) {
  const mx_maddpg_cfg& c = h->cfg;
#if !MX_EMU
  g_mx_pdl_auto = 1;      // ~40 small dependent launches per update: programmatic dependent launch measured 491 -> 469 us (R-MADDPG), 372 -> 355 us (R-MATD3)
#endif
  if (!b || b->B <= 0 || b->B > c.max_batch) { mx_set_error("maddpg step: batch size outside [1, max_batch=%d]", c.max_batch); return 1; }
  if (!b->obs || !b->share || !b->acts || !b->rewards || !b->dones || !b->dones_env) { mx_set_error("maddpg step: missing batch field"); return 1; }
  if (c.use_per && !b->weights) { mx_set_error("maddpg step: use_per set but batch has no importance weights"); return 1; }
  if (c.target_noise > 0.f && !target_noise_dev) { mx_set_error("maddpg step: MATD3 target noise expected"); return 1; }
  const bool update_actor = h->force_update_actor >= 0 ? h->force_update_actor != 0
                                                     : (h->num_updates % (c.actor_update_interval > 0 ? c.actor_update_interval : 1)) == 0;
  {
    const bool upd = update_actor;
    if (c.discrete && upd && !actor_noise_dev) { mx_set_error("maddpg step: discrete actor update needs the Gumbel draws (actor_noise_dev)"); return 1; }
  }
  cudaStream_t s = (cudaStream_t)stream;
  if (c.mlp) {
    if (maddpg_step_mlp(h, b, target_noise_dev, actor_noise_dev, update_actor, s)) return 1;
    if (update_actor_out) *update_actor_out = update_actor ? 1 : 0;
    if (h->force_update_actor < 0) h->num_updates += 1;
    return 0;
  }
  float* ws = h->ws;
  const MxMaddpgWs& W = h->W;
  const int B = b->B, T = c.episode_len, N = c.n_agents, K = c.num_q, Ac = c.act_dim, S = c.state_dim;
  const int Ma = B * (T + 1) * N, Mc = B * T, Mr = N * B * T;
  const int ldc = mx_round_up(critic_in_dim(&c), 4);
  const MxNetLayout& LA = h->actor;
  const MxNetLayout& LC = h->critic;
  const int hstride = MX_H + 4;
  const bool multi = c.cent_act_dim > 0;       // several policies: the centralised action vectors were assembled by mx_maddpg_cent_contribute

  // ---------- A. actor: live + target over the T+1 steps ----------
  FrontFwdArgs ff;
  memset(&ff, 0, sizeof(ff));
  ff.tc_acc = ws + W.tc_acc; ff.tc_acc_cols = (int)W.tc_acc_cols;
  ff.X = b->obs; ff.ldx = b->obs_ld; ff.M = Ma; ff.feature_norm = c.no_feature_norm ? 0 : 1; ff.act_tanh = c.use_tanh;
  ff.theta[0] = h->th_a; ff.theta[1] = h->th_a_tgt; ff.L = LA;
  ff.gi[0] = ws + W.a_gi[0]; ff.gi[1] = ws + W.a_gi[1];
  ff.u1 = ws + W.a_u1; ff.u2 = ws + W.a_u2; ff.st0 = ws + W.a_st0; ff.st1 = ws + W.a_st1; ff.st2 = ws + W.a_st2;
  if (mx_launch_front_fwd(ff, 2, s)) return 1;
  GruFwdArgs gf;
  memset(&gf, 0, sizeof(gf));
  gf.theta[0] = h->th_a; gf.theta[1] = h->th_a_tgt; gf.whh = LA.whh; gf.bhh = LA.bhh;
  gf.gi[0] = ff.gi[0]; gf.gi[1] = ff.gi[1]; gf.hall[0] = ws + W.a_h[0]; gf.hall[1] = ws + W.a_h[1];
  gf.gates = ws + W.a_gates; gf.hn = ws + W.a_hn; gf.R = B * N; gf.T = T; gf.N = N;
  if (mx_launch_gru_fwd(gf, 2, s)) return 1;
  HeadArgs ha;
  memset(&ha, 0, sizeof(ha));
  ha.lno_g = LA.lno_g; ha.lno_b = LA.lno_b; ha.w = LA.wq; ha.b = LA.bq; ha.OD = Ac; ha.b_stride = 1; ha.w_stride = MX_H; ha.M = Ma;
  ha.theta = h->th_a; ha.h = gf.hall[0]; ha.sto = ws + W.a_sto; ha.out = ws + W.a_out;
  MX_LAUNCH(k_head_fwd, dim3(launch1d((long long)Ma * 32)), dim3(256), 0, s, ha); MX_COUNT(); MX_MARK("k_head_fwd", s);
  ha.theta = h->th_a_tgt; ha.h = gf.hall[1]; ha.sto = nullptr; ha.out = ws + W.a_nact; ha.noise = c.target_noise > 0.f ? target_noise_dev : nullptr;
  MX_LAUNCH(k_head_fwd, dim3(launch1d((long long)Ma * 32)), dim3(256), 0, s, ha); MX_COUNT(); MX_MARK("k_head_fwd", s);
  if (c.discrete) {      // target actions: arg-max one-hot (MADDPG) / hard Gumbel-softmax sample (MATD3; the head added the draw)
    ActXformArgs ax = act_xform_args(&c, Ma, c.target_noise > 0.f ? 1 : 0, b->avail, b->act_ld);
    ax.logits = ws + W.a_nact; ax.out = ws + W.a_nact;
    MX_LAUNCH(k_act_transform, dim3(launch1d(Ma)), dim3(256), 0, s, ax); MX_COUNT(); MX_MARK("k_act_transform", s);
  }

  // ---------- B. critic over the buffer sequence (live + target) ----------
  PackArgs pk;
  memset(&pk, 0, sizeof(pk));
  pk.B = B; pk.T = T; pk.N = N; pk.S = S; pk.Ac = Ac; pk.share = b->share; pk.share_ld = b->share_ld; pk.acts = b->acts; pk.act_ld = b->act_ld;
  pk.ldx = ldc;
  if (multi) { pk.CA = c.cent_act_dim; pk.off = c.act_offset; pk.ca_ld = mx_round_up(c.cent_act_dim, 4); pk.cent_acts = ws + W.cent_acts; pk.cent_nacts = ws + W.cent_nacts; }
  pk.mode = 0; pk.x = ws + W.c_x;
  MX_LAUNCH(k_pack_critic_in, dim3(launch1d((long long)Mc * ldc)), dim3(256), 0, s, pk); MX_COUNT(); MX_MARK("k_pack_critic_in", s);
  FrontFwdArgs fc;
  memset(&fc, 0, sizeof(fc));
  fc.tc_acc = ws + W.tc_acc; fc.tc_acc_cols = (int)W.tc_acc_cols;
  fc.X = ws + W.c_x; fc.ldx = ldc; fc.M = Mc; fc.feature_norm = c.no_feature_norm ? 0 : 1; fc.act_tanh = c.use_tanh;
  fc.theta[0] = h->th_c; fc.theta[1] = h->th_c_tgt; fc.L = LC;
  fc.gi[0] = ws + W.c_gi[0]; fc.gi[1] = ws + W.c_gi[1];
  fc.u1 = ws + W.c_u1; fc.u2 = ws + W.c_u2; fc.st0 = ws + W.c_st0; fc.st1 = ws + W.c_st1; fc.st2 = ws + W.c_st2;
  if (mx_launch_front_fwd(fc, 2, s)) return 1;
  GruFwdArgs gc;
  memset(&gc, 0, sizeof(gc));
  gc.theta[0] = h->th_c; gc.theta[1] = h->th_c_tgt; gc.whh = LC.whh; gc.bhh = LC.bhh;
  gc.gi[0] = fc.gi[0]; gc.gi[1] = fc.gi[1]; gc.hall[0] = ws + W.c_h[0]; gc.hall[1] = ws + W.c_h[1];
  gc.gates = ws + W.c_gates; gc.hn = ws + W.c_hn; gc.R = B; gc.T = T - 1; gc.N = 1;
  if (mx_launch_gru_fwd(gc, 2, s)) return 1;
  HeadArgs hc;
  memset(&hc, 0, sizeof(hc));
  hc.lno_g = LC.lno_g; hc.lno_b = LC.lno_b; hc.w = LC.wq; hc.b = LC.wq + MX_H; hc.OD = K; hc.b_stride = hstride; hc.w_stride = hstride; hc.M = Mc;
  hc.theta = h->th_c; hc.h = gc.hall[0]; hc.sto = ws + W.c_sto; hc.out = ws + W.c_q;
  MX_LAUNCH(k_head_fwd, dim3(launch1d((long long)Mc * 32)), dim3(256), 0, s, hc); MX_COUNT(); MX_MARK("k_head_fwd", s);

  // ---------- C. target Q: one branch step per (b,t) from the target critic's buffer state ----------
  pk.mode = 1; pk.x = ws + W.t_x; pk.actor_out = ws + W.a_nact;
  MX_LAUNCH(k_pack_critic_in, dim3(launch1d((long long)Mc * ldc)), dim3(256), 0, s, pk); MX_COUNT(); MX_MARK("k_pack_critic_in", s);
  FrontFwdArgs ft;
  memset(&ft, 0, sizeof(ft));
  ft.tc_acc = ws + W.tc_acc; ft.tc_acc_cols = (int)W.tc_acc_cols;
  ft.X = ws + W.t_x; ft.ldx = ldc; ft.M = Mc; ft.feature_norm = c.no_feature_norm ? 0 : 1; ft.act_tanh = c.use_tanh; ft.theta[0] = h->th_c_tgt; ft.L = LC; ft.gi[0] = ws + W.t_gi;
  if (mx_launch_front_fwd(ft, 1, s)) return 1;
  GruFwdArgs gt;
  memset(&gt, 0, sizeof(gt));
  gt.theta[0] = h->th_c_tgt; gt.whh = LC.whh; gt.bhh = LC.bhh; gt.gi[0] = ft.gi[0]; gt.hall[0] = ws + W.t_h;
  gt.gates = nullptr; gt.hn = nullptr; gt.R = Mc; gt.T = 0; gt.N = 1; gt.h0 = gc.hall[1];
  if (mx_launch_gru_fwd(gt, 1, s)) return 1;
  HeadArgs ht = hc;
  ht.theta = h->th_c_tgt; ht.h = gt.hall[0]; ht.sto = nullptr; ht.out = ws + W.t_q; ht.out_min = ws + W.t_qmin;
  MX_LAUNCH(k_head_fwd, dim3(launch1d((long long)Mc * 32)), dim3(256), 0, s, ht); MX_COUNT(); MX_MARK("k_head_fwd", s);

  // ---------- D. TD target, critic loss ----------
  CriticLossArgs cl;
  memset(&cl, 0, sizeof(cl));
  cl.B = B; cl.T = T; cl.N = N; cl.K = K; cl.ld_tn = b->ep_tn_ld > 0 ? b->ep_tn_ld : T * N; cl.ld_t = b->ep_t_ld > 0 ? b->ep_t_ld : T; cl.qpred = ws + W.c_q; cl.qnext_min = ws + W.t_qmin; cl.rewards = b->rewards; cl.dones_env = b->dones_env;
  cl.weights = c.use_per ? b->weights : nullptr; cl.gamma = c.gamma; cl.huber_delta = c.huber_delta; cl.per_nu = c.per_nu; cl.per_eps = c.per_eps;
  cl.use_huber = c.use_huber; cl.dq = ws + W.c_dq; cl.err = ws + W.c_err; cl.scal = ws + W.scal_c; cl.prio = c.use_per ? ws + W.prio : nullptr;
  MX_LAUNCH(k_critic_loss, dim3(1), dim3(256), 0, s, cl); MX_COUNT(); MX_MARK("k_critic_loss", s);

  // ---------- E. critic backward + Adam ----------
  const int head_grid = mx_imin_host(mx_num_sms(), mx_ceil_div(Mc, 32));
  HeadBwdArgs hb;
  memset(&hb, 0, sizeof(hb));
  hb.theta = h->th_c; hb.lno_g = LC.lno_g; hb.lno_b = LC.lno_b; hb.w = LC.wq; hb.b = LC.wq + MX_H; hb.OD = K; hb.b_stride = hstride; hb.w_stride = hstride;
  hb.h = gc.hall[0]; hb.sto = ws + W.c_sto; hb.dout = ws + W.c_dq; hb.M = Mc; hb.dh_out = ws + W.c_dh; hb.gpart = ws + W.gpart_c; hb.P = h->Pc;
  MX_LAUNCH(k_head_bwd, dim3(head_grid), dim3(256), 0, s, hb); MX_COUNT(); MX_MARK("k_head_bwd", s);
  GruBwdArgs gb;
  memset(&gb, 0, sizeof(gb));
  gb.theta = h->th_c; gb.whh = LC.whh; gb.hall = gc.hall[0]; gb.gates = gc.gates; gb.hn = gc.hn; gb.dh_out = hb.dh_out; gb.dgi = ws + W.c_dgi;
  gb.R = B; gb.T = T; gb.N = 1; gb.T1 = T;
  if (mx_launch_gru_bwd(gb, s)) return 1;
  int parts[2] = {0, 0};
  FrontBwdArgs fb;
  memset(&fb, 0, sizeof(fb));
  fb.X = ws + W.c_x; fb.ldx = ldc; fb.M = Mc; fb.T = T; fb.N = 1; fb.T1 = T; fb.feature_norm = c.no_feature_norm ? 0 : 1; fb.act_tanh = c.use_tanh; fb.theta = h->th_c; fb.L = LC;
  fb.u1 = fc.u1; fb.u2 = fc.u2; fb.st0 = fc.st0; fb.st1 = fc.st1; fb.st2 = fc.st2; fb.dgi = gb.dgi; fb.gates = gc.gates; fb.hall = gc.hall[0];
  fb.gpart = ws + W.gpart_c; fb.P = h->Pc;
  fb.da2_out = ws + W.tc_da2; fb.da1_out = ws + W.tc_da1; fb.tc_imgT = ws + W.tc_imgT;      // (option wgrad_tc)
  fb.tc_acc = ws + W.tc_acc; fb.tc_acc_cols = (int)W.tc_acc_cols;
  if (mx_launch_front_bwd(fb, &parts[0], s)) return 1;
  if (optimise(h, false, parts, head_grid, s)) return 1;

  // ---------- F. actor update with the UPDATED critic ----------
  if (update_actor) {
    // live critic recurrence over the buffer sequence again (its parameters just changed)
    FrontFwdArgs f2;
    memset(&f2, 0, sizeof(f2));
    f2.tc_acc = ws + W.tc_acc; f2.tc_acc_cols = (int)W.tc_acc_cols;
    f2.X = ws + W.c_x; f2.ldx = ldc; f2.M = Mc; f2.feature_norm = c.no_feature_norm ? 0 : 1; f2.act_tanh = c.use_tanh; f2.theta[0] = h->th_c; f2.L = LC; f2.gi[0] = ws + W.c_gi[0];
    if (mx_launch_front_fwd(f2, 1, s)) return 1;
    GruFwdArgs g2;
    memset(&g2, 0, sizeof(g2));
    g2.theta[0] = h->th_c; g2.whh = LC.whh; g2.bhh = LC.bhh; g2.gi[0] = f2.gi[0]; g2.hall[0] = ws + W.c_h[0]; g2.R = B; g2.T = T - 1; g2.N = 1;
    g2.gates = ws + W.c_gates; g2.hn = ws + W.c_hn;
    if (mx_launch_gru_fwd(g2, 1, s)) return 1;
    if (c.discrete) {    // the live actor's hard Gumbel-softmax sample (straight-through), r_maddpg.py:277
      ActXformArgs ax = act_xform_args(&c, Ma, 1, b->avail, b->act_ld);
      ax.logits = ws + W.a_out; ax.gumbel = actor_noise_dev; ax.out = ws + W.a_act; ax.soft = ws + W.a_soft;
      MX_LAUNCH(k_act_transform, dim3(launch1d(Ma)), dim3(256), 0, s, ax); MX_COUNT(); MX_MARK("k_act_transform", s);
    }
    pk.mode = 2; pk.x = ws + W.r_x; pk.actor_out = ws + (c.discrete ? W.a_act : W.a_out); pk.hseq = g2.hall[0]; pk.h0 = ws + W.r_h0;
    MX_LAUNCH(k_pack_critic_in, dim3(launch1d((long long)Mr * ldc)), dim3(256), 0, s, pk); MX_COUNT(); MX_MARK("k_pack_critic_in", s);
    FrontFwdArgs fr;
    memset(&fr, 0, sizeof(fr));
    fr.tc_acc = ws + W.tc_acc; fr.tc_acc_cols = (int)W.tc_acc_cols;
    fr.X = ws + W.r_x; fr.ldx = ldc; fr.M = Mr; fr.feature_norm = c.no_feature_norm ? 0 : 1; fr.act_tanh = c.use_tanh; fr.theta[0] = h->th_c; fr.L = LC; fr.gi[0] = ws + W.r_gi;
    fr.u1 = ws + W.r_u1; fr.u2 = ws + W.r_u2; fr.st0 = ws + W.r_st0; fr.st1 = ws + W.r_st1; fr.st2 = ws + W.r_st2;
    if (mx_launch_front_fwd(fr, 1, s)) return 1;
    GruFwdArgs gr;
    memset(&gr, 0, sizeof(gr));
    gr.theta[0] = h->th_c; gr.whh = LC.whh; gr.bhh = LC.bhh; gr.gi[0] = fr.gi[0]; gr.hall[0] = ws + W.r_h;
    gr.gates = ws + W.r_gates; gr.hn = ws + W.r_hn; gr.R = Mr; gr.T = 0; gr.N = 1; gr.h0 = ws + W.r_h0;
    if (mx_launch_gru_fwd(gr, 1, s)) return 1;
    HeadArgs hr = hc;
    hr.theta = h->th_c; hr.h = gr.hall[0]; hr.sto = ws + W.r_sto; hr.out = ws + W.r_q; hr.out_min = nullptr; hr.M = Mr;
    MX_LAUNCH(k_head_fwd, dim3(launch1d((long long)Mr * 32)), dim3(256), 0, s, hr); MX_COUNT(); MX_MARK("k_head_fwd", s);
    ActorLossArgs al;
    memset(&al, 0, sizeof(al));
    al.B = B; al.T = T; al.N = N; al.K = K; al.ld_tn = b->ep_tn_ld > 0 ? b->ep_tn_ld : T * N; al.qa = ws + W.r_q; al.dones = b->dones; al.dout = ws + W.r_dout; al.scal = ws + W.scal_a;
    MX_LAUNCH(k_actor_loss, dim3(1), dim3(256), 0, s, al); MX_COUNT(); MX_MARK("k_actor_loss", s);
    // back through the (frozen) critic to its action inputs
    HeadBwdArgs hbr = hb;
    hbr.h = gr.hall[0]; hbr.sto = ws + W.r_sto; hbr.dout = ws + W.r_dout; hbr.M = Mr; hbr.dh_out = ws + W.r_dh; hbr.gpart = nullptr;
    MX_LAUNCH(k_head_bwd, dim3(mx_imin_host(mx_num_sms(), mx_ceil_div(Mr, 32))), dim3(256), 0, s, hbr); MX_COUNT(); MX_MARK("k_head_bwd", s);
    GruBwdArgs gbr;
    memset(&gbr, 0, sizeof(gbr));
    gbr.theta = h->th_c; gbr.whh = LC.whh; gbr.hall = gr.hall[0]; gbr.gates = gr.gates; gbr.hn = gr.hn; gbr.dh_out = hbr.dh_out; gbr.dgi = ws + W.r_dgi;
    gbr.R = Mr; gbr.T = 1; gbr.N = 1; gbr.T1 = 1; gbr.h0 = ws + W.r_h0;
    if (mx_launch_gru_bwd(gbr, s)) return 1;
    FrontBwdArgs fbr;
    memset(&fbr, 0, sizeof(fbr));
    fbr.X = ws + W.r_x; fbr.ldx = ldc; fbr.M = Mr; fbr.T = 0; fbr.N = 1; fbr.T1 = 1; fbr.h0 = ws + W.r_h0; fbr.feature_norm = c.no_feature_norm ? 0 : 1; fbr.act_tanh = c.use_tanh; fbr.theta = h->th_c; fbr.L = LC;
    fbr.u1 = fr.u1; fbr.u2 = fr.u2; fbr.st0 = fr.st0; fbr.st1 = fr.st1; fbr.st2 = fr.st2; fbr.dgi = gbr.dgi; fbr.gates = gr.gates; fbr.hall = gr.hall[0];
    fbr.gpart = ws + W.gpart_c; fbr.P = h->Pc; fbr.dX = ws + W.r_dx; fbr.skip_wgrad = 1;
    int dummy = 0;
    if (mx_launch_front_bwd(fbr, &dummy, s)) return 1;
    MX_LAUNCH(k_scatter_actor_grad, dim3(launch1d(Ma)), dim3(256), 0, s, (const float*)(ws + W.r_dx), ldc, B, T, N, S, Ac,
              (const float*)(c.discrete ? ws + W.a_soft : nullptr), ws + W.a_dout, multi ? c.act_offset : 0, Ac, act_segs(&c));
    MX_COUNT(); MX_MARK("k_scatter_actor_grad", s);
    // actor backward + Adam
    const int ahead_grid = mx_imin_host(mx_num_sms(), mx_ceil_div(Ma, 32));
    HeadBwdArgs hba;
    memset(&hba, 0, sizeof(hba));
    hba.theta = h->th_a; hba.lno_g = LA.lno_g; hba.lno_b = LA.lno_b; hba.w = LA.wq; hba.b = LA.bq; hba.OD = Ac; hba.b_stride = 1; hba.w_stride = MX_H;
    hba.h = gf.hall[0]; hba.sto = ws + W.a_sto; hba.dout = ws + W.a_dout; hba.M = Ma; hba.dh_out = ws + W.a_dh; hba.gpart = ws + W.gpart_a; hba.P = h->Pa;
    MX_LAUNCH(k_head_bwd, dim3(ahead_grid), dim3(256), 0, s, hba); MX_COUNT(); MX_MARK("k_head_bwd", s);
    GruBwdArgs gba;
    memset(&gba, 0, sizeof(gba));
    gba.theta = h->th_a; gba.whh = LA.whh; gba.hall = gf.hall[0]; gba.gates = gf.gates; gba.hn = gf.hn; gba.dh_out = hba.dh_out; gba.dgi = ws + W.a_dgi;
    gba.R = B * N; gba.T = T; gba.N = N; gba.T1 = T + 1;
    if (mx_launch_gru_bwd(gba, s)) return 1;
    FrontBwdArgs fba;
    memset(&fba, 0, sizeof(fba));
    fba.X = b->obs; fba.ldx = b->obs_ld; fba.M = Ma; fba.T = T; fba.N = N; fba.feature_norm = c.no_feature_norm ? 0 : 1; fba.act_tanh = c.use_tanh; fba.theta = h->th_a; fba.L = LA;
    fba.u1 = ff.u1; fba.u2 = ff.u2; fba.st0 = ff.st0; fba.st1 = ff.st1; fba.st2 = ff.st2; fba.dgi = gba.dgi; fba.gates = gf.gates; fba.hall = gf.hall[0];
    fba.gpart = ws + W.gpart_a; fba.P = h->Pa;
    fba.da2_out = ws + W.tc_da2; fba.da1_out = ws + W.tc_da1; fba.tc_imgT = ws + W.tc_imgT;
    fba.tc_acc = ws + W.tc_acc; fba.tc_acc_cols = (int)W.tc_acc_cols;
    int aparts[2] = {0, 0};
    if (mx_launch_front_bwd(fba, &aparts[0], s)) return 1;
    if (optimise(h, true, aparts, ahead_grid, s)) return 1;
  }
  if (update_actor_out) *update_actor_out = update_actor ? 1 : 0;
  if (h->force_update_actor < 0) h->num_updates += 1;      // (graph replays count in mx_graph_launch)
  return 0;
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
  float* ws = src->ws;
  const MxMaddpgWs& W = src->W;
  const int B = b->B, T = c.episode_len, N = c.n_agents, Ac = c.act_dim;
  const int Ma = B * (T + 1) * N;
  const MxNetLayout& LA = src->actor;
  FrontFwdArgs ff;
  memset(&ff, 0, sizeof(ff));
  ff.tc_acc = ws + W.tc_acc; ff.tc_acc_cols = (int)W.tc_acc_cols;
  ff.X = b->obs; ff.ldx = b->obs_ld; ff.M = Ma; ff.feature_norm = c.no_feature_norm ? 0 : 1; ff.act_tanh = c.use_tanh;
  ff.theta[0] = src->th_a_tgt; ff.L = LA; ff.gi[0] = ws + W.a_gi[1];
  if (mx_launch_front_fwd(ff, 1, s)) return 1;
  if (c.mlp) {
    // maddpg.py:64-74: no recurrence, the head sits in the weight_ih slot (as maddpg_step_mlp phase A).  The noise rows are the
    // step-1 (next-observation) rows [b][2][N][Ac]; k_cent_scatter's row (b*(T+1)+t+1)*N+n with T = 1, t = 0 is that same step.
    MX_LAUNCH(k_mlp_head_cols, dim3(launch1d(Ma)), dim3(256), 0, s, (const float*)ff.gi[0], Ma, Ac, c.target_noise > 0.f ? target_noise_dev : nullptr,
              ws + W.a_nact, nullptr);
    MX_COUNT(); MX_MARK("k_mlp_head_cols", s);
  } else {
    GruFwdArgs gf;
    memset(&gf, 0, sizeof(gf));
    gf.theta[0] = src->th_a_tgt; gf.whh = LA.whh; gf.bhh = LA.bhh; gf.gi[0] = ff.gi[0]; gf.hall[0] = ws + W.a_h[1]; gf.R = B * N; gf.T = T; gf.N = N;
    if (mx_launch_gru_fwd(gf, 1, s)) return 1;
    HeadArgs ha;
    memset(&ha, 0, sizeof(ha));
    ha.lno_g = LA.lno_g; ha.lno_b = LA.lno_b; ha.w = LA.wq; ha.b = LA.bq; ha.OD = Ac; ha.b_stride = 1; ha.w_stride = MX_H; ha.M = Ma;
    ha.theta = src->th_a_tgt; ha.h = gf.hall[0]; ha.out = ws + W.a_nact; ha.noise = c.target_noise > 0.f ? target_noise_dev : nullptr;
    MX_LAUNCH(k_head_fwd, dim3(launch1d((long long)Ma * 32)), dim3(256), 0, s, ha); MX_COUNT(); MX_MARK("k_head_fwd", s);
  }
  if (c.discrete) {      // one-hot with the next-avail mask (MADDPG) / hard Gumbel-softmax (MATD3)
    ActXformArgs ax = act_xform_args(&c, Ma, c.target_noise > 0.f ? 1 : 0, b->avail, b->act_ld);
    ax.logits = ws + W.a_nact; ax.out = ws + W.a_nact;
    MX_LAUNCH(k_act_transform, dim3(launch1d(Ma)), dim3(256), 0, s, ax); MX_COUNT(); MX_MARK("k_act_transform", s);
  }
  MX_LAUNCH(k_cent_scatter, dim3(launch1d((long long)B * T * N * Ac)), dim3(256), 0, s, (const float*)(ws + W.a_nact), b->acts, b->act_ld, B, T, N, Ac,
            dst->ws + dst->W.cent_acts, dst->ws + dst->W.cent_nacts, mx_round_up(d.cent_act_dim, 4), c.act_offset);
  MX_COUNT(); MX_MARK("k_cent_scatter", s);
  return MX_CHECK_LAUNCH("cent_contribute");
}

// [sample ->] shared_train_policy_on_batch [-> PER write-back] [-> soft update] as one CUDA graph.  The actor is updated only
// every actor_update_interval-th call, so the caller records one graph per variant (update_actor = 1 / 0) and replays the one
// the update counter asks for; the noise buffers are fixed device buffers the caller refills before each launch.
extern "C" int mx_maddpg_graph_capture(mx_replay* r, mx_maddpg* h, int32_t B, double beta, uint32_t flags, const float* target_noise_dev,
                                       const float* actor_noise_dev, int32_t update_actor, void* stream, mx_graph** out) {
  if (!r || !h || !out) { mx_set_error("mx_maddpg_graph_capture: null argument"); return 1; }
  if (h->cfg.mlp && h->cfg.cent_act_dim > 0) {      // the graph would replay the step without the other policies' contributions
    mx_set_error("mx_maddpg_graph_capture: an MLP learner with several policies (cent_act_dim > 0) cannot be captured: its step needs "
                 "mx_maddpg_cent_contribute from every policy first; run it eagerly");
    return 1;
  }
  if ((flags & 2u) && mx_replay_set_beta(r, beta, stream)) return 1;
  auto seq = [=](void* st) -> int {
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
extern "C" int64_t mx_maddpg_num_updates(const mx_maddpg* h) { return h->num_updates; }

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
