// Rollout-time single step of an RNNBase + Linear-head network: the per-env-step policy call of the runners.
//
// reference: QMixPolicy.get_q_values / get_actions on one step (qmix/algorithm/QMixPolicy.py:42-67, 95-174; the greedy branch
// of actions_from_q with the -1e10 availability mask, utils/util.py:297-302) and the actor forward of
// R_MADDPGPolicy.get_actions (r_maddpg/algorithm/rMADDPGPolicy.py:77-103); network = algorithms/utils/{mlp,rnn,act}.py
// (LN -> fc1 -> ReLU -> LN -> fc2 -> ReLU -> LN -> GRU cell -> LN -> Linear).  The reference issues ~25 tiny ATen ops per env
// step; here it is ONE launch: one CTA per row (row = one agent of one env), activations in shared memory, every dot product
// split over 4 lanes.  Exploration noise (epsilon-greedy / Gumbel / Gaussian) stays on the host because the reference draws
// it from the process-global NumPy / torch CPU generators.
#include <math.h>
#include <string.h>

#include "mx_internal.h"
#include "mx_kernels.h"

#define MX_ROLL_THREADS 256
#define MX_ROLL_MAX_IN 1024

struct RollArgs {
  const float* theta;
  MxNetLayout L;
  const float* x; int x_ld;
  const float* h_in;       // [R][H] or null (zeros)
  float* h_out;            // [R][H]
  float* h_copy;           // optional second copy of the new state (mapped host memory) or null
  float* out;              // [R][out_dim]
  const float* avail; int avail_ld;
  int32_t* greedy;         // [R] or null
  float* greedy_q;         // [R] or null
  int R;
  int mlp;                 // non-recurrent net: head = first out_dim rows of the W_ih slot applied to the MLPBase output
  int no_feature_norm;     // no input LayerNorm (--use_feature_normalization switched off)
  int act_tanh;            // tanh instead of ReLU (--use_ReLU switched off)
};

// LayerNorm of v[0..n) in shared memory, in place (two-pass, biased variance, eps inside the sqrt like ATen); warp 0 only
MX_DEVINL void roll_layer_norm(float* v, int n, const float* __restrict__ g, const float* __restrict__ b) {
  const int lane = threadIdx.x & 31;
  if (threadIdx.x < 32) {
    float s = 0.f;
    for (int k = lane; k < n; k += 32) s += v[k];
    const float mean = mx_warp_sum(s) / (float)n;
    float q = 0.f;
    for (int k = lane; k < n; k += 32) { const float d = v[k] - mean; q = fmaf(d, d, q); }
    const float rstd = 1.0f / sqrtf(mx_warp_sum(q) / (float)n + MX_LN_EPS);
    for (int k = lane; k < n; k += 32) v[k] = (v[k] - mean) * rstd * g[k] + b[k];
  }
  __syncthreads();
}

// partial dot product of W[row][0..K) with v[0..K) over the k-slice of lane q (k = q, q+4, ...), reduced over the 4 lanes
MX_DEVINL float roll_dot4(const float* __restrict__ Wrow, const float* v, int K, int q) {
  float a = 0.f;
  for (int k = q; k < K; k += 4) a = fmaf(Wrow[k], v[k], a);
  a += __shfl_xor_sync(0xffffffffu, a, 1);
  a += __shfl_xor_sync(0xffffffffu, a, 2);
  return a;
}

__global__ void __launch_bounds__(MX_ROLL_THREADS) k_policy_step(RollArgs a) {
  __shared__ float xs[MX_ROLL_MAX_IN];
  __shared__ float v1[MX_H], v2[MX_H], hs[MX_H], hn[MX_H];
  __shared__ float qs[64];
  const int tid = threadIdx.x, u = tid >> 2, q = tid & 3;
  const MxNetLayout& L = a.L;
  const float* th = a.theta;
  const int I = L.in_dim, A = L.out_dim;
  for (int r = blockIdx.x; r < a.R; r += gridDim.x) {
    for (int k = tid; k < I; k += MX_ROLL_THREADS) xs[k] = a.x[(size_t)r * a.x_ld + k];
    if (tid < MX_H) hs[tid] = a.h_in ? a.h_in[(size_t)r * MX_H + tid] : 0.f;
    __syncthreads();
    if (!a.no_feature_norm) roll_layer_norm(xs, I, th + L.fn_g, th + L.fn_b);            // mlp.py:64-65 (block-uniform branch)
    {   // fc1: Linear -> ReLU -> LayerNorm                                               mlp.py:19-20
      const float d = roll_dot4(th + L.w1 + (size_t)u * I, xs, I, q);
      if (q == 0) { const float z = d + th[L.b1 + u]; v1[u] = a.act_tanh ? tanhf(z) : fmaxf(z, 0.f); }
    }
    __syncthreads();
    roll_layer_norm(v1, MX_H, th + L.ln1_g, th + L.ln1_b);
    {   // fc2[0]                                                                          mlp.py:21-29
      const float d = roll_dot4(th + L.w2 + (size_t)u * MX_H, v1, MX_H, q);
      if (q == 0) { const float z = d + th[L.b2 + u]; v2[u] = a.act_tanh ? tanhf(z) : fmaxf(z, 0.f); }
    }
    __syncthreads();
    roll_layer_norm(v2, MX_H, th + L.ln2_g, th + L.ln2_b);
    if (a.mlp) {   // M_QMixPolicy: Q = Linear(H, A)(MLPBase(x)); the head sits in the W_ih slot (agent_q_function.py:24-33)
      const float d = roll_dot4(th + L.wih + (size_t)(u < A ? u : 0) * MX_H, v2, MX_H, q);
      if (q == 0 && u < A) {
        const float o = d + th[L.bih + u];
        qs[u] = o;
        a.out[(size_t)r * A + u] = o;
      }
    } else {
    {   // GRU cell, PyTorch gate order [r; z; n]                                          rnn.py:8, 33-47
      float gi[3], gh[3];
#pragma unroll
      for (int g = 0; g < 3; ++g) {
        gi[g] = roll_dot4(th + L.wih + (size_t)(g * MX_H + u) * MX_H, v2, MX_H, q) + th[L.bih + g * MX_H + u];
        gh[g] = roll_dot4(th + L.whh + (size_t)(g * MX_H + u) * MX_H, hs, MX_H, q) + th[L.bhh + g * MX_H + u];
      }
      if (q == 0) {
        const float rg = 1.0f / (1.0f + expf(-(gi[0] + gh[0])));
        const float zg = 1.0f / (1.0f + expf(-(gi[1] + gh[1])));
        const float ng = tanhf(gi[2] + rg * gh[2]);
        const float hnew = (1.0f - zg) * ng + zg * hs[u];
        hn[u] = hnew;
        a.h_out[(size_t)r * MX_H + u] = hnew;                                             // carried state is the raw h' (rnn.py:21-23)
        if (a.h_copy) a.h_copy[(size_t)r * MX_H + u] = hnew;
      }
    }
    __syncthreads();
    roll_layer_norm(hn, MX_H, th + L.lno_g, th + L.lno_b);
    {   // head: Linear(H, out_dim)  (every lane runs the shuffles; rows >= out_dim are clamped and discarded)   act.py:19,32
      const float d = roll_dot4(th + L.wq + (size_t)(u < A ? u : 0) * MX_H, hn, MX_H, q);
      if (q == 0 && u < A) {
        const float o = d + th[L.bq + u];
        qs[u] = o;
        a.out[(size_t)r * A + u] = o;
      }
    }
    }
    __syncthreads();
    if (tid == 0 && a.greedy) {   // greedy action: unavailable actions forced to -1e10, first maximum wins (util.py:297-302, torch.max)
      int best = 0;
      float bv = 0.f;
      for (int k = 0; k < A; ++k) {
        const float v = (a.avail && a.avail[(size_t)r * a.avail_ld + k] == 0.f) ? -1e10f : qs[k];
        if (k == 0 || v > bv) { bv = v; best = k; }
      }
      a.greedy[r] = best;
      if (a.greedy_q) a.greedy_q[r] = bv;
    }
    __syncthreads();
  }
}

extern "C" int mx_policy_step(const mx_policy_step_args* p, void* stream) {
  if (!p || !p->theta || !p->x || (!p->h_out && !p->mlp) || !p->out) { mx_set_error("mx_policy_step: null argument"); return 1; }
  if (p->rows <= 0) { mx_set_error("mx_policy_step: rows must be positive"); return 1; }
  if (p->in_dim <= 0 || p->in_dim > MX_ROLL_MAX_IN) { mx_set_error("mx_policy_step: in_dim %d outside [1, %d]", p->in_dim, MX_ROLL_MAX_IN); return 1; }
  if (p->out_dim <= 0 || p->out_dim > 64) { mx_set_error("mx_policy_step: out_dim %d outside [1, 64]", p->out_dim); return 1; }
  if (p->x_ld < p->in_dim || (p->avail && p->avail_ld < p->out_dim)) { mx_set_error("mx_policy_step: row stride smaller than the row"); return 1; }
  RollArgs a;
  memset(&a, 0, sizeof(a));
  a.theta = p->theta;
  mx_net_layout(p->in_dim, p->out_dim, 0, &a.L);
  a.x = p->x; a.x_ld = p->x_ld; a.h_in = p->h_in; a.h_out = p->h_out; a.h_copy = p->h_copy; a.out = p->out;
  a.avail = p->avail; a.avail_ld = p->avail_ld; a.greedy = p->greedy; a.greedy_q = p->greedy_q; a.R = p->rows; a.mlp = p->mlp; a.no_feature_norm = p->no_feature_norm; a.act_tanh = p->use_tanh;
  int grid = p->rows;
  const int cap = mx_num_sms() * 4;
  if (grid > cap) grid = cap;
  cudaStream_t s = (cudaStream_t)stream;
  return mx_launch("k_policy_step", k_policy_step, dim3(grid), dim3(MX_ROLL_THREADS), 0, s, MX_PLAIN, a);
}
