// Kernel argument blocks + launcher prototypes (internal).
#pragma once
#include "mx_internal.h"

struct FrontFwdArgs {
  const float* X;          // [M][ldx] dense input rows
  int ldx, M;
  int feature_norm;
  const float* theta[2];   // live, target flat parameter vectors
  MxNetLayout L;
  float* gi[2];            // [M][3H]
  float *u1, *u2;          // live: post-ReLU pre-LN activations [M][H]
  float *st0, *st1, *st2;  // live: (mean, rstd) per row for the three LayerNorms
  const float* tc_img[2];  // optional: pre-split TF32 hi/lo weight images in the wgmma operand layout (mx_launch_tc_prep_weights)
  float* tc_acc;           // with tc_img: the tensor-core accumulators, tc_acc_cols x 128 floats (CTAs x columns per CTA <= tc_acc_cols)
  int tc_acc_cols;
  int act_tanh;            // 1: tanh instead of ReLU after fc1 / fc2 (--use_ReLU switched off)
};
size_t mx_tc_image_floats(int in_dim);
// accumulator floats a learner's tensor-core launches over at most M rows need (FrontFwdArgs / FrontBwdArgs tc_acc); columns = floats / 128
size_t mx_tc_acc_floats(int64_t M);
int mx_launch_tc_prep_weights(const float* const theta[2], const MxNetLayout& L, float* const img[2], int nets, cudaStream_t s);
size_t mx_front_fwd_smem(int in_dim, int RM);
int mx_launch_front_fwd(const FrontFwdArgs& a, int nets, cudaStream_t s);

// prev_act_inp: X[m] = [obs[m] | acts[b][t-1][n]] (zeros at t = 0) for m = (b (T+1) + t) N + n   (qmix.py:122-127)
int mx_launch_pack_prev_act(const float* obs, int obs_ld, const float* acts, int act_ld, float* X, int ldx, int B, int T, int N, int O, int A,
                            cudaStream_t s);

struct GruFwdArgs {
  const float* theta[2];
  int whh, bhh;
  const float* gi[2];
  float* hall[2];          // [M][H]  h_t after step t
  float* gates;            // live [M][3H] (r, z, n)
  float* hn;               // live [M][H]  W_hn h + b_hn
  int R, T, N;             // rows, steps-1 (the kernel runs T+1 steps), agents interleaved per step (m = (b*(T+1)+t)*N + n)
  const float* h0;         // optional initial hidden state [R][H] (branch steps); null -> zeros
};
int mx_launch_gru_fwd(const GruFwdArgs& a, int nets, cudaStream_t s);

struct QHeadArgs {
  const float* theta[2];
  int wq, bq, lno_g, lno_b;
  const float* hall[2];
  float* sto;              // live post-GRU LN stats [M][2]
  const int32_t* act_idx;  // [B][T][N]
  const float* avail;      // [M][act_ld] or null
  int act_ld;
  int M, T, N, A, double_q;
  int ld_tn;               // floats between consecutive episodes of act_idx (>= T*N)
  float *q_taken, *q_next; // [B*T][N]
  int32_t* greedy;         // [M] (debug)
  float *qall0, *qall1;    // [M][A] (debug) or null
};
int mx_launch_qhead(const QHeadArgs& a, cudaStream_t s);

struct MixerArgs {
  const float *theta, *theta_tgt;
  MxMixLayout L;
  int vdn;
  const float* share;      // [B][T+1][share_ld]
  int share_ld;
  const float *q_taken, *q_next;   // [E][N]
  const float* rewards;    // [B][T][N]
  const float* dones_env;  // [B][T]
  const float* weights;    // [B] or null
  int B, T, N;
  int ld_tn, ld_t;         // floats between consecutive episodes of rewards (>= T*N) and dones_env (>= T)
  float gamma, huber_delta;
  int use_huber;
  float *qtot, *qtot_next, *err;   // [E]
  float* dq_taken;         // [E][N]
  float* gpart;            // [npart][P]   this kernel writes the mixer slice of partial blockIdx.x
  long long P;
  float* spart;            // [npart][8]   (sum(1-bad), loss numerator, sum Q_tot(1-bad))
  // ---- split pipeline (mx_launch_mix_hyper_fwd / _core / _hyper_bwd): per-element hypernet outputs kept in global memory so
  // that the state-only hypernet layers run beside the agent-net kernels instead of between them (row strides gH/gP/gM floats)
  float *hyp_h1, *hyp_h2, *hyp_hb;                        // live [E][gH]: post-ReLU hidden layers of hyper_w1 / hyper_w2 / hyper_b2
  float *hyp_p1[2], *hyp_b1[2], *hyp_p2[2], *hyp_b2[2];   // [live|target]: raw hyper_w1 out [E][gP], hyper_b1 [E][gM], hyper_w2 [E][gM], b2 [E]
  float *d_q, *d_hp, *d_p2, *d_p1;                        // dL/dQ_tot [E], d(hidden pre-ELU) [E][gM], d(hyper_w2 out) [E][gM], d(hyper_w1 out) [E][gP]
  int gH, gP, gM;
  // ---- wide-state path (mx_mix_wide_state): the hypernetworks' state-reading first layers run as one tensor-core GEMM (mixer_wide.cu);
  // the hypernet kernels read its pre-activations instead of the state rows and hand back the gradient at them
  int wide;
  MxMixWide wl;
  float* wimg;             // [net][hi Cp*Sp | lo Cp*Sp | bias Cp]: TF32 hi / lo split of the stacked state-layer weights, row-major
  float* pre;              // [net][B*(T+1)][Cp]: state-layer pre-activations (bias added, no activation) of every state row
  float* d_pre;            // [E][Cp]: live net's gradient at those pre-activations (ReLU-masked where the layer has one)
};
int mx_launch_mixer(const MixerArgs& a, int* nparts_used, cudaStream_t s);
// wide-state path (mixer_wide.cu): weight images + state-layer GEMM (before the hypernet forward), state-layer weight gradient (after the
// hypernet backward: writes the state layers' weights and biases as gradient partial 0)
int mx_launch_mixw_state_fwd(const MixerArgs& a, cudaStream_t s);
int mx_launch_mixw_state_wgrad(const MixerArgs& a, cudaStream_t s);
size_t mx_mixw_image_floats(const MxMixWide& w);
// split form of the same computation (k_mixer == hyper_fwd ; core ; hyper_bwd).  hyper_fwd depends only on the batch's states and
// the parameters, hyper_bwd only on core's outputs: the learner runs them on a forked branch next to the agent-net kernels.
int mx_mixer_split_supported(const MxMixLayout& L);
int mx_launch_mix_hyper_fwd(const MixerArgs& a, cudaStream_t s);
int mx_launch_mix_core(const MixerArgs& a, int* scalar_parts_used, cudaStream_t s);
int mx_launch_mix_hyper_bwd(const MixerArgs& a, int* nparts_used, cudaStream_t s);

// k_qhead + k_mix_core + k_qhead_bwd in one launch (mid.cu); `mix` carries the hypernet outputs / mixer scalars, the rest is the head
struct MidArgs {
  MixerArgs mix;
  int wq, bq, lno_g, lno_b;
  const float* hall[2];    // live, target [M][H]
  const int32_t* act_idx;  // [B][T][N]
  const float* avail;      // [M][act_ld] or null
  int act_ld;
  int T, N, A, double_q;
  int ld_tn;               // episode stride of act_idx (rewards / dones_env strides are in `mix`)
  float* dh_out;           // [M][H]
  float* gpart;            // head + post-GRU LayerNorm gradient partial of CTA blockIdx.x
  long long P;
};
int mx_mid_supported(const MidArgs& a);
int mx_launch_mid(const MidArgs& a, int* parts_used, cudaStream_t s);   // parts_used: gradient partials == scalar partials

// ---- transition-level MLP variant (cfg.mlp): the Q head is the first A rows of the W_ih slot, so Q[m][k] = gi[m][k] ----
struct MlpQSelArgs {
  const float* gi[2];      // live, target [M][3H]: columns [0, A) are the Q values of row m = (b*2 + t)*N + n
  const int32_t* act_idx;  // [B][1][N] (episode stride ld_tn)
  const float* avail;      // [M][act_ld] or null (rows t = 1 = next_avail)
  int act_ld, ld_tn;
  int B, N, A, double_q;
  float *q_taken, *q_next; // [B][N]
  float *qall0, *qall1;    // debug [M][A] or null
  int32_t* greedy;         // debug [M] or null
};
int mx_launch_mlp_qselect(const MlpQSelArgs& a, cudaStream_t s);
// dgi[M][3H] = 0 except (row of step 0, column act) = dq_taken[b][n]
int mx_launch_mlp_dgi(const float* dq_taken, const int32_t* act_idx, int ld_tn, float* dgi, int B, int N, cudaStream_t s);

struct QHeadBwdArgs {
  const float* theta;
  int wq, bq, lno_g, lno_b;
  const float* hall;       // live [M][H]
  const float* sto;        // [M][2]
  const int32_t* act_idx;
  const float* dq_taken;   // [E][N]
  int M, T, N, A;
  int ld_tn;               // episode stride of act_idx
  float* dh_out;           // [M][H]
  float* gpart;
  long long P;
};
int mx_launch_qhead_bwd(const QHeadBwdArgs& a, int* nparts_used, cudaStream_t s);

struct GruBwdArgs {
  const float* theta;
  int whh;
  const float* hall;       // live [M][H]
  const float* gates;      // [M][3H]
  const float* hn;         // [M][H]
  const float* dh_out;     // [M][H]
  float* dgi;              // [M][3H]   d(loss)/d(gi) ; rows t >= TB are zero-filled
  int R, T, N;             // T = number of steps to back-propagate (TB)
  int T1;                  // steps per sequence in memory (0 -> T + 1, the QMIX layout where the bootstrap step has no gradient)
  const float* h0;         // optional initial hidden state [R][H] used as h_{-1}; null -> zeros
};
int mx_launch_gru_bwd(const GruBwdArgs& a, cudaStream_t s);

struct FrontBwdArgs {
  const float* X;          // [M][ldx]
  int ldx, M, T, N;         // T: episode length when T1 == 0 (steps per sequence = T + 1)
  int T1;                   // steps per sequence in memory (0 -> T + 1)
  const float* h0;          // optional h_{-1} rows [M / T1 ...]: only for T1 == 1 branch rows ([M][H])
  int feature_norm;
  const float* theta;
  MxNetLayout L;
  const float *u1, *u2, *st0, *st1, *st2;
  const float* dgi;        // [M][3H]
  const float* gates;      // [M][3H] (r needed for dgh_n)
  const float* hall;       // [M][H]
  float* gpart;
  long long P;
  int no_gru;              // 1: MLP variant -- no recurrent weights: gates / hall are not read, dW_hh / db_hh are not produced
  float* dX;               // optional: gradient w.r.t. the input rows [M][ldx] (through the feature LayerNorm)
  int skip_wgrad;          // 1: data gradient only (frozen network)
  // tensor-core weight gradients (tc_bwd.cu, option wgrad_tc): when both buffers are given and the option is on, k_front_bwd keeps
  // the data-gradient chain and the LayerNorm gain / bias gradients, writes the two intermediate row gradients here, and
  // k_wgrad_tc produces every dW / db of the front layers and the GRU input / recurrent matrices from them
  float *da2_out, *da1_out;   // [M][H] each: gradient at the fc2 / fc1 pre-activation outputs (after the ReLU mask)
  int wgrad_external;      // set by the launcher, not by callers
  float* tc_imgT;          // scratch for the transposed TF32 weight images of the all-tensor-core backward (option wgrad_tc = 2)
  int tc_imgT_ready;       // 1: the caller already built them for the current parameters (mx_launch_tc_prep_weights_T)
  float* tc_acc;           // with tc_imgT or the tensor-core weight gradients: accumulators, as FrontFwdArgs::tc_acc
  int tc_acc_cols;
  int act_tanh;            // 1: tanh instead of ReLU (the saved u1 / u2 are the activations' outputs: tanh' = 1 - u^2)
  float* ln_part;          // optional [ln_part_rows][512] side array: lets k_front_bwd_tc run more CTAs than there are gradient partial rows (streamed mode)
  int ln_part_rows;
  int gru_wgrad_ext;       // 1: dW_ih / dW_hh / db_ih / db_hh come from k_gru_wgrad (mx_launch_gru_wgrad with these same arguments), not from k_front_bwd
};
bool mx_gru_wgrad_split_usable(const FrontBwdArgs& a);      // with gru_wgrad_ext = 0
int mx_launch_gru_wgrad(const FrontBwdArgs& a, cudaStream_t s);
int mx_launch_tc_prep_weights_T(const float* theta, const MxNetLayout& L, float* imgT, cudaStream_t s);
bool mx_tc_prep_T_wanted(int in_dim);
size_t mx_tc_imageT_floats(int in_dim);
int mx_launch_front_bwd(const FrontBwdArgs& a, int* nparts_used, cudaStream_t s);
// the widest agent-net input k_front_bwd's shared memory holds (gru_ext: with k_gru_wgrad beside it, as in the recurrent QMIX step);
// the learners refuse wider inputs at creation
int mx_front_bwd_max_in_dim(bool gru_ext);
int mx_launch_wgrad_tc(const FrontBwdArgs& a, int nparts, cudaStream_t s);
bool mx_wgrad_tc_usable(const FrontBwdArgs& a);

struct OptimArgs {
  float *theta, *theta_tgt, *adam_m, *adam_v;
  const float* gpart;
  float* grad;             // [P + 8]
  long long P;             // parameters the optimiser updates: [0, P) of theta / theta_tgt / adam_m / adam_v
  long long gpart_ld;      // floats between consecutive gradient partials (0: P); larger when the partials also hold frozen tensors past P
  int seg_begin[8], seg_end[8], seg_parts[8], nseg;   // parameter segments and how many partials each has
  const float* spart;
  int spart_n;
  float* info;             // [8]
  const float* abort;      // k_adam applies nothing while *abort < 0 (a peer-memory exchange timed out); null: info[7] is that word
  double* adam_t;          // [4]
  // loss / PER finalisation
  const float* err;        // [B][T] masked TD errors
  int B, T;
  float per_nu, per_eps;
  float* prio;             // [B] or null
  float lr, beta1, beta2, eps, max_grad_norm, tau;
  int world_size;
  float* normpart;          // [mx_grad_reduce_blocks(P)] per-block sum of squares of the reduced numerators (k_grad_reduce -> k_adam),
  int normpart_n;           //   or null when the gradient is all-reduced in between (world_size > 1)
  int fuse_polyak;          // Adam epilogue also applies the soft target update (graph mode)
  float weight_decay;       // torch.optim.Adam(weight_decay): g += wd * p after clipping
  // k_optim_fused: grid barrier words (device, zero-initialised): [0] exchange arrivals, [1] barrier arrivals, [2] barrier generation,
  // [3] sticky abort flag (a peer never arrived)
  unsigned* sync;
  int phase;                // k_optim_fused: 0 = whole kernel (grid barrier); 1 / 2 = the halves before / after the barrier as two launches (emulator)
  // data-parallel exchange over peer memory (p2p.cu layout): base of every rank's symmetric block, floats per slot, rank / world (0: none)
  float* p2p_blocks[16];
  unsigned long long p2p_timeout_ns;      // a peer that has not delivered after this long sets the sticky abort word (option p2p_timeout_ms, default 10 s)
  int p2p_ll;              // 1: flag-in-data exchange lines (option p2p_ll, default); 0: slots + one flag per rank
  float* xstat;             // [8] accumulated by the scalar block (data parallel only): ns spent in push+fence, wait for peers, local sum; launches; max wait
  long long p2p_slot;
  int p2p_rank, p2p_world;
};
static inline int mx_grad_reduce_blocks(long long P) { return (int)((P + 255) / 256); }   // 256 parameters per block
int mx_launch_grad_reduce(const OptimArgs& a, cudaStream_t s);
int mx_launch_adam(const OptimArgs& a, cudaStream_t s);
// reduce + [peer-memory all-reduce] + clip + Adam [+ Polyak] in ONE launch (grid barrier); returns -1 when the configuration cannot use
// it (the caller then launches k_grad_reduce / [exchange] / k_adam)
int mx_launch_optim_fused(const OptimArgs& a, cudaStream_t s);
extern int g_mx_optim_fused;
int mx_launch_polyak(float* tgt, const float* src, long long n, float tau, cudaStream_t s);
