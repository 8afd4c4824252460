/* marl_b200.h -- C-ABI of the H100-native recurrent off-policy MARL update engine (libmarl_b200.so).
 *
 * The reference (marlbenchmark/off-policy) is pure Python and has NO FFI/plugin interface
 * (SURVEY.md section 8(b)): the seam is Python class construction by dotted module path inside
 * offpolicy/runner/rnn/base_runner.py:7,110-178.  This header is therefore the boundary a maintainer
 * would bind with ctypes from drop-in classes of the same dotted names (see INTEGRATION.md); every
 * entry point below cites the reference function it replaces.
 *
 * Conventions
 *   - plain C: opaque handles, POD structs, raw pointers and sizes; no torch / C++ types.
 *   - every function returns 0 on success, non-zero on error; mx_last_error() gives the message
 *     (the reference signals errors with Python asserts/exceptions; the Python mirror re-raises).
 *   - nothing here allocates device memory: the caller owns every device buffer (sizes come from the
 *     *_layout / *_bytes queries, which need no GPU) and passes raw device pointers.  (A learner handle
 *     owns one non-blocking CUDA stream + a few events: kernels that do not depend on the agent nets run
 *     on that forked branch, ordered against the caller's stream by events -- parallel graph branches
 *     under stream capture.)
 *   - every launch is ordered on the cudaStream_t given (as void*), is asynchronous and never synchronises,
 *     except the calls documented as synchronising (mx_replay_restore, mx_replay_get_rng_state, mx_trng_seed / set_state /
 *     get_state, mx_profile_end).
 *     Host pointers given to *_async calls must stay valid until the stream reaches that point
 *     (cudaMemcpyAsync rules); use pinned memory for real asynchrony.
 *   - all floating-point data is fp32 unless stated; PER trees are fp64 like the reference
 *     (offpolicy/utils/segment_tree.py:38,104).
 */
#ifndef MARL_B200_H
#define MARL_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MX_ABI_VERSION 5
#define MX_MAX_NAME 64
#define MX_MAX_ACT_SEG 4       /* mx_maddpg_cfg.act_seg: MultiDiscrete sub-spaces per agent */

typedef struct mx_replay mx_replay;   /* one policy's episode store + sampler (RecPolicyBuffer + PER trees) */
typedef struct mx_qmix mx_qmix;       /* recurrent QMIX / VDN learner (QMix trainer + QMixPolicy nets + QMixer) */

const char* mx_last_error(void);
int mx_abi_version(void);
/* sizeof() of a public struct by its C name ("mx_batch", "mx_replay_cfg", "mx_replay_layout", "mx_qmix_cfg", "mx_maddpg_cfg",
 * "mx_param_entry", "mx_policy_step_args", "mx_episodes", "mx_trng_draw"); -1 for an unknown name.  Lets a binding written in another
 * language verify its struct mirrors at load time. */
int64_t mx_sizeof(const char* struct_name);
/* Host fences for pinned staging buffers a binding reuses: alloc once (id >= 0, -1 on error); record after enqueueing the copy that reads
 * the buffer; wait before rewriting it (returns at once if never recorded); release when the buffer is dropped (waits for its last
 * record; the id may then be handed out again).  Not thread-safe; at most 256 fences held at once per process. */
int mx_host_fence_alloc(void);
int mx_host_fence_record(int id, void* stream);
int mx_host_fence_wait(int id);
int mx_host_fence_release(int id);
/* 1 when built by nvcc for sm_90a, 0 for the CPU-emulated unit-test build (tests/emu; never shipped) */
int mx_is_cuda_build(void);

/* ------------------------------------------------------------------------------------------------
 * Episode replay (HBM-resident SoA, episode-major).
 * Replaces RecPolicyBuffer.__init__/insert/sample_inds (offpolicy/utils/rec_buffer.py:85-240),
 * RecReplayBuffer.sample (:62-82) and PrioritizedRecReplayBuffer (:243-324) + SumSegmentTree /
 * MinSegmentTree (offpolicy/utils/segment_tree.py).
 * ------------------------------------------------------------------------------------------------ */
typedef struct mx_replay_cfg {
  int32_t capacity;        /* buffer_size: max episodes                              rec_buffer.py:103 */
  int32_t episode_len;     /* T                                                      rec_buffer.py:104 */
  int32_t n_agents;        /* N                                                                        */
  int32_t obs_dim;         /* O                                                                        */
  int32_t share_dim;       /* S (use_same_share_obs=True layout: one state per step) rec_buffer.py:123 */
  int32_t act_dim;         /* A (one-hot width, or continuous action width)                            */
  int32_t use_avail;       /* store avail_acts                                       rec_buffer.py:131 */
  int32_t use_per;         /* allocate fp64 sum/min trees                            rec_buffer.py:252 */
  int32_t reward_norm;     /* use_reward_normalization                               rec_buffer.py:209 */
  int32_t max_batch;       /* largest batch_size that will be sampled                                  */
  double per_alpha;        /* PER exponent                                           rec_buffer.py:250 */
} mx_replay_cfg;

/* byte offsets of every region inside the single device blob the caller allocates for a replay */
typedef struct mx_replay_layout {
  int32_t obs_ld, share_ld, act_ld;         /* padded innermost strides (multiples of 4 floats)       */
  int64_t ep_obs, ep_share, ep_acts, ep_avail, ep_rew, ep_dones, ep_dones_env, ep_actidx; /* floats per episode (padded) */
  int64_t off_obs, off_share, off_acts, off_avail, off_rew, off_dones, off_dones_env, off_actidx;
  int64_t off_sum_tree, off_min_tree;       /* fp64 [2*tree_cap] each                                  */
  int64_t off_rng;                          /* uint32 key[624] + pos                                   */
  int64_t off_state;                        /* device scalars: filled, cursor, max_priority (fp64) ... */
  int64_t off_stage;                        /* staging area for one insert call (time-major raw)       */
  int64_t stage_bytes;
  /* batch region (the sampled batch, same field layout with capacity -> max_batch) */
  int64_t off_b_obs, off_b_share, off_b_acts, off_b_avail, off_b_rew, off_b_dones, off_b_dones_env, off_b_actidx;
  int64_t off_b_idx;                        /* int64 [max_batch]   sampled episode indices             */
  int64_t off_b_weights;                    /* fp64  [max_batch]   PER importance weights              */
  int64_t off_b_wf32;                       /* fp32  [max_batch]   same, as consumed by the learner    */
  int64_t off_rstats;                       /* fp64 [4]: masked sum, sumsq of r - K, count, K          */
  int32_t tree_cap;                         /* next pow2 >= capacity                                   */
  int64_t total_bytes;
} mx_replay_layout;

int mx_replay_layout_query(const mx_replay_cfg* cfg, mx_replay_layout* out);

/* `blob` = device memory of layout.total_bytes, zero-filled by the caller before create. */
int mx_replay_create(const mx_replay_cfg* cfg, void* blob, void* stream, mx_replay** out);
void mx_replay_destroy(mx_replay* r);

/* Ring insert of n_ep whole episodes (rec_buffer.py:146-190).  Arrays are the runner's time-major
 * host (or device) arrays: obs (T+1,n_ep,N,O), share_obs (T+1,n_ep,S) [agent axis already dropped],
 * acts (T,n_ep,N,A), rewards (T,n_ep,N), dones (T,n_ep,N), dones_env (T,n_ep), avail (T+1,n_ep,N,A)
 * or NULL.  `first_slot_out` receives current_i before the insert; slots wrap modulo capacity.
 * PER: every inserted slot's leaf is primed with max_priority**alpha (intent of rec_buffer.py:263-268). */
typedef struct mx_episodes {
  const float *obs, *share_obs, *acts, *rewards, *dones, *dones_env, *avail;
} mx_episodes;
int mx_replay_insert_async(mx_replay* r, const mx_episodes* ep, int32_t n_ep, int32_t* first_slot_out, void* stream);
/* Same insert from ONE packed host block (a single host->device copy): fields in the order obs, share_obs, acts,
 * rewards, dones, dones_env, avail, each starting at the 256-byte aligned offset reported by
 * mx_replay_insert_packed_layout (which returns the packed size in bytes for n_ep episodes). */
int64_t mx_replay_insert_packed_layout(const mx_replay* r, int32_t n_ep, int64_t offsets[7], int64_t counts[7]);
int mx_replay_insert_packed_async(mx_replay* r, const void* packed, int64_t nbytes, int32_t n_ep, int32_t* first_slot_out, void* stream);
/* Checkpoint / resume (SURVEY.md section 8(f).3; the reference saves network weights only, runner/rnn/base_runner.py:286-337):
 * the blob IS the replay's whole state (episodes, PER trees, MT19937 key, ring position), so a snapshot is a copy of the blob;
 * after copying one back, mx_replay_restore re-reads the host mirror of the ring position from it (synchronises). */
int mx_replay_restore(mx_replay* r, void* stream);
int32_t mx_replay_len(const mx_replay* r);      /* filled_i  (rec_buffer.py:36-37)  */
int32_t mx_replay_cursor(const mx_replay* r);   /* current_i                         */

/* NumPy legacy MT19937 state living on the device (np.random.seed / get_state, SURVEY.md App. C) */
int mx_replay_seed(mx_replay* r, uint32_t seed, void* stream);
int mx_replay_set_rng_state(mx_replay* r, const uint32_t key[624], int32_t pos, void* stream);
int mx_replay_get_rng_state(mx_replay* r, uint32_t key[624], int32_t* pos, void* stream); /* synchronises */

/* RecReplayBuffer.sample (rec_buffer.py:62-82): draw B indices with np.random.choice semantics from the
 * device-resident stream, then gather every field of those episodes into the batch region. */
int mx_replay_sample_uniform(mx_replay* r, int32_t B, void* stream);
/* Same gather for caller-provided indices (host-drawn np.random.choice keeps the process-global NumPy
 * stream shared with the env loop, exactly like the reference).  idx_dev: int64[B] on the device. */
int mx_replay_gather(mx_replay* r, const int64_t* idx_dev, int32_t B, void* stream);
/* same, indices in (pinned) host memory: one async H2D copy of B int64 + the gather */
int mx_replay_gather_host(mx_replay* r, const int64_t* idx_host, int32_t B, void* stream);
/* PrioritizedRecReplayBuffer.sample (rec_buffer.py:272-304): masses from np.random.random semantics,
 * fp64 prefix-sum descent, IS weights, gather. */
int mx_replay_sample_per(mx_replay* r, int32_t B, double beta, void* stream);
/* The PER draw inside a captured whole-step sequence (mx_graph_capture / mx_maddpg_graph_capture with flag 2) reads its
 * importance-sampling exponent from a device scalar, initialised with the `beta` given at capture.  The reference anneals beta
 * towards 1 on every train step (runner/rnn/base_runner.py:159-160,235 -> rec_buffer.py:278): call this before a mx_graph_launch
 * to change it (one tiny launch on `stream`, by-value argument, no synchronisation). */
int mx_replay_set_beta(mx_replay* r, double beta, void* stream);
/* update_priorities (rec_buffer.py:306-324): leaf = prio**alpha into both trees, duplicate idx: last wins;
 * max_priority = max(max_priority, max(prio)).  prio_dev fp32[B] (the trainer hands NumPy fp32), or pass
 * leaves_f64_dev != NULL to store pre-powered fp64 leaf values verbatim (parity tests). */
int mx_replay_update_priorities(mx_replay* r, const int64_t* idx_dev, const float* prio_dev,
                                const double* leaves_f64_dev, const double* max_prio_host, int32_t B, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Recurrent QMIX / VDN learner.
 * Replaces QMix.__init__/train_policy_on_batch/soft_target_updates/hard_target_updates
 * (offpolicy/algorithms/qmix/qmix.py:11-216), QMixPolicy.get_q_values/q_values_from_actions/
 * actions_from_q (qmix/algorithm/QMixPolicy.py:42-174), AgentQFunction.forward
 * (agent_q_function.py:34-67), RNNBase/MLPBase/ACTLayer (algorithms/utils/{rnn,mlp,act}.py),
 * QMixer.forward (q_mixer.py:68-94), clip_grad_norm_ + Adam (qmix.py:190-193), soft_update
 * (utils/util.py:123-134).
 * ------------------------------------------------------------------------------------------------ */
typedef struct mx_qmix_cfg {
  int32_t n_agents, obs_dim, act_dim, state_dim;   /* n_agents <= 32, act_dim <= 64 (SMAC: 6 + enemies, 36 on 27m_vs_30m) */
  int32_t hidden;            /* must be 64 (config.py:63 default)                  */
  int32_t mixer_hidden;      /* mixer_hidden_dim (32)                              */
  int32_t hyper_hidden;      /* hypernet_hidden_dim (64)                           */
  int32_t hyper_layers;      /* 1 or 2                                             */
  int32_t episode_len;       /* T                                                  */
  int32_t max_batch;         /* B upper bound (workspace sizing)                   */
  int32_t vdn;               /* 1: sum mixer (vdn_mixer.py:28-40 intent)           */
  int32_t double_q;          /* use_double_q                                       */
  int32_t use_huber;         /* use_huber_loss                                     */
  int32_t use_per;           /* importance weights + new priorities                */
  int32_t use_avail;         /* (informational) masks follow the batch: batch->avail may be NULL, e.g. MPE */
  int32_t world_size;        /* data-parallel ranks (1 = single GPU)               */
  float gamma, huber_delta, per_nu, per_eps;
  float lr, adam_beta1, adam_beta2, adam_eps, max_grad_norm, tau;
  int32_t prev_act_inp;      /* --prev_act_inp (config.py:81): the agent net's input is [obs | previous one-hot action]
                                (QMixPolicy.py:29,54-58; qmix.py:122-127: zeros at t = 0, then the buffer's actions) */
  int32_t mlp;               /* 1: the transition-level (non-recurrent) variant M_QMix / M_VDN (algorithms/mqmix/mqmix.py:67-216): the agent
                                net is MLPBase + Linear head without a GRU (mqmix/algorithm/agent_q_function.py), a "batch" is B single
                                transitions stored as episodes of length 1 (step 0 = obs, step 1 = next_obs), episode_len must be 1.
                                The head occupies the first act_dim rows of the (otherwise zero) weight_ih slot of the flat vector. */
  int32_t no_feature_norm;   /* 1: --use_feature_normalization switched off (config.py: store_false; mlp.py:64-65): the input LayerNorm
                                is skipped and its two tensors are absent from the parameter list */
  int32_t use_tanh;          /* 1: --use_ReLU switched off (config.py: store_false; mlp.py:12,19-22): tanh instead of ReLU in fc1 / fc2 */
} mx_qmix_cfg;

typedef struct mx_param_entry {
  char name[MX_MAX_NAME];    /* reference state_dict key, prefixed "agent." or "mixer." (SURVEY.md App. E) */
  int64_t offset;            /* in floats, inside the flat parameter vector; 16-byte aligned */
  int32_t rows, cols;        /* cols == 0 for 1-D tensors */
} mx_param_entry;

/* Flat parameter vector layout.  Returns the number of entries (<= max_entries); *total_floats = padded P. */
int mx_qmix_param_layout(const mx_qmix_cfg* cfg, mx_param_entry* out, int32_t max_entries, int64_t* total_floats);
int64_t mx_qmix_workspace_bytes(const mx_qmix_cfg* cfg);

/* device buffers, each `total_floats` fp32: theta (live), theta_tgt, adam_m, adam_v; workspace zero-filled. */
int mx_qmix_create(const mx_qmix_cfg* cfg, float* theta, float* theta_tgt, float* adam_m, float* adam_v,
                   void* workspace, int64_t workspace_bytes, mx_qmix** out);
void mx_qmix_destroy(mx_qmix* q);

/* The sampled batch (device pointers, episode-major, padded strides as in mx_replay_layout). */
typedef struct mx_batch {
  int32_t B;
  int32_t obs_ld, share_ld, act_ld;
  const float* obs;        /* [B][T+1][N][obs_ld]  */
  const float* share;      /* [B][T+1][share_ld]   */
  const float* acts;       /* [B][T][N][act_ld]  one-hot (unused by QMIX when act_idx given) */
  const int32_t* act_idx;  /* [B][T][N]            argmax of the one-hot action (QMixPolicy.py:89); episode stride ep_tn_ld */
  const float* avail;      /* [B][T+1][N][act_ld]  or NULL */
  const float* rewards;    /* [B][T][N]            agent 0's stream is used (qmix.py:159); episode stride ep_tn_ld */
  const float* dones;      /* [B][T][N]            (unused by QMIX) */
  const float* dones_env;  /* [B][T]               */
  const float* weights;    /* [B] fp32 PER importance weights or NULL */
  const int64_t* idx;      /* [B] or NULL */
  /* floats between consecutive episodes of the per-step fields: rewards / dones / act_idx (>= T*N) and dones_env (>= T).
   * 0 = dense.  The replay's batch region pads every episode row to 16 bytes, so it reports round_up(T*N, 4) / round_up(T, 4). */
  int32_t ep_tn_ld, ep_t_ld;
} mx_batch;
int mx_replay_batch(const mx_replay* r, int32_t B, mx_batch* out);   /* view of the replay's batch region */

/* One learner step = QMix.train_policy_on_batch (qmix.py:77-200): forward (live + target agent nets over
 * T+1 steps, mixers), TD target, masked MSE/Huber, BPTT, global-norm clip, Adam.  With world_size > 1 the
 * step stops after producing the flat gradient-numerator buffer; the caller all-reduces
 * mx_qmix_grad_buffer() (sum) and calls mx_qmix_apply(). */
int mx_qmix_step(mx_qmix* q, const mx_batch* batch, void* stream);
/* flags: MX_STEP_FUSE_SOFT_UPDATE -> the Adam kernel's epilogue also applies the Polyak target update
 * (= train_policy_on_batch immediately followed by soft_target_updates, base_runner.py:272-280, one launch fewer). */
#define MX_STEP_FUSE_SOFT_UPDATE 1u
int mx_qmix_step_ex(mx_qmix* q, const mx_batch* batch, uint32_t flags, void* stream);
int mx_qmix_apply_ex(mx_qmix* q, uint32_t flags, void* stream);
/* parity/debug: also materialise per-action Q values ("q_live"/"q_tgt") and greedy actions in the workspace */
int mx_qmix_set_debug(mx_qmix* q, int32_t on);
int mx_qmix_backward_only(mx_qmix* q, const mx_batch* batch, void* stream);  /* everything up to the reduced grads */
int mx_qmix_apply(mx_qmix* q, void* stream);                                 /* norm + clip + Adam + info scalars   */
/* flat fp32 buffer to all-reduce: [grad numerators (P) | sum(1-bad) | loss numerator | sum Q_tot(1-bad) | elements ] */
float* mx_qmix_grad_buffer(mx_qmix* q, int64_t* n_floats);
/* device fp32[4]: loss, grad_norm (pre-clip), Q_tot, denom -- qmix.py:195-198 */
const float* mx_qmix_info(mx_qmix* q);
/* device fp32[B] new PER priorities (qmix.py:179-181) valid after a step with use_per */
const float* mx_qmix_priorities(mx_qmix* q);

/* Data-parallel exchange over NVLink peer memory instead of an NCCL call (no reference counterpart: the reference is single
 * process; DESIGN.md section 6).  Every rank allocates one SYMMETRIC block of mx_qmix_p2p_block_bytes() (zero-filled, mapped into
 * every peer: torch.distributed._symmetric_memory / cudaIpc) and hands the world's block addresses, in rank order, to
 * mx_qmix_set_peers together with a zeroed local uint32 counter.  From then on mx_qmix_step[_ex] with world_size > 1 is complete:
 * backward -> publish (copy grad[P+4] into the own block, signal the peers) -> reduce (wait for every peer's signal, add all
 * blocks in rank order: bit-identical on every rank) -> clip + Adam.  The two halves are exported for tests. */
int64_t mx_qmix_p2p_block_bytes(const mx_qmix* q);
int mx_qmix_set_peers(mx_qmix* q, int32_t rank, int32_t world, void* const* peer_blocks, uint32_t* counter_dev);
int mx_qmix_p2p_publish(mx_qmix* q, void* stream);
int mx_qmix_p2p_reduce(mx_qmix* q, void* stream);

int mx_qmix_soft_update(mx_qmix* q, void* stream);   /* qmix.py:211-216 + util.py:123-134 (all registered params) */
int mx_qmix_hard_update(mx_qmix* q, void* stream);   /* qmix.py:203-209 */

/* ------------------------------------------------------------------------------------------------
 * Recurrent MADDPG / MATD3 learner (shared centralised observation, continuous actions).
 * Replaces R_MADDPG.shared_train_policy_on_batch / get_update_info (offpolicy/algorithms/r_maddpg/r_maddpg.py:44-331),
 * R_MADDPG_Actor / R_MADDPG_Critic forward (r_maddpg/algorithm/r_actor_critic.py:7-130), the two Adam steps and
 * soft/hard target updates of R_MADDPGPolicy (rMADDPGPolicy.py:53-54,162-170), and the R_MATD3 variants
 * (r_matd3/...: two Q heads, actor every 2nd update, Gaussian target-action noise).
 * ------------------------------------------------------------------------------------------------ */
typedef struct mx_maddpg mx_maddpg;
typedef struct mx_maddpg_cfg {
  int32_t n_agents, obs_dim, act_dim, state_dim;   /* act_dim: width of one agent's continuous action; state_dim = cent_obs_dim */
  int32_t hidden;                 /* must be 64 */
  int32_t episode_len, max_batch;
  int32_t num_q;                  /* Q heads: 1 (MADDPG) or 2 (MATD3)                    r_actor_critic.py:93 */
  int32_t actor_update_interval;  /* 1 (MADDPG) or 2 (MATD3)                             r_maddpg.py:125      */
  int32_t use_huber, use_per;
  float gamma, huber_delta, per_nu, per_eps;
  float lr, adam_beta1, adam_beta2, adam_eps, max_grad_norm, tau, weight_decay;
  float target_noise;             /* > 0: the caller passes noise for the target actions (MATD3): N(0, target_noise) samples for
                                     Box actions (util.py:217-218), Gumbel(0,1) draws for Discrete actions (util.py:127-130) */
  int32_t discrete;               /* 1: Discrete(act_dim) actions -- one-hot buffer actions, arg-max one-hot / hard Gumbel-softmax
                                     actor outputs (rMADDPGPolicy.py:104-120, util.py:106-166); 0: Box(act_dim)              */
  int32_t no_feature_norm;   /* 1: --use_feature_normalization switched off: no input LayerNorm in the actor and the critic */
  int32_t use_tanh;          /* 1: --use_ReLU switched off: tanh instead of ReLU in the fc1 / fc2 blocks of both networks */
  /* several policies (config.py:61 share_policy = False, train/train_mpe.py:139-150: one policy per agent, possibly with different
   * observation / action spaces): every policy owns one mx_maddpg for ITS n_agents agents; the centralised critic still sees the
   * actions of all agents.  cent_act_dim = total action width over all agents (policy_info['cent_act_dim']), act_offset = first
   * column of this policy's agents inside it.  0 / 0 = one shared policy (cent_act_dim = n_agents * act_dim). */
  int32_t cent_act_dim, act_offset;
  /* 1: transition-level MADDPG / MATD3 (algorithms/maddpg/maddpg.py:90-249, maddpg/algorithm/actor_critic.py): MLP actor and critic
   * without recurrence, a batch = B transitions stored as episodes of length 1 (episode_len must be 1; step 0 = obs, step 1 = next
   * obs).  The critic's K Q heads are not trained (a plain list in the reference, SURVEY.md App. D-6): the live and the target heads
   * are two fixed initialisations kept behind the critic's trunk, outside the range Adam, clipping and the target updates touch.
   * The actor loss is masked by valid_transition (mx_maddpg_set_valid).  Several policies work as in the recurrent learner
   * (cent_act_dim > 0, mx_maddpg_cent_contribute before every step).  mx_maddpg_graph_capture(_ex) takes one shared policy only;
   * several policies are captured together, a whole batch_train per graph, by mx_maddpg_batch_graph_capture (recurrent or mlp). */
  int32_t mlp;
  /* MultiDiscrete actions (envs/mpe/multi_discrete.py, act.py:15-17: one Linear head per sub-space): the action is n_act_seg one-hot
   * blocks of act_seg[i] columns, act_dim = their sum.  Arg-max, hard Gumbel-softmax and its straight-through gradient work per block,
   * and the available-action mask is ignored (MADDPGPolicy.py:73-89) -- also with n_act_seg = 1, which is a MultiDiscrete space of one
   * sub-space.  0 = one block of act_dim (Box / Discrete, the mask applies).  Segments need discrete and mlp (the recurrent learner
   * takes none and keeps act_dim <= 8).  The MLP learner takes act_dim <= 32 (Box, Discrete or MultiDiscrete). */
  int32_t n_act_seg;
  int32_t act_seg[MX_MAX_ACT_SEG];
} mx_maddpg_cfg;
/* which = 0: actor ("rnn.*", "act.action_out.*"), 1: critic ("rnn.*", "q_outs.k.*"); names = reference state_dict keys.
 * cfg.mlp: actor "mlp.*", "act.action_out.*" (with n_act_seg > 0: "act.action_outs.i.*", consecutive row blocks of one head); critic "mlp.*" (the trained trunk); which = 2: the critic's frozen heads "q_outs.k.*",
 * located in the live and in the target critic vector alike. */
int mx_maddpg_param_layout(const mx_maddpg_cfg* cfg, int32_t which, mx_param_entry* out, int32_t max_entries, int64_t* total_floats);
int64_t mx_maddpg_workspace_bytes(const mx_maddpg_cfg* cfg);
/* actor_vecs / critic_vecs: {theta, theta_target, adam_m, adam_v}, each of the layout's total_floats; workspace zero-filled */
int mx_maddpg_create(const mx_maddpg_cfg* cfg, float* const actor_vecs[4], float* const critic_vecs[4], void* workspace,
                     int64_t workspace_bytes, mx_maddpg** out);
void mx_maddpg_destroy(mx_maddpg* h);
/* One update = shared_train_policy_on_batch: critic update, then (every actor_update_interval-th call) the actor update with
 * the updated critic.  target_noise_dev: fp32 [(T+1)][B][N][act_dim] in batch row order (row = (b*(T+1)+t)*N + n) or NULL.
 * *update_actor_out tells the caller whether the actor was updated (train_info['update_actor']). */
int mx_maddpg_step(mx_maddpg* h, const mx_batch* batch, const float* target_noise_dev, int32_t* update_actor_out, void* stream);
/* Same, for Discrete actors: actor_noise_dev = the Gumbel(0,1) draws of the actor update's `use_gumbel=True` call
 * (r_maddpg.py:277), fp32 [B][T+1][N][act_dim] in batch row order (the t = T slice is ignored), required on calls that
 * update the actor; batch->avail (or NULL) masks unavailable actions to -1e10 like util.py:115,141. */
int mx_maddpg_step_ex(mx_maddpg* h, const mx_batch* batch, const float* target_noise_dev, const float* actor_noise_dev,
                      int32_t* update_actor_out, void* stream);
/* Several policies: r_maddpg.py:40-105 / maddpg.py:38-81 (get_update_info).  Runs src's TARGET actor over src_batch (noise as in
 * mx_maddpg_step_ex) and writes src's columns of the two centralised action vectors (buffer actions; target actions at t+1; for
 * cfg.mlp the next-observation step of the transition) into dst's workspace.  Before mx_maddpg_step_ex(dst, ...) call it once per
 * policy, dst itself included (same stream). */
int mx_maddpg_cent_contribute(mx_maddpg* src, const mx_batch* src_batch, const float* target_noise_dev, mx_maddpg* dst, void* stream);
/* Whole-update CUDA graph (declared with mx_graph below): [sample ->] step [-> PER write-back] [-> soft update when the actor
 * was updated, base_runner.py:250-252]; flags as for mx_graph_capture.  One graph per variant (update_actor = 1 / 0); the two
 * noise pointers are fixed device buffers the caller refills before every mx_graph_launch.  A learner of several policies
 * (cent_act_dim > 0) is refused: its step needs every policy's contribution first (mx_maddpg_batch_graph_capture). */
struct mx_graph;
int mx_maddpg_graph_capture(mx_replay* r, mx_maddpg* h, int32_t B, double beta, uint32_t flags, const float* target_noise_dev,
                            const float* actor_noise_dev, int32_t update_actor, void* stream, struct mx_graph** out);

/* torch's CPU generator on the device (the mt19937 behind torch.manual_seed / uniform_ / normal_): the noise draws of an update
 * without host work.  The state is caller-owned device memory of MX_TRNG_WORDS uint32: key[624], then torch's `left` and `next`
 * (the next word read is key[625 - left], after a twist when that is 624).  One fill reproduces one torch call on a contiguous float
 * tensor of shape (T, rows_n * rows_b, cols) -- it consumes exactly the words torch would, the uniforms are bit-identical, the Gumbel
 * and normal transforms agree with torch's to a few ulps -- and writes value (t, n * rows_b + b, c) to
 * dst[t * ld_t + n * ld_n + b * ld_b + c].  Kinds: uniform_; uniform_ then -log(-log(u + 1e-20) + 1e-20) (sample_gumbel,
 * utils/util.py:127-130); normal_(0, std) of >= 16 values (torch's Box-Muller over blocks of 16 with the redrawn tail block; a smaller
 * normal draw takes torch's scalar path and is refused). */
#define MX_TRNG_WORDS 640
#define MX_TRNG_UNIFORM 0
#define MX_TRNG_GUMBEL 1
#define MX_TRNG_NORMAL 2
typedef struct mx_trng_draw {
  int32_t kind;
  int32_t T, rows_n, rows_b, cols;   /* source shape (T, rows_n * rows_b, cols), rows agent-major: row = n * rows_b + b */
  float std;                         /* MX_TRNG_NORMAL */
  float* dst;                        /* device fp32, first column of the destination block */
  int64_t ld_t, ld_n, ld_b;          /* destination strides in floats */
} mx_trng_draw;
int mx_trng_seed(uint32_t* state_dev, uint64_t seed, void* stream);      /* torch.manual_seed(seed); synchronises */
int mx_trng_set_state(uint32_t* state_dev, const uint32_t key[624], int32_t left, int32_t next, void* stream);   /* synchronises */
int mx_trng_get_state(const uint32_t* state_dev, uint32_t key[624], int32_t* left, int32_t* next, void* stream); /* synchronises */
/* MT19937 words the fill consumes (the scratch it needs), or -1 and mx_last_error for a bad fill */
int64_t mx_trng_words(const mx_trng_draw* f);
/* Enqueue one fill on `stream` (two launches); advances the device state.  scratch_dev: device uint32[scratch_words >= mx_trng_words]. */
int mx_trng_fill(uint32_t* state_dev, const mx_trng_draw* f, uint32_t* scratch_dev, int64_t scratch_words, void* stream);
/* mx_maddpg_graph_capture with the update's noise draws at the head of the graph: the n_fills fills (in the order torch's calls would
 * make them, into target_noise_dev / actor_noise_dev) run from state_dev before the sample, so one mx_graph_launch is the whole update.
 * The fills share the scratch, which must hold the largest of them. */
int mx_maddpg_graph_capture_ex(mx_replay* r, mx_maddpg* h, int32_t B, double beta, uint32_t flags, const float* target_noise_dev,
                               const float* actor_noise_dev, int32_t update_actor, uint32_t* state_dev, const mx_trng_draw* fills,
                               int32_t n_fills, uint32_t* scratch_dev, int64_t scratch_words, void* stream, struct mx_graph** out);
/* Several policies (cent_act_dim > 0; mx_maddpg_graph_capture(_ex) refuses such a learner): one batch_train of the runner
 * (runner/{rnn,mlp}/base_runner.py) as one CUDA graph.  stores / learners: the P >= 2 policies' replays and learners in policy-id order
 * (act_offsets tiling cent_act_dim).  Per policy p: its fill_counts[p] fills (the next ones of `fills`, in the order torch's calls would
 * make them: the target noise of every policy q in id order, then p's actor draws), the sample (flags bit0: one uniform draw on
 * stores[uniform_store]; bit1: a PER draw from p's tree) gathered into every other store, mx_maddpg_cent_contribute of every q into p,
 * the step of p, and (bit3) the write-back to p's tree; then (bit2) the soft updates of all P learners in the update_actor variant.
 * target_noise_dev[p * P + q]: q's target noise in p's update; actor_noise_dev[p]: p's actor draws (NULL where none is taken; one
 * buffer may serve every p when the fills write it inside the graph).  Each replay advances every learner's update count. */
int mx_maddpg_batch_graph_capture(mx_replay* const* stores, mx_maddpg* const* learners, int32_t n_policies, int32_t uniform_store, int32_t B,
                                  double beta, uint32_t flags, const float* const* target_noise_dev, const float* const* actor_noise_dev,
                                  int32_t update_actor, uint32_t* state_dev, const mx_trng_draw* fills, const int32_t* fill_counts,
                                  uint32_t* scratch_dev, int64_t scratch_words, void* stream, struct mx_graph** out);
/* cfg.mlp: valid_transition of the transition store, device fp32 [rows][n_agents] (mlp_buffer.py:156).  The actor loss of a batch
 * reads row batch->idx[b] (row b when the batch has no indices); NULL: every transition is valid.  The pointer is kept, so a
 * captured graph reads the store as it is at replay time. */
int mx_maddpg_set_valid(mx_maddpg* h, const float* valid_dev);
int64_t mx_maddpg_num_updates(const mx_maddpg* h);   /* updates done so far (self.num_updates[p_id], r_maddpg.py:125) */
int mx_maddpg_set_num_updates(mx_maddpg* h, int64_t n);   /* restore the update count (checkpoint resume); n >= 0 */
/* Named workspace region (byte offset, length in 4-byte words): "adam_ta" / "adam_tc", the actor / critic Adam step counters (fp64)
 * a checkpoint saves beside the parameter vectors.  Non-zero and mx_last_error for an unknown name. */
int mx_maddpg_ws_lookup(const mx_maddpg* h, const char* name, int64_t* byte_offset, int64_t* n_elems);
/* device fp32[8]: critic_loss, critic_grad_norm, -, denom, actor_loss, actor_grad_norm, -, denom */
const float* mx_maddpg_info(mx_maddpg* h);
const float* mx_maddpg_priorities(mx_maddpg* h);
int mx_maddpg_grad_views(mx_maddpg* h, int64_t* actor_off_bytes, int64_t* critic_off_bytes);   /* parity tests: numerator grads in the workspace */
int mx_maddpg_soft_update(mx_maddpg* h, void* stream);   /* rMADDPGPolicy.py:162-165 */
int mx_maddpg_hard_update(mx_maddpg* h, void* stream);   /* rMADDPGPolicy.py:167-170 */

/* ------------------------------------------------------------------------------------------------
 * Rollout-time policy step (one env step of the runners' collect_rollout loops, runner/rnn/smac_runner.py:73-98,
 * runner/rnn/mpe_runner.py): ONE launch for the whole RNNBase + Linear-head forward of `rows` = n_envs * n_agents rows.
 * Replaces the single-step branch of QMixPolicy.get_q_values / get_actions (qmix/algorithm/QMixPolicy.py:42-67, 95-174, greedy
 * arg-max with the -1e10 availability mask of utils/util.py:297-302) and the actor forward of R_MADDPGPolicy.get_actions
 * (r_maddpg/algorithm/rMADDPGPolicy.py:77-103).  `theta` is a flat vector in the agent-net layout (mx_qmix_param_layout's
 * "agent." block / mx_maddpg_param_layout which = 0), i.e. the live or the target vector of a learner.  Exploration noise is
 * applied by the caller (the reference draws it from the process-global NumPy / torch CPU generators).
 * ------------------------------------------------------------------------------------------------ */
typedef struct mx_policy_step_args {
  const float* theta;      /* device: flat parameters of the network                                   */
  int32_t in_dim, out_dim; /* obs_dim, act_dim (hidden size is 64)                                     */
  int32_t rows;            /* n_envs * n_agents                                                        */
  int32_t x_ld, avail_ld;  /* row strides of x and avail in floats                                     */
  const float* x;          /* device [rows][x_ld]      observations of this step                       */
  const float* h_in;       /* device [rows][64]        recurrent state, or NULL for zeros (init_hidden) */
  float* h_out;            /* device [rows][64]        new recurrent state (may alias h_in)            */
  float* out;              /* device [rows][out_dim]   Q values / action logits / continuous actions   */
  const float* avail;      /* device [rows][avail_ld]  available-action mask or NULL                   */
  int32_t* greedy;         /* device [rows] arg-max action under the mask, or NULL                     */
  float* greedy_q;         /* device [rows] its value (the reference's greedy_Qs), or NULL             */
  float* h_copy;           /* optional second destination of the new state [rows][64] (e.g. mapped pinned host memory), or NULL */
  int32_t mlp;             /* 1: non-recurrent net (M_QMixPolicy.get_actions, mQMixPolicy.py:60-110): MLPBase -> head stored in the
                              weight_ih slot (see mx_qmix_cfg.mlp); h_in / h_out are ignored (h_out may be NULL) */
  int32_t no_feature_norm; /* 1: the network has no input LayerNorm (mx_qmix_cfg.no_feature_norm) */
  int32_t use_tanh;        /* 1: tanh instead of ReLU in fc1 / fc2 (mx_qmix_cfg.use_tanh) */
} mx_policy_step_args;
/* x / avail / out / greedy / greedy_q / h_copy may point into MAPPED PINNED HOST memory (cudaHostAlloc; same address on the
 * device under UVA): the kernel then reads the observation and writes the actions straight over PCIe and one env step costs one
 * launch + one stream synchronisation, no memcpy calls. */
int mx_policy_step(const mx_policy_step_args* args, void* stream);

/* Debug / parity: look up a named fp32 (or int32) region of the workspace written by the last step.
 * Returns byte offset into the workspace and element count; names are listed in DESIGN.md. */
int mx_qmix_ws_lookup(const mx_qmix* q, const char* name, int64_t* byte_offset, int64_t* n_elems);

/* Whole-step CUDA graph: [sample (uniform|per) ->] step [-> priority write-back] [-> soft update], captured once
 * and replayed.  flags: bit0 sample uniform, bit1 sample PER, bit2 soft update, bit3 PER write-back. */
typedef struct mx_graph mx_graph;
int mx_graph_capture(mx_replay* r, mx_qmix* q, int32_t B, double beta, uint32_t flags, void* stream, mx_graph** out);
int mx_graph_launch(mx_graph* g, void* stream);
void mx_graph_destroy(mx_graph* g);

/* Tensor-core building block probe (parity tests): Y[M][N] = X[M][K] . W[N][K]^T with wgmma on TF32
 * operands; passes = 1 (plain TF32) or 3 (3xTF32 hi/lo split, fp32-level accuracy); swap_ls selects which descriptor field
 * carries the K-direction core-matrix stride (the kernels use swap_ls = 0).  N % 16 == 0, N <= 256, K % 8 == 0, K <= 64. */
int mx_tc_linear_probe(const float* X, const float* W, float* Y, int32_t M, int32_t N, int32_t K, int32_t passes, int32_t swap_ls, void* stream);

/* Runtime options (process-wide switches between paths that are each the default for some input or build).
 * Returns 1 for an unknown name.  (default)
 *   front_tc (1)            time-batched front layers on the wgmma 3xTF32 kernels (inputs <= 128); 0 = the FFMA kernel
 *   wgrad_tc (-1)           backward of the front layers on the tensor cores: -1 = by input width (inputs > 64: mode 2), 0 = FFMA k_front_bwd,
 *                           1 = k_wgrad_tc beside k_front_bwd, 2 = k_front_bwd_tc + k_wgrad_tc
 *   overlap (1) / overlap_rows (2^20)   state-only kernels on a forked stream / graph branch: 0 off, 1 when B*(T+1)*N <= overlap_rows, 2 always
 *   mixer_split (1), mid_fused (1)      split hypernet / core mixer kernels; k_mid between the recurrences (0 = separate kernels)
 *   optim_fused (1)         one-launch reduce + [exchange] + clip + Adam + Polyak (0: k_grad_reduce + k_adam)
 *   p2p_ll (1)              data-parallel exchange as flag-in-data lines (0: slots + one flag per rank); p2p_timeout_ms (10000) wait for a peer
 *   gather_tma (1)          episode gather on the TMA unit (0: vectorised loads; 2: TMA at every size)
 *   pdl (-1)                programmatic dependent launch: -1 = QMIX steps of <= pdl_rows (12288) rows and the R-MADDPG update, 0 never, 1 always
 *   smem_carveout (100)     preferred shared-memory carveout (percent) of every step kernel; -1 = driver default */
int mx_set_option(const char* name, int32_t value);

/* number of kernel launches issued by this library since load (bench.py's gpu_launches counter) */
int64_t mx_launch_count(void);

/* Per-kernel device timing for bench.py's roofline: between begin and end every launch of this library on
 * `stream` is bracketed by CUDA events.  mx_profile_end synchronises the stream and returns the number of
 * launches; names are written ';'-separated into names_buf, durations in milliseconds into ms[]. */
int mx_profile_begin(void* stream);
int mx_profile_end(void* stream, char* names_buf, int32_t buf_len, float* ms, int32_t max_n);
/* number of kernel nodes one mx_graph_launch replays */
int32_t mx_graph_num_kernels(const mx_graph* g);

#ifdef __cplusplus
}
#endif
#endif
