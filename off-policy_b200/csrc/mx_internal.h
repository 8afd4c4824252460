// Internal host-side structures shared by the translation units of libmarl_b200.
#pragma once
#include "../../include/marl_b200.h"
#include "mx_common.cuh"

#include <functional>
#include <string>

void mx_set_error(const char* fmt, ...);
extern long long g_mx_launches;
extern int g_mx_prof_on;
void mx_prof_mark(const char* name, cudaStream_t s);
extern int g_mx_mixer_split, g_mx_overlap, g_mx_overlap_rows, g_mx_mid_fused, g_mx_optim_fused, g_mx_p2p_ll, g_mx_p2p_timeout_ms;
int mx_set_option_common(const char* name, int value);   // 0 when `name` was one of the build-independent options
#define MX_MARK(name, s) do { if (g_mx_prof_on) mx_prof_mark((name), (s)); } while (0)

#if MX_EMU
static inline int mx_num_sms() { return 4; }
static inline int mx_check_launch(const char*) { return 0; }
#else
int mx_num_sms();
int mx_check_launch(const char* what);
#endif

// ---- launching a kernel ------------------------------------------------------------------------------------------------------------
// Every kernel launch goes through mx_launch: it raises the kernel's dynamic shared-memory limit when `smem` needs it, applies the
// launch policy of `kind`, launches, counts the launch (mx_launch_count), marks `name` for the profiler and returns the launch status:
// 0, MX_ERR_SMEM when the kernel cannot be given `smem` bytes (mx_last_error says so), or mx_check_launch's code.
//
// MX_STEP launches are the learner-step kernels, whose device code calls MX_PDL_WAIT():
//  * Programmatic dependent launch (PDL).  Such a kernel may begin while its stream predecessor is still running; everything it does
//    before MX_PDL_WAIT() overlaps the predecessor's tail, so that part may only touch state the predecessor does not write: its own
//    shared memory / tensor-core accumulator and the parameter vectors theta / theta_target.  Those are written only by the optimiser
//    kernels, which call MX_PDL_THETA_WRITTEN() so that the NEXT launch is a plain, fully ordered one.
//  * Kernels of the two branches of a step only share an SM if the SM's L1 / shared-memory split, fixed while any CTA is resident,
//    leaves room for both: every step kernel asks for the largest shared-memory carveout (option smem_carveout, percent; < 0 = driver
//    default), once per kernel and again after the option changes.
// MX_PLAIN launches (replay, rollout, exchange, noise and actor-critic head kernels, the probe) are ordinary launches.
enum MxLaunchKind { MX_PLAIN, MX_STEP };
constexpr size_t MX_SMEM_OPTIN_MAX = 227 * 1024;   // dynamic shared memory one block may opt in to on sm_90
constexpr int MX_ERR_SMEM = 1;

#if MX_EMU
template <typename... KArgs, typename... Args>
static inline int mx_launch(const char* name, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, MxLaunchKind,
                            Args&&... args) {
  emu::launch(grid, block, smem, [&]() { kern(args...); });
  ++g_mx_launches;
  MX_MARK(name, s);
  return 0;
}
#else
int mx_launch_config(const char* name, const void* kern, size_t smem, MxLaunchKind kind, cudaLaunchConfig_t* cfg);   // opt-in, carveout, PDL
int mx_launch_done(const char* name, cudaStream_t s);                                                              // count, mark, check
template <typename... KArgs, typename... Args>
static inline int mx_launch(const char* name, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, MxLaunchKind kind,
                            Args&&... args) {
  cudaLaunchAttribute at[1];
  cudaLaunchConfig_t cfg;
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
  cfg.attrs = at; cfg.numAttrs = 0;
  if (const int rc = mx_launch_config(name, reinterpret_cast<const void*>(kern), smem, kind, &cfg)) return rc;
  cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
  return mx_launch_done(name, s);
}
#endif

// whole-step CUDA graph (qmix.cu): the recorded launch sequence, kept for the emulated build which simply re-runs it
struct mx_graph {
#if !MX_EMU
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t exec = nullptr;
#endif
  std::function<int(void*)> seq;
  std::function<void()> after_launch;     // host-side bookkeeping a replay must repeat (e.g. the learner's update counter)
  int n_kernels = 0;
};
int mx_graph_capture_seq(std::function<int(void*)> seq, std::function<void()> after_launch, void* stream, mx_graph** out);

// ---- replay ------------------------------------------------------------------------------------
struct MxReplayState {   // device-resident scalars (off_state)
  int32_t filled;
  int32_t cursor;
  int32_t rng_pos;
  int32_t pad;
  double max_priority;
  double reward_mean, reward_std;
  double per_beta;          // importance-sampling exponent read by the captured PER draw (mx_replay_set_beta); eager calls pass it by value
};

struct mx_replay {
  mx_replay_cfg cfg;
  mx_replay_layout L;
  char* blob;
  int32_t filled, cursor;   // host mirror (inserts are host-driven)
  void* tma = nullptr;      // tensor maps of the fields (gather_tma.cu), null: vectorised gather
};
void* mx_gather_tma_create(mx_replay* r);
void mx_gather_tma_destroy(void* p);
int mx_launch_gather_tma(void* p, const int64_t* idx_dev, int B, cudaStream_t s);     // -1: not available
extern int g_mx_gather_tma;

// ---- agent net / mixer parameter layouts (offsets in floats inside the flat vector) --------------
struct MxNetLayout {       // RNNBase (LN -> fc1 -> LN -> fc2 -> LN -> GRU -> LN) + Linear head
  int in_dim, out_dim;
  int fn_g, fn_b;
  int w1, b1, ln1_g, ln1_b;
  int wh, bh, lnh_g, lnh_b;   // fc_h: registered, unused in forward (mlp.py:21-29); polyak-averaged only
  int w2, b2, ln2_g, ln2_b;
  int wih, whh, bih, bhh;
  int lno_g, lno_b;
  int wq, bq;
  int size;                   // floats, multiple of 4
};
struct MxMixLayout {
  int S, N, ME, HY, layers;
  int w1a, b1a, w1b, b1b;     // hyper_w1: (layers==2) Linear(S,HY) -> ReLU -> Linear(HY,N*ME); (layers==1) only "b" = Linear(S,N*ME)
  int w2a, b2a, w2b, b2b;     // hyper_w2
  int wb1, bb1;               // hyper_b1 Linear(S,ME)
  int wb2a, bb2a, wb2b, bb2b; // hyper_b2 Linear(S,HY) -> ReLU -> Linear(HY,1)
  int size;
};
int mx_net_layout(int in_dim, int out_dim, int base, MxNetLayout* L);
int mx_mix_layout(int S, int N, int ME, int HY, int layers, int base, MxMixLayout* L);
// Wide-state path: the hypernetworks' four state-reading first layers stacked as the columns of one GEMM.  Block order: 0 = hyper_w1
// (w1a, or w1b with 1-layer hypernets), 1 = hyper_w2 (w2a / w2b), 2 = hyper_b2's first layer (wb2a, ReLU), 3 = hyper_b1 (wb1).
struct MxMixWide {
  int C, Cp, Sp;              // stacked columns per net, padded to 16; state width padded to the GEMM's K chunk
  int col[4], rows[4], w[4], b[4];   // block: first column (multiple of 4), rows, weight / bias offsets in the flat parameters
};
// true when the hypernet tile of the shared-memory mixer kernels does not fit in an SM at its largest tile height: such a learner takes
// the wide-state path.  Depends on the layout only (not on the build, the batch size or the device).
bool mx_mix_wide_state(const MxMixLayout& L);
void mx_mix_wide_layout(const MxMixLayout& L, MxMixWide* w);

// ---- QMIX learner workspace -----------------------------------------------------------------------
struct MxQmixWs {           // offsets in floats into the workspace
  int64_t gi[2], hall[2];   // [net][M][3H], [net][M][H]
  int64_t u1, u2, st0, st1, st2, sto, gates, hn;   // live-net activations kept for backward
  int64_t qall[2];          // [net][M][A]  (debug + greedy)
  int64_t greedy;           // int32 [M]
  int64_t q_taken, q_next;  // [B*T][N]
  int64_t qtot, qtot_next, err;  // [B*T]
  int64_t dq_taken;         // [B*T][N]
  int64_t dh_out;           // [M][H]
  int64_t dgi;              // [M][3H]
  int64_t gpart;            // [npart][P]
  int64_t lnpart;           // [2 npart][512]: LayerNorm gain / bias sums of k_front_bwd_tc CTAs (streamed mode, two CTAs per SM)
  int64_t grad;             // [P + 8]   flat gradient numerators + scalars (all-reduce payload)
  int64_t info;             // [8]
  int64_t prio;             // [max_batch]
  int64_t spart;            // [npart][8] per-CTA scalar partials (denominator, loss numerator, sum Q_tot)
  int64_t adam_t;           // double[4]: step count, beta1^t, beta2^t
  int64_t normpart;         // [ceil(P/256)] per-block sums of squares of the reduced gradient numerators
  int64_t xstat;            // float[8]: exchange breakdown accumulated by k_optim_fused (ns: push, wait, sum; launches; max wait)
  int64_t sync;             // uint32[8]: grid-barrier / exchange words of k_optim_fused (zero-initialised with the workspace)
  int64_t tcimg[2];         // pre-split TF32 weight images of the agent front layers (live, target)
  int64_t xin;              // prev_act_inp: packed network input rows [M][round_up(O + A, 4)]
  int64_t tcimgT;           // transposed TF32 weight images for k_front_bwd_tc
  int64_t tcacc, tcacc_cols; // tensor-core accumulators (mx_tc_acc_floats of the largest batch) and their columns
  int64_t da2, da1;         // [M][H] each: row gradients handed from k_front_bwd to k_wgrad_tc (option wgrad_tc)
  // split mixer pipeline: per-element hypernet outputs (live: kept for backward; target: forward only) and core's gradients
  int64_t hyp_h1, hyp_h2, hyp_hb;               // live [E][gH]
  int64_t hyp_p1[2], hyp_b1[2], hyp_p2[2], hyp_b2[2];
  int64_t d_q, d_hp, d_p2, d_p1;
  int64_t wimg, pre, d_pre;  // wide-state path only (empty otherwise): state-layer weight images, pre-activations, their gradient
  int64_t total;
};

// the QMIX step's fork / join points (qmix.cu), one event each: mx_qmix_prefork's fork and its weight images done; the hypernet
// forward's fork and join; the hypernet backward's fork; the step's final join; the GRU weight gradients' fork
enum MxQmixEvent { MX_EV_FORK, MX_EV_PREP, MX_EV_BATCH, MX_EV_HYPER, MX_EV_CORE, MX_EV_HBWD, MX_EV_GBWD, MX_EV_COUNT };

struct mx_qmix {
  mx_qmix_cfg cfg;
  MxNetLayout agent;
  MxMixLayout mix;
  int64_t P;               // padded parameter count
  int npart;               // number of per-CTA gradient partials
  int debug;               // also materialise q_all / greedy (parity tests)
  float *theta, *theta_tgt, *adam_m, *adam_v;
  float* ws;
  int64_t ws_bytes;
  MxQmixWs W;
  int split_ok;            // the split mixer pipeline supports this configuration
  int wide;                // wide-state path (mx_mix_wide_state): state layers on the tensor cores, always the split pipeline
  MxMixWide wl;
  // data-parallel exchange over peer memory (p2p.cu): symmetric blocks of every rank, set by mx_qmix_set_peers
  int p2p_rank = 0, p2p_world = 0;
  float* p2p_blocks[16] = {nullptr};
  uint32_t* p2p_counter = nullptr;
  // forked branch for the state-only kernels (weight-image prep, mixer hypernets): one non-blocking stream + fork/join events;
  // inside a stream capture the same record/wait calls turn into parallel graph branches.  The emulator has neither.
  cudaStream_t side = nullptr;
#if !MX_EMU
  cudaEvent_t ev[MX_EV_COUNT] = {};
#endif
  int prep_pending = 0;    // mx_qmix_prefork() already launched the weight-image prep for the coming step
  int imgT_fresh = 0;      // the transposed images (tensor-core backward) were rebuilt with the forward ones for this step
};
// ---- data-parallel exchange over peer memory (p2p.cu), for any learner's flat gradient buffer ----
#define MX_P2P_MAX_WORLD 16
// what one exchange sums: grad[P + 4] (gradient numerators, then the four loss scalars), keyed to the network's Adam step count (slot
// parity and flag value; already bumped by k_grad_reduce), and the learner's sticky abort word (-1 after a peer time-out)
struct MxP2pPayload {
  float* grad;
  int64_t P;                  // a multiple of 4
  const double* adam_t;
  float* abort;
};
struct MxP2pPeers {         // the world's symmetric blocks in rank order and this rank's local arrival counter
  int rank = 0, world = 0;
  float* blocks[MX_P2P_MAX_WORLD] = {nullptr};
  uint32_t* counter = nullptr;
};
int64_t mx_p2p_slot_floats(int64_t P);
// floats of one symmetric block laid out for `layout_world` ranks: slots of both parities [2][layout_world][slot] | 64 flag words
int64_t mx_p2p_block_floats(int64_t P, int layout_world);
int mx_p2p_set_peers(const char* who, MxP2pPeers* out, int32_t rank, int32_t world, void* const* peer_blocks, uint32_t* counter_dev);
int mx_p2p_publish(const MxP2pPeers& peers, const MxP2pPayload& pl, int layout_world, cudaStream_t s);
int mx_p2p_reduce(const MxP2pPeers& peers, const MxP2pPayload& pl, int layout_world, cudaStream_t s);

int mx_replay_sample_per_state_beta(mx_replay* r, int32_t B, void* stream);   // PER draw whose exponent is the device scalar (captured sequences)
int mx_qmix_prefork(mx_qmix* q, int B, void* stream);   // optional: start the parameter-only work of the next step before its batch is sampled
