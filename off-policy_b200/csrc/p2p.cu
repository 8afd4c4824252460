// Data-parallel gradient exchange over NVLink peer memory: a one-shot all-reduce written for THIS payload (one flat fp32
// vector of 0.2-0.4 MB per step: gradient numerators + loss denominators) instead of an NCCL call.
//
// The reference has no distributed path (utils/util.py:148-153 is dead code); the data-parallel learner of this repository
// (DESIGN.md section 6) sums the per-rank buffers `grad[P+4]` of every step.  PUSH model: every rank stores its buffer into slot
// [step parity][own rank] of EVERY rank's symmetric (peer-mapped) block -- remote stores are fire-and-forget, so the wire time hides
// behind the sender's own work -- then raises flag[own rank] = step on every rank; a rank that has seen all flags adds the `world`
// slots of its OWN block (local reads) in rank order.  Every rank computes bit-identical sums, so the replicas never diverge.
//
//   symmetric block of rank r (same layout on every rank):  [ recv[2][world][slot] | flags[world] (uint32, one per writer) ]
//
// Slots alternate with the step parity: a rank overwrites recv[s & 1] at step s + 2, which it reaches only after every peer has
// signalled step s + 1, i.e. has finished reading step s -- no acknowledgement round is needed.
// In the product path the whole exchange lives INSIDE the optimiser kernel (optim.cu: k_optim_fused -- the blocks that reduce the
// gradient partials push their columns straight from registers and apply Adam to the summed columns); the two kernels below are the
// same protocol as separate launches: start-up self-test, the emulated two-rank test, and `mx_set_option("optim_fused", 0)`.
//
// The helpers take a payload (buffer, P, Adam step count, abort word) rather than a learner.  The actor-critic learner (maddpg.cu)
// exchanges two payloads per update, the critic's and then the actor's, each over its own block, flags and arrival counter and keyed
// to its own Adam step count (the two counts advance at different rates when the actor trains every other update).  Its blocks are
// laid out for MX_P2P_MAX_WORLD ranks, so they can be sized before the world is known; the flags sit behind those slots.
#include <string.h>

#include "mx_internal.h"
#include "mx_kernels.h"

struct P2pArgs {
  float* grad;                 // [n] local flat buffer (k_grad_reduce output / k_adam input)
  float* blk[MX_P2P_MAX_WORLD];        // base of every rank's symmetric block (own block at index `rank`)
  long long n4;                // float4 per slot
  long long slot_floats;       // floats per slot (padded)
  long long flags_off;         // floats from a block's base to its flag words (behind the slots of both parities)
  const double* adam_t;        // adam_t[0] = 1-based step count, already bumped by k_grad_reduce
  unsigned* counter;           // local: CTAs of k_p2p_push that have finished
  float* abort;                // sticky abort word: -1 when a peer never arrived (time-out)
  int rank, world;
  unsigned long long timeout_ns;   // option p2p_timeout_ms (default 10 s)
};

MX_DEVINL unsigned* p2p_flags(float* block, long long flags_off) { return reinterpret_cast<unsigned*>(block + flags_off); }

__global__ void __launch_bounds__(256) k_p2p_push(P2pArgs a) {
  const unsigned step = (unsigned)a.adam_t[0];
  const size_t off = ((size_t)(step & 1u) * a.world + a.rank) * a.slot_floats;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = mx_ld4(a.grad + 4 * i);
    for (int p = 0; p < a.world; ++p) mx_st4(a.blk[p] + off + 4 * i, v);
  }
  __threadfence_system();                // this thread's slot writes are visible to the peers before anything that follows
  __syncthreads();
  __shared__ unsigned s_last;
  if (threadIdx.x == 0) s_last = (atomicAdd(a.counter, 1u) == gridDim.x - 1) ? 1u : 0u;
  __syncthreads();
  if (s_last) {                          // every CTA has fenced its part of the slot: tell the peers (and ourselves)
    if (threadIdx.x == 0) *a.counter = 0u;
    if ((int)threadIdx.x < a.world) {
      __threadfence_system();
      volatile unsigned* f = p2p_flags(a.blk[threadIdx.x], a.flags_off) + a.rank;
      *f = step;
    }
  }
}

MX_DEVINL float4 p2p_ld4(const float* p) {
#if MX_EMU
  return *reinterpret_cast<const float4*>(p);
#else
  float4 r;      // volatile: never served from a stale L1 line (memory written by another GPU)
  asm volatile("ld.volatile.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
#endif
}

__global__ void __launch_bounds__(256) k_p2p_sum(P2pArgs a) {
  const unsigned step = (unsigned)a.adam_t[0];
  __shared__ int s_bad;
  if (threadIdx.x == 0) s_bad = 0;
  __syncthreads();
  if ((int)threadIdx.x < a.world) {
    volatile unsigned* f = p2p_flags(a.blk[a.rank], a.flags_off) + threadIdx.x;
#if !MX_EMU
    unsigned long long t0, t1;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    while (*f < step) {
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
      if (t1 - t0 > a.timeout_ns) { s_bad = 1; break; }      // 10 s: a peer died; do not hang the device
    }
    __threadfence_system();              // acquire: the peer's slot writes precede its flag store
#else
    if (*f < step) s_bad = 1;            // the emulated test publishes every rank before it reduces
#endif
  }
  __syncthreads();
  if (s_bad) {                           // fatal: k_adam applies nothing while the abort word is < 0 and the host raises
    if (threadIdx.x == 0) *a.abort = -1.f;
    return;
  }
  const size_t off = (size_t)(step & 1u) * a.world * a.slot_floats;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.n4; i += (long long)gridDim.x * blockDim.x) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int p = 0; p < a.world; ++p) {  // rank order on every rank: bit-identical sums everywhere
      const float4 v = p2p_ld4(a.blk[a.rank] + off + (size_t)p * a.slot_floats + 4 * i);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    mx_st4(a.grad + 4 * i, acc);
  }
}

// ---- the protocol for any payload: block sizing, peer validation and the two launches ----
int64_t mx_p2p_slot_floats(int64_t P) { return mx_round_up64(P + 8, 64); }
int64_t mx_p2p_block_floats(int64_t P, int layout_world) { return 2 * (int64_t)layout_world * mx_p2p_slot_floats(P) + 64; }

int mx_p2p_set_peers(const char* who, MxP2pPeers* out, int32_t rank, int32_t world, void* const* peer_blocks, uint32_t* counter_dev) {
  if (!peer_blocks || !counter_dev) { mx_set_error("%s: null argument", who); return 1; }
  if (world < 2 || world > MX_P2P_MAX_WORLD || rank < 0 || rank >= world) { mx_set_error("%s: rank %d / world %d unsupported (max %d)", who, rank, world, MX_P2P_MAX_WORLD); return 1; }
  for (int p = 0; p < world; ++p)
    if (!peer_blocks[p]) { mx_set_error("%s: null peer block %d", who, p); return 1; }
  out->rank = rank; out->world = world; out->counter = counter_dev;
  for (int p = 0; p < world; ++p) out->blocks[p] = (float*)peer_blocks[p];
  return 0;
}

static P2pArgs p2p_args(const MxP2pPeers& peers, const MxP2pPayload& pl, int layout_world) {
  P2pArgs a;
  memset(&a, 0, sizeof(a));
  a.grad = pl.grad;
  for (int p = 0; p < peers.world; ++p) a.blk[p] = peers.blocks[p];
  a.n4 = (pl.P + 4) / 4;
  a.slot_floats = mx_p2p_slot_floats(pl.P);
  a.flags_off = 2 * (long long)layout_world * a.slot_floats;
  a.adam_t = pl.adam_t;
  a.counter = peers.counter;
  a.abort = pl.abort;
  a.rank = peers.rank; a.world = peers.world;
  a.timeout_ns = (unsigned long long)(g_mx_p2p_timeout_ms > 0 ? g_mx_p2p_timeout_ms : 10000) * 1000000ull;
  return a;
}

static int p2p_grid(const P2pArgs& a) {
  int grid = (int)((a.n4 + 255) / 256);
  const int sms = mx_num_sms();
  if (grid > sms) grid = sms;
  return grid < 1 ? 1 : grid;
}

int mx_p2p_publish(const MxP2pPeers& peers, const MxP2pPayload& pl, int layout_world, cudaStream_t s) {
  P2pArgs a = p2p_args(peers, pl, layout_world);
  return mx_launch("k_p2p_push", k_p2p_push, dim3(p2p_grid(a)), dim3(256), 0, s, MX_PLAIN, a);
}

int mx_p2p_reduce(const MxP2pPeers& peers, const MxP2pPayload& pl, int layout_world, cudaStream_t s) {
  P2pArgs a = p2p_args(peers, pl, layout_world);
  return mx_launch("k_p2p_sum", k_p2p_sum, dim3(p2p_grid(a)), dim3(256), 0, s, MX_PLAIN, a);
}

// ---- QMIX: one payload, the learner's grad[P+4]; its block also holds k_optim_fused's line arrays ----
extern "C" int64_t mx_qmix_p2p_block_bytes(const mx_qmix* q) {
  const int64_t slot = mx_p2p_slot_floats(q->P);
  const int64_t world = q->cfg.world_size > 1 ? q->cfg.world_size : 1;
  return (mx_p2p_block_floats(q->P, (int)world) + 2 * world * 2 * slot) * 4;      // slots of both parities | flags | flag-in-data line arrays of both parities (k_optim_fused)
}

extern "C" int mx_qmix_set_peers(mx_qmix* q, int32_t rank, int32_t world, void* const* peer_blocks, uint32_t* counter_dev) {
  if (!q) { mx_set_error("mx_qmix_set_peers: null argument"); return 1; }
  MxP2pPeers peers;
  if (mx_p2p_set_peers("mx_qmix_set_peers", &peers, rank, world, peer_blocks, counter_dev)) return 1;
  if (world != q->cfg.world_size) { mx_set_error("mx_qmix_set_peers: world %d != cfg.world_size %d", world, q->cfg.world_size); return 1; }
  q->p2p_rank = rank; q->p2p_world = world; q->p2p_counter = counter_dev;
  for (int p = 0; p < world; ++p) q->p2p_blocks[p] = peers.blocks[p];
  return 0;
}

static void qmix_p2p(mx_qmix* q, MxP2pPeers* peers, MxP2pPayload* pl) {
  peers->rank = q->p2p_rank; peers->world = q->p2p_world; peers->counter = q->p2p_counter;
  for (int p = 0; p < q->p2p_world; ++p) peers->blocks[p] = q->p2p_blocks[p];
  pl->grad = q->ws + q->W.grad; pl->P = q->P;
  pl->adam_t = reinterpret_cast<const double*>(q->ws + q->W.adam_t);
  pl->abort = q->ws + q->W.info + 7;
}

extern "C" int mx_qmix_p2p_publish(mx_qmix* q, void* stream) {
  if (!q->p2p_world) { mx_set_error("mx_qmix_p2p_publish: mx_qmix_set_peers was not called"); return 1; }
  MxP2pPeers peers;
  MxP2pPayload pl;
  qmix_p2p(q, &peers, &pl);
  return mx_p2p_publish(peers, pl, q->p2p_world, (cudaStream_t)stream);
}

extern "C" int mx_qmix_p2p_reduce(mx_qmix* q, void* stream) {
  if (!q->p2p_world) { mx_set_error("mx_qmix_p2p_reduce: mx_qmix_set_peers was not called"); return 1; }
  MxP2pPeers peers;
  MxP2pPayload pl;
  qmix_p2p(q, &peers, &pl);
  return mx_p2p_reduce(peers, pl, q->p2p_world, (cudaStream_t)stream);
}
