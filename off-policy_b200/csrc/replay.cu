// HBM-resident episode replay: ring insert, NumPy-legacy index draw, vectorised gather, fp64 PER trees.
//
// Layout (DESIGN.md "replay SoA"): every field is EPISODE-major -- one episode's slice of a field is a
// single contiguous, 16-byte aligned chunk (innermost dim padded to a multiple of 4 floats) -- so sampling
// B episodes is B straight 128-bit copies per field.  The reference keeps time-major NumPy arrays
// (T+1, E, N, D) and pays a strided fancy-index copy per field (rec_buffer.py:120-141, 192-240).
#include <math.h>
#include <stddef.h>
#include <stdio.h>
#include <string.h>

#include "mx_internal.h"
#include "mx_mt19937.cuh"

// =====================================================================================================
// layout
// =====================================================================================================
static int64_t align_up(int64_t v, int64_t a) { return (v + a - 1) / a * a; }

extern "C" int mx_replay_layout_query(const mx_replay_cfg* c, mx_replay_layout* L) {
  if (!c || !L) { mx_set_error("null argument"); return 1; }
  if (c->capacity <= 0 || c->episode_len <= 0 || c->n_agents <= 0 || c->obs_dim <= 0 || c->share_dim <= 0 || c->act_dim <= 0 ||
      c->max_batch <= 0) {
    mx_set_error("mx_replay_layout_query: non-positive dimension");
    return 1;
  }
  memset(L, 0, sizeof(*L));
  const int T = c->episode_len, N = c->n_agents;
  L->obs_ld = mx_round_up(c->obs_dim, 4);
  L->share_ld = mx_round_up(c->share_dim, 4);
  L->act_ld = mx_round_up(c->act_dim, 4);
  L->ep_obs = (int64_t)(T + 1) * N * L->obs_ld;
  L->ep_share = (int64_t)(T + 1) * L->share_ld;
  L->ep_acts = (int64_t)T * N * L->act_ld;
  L->ep_avail = c->use_avail ? (int64_t)(T + 1) * N * L->act_ld : 0;
  L->ep_rew = mx_round_up(T * N, 4);
  L->ep_dones = mx_round_up(T * N, 4);
  L->ep_dones_env = mx_round_up(T, 4);
  L->ep_actidx = mx_round_up(T * N, 4);
  int cap = 1;
  while (cap < c->capacity) cap *= 2;
  L->tree_cap = cap;
  int64_t off = 0;
  auto take = [&](int64_t bytes) { int64_t o = off; off = align_up(off + bytes, 256); return o; };
  const int64_t E = c->capacity, MB = c->max_batch;
  L->off_obs = take(E * L->ep_obs * 4);
  L->off_share = take(E * L->ep_share * 4);
  L->off_acts = take(E * L->ep_acts * 4);
  L->off_avail = take(E * L->ep_avail * 4);
  L->off_rew = take(E * L->ep_rew * 4);
  L->off_dones = take(E * L->ep_dones * 4);
  L->off_dones_env = take(E * L->ep_dones_env * 4);
  L->off_actidx = take(E * L->ep_actidx * 4);
  L->off_sum_tree = take(c->use_per ? (int64_t)2 * cap * 8 : 0);
  L->off_min_tree = take(c->use_per ? (int64_t)2 * cap * 8 : 0);
  L->off_rng = take(625 * 4);
  L->off_state = take(sizeof(MxReplayState));
  L->off_rstats = take(4 * 8);
  L->off_b_obs = take(MB * L->ep_obs * 4);
  L->off_b_share = take(MB * L->ep_share * 4);
  L->off_b_acts = take(MB * L->ep_acts * 4);
  L->off_b_avail = take(MB * L->ep_avail * 4);
  L->off_b_rew = take(MB * L->ep_rew * 4);
  L->off_b_dones = take(MB * L->ep_dones * 4);
  L->off_b_dones_env = take(MB * L->ep_dones_env * 4);
  L->off_b_actidx = take(MB * L->ep_actidx * 4);
  L->off_b_idx = take(MB * 8);
  L->off_b_weights = take(MB * 8);
  L->off_b_wf32 = take(MB * 4);
  // staging for ONE insert call of up to max_batch episodes, raw time-major as handed in
  int64_t per_ep = (int64_t)(T + 1) * N * c->obs_dim + (int64_t)(T + 1) * c->share_dim + (int64_t)T * N * c->act_dim +
                   (c->use_avail ? (int64_t)(T + 1) * N * c->act_dim : 0) + 2 * (int64_t)T * N + T;
  L->stage_bytes = align_up(per_ep * 4 * MB + 7 * 256, 256);
  L->off_stage = take(L->stage_bytes);
  L->total_bytes = off;
  return 0;
}

// =====================================================================================================
// insert: time-major staging -> episode-major padded SoA
// =====================================================================================================
struct InsField {
  const float* src;   // (Tf, n_ep, rows, D) raw
  float* dst;         // [E][ep_stride]
  int Tf, rows, D, ld;
  long long ep_stride;
  long long count;    // Tf * n_ep * rows * D
};
struct InsArgs {
  InsField f[7];
  int nf;
  int n_ep, first_slot, capacity;
  int T, N, A, act_ld;
  const float* acts_src;   // for act_idx
  int32_t* actidx;         // [E][ep_actidx]
  long long ep_actidx;
  MxReplayState* state;
  int new_filled, new_cursor;
  double* sum_tree;        // PER priming (may be null)
  double* min_tree;
  int tree_cap;
  double alpha;
};

__global__ void k_insert_scatter(InsArgs a) {
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nth = (long long)gridDim.x * blockDim.x;
  for (int fi = 0; fi < a.nf; ++fi) {
    const InsField f = a.f[fi];
    for (long long i = tid; i < f.count; i += nth) {
      int d = (int)(i % f.D);
      long long r = i / f.D;
      int row = (int)(r % f.rows);
      r /= f.rows;
      int e = (int)(r % a.n_ep);
      int t = (int)(r / a.n_ep);
      int slot = (a.first_slot + e) % a.capacity;
      f.dst[(long long)slot * f.ep_stride + ((long long)t * f.rows + row) * f.ld + d] = f.src[i];
    }
  }
  // action index = argmax of the one-hot action, first maximum (QMixPolicy.py:89)
  const long long na = (long long)a.T * a.n_ep * a.N;
  for (long long i = tid; i < na; i += nth) {
    int n = (int)(i % a.N);
    long long r = i / a.N;
    int e = (int)(r % a.n_ep);
    int t = (int)(r / a.n_ep);
    const float* p = a.acts_src + i * a.A;
    int best = 0;
    float bv = p[0];
    for (int k = 1; k < a.A; ++k)
      if (p[k] > bv) { bv = p[k]; best = k; }
    int slot = (a.first_slot + e) % a.capacity;
    a.actidx[(long long)slot * a.ep_actidx + t * a.N + n] = best;
  }
  if (tid == 0) {
    a.state->filled = a.new_filled;
    a.state->cursor = a.new_cursor;
  }
}

// PER tree maintenance for a set of leaves: values[i] -> leaf idx[i]; duplicates: LAST write wins
// (NumPy fancy assignment, rec_buffer.py:320-321), then parents are recomputed level by level
// (segment_tree.py:74-89).  One CTA.
struct TreeUpd {
  double *sum_tree, *min_tree;
  int cap, n;
  const long long* idx;       // device int64[n] or null -> ring slots first_slot..+n
  int first_slot, capacity;
  const float* prio;          // fp32 priorities (powered by alpha here) or null
  const double* leaves;       // pre-powered fp64 leaves or null
  double alpha;
  int prime_from_max;         // leaf = max_priority ** alpha
  MxReplayState* state;
  int update_max;
};

__global__ void k_tree_update(TreeUpd u) {
  __shared__ long long s_idx[1024];
  const int tid = threadIdx.x;
  long long my = -1;
  double val = 0.0;
  float myp = 0.f;
  if (tid < u.n) {
    my = u.idx ? u.idx[tid] : (long long)((u.first_slot + tid) % u.capacity);
    if (u.prime_from_max) val = pow(u.state->max_priority, u.alpha);
    else if (u.leaves) val = u.leaves[tid];
    else {
      myp = u.prio[tid];
      val = (double)(float)pow((double)myp, u.alpha);   // fp32 result like NumPy's float32 ** python-float
    }
  }
  if (tid < 1024) s_idx[tid] = my;
  __syncthreads();
  bool writer = tid < u.n;
  if (writer)
    for (int j = tid + 1; j < u.n; ++j)
      if (s_idx[j] == my) { writer = false; break; }
  if (writer) {
    u.sum_tree[u.cap + my] = val;
    u.min_tree[u.cap + my] = val;
  }
  __syncthreads();
  for (int shift = 1; (u.cap >> shift) >= 1; ++shift) {
    if (tid < u.n) {
      long long node = (u.cap + my) >> shift;
      u.sum_tree[node] = u.sum_tree[2 * node] + u.sum_tree[2 * node + 1];
      double l = u.min_tree[2 * node], r = u.min_tree[2 * node + 1];
      u.min_tree[node] = l < r ? l : r;
    }
    __syncthreads();
  }
  if (u.update_max && u.prio) {
    // max_priority = max(max_priority, max(prio))  (rec_buffer.py:323-324)
    __shared__ float s_max[32];
    float m = tid < u.n ? myp : 0.f;
    m = mx_warp_max(m);
    if ((tid & 31) == 0) s_max[tid >> 5] = m;
    __syncthreads();
    if (tid == 0) {
      float mm = 0.f;
      for (int w = 0; w < (int)((blockDim.x + 31) / 32); ++w) mm = fmaxf(mm, s_max[w]);
      if ((double)mm > u.state->max_priority) u.state->max_priority = (double)mm;
    }
  }
}

// =====================================================================================================
// NumPy legacy MT19937 on the device (SURVEY.md App. C; oracle/mt19937.py is the CPU restatement; generator core: mx_mt19937.cuh)
// =====================================================================================================
struct DrawArgs {
  uint32_t* rng;               // key[624]
  MxReplayState* state;
  int B;
  int per;                     // 0: uniform randint(0, filled)   1: PER masses
  long long* idx_out;          // int64 [B]
  // PER
  const double *sum_tree, *min_tree;
  int cap;
  double beta;                 // < 0: read state->per_beta (whole-step graphs: the exponent anneals between replays of one captured launch)
  double* w_out;               // fp64 [B]
  float* w32_out;              // fp32 [B]
};

__global__ void __launch_bounds__(256) k_draw(DrawArgs a) {
  __shared__ uint32_t key[MT_N];
  __shared__ int s_pos, s_done, s_next;
  __shared__ double s_u[1024];
  __shared__ uint32_t s_half;   // PER: first word of a double already drawn
  __shared__ int s_havehalf;
  const int tid = threadIdx.x;
  // ---- fast path (uniform draw, no regeneration needed within the next 256 words): the stream is consumed straight from
  // global memory -- all 256 candidate words are tempered and rejection-tested in parallel, accepted ones are compacted in
  // stream order with ballots, and only `rng_pos` is written back.  Falls through to the general path otherwise.
  if (!a.per && blockDim.x == 256) {
    __shared__ int s_wcnt[8], s_used;
    const int pos0 = a.state->rng_pos, n0 = a.state->filled;
    const uint32_t rng0 = (uint32_t)(n0 - 1);
    if (rng0 != 0 && pos0 + 256 <= MT_N && a.B <= 256) {       // block-uniform condition
      uint32_t mask0 = rng0;
      mask0 |= mask0 >> 1; mask0 |= mask0 >> 2; mask0 |= mask0 >> 4; mask0 |= mask0 >> 8; mask0 |= mask0 >> 16;
      const uint32_t v = mt_temper(a.rng[pos0 + tid]) & mask0;   // masked rejection (legacy randint)
      const bool acc = v <= rng0;
      const unsigned bal = __ballot_sync(0xffffffffu, acc);
      const int lane = tid & 31, warp = tid >> 5;
      if (lane == 0) s_wcnt[warp] = __popc(bal);
      if (tid == 0) s_used = -1;
      __syncthreads();
      int before = 0, total_acc = 0;
      for (int w = 0; w < 8; ++w) { if (w < warp) before += s_wcnt[w]; total_acc += s_wcnt[w]; }
      if (total_acc >= a.B) {                                    // block-uniform
        const int k = before + __popc(bal & ((1u << lane) - 1u));
        if (acc && k < a.B) {
          a.idx_out[k] = (long long)v;
          if (k == a.B - 1) s_used = tid + 1;                    // words consumed = position of the B-th accepted word + 1
        }
        __syncthreads();
        if (tid == 0) a.state->rng_pos = pos0 + s_used;
        return;
      }
      __syncthreads();
    }
  }
  for (int i = tid; i < MT_N; i += blockDim.x) key[i] = a.rng[i];
  if (tid == 0) {
    s_pos = a.state->rng_pos;
    s_done = 0;
    s_next = 0;
    s_havehalf = 0;
  }
  __syncthreads();
  const int n = a.state->filled;
  const uint32_t rng = (uint32_t)(n - 1);
  uint32_t mask = rng;
  mask |= mask >> 1; mask |= mask >> 2; mask |= mask >> 4; mask |= mask >> 8; mask |= mask >> 16;
  while (true) {
    if (tid == 0) {
      int pos = s_pos, k = s_next;
      if (!a.per) {
        if (rng == 0) {           // n == 1 consumes nothing
          for (; k < a.B; ++k) a.idx_out[k] = 0;
        }
        while (k < a.B && pos < MT_N) {
          uint32_t v = mt_temper(key[pos++]) & mask;   // masked rejection (legacy randint)
          if (v <= rng) a.idx_out[k++] = (long long)v;
        }
      } else {
        while (k < a.B && pos < MT_N) {
          uint32_t w = mt_temper(key[pos++]);
          if (!s_havehalf) { s_half = w; s_havehalf = 1; }
          else {
            s_u[k++] = ((double)(s_half >> 5) * 67108864.0 + (double)(w >> 6)) / 9007199254740992.0;
            s_havehalf = 0;
          }
        }
      }
      s_pos = pos;
      s_next = k;
      s_done = (k >= a.B);
    }
    __syncthreads();
    if (s_done) break;
    mt_twist_cta(key);
    if (tid == 0) s_pos = 0;
    __syncthreads();
  }
  for (int i = tid; i < MT_N; i += blockDim.x) a.rng[i] = key[i];
  if (tid == 0) a.state->rng_pos = s_pos;
  if (!a.per) return;

  // ---- proportional sampling (rec_buffer.py:272-296, segment_tree.py:43-72,115-146) ----
  __shared__ double s_total, s_all, s_min;
  if (tid == 0) {
    // sum over leaves [0, n-1) with the reference's recursion order: v[L1] + (v[L2] + (...)) right-nested
    double stack[40];
    int sp = 0;
    int s = 0, e = n - 2;            // reduce(0, n-1): end exclusive -> inclusive n-2
    int node = 1, ns = 0, ne = a.cap - 1;
    while (true) {
      if (s == ns && e == ne) { stack[sp++] = a.sum_tree[node]; break; }
      int mid = (ns + ne) / 2;
      if (e <= mid) { node = 2 * node; ne = mid; }
      else if (mid + 1 <= s) { node = 2 * node + 1; ns = mid + 1; }
      else {
        stack[sp++] = a.sum_tree[2 * node];   // left part is exactly the left child (s == ns)
        node = 2 * node + 1;
        s = mid + 1;
        ns = mid + 1;
      }
    }
    double acc = stack[sp - 1];
    for (int i = sp - 2; i >= 0; --i) acc = stack[i] + acc;
    s_total = acc;
    s_all = a.sum_tree[1];
    s_min = a.min_tree[1];
  }
  __syncthreads();
  for (int i = tid; i < a.B; i += blockDim.x) {
    double m = s_u[i] * s_total;
    int node = 1;
    while (node < a.cap) {
      int left = 2 * node;
      double lv = a.sum_tree[left];
      if (lv <= m) { m -= lv; node = left + 1; }
      else node = left;
    }
    int leaf = node - a.cap;
    a.idx_out[i] = leaf;
    const double beta = a.beta < 0.0 ? a.state->per_beta : a.beta;
    double p_min = s_min / s_all;
    double max_w = pow(p_min * (double)n, -beta);
    double p_s = a.sum_tree[a.cap + leaf] / s_all;
    double w = pow(p_s * (double)n, -beta) / max_w;
    a.w_out[i] = w;
    a.w32_out[i] = (float)w;
  }
}

// =====================================================================================================
// reward normalisation statistics (rec_buffer.py:209-220): nan-masked mean / population std over every
// filled reward; a step is masked when the env was already done at the previous step.
//
// The reference rescans the whole buffer on every sample() (7 ms at 5 000 episodes, SURVEY.md section 8(f).2).  Here the
// masked sum / sum of squares / count are running fp64 totals in the blob, updated at insert time: the episodes an insert
// evicts are subtracted (read from the SoA before the scatter overwrites them), the new ones added (read from the insert
// staging area).  One CTA, fixed summation order -> deterministic; sample() only reads the two resulting scalars.
// =====================================================================================================
struct RewStatArgs {
  const float *rew_soa, *de_soa;     // [E][ep_rew], [E][ep_de]
  long long ep_rew, ep_de;
  const float *rew_stage, *de_stage; // raw time-major (T, n_ep, N), (T, n_ep)
  int T, N, n_ep, first_slot, capacity, filled_before;
  double* rstats;                    // [4]: sum, sum of squares, count
  MxReplayState* state;
};
__global__ void __launch_bounds__(256) k_reward_stats_update(RewStatArgs a) {
  __shared__ double red[3][8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double s = 0, s2 = 0, c = 0;
  const int per = a.T * a.N;
  for (int e = 0; e < a.n_ep; ++e) {
    const int slot = (a.first_slot + e) % a.capacity;
    const bool evict = slot < a.filled_before;
    for (int i = tid; i < per; i += blockDim.x) {
      const int t = i / a.N, n = i - t * a.N;
      if (!(t > 0 && a.de_stage[(size_t)(t - 1) * a.n_ep + e] == 1.0f)) {
        const double v = (double)a.rew_stage[((size_t)t * a.n_ep + e) * a.N + n];
        s += v; s2 += v * v; c += 1.0;
      }
      if (evict && !(t > 0 && a.de_soa[(size_t)slot * a.ep_de + t - 1] == 1.0f)) {
        const double v = (double)a.rew_soa[(size_t)slot * a.ep_rew + i];
        s -= v; s2 -= v * v; c -= 1.0;
      }
    }
  }
  s = mx_warp_sum_d(s); s2 = mx_warp_sum_d(s2); c = mx_warp_sum_d(c);
  if (lane == 0) { red[0][warp] = s; red[1][warp] = s2; red[2][warp] = c; }
  __syncthreads();
  if (tid == 0) {
    double t0 = a.rstats[0], t1 = a.rstats[1], t2 = a.rstats[2];
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { t0 += red[0][w]; t1 += red[1][w]; t2 += red[2][w]; }
    a.rstats[0] = t0; a.rstats[1] = t1; a.rstats[2] = t2;
    if (t2 > 0.0) {
      const double mean = t0 / t2;
      const double var = t1 / t2 - mean * mean;
      a.state->reward_mean = (double)(float)mean;                      // the reference's statistics are np.float32 scalars
      a.state->reward_std = (double)(float)sqrt(var > 0 ? var : 0.0);
    }
  }
}

// =====================================================================================================
// gather: B sampled episodes x every field, 128-bit loads/stores, grid sized to the SM count
// =====================================================================================================
struct GatherField {
  const float* src;
  float* dst;
  long long ep4;     // float4s per episode
};
struct GatherArgs {
  GatherField f[8];
  long long cum4[9]; // cumulative float4 counts per (field x one episode)
  int nf, B;
  const long long* idx;
  int rew_field;     // index of the reward field or -1: apply (r - mean) / std there
  const MxReplayState* state;
};

// One float4 of the batch: flat index i -> (episode b, field, offset) -> source / destination addresses.
MX_DEVINL void gather_addr(const GatherArgs& a, unsigned i, unsigned per_ep, const float*& src, float*& dst, bool& is_rew) {
  const unsigned b = i / per_ep;
  const unsigned r = i - b * per_ep;
  int fi = 0;
#pragma unroll
  for (int k = 1; k < 8; ++k)
    if (k < a.nf && r >= (unsigned)a.cum4[k]) fi = k;
  const long long off = (long long)r - a.cum4[fi];
  const long long e = a.idx[b];
  src = a.f[fi].src + (e * a.f[fi].ep4 + off) * 4;
  dst = a.f[fi].dst + ((long long)b * a.f[fi].ep4 + off) * 4;
  is_rew = (fi == a.rew_field);
}

// HBM-bound copy: every thread keeps FOUR independent 16-byte loads in flight per iteration (8 resident CTAs x 256 threads x
// 64 B = 128 KB in flight per SM), consecutive threads touch consecutive 16-byte words, 32-bit index arithmetic.
__global__ void __launch_bounds__(256) k_gather(GatherArgs a) {
  const unsigned per_ep = (unsigned)a.cum4[a.nf];
  const unsigned total = per_ep * (unsigned)a.B;            // < 2^31 float4 (checked by the launcher)
  float mean = 0.f, stdv = 1.f;
  MX_PDL_WAIT();
  if (a.rew_field >= 0) { mean = (float)a.state->reward_mean; stdv = (float)a.state->reward_std; }
  const unsigned step = gridDim.x * blockDim.x * 4u;
  for (unsigned base = blockIdx.x * blockDim.x * 4u + threadIdx.x; base < total; base += step) {
    const float* src[4];
    float* dst[4];
    bool rw[4], ok[4];
    float4 v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const unsigned i = base + j * blockDim.x;
      ok[j] = i < total;
      if (ok[j]) gather_addr(a, i, per_ep, src[j], dst[j], rw[j]);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (ok[j]) v[j] = mx_ld4_stream(src[j]);
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (ok[j]) {
        if (rw[j]) { v[j].x = (v[j].x - mean) / stdv; v[j].y = (v[j].y - mean) / stdv; v[j].z = (v[j].z - mean) / stdv; v[j].w = (v[j].w - mean) / stdv; }
        mx_st4_stream(dst[j], v[j]);
      }
  }
}

// =====================================================================================================
// host API
// =====================================================================================================
extern "C" int mx_replay_create(const mx_replay_cfg* cfg, void* blob, void* stream, mx_replay** out) {
  (void)stream;
  if (!cfg || !blob || !out) { mx_set_error("mx_replay_create: null argument"); return 1; }
  mx_replay* r = new mx_replay();
  r->cfg = *cfg;
  if (mx_replay_layout_query(cfg, &r->L)) { delete r; return 1; }
  if (cfg->max_batch > 1024) { mx_set_error("mx_replay_create: max_batch > 1024 unsupported"); delete r; return 1; }
  r->blob = (char*)blob;
  r->filled = 0;
  r->cursor = 0;
  // device state: max_priority = 1.0 (rec_buffer.py:260); rng_pos = 624 until seeded
  MxReplayState st;
  memset(&st, 0, sizeof(st));
  st.rng_pos = MT_N;
  st.max_priority = 1.0;
  st.reward_mean = 0.0;
  st.reward_std = 1.0;
  cudaMemcpyAsync(r->blob + r->L.off_state, &st, sizeof(st), cudaMemcpyHostToDevice, (cudaStream_t)stream);
  cudaStreamSynchronize((cudaStream_t)stream);
  if (cfg->use_per) {
    // min-tree neutral element is +inf (segment_tree.py:151)
    const int64_t n = 2 * (int64_t)r->L.tree_cap;
    double* tmp = new double[n];
    for (int64_t i = 0; i < n; ++i) tmp[i] = INFINITY;
    cudaMemcpyAsync(r->blob + r->L.off_min_tree, tmp, n * 8, cudaMemcpyHostToDevice, (cudaStream_t)stream);
    cudaStreamSynchronize((cudaStream_t)stream);
    delete[] tmp;
  }
  r->tma = mx_gather_tma_create(r);
  *out = r;
  return 0;
}
extern "C" void mx_replay_destroy(mx_replay* r) {
  if (r) mx_gather_tma_destroy(r->tma);
  delete r;
}
// Checkpoint restore: after the caller has copied a saved blob back into device memory, re-read the host mirror of the ring
// position from the blob's device scalars (synchronises the stream).
extern "C" int mx_replay_restore(mx_replay* r, void* stream) {
  if (!r) { mx_set_error("mx_replay_restore: null handle"); return 1; }
  MxReplayState st;
  cudaMemcpyAsync(&st, r->blob + r->L.off_state, sizeof(st), cudaMemcpyDeviceToHost, (cudaStream_t)stream);
  cudaStreamSynchronize((cudaStream_t)stream);
  if (st.filled < 0 || st.filled > r->cfg.capacity || st.cursor < 0 || st.cursor > r->cfg.capacity) {
    mx_set_error("mx_replay_restore: blob does not hold a replay of this shape (filled %d, cursor %d, capacity %d)", st.filled, st.cursor, r->cfg.capacity);
    return 1;
  }
  r->filled = st.filled;
  r->cursor = st.cursor;
  return 0;
}
extern "C" int32_t mx_replay_len(const mx_replay* r) { return r->filled; }
extern "C" int32_t mx_replay_cursor(const mx_replay* r) { return r->cursor; }

template <class T> static T* at(mx_replay* r, int64_t off) { return reinterpret_cast<T*>(r->blob + off); }
template <class T> static const T* cat(const mx_replay* r, int64_t off) { return reinterpret_cast<const T*>(r->blob + off); }

// field table of one insert call: element counts and byte offsets inside the (256-byte aligned) staging layout
struct StageField { int64_t count, offset; };
static int stage_fields(const mx_replay* r, int n_ep, StageField f[7], int64_t* total) {
  const mx_replay_cfg& c = r->cfg;
  const int T = c.episode_len, N = c.n_agents;
  const int64_t cnt[7] = {(int64_t)(T + 1) * n_ep * N * c.obs_dim, (int64_t)(T + 1) * n_ep * c.share_dim, (int64_t)T * n_ep * N * c.act_dim,
                          (int64_t)T * n_ep * N, (int64_t)T * n_ep * N, (int64_t)T * n_ep, c.use_avail ? (int64_t)(T + 1) * n_ep * N * c.act_dim : 0};
  int64_t so = 0;
  for (int i = 0; i < 7; ++i) { f[i].count = cnt[i]; f[i].offset = so; so = align_up(so + cnt[i] * 4, 256); }
  *total = so;
  return 0;
}

static int insert_staged(mx_replay* r, int32_t n_ep, int32_t* first_slot_out, cudaStream_t s) {
  const mx_replay_cfg& c = r->cfg;
  const mx_replay_layout& L = r->L;
  const int T = c.episode_len, N = c.n_agents;
  StageField sf[7];
  int64_t total;
  stage_fields(r, n_ep, sf, &total);
  char* stage = r->blob + L.off_stage;
  InsArgs a;
  memset(&a, 0, sizeof(a));
  int nf = 0;
  auto add = [&](int fi, float* dst, int Tf, int rows, int D, int ld, int64_t ep_stride) {
    a.f[nf].src = reinterpret_cast<const float*>(stage + sf[fi].offset); a.f[nf].dst = dst; a.f[nf].Tf = Tf; a.f[nf].rows = rows; a.f[nf].D = D;
    a.f[nf].ld = ld; a.f[nf].ep_stride = ep_stride; a.f[nf].count = sf[fi].count;
    ++nf;
  };
  add(0, at<float>(r, L.off_obs), T + 1, N, c.obs_dim, L.obs_ld, L.ep_obs);
  add(1, at<float>(r, L.off_share), T + 1, 1, c.share_dim, L.share_ld, L.ep_share);
  add(2, at<float>(r, L.off_acts), T, N, c.act_dim, L.act_ld, L.ep_acts);
  add(3, at<float>(r, L.off_rew), T, N, 1, 1, L.ep_rew);
  add(4, at<float>(r, L.off_dones), T, N, 1, 1, L.ep_dones);
  add(5, at<float>(r, L.off_dones_env), T, 1, 1, 1, L.ep_dones_env);
  if (c.use_avail) add(6, at<float>(r, L.off_avail), T + 1, N, c.act_dim, L.act_ld, L.ep_avail);
  a.nf = nf;
  const int first = r->cursor % c.capacity;                    // current_i may equal capacity (rec_buffer.py:187)
  a.n_ep = n_ep; a.first_slot = first; a.capacity = c.capacity;
  a.T = T; a.N = N; a.A = c.act_dim; a.act_ld = L.act_ld;
  a.acts_src = reinterpret_cast<const float*>(stage + sf[2].offset);
  a.actidx = at<int32_t>(r, L.off_actidx);
  a.ep_actidx = L.ep_actidx;
  a.state = at<MxReplayState>(r, L.off_state);
  const int last = (first + n_ep - 1) % c.capacity;
  a.new_cursor = last + 1;                                     // rec_buffer.py:187 (not wrapped until the next insert)
  a.new_filled = r->filled + n_ep < c.capacity ? r->filled + n_ep : c.capacity;
  if (c.reward_norm) {     // running reward statistics: must read the evicted episodes before the scatter overwrites them
    RewStatArgs rs;
    memset(&rs, 0, sizeof(rs));
    rs.rew_soa = cat<float>(r, L.off_rew); rs.de_soa = cat<float>(r, L.off_dones_env); rs.ep_rew = L.ep_rew; rs.ep_de = L.ep_dones_env;
    rs.rew_stage = reinterpret_cast<const float*>(stage + sf[3].offset); rs.de_stage = reinterpret_cast<const float*>(stage + sf[5].offset);
    rs.T = T; rs.N = N; rs.n_ep = n_ep; rs.first_slot = first; rs.capacity = c.capacity; rs.filled_before = r->filled;
    rs.rstats = at<double>(r, L.off_rstats); rs.state = a.state;
    if (const int rc = mx_launch("k_reward_stats_update", k_reward_stats_update, dim3(1), dim3(256), 0, s, MX_PLAIN, rs)) return rc;
  }
  int64_t work = a.f[0].count;
  int grid = (int)((work + 255) / 256);
  int maxg = mx_num_sms() * 8;
  if (grid > maxg) grid = maxg;
  if (grid < 1) grid = 1;
  if (const int rc = mx_launch("k_insert_scatter", k_insert_scatter, dim3(grid), dim3(256), 0, s, MX_PLAIN, a)) return rc;
  if (c.use_per) {
    TreeUpd u;
    memset(&u, 0, sizeof(u));
    u.sum_tree = at<double>(r, L.off_sum_tree); u.min_tree = at<double>(r, L.off_min_tree);
    u.cap = L.tree_cap; u.n = n_ep; u.idx = nullptr; u.first_slot = first; u.capacity = c.capacity;
    u.alpha = c.per_alpha; u.prime_from_max = 1; u.state = a.state; u.update_max = 0;
    if (const int rc = mx_launch("k_tree_update", k_tree_update, dim3(1), dim3(mx_round_up(n_ep, 32)), 0, s, MX_PLAIN, u)) return rc;
  }
  if (first_slot_out) *first_slot_out = first;
  r->cursor = a.new_cursor;
  r->filled = a.new_filled;
  return 0;
}

static int check_insert(mx_replay* r, int32_t n_ep) {
  const mx_replay_cfg& c = r->cfg;
  if (n_ep <= 0 || n_ep > c.max_batch || n_ep > c.capacity) { mx_set_error("mx_replay_insert: n_ep=%d out of range (max_batch %d)", n_ep, c.max_batch); return 1; }
  return 0;
}

extern "C" int mx_replay_insert_async(mx_replay* r, const mx_episodes* ep, int32_t n_ep, int32_t* first_slot_out, void* stream) {
  if (check_insert(r, n_ep)) return 1;
  if (!ep->obs || !ep->share_obs || !ep->acts || !ep->rewards || !ep->dones || !ep->dones_env || (r->cfg.use_avail && !ep->avail)) {
    mx_set_error("mx_replay_insert: missing field");
    return 1;
  }
  cudaStream_t s = (cudaStream_t)stream;
  StageField sf[7];
  int64_t total;
  stage_fields(r, n_ep, sf, &total);
  if (total > r->L.stage_bytes) { mx_set_error("mx_replay_insert: staging overflow"); return 1; }
  const float* src[7] = {ep->obs, ep->share_obs, ep->acts, ep->rewards, ep->dones, ep->dones_env, ep->avail};
  char* stage = r->blob + r->L.off_stage;
  for (int i = 0; i < 7; ++i)
    if (sf[i].count) cudaMemcpyAsync(stage + sf[i].offset, src[i], sf[i].count * 4, cudaMemcpyDefault, s);
  return insert_staged(r, n_ep, first_slot_out, s);
}

extern "C" int64_t mx_replay_insert_packed_layout(const mx_replay* r, int32_t n_ep, int64_t offsets[7], int64_t counts[7]) {
  StageField sf[7];
  int64_t total;
  stage_fields(r, n_ep, sf, &total);
  for (int i = 0; i < 7; ++i) { offsets[i] = sf[i].offset; counts[i] = sf[i].count; }
  return total;
}

extern "C" int mx_replay_insert_packed_async(mx_replay* r, const void* packed, int64_t nbytes, int32_t n_ep, int32_t* first_slot_out, void* stream) {
  if (check_insert(r, n_ep)) return 1;
  StageField sf[7];
  int64_t total;
  stage_fields(r, n_ep, sf, &total);
  if (nbytes != total || total > r->L.stage_bytes) { mx_set_error("mx_replay_insert_packed: expected %lld bytes, got %lld", (long long)total, (long long)nbytes); return 1; }
  cudaStream_t s = (cudaStream_t)stream;
  cudaMemcpyAsync(r->blob + r->L.off_stage, packed, (size_t)nbytes, cudaMemcpyDefault, s);     // ONE host->device copy per insert
  return insert_staged(r, n_ep, first_slot_out, s);
}

extern "C" int mx_replay_seed(mx_replay* r, uint32_t seed, void* stream) {
  uint32_t key[MT_N];
  uint32_t s = seed;
  for (int i = 0; i < MT_N; ++i) {
    key[i] = s;
    s = 1812433253u * (s ^ (s >> 30)) + (uint32_t)(i + 1);
  }
  return mx_replay_set_rng_state(r, key, MT_N, stream);
}
extern "C" int mx_replay_set_rng_state(mx_replay* r, const uint32_t key[624], int32_t pos, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  cudaMemcpyAsync(r->blob + r->L.off_rng, key, MT_N * 4, cudaMemcpyHostToDevice, s);
  cudaMemcpyAsync(r->blob + r->L.off_state + offsetof(MxReplayState, rng_pos), &pos, 4, cudaMemcpyHostToDevice, s);
  cudaStreamSynchronize(s);   // `key`/`pos` are caller stack memory
  return 0;
}
extern "C" int mx_replay_get_rng_state(mx_replay* r, uint32_t key[624], int32_t* pos, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  cudaMemcpyAsync(key, r->blob + r->L.off_rng, MT_N * 4, cudaMemcpyDeviceToHost, s);
  cudaMemcpyAsync(pos, r->blob + r->L.off_state + offsetof(MxReplayState, rng_pos), 4, cudaMemcpyDeviceToHost, s);
  cudaStreamSynchronize(s);
  return 0;
}

static int launch_gather(mx_replay* r, const int64_t* idx_dev, int B, cudaStream_t s) {
  {
    const int rc = mx_launch_gather_tma(r->tma, idx_dev, B, s);      // TMA tile copies (gather_tma.cu); -1: vectorised loads below
    if (rc >= 0) return rc;
  }
  const mx_replay_cfg& c = r->cfg;
  const mx_replay_layout& L = r->L;
  GatherArgs g;
  memset(&g, 0, sizeof(g));
  int nf = 0;
  long long cum = 0;
  auto add = [&](int64_t src_off, int64_t dst_off, int64_t ep_floats) {
    if (ep_floats == 0) return;
    g.f[nf].src = cat<float>(r, src_off);
    g.f[nf].dst = at<float>(r, dst_off);
    g.f[nf].ep4 = ep_floats / 4;
    g.cum4[nf] = cum;
    cum += ep_floats / 4;
    ++nf;
  };
  add(L.off_obs, L.off_b_obs, L.ep_obs);
  add(L.off_share, L.off_b_share, L.ep_share);
  add(L.off_acts, L.off_b_acts, L.ep_acts);
  add(L.off_avail, L.off_b_avail, L.ep_avail);
  g.rew_field = c.reward_norm ? nf : -1;
  add(L.off_rew, L.off_b_rew, L.ep_rew);
  add(L.off_dones, L.off_b_dones, L.ep_dones);
  add(L.off_dones_env, L.off_b_dones_env, L.ep_dones_env);
  add(L.off_actidx, L.off_b_actidx, L.ep_actidx);
  g.cum4[nf] = cum;
  g.nf = nf;
  g.B = B;
  g.idx = (const long long*)idx_dev;
  g.state = cat<MxReplayState>(r, L.off_state);
  long long total = cum * B;
  if (total >= (1ll << 31)) { mx_set_error("gather: batch of %lld 16-byte words exceeds the 32-bit index range", total); return 1; }
  // each thread moves >= 4 float4 per iteration; grid is a multiple of the SM count (persistent-style, grid-stride)
  long long want = (total + 1023) / 1024;
  int sms = mx_num_sms();
  int grid = (int)(want < 1 ? 1 : want);
  if (grid > sms * 8) grid = sms * 8;
  else if (grid > sms) grid = grid / sms * sms;
  return mx_launch("k_gather", k_gather, dim3(grid), dim3(256), 0, s, MX_STEP, g);
}

static int check_sample(mx_replay* r, int B) {
  if (B <= 0 || B > r->cfg.max_batch) { mx_set_error("sample: batch_size %d outside [1, max_batch=%d]", B, r->cfg.max_batch); return 1; }
  if (r->filled <= 0) { mx_set_error("sample: buffer is empty"); return 1; }
  return 0;
}

extern "C" int mx_replay_sample_uniform(mx_replay* r, int32_t B, void* stream) {
  if (check_sample(r, B)) return 1;
  cudaStream_t s = (cudaStream_t)stream;
  DrawArgs d;
  memset(&d, 0, sizeof(d));
  d.rng = at<uint32_t>(r, r->L.off_rng);
  d.state = at<MxReplayState>(r, r->L.off_state);
  d.B = B; d.per = 0;
  d.idx_out = at<long long>(r, r->L.off_b_idx);
  if (const int rc = mx_launch("k_draw", k_draw, dim3(1), dim3(256), 0, s, MX_PLAIN, d)) return rc;
  return launch_gather(r, at<int64_t>(r, r->L.off_b_idx), B, s);
}

extern "C" int mx_replay_gather(mx_replay* r, const int64_t* idx_dev, int32_t B, void* stream) {
  if (check_sample(r, B)) return 1;
  cudaStream_t s = (cudaStream_t)stream;
  if (idx_dev != at<int64_t>(r, r->L.off_b_idx)) cudaMemcpyAsync(at<int64_t>(r, r->L.off_b_idx), idx_dev, (size_t)B * 8, cudaMemcpyDeviceToDevice, s);
  return launch_gather(r, at<int64_t>(r, r->L.off_b_idx), B, s);
}

// Same gather with the indices still on the host (np.random.choice result in pinned memory): one H2D copy + the gather.
extern "C" int mx_replay_gather_host(mx_replay* r, const int64_t* idx_host, int32_t B, void* stream) {
  if (check_sample(r, B)) return 1;
  if (!idx_host) { mx_set_error("gather_host: null indices"); return 1; }
  cudaStream_t s = (cudaStream_t)stream;
  cudaMemcpyAsync(at<int64_t>(r, r->L.off_b_idx), idx_host, (size_t)B * 8, cudaMemcpyHostToDevice, s);
  return launch_gather(r, at<int64_t>(r, r->L.off_b_idx), B, s);
}

__global__ void k_set_beta(MxReplayState* st, double beta) { st->per_beta = beta; }

// Importance-sampling exponent for the NEXT replays of a captured whole-step sequence (rec_buffer.py:278: beta is an argument of every
// sample() and the runner anneals it, base_runner.py:159-160,235): a by-value kernel argument, so no host memory has to stay alive.
extern "C" int mx_replay_set_beta(mx_replay* r, double beta, void* stream) {
  if (!r || !r->cfg.use_per) { mx_set_error("mx_replay_set_beta: replay created without use_per"); return 1; }
  if (!(beta > 0)) { mx_set_error("mx_replay_set_beta: beta must be > 0"); return 1; }
  MX_LAUNCH(k_set_beta, dim3(1), dim3(1), 0, (cudaStream_t)stream, at<MxReplayState>(r, r->L.off_state), beta);   // (not counted or marked)
  return mx_check_launch("set_beta");
}

static int sample_per_impl(mx_replay* r, int32_t B, double beta, void* stream);
extern "C" int mx_replay_sample_per(mx_replay* r, int32_t B, double beta, void* stream) {
  if (!(beta > 0)) { mx_set_error("sample_per: beta must be > 0"); return 1; }                                                                  // rec_buffer.py:289
  return sample_per_impl(r, B, beta, stream);
}
int mx_replay_sample_per_state_beta(mx_replay* r, int32_t B, void* stream) { return sample_per_impl(r, B, -1.0, stream); }
static int sample_per_impl(mx_replay* r, int32_t B, double beta, void* stream) {
  if (check_sample(r, B)) return 1;
  if (!r->cfg.use_per) { mx_set_error("sample_per: replay created without use_per"); return 1; }
  if (!(r->filled > B)) { mx_set_error("Cannot sample with no completed episodes in the buffer! (len %d <= batch %d)", r->filled, B); return 1; }  // rec_buffer.py:287-288
  cudaStream_t s = (cudaStream_t)stream;
  DrawArgs d;
  memset(&d, 0, sizeof(d));
  d.rng = at<uint32_t>(r, r->L.off_rng);
  d.state = at<MxReplayState>(r, r->L.off_state);
  d.B = B; d.per = 1;
  d.idx_out = at<long long>(r, r->L.off_b_idx);
  d.sum_tree = at<double>(r, r->L.off_sum_tree);
  d.min_tree = at<double>(r, r->L.off_min_tree);
  d.cap = r->L.tree_cap;
  d.beta = beta;
  d.w_out = at<double>(r, r->L.off_b_weights);
  d.w32_out = at<float>(r, r->L.off_b_wf32);
  if (const int rc = mx_launch("k_draw", k_draw, dim3(1), dim3(256), 0, s, MX_PLAIN, d)) return rc;
  return launch_gather(r, at<int64_t>(r, r->L.off_b_idx), B, s);
}

extern "C" int mx_replay_update_priorities(mx_replay* r, const int64_t* idx_dev, const float* prio_dev, const double* leaves_f64_dev,
                                           const double* max_prio_host, int32_t B, void* stream) {
  if (!r->cfg.use_per) { mx_set_error("update_priorities: replay created without use_per"); return 1; }
  if (B <= 0 || B > 1024) { mx_set_error("update_priorities: B out of range"); return 1; }
  cudaStream_t s = (cudaStream_t)stream;
  (void)max_prio_host;
  TreeUpd u;
  memset(&u, 0, sizeof(u));
  u.sum_tree = at<double>(r, r->L.off_sum_tree); u.min_tree = at<double>(r, r->L.off_min_tree);
  u.cap = r->L.tree_cap; u.n = B; u.idx = (const long long*)idx_dev; u.capacity = r->cfg.capacity;
  u.prio = prio_dev; u.leaves = leaves_f64_dev; u.alpha = r->cfg.per_alpha; u.prime_from_max = 0;
  u.state = at<MxReplayState>(r, r->L.off_state); u.update_max = 1;
  return mx_launch("k_tree_update", k_tree_update, dim3(1), dim3(mx_round_up(B, 32)), 0, s, MX_PLAIN, u);
}

extern "C" int mx_replay_batch(const mx_replay* r, int32_t B, mx_batch* out) {
  if (B <= 0 || B > r->cfg.max_batch) { mx_set_error("mx_replay_batch: bad B"); return 1; }
  const mx_replay_layout& L = r->L;
  memset(out, 0, sizeof(*out));
  out->B = B;
  out->obs_ld = L.obs_ld; out->share_ld = L.share_ld; out->act_ld = L.act_ld;
  out->obs = cat<float>(r, L.off_b_obs);
  out->share = cat<float>(r, L.off_b_share);
  out->acts = cat<float>(r, L.off_b_acts);
  out->act_idx = cat<int32_t>(r, L.off_b_actidx);
  out->avail = r->cfg.use_avail ? cat<float>(r, L.off_b_avail) : nullptr;
  out->rewards = cat<float>(r, L.off_b_rew);
  out->dones = cat<float>(r, L.off_b_dones);
  out->dones_env = cat<float>(r, L.off_b_dones_env);
  out->weights = r->cfg.use_per ? cat<float>(r, L.off_b_wf32) : nullptr;
  out->idx = cat<int64_t>(r, L.off_b_idx);
  out->ep_tn_ld = (int32_t)L.ep_rew;          // == ep_dones == ep_actidx: round_up(T * N, 4)
  out->ep_t_ld = (int32_t)L.ep_dones_env;     // round_up(T, 4)
  return 0;
}
