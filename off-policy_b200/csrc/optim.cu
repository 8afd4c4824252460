// Gradient partial reduction, loss / PER finalisation, global-norm clip + Adam, Polyak target update.
//
// reference: torch.nn.utils.clip_grad_norm_(params, max_grad_norm) + torch.optim.Adam.step (qmix.py:190-193),
// soft_update (utils/util.py:123-134), PER priorities (qmix.py:176-181), train_info (qmix.py:195-198).
//
// Pipeline:  k_grad_reduce  : grad[i] = sum over per-CTA partials (deterministic order); block `gridDim.x-1`
//                             also finalises the scalar sums, the PER priorities and bumps the Adam step count
//            [NCCL all-reduce of grad[0 .. P+4) when world_size > 1]
//            k_adam         : every CTA recomputes ||grad||^2 over the whole (L2-resident) buffer in the same
//                             order -- no grid-wide barrier needed -- then clips and updates its own slice.
#include <math.h>

#include "mx_internal.h"
#include "mx_kernels.h"

// ---- phase 1 of the optimiser, shared by k_grad_reduce and k_optim_fused -------------------------------------------------------------
// scalar block: sum(1-bad), loss numerator, sum Q_tot(1-bad), element count -> grad[P .. P+3]; PER priorities.  Returns the four scalars.
MX_DEVINL float4 optim_scalars(const OptimArgs& a) {
  const int tid = threadIdx.x;
  __shared__ float red[3][256];
  __shared__ float4 s_out;
  float s0 = 0.f, s1 = 0.f, s2 = 0.f;
  for (int i = tid; i < a.spart_n; i += blockDim.x) { s0 += a.spart[i * 8]; s1 += a.spart[i * 8 + 1]; s2 += a.spart[i * 8 + 2]; }
  red[0][tid] = s0; red[1][tid] = s1; red[2][tid] = s2;
  __syncthreads();
  if (tid == 0) {
    float t0 = 0.f, t1 = 0.f, t2 = 0.f;
    for (int i = 0; i < (int)blockDim.x; ++i) { t0 += red[0][i]; t1 += red[1][i]; t2 += red[2][i]; }
    s_out = make_float4(t0, t1, t2, (float)(a.B * a.T));
    mx_st4(a.grad + a.P, s_out);
  }
  // ---- PER: new priority = (1-nu) * mean_t|e| + nu * max_t|e| + eps  (mean over all T, masked steps are zeros) ----
  if (a.prio) {
    for (int b = tid; b < a.B; b += blockDim.x) {
      float mx = 0.f, sm = 0.f;
      for (int t = 0; t < a.T; ++t) {
        const float e = fabsf(a.err[(size_t)b * a.T + t]);
        sm += e;
        mx = fmaxf(mx, e);
      }
      a.prio[b] = (1.f - a.per_nu) * (sm / (float)a.T) + a.per_nu * mx + a.per_eps;
    }
  }
  __syncthreads();
  return s_out;
}

// parameter block: 64 float4 columns (256 parameters) per block x 4 slices of the partial index: thread (c, sl) sums partials sl, sl+4, ...
// of its column with 16-byte loads (8 in flight), then the four slices are added in fixed order -> deterministic result.  Threads
// tid < 64 return the reduced float4 of column tid (zeros past P).
MX_DEVINL float4 optim_reduce_partials(const OptimArgs& a) {
  const int tid = threadIdx.x;
  __shared__ float4 sl_sum[4][64];
  const int c = tid & 63, sl = tid >> 6;
  const long long i = ((long long)blockIdx.x * 64 + c) * 4;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (i < a.P) {
    int parts = 0;
    for (int s = 0; s < a.nseg; ++s)
      if (i >= a.seg_begin[s] && i < a.seg_end[s]) parts = a.seg_parts[s];     // segment bounds are multiples of 4 floats
    const float* gp = a.gpart + i;
    const long long ld = a.gpart_ld > 0 ? a.gpart_ld : a.P;
    float4 b0 = acc, b1 = acc, b2 = acc, b3 = acc;
    int p = sl;
    for (; p + 28 < parts; p += 32) {
      const float4 v0 = mx_ld4(gp + (size_t)p * ld), v1 = mx_ld4(gp + (size_t)(p + 4) * ld);
      const float4 v2 = mx_ld4(gp + (size_t)(p + 8) * ld), v3 = mx_ld4(gp + (size_t)(p + 12) * ld);
      const float4 v4 = mx_ld4(gp + (size_t)(p + 16) * ld), v5 = mx_ld4(gp + (size_t)(p + 20) * ld);
      const float4 v6 = mx_ld4(gp + (size_t)(p + 24) * ld), v7 = mx_ld4(gp + (size_t)(p + 28) * ld);
      b0.x += v0.x; b0.y += v0.y; b0.z += v0.z; b0.w += v0.w;
      b1.x += v1.x; b1.y += v1.y; b1.z += v1.z; b1.w += v1.w;
      b2.x += v2.x; b2.y += v2.y; b2.z += v2.z; b2.w += v2.w;
      b3.x += v3.x; b3.y += v3.y; b3.z += v3.z; b3.w += v3.w;
      b0.x += v4.x; b0.y += v4.y; b0.z += v4.z; b0.w += v4.w;
      b1.x += v5.x; b1.y += v5.y; b1.z += v5.z; b1.w += v5.w;
      b2.x += v6.x; b2.y += v6.y; b2.z += v6.z; b2.w += v6.w;
      b3.x += v7.x; b3.y += v7.y; b3.z += v7.z; b3.w += v7.w;
    }
    for (; p < parts; p += 4) {
      const float4 v = mx_ld4(gp + (size_t)p * ld);
      b0.x += v.x; b0.y += v.y; b0.z += v.z; b0.w += v.w;
    }
    acc.x = (b0.x + b1.x) + (b2.x + b3.x); acc.y = (b0.y + b1.y) + (b2.y + b3.y);
    acc.z = (b0.z + b1.z) + (b2.z + b3.z); acc.w = (b0.w + b1.w) + (b2.w + b3.w);
  }
  sl_sum[sl][c] = acc;
  __syncthreads();
  float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
  if (tid < 64) {
    const float4 s0 = sl_sum[0][tid], s1 = sl_sum[1][tid], s2 = sl_sum[2][tid], s3 = sl_sum[3][tid];
    g.x = (s0.x + s1.x) + (s2.x + s3.x); g.y = (s0.y + s1.y) + (s2.y + s3.y);
    g.z = (s0.z + s1.z) + (s2.z + s3.z); g.w = (s0.w + s1.w) + (s2.w + s3.w);
  }
  return g;
}

// per-block sum of squares of the reduced float4 columns (threads tid < 64) -> normpart[blockIdx.x]
MX_DEVINL void optim_block_sumsq(const OptimArgs& a, float4 g, long long j) {
  const int tid = threadIdx.x;
  __shared__ float sq[2];
  if (tid < 64) {
    float q = (j < a.P) ? (g.x * g.x + g.y * g.y) + (g.z * g.z + g.w * g.w) : 0.f;
    q = mx_warp_sum(q);
    if ((tid & 31) == 0) sq[tid >> 5] = q;
  }
  __syncthreads();
  if (tid == 0 && a.normpart) a.normpart[blockIdx.x] = sq[0] + sq[1];
}

// Adam step count (1-based) and the running powers beta^t for the bias corrections (first step: 1 * beta)
MX_DEVINL void optim_bump_step(const OptimArgs& a) {
  const double t_old = a.adam_t[0];
  a.adam_t[0] = t_old + 1.0;
  a.adam_t[1] = (t_old == 0.0 ? 1.0 : a.adam_t[1]) * (double)a.beta1;
  a.adam_t[2] = (t_old == 0.0 ? 1.0 : a.adam_t[2]) * (double)a.beta2;
}

__global__ void __launch_bounds__(256) k_grad_reduce(OptimArgs a) {
  const int tid = threadIdx.x;
  MX_PDL_WAIT();
  if (blockIdx.x == gridDim.x - 1) {
    optim_scalars(a);
    if (tid == 0) optim_bump_step(a);
    return;
  }
  const float4 g = optim_reduce_partials(a);
  const long long j = ((long long)blockIdx.x * 64 + tid) * 4;
  if (tid < 64 && j < a.P) mx_st4(a.grad + j, g);
  optim_block_sumsq(a, g, j);      // lets k_adam skip re-reading the whole gradient
}

// ---- one-launch optimiser: partial reduction -> [all-reduce over peer memory] -> global-norm clip -> Adam [-> Polyak] ----------------
// Grid = the k_grad_reduce grid (one block per 256 parameters + the scalar block), all co-resident (checked by the launcher), joined
// by ONE grid barrier (sense-reversing counter in device memory) between the reduction and the update: the global gradient norm needs
// every block's sum of squares.  The reduced gradient never leaves the registers of the 64 threads that apply it.
// Data parallel (a.p2p_world > 1): every block PUSHES its reduced columns into slot [step parity][own rank] of every peer's symmetric
// block (remote stores are fire-and-forget; the later reads are local), the last block to finish raises flag[own rank] = step on
// every peer, all blocks wait for the world's flags (which also orders the local blocks) and add the slots in rank order -- every
// rank computes the same bits.  A peer that never arrives (10 s) sets the sticky abort word: NO rank-local update is applied and
// info[7] = -1 tells the host, which raises.
MX_DEVINL unsigned optim_ld_volatile(const unsigned* p) { return *reinterpret_cast<const volatile unsigned*>(p); }
MX_DEVINL float4 optim_ld4_volatile(const float* p) {
#if MX_EMU
  return *reinterpret_cast<const float4*>(p);
#else
  float4 r;      // never served from a stale L1 line (written by another GPU / another SM during this kernel)
  asm volatile("ld.volatile.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
#endif
}

// ---- flag-in-data ("LL") exchange lines: a float4 of gradient columns travels as two 16-byte lines {x, flag, y, flag} {z, flag, w, flag};
// a line is written by ONE vector store and read by ONE vector load, so data and flags arrive together: no fence, no arrival counter,
// no separate flag hop -- a column's owner thread adds a peer's contribution the moment that peer's two lines show this step's flag.
#if !MX_EMU
__device__ __forceinline__ void optim_ll_store(float* dst, float4 v, unsigned flag) {
  asm volatile("st.volatile.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "r"(__float_as_uint(v.x)), "r"(flag), "r"(__float_as_uint(v.y)), "r"(flag) : "memory");
  asm volatile("st.volatile.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(dst + 4), "r"(__float_as_uint(v.z)), "r"(flag), "r"(__float_as_uint(v.w)), "r"(flag) : "memory");
}
__device__ __forceinline__ bool optim_ll_load(const float* src, float4* v, unsigned flag) {
  unsigned a0, a1, a2, a3, b0, b1, b2, b3;
  asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(a0), "=r"(a1), "=r"(a2), "=r"(a3) : "l"(src) : "memory");
  asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(b0), "=r"(b1), "=r"(b2), "=r"(b3) : "l"(src + 4) : "memory");
  *v = make_float4(__uint_as_float(a0), __uint_as_float(a2), __uint_as_float(b0), __uint_as_float(b2));
  return a1 == flag && a3 == flag && b1 == flag && b3 == flag;
}
#endif

__global__ void __launch_bounds__(256) k_optim_fused(OptimArgs a) {
  const int tid = threadIdx.x;
  const bool scalar_blk = blockIdx.x == gridDim.x - 1;
  __shared__ unsigned s_gen, s_last;
  __shared__ double red[8];
  __shared__ float s_scale, s_step, s_bc2s;
  MX_PDL_WAIT();
  if (tid == 0) s_gen = optim_ld_volatile(a.sync + 2);       // barrier generation, read before this block arrives anywhere
  const double t_old = a.adam_t[0];                          // (rewritten by the scalar block only after the grid barrier)
  const double b1p = (t_old == 0.0 ? 1.0 : a.adam_t[1]) * (double)a.beta1, b2p = (t_old == 0.0 ? 1.0 : a.adam_t[2]) * (double)a.beta2;
  const unsigned step = (unsigned)t_old + 1u;
  const long long j = ((long long)blockIdx.x * 64 + tid) * 4;
  float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 sc = g;
  if (a.phase == 2) {                    // second launch of the two-launch form: the reduced columns come back from memory
    if (!scalar_blk && tid < 64 && j < a.P) g = mx_ld4(a.grad + j);
  } else if (scalar_blk) sc = optim_scalars(a);
  else {
    g = optim_reduce_partials(a);
    if (a.p2p_world <= 1 && tid < 64 && j < a.P) mx_st4(a.grad + j, g);
  }
#if !MX_EMU
  if (a.p2p_world > 1 && a.phase == 0 && a.p2p_ll) {
    // ---- data-parallel exchange, flag-in-data lines (default): push this rank's columns into every peer's line array of this step's
    //      parity, then add the peers' lines in rank order as they arrive (the line arrays follow the slots + flags of the protocol below) ----
    const int W = a.p2p_world;
    unsigned long long ts0 = 0, ts1 = 0, ts2 = 0;
    const bool stamp = scalar_blk && tid == 0 && a.xstat;
    if (stamp) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(ts0));
    const long long col = scalar_blk ? a.P : j;
    const bool owner = scalar_blk ? tid == 0 : (tid < 64 && j < a.P);
    const float4 mine = scalar_blk ? sc : g;
    const size_t ll0 = 2 * (size_t)W * a.p2p_slot + 64 + (size_t)(step & 1u) * W * 2 * a.p2p_slot;
    if (owner) {
      for (int p = 0; p < W; ++p)
        if (p != a.p2p_rank) optim_ll_store(a.p2p_blocks[p] + ll0 + (size_t)a.p2p_rank * 2 * a.p2p_slot + 2 * col, mine, step);
      if (stamp) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(ts1));
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      unsigned long long t0 = 0;
      for (int p = 0; p < W; ++p) {        // rank order on every rank: bit-identical sums everywhere
        float4 v = mine;
        if (p != a.p2p_rank) {
          const float* src = a.p2p_blocks[a.p2p_rank] + ll0 + (size_t)p * 2 * a.p2p_slot + 2 * col;
          unsigned spins = 0;
          while (!optim_ll_load(src, &v, step)) {
            if ((++spins & 1023u) == 0) {
              unsigned long long t1;
              asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
              if (t0 == 0) t0 = t1;
              if (t1 - t0 > a.p2p_timeout_ns || optim_ld_volatile(a.sync + 3)) { atomicExch(a.sync + 3, 1u); break; }     // 10 s: a peer died; do not hang the device
            }
          }
        }
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
      }
      mx_st4(a.grad + col, acc);
      if (scalar_blk) sc = acc; else g = acc;
      if (stamp) {
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(ts2));
        const float w = (float)(ts2 - ts1);
        a.xstat[0] += (float)(ts1 - ts0); a.xstat[1] += w; a.xstat[3] += 1.f;
        if (w > a.xstat[4]) a.xstat[4] = w;
      }
    }
  } else
#endif
  if (a.p2p_world > 1 && a.phase == 0) {
    const int W = a.p2p_world;
#if !MX_EMU
    unsigned long long ts0 = 0, ts1 = 0, ts2 = 0, ts3 = 0;       // exchange breakdown (scalar block, thread 0): where the data-parallel step loses time
    const bool stamp = scalar_blk && tid == 0 && a.xstat;
    if (stamp) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(ts0));
#endif
    const size_t slot0 = (size_t)(step & 1u) * W * a.p2p_slot;
    const long long col = scalar_blk ? a.P : j;                       // the scalar block owns the four scalars behind the parameters
    const bool owner = scalar_blk ? tid == 0 : (tid < 64 && j < a.P);
    const float4 mine = scalar_blk ? sc : g;
    if (owner)
      for (int p = 0; p < W; ++p) mx_st4(a.p2p_blocks[p] + slot0 + (size_t)a.p2p_rank * a.p2p_slot + col, mine);
    __syncthreads();                     // every thread of the block has issued its remote stores ...
    if (tid == 0) {
      __threadfence_system();            // ... ONE system-scope fence per block orders them (cumulative through the barrier) before the arrival below;
                                         // a fence in every thread costs ~7 us here (56k fences wait for their NVLink acknowledgements at once)
      const unsigned last = (atomicAdd(a.sync + 0, 1u) == gridDim.x - 1) ? 1u : 0u;
      if (last) a.sync[0] = 0u;
      s_last = last;
    }
    __syncthreads();
    unsigned* my_flags = reinterpret_cast<unsigned*>(a.p2p_blocks[a.p2p_rank] + 2 * (size_t)W * a.p2p_slot);
    if (s_last && tid < W) {             // every block of this rank has fenced its part of the slot: tell the peers (and ourselves)
      __threadfence_system();
      volatile unsigned* f = reinterpret_cast<unsigned*>(a.p2p_blocks[tid] + 2 * (size_t)W * a.p2p_slot) + a.p2p_rank;
      *f = step;
    }
#if !MX_EMU
    if (stamp) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(ts1));
#endif
    if (tid < W) {
#if !MX_EMU
      unsigned long long t0, t1;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
      while (optim_ld_volatile(my_flags + tid) < step) {
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        if (t1 - t0 > a.p2p_timeout_ns) { atomicExch(a.sync + 3, 1u); break; }      // 10 s: a peer died; do not hang the device
      }
      __threadfence_system();            // acquire: the peer's slot writes precede its flag store
#endif
    }
    __syncthreads();
#if !MX_EMU
    if (stamp) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(ts2));
#endif
    if (owner) {
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int p = 0; p < W; ++p) {      // rank order on every rank: bit-identical sums everywhere
        const float4 v = optim_ld4_volatile(a.p2p_blocks[a.p2p_rank] + slot0 + (size_t)p * a.p2p_slot + col);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
      }
      mx_st4(a.grad + col, acc);
      if (scalar_blk) sc = acc; else g = acc;
    }
#if !MX_EMU
    if (stamp) {
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(ts3));
      const float w = (float)(ts2 - ts1);
      a.xstat[0] += (float)(ts1 - ts0); a.xstat[1] += w; a.xstat[2] += (float)(ts3 - ts2); a.xstat[3] += 1.f;
      if (w > a.xstat[4]) a.xstat[4] = w;
    }
#endif
  }
  if (!scalar_blk && a.phase != 2) optim_block_sumsq(a, g, j);
  if (a.phase == 1) return;
  // ---- grid barrier ----
  __syncthreads();
  if (tid == 0 && a.phase == 0) {
    __threadfence();
    if (atomicAdd(a.sync + 1, 1u) == gridDim.x - 1) {
      a.sync[1] = 0u;
      __threadfence();
      atomicAdd(a.sync + 2, 1u);
    } else {
      while (optim_ld_volatile(a.sync + 2) == s_gen) {}
    }
    __threadfence();
  }
  __syncthreads();
  if (optim_ld_volatile(a.sync + 3)) {       // a peer never arrived: nothing is applied anywhere on this rank
    if (blockIdx.x == 0 && tid == 0) a.info[7] = -1.f;
    return;
  }
  // ---- ||g||, clip, Adam on the columns still held in registers ----
  const float* gtail = a.grad + a.P;
  const float denom = __ldcg(gtail + 0);
  const float invd = 1.0f / denom;
  double sp = 0.0;
  for (int i = tid; i < a.normpart_n; i += blockDim.x) sp += (double)__ldcg(a.normpart + i);
  sp = mx_warp_sum_d(sp);
  if ((tid & 31) == 0) red[tid >> 5] = sp;
  __syncthreads();
  if (tid == 0) {
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
    const float norm = (float)sqrt(t * ((double)invd * (double)invd));
    float coef = a.max_grad_norm / (norm + 1e-6f);       // clip_grad_norm_: always applied, clamped to 1
    if (coef > 1.f) coef = 1.f;
    s_scale = coef * invd;
    s_step = a.lr / (float)(1.0 - b1p);
    s_bc2s = (float)sqrt(1.0 - b2p);
    if (blockIdx.x == 0) {
      a.info[0] = __ldcg(gtail + 1) * invd;                // loss
      a.info[1] = norm;                                    // grad_norm (pre-clip)
      a.info[2] = __ldcg(gtail + 2) / __ldcg(gtail + 3);   // Q_tot mean over all (t,b)
      a.info[3] = denom;
    }
    if (scalar_blk) { a.adam_t[0] = t_old + 1.0; a.adam_t[1] = b1p; a.adam_t[2] = b2p; }
  }
  __syncthreads();
  if (scalar_blk || tid >= 64 || j >= a.P) return;
  const float scale = s_scale, stp = s_step, bc2s = s_bc2s;
  const float gg[4] = {g.x, g.y, g.z, g.w};
  const float4 th4 = mx_ld4(a.theta + j), m4 = mx_ld4(a.adam_m + j), v4 = mx_ld4(a.adam_v + j);
  float th[4] = {th4.x, th4.y, th4.z, th4.w}, m[4] = {m4.x, m4.y, m4.z, m4.w}, v[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    float ge = gg[e] * scale;
    if (a.weight_decay != 0.f) ge = fmaf(a.weight_decay, th[e], ge);     // torch Adam: grad.add(param, alpha=weight_decay)
    m[e] = m[e] + (ge - m[e]) * (1.f - a.beta1);                         // exp_avg.lerp_(grad, 1 - beta1)
    v[e] = v[e] * a.beta2 + (1.f - a.beta2) * ge * ge;                   // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2)
    const float den = sqrtf(v[e]) / bc2s + a.eps;
    th[e] = th[e] - stp * (m[e] / den);
  }
  mx_st4(a.theta + j, make_float4(th[0], th[1], th[2], th[3]));
  mx_st4(a.adam_m + j, make_float4(m[0], m[1], m[2], m[3]));
  mx_st4(a.adam_v + j, make_float4(v[0], v[1], v[2], v[3]));
  if (a.fuse_polyak) {                                                    // util.py:132-134 fused epilogue
    const float4 t4 = mx_ld4(a.theta_tgt + j);
    mx_st4(a.theta_tgt + j, make_float4(t4.x * (1.0f - a.tau) + th[0] * a.tau, t4.y * (1.0f - a.tau) + th[1] * a.tau,
                                        t4.z * (1.0f - a.tau) + th[2] * a.tau, t4.w * (1.0f - a.tau) + th[3] * a.tau));
  }
}

__global__ void __launch_bounds__(1024) k_adam(OptimArgs a) {
  __shared__ double red[32];
  __shared__ float s_scale, s_step, s_bc2s;
  const int tid = threadIdx.x;
  MX_PDL_WAIT();
  if ((a.abort ? *a.abort : a.info[7]) < 0.f) return;     // the peer-memory exchange timed out (p2p.cu): the sums are not trustworthy, apply nothing
  const float denom = a.grad[a.P + 0];
  const float invd = 1.0f / denom;
  // ||g||^2 over the full vector, identical summation order in every CTA (no grid-wide barrier needed)
  double ds;
  if (a.normpart) {       // single GPU: per-block sums of squares of the numerators left by k_grad_reduce
    double sp = 0.0;
    for (int i = tid; i < a.normpart_n; i += blockDim.x) sp += (double)a.normpart[i];
    ds = mx_warp_sum_d(sp) * ((double)invd * (double)invd);
  } else {                // data parallel: the gradient was all-reduced after k_grad_reduce
    float sf = 0.f;
    const long long P4 = a.P / 4;
#pragma unroll 4
    for (long long i = tid; i < P4; i += blockDim.x) {
      const float4 g = mx_ld4(a.grad + 4 * i);
      const float gx = g.x * invd, gy = g.y * invd, gz = g.z * invd, gw = g.w * invd;
      sf += (gx * gx + gy * gy) + (gz * gz + gw * gw);
    }
    ds = mx_warp_sum_d((double)sf);
  }
  if ((tid & 31) == 0) red[tid >> 5] = ds;
  __syncthreads();
  if (tid < 32) {
    double t = tid < (int)(blockDim.x >> 5) ? red[tid] : 0.0;
    t = mx_warp_sum_d(t);
    if (tid == 0) {
      const float norm = (float)sqrt(t);
      float coef = a.max_grad_norm / (norm + 1e-6f);       // clip_grad_norm_: always applied, clamped to 1
      if (coef > 1.f) coef = 1.f;
      s_scale = coef * invd;
      s_step = a.lr / (float)(1.0 - a.adam_t[1]);          // beta1^t, beta2^t maintained by k_grad_reduce
      s_bc2s = (float)sqrt(1.0 - a.adam_t[2]);
      if (blockIdx.x == 0) {
        a.info[0] = a.grad[a.P + 1] * invd;                // loss
        a.info[1] = norm;                                  // grad_norm (pre-clip)
        a.info[2] = a.grad[a.P + 2] / a.grad[a.P + 3];     // Q_tot mean over all (t,b)
        a.info[3] = denom;
      }
    }
  }
  __syncthreads();
  const float scale = s_scale, step = s_step, bc2s = s_bc2s;
  for (long long i = (long long)blockIdx.x * blockDim.x + tid; i < a.P; i += (long long)gridDim.x * blockDim.x) {
    float g = a.grad[i] * scale;
    if (a.weight_decay != 0.f) g = fmaf(a.weight_decay, a.theta[i], g);     // torch Adam: grad.add(param, alpha=weight_decay)
    float m = a.adam_m[i], v = a.adam_v[i];
    m = m + (g - m) * (1.f - a.beta1);                   // exp_avg.lerp_(grad, 1 - beta1)
    v = v * a.beta2 + (1.f - a.beta2) * g * g;           // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2)
    const float den = sqrtf(v) / bc2s + a.eps;
    const float th_new = a.theta[i] - step * (m / den);
    a.theta[i] = th_new;
    a.adam_m[i] = m;
    a.adam_v[i] = v;
    if (a.fuse_polyak) a.theta_tgt[i] = a.theta_tgt[i] * (1.0f - a.tau) + th_new * a.tau;   // util.py:132-134 fused epilogue
  }
}

__global__ void __launch_bounds__(256) k_polyak(float* __restrict__ tgt, const float* __restrict__ src, long long n4, float tau) {
  MX_PDL_WAIT();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 t = mx_ld4(tgt + 4 * i);
    const float4 s = mx_ld4(src + 4 * i);
    t.x = t.x * (1.0f - tau) + s.x * tau;                // util.py:132-134
    t.y = t.y * (1.0f - tau) + s.y * tau;
    t.z = t.z * (1.0f - tau) + s.z * tau;
    t.w = t.w * (1.0f - tau) + s.w * tau;
    mx_st4(tgt + 4 * i, t);
  }
}

int mx_launch_grad_reduce(const OptimArgs& a, cudaStream_t s) {
  const int grid = mx_grad_reduce_blocks(a.P) + 1;
  return mx_launch("k_grad_reduce", k_grad_reduce, dim3(grid), dim3(256), 0, s, MX_STEP, a);
}
int g_mx_optim_fused = 1;
int mx_launch_optim_fused(const OptimArgs& a, cudaStream_t s) {
#if MX_EMU
  // the emulator runs one CTA at a time, so a grid barrier cannot complete there: the same kernel as two launches (before / after
  // the barrier).  The peer-memory exchange inside the kernel needs concurrently running ranks: the emulated tests use the separate
  // exchange kernels (p2p.cu) instead.
  if (!g_mx_optim_fused || !a.sync || !a.normpart || a.p2p_world > 1) return -1;
  OptimArgs b = a;
  const int grid = mx_grad_reduce_blocks(a.P) + 1;
  b.phase = 1;
  MX_LAUNCH(k_optim_fused, dim3(grid), dim3(256), 0, s, b);      // uncounted: the two phases are one launch on the device
  b.phase = 2;
  return mx_launch("k_optim_fused", k_optim_fused, dim3(grid), dim3(256), 0, s, MX_PLAIN, b);
#else
  if (!g_mx_optim_fused || !a.sync || !a.normpart) return -1;
  const int grid = mx_grad_reduce_blocks(a.P) + 1;
  static int per_sm = -1;
  if (per_sm < 0 && cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_optim_fused, 256, 0) != cudaSuccess) per_sm = 0;
  if (grid > per_sm * mx_num_sms()) return -1;        // not all blocks co-resident: no grid barrier
  const int rc = mx_launch("k_optim_fused", k_optim_fused, dim3(grid), dim3(256), 0, s, MX_STEP, a);
  MX_PDL_THETA_WRITTEN();
  return rc;
#endif
}
int mx_launch_adam(const OptimArgs& a, cudaStream_t s) {
  int grid = (int)((a.P + 4095) / 4096);
  const int sms = mx_num_sms();
  if (grid > sms) grid = sms;
  const int rc = mx_launch("k_adam", k_adam, dim3(grid), dim3(1024), 0, s, MX_STEP, a);
  MX_PDL_THETA_WRITTEN();
  return rc;
}
int mx_launch_polyak(float* tgt, const float* src, long long n, float tau, cudaStream_t s) {
  const long long n4 = n / 4;
  int grid = (int)((n4 + 255) / 256);
  const int sms = mx_num_sms();
  if (grid > sms) grid = sms;
  if (grid < 1) grid = 1;
  const int rc = mx_launch("k_polyak", k_polyak, dim3(grid), dim3(256), 0, s, MX_STEP, tgt, src, n4, tau);
  MX_PDL_THETA_WRITTEN();
  return rc;
}
