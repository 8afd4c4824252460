// QMIX monotonic hypernetwork mixer: target forward, live forward, TD target / masked loss, and the live
// mixer's backward -- one kernel, one CTA per tile of 16*RM (b,t) elements, weights streamed through shared
// memory in 64-row chunks.
//
// reference: algorithms/qmix/algorithm/q_mixer.py:68-94 (abs hyper-weights, ELU), qmix.py:155-187
// (Q_tot, TD target with (1-dones_env)*gamma, bad-transition mask shifted by one step, MSE/Huber, PER weights).
// VDN (vdn_mixer.py:28-40 intent): Q_tot = sum_n q_n.
//
// Gradients are accumulated as NUMERATORS (no division by sum(1-bad)): the optimiser kernel divides by the
// (all-reduced) denominator, so data-parallel ranks can simply sum their buffers.
#include "mx_internal.h"
#include "mx_kernels.h"
#include "mx_tile.cuh"

#include <string.h>

struct MixSmem {
  int ldS, ldH, ldP, ldM, ldw;
  int o_s, o_h1, o_h2, o_hb, o_p1, o_b1, o_p2, o_hid, o_q, o_vec, o_wc, total;
};
// wide: no state tile (the wide-state path reads the state layers' pre-activations instead)
static MixSmem mix_smem_layout(const MxMixLayout& L, int TE, bool wide = false) {
  MixSmem m;
  const int S64 = wide ? 0 : mx_round_up(L.S, 64), H64 = mx_round_up(L.HY, 64), P64 = mx_round_up(L.N * L.ME, 64), M64 = mx_round_up(L.ME, 64);
  m.ldS = mx_ld(S64); m.ldH = mx_ld(H64); m.ldP = mx_ld(P64); m.ldM = mx_ld(M64);
  m.ldw = mx_ld(S64 > H64 ? S64 : H64);
  int o = 0;
  m.o_s = o; o += wide ? 0 : TE * m.ldS;
  m.o_h1 = o; o += TE * m.ldH;
  m.o_h2 = o; o += TE * m.ldH;
  m.o_hb = o; o += TE * m.ldH;
  m.o_p1 = o; o += TE * m.ldP;
  m.o_b1 = o; o += TE * m.ldM;
  m.o_p2 = o; o += TE * m.ldM;
  m.o_hid = o; o += TE * m.ldM;
  m.o_q = o; o += TE * 32;
  m.o_vec = o; o += 8 * TE;         // b2, Q, Qn, dQ, valid, ...
  m.o_wc = o; o += 64 * m.ldw;
  m.total = o;
  return m;
}

bool mx_mix_wide_state(const MxMixLayout& L) { return (size_t)mix_smem_layout(L, 32).total * sizeof(float) + 16 > MX_SMEM_OPTIN_MAX; }

void mx_mix_wide_layout(const MxMixLayout& L, MxMixWide* w) {
  memset(w, 0, sizeof(*w));
  const int NM = L.N * L.ME;
  const int rows[4] = {L.layers == 2 ? L.HY : NM, L.layers == 2 ? L.HY : L.ME, L.HY, L.ME};
  const int wo[4] = {L.layers == 2 ? L.w1a : L.w1b, L.layers == 2 ? L.w2a : L.w2b, L.wb2a, L.wb1};
  const int bo[4] = {L.layers == 2 ? L.b1a : L.b1b, L.layers == 2 ? L.b2a : L.b2b, L.bb2a, L.bb1};
  int c = 0;
  for (int j = 0; j < 4; ++j) { w->col[j] = c; w->rows[j] = rows[j]; w->w[j] = wo[j]; w->b[j] = bo[j]; c += mx_round_up(rows[j], 4); }
  w->C = c;
  w->Cp = mx_round_up(c, 16);
  w->Sp = mx_round_up(L.S, 32);
}

// Y_s[r][c] = act(sum_k X_s[r][k] W[c][k] + b[c]) for c < Nout (columns up to round_up(Nout,64) are written, zeros beyond)
template <int RM>
__device__ MX_NOINLINE void tile_linear(const float* X_s, int ldx, int K, const float* __restrict__ W, const float* __restrict__ b, int Nout, float* Y_s,
                           int ldy, bool relu, float* Wc, int ldw) {
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int Kpad = (K + 3) & ~3;
  for (int nc = 0; nc * 64 < Nout; ++nc) {
    mx_stage_weight(Wc, ldw, W, Nout, K, K, nc * 64, 0, Kpad);
    __syncthreads();
    float acc[RM][4];
#pragma unroll
    for (int i = 0; i < RM; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    mx_mm_nt<RM>(X_s, ldx, Wc, ldw, Kpad, acc);
#pragma unroll
    for (int i = 0; i < RM; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = nc * 64 + tx + 16 * j;
        float v = 0.f;
        if (c < Nout) {
          v = acc[i][j] + b[c];
          if (relu) v = fmaxf(v, 0.f);
        }
        Y_s[(ty * RM + i) * ldy + c] = v;
      }
    __syncthreads();
  }
}

// dX_s[r][k] = (mask_s[r][k] > 0 ? 1 : 0) * sum_n dY_s[r][n] W[n][k]   for k < K (written over round_up(K,64) cols).
// dX_s may alias mask_s (each element is read and written by the same thread).
template <int RM>
__device__ MX_NOINLINE void tile_dgrad_relu(const float* dY_s, int ldy, int Nout, const float* __restrict__ W, int K, float* dX_s, const float* mask_s,
                               int ldx, float* Wc, int ldw) {
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  for (int kb = 0; kb * 64 < K; ++kb) {
    float acc[RM][4];
#pragma unroll
    for (int i = 0; i < RM; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    for (int nc = 0; nc * 64 < Nout; ++nc) {
      mx_stage_weight(Wc, ldw, W, Nout, K, K, nc * 64, kb * 64, 64);
      __syncthreads();
      mx_mm_nn<RM>(dY_s + nc * 64, ldy, Wc, ldw, acc);
      __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < RM; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int k = kb * 64 + 4 * tx + j;
        const int o = (ty * RM + i) * ldx + k;
        const float keep = (k < K && mask_s[o] > 0.f) ? 1.f : 0.f;
        dX_s[o] = keep * acc[i][j];
      }
  }
  __syncthreads();
}

// dW (+)= dY_s^T X_s ; db (+)= colsum(dY_s)
__device__ MX_NOINLINE void tile_wgrad(const float* dY_s, int ldy, int Nout, const float* X_s, int ldx, int K, int TE, float* dW, float* db, bool accumulate) {
  for (int nb = 0; nb * 64 < Nout; ++nb)
    for (int kb = 0; kb * 64 < K; ++kb) mx_wgrad_block(dY_s + nb * 64, ldy, X_s + kb * 64, ldx, TE, dW, Nout, K, nb * 64, kb * 64, accumulate);
  mx_colsum(dY_s, ldy, TE, Nout, db, accumulate);
}

// the state-only hypernetwork layers of one tile: h1/h2/hb (post-ReLU), p1 = hyper_w1(s), p2 = hyper_w2(s), b1 = hyper_b1(s)
template <int RM>
MX_DEVINL void mixer_hyper(const float* __restrict__ th, const MxMixLayout& L, const MixSmem& sm, float* smem) {
  float* s_s = smem + sm.o_s;
  float* h1_s = smem + sm.o_h1; float* h2_s = smem + sm.o_h2; float* hb_s = smem + sm.o_hb;
  float* p1_s = smem + sm.o_p1; float* b1_s = smem + sm.o_b1; float* p2_s = smem + sm.o_p2;
  float* Wc = smem + sm.o_wc;
  const int NM = L.N * L.ME;
  if (L.layers == 2) {
    tile_linear<RM>(s_s, sm.ldS, L.S, th + L.w1a, th + L.b1a, L.HY, h1_s, sm.ldH, true, Wc, sm.ldw);
    tile_linear<RM>(h1_s, sm.ldH, L.HY, th + L.w1b, th + L.b1b, NM, p1_s, sm.ldP, false, Wc, sm.ldw);
    tile_linear<RM>(s_s, sm.ldS, L.S, th + L.w2a, th + L.b2a, L.HY, h2_s, sm.ldH, true, Wc, sm.ldw);
    tile_linear<RM>(h2_s, sm.ldH, L.HY, th + L.w2b, th + L.b2b, L.ME, p2_s, sm.ldM, false, Wc, sm.ldw);
  } else {
    tile_linear<RM>(s_s, sm.ldS, L.S, th + L.w1b, th + L.b1b, NM, p1_s, sm.ldP, false, Wc, sm.ldw);
    tile_linear<RM>(s_s, sm.ldS, L.S, th + L.w2b, th + L.b2b, L.ME, p2_s, sm.ldM, false, Wc, sm.ldw);
  }
  tile_linear<RM>(s_s, sm.ldS, L.S, th + L.wb1, th + L.bb1, L.ME, b1_s, sm.ldM, false, Wc, sm.ldw);
  tile_linear<RM>(s_s, sm.ldS, L.S, th + L.wb2a, th + L.bb2a, L.HY, hb_s, sm.ldH, true, Wc, sm.ldw);
}

template <int RM>
MX_DEVINL void mixer_forward(const float* __restrict__ th, const MxMixLayout& L, const MixSmem& sm, float* smem, float* Qout /*[TE] in smem*/) {
  constexpr int TE = 16 * RM;
  float* hb_s = smem + sm.o_hb;
  float* p1_s = smem + sm.o_p1; float* b1_s = smem + sm.o_b1; float* p2_s = smem + sm.o_p2; float* hid_s = smem + sm.o_hid;
  float* q_s = smem + sm.o_q;
  mixer_hyper<RM>(th, L, sm, smem);
  // hidden = ELU(q . |w1| + b1)   (pre-activation kept in hid_s)
  for (int idx = threadIdx.x; idx < TE * L.ME; idx += MX_TILE_THREADS) {
    const int e = idx / L.ME, k = idx % L.ME;
    float v = b1_s[e * sm.ldM + k];
    for (int n = 0; n < L.N; ++n) v = fmaf(q_s[e * 32 + n], fabsf(p1_s[e * sm.ldP + n * L.ME + k]), v);
    hid_s[e * sm.ldM + k] = v;
  }
  __syncthreads();
  // Q_tot = ELU(hid) . |w2| + b2 ; b2 = hb . Wb2b + bb2b   (one half-warp of 16 lanes per element)
  {
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    for (int i = 0; i < RM; ++i) {
      const int e = ty * RM + i;
      float v = 0.f;
      for (int k = tx; k < L.ME; k += 16) {
        const float hp = hid_s[e * sm.ldM + k];
        const float hv = hp > 0.f ? hp : (expf(hp) - 1.f);
        v = fmaf(hv, fabsf(p2_s[e * sm.ldM + k]), v);
      }
      for (int k = tx; k < L.HY; k += 16) v = fmaf(hb_s[e * sm.ldH + k], th[L.wb2b + k], v);
      v = mx_row16_sum(v);
      if (tx == 0) Qout[e] = v + th[L.bb2b];
    }
  }
  __syncthreads();
}

template <int RM>
__global__ void __launch_bounds__(MX_TILE_THREADS) k_mixer(MixerArgs a, MixSmem sm) {
  constexpr int TE = 16 * RM;
  MX_DYN_SMEM(smem);
  const MxMixLayout L = a.L;
  const int tid = threadIdx.x;
  const int E = a.B * a.T;
  const int ntiles = (E + TE - 1) / TE;
  float* s_s = smem + sm.o_s;
  float* h1_s = smem + sm.o_h1; float* h2_s = smem + sm.o_h2; float* hb_s = smem + sm.o_hb;
  float* p1_s = smem + sm.o_p1; float* p2_s = smem + sm.o_p2; float* hid_s = smem + sm.o_hid;
  float* q_s = smem + sm.o_q; float* Wc = smem + sm.o_wc;
  float* Q_s = smem + sm.o_vec;          // [TE]
  float* Qn_s = Q_s + TE;                // [TE]
  float* dQ_s = Qn_s + TE;               // [TE]
  float* sc_s = dQ_s + TE;               // [3*TE] per-element scalar contributions
  float* gp = a.gpart + (size_t)blockIdx.x * a.P;
  float part_den = 0.f, part_loss = 0.f, part_q = 0.f;   // thread 0 only
  const int S64 = mx_round_up(L.S, 64);
  int iter = 0;
  MX_PDL_WAIT();

  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++iter) {
    const int e0 = tile * TE;
    const bool accum = iter > 0;
    // ================= target forward: Q_tot'(q_next[t], s[t+1]) =================
    for (int pass = 0; pass < 2; ++pass) {
      const bool tgt = (pass == 0);
      {   // state rows: 16-byte async copies (share_ld is a multiple of 4 and its pad columns are zero)
        const int nc4 = S64 >> 2, src4 = a.share_ld >> 2;
        for (int r = tid >> 4; r < TE; r += MX_TILE_THREADS / 16) {
          const int e = e0 + r;
          const float* src = nullptr;
          if (e < E) {
            const int b = e / a.T, t = e % a.T;
            src = a.share + ((size_t)b * (a.T + 1) + t + (tgt ? 1 : 0)) * a.share_ld;
          }
          for (int c4 = tid & 15; c4 < nc4; c4 += 16) {
            float* d = s_s + r * sm.ldS + 4 * c4;
            if (src && c4 < src4) mx_cp16(d, src + 4 * c4);
            else mx_st4(d, make_float4(0.f, 0.f, 0.f, 0.f));
          }
        }
        mx_cp_commit();
      }
      for (int idx = tid; idx < TE * 32; idx += MX_TILE_THREADS) {
        const int r = idx / 32, n = idx % 32;
        const int e = e0 + r;
        float v = 0.f;
        if (e < E && n < L.N) v = (tgt ? a.q_next : a.q_taken)[(size_t)e * L.N + n];
        q_s[idx] = v;
      }
      mx_cp_wait<0>();
      __syncthreads();
      mixer_forward<RM>(tgt ? a.theta_tgt : a.theta, L, sm, smem, tgt ? Qn_s : Q_s);
    }
    // ================= TD target, masked loss, dQ =================
    if (tid < TE) {
      const int e = e0 + tid;
      float dq = 0.f, den = 0.f, ls = 0.f, qs = 0.f;
      if (e < E) {
        const int b = e / a.T, t = e % a.T;
        const float rew = a.rewards[(size_t)b * a.ld_tn + (size_t)t * L.N];              // agent 0 (qmix.py:159)
        const float de = a.dones_env[(size_t)b * a.ld_t + t];
        const float bad = t > 0 ? a.dones_env[(size_t)b * a.ld_t + t - 1] : 0.f;     // qmix.py:161
        const float y = rew + (1.f - de) * a.gamma * Qn_s[tid];
        const float keep = 1.f - bad;
        const float err = (Q_s[tid] - y) * keep;
        const float w = a.weights ? a.weights[b] : 1.f;
        float le, dle;
        if (a.use_huber) {
          const float ae = fabsf(err);
          if (ae <= a.huber_delta) { le = 0.5f * err * err; dle = err; }
          else { le = a.huber_delta * (ae - 0.5f * a.huber_delta); dle = err > 0.f ? a.huber_delta : -a.huber_delta; }
        } else { le = err * err; dle = 2.f * err; }
        dq = dle * keep * w;
        den = keep; ls = le * w; qs = Q_s[tid] * keep;
        a.qtot[e] = Q_s[tid];
        a.qtot_next[e] = Qn_s[tid];
        a.err[e] = err;
      }
      dQ_s[tid] = dq;
      sc_s[tid] = den; sc_s[TE + tid] = ls; sc_s[2 * TE + tid] = qs;
    }
    __syncthreads();
    if (tid == 0)
      for (int r = 0; r < TE; ++r) { part_den += sc_s[r]; part_loss += sc_s[TE + r]; part_q += sc_s[2 * TE + r]; }

    // ================= backward through the live mixer =================
    const int NM = L.N * L.ME;
    // -- b2 path: d Wb2b, d bb2b, then hb_s <- d(pre-ReLU hb)
    for (int k = tid; k < L.HY; k += MX_TILE_THREADS) {
      float s = 0.f;
      for (int r = 0; r < TE; ++r) s = fmaf(dQ_s[r], hb_s[r * sm.ldH + k], s);
      float* p = gp + L.wb2b + k;
      *p = accum ? (*p + s) : s;
    }
    if (tid == 0) {
      float s = 0.f;
      for (int r = 0; r < TE; ++r) s += dQ_s[r];
      float* p = gp + L.bb2b;
      *p = accum ? (*p + s) : s;
    }
    __syncthreads();
    for (int idx = tid; idx < TE * sm.ldH; idx += MX_TILE_THREADS) {
      const int r = idx / sm.ldH, k = idx % sm.ldH;
      float v = 0.f;
      if (k < L.HY && hb_s[idx] > 0.f) v = dQ_s[r] * a.theta[L.wb2b + k];
      hb_s[idx] = v;
    }
    // -- elementwise: d hid_pre (into hid_s), d p2 (into p2_s)
    for (int idx = tid; idx < TE * sm.ldM; idx += MX_TILE_THREADS) {
      const int r = idx / sm.ldM, k = idx % sm.ldM;
      float dp2 = 0.f, dhp = 0.f;
      if (k < L.ME) {
        const float hp = hid_s[idx], p2 = p2_s[idx];
        const float hv = hp > 0.f ? hp : (expf(hp) - 1.f);
        const float dhid = dQ_s[r] * fabsf(p2);
        dhp = dhid * (hp > 0.f ? 1.f : (hv + 1.f));                      // ELU'(x) = exp(x) for x <= 0
        dp2 = dQ_s[r] * hv * (p2 > 0.f ? 1.f : (p2 < 0.f ? -1.f : 0.f));   // d|x| = sign(x)
      }
      hid_s[idx] = dhp;
      p2_s[idx] = dp2;
    }
    __syncthreads();
    // -- d q_taken[e][n] = sum_k |w1[n][k]| dhid_pre[k]     (half-warp per element)
    {
      const int tx = tid & 15, ty = tid >> 4;
      for (int i = 0; i < RM; ++i) {
        const int r = ty * RM + i;
        for (int n = 0; n < L.N; ++n) {
          float v = 0.f;
          for (int k = tx; k < L.ME; k += 16) v = fmaf(fabsf(p1_s[r * sm.ldP + n * L.ME + k]), hid_s[r * sm.ldM + k], v);
          v = mx_row16_sum(v);
          if (tx == 0 && e0 + r < E) a.dq_taken[(size_t)(e0 + r) * L.N + n] = v;
        }
      }
    }
    __syncthreads();
    // -- p1_s <- d p1 = q_n * dhid_pre[k] * sign(p1)
    for (int idx = tid; idx < TE * sm.ldP; idx += MX_TILE_THREADS) {
      const int r = idx / sm.ldP, c = idx % sm.ldP;
      float v = 0.f;
      if (c < NM) {
        const int n = c / L.ME, k = c % L.ME;
        const float p1 = p1_s[idx];
        v = q_s[r * 32 + n] * hid_s[r * sm.ldM + k] * (p1 > 0.f ? 1.f : (p1 < 0.f ? -1.f : 0.f));
      }
      p1_s[idx] = v;
    }
    __syncthreads();
    // -- hyper_b2 first layer, hyper_b1
    tile_wgrad(hb_s, sm.ldH, L.HY, s_s, sm.ldS, L.S, TE, gp + L.wb2a, gp + L.bb2a, accum);
    tile_wgrad(hid_s, sm.ldM, L.ME, s_s, sm.ldS, L.S, TE, gp + L.wb1, gp + L.bb1, accum);
    if (L.layers == 2) {
      // -- hyper_w2
      tile_wgrad(p2_s, sm.ldM, L.ME, h2_s, sm.ldH, L.HY, TE, gp + L.w2b, gp + L.b2b, accum);
      __syncthreads();
      tile_dgrad_relu<RM>(p2_s, sm.ldM, L.ME, a.theta + L.w2b, L.HY, h2_s, h2_s, sm.ldH, Wc, sm.ldw);
      tile_wgrad(h2_s, sm.ldH, L.HY, s_s, sm.ldS, L.S, TE, gp + L.w2a, gp + L.b2a, accum);
      // -- hyper_w1
      tile_wgrad(p1_s, sm.ldP, NM, h1_s, sm.ldH, L.HY, TE, gp + L.w1b, gp + L.b1b, accum);
      __syncthreads();
      tile_dgrad_relu<RM>(p1_s, sm.ldP, NM, a.theta + L.w1b, L.HY, h1_s, h1_s, sm.ldH, Wc, sm.ldw);
      tile_wgrad(h1_s, sm.ldH, L.HY, s_s, sm.ldS, L.S, TE, gp + L.w1a, gp + L.b1a, accum);
    } else {
      tile_wgrad(p2_s, sm.ldM, L.ME, s_s, sm.ldS, L.S, TE, gp + L.w2b, gp + L.b2b, accum);
      tile_wgrad(p1_s, sm.ldP, NM, s_s, sm.ldS, L.S, TE, gp + L.w1b, gp + L.b1b, accum);
    }
    __syncthreads();
  }
  if (tid == 0) {
    float* sp = a.spart + (size_t)blockIdx.x * 8;
    sp[0] = part_den; sp[1] = part_loss; sp[2] = part_q;
  }
}

// VDN: Q_tot = sum_n q_n (no parameters); same loss / dQ code path, one thread per element.
__global__ void __launch_bounds__(256) k_vdn_mix(MixerArgs a) {
  const int E = a.B * a.T;
  const int N = a.N;
  float den = 0.f, ls = 0.f, qs = 0.f;
  MX_PDL_WAIT();
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < E; e += gridDim.x * blockDim.x) {
    float Q = 0.f, Qn = 0.f;
    for (int n = 0; n < N; ++n) { Q += a.q_taken[(size_t)e * N + n]; Qn += a.q_next[(size_t)e * N + n]; }
    const int b = e / a.T, t = e % a.T;
    const float rew = a.rewards[(size_t)b * a.ld_tn + (size_t)t * N];
    const float de = a.dones_env[(size_t)b * a.ld_t + t];
    const float bad = t > 0 ? a.dones_env[(size_t)b * a.ld_t + t - 1] : 0.f;
    const float y = rew + (1.f - de) * a.gamma * Qn;
    const float keep = 1.f - bad;
    const float err = (Q - y) * keep;
    const float w = a.weights ? a.weights[b] : 1.f;
    float le, dle;
    if (a.use_huber) {
      const float ae = fabsf(err);
      if (ae <= a.huber_delta) { le = 0.5f * err * err; dle = err; }
      else { le = a.huber_delta * (ae - 0.5f * a.huber_delta); dle = err > 0.f ? a.huber_delta : -a.huber_delta; }
    } else { le = err * err; dle = 2.f * err; }
    const float dq = dle * keep * w;
    for (int n = 0; n < N; ++n) a.dq_taken[(size_t)e * N + n] = dq;
    a.qtot[e] = Q; a.qtot_next[e] = Qn; a.err[e] = err;
    den += keep; ls += le * w; qs += Q * keep;
  }
  __shared__ float red[3][256];
  red[0][threadIdx.x] = den; red[1][threadIdx.x] = ls; red[2][threadIdx.x] = qs;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s0 = 0.f, s1 = 0.f, s2 = 0.f;
    for (int i = 0; i < (int)blockDim.x; ++i) { s0 += red[0][i]; s1 += red[1][i]; s2 += red[2][i]; }
    float* sp = a.spart + (size_t)blockIdx.x * 8;
    sp[0] = s0; sp[1] = s1; sp[2] = s2;
  }
}

// =====================================================================================================
// Split pipeline: hyper_fwd ; core ; hyper_bwd  ==  k_mixer, with the per-element hypernet outputs in global
// memory (L2-resident).  hyper_fwd needs only the sampled states and the parameters, hyper_bwd only core's
// outputs, so the learner (qmix.cu) runs both on a forked branch beside the agent-net kernels; only the tiny
// q-dependent core stays between k_qhead and k_qhead_bwd.
// =====================================================================================================
// state rows of tile [e0, e0+TE) -> s_s (16-byte async copies; pad columns and rows >= E zero-filled)
MX_DEVINL void mix_stage_states(const MixerArgs& a, const MixSmem& sm, float* s_s, int e0, int E, int TE, int S64, int tshift) {
  const int tid = threadIdx.x;
  const int nc4 = S64 >> 2, src4 = a.share_ld >> 2;
  for (int r = tid >> 4; r < TE; r += MX_TILE_THREADS / 16) {
    const int e = e0 + r;
    const float* src = nullptr;
    if (e < E) {
      const int b = e / a.T, t = e % a.T;
      src = a.share + ((size_t)b * (a.T + 1) + t + tshift) * a.share_ld;
    }
    for (int c4 = tid & 15; c4 < nc4; c4 += 16) {
      float* d = s_s + r * sm.ldS + 4 * c4;
      if (src && c4 < src4) mx_cp16(d, src + 4 * c4);
      else mx_st4(d, make_float4(0.f, 0.f, 0.f, 0.f));
    }
  }
}
// smem tile [TE][lds] (columns [0, gcols) ) -> global rows e0.. of dst[E][gcols]   (gcols % 4 == 0)
MX_DEVINL void mix_tile_store(const float* src_s, int lds, float* __restrict__ dst, int gcols, int e0, int E, int TE) {
  const int nc4 = gcols >> 2;
  for (int idx = threadIdx.x; idx < TE * nc4; idx += MX_TILE_THREADS) {
    const int r = idx / nc4, c4 = idx - r * nc4;
    if (e0 + r < E) mx_st4(dst + (size_t)(e0 + r) * gcols + 4 * c4, mx_ld4(src_s + r * lds + 4 * c4));
  }
}
// global rows e0.. of src[E][gcols] -> smem tile [TE][lds], zero-filled out to `width` columns (width % 4 == 0, width <= lds)
MX_DEVINL void mix_tile_load(float* dst_s, int lds, int width, const float* __restrict__ src, int gcols, int e0, int E, int TE) {
  const int nc4 = width >> 2, g4 = gcols >> 2;
  for (int idx = threadIdx.x; idx < TE * nc4; idx += MX_TILE_THREADS) {
    const int r = idx / nc4, c4 = idx - r * nc4;
    float* d = dst_s + r * lds + 4 * c4;
    if (e0 + r < E && c4 < g4) mx_cp16(d, src + (size_t)(e0 + r) * gcols + 4 * c4);
    else mx_st4(d, make_float4(0.f, 0.f, 0.f, 0.f));
  }
}

// wide-state path: block `blk` of net `net`'s state-layer pre-activations for the tile's elements (state row b (T+1) + t + net),
// ReLU applied when `relu`, zero-filled out to `width` columns
MX_DEVINL void mix_pre_load(float* dst_s, int lds, int width, const MixerArgs& a, int net, int blk, bool relu, int e0, int E, int TE) {
  const float* pre = a.pre + (size_t)net * a.B * (a.T + 1) * a.wl.Cp + a.wl.col[blk];
  const int nc4 = width >> 2, g4 = mx_round_up(a.wl.rows[blk], 4) >> 2;
  for (int idx = threadIdx.x; idx < TE * nc4; idx += MX_TILE_THREADS) {
    const int r = idx / nc4, c4 = idx - r * nc4, e = e0 + r;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (e < E && c4 < g4) {
      const int b = e / a.T, t = e - b * a.T;
      v = mx_ld4(pre + ((size_t)b * (a.T + 1) + t + net) * a.wl.Cp + 4 * c4);
      if (relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
    }
    mx_st4(dst_s + r * lds + 4 * c4, v);
  }
}
// wide-state path: the tile's gradient at block `blk`'s pre-activations -> d_pre rows e0..
MX_DEVINL void mix_dpre_store(const float* src_s, int lds, const MixerArgs& a, int blk, int e0, int E, int TE) {
  const int nc4 = mx_round_up(a.wl.rows[blk], 4) >> 2;
  for (int idx = threadIdx.x; idx < TE * nc4; idx += MX_TILE_THREADS) {
    const int r = idx / nc4, c4 = idx - r * nc4;
    if (e0 + r < E) mx_st4(a.d_pre + (size_t)(e0 + r) * a.wl.Cp + a.wl.col[blk] + 4 * c4, mx_ld4(src_s + r * lds + 4 * c4));
  }
}

// blockIdx.y = 0: live net on s[t]; 1: target net on s[t+1] (qmix.py:155-157)
// WIDE: the state-reading layers come from the state-layer GEMM (mixer_wide.cu); only the second layers run here
template <int RM, bool WIDE>
__global__ void __launch_bounds__(MX_TILE_THREADS) k_mix_hyper_fwd(MixerArgs a, MixSmem sm) {
  constexpr int TE = 16 * RM;
  MX_DYN_SMEM(smem);
  const MxMixLayout L = a.L;
  const int E = a.B * a.T;
  const int ntiles = (E + TE - 1) / TE;
  const int net = blockIdx.y;
  const float* th = net ? a.theta_tgt : a.theta;
  float* s_s = smem + sm.o_s;
  float* h1_s = smem + sm.o_h1; float* h2_s = smem + sm.o_h2; float* hb_s = smem + sm.o_hb;
  float* p1_s = smem + sm.o_p1; float* b1_s = smem + sm.o_b1; float* p2_s = smem + sm.o_p2;
  const int S64 = mx_round_up(L.S, 64);
  MX_PDL_WAIT();
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int e0 = tile * TE;
    if constexpr (WIDE) {
      const int H64 = mx_round_up(L.HY, 64), P64 = mx_round_up(L.N * L.ME, 64), M64 = mx_round_up(L.ME, 64);
      if (L.layers == 2) {
        mix_pre_load(h1_s, sm.ldH, H64, a, net, 0, true, e0, E, TE);
        mix_pre_load(h2_s, sm.ldH, H64, a, net, 1, true, e0, E, TE);
      } else {
        mix_pre_load(p1_s, sm.ldP, P64, a, net, 0, false, e0, E, TE);
        mix_pre_load(p2_s, sm.ldM, M64, a, net, 1, false, e0, E, TE);
      }
      mix_pre_load(hb_s, sm.ldH, H64, a, net, 2, true, e0, E, TE);
      mix_pre_load(b1_s, sm.ldM, M64, a, net, 3, false, e0, E, TE);
      __syncthreads();
      if (L.layers == 2) {
        float* Wc = smem + sm.o_wc;
        tile_linear<RM>(h1_s, sm.ldH, L.HY, th + L.w1b, th + L.b1b, L.N * L.ME, p1_s, sm.ldP, false, Wc, sm.ldw);
        tile_linear<RM>(h2_s, sm.ldH, L.HY, th + L.w2b, th + L.b2b, L.ME, p2_s, sm.ldM, false, Wc, sm.ldw);
      }
    } else {
      mix_stage_states(a, sm, s_s, e0, E, TE, S64, net);
      mx_cp_commit();
      mx_cp_wait<0>();
      __syncthreads();
      mixer_hyper<RM>(th, L, sm, smem);
    }
    // b2 = hb . Wb2b + bb2b   (one half-warp per element)
    {
      const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
      for (int i = 0; i < RM; ++i) {
        const int r = ty * RM + i;
        float v = 0.f;
        for (int k = tx; k < L.HY; k += 16) v = fmaf(hb_s[r * sm.ldH + k], th[L.wb2b + k], v);
        v = mx_row16_sum(v);
        if (tx == 0 && e0 + r < E) a.hyp_b2[net][e0 + r] = v + th[L.bb2b];
      }
    }
    mix_tile_store(p1_s, sm.ldP, a.hyp_p1[net], a.gP, e0, E, TE);
    mix_tile_store(b1_s, sm.ldM, a.hyp_b1[net], a.gM, e0, E, TE);
    mix_tile_store(p2_s, sm.ldM, a.hyp_p2[net], a.gM, e0, E, TE);
    if (net == 0) {     // kept for the backward pass
      if (L.layers == 2) {
        mix_tile_store(h1_s, sm.ldH, a.hyp_h1, a.gH, e0, E, TE);
        mix_tile_store(h2_s, sm.ldH, a.hyp_h2, a.gH, e0, E, TE);
      }
      mix_tile_store(hb_s, sm.ldH, a.hyp_hb, a.gH, e0, E, TE);
    }
    __syncthreads();
  }
}

// One warp per (b,t) element, lanes over the mixer's hidden units: Q_tot' (target), Q_tot (live), TD target, masked loss,
// dL/dQ_tot and the elementwise part of the live mixer's backward (q_mixer.py:82-93, qmix.py:159-187).
#define MX_MIX_MAXK 2      // mixer_hidden <= 64
__global__ void __launch_bounds__(512) k_mix_core(MixerArgs a) {
  const MxMixLayout L = a.L;
  const int E = a.B * a.T, N = L.N, ME = L.ME;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  float den = 0.f, lsum = 0.f, qsum = 0.f;
  MX_PDL_WAIT();
  for (int e = blockIdx.x * nw + warp; e < E; e += gridDim.x * nw) {
    float Qv[2];
    float hp[MX_MIX_MAXK], hvv[MX_MIX_MAXK], p2v[MX_MIX_MAXK];
    // independent scalar loads first: their latency overlaps the two mixing passes
    const int b = e / a.T, t = e % a.T;
    const float rew = a.rewards[(size_t)b * a.ld_tn + (size_t)t * N];              // agent 0 (qmix.py:159)
    const float de = a.dones_env[(size_t)b * a.ld_t + t];
    const float bad = t > 0 ? a.dones_env[(size_t)b * a.ld_t + t - 1] : 0.f;     // qmix.py:161
    const float w = a.weights ? a.weights[b] : 1.f;
    const float b2v[2] = {a.hyp_b2[0][e], a.hyp_b2[1][e]};
#pragma unroll
    for (int net = 1; net >= 0; --net) {
      const float* q = (net ? a.q_next : a.q_taken) + (size_t)e * N;
      const float* p1 = a.hyp_p1[net] + (size_t)e * a.gP;
      float part = 0.f;
#pragma unroll
      for (int j = 0; j < MX_MIX_MAXK; ++j) {
        const int k = lane + 32 * j;
        if (k < ME) {
          float v = a.hyp_b1[net][(size_t)e * a.gM + k];
          for (int n = 0; n < N; ++n) v = fmaf(q[n], fabsf(p1[n * ME + k]), v);
          const float hv = v > 0.f ? v : (expf(v) - 1.f);
          const float p2 = a.hyp_p2[net][(size_t)e * a.gM + k];
          part = fmaf(hv, fabsf(p2), part);
          if (net == 0) { hp[j] = v; hvv[j] = hv; p2v[j] = p2; }
        }
      }
      Qv[net] = mx_warp_sum(part) + b2v[net];
    }
    const float y = rew + (1.f - de) * a.gamma * Qv[1];
    const float keep = 1.f - bad;
    const float err = (Qv[0] - y) * keep;
    float le, dle;
    if (a.use_huber) {
      const float ae = fabsf(err);
      if (ae <= a.huber_delta) { le = 0.5f * err * err; dle = err; }
      else { le = a.huber_delta * (ae - 0.5f * a.huber_delta); dle = err > 0.f ? a.huber_delta : -a.huber_delta; }
    } else { le = err * err; dle = 2.f * err; }
    const float dq = dle * keep * w;
    if (lane == 0) {
      a.qtot[e] = Qv[0]; a.qtot_next[e] = Qv[1]; a.err[e] = err; a.d_q[e] = dq;
      den += keep; lsum += le * w; qsum += Qv[0] * keep;
    }
    // elementwise backward: d hid_pre, d p2 ; then d q_taken and d p1
    float dhp[MX_MIX_MAXK];
#pragma unroll
    for (int j = 0; j < MX_MIX_MAXK; ++j) {
      const int k = lane + 32 * j;
      dhp[j] = 0.f;
      if (k < ME) {
        const float dhid = dq * fabsf(p2v[j]);
        dhp[j] = dhid * (hp[j] > 0.f ? 1.f : (hvv[j] + 1.f));                      // ELU'(x) = exp(x) for x <= 0
        a.d_hp[(size_t)e * a.gM + k] = dhp[j];
        a.d_p2[(size_t)e * a.gM + k] = dq * hvv[j] * (p2v[j] > 0.f ? 1.f : (p2v[j] < 0.f ? -1.f : 0.f));   // d|x| = sign(x)
      }
    }
    const float* p1 = a.hyp_p1[0] + (size_t)e * a.gP;
    const float* q = a.q_taken + (size_t)e * N;
    for (int n = 0; n < N; ++n) {
      float acc = 0.f;
      const float qn = q[n];
#pragma unroll
      for (int j = 0; j < MX_MIX_MAXK; ++j) {
        const int k = lane + 32 * j;
        if (k < ME) {
          const float pv = p1[n * ME + k];
          acc = fmaf(fabsf(pv), dhp[j], acc);
          a.d_p1[(size_t)e * a.gP + n * ME + k] = qn * dhp[j] * (pv > 0.f ? 1.f : (pv < 0.f ? -1.f : 0.f));
        }
      }
      acc = mx_warp_sum(acc);
      if (lane == 0) a.dq_taken[(size_t)e * N + n] = acc;
    }
  }
  __shared__ float red[3][16];
  if (lane == 0) { red[0][warp] = den; red[1][warp] = lsum; red[2][warp] = qsum; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float s0 = 0.f, s1 = 0.f, s2 = 0.f;
    for (int i = 0; i < nw; ++i) { s0 += red[0][i]; s1 += red[1][i]; s2 += red[2][i]; }
    float* sp = a.spart + (size_t)blockIdx.x * 8;
    sp[0] = s0; sp[1] = s1; sp[2] = s2;
  }
}

// parameter gradients of the live hypernetworks from core's d p1 / d p2 / d hid_pre / dQ (per-CTA partials like k_mixer)
// WIDE: the state layers' weight gradients are left to the state-layer GEMM; this kernel writes the gradient at their pre-activations
template <int RM, bool WIDE>
__global__ void __launch_bounds__(MX_TILE_THREADS) k_mix_hyper_bwd(MixerArgs a, MixSmem sm) {
  constexpr int TE = 16 * RM;
  MX_DYN_SMEM(smem);
  const MxMixLayout L = a.L;
  const int tid = threadIdx.x;
  const int E = a.B * a.T;
  const int ntiles = (E + TE - 1) / TE;
  float* s_s = smem + sm.o_s;
  float* h1_s = smem + sm.o_h1; float* h2_s = smem + sm.o_h2; float* hb_s = smem + sm.o_hb;
  float* p1_s = smem + sm.o_p1; float* p2_s = smem + sm.o_p2; float* hid_s = smem + sm.o_hid;
  float* Wc = smem + sm.o_wc;
  float* dQ_s = smem + sm.o_vec;          // [TE]
  float* gp = a.gpart + (size_t)blockIdx.x * a.P;
  const int S64 = mx_round_up(L.S, 64), H64 = mx_round_up(L.HY, 64), P64 = mx_round_up(L.N * L.ME, 64), M64 = mx_round_up(L.ME, 64);
  const int NM = L.N * L.ME;
  int iter = 0;
  MX_PDL_WAIT();
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++iter) {
    const int e0 = tile * TE;
    const bool accum = iter > 0;
    if constexpr (!WIDE) mix_stage_states(a, sm, s_s, e0, E, TE, S64, 0);
    if (L.layers == 2) {
      mix_tile_load(h1_s, sm.ldH, H64, a.hyp_h1, a.gH, e0, E, TE);
      mix_tile_load(h2_s, sm.ldH, H64, a.hyp_h2, a.gH, e0, E, TE);
    }
    mix_tile_load(hb_s, sm.ldH, H64, a.hyp_hb, a.gH, e0, E, TE);
    mix_tile_load(p1_s, sm.ldP, P64, a.d_p1, a.gP, e0, E, TE);
    mix_tile_load(p2_s, sm.ldM, M64, a.d_p2, a.gM, e0, E, TE);
    mix_tile_load(hid_s, sm.ldM, M64, a.d_hp, a.gM, e0, E, TE);
    mx_cp_commit();
    if (tid < TE) dQ_s[tid] = (e0 + tid < E) ? a.d_q[e0 + tid] : 0.f;
    mx_cp_wait<0>();
    __syncthreads();
    // -- b2 path: d Wb2b, d bb2b, then hb_s <- d(pre-ReLU hb)
    for (int k = tid; k < L.HY; k += MX_TILE_THREADS) {
      float s = 0.f;
      for (int r = 0; r < TE; ++r) s = fmaf(dQ_s[r], hb_s[r * sm.ldH + k], s);
      float* p = gp + L.wb2b + k;
      *p = accum ? (*p + s) : s;
    }
    if (tid == 0) {
      float s = 0.f;
      for (int r = 0; r < TE; ++r) s += dQ_s[r];
      float* p = gp + L.bb2b;
      *p = accum ? (*p + s) : s;
    }
    __syncthreads();
    for (int idx = tid; idx < TE * sm.ldH; idx += MX_TILE_THREADS) {
      const int r = idx / sm.ldH, k = idx % sm.ldH;
      float v = 0.f;
      if (k < L.HY && hb_s[idx] > 0.f) v = dQ_s[r] * a.theta[L.wb2b + k];
      hb_s[idx] = v;
    }
    __syncthreads();
    if constexpr (WIDE) {
      mix_dpre_store(hb_s, sm.ldH, a, 2, e0, E, TE);
      mix_dpre_store(hid_s, sm.ldM, a, 3, e0, E, TE);
      if (L.layers == 2) {
        tile_wgrad(p2_s, sm.ldM, L.ME, h2_s, sm.ldH, L.HY, TE, gp + L.w2b, gp + L.b2b, accum);
        __syncthreads();
        tile_dgrad_relu<RM>(p2_s, sm.ldM, L.ME, a.theta + L.w2b, L.HY, h2_s, h2_s, sm.ldH, Wc, sm.ldw);
        mix_dpre_store(h2_s, sm.ldH, a, 1, e0, E, TE);
        tile_wgrad(p1_s, sm.ldP, NM, h1_s, sm.ldH, L.HY, TE, gp + L.w1b, gp + L.b1b, accum);
        __syncthreads();
        tile_dgrad_relu<RM>(p1_s, sm.ldP, NM, a.theta + L.w1b, L.HY, h1_s, h1_s, sm.ldH, Wc, sm.ldw);
        mix_dpre_store(h1_s, sm.ldH, a, 0, e0, E, TE);
      } else {
        mix_dpre_store(p2_s, sm.ldM, a, 1, e0, E, TE);
        mix_dpre_store(p1_s, sm.ldP, a, 0, e0, E, TE);
      }
      __syncthreads();
      continue;
    }
    // -- hyper_b2 first layer, hyper_b1
    tile_wgrad(hb_s, sm.ldH, L.HY, s_s, sm.ldS, L.S, TE, gp + L.wb2a, gp + L.bb2a, accum);
    tile_wgrad(hid_s, sm.ldM, L.ME, s_s, sm.ldS, L.S, TE, gp + L.wb1, gp + L.bb1, accum);
    if (L.layers == 2) {
      // -- hyper_w2
      tile_wgrad(p2_s, sm.ldM, L.ME, h2_s, sm.ldH, L.HY, TE, gp + L.w2b, gp + L.b2b, accum);
      __syncthreads();
      tile_dgrad_relu<RM>(p2_s, sm.ldM, L.ME, a.theta + L.w2b, L.HY, h2_s, h2_s, sm.ldH, Wc, sm.ldw);
      tile_wgrad(h2_s, sm.ldH, L.HY, s_s, sm.ldS, L.S, TE, gp + L.w2a, gp + L.b2a, accum);
      // -- hyper_w1
      tile_wgrad(p1_s, sm.ldP, NM, h1_s, sm.ldH, L.HY, TE, gp + L.w1b, gp + L.b1b, accum);
      __syncthreads();
      tile_dgrad_relu<RM>(p1_s, sm.ldP, NM, a.theta + L.w1b, L.HY, h1_s, h1_s, sm.ldH, Wc, sm.ldw);
      tile_wgrad(h1_s, sm.ldH, L.HY, s_s, sm.ldS, L.S, TE, gp + L.w1a, gp + L.b1a, accum);
    } else {
      tile_wgrad(p2_s, sm.ldM, L.ME, s_s, sm.ldS, L.S, TE, gp + L.w2b, gp + L.b2b, accum);
      tile_wgrad(p1_s, sm.ldP, NM, s_s, sm.ldS, L.S, TE, gp + L.w1b, gp + L.b1b, accum);
    }
    __syncthreads();
  }
}

int mx_launch_mixer(const MixerArgs& a, int* nparts_used, cudaStream_t s) {
  const int E = a.B * a.T;
  const int sms = mx_num_sms();
  if (a.vdn) {
    int grid = mx_ceil_div(E, 256);
    if (grid > sms) grid = sms;
    *nparts_used = grid;
    return mx_launch("k_vdn_mix", k_vdn_mix, dim3(grid), dim3(256), 0, s, MX_STEP, a);
  }
  if (a.L.N > 32) { mx_set_error("mixer: n_agents > 32 unsupported"); return 1; }
  const int RM = (E > 16 * sms) ? 2 : 1;
  const int TE = 16 * RM;
  MixSmem sm = mix_smem_layout(a.L, TE);
  const size_t smem = (size_t)sm.total * sizeof(float) + 16;
  int grid = mx_ceil_div(E, TE);
  if (grid > sms) grid = sms;
#if !MX_EMU
  if (smem > MX_SMEM_OPTIN_MAX) { mx_set_error("mixer: %zu bytes of shared memory needed (state_dim / n_agents too large)", smem); return 1; }
#endif
  *nparts_used = grid;
  return mx_launch("k_mixer", RM == 1 ? k_mixer<1> : k_mixer<2>, dim3(grid), dim3(MX_TILE_THREADS), smem, s, MX_STEP, a, sm);
}

int mx_mixer_split_supported(const MxMixLayout& L) { return L.ME <= 32 * MX_MIX_MAXK && L.N <= 32; }

static int mix_split_rm(int E) {
  return (E > 16 * mx_num_sms()) ? 2 : 1;
}

int mx_launch_mix_hyper_fwd(const MixerArgs& a, cudaStream_t s) {
  const int E = a.B * a.T;
  const int RM = mix_split_rm(E), TE = 16 * RM;
  MixSmem sm = mix_smem_layout(a.L, TE, a.wide != 0);
  const size_t smem = (size_t)sm.total * sizeof(float) + 16;
  int grid = mx_ceil_div(E, TE);
  if (grid > mx_num_sms()) grid = mx_num_sms();
  if (a.wide && mx_launch_mixw_state_fwd(a, s)) return 1;
  auto kern = a.wide ? (RM == 1 ? k_mix_hyper_fwd<1, true> : k_mix_hyper_fwd<2, true>)
                     : (RM == 1 ? k_mix_hyper_fwd<1, false> : k_mix_hyper_fwd<2, false>);
  return mx_launch(a.wide ? "k_mix_hyper_fwd_wide" : "k_mix_hyper_fwd", kern, dim3(grid, 2), dim3(MX_TILE_THREADS), smem, s, MX_STEP, a, sm);
}

int mx_launch_mix_core(const MixerArgs& a, int* scalar_parts_used, cudaStream_t s) {
  const int E = a.B * a.T;
  int grid = mx_ceil_div(E, 16);                  // one warp per element, 16 warps per CTA: 3m (1 920 elements) = 120 CTAs, one pass
  if (grid > mx_num_sms()) grid = mx_num_sms();   // (spart holds one scalar partial per SM)
  *scalar_parts_used = grid;
  return mx_launch("k_mix_core", k_mix_core, dim3(grid), dim3(512), 0, s, MX_STEP, a);
}

int mx_launch_mix_hyper_bwd(const MixerArgs& a, int* nparts_used, cudaStream_t s) {
  const int E = a.B * a.T;
  const int RM = mix_split_rm(E), TE = 16 * RM;
  MixSmem sm = mix_smem_layout(a.L, TE, a.wide != 0);
  const size_t smem = (size_t)sm.total * sizeof(float) + 16;
  int grid = mx_ceil_div(E, TE);
  if (grid > mx_num_sms()) grid = mx_num_sms();
  auto kern = a.wide ? (RM == 1 ? k_mix_hyper_bwd<1, true> : k_mix_hyper_bwd<2, true>)
                     : (RM == 1 ? k_mix_hyper_bwd<1, false> : k_mix_hyper_bwd<2, false>);
  *nparts_used = grid;
  if (const int rc = mx_launch(a.wide ? "k_mix_hyper_bwd_wide" : "k_mix_hyper_bwd", kern, dim3(grid), dim3(MX_TILE_THREADS), smem, s, MX_STEP, a, sm))
    return rc;
  return a.wide ? mx_launch_mixw_state_wgrad(a, s) : 0;
}
