// The middle of the QMIX step in ONE kernel: Q head (live rows t and t+1, target rows t+1) -> taken / greedy / bootstrap Q values
// -> mixer core (Q_tot', Q_tot, TD target, masked loss, dQ_tot, elementwise mixer backward) -> Q head backward (post-GRU LayerNorm
// backward -> dL/dh_t, head + LayerNorm parameter gradients).  It replaces the three latency-bound launches k_qhead, k_mix_core and
// k_qhead_bwd that sit between the forward and the backward recurrence (same arithmetic, same references: QMixPolicy.py:69-93,
// qmix.py:138-187, q_mixer.py:82-93, act.py:19-32, rnn.py:21-23).
//
// One warp per (b, t) element: the N agents of an element are N consecutive rows m = (b (T+1) + t) N + n, so everything the
// element needs (q_taken[n], q_next[n], dq_taken[n]) stays in the warp's registers.  The head is evaluated with one lane per
// action (two half-dot-products per action when A <= 16; two actions per lane, k = lane and lane + 32, when 32 < A <= 64: the
// APL = 2 instantiation) on the LayerNorm output parked in a per-warp shared-memory row, so a
// 9-action head costs ~35 FMAs + 1 shuffle per lane instead of 9 five-step warp reductions.  The live head is evaluated twice per
// row (as "t" for the taken action, as "t+1" for the double-Q arg-max): 64 x A MACs, cheaper than a round trip through memory.
// Head-weight gradients accumulate in per-warp private shared-memory slices and are summed over the warps in fixed order
// (deterministic, no atomics).
#include "mx_internal.h"
#include "mx_kernels.h"

#define MID_WARPS_MAX 16      // 16 warps per CTA when the per-warp slices fit in shared memory, 8 otherwise (SMAC 8m: 8 agents x 14 actions)
// Head-weight row k lives at k * 66 with column j at j + (j >= 32): the two half-warps of the A <= 16 path (columns 0..31 and
// 32..63 of the same rows) then read banks 2k + j and 2k + 1 + j -- all 32 lanes conflict-free; the LayerNorm output row uses the
// same one-float gap, so its two broadcast reads per step also hit different banks.
#define MID_WLD 66
#define MID_YLD 66
MX_DEVINL int mid_col(int j) { return j + (j >> 5); }

struct MidSmem { int o_wq, o_bq, o_ln, o_y, o_dw, o_db, o_dg, o_stage, stage_ld, total; };
// APL: actions per lane (1: A <= 32, 2: A <= 64); the head, bias, availability and bias-gradient tiles have 32 * APL rows
static MidSmem mid_smem(int A, int N, int gP, int gM, int MID_WARPS, int APL) {
  MidSmem s;
  const int AR = 32 * APL;
  int o = 0;
  s.o_wq = o; o += 2 * AR * MID_WLD;            // [net][32 APL][65]
  s.o_bq = o; o += 2 * AR;
  s.o_ln = o; o += 4 * MX_H;                    // live gamma, beta, target gamma, beta
  s.o_y = o; o += MID_WARPS * MID_YLD;          // per-warp LayerNorm output row (gapped)
  s.o_dw = o; o += MID_WARPS * A * MX_H;        // per-warp private dWq
  s.o_db = o; o += MID_WARPS * AR;              // per-warp private dbq
  s.o_dg = o; o += 2 * MID_WARPS * MX_H;        // per-warp d gamma, d beta
  // per-warp operand staging (cp.async at the top of an element, ONE exposed L2 latency instead of one per agent and per mixer term):
  // h rows [live t | live t+1 | target t+1][N][64], mixer hypernet outputs p1[2][gP], b1[2][gM], p2[2][gM], availability [N][32 APL]
  s.stage_ld = (3 * N * MX_H + 2 * gP + 4 * gM + N * AR + 3) & ~3;
  s.o_stage = o; o += MID_WARPS * s.stage_ld;
  s.total = o;
  return s;
}

// LayerNorm of one row held as (v0 = h[lane], v1 = h[lane + 32]) -> normalised xh and y = xh * g + b
MX_DEVINL void mid_ln(float v0, float v1, const float* g, const float* b, int lane, float& xh0, float& xh1, float& y0, float& y1, float& rstd) {
  const float mean = mx_warp_sum(v0 + v1) * (1.f / MX_H);
  const float d0 = v0 - mean, d1 = v1 - mean;
  rstd = rsqrtf(mx_warp_sum(d0 * d0 + d1 * d1) * (1.f / MX_H) + MX_LN_EPS);
  xh0 = d0 * rstd; xh1 = d1 * rstd;
  y0 = xh0 * g[lane] + b[lane]; y1 = xh1 * g[lane + 32] + b[lane + 32];
}

// q_k for k = lane (A > 16) or k = lane & 15 (A <= 16, both half-warps end with the full value); lanes with k >= A return 0
MX_DEVINL float mid_head(const float* ys, const float* wq, const float* bq, int A, int lane) {
  float q;
  if (A <= 16) {
    const int k = lane & 15, j0 = (lane >> 4) * 33;         // second half starts one float later (mid_col)
    const float* w = wq + (k < A ? k : 0) * MID_WLD + j0;
    float s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int j = 0; j < 32; j += 2) { s0 = fmaf(ys[j0 + j], w[j], s0); s1 = fmaf(ys[j0 + j + 1], w[j + 1], s1); }
    q = s0 + s1;
    q += __shfl_xor_sync(0xffffffffu, q, 16);
    q = k < A ? q + bq[k] : 0.f;
  } else {
    const int k = lane;
    const float* w = wq + (k < A ? k : 0) * MID_WLD;
    float s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int j = 0; j < MX_H; j += 2) { s0 = fmaf(ys[mid_col(j)], w[mid_col(j)], s0); s1 = fmaf(ys[mid_col(j + 1)], w[mid_col(j + 1)], s1); }
    q = k < A ? (s0 + s1) + bq[k] : 0.f;
  }
  return q;
}

// 32 < A <= 64: q_k for k = lane (qa) and k = lane + 32 (qb, 0 when k >= A), same summation order as the one-action path
MX_DEVINL void mid_head2(const float* ys, const float* wq, const float* bq, int A, int lane, float& qa, float& qb) {
  const int kb = lane + 32;
  const float* wa = wq + lane * MID_WLD;
  const float* wb = wq + (kb < A ? kb : 0) * MID_WLD;
  float s0 = 0.f, s1 = 0.f, t0 = 0.f, t1 = 0.f;
#pragma unroll
  for (int j = 0; j < MX_H; j += 2) {
    const float y0 = ys[mid_col(j)], y1 = ys[mid_col(j + 1)];
    s0 = fmaf(y0, wa[mid_col(j)], s0); s1 = fmaf(y1, wa[mid_col(j + 1)], s1);
    t0 = fmaf(y0, wb[mid_col(j)], t0); t1 = fmaf(y1, wb[mid_col(j + 1)], t1);
  }
  qa = (s0 + s1) + bq[lane];
  qb = kb < A ? (t0 + t1) + bq[kb] : 0.f;
}

// the value of action k, held by lane k & 31 as lo (k < 32) or hi (k >= 32); every lane returns it
template <int APL>
MX_DEVINL float mid_pick(float lo, float hi, int k) {
  if constexpr (APL == 1) return __shfl_sync(0xffffffffu, lo, k);
  else return __shfl_sync(0xffffffffu, k < 32 ? lo : hi, k & 31);
}

// arg-max with "first maximum wins" over lanes k < A (value v in lane k); every lane returns the winner
MX_DEVINL void mid_argmax(float v, int A, int lane, float& best, int& idx) {
  float bv = lane < A ? v : -3.0e38f;
  int bi = lane < A ? lane : 1 << 20;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
  }
  best = bv; idx = bi;
}

// the same over 32 < A <= 64 actions, va for k = lane and vb for k = lane + 32: the lane keeps its lower action on a tie, then the
// warp reduction prefers the lower index, so the first maximum still wins
MX_DEVINL void mid_argmax2(float va, float vb, int A, int lane, float& best, int& idx) {
  float bv = va;
  int bi = lane;
  if (lane + 32 < A && vb > bv) { bv = vb; bi = lane + 32; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
  }
  best = bv; idx = bi;
}

template <int MID_WARPS, int APL>
__global__ void __launch_bounds__(32 * MID_WARPS) k_mid(MidArgs a, MidSmem sm) {
  constexpr int MID_THREADS = 32 * MID_WARPS;
  constexpr int AR = 32 * APL;                       // rows of the head / bias / availability tiles
  MX_DYN_SMEM(smem);
  const MxMixLayout L = a.mix.L;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int A = a.A, N = a.N, T = a.T, T1 = a.T + 1, ME = L.ME;
  const int E = a.mix.B * T;
  float* wq_s = smem + sm.o_wq; float* bq_s = smem + sm.o_bq; float* ln_s = smem + sm.o_ln;
  float* ys = smem + sm.o_y + warp * MID_YLD;
  float* my_dw = smem + sm.o_dw + warp * A * MX_H;
  float* my_db = smem + sm.o_db + warp * AR;
  float* stg = smem + sm.o_stage + warp * sm.stage_ld;
  for (int net = 0; net < 2; ++net) {
    const float* th = net ? a.mix.theta_tgt : a.mix.theta;
    for (int i = tid; i < A * MX_H; i += MID_THREADS) wq_s[net * AR * MID_WLD + (i / MX_H) * MID_WLD + mid_col(i % MX_H)] = th[a.wq + i];
    for (int i = tid; i < AR; i += MID_THREADS) bq_s[net * AR + i] = i < A ? th[a.bq + i] : 0.f;
    for (int i = tid; i < MX_H; i += MID_THREADS) { ln_s[net * 2 * MX_H + i] = th[a.lno_g + i]; ln_s[net * 2 * MX_H + MX_H + i] = th[a.lno_b + i]; }
  }
  for (int i = tid; i < MID_WARPS * A * MX_H; i += MID_THREADS) smem[sm.o_dw + i] = 0.f;
  for (int i = tid; i < MID_WARPS * AR; i += MID_THREADS) smem[sm.o_db + i] = 0.f;
  MX_PDL_WAIT();
  __syncthreads();
  const float* lg = ln_s; const float* lb = ln_s + MX_H; const float* tg = ln_s + 2 * MX_H; const float* tb = ln_s + 3 * MX_H;
  const float* wq0 = wq_s; const float* wq1 = wq_s + AR * MID_WLD;
  float den = 0.f, lsum = 0.f, qsum = 0.f;           // lane 0
  float dg0 = 0.f, dg1 = 0.f, db0 = 0.f, db1 = 0.f;   // LayerNorm gamma / beta gradients of this warp's rows

  for (int e = blockIdx.x * MID_WARPS + warp; e < E; e += gridDim.x * MID_WARPS) {
    const int b = e / T, t = e - b * T;
    const size_t m0 = ((size_t)b * T1 + t) * N;          // rows of step t;  rows of step t+1 start at m0 + N
    // independent scalar loads first
    const float rew = a.mix.rewards[(size_t)b * a.mix.ld_tn + (size_t)t * N];
    const float de = a.mix.dones_env[(size_t)b * a.mix.ld_t + t];
    const float bad = t > 0 ? a.mix.dones_env[(size_t)b * a.mix.ld_t + t - 1] : 0.f;
    const float w = a.mix.weights ? a.mix.weights[b] : 1.f;
    const float b2v[2] = {a.mix.hyp_b2[0][e], a.mix.hyp_b2[1][e]};
    float qt_reg = 0.f, qn_reg = 0.f;                     // lane n: q_taken[n], q_next[n]
    // ---- stage every operand of this element with asynchronous copies: all of them are in flight at once ----
    float* st_h = stg;                                    // [3][N][64]: live t, live t+1, target t+1
    float* st_p1 = st_h + 3 * N * MX_H;                   // [2][gP]
    float* st_b1 = st_p1 + 2 * a.mix.gP;                  // [2][gM]
    float* st_p2 = st_b1 + 2 * a.mix.gM;                  // [2][gM]
    float* st_av = st_p2 + 2 * a.mix.gM;                  // [N][32 APL]
    {
      const int hv = N * (MX_H / 4);                      // 16-byte pieces per block of N rows (rows of a step are contiguous)
      const float* s0 = a.hall[0] + m0 * MX_H;
      const float* s1 = a.hall[0] + (m0 + N) * MX_H;
      const float* s2 = a.hall[1] + (m0 + N) * MX_H;
      for (int i = lane; i < hv; i += 32) { mx_cp16(st_h + 4 * i, s0 + 4 * i); mx_cp16(st_h + N * MX_H + 4 * i, s1 + 4 * i); mx_cp16(st_h + 2 * N * MX_H + 4 * i, s2 + 4 * i); }
      for (int net = 0; net < 2; ++net) {
        const float* p1 = a.mix.hyp_p1[net] + (size_t)e * a.mix.gP;
        for (int i = lane; i < a.mix.gP / 4; i += 32) mx_cp16(st_p1 + net * a.mix.gP + 4 * i, p1 + 4 * i);
        const float* b1 = a.mix.hyp_b1[net] + (size_t)e * a.mix.gM;
        const float* p2 = a.mix.hyp_p2[net] + (size_t)e * a.mix.gM;
        for (int i = lane; i < a.mix.gM / 4; i += 32) { mx_cp16(st_b1 + net * a.mix.gM + 4 * i, b1 + 4 * i); mx_cp16(st_p2 + net * a.mix.gM + 4 * i, p2 + 4 * i); }
      }
      if (a.avail && lane < A)
        for (int n = 0; n < N; ++n) mx_cp4(st_av + n * AR + lane, a.avail + (m0 + N + n) * a.act_ld + lane);
      if (APL == 2 && a.avail && lane + 32 < A)
        for (int n = 0; n < N; ++n) mx_cp4(st_av + n * AR + lane + 32, a.avail + (m0 + N + n) * a.act_ld + lane + 32);
      mx_cp_commit();
    }
    const int act_l = lane < N ? a.act_idx[(size_t)b * a.ld_tn + (size_t)t * N + lane] : 0;       // lane n: taken action of agent n
    mx_cp_wait<0>();
    __syncwarp();
    // ---------------- Q head: taken-action Q (live, t), greedy action (live, t+1), bootstrap Q (target, t+1) ----------------
    for (int n = 0; n < N; ++n) {
      const float* hl = st_h + n * MX_H;
      const float* hl1 = st_h + (N + n) * MX_H;
      const float* ht1 = st_h + (2 * N + n) * MX_H;
      const float h0a = hl[lane], h0b = hl[lane + 32], h1a = hl1[lane], h1b = hl1[lane + 32], g1a = ht1[lane], g1b = ht1[lane + 32];
      const int act = __shfl_sync(0xffffffffu, act_l, n);
      float av = 1.f, av2 = 1.f;                         // availability of actions lane and lane + 32
      if (a.avail && lane < A) av = st_av[n * AR + lane];
      if (APL == 2 && a.avail && lane + 32 < A) av2 = st_av[n * AR + lane + 32];
      float xh0, xh1, y0, y1, rstd;
      // Q of actions lane (q) and lane + 32 (q_hi, APL = 2 only)
      auto head = [&](const float* wq, const float* bq, float& q, float& q_hi) {
        if constexpr (APL == 1) q = mid_head(ys, wq, bq, A, lane);
        else mid_head2(ys, wq, bq, A, lane, q, q_hi);
      };
      mid_ln(h0a, h0b, lg, lb, lane, xh0, xh1, y0, y1, rstd);
      ys[lane] = y0; ys[lane + 33] = y1;
      __syncwarp();
      float q_t, q_t_hi = 0.f;
      head(wq0, bq_s, q_t, q_t_hi);
      const float q_taken = mid_pick<APL>(q_t, q_t_hi, act);
      __syncwarp();
      mid_ln(h1a, h1b, lg, lb, lane, xh0, xh1, y0, y1, rstd);
      ys[lane] = y0; ys[lane + 33] = y1;
      __syncwarp();
      float q_t1, q_t1_hi = 0.f;
      head(wq0, bq_s, q_t1, q_t1_hi);
      float gbest; int greedy;
      if constexpr (APL == 1) mid_argmax(av != 0.f ? q_t1 : -1e10f, A, lane, gbest, greedy);          // util.py:297-302, first maximum wins
      else mid_argmax2(av != 0.f ? q_t1 : -1e10f, av2 != 0.f ? q_t1_hi : -1e10f, A, lane, gbest, greedy);
      __syncwarp();
      mid_ln(g1a, g1b, tg, tb, lane, xh0, xh1, y0, y1, rstd);
      ys[lane] = y0; ys[lane + 33] = y1;
      __syncwarp();
      float tq, tq_hi = 0.f;
      head(wq1, bq_s + AR, tq, tq_hi);
      float q_next;
      if (a.double_q) q_next = mid_pick<APL>(tq, tq_hi, greedy);
      else if constexpr (APL == 1) { int dummy; mid_argmax(tq, A, lane, q_next, dummy); }              // plain max, no avail mask (qmix.py:144)
      else { int dummy; mid_argmax2(tq, tq_hi, A, lane, q_next, dummy); }
      __syncwarp();
      if (lane == n) { qt_reg = q_taken; qn_reg = q_next; }
    }
    // ---------------- mixer core (same arithmetic as k_mix_core) ----------------
    float Qv[2];
    float hp[2], hvv[2], p2v[2];
#pragma unroll
    for (int net = 1; net >= 0; --net) {
      const float* p1 = st_p1 + net * a.mix.gP;
      float part = 0.f;
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int k = lane + 32 * j;
        float v = k < ME ? st_b1[net * a.mix.gM + k] : 0.f;
        for (int n = 0; n < N; ++n) {
          const float qv = __shfl_sync(0xffffffffu, net ? qn_reg : qt_reg, n);
          if (k < ME) v = fmaf(qv, fabsf(p1[n * ME + k]), v);
        }
        if (k < ME) {
          const float hv = v > 0.f ? v : (expf(v) - 1.f);
          const float p2 = st_p2[net * a.mix.gM + k];
          part = fmaf(hv, fabsf(p2), part);
          if (net == 0) { hp[j] = v; hvv[j] = hv; p2v[j] = p2; }
        }
      }
      Qv[net] = mx_warp_sum(part) + b2v[net];
    }
    const float y = rew + (1.f - de) * a.mix.gamma * Qv[1];
    const float keep = 1.f - bad;
    const float err = (Qv[0] - y) * keep;
    float le, dle;
    if (a.mix.use_huber) {
      const float ae = fabsf(err);
      if (ae <= a.mix.huber_delta) { le = 0.5f * err * err; dle = err; }
      else { le = a.mix.huber_delta * (ae - 0.5f * a.mix.huber_delta); dle = err > 0.f ? a.mix.huber_delta : -a.mix.huber_delta; }
    } else { le = err * err; dle = 2.f * err; }
    const float dq = dle * keep * w;
    if (lane == 0) {
      a.mix.qtot[e] = Qv[0]; a.mix.qtot_next[e] = Qv[1]; a.mix.err[e] = err; a.mix.d_q[e] = dq;
      den += keep; lsum += le * w; qsum += Qv[0] * keep;
    }
    float dhp[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int k = lane + 32 * j;
      dhp[j] = 0.f;
      if (k < ME) {
        const float dhid = dq * fabsf(p2v[j]);
        dhp[j] = dhid * (hp[j] > 0.f ? 1.f : (hvv[j] + 1.f));
        a.mix.d_hp[(size_t)e * a.mix.gM + k] = dhp[j];
        a.mix.d_p2[(size_t)e * a.mix.gM + k] = dq * hvv[j] * (p2v[j] > 0.f ? 1.f : (p2v[j] < 0.f ? -1.f : 0.f));
      }
    }
    float dqt_reg = 0.f;                                   // lane n: d q_taken[n]
    {
      const float* p1 = st_p1;
      for (int n = 0; n < N; ++n) {
        const float qn = __shfl_sync(0xffffffffu, qt_reg, n);
        float acc = 0.f;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int k = lane + 32 * j;
          if (k < ME) {
            const float pv = p1[n * ME + k];
            acc = fmaf(fabsf(pv), dhp[j], acc);
            a.mix.d_p1[(size_t)e * a.mix.gP + n * ME + k] = qn * dhp[j] * (pv > 0.f ? 1.f : (pv < 0.f ? -1.f : 0.f));
          }
        }
        acc = mx_warp_sum(acc);
        if (lane == n) dqt_reg = acc;
      }
    }
    // ---------------- Q head backward for the rows of step t ----------------
    for (int n = 0; n < N; ++n) {
      const float dqv = __shfl_sync(0xffffffffu, dqt_reg, n);
      const int act = __shfl_sync(0xffffffffu, act_l, n);
      const float* hl = st_h + n * MX_H;
      float xh0, xh1, y0, y1, rstd;
      mid_ln(hl[lane], hl[lane + 32], lg, lb, lane, xh0, xh1, y0, y1, rstd);
      const float dy0 = dqv * wq0[act * MID_WLD + lane], dy1 = dqv * wq0[act * MID_WLD + lane + 33];
      my_dw[act * MX_H + lane] += dqv * y0;
      my_dw[act * MX_H + lane + 32] += dqv * y1;
      if (lane == 0) my_db[act] += dqv;
      dg0 += dy0 * xh0; dg1 += dy1 * xh1; db0 += dy0; db1 += dy1;
      const float dx0 = dy0 * lg[lane], dx1 = dy1 * lg[lane + 32];
      const float c1 = mx_warp_sum(dx0 + dx1) * (1.f / MX_H);
      const float c2 = mx_warp_sum(dx0 * xh0 + dx1 * xh1) * (1.f / MX_H);
      float* out = a.dh_out + (m0 + n) * MX_H;
      out[lane] = rstd * (dx0 - c1 - xh0 * c2);
      out[lane + 32] = rstd * (dx1 - c1 - xh1 * c2);
      if (t == T - 1) {                                     // Q at the bootstrap step only feeds the (detached) target
        float* oz = a.dh_out + (m0 + N + n) * MX_H;
        oz[lane] = 0.f; oz[lane + 32] = 0.f;
      }
    }
  }
  // ---------------- per-CTA partials: scalars, head + LayerNorm parameter gradients (warps added in fixed order) ----------------
  float* dgw = smem + sm.o_dg;
  dgw[warp * MX_H + lane] = dg0; dgw[warp * MX_H + lane + 32] = dg1;
  dgw[(MID_WARPS + warp) * MX_H + lane] = db0; dgw[(MID_WARPS + warp) * MX_H + lane + 32] = db1;
  __shared__ float red[3][MID_WARPS];
  if (lane == 0) { red[0][warp] = den; red[1][warp] = lsum; red[2][warp] = qsum; }
  __syncthreads();
  if (tid == 0) {
    float s0 = 0.f, s1 = 0.f, s2 = 0.f;
    for (int i = 0; i < MID_WARPS; ++i) { s0 += red[0][i]; s1 += red[1][i]; s2 += red[2][i]; }
    float* sp = a.mix.spart + (size_t)blockIdx.x * 8;
    sp[0] = s0; sp[1] = s1; sp[2] = s2;
  }
  float* gp = a.gpart + (size_t)blockIdx.x * a.P;
  const float* dw_all = smem + sm.o_dw;
  const float* db_all = smem + sm.o_db;
  for (int i = tid; i < A * MX_H; i += MID_THREADS) {
    float v = 0.f;
#pragma unroll
    for (int wv = 0; wv < MID_WARPS; ++wv) v += dw_all[wv * A * MX_H + i];
    gp[a.wq + i] = v;
  }
  for (int i = tid; i < A; i += MID_THREADS) {
    float v = 0.f;
#pragma unroll
    for (int wv = 0; wv < MID_WARPS; ++wv) v += db_all[wv * AR + i];
    gp[a.bq + i] = v;
  }
  for (int i = tid; i < MX_H; i += MID_THREADS) {
    float g = 0.f, bb = 0.f;
#pragma unroll
    for (int wv = 0; wv < MID_WARPS; ++wv) { g += dgw[wv * MX_H + i]; bb += dgw[(MID_WARPS + wv) * MX_H + i]; }
    gp[a.lno_g + i] = g; gp[a.lno_b + i] = bb;
  }
}

static int mid_apl(const MidArgs& a) { return a.A > 32 ? 2 : 1; }
static int mid_pick_warps(const MidArgs& a) {      // 0: does not fit even with 8 warps
  for (int w = MID_WARPS_MAX; w >= 8; w >>= 1) {
    const MidSmem sm = mid_smem(a.A, a.N, a.mix.gP, a.mix.gM, w, mid_apl(a));
    if ((size_t)sm.total * sizeof(float) + 16 <= 220 * 1024) return w;
  }
  return 0;
}
int mx_mid_supported(const MidArgs& a) {
  if (!(mx_mixer_split_supported(a.mix.L) && a.A <= 64 && a.N <= 32)) return 0;
  return mid_pick_warps(a) != 0;          // the per-warp operand staging must fit
}

int mx_launch_mid(const MidArgs& a, int* parts_used, cudaStream_t s) {
  const int w = mid_pick_warps(a), apl = a.A <= 32 ? 1 : 2;
  if (a.A > 64 || (w != 16 && w != 8)) {
    mx_set_error("mid: configuration does not fit (N %d, A %d)", a.N, a.A);
    return 1;
  }
  auto kern = w == 16 ? (apl == 1 ? k_mid<16, 1> : k_mid<16, 2>) : (apl == 1 ? k_mid<8, 1> : k_mid<8, 2>);
  int grid = mx_ceil_div(a.mix.B * a.T, w);
  if (grid > mx_num_sms()) grid = mx_num_sms();
  MidSmem sm = mid_smem(a.A, a.N, a.mix.gP, a.mix.gM, w, apl);
  *parts_used = grid;
  return mx_launch("k_mid", kern, dim3(grid), dim3(32 * w), (size_t)sm.total * sizeof(float) + 16, s, MX_STEP, a, sm);
}
