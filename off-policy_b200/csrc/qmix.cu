// Recurrent QMIX / VDN learner: parameter + workspace layout, the step's launch sequence, CUDA-graph capture.
// reference: offpolicy/algorithms/qmix/qmix.py (QMix), see include/marl_b200.h for the per-entry-point mapping.
#include <stdio.h>
#include <string.h>

#include <string>
#include <vector>

#include "mx_internal.h"
#include "mx_kernels.h"

extern int g_mx_front_tc;
bool mx_front_tc_usable(int in_dim, bool have_image);

// =====================================================================================================
// parameter layouts (names = the reference's state_dict keys, SURVEY.md App. E)
// =====================================================================================================
static int take(int& off, int n) { int o = off; off += mx_round_up(n, 4); return o; }

int mx_net_layout(int in_dim, int out_dim, int base, MxNetLayout* L) {
  const int H = MX_H;
  int o = base;
  L->in_dim = in_dim; L->out_dim = out_dim;
  L->fn_g = take(o, in_dim); L->fn_b = take(o, in_dim);
  L->w1 = take(o, H * in_dim); L->b1 = take(o, H); L->ln1_g = take(o, H); L->ln1_b = take(o, H);
  L->wh = take(o, H * H); L->bh = take(o, H); L->lnh_g = take(o, H); L->lnh_b = take(o, H);
  L->w2 = take(o, H * H); L->b2 = take(o, H); L->ln2_g = take(o, H); L->ln2_b = take(o, H);
  L->wih = take(o, 3 * H * H); L->whh = take(o, 3 * H * H); L->bih = take(o, 3 * H); L->bhh = take(o, 3 * H);
  L->lno_g = take(o, H); L->lno_b = take(o, H);
  L->wq = take(o, out_dim * H); L->bq = take(o, out_dim);
  L->size = o - base;
  return 0;
}

int mx_mix_layout(int S, int N, int ME, int HY, int layers, int base, MxMixLayout* L) {
  int o = base;
  L->S = S; L->N = N; L->ME = ME; L->HY = HY; L->layers = layers;
  if (layers == 2) {
    L->w1a = take(o, HY * S); L->b1a = take(o, HY); L->w1b = take(o, N * ME * HY); L->b1b = take(o, N * ME);
    L->w2a = take(o, HY * S); L->b2a = take(o, HY); L->w2b = take(o, ME * HY); L->b2b = take(o, ME);
  } else {
    L->w1a = L->b1a = L->w2a = L->b2a = -1;
    L->w1b = take(o, N * ME * S); L->b1b = take(o, N * ME);
    L->w2b = take(o, ME * S); L->b2b = take(o, ME);
  }
  L->wb1 = take(o, ME * S); L->bb1 = take(o, ME);
  L->wb2a = take(o, HY * S); L->bb2a = take(o, HY); L->wb2b = take(o, HY); L->bb2b = take(o, 1);
  L->size = o - base;
  return 0;
}

static int check_cfg(const mx_qmix_cfg* c) {
  if (!c) { mx_set_error("null cfg"); return 1; }
  if (c->hidden != MX_H) { mx_set_error("hidden_size %d unsupported: kernels are specialised for %d", c->hidden, MX_H); return 1; }
  if (c->n_agents <= 0 || c->obs_dim <= 0 || c->act_dim <= 0 || c->state_dim <= 0 || c->episode_len <= 0 || c->max_batch <= 0) {
    mx_set_error("mx_qmix: non-positive dimension"); return 1;
  }
  if (c->act_dim > 64 || c->n_agents > 32) { mx_set_error("mx_qmix: act_dim must be <= 64 and n_agents <= 32"); return 1; }
  if (!c->vdn && c->hyper_layers != 1 && c->hyper_layers != 2) { mx_set_error("hypernet_layers must be 1 or 2"); return 1; }
  if (c->mlp && c->episode_len != 1) { mx_set_error("mx_qmix: the MLP (transition-level) variant stores transitions as episodes of length 1"); return 1; }
  if (c->mlp && c->prev_act_inp) { mx_set_error("mx_qmix: prev_act_inp is a recurrent-policy option"); return 1; }
  {     // the recurrent step runs k_gru_wgrad beside k_front_bwd above 128 input columns; the MLP variant has no GRU
    const int in_dim = c->obs_dim + (c->prev_act_inp ? c->act_dim : 0), lim = mx_front_bwd_max_in_dim(!c->mlp);
    if (in_dim > lim) {
      mx_set_error("mx_qmix: agent input width %d (obs_dim %d%s) exceeds %d, the widest k_front_bwd's shared memory holds", in_dim, c->obs_dim,
                   c->prev_act_inp ? " + act_dim with prev_act_inp" : "", lim);
      return 1;
    }
  }
  return 0;
}

static inline int agent_in_dim(const mx_qmix_cfg* c) { return c->obs_dim + (c->prev_act_inp ? c->act_dim : 0); }

static void layouts(const mx_qmix_cfg* c, MxNetLayout* A, MxMixLayout* M, int64_t* P) {
  mx_net_layout(agent_in_dim(c), c->act_dim, 0, A);
  memset(M, 0, sizeof(*M));
  M->size = 0;
  if (!c->vdn) mx_mix_layout(c->state_dim, c->n_agents, c->mixer_hidden, c->hyper_hidden, c->hyper_layers, A->size, M);
  *P = (int64_t)A->size + M->size;
}

extern "C" int mx_qmix_param_layout(const mx_qmix_cfg* c, mx_param_entry* out, int32_t max_entries, int64_t* total_floats) {
  if (check_cfg(c)) return -1;
  MxNetLayout A; MxMixLayout M; int64_t P;
  layouts(c, &A, &M, &P);
  std::vector<mx_param_entry> v;
  auto add = [&](const char* name, int off, int rows, int cols) {
    mx_param_entry e;
    memset(&e, 0, sizeof(e));
    snprintf(e.name, MX_MAX_NAME, "%s", name);
    e.offset = off; e.rows = rows; e.cols = cols;
    v.push_back(e);
  };
  const int H = MX_H, I = agent_in_dim(c), Aq = c->act_dim;
  if (c->mlp) {     // M_QMixPolicy.q_network = AgentQFunction(MLPBase + ACTLayer) (mqmix/algorithm/agent_q_function.py): reference key names;
                    // the head lives in the first act_dim rows of the weight_ih slot, the remaining recurrent slots stay zero
    if (!c->no_feature_norm) { add("agent.mlp.feature_norm.weight", A.fn_g, I, 0); add("agent.mlp.feature_norm.bias", A.fn_b, I, 0); }
    add("agent.mlp.mlp.fc1.0.weight", A.w1, H, I); add("agent.mlp.mlp.fc1.0.bias", A.b1, H, 0);
    add("agent.mlp.mlp.fc1.2.weight", A.ln1_g, H, 0); add("agent.mlp.mlp.fc1.2.bias", A.ln1_b, H, 0);
    add("agent.mlp.mlp.fc_h.0.weight", A.wh, H, H); add("agent.mlp.mlp.fc_h.0.bias", A.bh, H, 0);
    add("agent.mlp.mlp.fc_h.2.weight", A.lnh_g, H, 0); add("agent.mlp.mlp.fc_h.2.bias", A.lnh_b, H, 0);
    add("agent.mlp.mlp.fc2.0.0.weight", A.w2, H, H); add("agent.mlp.mlp.fc2.0.0.bias", A.b2, H, 0);
    add("agent.mlp.mlp.fc2.0.2.weight", A.ln2_g, H, 0); add("agent.mlp.mlp.fc2.0.2.bias", A.ln2_b, H, 0);
    add("agent.q.action_out.weight", A.wih, Aq, H); add("agent.q.action_out.bias", A.bih, Aq, 0);
  } else {
  if (!c->no_feature_norm) { add("agent.rnn.feature_norm.weight", A.fn_g, I, 0); add("agent.rnn.feature_norm.bias", A.fn_b, I, 0); }
  add("agent.rnn.mlp.fc1.0.weight", A.w1, H, I); add("agent.rnn.mlp.fc1.0.bias", A.b1, H, 0);
  add("agent.rnn.mlp.fc1.2.weight", A.ln1_g, H, 0); add("agent.rnn.mlp.fc1.2.bias", A.ln1_b, H, 0);
  add("agent.rnn.mlp.fc_h.0.weight", A.wh, H, H); add("agent.rnn.mlp.fc_h.0.bias", A.bh, H, 0);
  add("agent.rnn.mlp.fc_h.2.weight", A.lnh_g, H, 0); add("agent.rnn.mlp.fc_h.2.bias", A.lnh_b, H, 0);
  add("agent.rnn.mlp.fc2.0.0.weight", A.w2, H, H); add("agent.rnn.mlp.fc2.0.0.bias", A.b2, H, 0);
  add("agent.rnn.mlp.fc2.0.2.weight", A.ln2_g, H, 0); add("agent.rnn.mlp.fc2.0.2.bias", A.ln2_b, H, 0);
  add("agent.rnn.rnn.rnn.weight_ih_l0", A.wih, 3 * H, H); add("agent.rnn.rnn.rnn.weight_hh_l0", A.whh, 3 * H, H);
  add("agent.rnn.rnn.rnn.bias_ih_l0", A.bih, 3 * H, 0); add("agent.rnn.rnn.rnn.bias_hh_l0", A.bhh, 3 * H, 0);
  add("agent.rnn.rnn.norm.weight", A.lno_g, H, 0); add("agent.rnn.rnn.norm.bias", A.lno_b, H, 0);
  add("agent.q.action_out.weight", A.wq, Aq, H); add("agent.q.action_out.bias", A.bq, Aq, 0);
  }
  if (!c->vdn) {
    const int S = c->state_dim, N = c->n_agents, ME = c->mixer_hidden, HY = c->hyper_hidden;
    if (c->hyper_layers == 2) {
      add("mixer.hyper_w1.0.weight", M.w1a, HY, S); add("mixer.hyper_w1.0.bias", M.b1a, HY, 0);
      add("mixer.hyper_w1.2.weight", M.w1b, N * ME, HY); add("mixer.hyper_w1.2.bias", M.b1b, N * ME, 0);
      add("mixer.hyper_w2.0.weight", M.w2a, HY, S); add("mixer.hyper_w2.0.bias", M.b2a, HY, 0);
      add("mixer.hyper_w2.2.weight", M.w2b, ME, HY); add("mixer.hyper_w2.2.bias", M.b2b, ME, 0);
    } else {
      add("mixer.hyper_w1.weight", M.w1b, N * ME, S); add("mixer.hyper_w1.bias", M.b1b, N * ME, 0);
      add("mixer.hyper_w2.weight", M.w2b, ME, S); add("mixer.hyper_w2.bias", M.b2b, ME, 0);
    }
    add("mixer.hyper_b1.weight", M.wb1, ME, S); add("mixer.hyper_b1.bias", M.bb1, ME, 0);
    add("mixer.hyper_b2.0.weight", M.wb2a, HY, S); add("mixer.hyper_b2.0.bias", M.bb2a, HY, 0);
    add("mixer.hyper_b2.2.weight", M.wb2b, 1, HY); add("mixer.hyper_b2.2.bias", M.bb2b, 1, 0);
  }
  if (total_floats) *total_floats = P;
  const int n = (int)v.size();
  if (out) for (int i = 0; i < n && i < max_entries; ++i) out[i] = v[i];
  return n;
}

// =====================================================================================================
// workspace
// =====================================================================================================
static int64_t ws_layout(const mx_qmix_cfg* c, int64_t P, int npart, MxQmixWs* W) {
  const int64_t B = c->max_batch, T = c->episode_len, N = c->n_agents;
  const int64_t M = B * (T + 1) * N, E = B * T;
  int64_t o = 0;
  auto tk = [&](int64_t n) { int64_t r = o; o += (n + 63) / 64 * 64; return r; };
  for (int k = 0; k < 2; ++k) { W->gi[k] = tk(M * MX_G); W->hall[k] = tk(M * MX_H); W->qall[k] = tk(M * c->act_dim); }
  W->u1 = tk(M * MX_H); W->u2 = tk(M * MX_H);
  W->st0 = tk(M * 2); W->st1 = tk(M * 2); W->st2 = tk(M * 2); W->sto = tk(M * 2);
  W->gates = tk(M * MX_G); W->hn = tk(M * MX_H);
  W->greedy = tk(M);
  W->q_taken = tk(E * N); W->q_next = tk(E * N);
  W->qtot = tk(E); W->qtot_next = tk(E); W->err = tk(E);
  W->dq_taken = tk(E * N);
  W->dh_out = tk(M * MX_H);
  W->dgi = tk(M * MX_G);
  W->gpart = tk((int64_t)npart * P);
  W->lnpart = tk((int64_t)2 * npart * 512);      // LayerNorm sums of k_front_bwd_tc when it runs two CTAs per SM
  W->grad = tk(P + 8);
  W->info = tk(8);
  W->prio = tk(B);
  W->spart = tk((int64_t)npart * 8);
  W->adam_t = tk(8);
  W->normpart = tk(mx_grad_reduce_blocks(P));
  W->sync = tk(8);
  W->xstat = tk(8);
  W->tcimg[0] = tk((int64_t)mx_tc_image_floats(agent_in_dim(c))); W->tcimg[1] = tk((int64_t)mx_tc_image_floats(agent_in_dim(c)));
  W->xin = tk(c->prev_act_inp ? M * mx_round_up(agent_in_dim(c), 4) : 0);
  W->da2 = tk(M * MX_H); W->da1 = tk(M * MX_H);
  W->tcimgT = tk((int64_t)mx_tc_imageT_floats(agent_in_dim(c)));
  W->tcacc = tk((int64_t)mx_tc_acc_floats(M)); W->tcacc_cols = (int64_t)mx_tc_acc_floats(M) / 128;
  {
    const int64_t gH = mx_round_up(c->hyper_hidden, 4), gM = mx_round_up(c->mixer_hidden, 4), gP = mx_round_up(c->n_agents * c->mixer_hidden, 4);
    const int64_t En = c->vdn ? 0 : E;
    W->hyp_h1 = tk(En * gH); W->hyp_h2 = tk(En * gH); W->hyp_hb = tk(En * gH);
    for (int k = 0; k < 2; ++k) { W->hyp_p1[k] = tk(En * gP); W->hyp_b1[k] = tk(En * gM); W->hyp_p2[k] = tk(En * gM); W->hyp_b2[k] = tk(En); }
    W->d_q = tk(En); W->d_hp = tk(En * gM); W->d_p2 = tk(En * gM); W->d_p1 = tk(En * gP);
  }
  {     // wide-state path: weight images, pre-activations of every state row for both nets, their gradient (live elements)
    MxNetLayout Al; MxMixLayout Ml; int64_t P2;
    layouts(c, &Al, &Ml, &P2);
    const bool wide = !c->vdn && mx_mix_wide_state(Ml);
    MxMixWide wl;
    mx_mix_wide_layout(Ml, &wl);
    W->wimg = tk(wide ? (int64_t)mx_mixw_image_floats(wl) : 0);
    W->pre = tk(wide ? 2 * B * (T + 1) * wl.Cp : 0);
    W->d_pre = tk(wide ? E * wl.Cp : 0);
  }
  W->total = o;
  return o * 4;
}

static int qmix_npart() { return mx_num_sms(); }

extern "C" int64_t mx_qmix_workspace_bytes(const mx_qmix_cfg* c) {
  if (check_cfg(c)) return -1;
  MxNetLayout A; MxMixLayout M; int64_t P;
  layouts(c, &A, &M, &P);
  MxQmixWs W;
  return ws_layout(c, P, qmix_npart(), &W);
}

extern "C" int mx_qmix_create(const mx_qmix_cfg* c, float* theta, float* theta_tgt, float* adam_m, float* adam_v, void* workspace,
                              int64_t workspace_bytes, mx_qmix** out) {
  if (check_cfg(c)) return 1;
  if (!theta || !theta_tgt || !adam_m || !adam_v || !workspace || !out) { mx_set_error("mx_qmix_create: null buffer"); return 1; }
  mx_qmix* q = new mx_qmix();
  q->cfg = *c;
  layouts(c, &q->agent, &q->mix, &q->P);
  q->npart = qmix_npart();
  q->debug = 0;
  const int64_t need = ws_layout(c, q->P, q->npart, &q->W);
  if (workspace_bytes < need) { mx_set_error("mx_qmix_create: workspace %lld < %lld bytes", (long long)workspace_bytes, (long long)need); delete q; return 1; }
  q->theta = theta; q->theta_tgt = theta_tgt; q->adam_m = adam_m; q->adam_v = adam_v;
  q->ws = (float*)workspace;
  q->ws_bytes = workspace_bytes;
  q->split_ok = !c->vdn && mx_mixer_split_supported(q->mix);
  q->wide = !c->vdn && mx_mix_wide_state(q->mix);
  mx_mix_wide_layout(q->mix, &q->wl);
  if (q->wide && !q->split_ok) { mx_set_error("mx_qmix_create: state_dim %d needs the wide-state mixer, which supports mixer_hidden <= 64", c->state_dim); delete q; return 1; }
#if !MX_EMU
  if (cudaStreamCreateWithFlags(&q->side, cudaStreamNonBlocking) != cudaSuccess) { mx_set_error("mx_qmix_create: cudaStreamCreate failed"); delete q; return 1; }
  for (cudaEvent_t& e : q->ev) cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
#endif
  *out = q;
  return 0;
}
extern "C" void mx_qmix_destroy(mx_qmix* q) {
  if (!q) return;
#if !MX_EMU
  for (cudaEvent_t e : q->ev) if (e) cudaEventDestroy(e);
  if (q->side) cudaStreamDestroy(q->side);
#endif
  delete q;
}

extern "C" int mx_qmix_ws_lookup(const mx_qmix* q, const char* name, int64_t* byte_offset, int64_t* n_elems) {
  const mx_qmix_cfg& c = q->cfg;
  const int64_t B = c.max_batch, T = c.episode_len, N = c.n_agents;
  const int64_t M = B * (T + 1) * N, E = B * T;
  struct Ent { const char* n; int64_t off, cnt; };
  const MxQmixWs& W = q->W;
  const Ent tab[] = {
      {"gi_live", W.gi[0], M * MX_G}, {"gi_tgt", W.gi[1], M * MX_G}, {"h_live", W.hall[0], M * MX_H}, {"h_tgt", W.hall[1], M * MX_H},
      {"q_live", W.qall[0], M * c.act_dim}, {"q_tgt", W.qall[1], M * c.act_dim}, {"u1", W.u1, M * MX_H}, {"u2", W.u2, M * MX_H},
      {"st0", W.st0, M * 2}, {"st1", W.st1, M * 2}, {"st2", W.st2, M * 2}, {"sto", W.sto, M * 2}, {"gates", W.gates, M * MX_G},
      {"hn", W.hn, M * MX_H}, {"greedy", W.greedy, M}, {"q_taken", W.q_taken, E * N}, {"q_next", W.q_next, E * N}, {"qtot", W.qtot, E},
      {"qtot_next", W.qtot_next, E}, {"err", W.err, E}, {"dq_taken", W.dq_taken, E * N}, {"dh_out", W.dh_out, M * MX_H},
      {"xstat", W.xstat, 8}, {"dgi", W.dgi, M * MX_G}, {"grad", W.grad, q->P + 8}, {"info", W.info, 8}, {"adam_t", W.adam_t, 8}, {"prio", W.prio, B}, {"gpart", W.gpart, (int64_t)q->npart * q->P},
      {"hyp_pre", W.pre, q->wide ? 2 * B * (T + 1) * q->wl.Cp : 0}, {"d_pre", W.d_pre, q->wide ? E * q->wl.Cp : 0},
  };
  for (const Ent& e : tab)
    if (!strcmp(e.n, name)) { *byte_offset = e.off * 4; *n_elems = e.cnt; return 0; }
  mx_set_error("ws_lookup: unknown region '%s'", name);
  return 1;
}

extern "C" float* mx_qmix_grad_buffer(mx_qmix* q, int64_t* n_floats) {
  if (n_floats) *n_floats = q->P + 4;
  return q->ws + q->W.grad;
}
extern "C" const float* mx_qmix_info(mx_qmix* q) { return q->ws + q->W.info; }
extern "C" const float* mx_qmix_priorities(mx_qmix* q) { return q->ws + q->W.prio; }

// =====================================================================================================
// the step
// =====================================================================================================
static int check_batch(const mx_qmix* q, const mx_batch* b) {
  const mx_qmix_cfg& c = q->cfg;
  if (!b || b->B <= 0 || b->B > c.max_batch) { mx_set_error("qmix step: batch size outside [1, max_batch=%d]", c.max_batch); return 1; }
  if (!b->obs || !b->share || !b->act_idx || !b->rewards || !b->dones_env) { mx_set_error("qmix step: missing batch field"); return 1; }
  // b->avail may be NULL: MPE has no available-action masks (runner/rnn/mpe_runner.py:62; qmix.py:141-147 masks only when given)
  if (c.use_per && !b->weights) { mx_set_error("qmix step: use_per set but batch has no importance weights"); return 1; }
  if (b->obs_ld < c.obs_dim || b->share_ld < c.state_dim) { mx_set_error("qmix step: batch strides smaller than dims"); return 1; }
  if ((b->ep_tn_ld > 0 && b->ep_tn_ld < c.episode_len * c.n_agents) || (b->ep_t_ld > 0 && b->ep_t_ld < c.episode_len)) {
    mx_set_error("qmix step: episode strides smaller than the episode"); return 1;
  }
  return 0;
}

static OptimArgs optim_args(mx_qmix* q, int B, const int parts[4], bool after_external_allreduce = false) {   // parts: front_bwd, qhead_bwd, mixer gradient partials, scalar partials
  const mx_qmix_cfg& c = q->cfg;
  OptimArgs o;
  memset(&o, 0, sizeof(o));
  float* ws = q->ws;
  o.theta = q->theta; o.theta_tgt = q->theta_tgt; o.adam_m = q->adam_m; o.adam_v = q->adam_v;
  o.gpart = ws + q->W.gpart; o.grad = ws + q->W.grad; o.P = q->P;
  o.nseg = c.vdn ? 2 : 3;
  o.seg_begin[0] = 0; o.seg_end[0] = q->agent.lno_g; o.seg_parts[0] = parts[0];
  o.seg_begin[1] = q->agent.lno_g; o.seg_end[1] = q->agent.size; o.seg_parts[1] = parts[1];
  o.seg_begin[2] = q->agent.size; o.seg_end[2] = (int)q->P; o.seg_parts[2] = parts[2];
  if (q->wide) {      // the state layers' gradients are ONE partial (k_mixw_wgrad), the rest of the mixer has the hypernet kernel's partials
    const MxMixLayout& L = q->mix;
    const int st = parts[2] > 0 ? 1 : 0;      // (0: the caller passes no partials at all)
    auto seg = [&](int b, int e, int np) { o.seg_begin[o.nseg] = b; o.seg_end[o.nseg] = e; o.seg_parts[o.nseg] = np; ++o.nseg; };
    o.nseg = 2;
    if (L.layers == 2) {
      seg(L.w1a, L.w1b, st); seg(L.w1b, L.w2a, parts[2]);
      seg(L.w2a, L.w2b, st); seg(L.w2b, L.wb1, parts[2]);
    }
    seg(L.layers == 2 ? L.wb1 : L.w1b, L.wb2b, st); seg(L.wb2b, (int)q->P, parts[2]);
  }
  o.spart = ws + q->W.spart; o.spart_n = parts[3];
  o.info = ws + q->W.info;
  o.adam_t = reinterpret_cast<double*>(ws + q->W.adam_t);
  o.err = ws + q->W.err; o.B = B; o.T = c.episode_len;
  o.per_nu = c.per_nu; o.per_eps = c.per_eps;
  o.prio = c.use_per ? ws + q->W.prio : nullptr;
  o.lr = c.lr; o.beta1 = c.adam_beta1; o.beta2 = c.adam_beta2; o.eps = c.adam_eps; o.max_grad_norm = c.max_grad_norm; o.tau = c.tau;
  o.world_size = c.world_size;
  // per-block sums of squares of the reduced numerators: valid for k_adam on one GPU and inside k_optim_fused (computed after its
  // exchange); k_adam after an external all-reduce (NCCL / the separate p2p kernels) recomputes the norm from the summed buffer
  if (c.world_size == 1 || !after_external_allreduce) { o.normpart = ws + q->W.normpart; o.normpart_n = mx_grad_reduce_blocks(q->P); }
  o.sync = reinterpret_cast<unsigned*>(ws + q->W.sync);
  o.xstat = ws + q->W.xstat;
  o.p2p_world = q->p2p_world; o.p2p_rank = q->p2p_rank; o.p2p_slot = mx_round_up64(q->P + 8, 64); o.p2p_ll = g_mx_p2p_ll ? 1 : 0;
  o.p2p_timeout_ns = (unsigned long long)(g_mx_p2p_timeout_ms > 0 ? g_mx_p2p_timeout_ms : 10000) * 1000000ull;
  for (int p = 0; p < q->p2p_world; ++p) o.p2p_blocks[p] = q->p2p_blocks[p];
  return o;
}

// ---- forked branch helpers ------------------------------------------------------------------------------------------
// `side` runs work that does not depend on the agent nets; events order it against the caller's stream.  While the caller's
// stream is being captured the same calls fork / join the capture, i.e. the graph gets two parallel branches.  The emulator has
// no events and no side stream: it runs every launch on the caller's stream, and the event calls do nothing.
#if !MX_EMU
static inline bool want_overlap(const mx_qmix* q, int B) {     // the policy decision
  if (!g_mx_overlap || !q->side) return false;
  const long long rows = (long long)B * (q->cfg.episode_len + 1) * q->cfg.n_agents;
  return g_mx_overlap >= 2 || rows <= g_mx_overlap_rows;     // large batches are throughput-bound: a second branch only adds contention
}
static inline void ev_record(mx_qmix* q, int e, cudaStream_t s) { cudaEventRecord(q->ev[e], s); }
static inline void ev_wait(mx_qmix* q, int e, cudaStream_t s) { cudaStreamWaitEvent(s, q->ev[e], 0); }
static inline void set_pdl_auto(int M) { g_mx_pdl_auto = M <= g_mx_pdl_rows ? 1 : 0; }
#else
// as wanted on a device: the policy keeps mixer_split = 1 on the split pipeline, which the emulator then runs serially
static inline bool want_overlap(const mx_qmix*, int) { return true; }
static inline void ev_record(mx_qmix*, int, cudaStream_t) {}
static inline void ev_wait(mx_qmix*, int, cudaStream_t) {}
static inline void set_pdl_auto(int) {}
#endif
// per-kernel profiling (mx_profile_begin) times the same kernels back to back on one stream
static inline bool use_overlap(const mx_qmix* q, int B) { return q->side && want_overlap(q, B) && !g_mx_prof_on; }
static inline void fork_to_side(mx_qmix* q, int e, cudaStream_t s) { ev_record(q, e, s); ev_wait(q, e, q->side); }
static inline void join_from_side(mx_qmix* q, int e, cudaStream_t s) { ev_record(q, e, q->side); ev_wait(q, e, s); }

static int launch_prep(mx_qmix* q, cudaStream_t s) {
  const float* const th2[2] = {q->theta, q->theta_tgt};
  float* const img2[2] = {q->ws + q->W.tcimg[0], q->ws + q->W.tcimg[1]};
  if (mx_launch_tc_prep_weights(th2, q->agent, img2, 2, s)) return 1;
  q->imgT_fresh = 0;
  if (mx_tc_prep_T_wanted(q->agent.in_dim)) {      // the backward's transposed images: same parameters, same (side) branch
    if (mx_launch_tc_prep_weights_T(q->theta, q->agent, q->ws + q->W.tcimgT, s)) return 1;
    q->imgT_fresh = 1;
  }
  return 0;
}

// Parameter-only work of the coming step (TF32 hi/lo weight images of the front layers), started on the side branch so that it
// overlaps the index draw and the gather.  Optional: mx_qmix_backward_only does it itself when this was not called.
int mx_qmix_prefork(mx_qmix* q, int B, void* stream) {
  if (!use_overlap(q, B) || !mx_front_tc_usable(q->agent.in_dim, true) || q->prep_pending) return 0;
  fork_to_side(q, MX_EV_FORK, (cudaStream_t)stream);
  if (launch_prep(q, q->side)) return 1;
  ev_record(q, MX_EV_PREP, q->side);
  q->prep_pending = 1;
  return 0;
}

// ---- the launches of one step: the schedule is decided once, each builder fills its arguments from the learner and the batch, and
// backward_core below lists the phases
namespace {
struct Step {
  mx_qmix* q;
  const mx_batch* b;
  cudaStream_t s, side;       // the caller's stream; the side branch, or s when the step runs serially
  const mx_qmix_cfg& c;
  const MxQmixWs& W;
  float* ws;
  int B, T, N, M, ld_tn, ld_t;      // ld_tn, ld_t: episode strides of the batch's [B][T][N] and [B][T] fields
  const float* X; int ldx;    // agent-net input rows: the observations, or [obs | previous action] packed by pack_input (prev_act_inp)
  bool overlap, wanted;       // the side branch runs beside the agent nets; the policy's wish (profiling turns overlap off)
  bool split;                 // the mixer as hypernet forward / core / hypernet backward, not the fused k_mixer
  bool mid;                   // the core is k_mid: the Q head, the mixer core and the Q head's backward in one launch
  bool gsplit;                // the GRU weight gradients as their own kernel (k_gru_wgrad), beside k_front_bwd when forked
  int parts[4] = {0, 0, 0, 0};      // gradient partials of front_bwd, the Q head, the mixer; scalar partials
  MixerArgs mx{};
  FrontFwdArgs ff{};
  MidArgs md{};
  FrontBwdArgs fb{};

  Step(mx_qmix* q_, const mx_batch* b_, cudaStream_t s_) : q(q_), b(b_), s(s_), c(q_->cfg), W(q_->W), ws(q_->ws) {
    B = b->B; T = c.episode_len; N = c.n_agents; M = B * (T + 1) * N;
    ld_tn = b->ep_tn_ld > 0 ? b->ep_tn_ld : T * N; ld_t = b->ep_t_ld > 0 ? b->ep_t_ld : T;
    X = c.prev_act_inp ? ws + W.xin : b->obs;
    ldx = c.prev_act_inp ? mx_round_up(c.obs_dim + c.act_dim, 4) : b->obs_ld;

    mx.theta = q->theta; mx.theta_tgt = q->theta_tgt; mx.L = q->mix; mx.vdn = c.vdn;
    mx.share = b->share; mx.share_ld = b->share_ld;
    mx.q_taken = ws + W.q_taken; mx.q_next = ws + W.q_next;
    mx.rewards = b->rewards; mx.dones_env = b->dones_env; mx.weights = c.use_per ? b->weights : nullptr;
    mx.ld_tn = ld_tn; mx.ld_t = ld_t;
    mx.B = B; mx.T = T; mx.N = N; mx.gamma = c.gamma; mx.huber_delta = c.huber_delta; mx.use_huber = c.use_huber;
    mx.qtot = ws + W.qtot; mx.qtot_next = ws + W.qtot_next; mx.err = ws + W.err; mx.dq_taken = ws + W.dq_taken;
    mx.gpart = ws + W.gpart; mx.P = q->P; mx.spart = ws + W.spart;
    mx.hyp_h1 = ws + W.hyp_h1; mx.hyp_h2 = ws + W.hyp_h2; mx.hyp_hb = ws + W.hyp_hb;
    for (int k = 0; k < 2; ++k) { mx.hyp_p1[k] = ws + W.hyp_p1[k]; mx.hyp_b1[k] = ws + W.hyp_b1[k]; mx.hyp_p2[k] = ws + W.hyp_p2[k]; mx.hyp_b2[k] = ws + W.hyp_b2[k]; }
    mx.d_q = ws + W.d_q; mx.d_hp = ws + W.d_hp; mx.d_p2 = ws + W.d_p2; mx.d_p1 = ws + W.d_p1;
    mx.gH = mx_round_up(c.hyper_hidden, 4); mx.gM = mx_round_up(c.mixer_hidden, 4); mx.gP = mx_round_up(c.n_agents * c.mixer_hidden, 4);
    mx.wide = q->wide; mx.wl = q->wl;
    if (q->wide) { mx.wimg = ws + W.wimg; mx.pre = ws + W.pre; mx.d_pre = ws + W.d_pre; }

    ff.X = X; ff.ldx = ldx; ff.M = M; ff.feature_norm = c.no_feature_norm ? 0 : 1; ff.act_tanh = c.use_tanh;
    ff.theta[0] = q->theta; ff.theta[1] = q->theta_tgt; ff.L = q->agent;
    ff.gi[0] = ws + W.gi[0]; ff.gi[1] = ws + W.gi[1];
    ff.u1 = ws + W.u1; ff.u2 = ws + W.u2; ff.st0 = ws + W.st0; ff.st1 = ws + W.st1; ff.st2 = ws + W.st2;
    if (mx_front_tc_usable(q->agent.in_dim, true)) {     // the TF32 hi/lo weight images, rebuilt by weight_images()
      ff.tc_img[0] = ws + W.tcimg[0]; ff.tc_img[1] = ws + W.tcimg[1];
      ff.tc_acc = ws + W.tcacc; ff.tc_acc_cols = (int)W.tcacc_cols;
    }

    md.mix = mx;
    head<true, true>(md);
    // the live net's backward through its front layers from the "gi" gradient rows, and through the GRU weights unless cfg.mlp
    fb.X = X; fb.ldx = ldx; fb.M = M; fb.T = T; fb.N = N; fb.feature_norm = c.no_feature_norm ? 0 : 1; fb.act_tanh = c.use_tanh;
    fb.theta = q->theta; fb.L = q->agent; fb.u1 = ff.u1; fb.u2 = ff.u2; fb.st0 = ff.st0; fb.st1 = ff.st1; fb.st2 = ff.st2;
    fb.dgi = ws + W.dgi; fb.gpart = mx.gpart; fb.P = q->P;
    if (c.mlp) fb.no_gru = 1;
    else { fb.gates = ws + W.gates; fb.hall = ws + W.hall[0]; }
    fb.ln_part = ws + W.lnpart; fb.ln_part_rows = 2 * q->npart;
    fb.da2_out = ws + W.da2; fb.da1_out = ws + W.da1; fb.tc_imgT = ws + W.tcimgT;
    fb.tc_acc = ws + W.tcacc; fb.tc_acc_cols = (int)W.tcacc_cols;

    overlap = use_overlap(q, B); wanted = want_overlap(q, B);
    side = overlap ? q->side : s;
    // the split mixer only pays off when its hypernet kernels run beside the agent nets (serial, the fused k_mixer moves less data)
    split = q->wide || (q->split_ok && (g_mx_mixer_split >= 2 || (g_mx_mixer_split == 1 && wanted)));
    // the debug mode of the parity tests keeps the separate kernels because it materialises every per-action Q value
    mid = !c.mlp && split && g_mx_mid_fused && !q->debug && mx_mid_supported(md);
    gsplit = mx_gru_wgrad_split_usable(fb);      // never with cfg.mlp (no_gru)
  }

  void fork(int e) { if (overlap) fork_to_side(q, e, s); }
  void join(int e) { if (overlap) join_from_side(q, e, s); }

  // the Q values a forward selects and, in debug mode, every per-action value and the greedy action (k_qhead, k_mlp_qselect)
  template <class Args> void q_outputs(Args& a) const {
    a.q_taken = ws + W.q_taken; a.q_next = ws + W.q_next;
    a.greedy = q->debug ? reinterpret_cast<int32_t*>(ws + W.greedy) : nullptr;
    a.qall0 = q->debug ? ws + W.qall[0] : nullptr; a.qall1 = q->debug ? ws + W.qall[1] : nullptr;
  }
  // the Q head (post-GRU LayerNorm + Linear) and the rows it reads: k_qhead, k_mid, k_qhead_bwd.  FWD: the forward over both nets;
  // GRAD: the backward into dh_out and the head's gradient partials
  template <bool FWD, bool GRAD, class Args> void head(Args& a) const {
    a.wq = q->agent.wq; a.bq = q->agent.bq; a.lno_g = q->agent.lno_g; a.lno_b = q->agent.lno_b;
    a.act_idx = b->act_idx; a.T = T; a.N = N; a.A = c.act_dim; a.ld_tn = ld_tn;
    if constexpr (FWD) { a.hall[0] = ws + W.hall[0]; a.hall[1] = ws + W.hall[1]; a.avail = b->avail; a.act_ld = b->act_ld; a.double_q = c.double_q; }
    if constexpr (GRAD) { a.dh_out = ws + W.dh_out; a.gpart = mx.gpart; a.P = q->P; }
  }

  // ---- the phases ----
  int pack_input() const {    // prev_act_inp: network input = [obs | previous action], packed once per step into the workspace
    if (!c.prev_act_inp) return 0;
    if (!b->acts) { mx_set_error("qmix step: prev_act_inp needs the batch's one-hot actions"); return 1; }
    return mx_launch_pack_prev_act(b->obs, b->obs_ld, b->acts, b->act_ld, ws + W.xin, ldx, B, T, N, c.obs_dim, c.act_dim, s);
  }

  // weights changed in the last Adam / Polyak: rebuild the TF32 hi/lo images (18k elements per net), unless mx_qmix_prefork()
  // launched it on the side branch before the batch was sampled
  int weight_images() const {
    if (!ff.tc_img[0]) return 0;
    if (!q->prep_pending) return launch_prep(q, s);
    ev_wait(q, MX_EV_PREP, s); q->prep_pending = 0;
    return 0;
  }

  // the mixer's hypernetworks depend on the sampled states and the parameters only: forked branch beside the agent nets, before the
  // front kernel (forked after it, beside the recurrence, the hypernet CTAs cost more)
  int hyper_fwd_forked() {
    if (!(split && overlap)) return 0;
    fork(MX_EV_BATCH);
    return mx_launch_mix_hyper_fwd(mx, side);
  }

  // the mixer between the agents' Q values and their gradient.  Split: the hypernet forward (here, unless it was forked), the core
  // -- k_mid, or k_mix_core between k_qhead and k_qhead_bwd -- then the hypernet backward, beside the agent-net backward when forked.
  // Otherwise the fused k_mixer.
  int mixer() {
    if (!split) { const int rc = mx_launch_mixer(mx, &parts[2], s); parts[3] = parts[2]; return rc; }
    if (!overlap && mx_launch_mix_hyper_fwd(mx, s)) return 1;
    join(MX_EV_HYPER);
    if (mid ? mx_launch_mid(md, &parts[1], s) : mx_launch_mix_core(mx, &parts[3], s)) return 1;
    if (mid) parts[3] = parts[1];
    fork(MX_EV_CORE);
    return mx_launch_mix_hyper_bwd(mx, &parts[2], side);
  }
  int mlp_qselect() const {
    MlpQSelArgs a{};
    a.gi[0] = ff.gi[0]; a.gi[1] = ff.gi[1]; a.act_idx = b->act_idx; a.avail = b->avail; a.act_ld = b->act_ld; a.ld_tn = ld_tn;
    a.B = B; a.N = N; a.A = c.act_dim; a.double_q = c.double_q;
    q_outputs(a);
    return mx_launch_mlp_qselect(a, s);
  }
  int gru_fwd() const {
    GruFwdArgs a{};
    a.theta[0] = q->theta; a.theta[1] = q->theta_tgt; a.whh = q->agent.whh; a.bhh = q->agent.bhh;
    a.gi[0] = ff.gi[0]; a.gi[1] = ff.gi[1]; a.hall[0] = ws + W.hall[0]; a.hall[1] = ws + W.hall[1];
    a.gates = ws + W.gates; a.hn = ws + W.hn; a.R = B * N; a.T = T; a.N = N;
    return mx_launch_gru_fwd(a, 2, s);
  }
  int qhead() const {
    QHeadArgs a{};
    head<true, false>(a);
    q_outputs(a);
    a.theta[0] = q->theta; a.theta[1] = q->theta_tgt; a.sto = ws + W.sto; a.M = M;
    return mx_launch_qhead(a, s);
  }
  int qhead_bwd() {
    QHeadBwdArgs a{};
    head<false, true>(a);
    a.theta = q->theta; a.hall = ws + W.hall[0]; a.sto = ws + W.sto; a.dq_taken = mx.dq_taken; a.M = M;
    return mx_launch_qhead_bwd(a, &parts[1], s);
  }
  int gru_bwd() const {
    GruBwdArgs a{};
    a.theta = q->theta; a.whh = q->agent.whh; a.hall = ws + W.hall[0]; a.gates = ws + W.gates; a.hn = ws + W.hn; a.dh_out = ws + W.dh_out;
    a.dgi = ws + W.dgi; a.R = B * N; a.T = T; a.N = N;
    return mx_launch_gru_bwd(a, s);
  }

  // k_gru_wgrad on the side branch (gsplit), k_front_bwd, then the one join of everything the side branch still runs
  int front_bwd() {
    fb.tc_imgT_ready = q->imgT_fresh; q->imgT_fresh = 0;
    if (gsplit) { fb.gru_wgrad_ext = 1; fork(MX_EV_GBWD); if (mx_launch_gru_wgrad(fb, side)) return 1; }
    if (mx_launch_front_bwd(fb, &parts[0], s)) return 1;
    if (split || gsplit) join(MX_EV_HBWD);
    return 0;
  }
};
}  // namespace

// everything of the step up to (not including) the optimiser: forward, loss, backward; leaves the per-CTA gradient partials and
// fills `*oa` with the optimiser's arguments
static int backward_core(mx_qmix* q, const mx_batch* b, void* stream, OptimArgs* oa) {
  if (check_batch(q, b)) return 1;
  Step st(q, b, (cudaStream_t)stream);
  set_pdl_auto(st.M);      // programmatic dependent launches for this step's kernels (and the sample that follows it)

  if (st.pack_input()) return 1;
  if (st.weight_images()) return 1;
  if (st.hyper_fwd_forked()) return 1;
  if (mx_launch_front_fwd(st.ff, 2, st.s)) return 1;
  if (q->cfg.mlp) {      // transition-level variant (M_QMix / M_VDN): no recurrence, Q = columns [0, A) of the "gi" rows
    if (st.mlp_qselect()) return 1;
    if (st.mixer()) return 1;
    if (mx_launch_mlp_dgi(st.mx.dq_taken, b->act_idx, st.ld_tn, st.ws + st.W.dgi, st.B, st.N, st.s)) return 1;
  } else {
    if (st.gru_fwd()) return 1;
    if (!st.mid && st.qhead()) return 1;      // k_mid runs the Q head and its backward around the mixer core
    if (st.mixer()) return 1;
    if (!st.mid && st.qhead_bwd()) return 1;
    if (st.gru_bwd()) return 1;
  }
  if (st.front_bwd()) return 1;
  *oa = optim_args(q, st.B, st.parts);
  return 0;
}

extern "C" int mx_qmix_backward_only(mx_qmix* q, const mx_batch* b, void* stream) {
  OptimArgs o;
  if (backward_core(q, b, stream, &o)) return 1;
  return mx_launch_grad_reduce(o, (cudaStream_t)stream);
}

extern "C" int mx_qmix_apply_ex(mx_qmix* q, uint32_t flags, void* stream) {
  const int parts[4] = {0, 0, 0, 0};
  OptimArgs o = optim_args(q, q->cfg.max_batch, parts, true);
  o.fuse_polyak = (flags & MX_STEP_FUSE_SOFT_UPDATE) ? 1 : 0;
  return mx_launch_adam(o, (cudaStream_t)stream);
}
extern "C" int mx_qmix_apply(mx_qmix* q, void* stream) { return mx_qmix_apply_ex(q, 0, stream); }

extern "C" int mx_qmix_step_ex(mx_qmix* q, const mx_batch* b, uint32_t flags, void* stream) {
  OptimArgs o;
  if (backward_core(q, b, stream, &o)) return 1;
  if (q->cfg.world_size == 1 || q->p2p_world) {      // ONE launch: partial reduction + [exchange over peer memory] + clip + Adam [+ Polyak]
    o.fuse_polyak = (flags & MX_STEP_FUSE_SOFT_UPDATE) ? 1 : 0;
    const int rc = mx_launch_optim_fused(o, (cudaStream_t)stream);
    if (rc >= 0) return rc;
  }
  if (mx_launch_grad_reduce(o, (cudaStream_t)stream)) return 1;
  if (q->cfg.world_size > 1) {
    if (!q->p2p_world) return 0;         // NCCL path: the caller all-reduces mx_qmix_grad_buffer(), then mx_qmix_apply[_ex]()
    if (mx_qmix_p2p_publish(q, stream) || mx_qmix_p2p_reduce(q, stream)) return 1;   // one-shot all-reduce over peer memory
  }
  return mx_qmix_apply_ex(q, flags, stream);
}
extern "C" int mx_qmix_step(mx_qmix* q, const mx_batch* b, void* stream) { return mx_qmix_step_ex(q, b, 0, stream); }
extern "C" int mx_qmix_set_debug(mx_qmix* q, int32_t on) { q->debug = on ? 1 : 0; return 0; }

extern "C" int mx_qmix_soft_update(mx_qmix* q, void* stream) {
  return mx_launch_polyak(q->theta_tgt, q->theta, q->P, q->cfg.tau, (cudaStream_t)stream);
}
extern "C" int mx_qmix_hard_update(mx_qmix* q, void* stream) {
  cudaMemcpyAsync(q->theta_tgt, q->theta, (size_t)q->P * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream);
  MX_MARK("hard_update_memcpy", (cudaStream_t)stream);
  return 0;
}

// =====================================================================================================
// whole-step CUDA graph
// =====================================================================================================
static int run_sequence(mx_replay* r, mx_qmix* q, int B, double beta, uint32_t flags, void* stream) {
  if ((flags & 3u) && mx_qmix_prefork(q, B, stream)) return 1;      // weight-image prep overlaps the draw + gather
  if (flags & 1u) { if (mx_replay_sample_uniform(r, B, stream)) return 1; }
  else if (flags & 2u) { (void)beta; if (mx_replay_sample_per_state_beta(r, B, stream)) return 1; }     // beta: device scalar, see mx_graph_capture
  mx_batch b;
  if (mx_replay_batch(r, B, &b)) return 1;
  const bool fuse = (flags & 4u) && (q->cfg.world_size == 1 || q->p2p_world);
  if (mx_qmix_step_ex(q, &b, fuse ? MX_STEP_FUSE_SOFT_UPDATE : 0u, stream)) return 1;
  if (flags & 8u) {
    if (mx_replay_update_priorities(r, b.idx, mx_qmix_priorities(q), nullptr, nullptr, B, stream)) return 1;
  }
  if ((flags & 4u) && !fuse) { if (mx_qmix_soft_update(q, stream)) return 1; }
  return 0;
}

// Record `seq` (the library's own launch sequence) on `stream` into an executable graph.
int mx_graph_capture_seq(std::function<int(void*)> seq, std::function<void()> after_launch, void* stream, mx_graph** out) {
  mx_graph* g = new mx_graph();
  g->seq = seq; g->after_launch = after_launch; g->n_kernels = 0;
#if !MX_EMU
  cudaStream_t s = (cudaStream_t)stream;
  if (!s) { mx_set_error("graph capture: needs a non-default stream (the legacy stream cannot be captured)"); delete g; return 1; }
  {
    cudaError_t be = cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal);
    if (be != cudaSuccess) {
      mx_set_error("cudaStreamBeginCapture failed: %s", cudaGetErrorString(be));
      cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
      if (cudaStreamIsCapturing(s, &st) == cudaSuccess && st != cudaStreamCaptureStatusNone) { cudaGraph_t tmp = nullptr; cudaStreamEndCapture(s, &tmp); if (tmp) cudaGraphDestroy(tmp); }
      cudaGetLastError();
      delete g;
      return 1;
    }
  }
  int rc = seq(stream);
  cudaError_t e = cudaStreamEndCapture(s, &g->graph);
  if (rc || e != cudaSuccess) { mx_set_error("graph capture failed: %s", rc ? mx_last_error() : cudaGetErrorString(e)); delete g; return 1; }
  if (cudaGraphInstantiate(&g->exec, g->graph, 0) != cudaSuccess) { mx_set_error("cudaGraphInstantiate failed"); delete g; return 1; }
  size_t nn = 0;
  cudaGraphGetNodes(g->graph, nullptr, &nn);
  std::vector<cudaGraphNode_t> nodes(nn);
  if (nn) cudaGraphGetNodes(g->graph, nodes.data(), &nn);
  for (size_t i = 0; i < nn; ++i) {
    cudaGraphNodeType ty;
    if (cudaGraphNodeGetType(nodes[i], &ty) == cudaSuccess && ty == cudaGraphNodeTypeKernel) g->n_kernels++;
  }
#endif
  *out = g;
  return 0;
}

extern "C" int mx_graph_capture(mx_replay* r, mx_qmix* q, int32_t B, double beta, uint32_t flags, void* stream, mx_graph** out) {
  if (!r || !q || !out) { mx_set_error("mx_graph_capture: null argument"); return 1; }
  if ((flags & 2u) && mx_replay_set_beta(r, beta, stream)) return 1;     // initial exponent; mx_replay_set_beta() before a launch changes it
  return mx_graph_capture_seq([=](void* st) { return run_sequence(r, q, B, beta, flags, st); }, nullptr, stream, out);
}

extern "C" int mx_graph_launch(mx_graph* g, void* stream) {
#if !MX_EMU
  if (cudaGraphLaunch(g->exec, (cudaStream_t)stream) != cudaSuccess) { mx_set_error("cudaGraphLaunch: %s", cudaGetErrorString(cudaGetLastError())); return 1; }
  g_mx_launches += g->n_kernels;   // kernel nodes replayed by this launch
  if (g->after_launch) g->after_launch();
  return 0;
#else
  const int rc = g->seq(stream);
  if (!rc && g->after_launch) g->after_launch();
  return rc;
#endif
}

extern "C" int32_t mx_graph_num_kernels(const mx_graph* g) { return g ? g->n_kernels : 0; }

extern "C" void mx_graph_destroy(mx_graph* g) {
  if (!g) return;
#if !MX_EMU
  cudaGraphExecDestroy(g->exec);
  cudaGraphDestroy(g->graph);
#endif
  delete g;
}
