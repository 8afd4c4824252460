"""Transition-level coverage of the MLP MADDPG / MATD3 learner (csrc/maddpg.cu maddpg_step_mlp) against a float64 oracle: shared by the
emulated (CPU) and the GPU test modules.

The lock-step checks (mlp_maddpg_checks.lockstep) compare whole-batch gradients per tensor at 1e-4 x max.  One transition is 1 / B of a
critic tensor and 1 / (2 N B) of the actor's rows, so a kernel that drops or double-counts the last partial tile of a row space is
invisible there.  The checks here make every transition count:

* isolated critic transition: PER on, importance weights one-hot on transition b.  The critic loss is linear in the weights, so its
  gradient is exactly b's one live row (plus its target row, through y).
* isolated actor row: valid_transition one-hot on (agent n, transition b).  The actor loss is -Q of that one agent-replaced copy, and the
  actor gradient comes from one actor row.  Its actor_loss is a per-row forward check of the live actor, the action transform, pack
  mode 2 and the critic forward.
* per-transition forward: PER weights all 1; every transition's priority (the mean over the K heads of |y - Q_k|) against float64: the
  target actor, the one-hot / Gumbel target actions, pack modes 0 and 1, both critic forwards and the min over the K heads, per row.
* batch size changing on one learner: max_batch, then 1, then a batch one tile smaller, each step against float64.

The isolated runs use lr 0: the actor phase then reads the critic the step started from, so a decision of the critic phase (a ReLU
kink on another transition's row) cannot reach the isolated actor row through Adam, and the learner's state is the same for every run.

Decisions -- the arg-max target actions, the hard Gumbel samples and the ReLU kinks -- change between fp32 and float64 only at near-ties.
Every decision the isolated transition's gradient depends on must have a float64 margin above DECISION_MARGIN; a transition that misses
it is redrawn (its observations, actions and shared observations) and the redraws are counted, never absorbed into a wider bound.
"""
import zlib

import numpy as np
import torch
import torch.nn.functional as F

import mlp_maddpg_checks as mc
import mlp_maddpg_md_checks as mdc
from row_coverage_checks import GRAD_TOL, ROW_TOL, TD_ULPS, TileRules, kernels_run  # noqa: F401 (TileRules: for the test modules)

from oracle.maddpg_mlp_md import MlpMaddpgMD, draw_noise_multi_md, step_multi_md

DECISION_MARGIN = 1e-3
SOFTMAX_SLACK = 0.05
MAX_REDRAWS = 40
# An isolated row whose gradient the fp32 oracle itself gets wrong by more than this share of GRAD_TOL is ill-conditioned, not a tile
# edge: above 128 critic columns the actor row's gradient is the critic's input-LayerNorm backward at the agent's action columns,
# rstd (d0 g - mean(d0 g) - xh mean(d0 g xh)), whose terms can cancel to a small share of their size.  Measured on the emulator at
# simple_spread N = 6 (critic 246): one copy row in four where the fp32 oracle is 8.4e-6 off float64 (4e-7 on the other three) and the
# engine 2.5e-5.  Such a transition is redrawn like a near-tie and counted (stats["ill_conditioned"], printed per case), never absorbed
# into a wider bound.  The rule applies only to critics wider than FP32_COND_MIN_CRITIC columns; narrower cases are checked as drawn.
FP32_COND_SHARE = 0.25
FP32_COND_MIN_CRITIC = 128


# ---- the learner pair ------------------------------------------------------------------------------------------------------
def build_pair(specs, S, B, discrete=True, td3=False, seed=11, **over):
    """(args, {policy_id: policy}, trainer, {policy_id: float64 MlpMaddpgMD}) with every tensor of every network randomised (the live
    nets around their initialisation, the targets near the live ones, both head sets), trainer max_batch = B.  specs as
    mlp_maddpg_md_checks.norm_specs; one spec is the shared-policy learner."""
    from offpolicy._b200.factory import build_mlp_maddpg_multi
    torch.manual_seed(seed)
    over.setdefault("max_grad_norm", 1e9)        # the isolated gradients are compared unclipped
    args, pols, tr, _ = build_mlp_maddpg_multi(specs, S, B, discrete=discrete, td3=td3, **over)
    gen = torch.Generator().manual_seed(seed)
    noisy = lambda sd, s: {k: v.cpu() + s * torch.randn(v.shape, generator=gen) for k, v in sd.items()}
    for p in sorted(pols):
        pol = pols[p]
        for live, tgt in ((pol.actor, pol.target_actor), (pol.critic, pol.target_critic)):
            sd = noisy(live.state_dict(), 0.2)
            live.load_state_dict(sd)
            tgt.load_state_dict(noisy(sd, 0.05))
        for heads in (pol.critic_heads, pol.target_critic_heads):
            heads.load_state_dict(noisy(heads.state_dict(), 0.3))
    return args, pols, tr, oracles64(args, pols)


def oracles64(args, pols, dtype=torch.float64):
    cpu = lambda m: {k: v.cpu() for k, v in m.state_dict().items()}
    return {p: MlpMaddpgMD(cpu(pol.actor), cpu(pol.critic), cpu(pol.critic_heads), cpu(pol.target_actor), cpu(pol.target_critic),
                           cpu(pol.target_critic_heads), pol.discrete, pol.td3, gamma=args.gamma, lr=args.lr, eps=args.opti_eps,
                           weight_decay=args.weight_decay, max_grad_norm=args.max_grad_norm, tau=args.tau, huber=args.use_huber_loss,
                           huber_delta=args.huber_delta, use_per=args.use_per, per_eps=args.per_eps, relu=bool(args.use_ReLU),
                           feature_norm=bool(args.use_feature_normalization), segs=pol.act_segs, dtype=dtype)
            for p, pol in pols.items()}


def step_both(tr, L64, p, batch, seed):
    """One engine step of policy p and the float64 oracle's, from the same torch RNG state (the same noise draws)."""
    torch.manual_seed(seed)
    info, prio, _ = tr.shared_train_policy_on_batch(p, batch)
    torch.manual_seed(seed)
    tn, an = draw_noise_multi_md(mdc.noise_shapes(tr), p, np.asarray(batch[0][p]).shape[1])
    ref, rprio, grads = step_multi_md(L64, p, batch, tn, an, dtype=torch.float64)
    return info, prio, ref, rprio, grads


# ---- float64 decisions --------------------------------------------------------------------------------------------------------
def _trunk(L, p, x):
    """MLPBase forward in float64 (oracle/maddpg_mlp.py _mlp), returning (output, [fc1 and fc2 pre-activations])."""
    act = torch.relu if L.relu else torch.tanh
    if L.feature_norm:
        x = F.layer_norm(x, x.shape[-1:], p["mlp.feature_norm.weight"], p["mlp.feature_norm.bias"])
    a1 = F.linear(x, p["mlp.mlp.fc1.0.weight"], p["mlp.mlp.fc1.0.bias"])
    h = F.layer_norm(act(a1), (64,), p["mlp.mlp.fc1.2.weight"], p["mlp.mlp.fc1.2.bias"])
    a2 = F.linear(h, p["mlp.mlp.fc2.0.0.weight"], p["mlp.mlp.fc2.0.0.bias"])
    return F.layer_norm(act(a2), (64,), p["mlp.mlp.fc2.0.2.weight"], p["mlp.mlp.fc2.0.2.bias"]), [a1, a2]


def _kinks(L, pre):
    """Per row: the smallest |pre-activation| of a ReLU net (inf for tanh, which has no kink)."""
    if not L.relu:
        return torch.full((pre[0].shape[0],), float("inf"), dtype=torch.float64)
    return torch.stack([a.abs().min(-1)[0] for a in pre]).min(0)[0]


def _gap(z, segs):
    """Per row: top-1 minus top-2 of z within each block of segs (the whole row when segs is None), the smallest over the blocks."""
    out = []
    for blk in (z.split(list(segs), -1) if segs else [z]):
        t = blk.topk(2, -1)[0] if blk.shape[-1] > 1 else torch.cat([blk, blk.new_full(blk.shape, -float("inf"))], -1)
        out.append(t[:, 0] - t[:, 1])
    return torch.stack(out).min(0)[0]


def _action_gap(L, out, noise, avail):
    """Per row: the arg-max margin of a Discrete action (logits, or logits + Gumbel for the hard Gumbel sample; masked entries -1e10 as
    the reference, blocks of a MultiDiscrete action on their own with no mask); inf for a Box action."""
    if not L.discrete:
        return torch.full((out.shape[0],), float("inf"), dtype=torch.float64)
    z = out + noise if noise is not None else out.clone()
    if avail is not None and L.segs is None:
        z = z.masked_fill(avail == 0, -1e10)
    return _gap(z, L.segs)


@torch.no_grad()
def margins(L64, p, batch, tn, an, slack=True):
    """float64 decision margins of policy p's update on `batch` with the draws (tn, an): {"critic": per transition, the smallest over
    the decisions its critic gradient depends on (every policy's target actor on its next observations and target action, the target
    critic's and the live critic's kinks), "actor": (N_p, B) per agent-replaced copy (the live actor's kinks and Gumbel sample, the critic's
    kinks on the copy), "target": per transition, the target actions' gaps alone (what its forward value depends on)}; and "qscale":
    (N_p, B) sum_j |w_j h_j| + |bias| of head 0 on each copy, the natural scale of that Q value's round-off; "qmag": per transition
    the same scale of its TD errors, the larger of the live heads' and |r| + gamma times the target heads'."""
    f = lambda x: None if x is None else torch.as_tensor(np.asarray(x)).double()
    obs, share, acts, rew, nobs, nshare, _d, dones_env, valid, avail, navail = batch[:11]
    ids = sorted(L64)
    B = np.asarray(obs[p]).shape[1]
    crit = torch.full((B,), float("inf"), dtype=torch.float64)
    tgt_gap = crit.clone()
    cent_act, cent_nact, start = [], [], 0
    for q in ids:
        Lq = L64[q]
        nob = f(nobs[q])
        Nq = nob.shape[0]
        if q == p:
            start = len(cent_act)
        h, pre = _trunk(Lq, Lq.target_actor, nob.reshape(Nq * B, -1))
        out = Lq.actor_out(Lq.target_actor, nob.reshape(Nq * B, -1)).detach()
        nav = None if navail is None or navail.get(q) is None else f(navail[q]).reshape(Nq * B, -1)
        noise = f(tn[q]) if (Lq.td3 and Lq.discrete) else None
        gap = _action_gap(Lq, out, noise, nav).view(Nq, B).min(0)[0]
        tgt_gap = torch.minimum(tgt_gap, gap)
        crit = torch.minimum(crit, torch.minimum(gap, _kinks(Lq, pre).view(Nq, B).min(0)[0]))
        nact = Lq.act_target(out, f(tn[q]), nav)
        cent_nact.append(torch.cat(nact.split(B, 0), -1))
        cent_act.extend(list(f(acts[q])))
    L = L64[p]
    # sum_j |w_kj h_j| + |b_k|, the largest over the K heads: the scale of a Q value's round-off
    head_scale = lambda hs, h: torch.stack([(h * hs["q_outs.%d.weight" % k][0]).abs().sum(-1) + hs["q_outs.%d.bias" % k][0].abs()
                                            for k in range(L.K)]).max(0)[0]
    h_t, pre_t = _trunk(L, L.target_critic, torch.cat([f(nshare[p]), torch.cat(cent_nact, -1)], 1))
    h_c, pre_c = _trunk(L, L.critic, torch.cat([f(share[p]), torch.cat(cent_act, -1)], 1))
    qmag = torch.maximum(head_scale(L.heads, h_c), f(rew[p])[0].view(-1).abs() + L.gamma * head_scale(L.target_heads, h_t))
    head = lambda hs, h: torch.stack([(h * hs["q_outs.%d.weight" % k][0]).sum(-1) + hs["q_outs.%d.bias" % k][0] for k in range(L.K)])
    y = f(rew[p])[0].view(-1) + L.gamma * (1 - f(dones_env[p]).view(-1)) * head(L.target_heads, h_t).min(0)[0]
    qmax = head(L.heads, h_c).max(0)[0]
    crit = torch.minimum(crit, torch.minimum(_kinks(L, pre_t), _kinks(L, pre_c)))
    ob = f(obs[p])
    Np = ob.shape[0]
    _, pre_a = _trunk(L, L.actor, ob.reshape(Np * B, -1))
    out = L.actor_out(L.actor, ob.reshape(Np * B, -1)).detach()
    av = None if avail is None or avail.get(p) is None else f(avail[p]).reshape(Np * B, -1)
    act_m = torch.minimum(_kinks(L, pre_a), _action_gap(L, out, f(an), av) if L.discrete else _kinks(L, pre_a))
    if L.discrete and slack:
        # the straight-through gradient is the softmax Jacobian's: at a saturated block (top probability 1 - d) its fp32 backward
        # y* (g* - sum_j y_j g_j) cancels to ~d of its terms, ~eps / d relative into every actor tensor (measured 2.3e-5 with d ~ 3e-3 on
        # an H100): each block's 1 - max softmax must stay above SOFTMAX_SLACK, scaled into the same margin
        z = out + f(an)
        if av is not None and L.segs is None:
            z = z.masked_fill(av == 0, -1e10)
        room = torch.stack([1.0 - F.softmax(blk, -1).max(-1)[0] for blk in (z.split(L.segs, -1) if L.segs else [z])]).min(0)[0]
        if av is not None and L.segs is None:       # one available action: the sample is exactly one-hot, its Jacobian exactly zero
            room = torch.where((av != 0).sum(-1) <= 1, torch.ones_like(room), room)
        act_m = torch.minimum(act_m, room * (DECISION_MARGIN / SOFTMAX_SLACK))
    pol = L.act_live(out, f(an), av).split(B, 0)
    rows = [torch.cat([pol[i] if j == start + i else cent_act[j] for j in range(len(cent_act))], -1) for i in range(Np)]
    h_r, pre_r = _trunk(L, L.critic, torch.cat([f(share[p]).repeat(Np, 1), torch.cat(rows, 0)], 1))
    act_m = torch.minimum(act_m, _kinks(L, pre_r)).view(Np, B)
    qscale = ((h_r * L.heads["q_outs.0.weight"][0]).abs().sum(-1) + L.heads["q_outs.0.bias"].abs()).view(Np, B)
    return {"critic": crit, "actor": act_m, "target": tgt_gap, "qscale": qscale, "qmag": qmag, "y": y, "qmax": qmax}


def noise_at(tr, p, B, seed):
    torch.manual_seed(seed)
    return draw_noise_multi_md(mdc.noise_shapes(tr), p, B)


def redraw(batch, rng, b, fields=(0, 1, 2, 4, 5)):
    """A copy of `batch` with transition b's observations, shared observations and buffer actions drawn anew (every policy's)."""
    out = [dict(d) if isinstance(d, dict) else d for d in batch]
    for i in fields:
        for q, v in batch[i].items():
            v = np.array(v, copy=True)
            if i == 2:                            # one-hot blocks stay one-hot; Box actions stay in (-1, 1)
                hot = v[..., b, :] > 0.5
                if np.array_equal(hot.sum(-1), np.ones(hot.shape[:-1])) and set(np.unique(v)) <= {0.0, 1.0}:
                    v[..., b, :] = np.roll(v[..., b, :], int(rng.integers(1, v.shape[-1] + 1)), -1)
                else:
                    v[..., b, :] = np.tanh(rng.standard_normal(v[..., b, :].shape)).astype(np.float32)
            elif v.ndim == 3:
                v[:, b] = rng.standard_normal(v[:, b].shape).astype(np.float32)
            else:
                v[b] = rng.standard_normal(v[b].shape).astype(np.float32)
            out[i][q] = v
    return tuple(out)


def settle(tr, L64, p, batch, checks, seed, rng, stats, slack=True):
    """Redraw transitions until every (key, row) of `checks` -- key "critic" with a transition index, "actor" with an (n, b) pair -- has a
    float64 decision margin above DECISION_MARGIN under the draws of `seed`; counts the redraws in stats["redraws"] and records the
    smallest margin kept."""
    B = np.asarray(batch[0][p]).shape[1]
    tn, an = noise_at(tr, p, B, seed)
    for _ in range(MAX_REDRAWS + 1):
        m = margins(L64, p, batch, tn, an, slack)
        low = {(r[1] if isinstance(r, tuple) else r) for key, r in checks if float(m[key][r]) <= DECISION_MARGIN}
        if not low:
            stats["min_margin"] = min([stats.get("min_margin", float("inf"))] + [float(m[key][r]) for key, r in checks])
            return batch
        for b in sorted(low):
            batch = redraw(batch, rng, b)
            stats["redraws"] = stats.get("redraws", 0) + 1
    raise AssertionError("no draw with every decision margin above %.0e after %d redraws" % (DECISION_MARGIN, MAX_REDRAWS))


# ---- tile rules of the MLP step ----------------------------------------------------------------------------------------------
def row_tiles(rules, M, in_dim, data_grad=False):
    """(kernel, rows per tile, tiles) of the backward that owns an M-row space of width in_dim on the MLP path.  No recurrence:
    k_front_bwd picks its tile height without the k_gru_wgrad extension.  At 65-128 columns the weight gradient runs on k_wgrad_tc's
    64-row chunks (after k_front_bwd_tc) -- except for a data-gradient launch (the agent-replaced copies: dX set, skip_wgrad), which
    neither tensor-core kernel takes (tc_bwd.cu mx_wgrad_tc_usable / mx_front_bwd_tc_usable).  Up to 64 and above 128 columns
    (WG_MAX_IN), and for the copies at every width: FFMA k_front_bwd, on 32-row tiles only above 128."""
    kern = "k_front_bwd" if data_grad else rules.row_kernel(in_dim)
    if kern == "k_front_bwd":
        TM = 16 * rules.front_bwd_rm(M, in_dim, False)
        return kern, TM, -(-M // TM)
    TM, nt, _ = rules.agent_rows(M, in_dim, gru_ext=False)[kern]
    return kern, TM, nt


def spaces(rules, B, N, O, cin):
    """The step's three row spaces: critic Mc = B at cin (row b), actor Ma = 2 B N at O (row (2 b + t) N + n, t = 1 the next
    observation, whose gradient is zero), agent-replaced copies Mr = N B at cin (row n B + b)."""
    return {"critic": (B,) + row_tiles(rules, B, cin), "actor": (2 * B * N,) + row_tiles(rules, 2 * B * N, O),
            "copies": (N * B,) + row_tiles(rules, N * B, cin, data_grad=True)}


def space_row(name, n, b, B, N):
    """Row of the isolated pair (agent n, transition b) in a row space."""
    return {"critic": b, "actor": 2 * b * N + n, "copies": n * B + b}[name]


def last_tile_pair(name, M, TM, nt, B, N):
    """An (n, b) whose row sits in the space's last tile: the tile's first live row (the actor's t = 1 rows carry no gradient), or
    None when the tile holds none."""
    for row in range((nt - 1) * TM, M):
        if name == "actor":
            if (row // N) % 2 == 0:
                return row % N, row // (2 * N)
        elif name == "copies":
            return row // B, row % B
        else:
            return 0, row
    return None


def edges_hit(rules, sp, B, N):
    """The edges the shape hits, counting a space's last tile only when it holds a live row."""
    hits = set()
    for name, (M, kern, TM, nt) in sp.items():
        if last_tile_pair(name, M, TM, nt, B, N) is None:
            continue
        if nt == 1:
            hits.add(name + " one tile")
        if M % TM == 1:
            hits.add(name + " tail 1")
        if M % TM == TM - 1:
            hits.add(name + " tail TM-1")
        if nt == rules.sms:
            hits.add(name + " tiles = sms")
        if nt == rules.sms + 1:
            hits.add(name + " tiles = sms+1")
    return hits


EDGE_TARGETS = ["one tile", "tail 1", "tail TM-1", "tiles = sms", "tiles = sms+1"]


def pick_batches(rules, N, O, cin, spaces_=("critic", "actor", "copies"), Bs=range(1, 9000)):
    """The cheapest batch size B per (row space, edge) whose edge tile holds a live row.  An edge that cannot occur takes the nearest
    count that does, and the note says so: a last tile of 1 or TM-1 rows in a space with an even row count (the actor's 2 B N, the copies'
    N B at even N), the actor's tails of N rows or fewer (its last N rows are next-observation rows), or a tile count the tile-height rule
    skips.  Returns [(B, [edges], note)]."""
    cands = []
    for B in Bs:
        sp = spaces(rules, B, N, O, cin)
        cands.append((B, edges_hit(rules, sp, B, N), sp))
    live = lambda c, name: last_tile_pair(name, c[2][name][0], c[2][name][2], c[2][name][3], c[0], N) is not None
    out, notes = {}, {}
    for name in spaces_:
        for e in EDGE_TARGETS:
            tgt = name + " " + e
            hit = next((c for c in cands if tgt in c[1]), None)
            if hit is None and e.startswith("tail"):
                tail = lambda c: c[2][name][0] % c[2][name][2]
                ok = [c for c in cands if live(c, name) and tail(c)]
                hit = min(ok, key=(lambda c: (tail(c), c[0])) if e == "tail 1" else (lambda c: (c[2][name][2] - tail(c), c[0])))
                notes[tgt] = "%s cannot occur (an even row count, or only next-observation rows in it); nearest: a last tile of %d of %d " \
                             "rows at B %d" % (tgt, tail(hit), hit[2][name][2], hit[0])
            elif hit is None:
                want = {"tiles = sms": rules.sms, "tiles = sms+1": rules.sms + 1}[e]
                ok = [c for c in cands if live(c, name) and c[2][name][3] >= want]
                hit = min(ok, key=lambda c: (c[2][name][3] - want, c[0]))
                notes[tgt] = "%s cannot occur (tile rule); nearest: %d tiles of %d rows at B %d" % (tgt, hit[2][name][3], hit[2][name][2], hit[0])
            out.setdefault(hit[0], []).append(tgt)
    return [(B, tg, "; ".join(notes[t] for t in tg if t in notes)) for B, tg in sorted(out.items())]


def pinned_pairs(B, N, sp):
    """[(n, b, {space: tile})]: the isolated (agent, transition) pairs of one batch and the tile each must land in.  (0, 0) pins every
    space's first tile; for each space, the first live row of its last tile; (N - 1, B - 1) the last live rows.  A space whose last tile
    holds only next-observation rows (the actor's, at a batch size picked for another space's edge) has nothing to pin there: its
    gradient partial is identically zero."""
    pairs = {(0, 0), (N - 1, B - 1)}
    live = []
    for name, (M, kern, TM, nt) in sp.items():
        pr = last_tile_pair(name, M, TM, nt, B, N)
        if pr is not None:
            pairs.add(pr)
            live.append(name)
    out = [(n, b, {name: space_row(name, n, b, B, N) // TM for name, (M, kern, TM, nt) in sp.items()}) for n, b in sorted(pairs)]
    for name in live:                   # every live last tile is pinned by one of the pairs
        assert any(t[name] == sp[name][3] - 1 for _, _, t in out), (name, "last tile not pinned", B)
    return out


def owner_launches(names):
    """The launches of one MLP step grouped by the row space they serve, from their order in maddpg_step_mlp: the critic backward
    between the critic's k_mlp_dgi_cols and its optimiser, the copies' between the actor's k_mlp_dgi_cols and k_scatter_actor_grad, the
    actor's between k_scatter_actor_grad and the actor's optimiser."""
    d = [i for i, k in enumerate(names) if k == "k_mlp_dgi_cols"]
    sc = names.index("k_scatter_actor_grad")
    red = [i for i, k in enumerate(names) if k == "k_grad_reduce"]
    assert len(d) == 2 and len(red) == 2 and d[0] < red[0] < d[1] < sc < red[1], names
    return {"critic": names[d[0] + 1:red[0]], "copies": names[d[1] + 1:sc], "actor": names[sc + 1:red[1]]}


def forward_launches(names):
    """The forward launches of one MLP step by the nets they run: a critic forward (live and target on the buffer rows, live on the
    agent-replaced copies) directly follows the k_pack_critic_in that built its input; every other k_front_fwd* launch is an actor's."""
    out = {"critic": [], "actor": []}
    after_pack = False
    for k in names:
        if k.startswith("k_front_fwd"):
            out["critic" if after_pack else "actor"].append(k)
        else:
            after_pack = k == "k_pack_critic_in"
    return out


# above WG_MAX_IN (128) input columns every net runs FFMA: k_front_fwd<2> forward (no tensor-core image), k_front_bwd backward
TC_KERNELS = ("k_front_fwd_tc", "k_front_fwd_tc1", "k_front_fwd_tc_wide", "k_front_bwd_tc", "k_wgrad_tc", "k_tc_prep_weights_T")


def assert_row_kernels(names, sp, n_policies=1, widths=None):
    """Each space's row kernel ran in the launch that owns that space; the copies' backward is exactly one k_front_bwd; every policy's
    cent_contribute ran (k_cent_scatter) when there are several.  widths {"critic": cin, "actor": obs}: a net above 128 columns ran
    only k_front_fwd forwards and only k_front_bwd in each of its spaces' own launches."""
    own = owner_launches(names)
    for name, (M, kern, TM, nt) in sp.items():
        assert kern in own[name], (name, kern, "did not run in its own launch", own[name])
    assert own["copies"] == ["k_front_bwd"], own["copies"]
    fwd = forward_launches(names)
    for net, w in (widths or {}).items():
        if w <= 128:
            continue
        assert fwd[net] and set(fwd[net]) == {"k_front_fwd"}, (net, w, "forward launches", fwd[net], names)
        for name in ("critic", "copies") if net == "critic" else ("actor",):
            assert own[name] == ["k_front_bwd"], (name, w, "backward launches", own[name])
        assert not any(k in TC_KERNELS for k in own["critic" if net == "critic" else "actor"]), (net, own)
    for k in ("k_mlp_head_cols", "k_critic_loss", "k_actor_loss", "k_pack_critic_in"):
        assert k in names, (k, "did not run")
    if n_policies > 1:
        assert names.count("k_cent_scatter") == n_policies, names


# ---- the checks -------------------------------------------------------------------------------------------------------------------
def grad_errs(ours, ref, tol, tag):
    """{tensor: max |engine - float64| / max |float64|} per tensor, asserted against tol; a tensor whose float64 gradient is exactly zero
    (fc_h, in no forward pass) must be exactly zero."""
    errs, bad = {}, []
    for net, d in ref.items():
        for k, r in d.items():
            r = r.detach().double()
            o = ours[net][k].reshape(r.shape)
            diff, scale = float((o - r).abs().max()), float(r.abs().max())
            if scale == 0.0:
                assert diff == 0.0, (tag, net, k, "gradient where the float64 one is exactly zero", diff)
                continue
            errs[net + "." + k] = diff / scale
            if diff > tol * scale:
                bad.append("%s %s.%s: err %.3e > %.1e x max|ref| %.3e" % (tag, net, k, diff, tol, scale))
    assert not bad, "\n".join(bad)
    return errs


def fp32_oracle_error(L32, L64, p, batch, tn, an):
    """The fp32 oracle's worst relative gradient error against float64 on `batch` (its conditioning, FP32_COND_SHARE).  Both steps run on
    copies, so neither oracle's Adam state moves."""
    import copy
    _, _, g32 = step_multi_md(copy.deepcopy(L32), p, batch, tn, an, dtype=torch.float32)
    _, _, g64 = step_multi_md(copy.deepcopy(L64), p, batch, tn, an, dtype=torch.float64)
    worst = 0.0
    for net, d in g64.items():
        for k, r in d.items():
            scale = float(r.detach().abs().max())
            if scale > 0.0:
                worst = max(worst, float((g32[net][k].detach().double() - r.detach()).abs().max()) / scale)
    return worst


def isolated(tr, pols, L64, p, batch, pairs, sp, seed, rng, stats, tol=GRAD_TOL, L32=None):
    """For each (n, b, tiles) of `pairs` (pinned_pairs): one engine step of policy p with PER weights one-hot on b and valid_transition
    one-hot on (n, b), against the float64 step: every critic and actor tensor within tol x max|ref|, and the isolated copy's actor_loss
    within ROW_TOL of its scale; the decisions settled first.  The pair's critic, actor and copy rows must sit in `tiles`.  Returns the
    worst relative error per tensor."""
    B = np.asarray(batch[0][p]).shape[1]
    Np = np.asarray(batch[0][p]).shape[0]
    worst = {}
    cond = pols[p].central_obs_dim + pols[p].central_act_dim > FP32_COND_MIN_CRITIC
    if cond and L32 is None:
        L32 = oracles64(tr.args, pols, torch.float32)
    stats.setdefault("ill_conditioned", 0)
    for i, (n, b, tiles) in enumerate(pairs):
        for name, t in tiles.items():
            assert space_row(name, n, b, B, Np) // sp[name][2] == t, (name, n, b, t)
        s = seed + 17 * i
        for _ in range(MAX_REDRAWS + 1):
            bt = settle(tr, L64, p, batch, [("critic", b), ("actor", (n, b))], s, rng, stats)
            bt = far_td_error(L64, p, bt, b, *noise_at(tr, p, B, s))
            w = np.zeros(B, np.float32)
            w[b] = 1.0
            valid = {q: np.array(v, copy=True) for q, v in bt[8].items()}
            valid[p][:] = 0.0
            valid[p][n, b] = 1.0
            bt = tuple(bt[:8]) + (valid,) + tuple(bt[9:11]) + (w, np.arange(B))
            if not cond or fp32_oracle_error(L32, L64, p, bt, *noise_at(tr, p, B, s)) <= FP32_COND_SHARE * tol:
                break
            batch = redraw(batch, rng, b)
            stats["redraws"] = stats.get("redraws", 0) + 1
            stats["ill_conditioned"] += 1
        else:
            raise AssertionError("transition %d: no draw the fp32 oracle gets within %.0e of float64" % (b, FP32_COND_SHARE * tol))
        qscale = float(margins(L64, p, bt, *noise_at(tr, p, B, s))["qscale"][n, b])
        info, _, ref, _, grads = step_both(tr, L64, p, bt, s)
        errs = grad_errs(mc.engine_grads(tr, pols[p], p), grads, tol, "transition %d (agent %d) of %d" % (b, n, B))
        d = abs(float(info["actor_loss"]) - ref["actor_loss"])
        assert d <= ROW_TOL * qscale, ("actor_loss of copy (%d, %d)" % (n, b), float(info["actor_loss"]), ref["actor_loss"], qscale)
        errs["actor_loss"] = d / qscale
        for k, v in errs.items():
            worst[k] = max(worst.get(k, 0.0), v)
    return worst


def far_td_error(L64, p, batch, b, tn, an):
    """Transition b's reward set so that y sits qmag above every head's Q (qmag: the round-off scale of its TD errors, margins).  One
    transition's critic gradient is its TD errors times d Q / d theta; an error y - Q_k that nearly cancels carries a relative fp32 error
    of ulps(qmag) / |y - Q_k| into every critic tensor (measured 2e-5 to 1e-4 on an H100), which is the TD error's precision, checked by
    per_transition_forward, not the row's."""
    m = margins(L64, p, batch, tn, an)
    rew = {q: np.array(v, copy=True) for q, v in batch[3].items()}
    rew[p][:, b] += np.float32(m["qmax"][b] - m["y"][b] + 2.0 * m["qmag"][b])
    return tuple(batch[:3]) + (rew,) + tuple(batch[4:])


def per_transition_forward(tr, L64, p, batch, seed, rng, stats):
    """PER weights all 1: every transition's priority (mean over the K heads of |y - Q_k|, + per_eps) within TD_ULPS fp32 ulps of the
    float64 one, ulps of the TD errors' round-off scale ("qmag" of margins: the heads' sum_j |w_j h_j| + |b|, not |Q|, which cancellation
    in the 64-term head dot product can make small -- measured up to 32 ulps of max(|Q|, |y|) on the emulator at simple_spread's shapes).
    The arg-max / Gumbel target actions of every transition are settled first (the forward value is continuous in everything else).
    Returns the worst error in ulps."""
    B = np.asarray(batch[0][p]).shape[1]
    tn, an = noise_at(tr, p, B, seed)
    for _ in range(MAX_REDRAWS + 1):
        gap = margins(L64, p, batch, tn, an)["target"]
        low = [b for b in range(B) if float(gap[b]) <= DECISION_MARGIN]
        if not low:
            break
        for b in low:
            batch = redraw(batch, rng, b, fields=(4, 5))
            stats["redraws"] = stats.get("redraws", 0) + 1
    else:
        raise AssertionError("target actions: no draw with every gap above %.0e" % DECISION_MARGIN)
    bt = tuple(batch[:11]) + (np.ones(B, np.float32), np.arange(B))
    _, prio, _, rprio, _ = step_both(tr, L64, p, bt, seed)
    scale = margins(L64, p, bt, *noise_at(tr, p, B, seed))["qmag"].numpy()
    ulps = np.abs(np.asarray(prio, dtype=np.float64) - rprio) / (2.0 ** -23 * scale)
    bad = np.nonzero(ulps > TD_ULPS)[0]
    assert bad.size == 0, ("priorities off float64 by more than %d ulps of their scale" % TD_ULPS, [(int(b), float(ulps[b])) for b in bad[:8]])
    return float(ulps.max())


def batch_size_sequence(args, tr, pols, L64, p, make, Bs, seed, rng, stats, rules, engine, stream=None, tol=GRAD_TOL, param_tol=5e-3):
    """Steps of policy p at the batch sizes Bs on ONE learner (max_batch = Bs[0]), each against the float64 step: every clipped gradient
    tensor, the losses, the priorities, the parameters after Adam and the targets after the soft update; each space's row kernel in the
    launch that owns it (tile rules `rules`).  Every decision of every row
    is settled first (not the softmax slack of an isolated row: one saturated row among thousands moves no tensor by a measurable share).
    Returns the worst relative gradient error."""
    worst = 0.0
    for s, B in enumerate(Bs):
        batch = make(B)
        N = np.asarray(batch[0][p]).shape[0]
        batch = settle(tr, L64, p, batch, [("critic", b) for b in range(B)] + [("actor", (n, b)) for n in range(N) for b in range(B)],
                       seed + s, rng, stats, slack=False)
        res = []
        names = kernels_run(engine.lib(), stream, lambda: res.append(step_both(tr, L64, p, batch, seed + s)))
        pol = pols[p]
        cin = pol.central_obs_dim + pol.central_act_dim
        assert_row_kernels(names, spaces(rules, B, N, pol.obs_dim, cin), len(pols), {"critic": cin, "actor": pol.obs_dim})
        info, prio, ref, rprio, grads = res[0]
        errs = grad_errs(mc.clipped_engine_grads(tr, pols[p], ref, args.max_grad_norm, p), grads, tol, "step %d at B = %d" % (s, B))
        worst = max([worst] + list(errs.values()))
        for k in ("critic_loss", "critic_grad_norm", "actor_loss", "actor_grad_norm"):
            assert abs(float(info[k]) - ref[k]) <= tol * max(1.0, abs(ref[k])), (s, B, k, float(info[k]), ref[k])
        if rprio is not None:
            assert np.abs(np.asarray(prio) - rprio).max() <= 1e-4 * max(1.0, np.abs(rprio).max()), (s, B, "priorities")
        for q in sorted(pols):
            pols[q].soft_target_updates()
            L64[q].soft_update()
        pol, L = pols[p], L64[p]
        for mod, ref_sd, lim in ((pol.actor, L.actor, param_tol * args.lr * (s + 1) + 1e-7), (pol.critic, L.critic, param_tol * args.lr * (s + 1) + 1e-7),
                                 (pol.target_actor, L.target_actor, 1e-6), (pol.target_critic, L.target_critic, 1e-6)):
            for k, v in mod.state_dict().items():
                d = float((v.cpu().double() - ref_sd[k].detach()).abs().max())
                assert d <= lim, (s, B, k, d)
    return worst


def make_batches(specs, S, discrete, avail=False):
    """B -> a batch of every policy in `specs` (PER weights in [0.2, 1.2)), Box or Discrete (mlp_maddpg_multi_checks) or with
    MultiDiscrete policies (mlp_maddpg_md_checks)."""
    import mlp_maddpg_multi_checks as mmc
    md = any(isinstance(s[1], (list, tuple)) for s in specs)
    rng = np.random.default_rng(zlib.crc32(repr((specs, S, discrete, avail)).encode()))
    if md:
        return lambda B: mdc.synth_batch_md(rng, specs, B, S, per=True)
    return lambda B: mmc.synth_batch_multi(rng, specs, B, S, discrete, avail=avail, per=True)


def geometry(specs, S, p):
    """(N_p, obs width of p, critic input width S + sum of every policy's action width)."""
    norm = mdc.norm_specs(specs)
    o, a, n = norm[p]
    return n, o, S + sum(mdc.width(aq) * nq for _, aq, nq in norm.values())


def run_case(engine, stream, rules, specs, S, discrete, td3, Bs, p="policy_0", avail=False, seed=3, **over):
    """Isolated transitions and the per-transition forward of policy p at each batch size of Bs (one learner, max_batch = max(Bs)),
    the pairs whose rows sit in each row space's last tile isolated; asserts that each space's row kernel ran in the launch that owns it.
    Returns (worst per check, stats)."""
    args, pols, tr, L64 = build_pair(specs, S, max(Bs), discrete, td3, seed=seed, use_per=True, lr=0.0, **over)
    make = make_batches(specs, S, discrete, avail)
    rng = np.random.default_rng(seed)
    N, O, cin = geometry(specs, S, p)
    worst, stats = {"grad": 0.0, "actor_loss": 0.0, "td_ulps": 0.0}, {"redraws": 0}
    for B in Bs:
        batch = make(B)
        sp = spaces(rules, B, N, O, cin)
        pairs = pinned_pairs(B, N, sp)
        ulps = []
        names = kernels_run(engine.lib(), stream, lambda: ulps.append(per_transition_forward(tr, L64, p, batch, seed + B, rng, stats)))
        worst["td_ulps"] = max(worst["td_ulps"], ulps[0])
        assert_row_kernels(names, sp, len(pols), {"critic": cin, "actor": O})
        if discrete:
            assert "k_act_transform" in names
        errs = isolated(tr, pols, L64, p, batch, pairs, sp, seed + 7 * B, rng, stats)
        worst["actor_loss"] = max(worst["actor_loss"], errs.pop("actor_loss"))
        worst["grad"] = max([worst["grad"]] + list(errs.values()))
    return worst, stats
