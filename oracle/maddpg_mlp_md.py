"""CPU restatement of the transition-level MADDPG / MATD3 update for MultiDiscrete action spaces (reference:
offpolicy/algorithms/maddpg/maddpg.py:38-249, maddpg/algorithm/MADDPGPolicy.py:63-129, algorithms/utils/act.py:15-29), on top of the
`MlpMaddpg` objects of oracle/maddpg_mlp.py.

A MultiDiscrete action (e.g. simple_reference: move Discrete(5) and speak Discrete(10)) is one one-hot block per sub-space, `segs` their
widths.  The actor has one head `act.action_outs.i` per sub-space; the target actions are the arg-max one-hot (MADDPG) or the hard
Gumbel-softmax (MATD3) of each block on its own, the actor update's action the hard Gumbel-softmax of each block, and the available-action
masks are ignored (MADDPGPolicy.py:73-89).  Every Gumbel draw is one call per sub-space, in sub-space order.  The critic sees the blocks
as plain columns.

`step_multi_md` is the update of one policy among several (share_policy off), as oracle/maddpg_mlp_multi.py; a single shared policy is
the case of one learner (`MlpMaddpgMD.step`).  Learners with `segs=None` are plain Box / Discrete policies, so Discrete and MultiDiscrete
policies can be mixed.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle.maddpg_mlp import MlpMaddpg, _mlp, gumbel_hard, onehot_from_logits


def _blocks(x, segs):
    return x.split(list(segs), -1)


def onehot_blocks(logits, avail=None, segs=None):
    """onehot_from_logits on the whole row (util.py:106-118), or on each block of `segs` with no mask (MADDPGPolicy.py:87-88)."""
    if segs is None:
        return onehot_from_logits(logits, avail)
    return torch.cat([onehot_from_logits(x) for x in _blocks(logits, segs)], -1)


def gumbel_hard_blocks(logits, g, avail=None, segs=None):
    """gumbel_hard on the whole row (util.py:184-215), or on each block of `segs`: its own softmax, no mask (MADDPGPolicy.py:74-76)."""
    if segs is None:
        return gumbel_hard(logits, g, avail)
    return torch.cat([gumbel_hard(x, gx) for x, gx in zip(_blocks(logits, segs), _blocks(g, segs))], -1)


class MlpMaddpgMD(MlpMaddpg):
    def __init__(self, *a, segs=None, **k):
        """As MlpMaddpg; segs: the MultiDiscrete sub-space widths, or None (Box / Discrete)."""
        MlpMaddpg.__init__(self, *a, **k)
        self.segs = None if segs is None else [int(n) for n in segs]

    def actor_out(self, p, obs):
        if self.segs is None:
            return MlpMaddpg.actor_out(self, p, obs)
        h = _mlp(p, obs, self.relu, self.feature_norm)           # act.py:26-29: the sub-space heads' outputs side by side
        return torch.cat([F.linear(h, p["act.action_outs.%d.weight" % i], p["act.action_outs.%d.bias" % i]) for i in range(len(self.segs))], -1)

    def act_target(self, out, noise, navail):
        """get_actions(nobs, navail, use_target=True) from the target actor's outputs (maddpg.py:71)."""
        if self.discrete:
            return gumbel_hard_blocks(out, noise, navail, self.segs) if self.td3 else onehot_blocks(out, navail, self.segs)
        return out + noise if self.td3 else out

    def act_live(self, out, noise, avail):
        """get_actions(obs, avail, use_gumbel=True) from the live actor's outputs (maddpg.py:209)."""
        return gumbel_hard_blocks(out, noise, avail, self.segs) if self.discrete else out

    def step(self, batch, target_noise=None, actor_noise=None):
        """One shared_train_policy_on_batch of policy_0, the only policy (as MlpMaddpg.step)."""
        return step_multi_md({"policy_0": self}, "policy_0", batch, {"policy_0": target_noise}, actor_noise, dtype=self.dtype)


def _f(x, dtype=torch.float32):
    return None if x is None else torch.as_tensor(np.asarray(x)).to(dtype)


def step_multi_md(learners, update_id, batch, target_noise, actor_noise=None, dtype=torch.float32):
    """One shared_train_policy_on_batch(update_id, batch).  learners: {policy_id: MlpMaddpgMD}, all built with `dtype`; batch: the 13-tuple
    of mlp_buffer.py with an entry per policy; target_noise: {policy_id: (N_q*B, A_q) draw or None}; actor_noise: p's (N_p*B, A_p) Gumbel
    draw or None.  Returns (train_info, priorities or None, clipped gradients)."""
    obs, share, acts, rew, nobs, nshare, _dones, dones_env, valid, avail, navail, weights, _idx = batch
    f = lambda x: _f(x, dtype)
    actor_noise = f(actor_noise)
    ids = sorted(learners)
    p = update_id
    L = learners[p]
    opt = lambda d, q: None if d is None or d.get(q) is None else f(d[q])
    cent_act, cent_nact, start, ind = [], [], None, 0
    with torch.no_grad():
        for q in ids:                                                         # maddpg.py:56-76
            Lq = learners[q]
            nob = f(nobs[q])
            Nq, B = nob.shape[0], nob.shape[1]
            if q == p:
                start = ind
            cent_act.extend(list(f(acts[q])))
            nav = opt(navail, q)
            out = Lq.actor_out(Lq.target_actor, nob.reshape(Nq * B, -1))
            nact = Lq.act_target(out, f(target_noise[q]), None if nav is None else nav.reshape(Nq * B, -1))
            cent_nact.append(torch.cat(nact.split(B, 0), -1))
            ind += Nq
        cent_nact = torch.cat(cent_nact, -1)
        qn = torch.cat(L.q(L.target_critic, L.target_heads, torch.cat([f(nshare[p]), cent_nact], 1)), -1).min(-1, keepdim=True)[0]
        y = f(rew[p])[0].view(-1, 1) + L.gamma * (1 - f(dones_env[p]).view(-1, 1)) * qn           # maddpg.py:113-126
    info = {}
    qs = L.q(L.critic, L.heads, torch.cat([f(share[p]), torch.cat(cent_act, -1)], 1))
    errors = [y - q for q in qs]
    loss_fn = (lambda e: torch.where(e.abs() <= L.huber_delta, 0.5 * e ** 2, L.huber_delta * (e.abs() - 0.5 * L.huber_delta))) \
        if L.huber else (lambda e: e ** 2)
    if L.use_per:                                                             # maddpg.py:134-144
        w = f(weights)
        critic_loss = torch.stack([(loss_fn(e).flatten() * w).mean() for e in errors]).sum(0)
        prio = np.stack([e.abs().detach().numpy().flatten() for e in errors]).mean(axis=0) + L.per_eps
    else:
        critic_loss = torch.stack([loss_fn(e).mean() for e in errors]).sum(0)
        prio = None
    L.critic_opt.zero_grad()
    critic_loss.backward()
    info["critic_loss"] = float(critic_loss.detach())
    info["critic_grad_norm"] = float(torch.nn.utils.clip_grad_norm_(list(L.critic.values()), L.max_grad_norm))
    g = lambda d: {k: v.grad.clone() if v.grad is not None else torch.zeros_like(v) for k, v in d.items()}     # fc_h: unused, no grad
    grads = {"critic": g(L.critic)}
    L.critic_opt.step()
    # actor update, every call (maddpg.py:100, 162-247: num_updates is never incremented)
    ob = f(obs[p])
    Np, B = ob.shape[0], ob.shape[1]
    out = L.actor_out(L.actor, ob.reshape(Np * B, -1))
    av = opt(avail, p)
    pol = L.act_live(out, actor_noise, None if av is None else av.reshape(Np * B, -1)).split(B, 0)
    rows = []
    for i in range(Np):                                                       # maddpg.py:183-227: agent replace_ind_start + i replaced
        rows.append(torch.cat([pol[i] if j == start + i else cent_act[j] for j in range(len(cent_act))], -1))
    frozen = {k: v.detach() for k, v in L.critic.items()}
    qa = L.q(frozen, L.heads, torch.cat([f(share[p]).repeat(Np, 1), torch.cat(rows, 0)], 1))[0]
    vmask = f(valid[p]).reshape(Np * B, 1)
    actor_loss = -(qa * vmask).sum() / vmask.sum()
    L.actor_opt.zero_grad()
    actor_loss.backward()
    info["actor_loss"] = float(actor_loss.detach())
    info["actor_grad_norm"] = float(torch.nn.utils.clip_grad_norm_(list(L.actor.values()), L.max_grad_norm))
    grads["actor"] = g(L.actor)
    L.actor_opt.step()
    return info, prio, grads


def _gumbel(rows, a):
    """Gumbel(0, 1) draws (util.py:178-181) for `rows` rows of an action of width a, or one call per sub-space when a is a list."""
    one = lambda n: -torch.log(-torch.log(torch.empty(rows, n).uniform_() + 1e-20) + 1e-20)
    return torch.cat([one(n) for n in a], -1) if isinstance(a, (list, tuple)) else one(a)


def draw_noise_multi_md(shapes, update_id, B):
    """The torch CPU draws of one update of policy `update_id`, in the reference's order: every policy's target draw in sorted-id order
    (get_update_info, maddpg.py:71: Gumbel for Discrete MATD3, N(0, std) for Box MATD3, nothing for MADDPG), then the updated policy's
    actor Gumbel draw (maddpg.py:209, Discrete only).  shapes: {policy_id: (n_agents, act, discrete, td3, target_std)} with act the
    action width, or the list of sub-space widths of a MultiDiscrete policy.
    Returns ({policy_id: (N_q*B, A_q) or None}, (N_p*B, A_p) or None)."""
    tn = {}
    for q in sorted(shapes):
        n, a, discrete, td3, std = shapes[q]
        tn[q] = (_gumbel(n * B, a) if discrete else torch.empty(n * B, a).normal_(mean=0, std=float(std))) if td3 else None
    n, a, discrete, _, _ = shapes[update_id]
    return tn, (_gumbel(n * B, a) if discrete else None)


def draw_noise_md(N, B, segs, td3):
    """draw_noise_multi_md for one MultiDiscrete policy: (target_noise or None, actor_noise), each (N*B, sum(segs))."""
    tn, an = draw_noise_multi_md({"policy_0": (N, list(segs), True, td3, 0.0)}, "policy_0", B)
    return tn["policy_0"], an
