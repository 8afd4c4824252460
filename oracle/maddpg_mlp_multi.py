"""CPU restatement of the transition-level MADDPG / MATD3 update with several policies (share_policy off; reference:
offpolicy/algorithms/maddpg/maddpg.py:38-249, get_update_info + shared_train_policy_on_batch), built on the single-policy `MlpMaddpg`
objects of oracle/maddpg_mlp.py: one per policy, each with its own observation / action widths.

The update of policy p:
- `cent_nact` is every policy's target-actor next action, in sorted-id order, each policy's agents in order (maddpg.py:55-79);
- `cent_act` is every policy's buffer actions in the same order;
- the critic target and loss use p's rewards, dones_env, shared observation and PER weights (maddpg.py:103-107);
- the actor loss replaces p's agents at `replace_ind_start` one at a time and is masked by p's valid_transition (maddpg.py:169-232).
"""
import numpy as np
import torch

from oracle.maddpg_mlp import gumbel_hard, onehot_from_logits


def _f(x, dtype=torch.float32):
    return None if x is None else torch.as_tensor(np.asarray(x)).to(dtype)


def step_multi(learners, update_id, batch, target_noise, actor_noise=None, dtype=torch.float32):
    """One shared_train_policy_on_batch(update_id, batch).  learners: {policy_id: MlpMaddpg}, all built with `dtype`; batch: the 13-tuple
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
            nav = None if nav is None else nav.reshape(Nq * B, -1)
            if Lq.discrete:
                nact = gumbel_hard(out, f(target_noise[q]), nav) if Lq.td3 else onehot_from_logits(out, nav)
            else:
                nact = out + f(target_noise[q]) if Lq.td3 else out
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
    g = lambda d: {k: v.grad.clone() if v.grad is not None else torch.zeros_like(v) for k, v in d.items()}
    grads = {"critic": g(L.critic)}
    L.critic_opt.step()
    # actor update, every call (maddpg.py:100, 162-247)
    ob = f(obs[p])
    Np, B = ob.shape[0], ob.shape[1]
    out = L.actor_out(L.actor, ob.reshape(Np * B, -1))
    av = opt(avail, p)
    pol = gumbel_hard(out, actor_noise, None if av is None else av.reshape(Np * B, -1)) if L.discrete else out
    pol = pol.split(B, 0)
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


def draw_noise_multi(shapes, update_id, B):
    """The torch CPU draws of one update of policy `update_id`, in the reference's order: every policy's target draw in sorted-id order
    (get_update_info, maddpg.py:71: Gumbel for Discrete MATD3, N(0, std) for Box MATD3, nothing for MADDPG), then the updated policy's
    actor Gumbel draw (maddpg.py:209, Discrete only).  shapes: {policy_id: (n_agents, act_dim, discrete, td3, target_std)}.
    Returns ({policy_id: (N_q*B, A_q) or None}, (N_p*B, A_p) or None)."""
    gumbel = lambda n, a: -torch.log(-torch.log(torch.empty(n * B, a).uniform_() + 1e-20) + 1e-20)     # util.py:178-181
    tn = {}
    for q in sorted(shapes):
        n, a, discrete, td3, std = shapes[q]
        tn[q] = (gumbel(n, a) if discrete else torch.empty(n * B, a).normal_(mean=0, std=float(std))) if td3 else None
    n, a, discrete, _, _ = shapes[update_id]
    return tn, (gumbel(n, a) if discrete else None)
