"""CPU restatement of the transition-level MADDPG / MATD3 update (reference: offpolicy/algorithms/maddpg/maddpg.py:90-249,
maddpg/algorithm/{MADDPGPolicy.py, actor_critic.py}, algorithms/utils/{mlp.py, act.py}, utils/util.py) for one shared policy.

`MlpMaddpg` holds the live / target actor and critic as plain fp32 tensors plus the two frozen head sets, runs one update on a batch in
the reference's NumPy layout with the noise draws handed in, and applies the soft / hard target updates.  It is the yardstick the
engine tests compare against where the reference checkout is absent.
"""
import numpy as np
import torch
import torch.nn.functional as F

H = 64


def _mlp(p, x, relu=True, feature_norm=True):
    """MLPBase.forward (mlp.py:77-89, layer_N = 1): [LayerNorm] -> fc1 (Linear, act, LayerNorm) -> fc2[0] (same)."""
    act = torch.relu if relu else torch.tanh
    if feature_norm:
        x = F.layer_norm(x, x.shape[-1:], p["mlp.feature_norm.weight"], p["mlp.feature_norm.bias"])
    x = F.layer_norm(act(F.linear(x, p["mlp.mlp.fc1.0.weight"], p["mlp.mlp.fc1.0.bias"])), (H,), p["mlp.mlp.fc1.2.weight"], p["mlp.mlp.fc1.2.bias"])
    return F.layer_norm(act(F.linear(x, p["mlp.mlp.fc2.0.0.weight"], p["mlp.mlp.fc2.0.0.bias"])), (H,), p["mlp.mlp.fc2.0.2.weight"],
                        p["mlp.mlp.fc2.0.2.bias"])


def onehot_from_logits(logits, avail=None):
    """util.py:156-170 (eps = 0): every maximal logit is hot."""
    logits = logits.clone()
    if avail is not None:
        logits[avail == 0] = -1e10
    return (logits == logits.max(-1, keepdim=True)[0]).to(logits.dtype)


def gumbel_hard(logits, g, avail=None):
    """util.py:184-215, hard = True, temperature 1, with the Gumbel draw g handed in."""
    y = logits + g
    if avail is not None:
        y = y.masked_fill(avail == 0, -1e10)
    y = F.softmax(y, dim=-1)
    return (onehot_from_logits(y) - y).detach() + y


class MlpMaddpg(object):
    def __init__(self, actor, critic, heads, target_actor, target_critic, target_heads, discrete, td3, gamma=0.99, lr=7e-4, eps=1e-5,
                 weight_decay=0.0, max_grad_norm=10.0, tau=0.005, huber=False, huber_delta=10.0, use_per=False, per_eps=1e-6, relu=True,
                 feature_norm=True, dtype=torch.float32):
        """actor / critic / target_*: {reference key: tensor}; heads / target_heads: {"q_outs.k.weight" / ".bias": tensor}.  dtype: of
        every tensor of the update (float64 for the row-coverage checks: batch, nets, heads, Adam, clip and Polyak all in float64)."""
        self.dtype = dtype
        t = lambda d, g: {k: torch.as_tensor(v).to(dtype).detach().clone().requires_grad_(g) for k, v in d.items()}
        self.actor, self.critic = t(actor, True), t(critic, True)
        self.target_actor, self.target_critic = t(target_actor, False), t(target_critic, False)
        self.heads, self.target_heads = t(heads, False), t(target_heads, False)
        self.K = len(self.heads) // 2
        self.discrete, self.td3 = discrete, td3
        self.gamma, self.huber, self.huber_delta, self.use_per, self.per_eps = gamma, huber, huber_delta, use_per, per_eps
        self.max_grad_norm, self.tau, self.relu, self.feature_norm = max_grad_norm, tau, relu, feature_norm
        # MADDPGPolicy.py:53-55: Adam over actor.parameters() / critic.parameters() -- the heads are not among them
        self.actor_opt = torch.optim.Adam(list(self.actor.values()), lr=lr, eps=eps, weight_decay=weight_decay)
        self.critic_opt = torch.optim.Adam(list(self.critic.values()), lr=lr, eps=eps, weight_decay=weight_decay)

    def actor_out(self, p, obs):
        return F.linear(_mlp(p, obs, self.relu, self.feature_norm), p["act.action_out.weight"], p["act.action_out.bias"])

    def q(self, p, heads, x):
        h = _mlp(p, x, self.relu, self.feature_norm)
        return [F.linear(h, heads["q_outs.%d.weight" % k], heads["q_outs.%d.bias" % k]) for k in range(self.K)]

    def step(self, batch, target_noise=None, actor_noise=None):
        """One shared_train_policy_on_batch of policy_0.  batch: the 13-tuple of mlp_buffer.py (policy_0 entries); target_noise /
        actor_noise: the (N*B, A) draws the reference makes in get_update_info (MATD3) and in the actor update (Discrete)."""
        obs, share, acts, rew, nobs, nshare, _dones, dones_env, valid, avail, navail, weights, _idx = batch
        f = lambda x: None if x is None else torch.as_tensor(np.asarray(x)).to(self.dtype)
        p = "policy_0"
        target_noise, actor_noise = f(target_noise), f(actor_noise)
        obs, nobs, acts = f(obs[p]), f(nobs[p]), f(acts[p])                 # (N, B, .)
        N, B = obs.shape[0], obs.shape[1]
        av = f(avail[p]) if avail is not None and avail[p] is not None else None
        nav = f(navail[p]) if navail is not None and navail[p] is not None else None
        cat = lambda x: x.reshape(N * B, -1)                                 # np.concatenate(x, axis=0): agent-major rows
        info = {}
        with torch.no_grad():                                                # maddpg.py:64-74: target actor on next_obs
            out = self.actor_out(self.target_actor, cat(nobs))
            if self.discrete:
                nact = gumbel_hard(out, target_noise, None if nav is None else cat(nav)) if self.td3 else \
                    onehot_from_logits(out, None if nav is None else cat(nav))
            else:
                nact = out + target_noise if self.td3 else out
            cent_nact = torch.cat(nact.split(B, 0), -1)
            qn = torch.cat(self.q(self.target_critic, self.target_heads, torch.cat([f(nshare[p]), cent_nact], 1)), -1).min(-1, keepdim=True)[0]
            y = f(rew[p])[0].view(-1, 1) + self.gamma * (1 - f(dones_env[p]).view(-1, 1)) * qn           # maddpg.py:119-126
        cent_act = torch.cat(list(acts), -1)
        qs = self.q(self.critic, self.heads, torch.cat([f(share[p]), cent_act], 1))
        errors = [y - q for q in qs]
        loss_fn = (lambda e: torch.where(e.abs() <= self.huber_delta, 0.5 * e ** 2, self.huber_delta * (e.abs() - 0.5 * self.huber_delta))) \
            if self.huber else (lambda e: e ** 2)
        if self.use_per:                                                     # maddpg.py:134-144
            w = f(weights)
            critic_loss = torch.stack([(loss_fn(e).flatten() * w).mean() for e in errors]).sum(0)
            prio = np.stack([e.abs().detach().numpy().flatten() for e in errors]).mean(axis=0) + self.per_eps
        else:
            critic_loss = torch.stack([loss_fn(e).mean() for e in errors]).sum(0)
            prio = None
        self.critic_opt.zero_grad()
        critic_loss.backward()
        info["critic_loss"] = float(critic_loss.detach())
        info["critic_grad_norm"] = float(torch.nn.utils.clip_grad_norm_(list(self.critic.values()), self.max_grad_norm))
        g = lambda d: {k: v.grad.clone() if v.grad is not None else torch.zeros_like(v) for k, v in d.items()}     # fc_h: unused, no grad
        grads = {"critic": g(self.critic)}
        self.critic_opt.step()
        # actor update, every call (maddpg.py:100, 162-247: num_updates is never incremented)
        out = self.actor_out(self.actor, cat(obs))
        if self.discrete:
            pol = gumbel_hard(out, actor_noise, None if av is None else cat(av))
        else:
            pol = out
        pol = pol.split(B, 0)
        rows = []
        for i in range(N):                                                   # the N agent-replaced copies, maddpg.py:183-227
            rows.append(torch.cat([pol[j] if j == i else acts[j] for j in range(N)], -1))
        frozen = {k: v.detach() for k, v in self.critic.items()}
        qa = self.q(frozen, self.heads, torch.cat([f(share[p]).repeat(N, 1), torch.cat(rows, 0)], 1))[0]
        vmask = f(valid[p]).reshape(N * B, 1)
        actor_loss = -(qa * vmask).sum() / vmask.sum()
        self.actor_opt.zero_grad()
        actor_loss.backward()
        info["actor_loss"] = float(actor_loss.detach())
        info["actor_grad_norm"] = float(torch.nn.utils.clip_grad_norm_(list(self.actor.values()), self.max_grad_norm))
        grads["actor"] = g(self.actor)
        self.actor_opt.step()
        return info, prio, grads

    def soft_update(self):
        """MADDPGPolicy.py:141-145 (util.py:123-134): the critic trunk and the actor; the heads are not parameters."""
        with torch.no_grad():
            for tgt, src in ((self.target_critic, self.critic), (self.target_actor, self.actor)):
                for k in tgt:
                    tgt[k].copy_(tgt[k] * (1.0 - self.tau) + src[k] * self.tau)

    def hard_update(self):
        with torch.no_grad():
            for tgt, src in ((self.target_critic, self.critic), (self.target_actor, self.actor)):
                for k in tgt:
                    tgt[k].copy_(src[k])


def draw_noise(N, B, A, discrete, td3, target_std):
    """The torch CPU draws one update of the reference makes, in its order: the target policy's (maddpg.py:71 -> MADDPGPolicy.py:93-94
    Gumbel for Discrete MATD3, :111-113 N(0, std) for Box MATD3), then the actor's Gumbel draw (maddpg.py:209, Discrete only).
    Returns (target_noise or None, actor_noise or None), each (N*B, A) in agent-major rows."""
    gumbel = lambda: -torch.log(-torch.log(torch.empty(N * B, A).uniform_() + 1e-20) + 1e-20)          # util.py:178-181
    tn = (gumbel() if discrete else torch.empty(N * B, A).normal_(mean=0, std=float(target_std))) if td3 else None
    an = gumbel() if discrete else None
    return tn, an
