"""Recurrent MADDPG / MATD3 learner step (shared centralised observation, continuous `Box` actions), restated in
CPU PyTorch (oracle; test infrastructure only).

Follows /root/reference/offpolicy/algorithms/r_maddpg/r_maddpg.py:114-331 (`shared_train_policy_on_batch`),
`get_update_info` (:44-105), the nets in r_maddpg/algorithm/r_actor_critic.py:7-130 and the policy wrapper
r_maddpg/algorithm/rMADDPGPolicy.py:11-170 (two Adams with weight_decay, Polyak on actor + critic):

  1. next actions: target actor over the full (T+1)-sequence of every agent (rows agent-major), Box actions are the raw
     output (MADDPG) or + N(0, target_noise) (MATD3, `gaussian_noise`, util.py:217-218 -- drawn by the caller from the
     torch CPU RNG exactly like the reference and handed in as `noise`); Discrete actions are the arg-max one-hot of the
     logits (MADDPG, `onehot_from_logits` util.py:106-125) or a hard Gumbel-softmax sample (MATD3, util.py:127-166;
     `noise` = the Gumbel(0,1) draws); drop t=0, concat agents on the feature axis.
  2. Q_k = critic(cent_obs[:-1], buffer cent_act) as one sequence from h0 = 0                                 (:162)
  3. target: h <- 0; for t: _, h = target_critic(obs_t, act_t, h); Q'_t = min_k target_critic(obs_{t+1}, nact_t, h)  (:168-182)
  4. y = r(agent 0) + gamma (1 - dones_env) Q'; Q_k, y masked by (1 - curr_dones) (dones_env shifted by one step);
     critic_loss = sum_k sum l(Q_k - y) / sum(1 - curr_dones); clip 10; Adam(critic)                         (:188-231)
  5. actor (every actor_update_interval updates), with the UPDATED critic: actor over obs[:-1]; N stacked copies of the
     batch, copy i has agent i's action replaced by the actor's; Q_t = critic(obs_t, replaced_t, h)[head 0] with h advanced on
     buffer actions only; actor_loss = -sum Q (1 - done_mask_i) / sum(1 - done_mask); clip 10; Adam(actor)    (:236-327)
     Discrete: the actor's actions are hard Gumbel-softmax samples with the straight-through gradient of the soft sample
     (`use_gumbel=True`, r_maddpg.py:277; `actor_noise` = the Gumbel draws of that call).
"""
import copy
from dataclasses import dataclass

import numpy as np
import torch
import torch.nn as nn

from oracle.qmix import _RNNBase, init_like_reference


@dataclass
class MaddpgConfig:
    n_agents: int = 3
    obs_dim: int = 18
    act_dim: int = 2
    state_dim: int = 54
    hidden: int = 64
    layer_n: int = 1
    feature_norm: bool = True
    relu: bool = True              # use_ReLU (store_false flag): False = tanh blocks
    gamma: float = 0.99
    lr: float = 5e-4
    opti_eps: float = 1e-5
    weight_decay: float = 0.0
    max_grad_norm: float = 10.0
    tau: float = 0.005
    huber: bool = False
    huber_delta: float = 10.0
    use_per: bool = False
    per_nu: float = 0.9
    per_eps: float = 1e-6
    td3: bool = False
    target_noise: float = 0.2
    actor_update_interval: int = 1
    gain: float = 0.01
    discrete: bool = False            # Discrete(act_dim): one-hot actions, Gumbel-softmax actor


def onehot_of_max(x, avail=None):
    """`onehot_from_logits` without exploration (util.py:106-118): every maximal entry is hot; unavailable -> -1e10."""
    if avail is not None:
        x = torch.where(avail == 0, torch.full_like(x, -1e10), x)
    return (x == x.max(dim=-1, keepdim=True)[0]).to(x.dtype)


def hard_gumbel_softmax(logits, gumbel, avail=None):
    """util.py:133-166 with temperature 1 and hard=True: value (y_hard - y) + y, gradient of the soft sample y."""
    y = logits + gumbel
    if avail is not None:
        y = torch.where(avail == 0, torch.full_like(y, -1e10), y)
    y = torch.softmax(y / 1.0, dim=-1)
    return (onehot_of_max(y) - y).detach() + y


def sample_gumbel(shape, eps=1e-20):
    """util.py:127-130: one uniform_ draw from torch's CPU generator."""
    u = torch.empty(*shape).uniform_()
    return -torch.log(-torch.log(u + eps) + eps)


class _ActHead(nn.Module):
    def __init__(self, h, a):
        super().__init__()
        self.action_out = nn.Linear(h, a)


class ActorNet(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.rnn = _RNNBase(cfg.obs_dim, cfg.hidden, cfg.layer_n, cfg.feature_norm, cfg.relu)
        self.act = _ActHead(cfg.hidden, cfg.act_dim)
        self.hidden = cfg.hidden

    def forward(self, x, h0=None):
        if h0 is None:
            h0 = torch.zeros(x.shape[1], self.hidden, dtype=x.dtype)
        y, hT = self.rnn(x, h0[None])
        return self.act.action_out(y), hT


class CriticNet(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        k = 2 if cfg.td3 else 1
        self.rnn = _RNNBase(cfg.state_dim + cfg.n_agents * cfg.act_dim, cfg.hidden, cfg.layer_n, cfg.feature_norm, cfg.relu)
        self.q_outs = nn.ModuleList([nn.Linear(cfg.hidden, 1) for _ in range(k)])
        self.hidden = cfg.hidden

    def forward(self, s, a, h0=None):
        seq = s.dim() == 3
        if not seq:
            s, a = s[None], a[None]
        if h0 is None:
            h0 = torch.zeros(s.shape[1], self.hidden, dtype=s.dtype)
        y, hT = self.rnn(torch.cat([s, a], dim=2), h0[None])
        qs = [q(y) for q in self.q_outs]
        if not seq:
            qs = [q[0] for q in qs]
        return qs, hT


class MaddpgLearner(object):
    """Batch = (obs (N,T+1,B,O), share (T+1,B,S), acts (N,T,B,Ac), rewards (N,T,B,1), dones (N,T,B,1), dones_env (T,B,1),
    avail None, weights (B,) | None, idx | None)."""

    def __init__(self, cfg, seed=1, dtype=torch.float32):
        """dtype: float32 is the reference's arithmetic; float64 runs the whole update (batch, noise, networks, both Adams, clipping,
        Polyak) in double precision from the same float32-drawn initial values (tests/row_coverage_checks.py)."""
        self.cfg = cfg
        self.dtype = dtype
        self.actor = init_like_reference(ActorNet(cfg), cfg, seed).to(dtype)
        self.critic = init_like_reference(CriticNet(cfg), cfg, seed + 1).to(dtype)
        self.sync_targets()
        kw = dict(lr=cfg.lr, eps=cfg.opti_eps, weight_decay=cfg.weight_decay)
        self.actor_opt = torch.optim.Adam(self.actor.parameters(), **kw)
        self.critic_opt = torch.optim.Adam(self.critic.parameters(), **kw)
        self.num_updates = 0

    def sync_targets(self):
        self.tgt_actor = copy.deepcopy(self.actor)
        self.tgt_critic = copy.deepcopy(self.critic)

    def stack(self, x):
        x = torch.as_tensor(x, dtype=getattr(self, "dtype", torch.float32))
        return torch.cat(list(x), dim=-2)          # (N,T,B,D) -> (T, N*B, D), row = n*B + b

    def _loss(self, e):
        if self.cfg.huber:
            d = self.cfg.huber_delta
            small = (e.abs() <= d).to(e.dtype)
            return small * e ** 2 / 2 + (1 - small) * d * (e.abs() - d / 2)
        return e ** 2

    def step(self, batch, noise=None, actor_noise=None):
        cfg = self.cfg
        obs, share, acts, rew, dones, dones_env, avail, weights, _idx = batch
        N, B, T = cfg.n_agents, obs.shape[2], acts.shape[1]
        dt = self.dtype
        t32 = lambda x: torch.as_tensor(x, dtype=dt)
        s = t32(share)
        de = t32(dones_env)
        r = t32(rew[0])
        curr = torch.cat([torch.zeros(1, B, 1, dtype=dt), de[:T - 1]], 0)
        x_all = self.stack(obs)                                        # (T+1, N*B, O)
        av_all = self.stack(avail) if (avail is not None and cfg.discrete) else None
        cent_act = torch.cat(list(t32(acts)), dim=-1)                  # (T, B, N*Ac) agents on the feature axis
        update_actor = self.num_updates % cfg.actor_update_interval == 0
        info = {}
        # 1. next actions from the target actor
        with torch.no_grad():
            nact, _ = self.tgt_actor(x_all)
            if cfg.discrete:
                nact = hard_gumbel_softmax(nact, t32(noise), av_all) if cfg.td3 else onehot_of_max(nact, av_all)
            elif cfg.td3:
                nact = nact + t32(noise)
            nact = nact[1:]
            cent_nact = torch.cat(nact.split(B, dim=1), dim=-1)        # (T, B, N*Ac)
        # 2. critic prediction
        q_seq, _ = self.critic(s[:-1], cent_act)
        # 3. target Q
        with torch.no_grad():
            h = torch.zeros(B, cfg.hidden, dtype=dt)
            nq = []
            for t in range(T):
                _, h = self.tgt_critic(s[t], cent_act[t], h)
                qs, _ = self.tgt_critic(s[t + 1], cent_nact[t], h)
                nq.append(torch.cat(qs, dim=-1).min(dim=-1, keepdim=True)[0])
            nq = (1 - de) * torch.stack(nq)
        target = (r + cfg.gamma * nq) * (1 - curr)
        errs = [q * (1 - curr) - target for q in q_seq]
        self.critic_errs = [e.detach() for e in errs]                  # (T, B, 1) per head: the TD errors of this update
        denom = (1 - curr).sum()
        prio = None
        if cfg.use_per:
            w = t32(weights)
            closs = torch.stack([(self._loss(e).sum(dim=0).flatten() * w).sum() / denom for e in errs]).sum()
            tds = [e.abs().detach().numpy() for e in errs]
            pr = [((1 - cfg.per_nu) * td.mean(axis=0) + cfg.per_nu * td.max(axis=0)).flatten() + cfg.per_eps for td in tds]
            prio = np.stack(pr).mean(axis=0) + cfg.per_eps
        else:
            closs = torch.stack([self._loss(e).sum() / denom for e in errs]).sum()
        self.critic_opt.zero_grad()
        closs.backward()
        cgn = torch.nn.utils.clip_grad_norm_(self.critic.parameters(), cfg.max_grad_norm)
        self.critic_grads = {k: p.grad.clone() for k, p in self.critic.named_parameters() if p.grad is not None}
        self.critic_opt.step()
        info["critic_loss"], info["critic_grad_norm"] = closs.detach(), cgn.detach()
        # 5. actor update with the updated critic
        if update_actor:
            for p in self.critic.parameters():
                p.requires_grad = False
            a_seq, _ = self.actor(x_all[:-1])                          # (T, N*B, Ac)
            if cfg.discrete:
                a_seq = hard_gumbel_softmax(a_seq, t32(actor_noise), None if av_all is None else av_all[:-1])
            agent_a = a_seq.split(B, dim=1)
            buf_a = list(t32(acts))
            dm = torch.cat([torch.cat([torch.zeros(1, B, 1, dtype=dt), t32(dones[i])[:T - 1]], 0) for i in range(N)], dim=1)   # (T, N*B, 1)
            h = torch.zeros(N * B, cfg.hidden, dtype=dt)
            s_rep = s[:-1].repeat(1, N, 1)
            batch_cent = cent_act.repeat(1, N, 1)
            repl = []
            for i in range(N):
                parts = [agent_a[j] if j == i else buf_a[j] for j in range(N)]
                repl.append(torch.cat(parts, dim=-1))
            repl = torch.cat(repl, dim=1)                               # (T, N*B, N*Ac): copy i has agent i replaced
            qs_t = []
            for t in range(T):
                q, _ = self.critic(s_rep[t], repl[t], h)
                qs_t.append(q[0])
                _, h = self.critic(s_rep[t], batch_cent[t], h)
            qa = torch.stack(qs_t) * (1 - dm)
            aloss = (-qa).sum() / (1 - dm).sum()
            self.critic_opt.zero_grad()
            self.actor_opt.zero_grad()
            aloss.backward()
            agn = torch.nn.utils.clip_grad_norm_(self.actor.parameters(), cfg.max_grad_norm)
            self.actor_grads = {k: p.grad.clone() for k, p in self.actor.named_parameters() if p.grad is not None}
            self.actor_opt.step()
            for p in self.critic.parameters():
                p.requires_grad = True
            info["actor_loss"], info["actor_grad_norm"] = aloss.detach(), agn.detach()
        info["update_actor"] = update_actor
        self.num_updates += 1
        return info, prio

    def soft_update(self):
        tau = self.cfg.tau
        with torch.no_grad():
            for tgt, src in ((self.tgt_critic, self.critic), (self.tgt_actor, self.actor)):
                for t, s in zip(tgt.parameters(), src.parameters()):
                    t.copy_(t * (1.0 - tau) + s * tau)


def synth_batch_cont(cfg, B, T, seed=0, var_len=True):
    rs = np.random.RandomState(seed)
    N, O, A, S = cfg.n_agents, cfg.obs_dim, cfg.act_dim, cfg.state_dim
    obs = rs.randn(N, T + 1, B, O).astype(np.float32)
    share = rs.randn(T + 1, B, S).astype(np.float32)
    acts = rs.uniform(-1, 1, (N, T, B, A)).astype(np.float32)
    r = rs.randn(T, B, 1).astype(np.float32)
    rew = np.repeat(r[None], N, axis=0)
    dones_env = np.zeros((T, B, 1), np.float32)
    dones = np.zeros((N, T, B, 1), np.float32)
    if var_len:
        L = rs.randint(T // 2, T + 1, size=B)
        for b in range(B):
            dones_env[L[b] - 1:, b, 0] = 1.0
            for n in range(N):
                dn = min(L[b], rs.randint(T // 3, T + 1))       # an agent may die earlier than the episode ends
                dones[n, dn - 1:, b, 0] = 1.0
    return obs, share, acts, rew, dones, dones_env, None


def synth_batch_disc(cfg, B, T, seed=0, var_len=True):
    """Same as `synth_batch_cont` with one-hot buffer actions (Discrete(act_dim))."""
    b = list(synth_batch_cont(cfg, B, T, seed, var_len))
    rs = np.random.RandomState(seed + 7919)
    a = rs.randint(0, cfg.act_dim, size=(cfg.n_agents, T, B))
    b[2] = np.eye(cfg.act_dim, dtype=np.float32)[a]
    return tuple(b)


def synth_avail(cfg, B, T, seed=0):
    """Bernoulli(0.7) availability, action 0 always available: (N, T+1, B, A)."""
    rs = np.random.RandomState(seed + 104729)
    av = (rs.rand(cfg.n_agents, T + 1, B, cfg.act_dim) < 0.7).astype(np.float32)
    av[..., 0] = 1.0
    return av


# =====================================================================================================================
# several policies (share_policy = False): config.py:61, scripts/train/train_mpe.py:139-150, r_maddpg.py:40-105 + 114-331
# =====================================================================================================================
class MaddpgMultiLearner(object):
    """One MaddpgLearner-like state per policy; `step(p, ...)` restates r_maddpg.py:114-331 for update_policy_id = policy p when every
    policy controls exactly its own agents (in the reference's scripts: one agent per policy, heterogeneous obs / action widths).

    specs: [(obs_dim, act_dim)] per policy (policy i controls agent i).  Batch per round: obs {p: (1,T+1,B,O_p)}, share (T+1,B,S),
    acts {p: (1,T,B,A_p)}, rew (T,B,1), dones {p: (1,T,B,1)}, dones_env (T,B,1).  The centralised action vector concatenates the
    policies' agents in sorted-id order (r_maddpg.py:62-105)."""

    def __init__(self, specs, state_dim, base_cfg):
        import dataclasses
        self.specs, self.S = list(specs), state_dim
        self.CA = sum(a for _, a in specs)
        self.cfgs, self.actor, self.critic, self.tgt_actor, self.tgt_critic, self.actor_opt, self.critic_opt = [], [], [], [], [], [], []
        for i, (o, a) in enumerate(specs):
            c = dataclasses.replace(base_cfg, n_agents=1, obs_dim=o, act_dim=a, state_dim=state_dim)
            self.cfgs.append(c)
            actor = init_like_reference(ActorNet(c), c, 1 + i)
            cc = dataclasses.replace(c, n_agents=1, act_dim=self.CA)            # critic input = state + all agents' actions
            critic = init_like_reference(CriticNet(cc), c, 2 + i)
            self.actor.append(actor); self.critic.append(critic)
            self.tgt_actor.append(copy.deepcopy(actor)); self.tgt_critic.append(copy.deepcopy(critic))
            kw = dict(lr=c.lr, eps=c.opti_eps, weight_decay=c.weight_decay)
            self.actor_opt.append(torch.optim.Adam(actor.parameters(), **kw))
            self.critic_opt.append(torch.optim.Adam(critic.parameters(), **kw))
        self.num_updates = [0] * len(specs)

    def _loss(self, cfg, e):
        if cfg.huber:
            d = cfg.huber_delta
            small = (e.abs() <= d).float()
            return small * e ** 2 / 2 + (1 - small) * d * (e.abs() - d / 2)
        return e ** 2

    def step(self, p, obs, share, acts, rew, dones, dones_env, noises=None, actor_noise=None):
        """noises: {q: (T+1, B, A_q)} target-action draws of every policy (MATD3) or None; actor_noise: (T, B, A_p) Gumbel draws (Discrete)."""
        cfg = self.cfgs[p]
        t32 = lambda x: torch.as_tensor(x, dtype=torch.float32)
        P = len(self.specs)
        T, B = acts[0].shape[1], acts[0].shape[2]
        s, de, r = t32(share), t32(dones_env), t32(rew)
        curr = torch.cat([torch.zeros(1, B, 1), de[:T - 1]], 0)
        cent_act = torch.cat([t32(acts[q][0]) for q in range(P)], dim=-1)                  # (T, B, CA)
        update_actor = self.num_updates[p] % cfg.actor_update_interval == 0
        info = {}
        with torch.no_grad():                                                            # r_maddpg.py:62-105, every policy's target actor
            nacts = []
            for q in range(P):
                cq = self.cfgs[q]
                na, _ = self.tgt_actor[q](t32(obs[q][0]))
                if cq.discrete:
                    na = hard_gumbel_softmax(na, t32(noises[q])) if cq.td3 else onehot_of_max(na)
                elif cq.td3:
                    na = na + t32(noises[q])
                nacts.append(na[1:])
            cent_nact = torch.cat(nacts, dim=-1)                                          # (T, B, CA)
        q_seq, _ = self.critic[p](s[:-1], cent_act)
        with torch.no_grad():
            h = torch.zeros(B, cfg.hidden)
            nq = []
            for t in range(T):
                _, h = self.tgt_critic[p](s[t], cent_act[t], h)
                qs, _ = self.tgt_critic[p](s[t + 1], cent_nact[t], h)
                nq.append(torch.cat(qs, dim=-1).min(dim=-1, keepdim=True)[0])
            nq = (1 - de) * torch.stack(nq)
        target = (r + cfg.gamma * nq) * (1 - curr)
        errs = [q * (1 - curr) - target for q in q_seq]
        denom = (1 - curr).sum()
        closs = torch.stack([self._loss(cfg, e).sum() / denom for e in errs]).sum()
        self.critic_opt[p].zero_grad()
        closs.backward()
        cgn = torch.nn.utils.clip_grad_norm_(self.critic[p].parameters(), cfg.max_grad_norm)
        self.critic_grads = {k: v.grad.clone() for k, v in self.critic[p].named_parameters() if v.grad is not None}
        self.critic_opt[p].step()
        info["critic_loss"], info["critic_grad_norm"] = closs.detach(), cgn.detach()
        if update_actor:                                                                 # r_maddpg.py:232-322 with num_update_agents = 1
            for prm in self.critic[p].parameters():
                prm.requires_grad = False
            a_seq, _ = self.actor[p](t32(obs[p][0])[:-1])
            if cfg.discrete:
                a_seq = hard_gumbel_softmax(a_seq, t32(actor_noise))
            parts = [a_seq if q == p else t32(acts[q][0]) for q in range(P)]
            repl = torch.cat(parts, dim=-1)
            dm = torch.cat([torch.zeros(1, B, 1), t32(dones[p][0])[:T - 1]], 0)
            h = torch.zeros(B, cfg.hidden)
            qs_t = []
            for t in range(T):
                q, _ = self.critic[p](s[t], repl[t], h)
                qs_t.append(q[0])
                _, h = self.critic[p](s[t], cent_act[t], h)
            qa = torch.stack(qs_t) * (1 - dm)
            aloss = (-qa).sum() / (1 - dm).sum()
            self.critic_opt[p].zero_grad()
            self.actor_opt[p].zero_grad()
            aloss.backward()
            agn = torch.nn.utils.clip_grad_norm_(self.actor[p].parameters(), cfg.max_grad_norm)
            self.actor_grads = {k: v.grad.clone() for k, v in self.actor[p].named_parameters() if v.grad is not None}
            self.actor_opt[p].step()
            for prm in self.critic[p].parameters():
                prm.requires_grad = True
            info["actor_loss"], info["actor_grad_norm"] = aloss.detach(), agn.detach()
        info["update_actor"] = update_actor
        self.num_updates[p] += 1
        return info

    def soft_update_all(self):
        with torch.no_grad():
            for p in range(len(self.specs)):
                tau = self.cfgs[p].tau
                for tgt, src in ((self.tgt_critic[p], self.critic[p]), (self.tgt_actor[p], self.actor[p])):
                    for t, s in zip(tgt.parameters(), src.parameters()):
                        t.copy_(t * (1.0 - tau) + s * tau)
