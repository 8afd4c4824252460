"""MLP (transition-level) QMIX / VDN learner step, restated in CPU PyTorch (oracle; test infra only).

Restates the call sites of the reference's non-recurrent path:

  agent net        /root/reference/offpolicy/algorithms/utils/mlp.py:7-29,52-89 (MLPBase), act.py:5-37,
                   mqmix/algorithm/agent_q_function.py:8-40
  mixer            mqmix/algorithm/q_mixer.py (same arithmetic as the recurrent one on (B, N) inputs; oracle.qmix.QMixerNet with T = 1)
  learner step     mqmix/mqmix.py:67-218 (stack agents, double-Q with the next-step availability mask, TD target, mean loss, PER
                   weights and |error| + eps priorities, clip, Adam)
  target updates   mqmix/mqmix.py:220-234 + utils/util.py:123-134

Pinned by tests/test_oracle_mqmix.py against the goldens the unmodified reference produced (tests/golden/mqmix_*.npz).
Module / parameter names reproduce the reference's state_dict keys, so the golden state_dicts load strictly.
"""
import copy

import numpy as np
import torch
import torch.nn as nn

from oracle.qmix import _MLP, _Head, QMixerNet, VDNMixerNet, init_like_reference, masked_argmax


class _MLPBase(nn.Module):
    def __init__(self, i, h, layer_n, feature_norm, relu=True):
        super().__init__()
        if feature_norm:
            self.feature_norm = nn.LayerNorm(i)
        self.mlp = _MLP(i, h, layer_n, relu)
        self._fn = feature_norm

    def forward(self, x):
        if self._fn:
            x = self.feature_norm(x)
        return self.mlp(x)


class MAgentNet(nn.Module):
    """agent_q_function.py:8-40: MLPBase -> Linear(H, A)."""

    def __init__(self, cfg):
        super().__init__()
        self.mlp = _MLPBase(cfg.obs_dim, cfg.hidden, cfg.layer_n, cfg.feature_norm, getattr(cfg, "relu", True))
        self.q = _Head(cfg.hidden, cfg.act_dim)

    def forward(self, x):
        return self.q.action_out(self.mlp(x))


class MqmixLearner(object):
    """State + one learner step.  Batch = the reference's 13-tuple restricted to policy_0, as arrays: obs (N,B,O), share (B,S),
    acts (N,B,A), rewards (N,B,1), nobs (N,B,O), nshare (B,S), dones (N,B,1), dones_env (B,1), valid (N,B,1), avail (N,B,A) | None,
    navail (N,B,A) | None, weights (B,) | None, idx | None."""

    def __init__(self, cfg, seed=1, device="cpu", dtype=torch.float32):
        """dtype: as oracle.qmix.QmixLearner (float64: the whole step in double precision, same initial values)."""
        self.cfg = cfg
        self.device = torch.device(device)
        self.dtype = dtype
        self.agent = init_like_reference(MAgentNet(cfg), cfg, seed).to(self.device, dtype)
        self.mixer = (VDNMixerNet() if cfg.vdn else init_like_reference(QMixerNet(cfg), cfg, seed + 1)).to(self.device, dtype)
        self.sync_targets()
        self.params = list(self.agent.parameters()) + list(self.mixer.parameters())      # mqmix.py:57-63
        self.opt = torch.optim.Adam(self.params, lr=cfg.lr, eps=cfg.opti_eps)

    def sync_targets(self):
        self.tgt_agent = copy.deepcopy(self.agent)
        self.tgt_mixer = copy.deepcopy(self.mixer)

    def _stack(self, x):
        """(N,B,D) -> (N*B, D), row = n*B + b (mqmix.py:100-103)."""
        return torch.as_tensor(np.asarray(x), dtype=self.dtype).to(self.device).reshape(-1, np.asarray(x).shape[-1])

    def loss_terms(self, batch):
        cfg, dev, dt = self.cfg, self.device, self.dtype
        obs, share, acts, rew, nobs, nshare, _dones, dones_env, _valid, _avail, navail, weights, _idx = batch
        B = np.asarray(obs).shape[1]
        s = torch.as_tensor(np.asarray(share), dtype=dt).to(dev)
        ns = torch.as_tensor(np.asarray(nshare), dtype=dt).to(dev)
        de = torch.as_tensor(np.asarray(dones_env), dtype=dt).to(dev)
        x, nx, a = self._stack(obs), self._stack(nobs), self._stack(acts)
        nav = self._stack(navail) if navail is not None else None

        q_all = self.agent(x)                                                   # (N*B, A)
        q_taken = q_all.gather(1, a.max(dim=-1)[1].unsqueeze(-1))               # mqmix.py:130-133
        q_taken = torch.cat(q_taken.split(B, dim=-2), dim=-1)                   # (B, N)
        with torch.no_grad():
            if cfg.double_q:
                greedy = masked_argmax(self.agent(nx), nav)                      # mqmix.py:141-162: live net picks, next-step mask
                tq = self.tgt_agent(nx).gather(1, greedy.unsqueeze(-1))
            else:
                tqa = self.tgt_agent(nx)                                         # mqmix.py:164-170 -> mQMixPolicy.get_actions(explore=False):
                if nav is not None:                                              # the greedy Q of the MASKED target values
                    tqa = tqa.clone()
                    tqa[nav == 0] = -1e10
                tq = tqa.max(dim=-1, keepdim=True)[0]
            tq = torch.cat(tq.split(B, dim=-2), dim=-1)                          # (B, N)
            q_tot_next = self.tgt_mixer(tq.unsqueeze(0), ns.unsqueeze(0))[0]     # (B, 1)
        q_tot = self.mixer(q_taken.unsqueeze(0), s.unsqueeze(0))[0]              # (B, 1)
        r = torch.as_tensor(np.asarray(rew)[0], dtype=dt).to(dev)     # agent 0's stream (mqmix.py:96)
        y = r + (1 - de) * cfg.gamma * q_tot_next                                # mqmix.py:187
        err = (q_tot - y.detach()).squeeze(-1)                                   # (B,)
        per_elem = self._huber(err) if cfg.huber else err ** 2
        prio = None
        if cfg.use_per:
            w = torch.as_tensor(np.asarray(weights), dtype=dt).to(dev)
            loss = (per_elem * w).mean()                                         # mqmix.py:192-198
            prio = err.abs().detach().cpu().numpy().flatten() + cfg.per_eps
        else:
            loss = per_elem.mean()
        return loss, prio, dict(q_all=q_all, q_taken=q_taken, tq_next=tq, q_tot=q_tot, q_tot_next=q_tot_next, target=y, err=err)

    def _huber(self, e):
        d = self.cfg.huber_delta
        small = (e.abs() <= d).to(e.dtype)
        return small * e ** 2 / 2 + (1 - small) * d * (e.abs() - d / 2)

    def step(self, batch):
        loss, prio, aux = self.loss_terms(batch)
        self.opt.zero_grad()
        loss.backward()
        gnorm = torch.nn.utils.clip_grad_norm_(self.params, self.cfg.max_grad_norm)
        self.opt.step()
        info = dict(loss=loss.detach(), grad_norm=gnorm.detach() if torch.is_tensor(gnorm) else torch.tensor(gnorm),
                    Q_tot=aux["q_tot"].mean().detach())
        return info, prio, aux

    def grads(self, batch):
        """Raw (unclipped) gradients, no parameter update."""
        loss, prio, aux = self.loss_terms(batch)
        for p in self.params:
            p.grad = None
        loss.backward()
        return loss.detach(), prio, aux

    def soft_update(self):
        tau = self.cfg.tau
        with torch.no_grad():
            for t, s in list(zip(self.tgt_agent.parameters(), self.agent.parameters())) + \
                        list(zip(self.tgt_mixer.parameters(), self.mixer.parameters())):
                t.copy_(t * (1.0 - tau) + s * tau)

    def hard_update(self):
        self.tgt_agent.load_state_dict(self.agent.state_dict())
        self.tgt_mixer.load_state_dict(self.mixer.state_dict())


def synth_transitions(cfg, B, seed=0, avail=True, avail_p=0.6):
    """Synthetic transition batch in the reference's MlpReplayBuffer.sample() layout."""
    rs = np.random.RandomState(seed)
    N, O, A, S = cfg.n_agents, cfg.obs_dim, cfg.act_dim, cfg.state_dim
    av = (rs.rand(N, B, A) < avail_p).astype(np.float32); av[..., 0] = 1.0
    nav = (rs.rand(N, B, A) < avail_p).astype(np.float32); nav[..., 0] = 1.0
    acts = np.eye(A, dtype=np.float32)[(rs.rand(N, B, A) + 10.0 * av).argmax(-1)]
    rew = np.repeat(rs.randn(1, B, 1).astype(np.float32), N, 0)
    return (rs.randn(N, B, O).astype(np.float32), rs.randn(B, S).astype(np.float32), acts, rew, rs.randn(N, B, O).astype(np.float32),
            rs.randn(B, S).astype(np.float32), np.zeros((N, B, 1), np.float32), (rs.rand(B, 1) < 0.3).astype(np.float32), np.ones((N, B, 1), np.float32),
            av if avail else None, nav if avail else None)


class TransitionReplay(object):
    """Transition store + uniform sampling, restated in NumPy from /root/reference/offpolicy/utils/mlp_buffer.py:
    storage and ring insert :101-205, np.random.choice sampling :83-98, sample layout and reward normalisation (mean / population std over
    ALL filled rewards) :207-257.  Pinned by tests/test_oracle_mqmix.py against tests/golden/mlp_replay_small.npz (the reference's own
    MlpReplayBuffer driven with the same inserts under the same NumPy seed)."""

    def __init__(self, capacity, N, O, S, A, use_avail=False, reward_norm=False):
        z = lambda *s: np.zeros(s, np.float32)
        self.capacity, self.use_avail, self.reward_norm = capacity, use_avail, reward_norm
        self.f = dict(obs=z(capacity, N, O), share=z(capacity, S), acts=z(capacity, N, A), rew=z(capacity, N, 1), nobs=z(capacity, N, O),
                      nshare=z(capacity, S), dones=np.ones((capacity, N, 1), np.float32), dones_env=np.ones((capacity, 1), np.float32),
                      valid=z(capacity, N, 1))
        if use_avail:
            self.f["avail"] = np.ones((capacity, N, A), np.float32)
            self.f["navail"] = np.ones((capacity, N, A), np.float32)
        self.filled = self.cur = 0

    def __len__(self):
        return self.filled

    def insert(self, n, obs, share, acts, rew, nobs, nshare, dones, dones_env, valid, avail=None, navail=None):
        idx = (self.cur + np.arange(n)) % self.capacity                       # mlp_buffer.py:179-183
        vals = dict(obs=obs, share=share, acts=acts, rew=rew, nobs=nobs, nshare=nshare, dones=dones, dones_env=dones_env, valid=valid)
        if self.use_avail:
            vals.update(avail=avail, navail=navail)
        for k, v in vals.items():
            self.f[k][idx] = v
        self.cur = int(idx[-1]) + 1
        self.filled = min(self.filled + n, self.capacity)
        return idx

    def gather(self, inds):
        f = self.f
        c = lambda x: x.transpose(1, 0, 2)                                    # (B, N, D) -> (N, B, D), mlp_buffer.py:6-7
        rew = f["rew"][inds]
        if self.reward_norm:
            allr = f["rew"][:self.filled]
            rew = (rew - allr.mean()) / allr.std()
        return (c(f["obs"][inds]), f["share"][inds], c(f["acts"][inds]), c(rew), c(f["nobs"][inds]), f["nshare"][inds], c(f["dones"][inds]),
                f["dones_env"][inds], c(f["valid"][inds]), c(f["avail"][inds]) if self.use_avail else None,
                c(f["navail"][inds]) if self.use_avail else None)

    def sample(self, B):
        inds = np.random.choice(self.filled, B)
        return self.gather(inds) + (None, None), inds


def transition_replay_script(seed=0):
    """Insert / sample schedule of tests/golden/mlp_replay_small.npz (shared by its generator and the tests that replay it): yields
    ("insert", n, fields) and ("sample", B, None); capacity 20, so the ring wraps."""
    N, O, A, S, E = 3, 6, 4, 7, 20
    rs = np.random.RandomState(seed)
    for k in range(31):
        n = 1 if k % 5 else 3
        f = dict(obs=rs.randn(n, N, O), share=rs.randn(n, S), acts=np.eye(A)[rs.randint(0, A, (n, N))], rew=2.0 + rs.randn(n, N, 1), nobs=rs.randn(n, N, O),
                 nshare=rs.randn(n, S), dones=(rs.rand(n, N, 1) < 0.2) * 1.0, dones_env=(rs.rand(n, 1) < 0.2) * 1.0, valid=(rs.rand(n, N, 1) < 0.9) * 1.0,
                 avail=(rs.rand(n, N, A) < 0.5) * 1.0, navail=(rs.rand(n, N, A) < 0.5) * 1.0)
        yield "insert", n, {kk: v.astype(np.float32) for kk, v in f.items()}
        if k >= 6:
            yield "sample", 8, None
