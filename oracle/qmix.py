"""Recurrent QMIX / VDN learner step, restated in CPU PyTorch (oracle; test infra only).

The reference's arithmetic on this path is eager PyTorch (third-party; torch==1.5.1 pinned
in requirements.txt:144, torch 2.11 installed here).  This file restates the *call sites*:

  agent net        /root/reference/offpolicy/algorithms/utils/mlp.py:7-29,52-89, rnn.py:4-47,
                   act.py:5-37, qmix/algorithm/agent_q_function.py:34-67
  mixer            qmix/algorithm/q_mixer.py:6-94          (VDN intent: vdn/algorithm/vdn_mixer.py:28-40)
  learner step     qmix/qmix.py:77-200                     (batch assembly, double-Q, TD target, loss, PER, clip, Adam)
  target updates   qmix/qmix.py:203-216 + utils/util.py:123-134
  argmax masking   utils/util.py:297-302 (-1e10 fill), QMixPolicy.py:69-93,167-172

Module/parameter names reproduce the reference's state_dict keys (SURVEY.md App. E) so the
golden state_dicts dumped from the real reference load with `load_state_dict(strict=True)`.

`agent_trace()` re-runs the agent net one GRU cell at a time and returns every
intermediate the CUDA kernels materialise (used only to localise kernel bugs).
"""
import copy
from dataclasses import dataclass

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F


@dataclass
class QmixConfig:
    n_agents: int = 3
    obs_dim: int = 30
    act_dim: int = 9
    state_dim: int = 48
    hidden: int = 64
    layer_n: int = 1
    mixer_hidden: int = 32
    hyper_hidden: int = 64
    hyper_layers: int = 2
    gamma: float = 0.99
    lr: float = 5e-4
    opti_eps: float = 1e-5
    max_grad_norm: float = 10.0
    tau: float = 0.005
    double_q: bool = True
    huber: bool = False
    huber_delta: float = 10.0
    use_per: bool = False
    per_nu: float = 0.9
    per_eps: float = 1e-6
    vdn: bool = False
    feature_norm: bool = True
    relu: bool = True              # config.py use_ReLU (store_false): False = tanh blocks (mlp.py:12,19-22)
    prev_act_inp: bool = False     # config.py:81: agent-net input = [obs | previous one-hot action] (QMixPolicy.py:29,54-58)
    gain: float = 0.01


def _lin(i, o):
    return nn.Linear(i, o)


class _Block(nn.Sequential):
    """Linear -> ReLU -> LayerNorm (mlp.py:19-23)."""

    def __init__(self, i, o, relu=True):
        super().__init__(_lin(i, o), nn.ReLU() if relu else nn.Tanh(), nn.LayerNorm(o))


class _MLP(nn.Module):
    def __init__(self, i, h, layer_n, relu=True):
        super().__init__()
        self.fc1 = _Block(i, h, relu)
        self.fc_h = _Block(h, h, relu)                      # registered, never used in forward (mlp.py:21-29)
        self.fc2 = nn.ModuleList([copy.deepcopy(self.fc_h) for _ in range(layer_n)])

    def forward(self, x):
        x = self.fc1(x)
        for blk in self.fc2:
            x = blk(x)
        return x


class _GRUWrap(nn.Module):
    def __init__(self, h):
        super().__init__()
        self.rnn = nn.GRU(h, h, num_layers=1)
        self.norm = nn.LayerNorm(h)


class _RNNBase(nn.Module):
    def __init__(self, i, h, layer_n, feature_norm, relu=True):
        super().__init__()
        if feature_norm:
            self.feature_norm = nn.LayerNorm(i)
        self.mlp = _MLP(i, h, layer_n, relu)
        self.rnn = _GRUWrap(h)
        self._fn = feature_norm

    def forward(self, x, h0):
        if self._fn:
            x = self.feature_norm(x)
        x = self.mlp(x)
        y, hT = self.rnn.rnn(x, h0)
        return self.rnn.norm(y), hT[0]                # LN on outputs only; carried state is raw h (rnn.py:21-23)


class _Head(nn.Module):
    def __init__(self, h, a):
        super().__init__()
        self.action_out = _lin(h, a)


class AgentNet(nn.Module):
    def __init__(self, cfg, in_dim=None, out_dim=None):
        super().__init__()
        self.rnn = _RNNBase(in_dim or cfg.obs_dim, cfg.hidden, cfg.layer_n, cfg.feature_norm, getattr(cfg, "relu", True))
        self.q = _Head(cfg.hidden, out_dim or cfg.act_dim)
        self.hidden = cfg.hidden

    def forward(self, x, h0=None):
        if h0 is None:
            h0 = torch.zeros(1, x.shape[1], self.hidden, dtype=x.dtype, device=x.device)
        y, hT = self.rnn(x, h0)
        return self.q.action_out(y), hT


class QMixerNet(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        S, N, ME, HY = cfg.state_dim, cfg.n_agents, cfg.mixer_hidden, cfg.hyper_hidden
        self.N, self.ME, self.S = N, ME, S
        if cfg.hyper_layers == 1:
            self.hyper_w1 = _lin(S, N * ME)
            self.hyper_w2 = _lin(S, ME)
        else:
            self.hyper_w1 = nn.Sequential(_lin(S, HY), nn.ReLU(), _lin(HY, N * ME))
            self.hyper_w2 = nn.Sequential(_lin(S, HY), nn.ReLU(), _lin(HY, ME))
        self.hyper_b1 = _lin(S, ME)
        self.hyper_b2 = nn.Sequential(_lin(S, HY), nn.ReLU(), _lin(HY, 1))

    def forward(self, q, s):
        T, B = q.shape[0], q.shape[1]
        q = q.reshape(T, B, 1, self.N)
        w1 = self.hyper_w1(s).abs().view(T, B, self.N, self.ME)
        b1 = self.hyper_b1(s).view(T, B, 1, self.ME)
        hid = F.elu(torch.matmul(q, w1) + b1)
        w2 = self.hyper_w2(s).abs().view(T, B, self.ME, 1)
        b2 = self.hyper_b2(s).view(T, B, 1, 1)
        return (torch.matmul(hid, w2) + b2).view(T, B, 1)


class VDNMixerNet(nn.Module):
    """Intent of vdn_mixer.py:28-40 (the shipped one is shape-broken, SURVEY.md App. D-1)."""

    def forward(self, q, s):
        return q.sum(dim=-1, keepdim=True)


def init_like_reference(net, cfg, seed):
    """Orthogonal/zero init in the spirit of mlp.py:14-17, rnn.py:9-16, act.py:10-12, q_mixer.py:33-35.
    Parity tests never depend on this (fixtures carry the state_dict); it only gives
    well-conditioned random weights for synthetic workloads."""
    g = torch.Generator().manual_seed(seed)
    relu_gain = nn.init.calculate_gain("relu")
    with torch.no_grad():
        for name, m in net.named_modules():
            if isinstance(m, nn.LayerNorm):
                m.weight.fill_(1.0)
                m.bias.zero_()
            elif isinstance(m, nn.Linear):
                gain = cfg.gain if name.endswith("action_out") else (1.0 if "hyper" in name else relu_gain)
                nn.init.orthogonal_(m.weight, gain=gain, generator=g)
                m.bias.zero_()
            elif isinstance(m, nn.GRU):
                for pn, p in m.named_parameters():
                    if "bias" in pn:
                        p.zero_()
                    else:
                        nn.init.orthogonal_(p, generator=g)
    return net


def randomize_all(net, seed, scale=0.2):
    """Make EVERY tensor non-trivial (LN gains != 1, biases != 0) so kernels' affine paths are exercised."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in net.named_parameters():
            if p.dim() == 1:
                is_gain = name.endswith("weight")
                p.copy_((1.0 if is_gain else 0.0) + scale * torch.randn(p.shape, generator=g))
            else:
                p.add_(0.05 * torch.randn(p.shape, generator=g))
    return net


def masked_argmax(q, avail):
    if avail is not None:
        q = q.clone()
        q[avail == 0] = -1e10                          # util.py:297-302
    return q.max(dim=-1)[1]


class QmixLearner(object):
    """State + one learner step.  Batch = the reference's 9-tuple restricted to policy_0,
    as arrays: obs (N,T+1,B,O), share (T+1,B,S), acts (N,T,B,A), rewards (N,T,B,1),
    dones (N,T,B,1), dones_env (T,B,1), avail (N,T+1,B,A) | None, weights (B,) | None, idx | None."""

    def __init__(self, cfg, seed=1, device="cpu", dtype=torch.float32):
        """device: "cpu" (parity oracle, CPU baseline) or a CUDA device -- the same eager PyTorch ops the reference issues with
        `--cuda` (bench.py's secondary baseline, SURVEY.md section 8(d)).  dtype: float32 is the reference's arithmetic; float64
        makes every tensor of the step (batch, networks, Adam moments, clipping, Polyak) double precision, a round-off-free yardstick
        for the kernels (tests/row_coverage_checks.py).  The initialisation is drawn in float32 either way, so a float64 learner
        with the same seed holds the same values as a float32 one."""
        self.cfg = cfg
        self.device = torch.device(device)
        self.dtype = dtype
        in_dim = cfg.obs_dim + cfg.act_dim if cfg.prev_act_inp else cfg.obs_dim
        self.agent = init_like_reference(AgentNet(cfg, in_dim=in_dim), cfg, seed).to(self.device, dtype)
        self.mixer = (VDNMixerNet() if cfg.vdn else init_like_reference(QMixerNet(cfg), cfg, seed + 1)).to(self.device, dtype)
        self.sync_targets()
        self.params = list(self.agent.parameters()) + list(self.mixer.parameters())   # qmix.py:66-72
        self.opt = torch.optim.Adam(self.params, lr=cfg.lr, eps=cfg.opti_eps)

    def sync_targets(self):
        self.tgt_agent = copy.deepcopy(self.agent)
        self.tgt_mixer = copy.deepcopy(self.mixer)

    # -- forward pieces ----------------------------------------------------------
    def stack_agents(self, x):
        """(N,T,B,D) -> (T, N*B, D), row = n*B + b (qmix.py:108-109)."""
        x = torch.as_tensor(x, dtype=getattr(self, "dtype", torch.float32)).to(getattr(self, "device", "cpu"))
        return torch.cat(list(x), dim=-2)

    def loss_terms(self, batch):
        cfg = self.cfg
        obs, share, acts, rew, _dones, dones_env, avail, weights, _idx = batch
        B = obs.shape[2]
        T = acts.shape[1]
        dev, dt = self.device, self.dtype
        s = torch.as_tensor(share, dtype=dt).to(dev)
        de = torch.as_tensor(dones_env, dtype=dt).to(dev)
        x = self.stack_agents(obs)
        a = self.stack_agents(acts)
        av = self.stack_agents(avail) if avail is not None else None
        if cfg.prev_act_inp:        # zeros at t = 0, then the buffer's actions (qmix.py:122-127)
            x = torch.cat((x, torch.cat((torch.zeros(1, a.shape[1], a.shape[2], dtype=dt, device=dev), a), 0)), -1)

        q_all, _ = self.agent(x)                                   # (T+1, N*B, A)
        a_idx = a.max(dim=-1)[1]
        q_taken = q_all[:-1].gather(2, a_idx.unsqueeze(-1))        # (T, N*B, 1)
        q_taken = torch.cat(q_taken.split(B, dim=-2), dim=-1)      # (T, B, N)
        with torch.no_grad():
            tq_all, _ = self.tgt_agent(x)
            if cfg.double_q:
                greedy = masked_argmax(q_all.detach(), av)         # avail-masked, all T+1 steps
                tq = tq_all.gather(2, greedy.unsqueeze(-1))
            else:
                tq = tq_all.max(dim=-1, keepdim=True)[0]           # no avail mask (qmix.py:144)
            tq = torch.cat(tq[1:].split(B, dim=-2), dim=-1)        # (T, B, N)
            q_tot_next = self.tgt_mixer(tq, s[1:])
        q_tot = self.mixer(q_taken, s[:-1])                        # (T, B, 1)
        r = torch.as_tensor(rew[0], dtype=dt).to(dev)   # agent 0's stream (qmix.py:159)
        bad = torch.cat([torch.zeros(1, B, 1, dtype=dt, device=dev), de[:T - 1]], 0)     # qmix.py:161
        y = r + (1 - de) * cfg.gamma * q_tot_next
        err = (q_tot - y.detach()) * (1 - bad)
        per_elem = self._huber(err) if cfg.huber else err ** 2
        denom = (1 - bad).sum()
        prio = None
        if cfg.use_per:
            w = torch.as_tensor(weights, dtype=dt).to(dev)
            loss = (per_elem.sum(dim=0).flatten() * w).sum() / denom
            td = err.abs().detach().cpu().numpy()
            prio = ((1 - cfg.per_nu) * td.mean(axis=0) + cfg.per_nu * td.max(axis=0)).flatten() + cfg.per_eps
        else:
            loss = per_elem.sum() / denom
        aux = dict(q_all=q_all, q_taken=q_taken, tq_next=tq, q_tot=q_tot, q_tot_next=q_tot_next,
                   target=y, err=err, bad=bad, denom=denom)
        return loss, prio, aux

    def _huber(self, e):
        d = self.cfg.huber_delta
        small = (e.abs() <= d).to(e.dtype)
        return small * e ** 2 / 2 + (1 - small) * d * (e.abs() - d / 2)

    # -- the step ------------------------------------------------------------------
    def step(self, batch):
        loss, prio, aux = self.loss_terms(batch)
        self.opt.zero_grad()
        loss.backward()
        gnorm = torch.nn.utils.clip_grad_norm_(self.params, self.cfg.max_grad_norm)
        self.opt.step()
        info = dict(loss=loss.detach(), grad_norm=gnorm.detach() if torch.is_tensor(gnorm) else torch.tensor(gnorm),
                    Q_tot=(aux["q_tot"] * (1 - aux["bad"])).mean().detach())
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


def agent_trace(net, x):
    """Cell-by-cell forward of AgentNet returning every intermediate, (T+1, R, .) tensors."""
    with torch.no_grad():
        rb = net.rnn
        x0 = rb.feature_norm(x) if rb._fn else x
        fc1 = rb.mlp.fc1
        u1 = fc1[1](fc1[0](x0))
        x1 = fc1[2](u1)
        blk = rb.mlp.fc2[0]
        u2 = blk[1](blk[0](x1))
        x2 = blk[2](u2)
        g = rb.rnn.rnn
        H = net.hidden
        gi = F.linear(x2, g.weight_ih_l0, g.bias_ih_l0)
        h = torch.zeros(x.shape[1], H, dtype=x.dtype, device=x.device)
        hs, rs, zs, ns, hns = [], [], [], [], []
        for t in range(x.shape[0]):
            gh = F.linear(h, g.weight_hh_l0, g.bias_hh_l0)
            r = torch.sigmoid(gi[t, :, :H] + gh[:, :H])
            z = torch.sigmoid(gi[t, :, H:2 * H] + gh[:, H:2 * H])
            n = torch.tanh(gi[t, :, 2 * H:] + r * gh[:, 2 * H:])
            h = (1 - z) * n + z * h
            hs.append(h); rs.append(r); zs.append(z); ns.append(n); hns.append(gh[:, 2 * H:])
        hseq = torch.stack(hs)
        y = rb.rnn.norm(hseq)
        q = net.q.action_out(y)
        return dict(x0=x0, u1=u1, x1=x1, u2=u2, x2=x2, gi=gi, h=hseq, r=torch.stack(rs), z=torch.stack(zs),
                    n=torch.stack(ns), hn=torch.stack(hns), y=y, q=q)


def synth_batch(cfg, B, T, seed=0, avail_p=None, var_len=False, dtype=np.float32):
    """Synthetic batch in the reference's sample() layout (BASELINE.md §3 item 2).  dtype: of the returned arrays; the values are
    drawn in float32 whatever it is, so a float64 batch holds exactly the float32 batch of the same seed."""
    rs = np.random.RandomState(seed)
    N, O, A, S = cfg.n_agents, cfg.obs_dim, cfg.act_dim, cfg.state_dim
    obs = rs.randn(N, T + 1, B, O).astype(np.float32).astype(dtype)
    share = rs.randn(T + 1, B, S).astype(np.float32).astype(dtype)
    if avail_p is None:
        avail = np.ones((N, T + 1, B, A), dtype)
    else:
        avail = (rs.rand(N, T + 1, B, A) < avail_p).astype(dtype)
        avail[..., 0] = 1.0
    # taken actions are always available ones
    logits = rs.rand(N, T, B, A) + 10.0 * avail[:, :T]
    a_idx = logits.argmax(-1)
    acts = np.eye(A, dtype=dtype)[a_idx]
    r = rs.randn(T, B, 1).astype(np.float32).astype(dtype)
    rew = np.repeat(r[None], N, axis=0)
    dones_env = np.zeros((T, B, 1), dtype)
    if var_len:
        L = rs.randint(T // 2, T + 1, size=B)
        for b in range(B):
            dones_env[L[b] - 1:, b, 0] = 1.0
    dones = np.repeat(dones_env[None], N, axis=0)
    return obs, share, acts, rew, dones, dones_env, avail
