"""Drop-in `R_MADDPGPolicy` (reference: offpolicy/algorithms/r_maddpg/algorithm/rMADDPGPolicy.py) for continuous (Box)
and Discrete action spaces.  `actor`, `critic`, `target_actor`, `target_critic` are named views (reference state_dict keys) of the flat
device vectors the CUDA learner updates in place; the two Adam states live beside them.  Rollout-time `get_actions`
(one env step) runs a handful of torch ops on those views; everything update-time is inside `mx_maddpg_step`.
Discrete actors follow rMADDPGPolicy.py:104-120: arg-max one-hot, hard Gumbel-softmax (draws from torch's CPU RNG like
utils/util.py:127-140) and epsilon-greedy exploration.  MultiDiscrete action spaces are not built and raise."""
import ctypes as C

import numpy as np
import torch
import torch.nn.functional as F

from offpolicy._b200 import capi
from offpolicy._b200.flat import FlatModule
from offpolicy._b200.host_util import space_dim, is_discrete, LinearDecay


def sample_gumbel(shape, eps=1e-20):
    """utils/util.py:127-130: one `uniform_` draw from torch's CPU generator."""
    u = torch.empty(*shape).uniform_()
    return -torch.log(-torch.log(u + eps) + eps)


def onehot_from_logits(logits, avail=None):
    """utils/util.py:106-118 (eps = 0): every maximal logit is hot; unavailable actions are forced to -1e10."""
    if avail is not None:
        logits = logits.clone()
        logits[torch.as_tensor(np.asarray(avail), dtype=torch.float32).to(logits.device) == 0] = -1e10
    return (logits == logits.max(dim=-1, keepdim=True)[0]).float()


def gumbel_softmax_hard(logits, avail=None):
    """utils/util.py:133-166 with hard=True, temperature 1: the Gumbel draw is added on the CPU (util.py:137-139)."""
    y = logits.cpu() + sample_gumbel(logits.shape)
    if avail is not None:
        y[torch.as_tensor(np.asarray(avail), dtype=torch.float32) == 0] = -1e10
    y = F.softmax(y / 1.0, dim=-1)
    return ((onehot_from_logits(y) - y) + y).to(logits.device)


def maddpg_cfg_struct(args, n_agents, obs_dim, act_dim, state_dim, episode_len, max_batch, td3, target_noise, actor_update_interval,
                      discrete=False, cent_act_dim=0, act_offset=0, mlp=False, act_segs=None):
    """act_segs: the MultiDiscrete sub-space widths (summing to act_dim), or None for one block (Box / Discrete)."""
    segs = [int(n) for n in act_segs] if act_segs is not None else []
    if len(segs) > capi.MAX_ACT_SEG:
        raise NotImplementedError("B200 MADDPG path: at most %d MultiDiscrete sub-spaces, got %d" % (capi.MAX_ACT_SEG, len(segs)))
    return capi.MaddpgCfg(n_agents=n_agents, obs_dim=obs_dim, act_dim=act_dim, state_dim=state_dim, hidden=args.hidden_size,
                          episode_len=episode_len, max_batch=max_batch, num_q=2 if td3 else 1, actor_update_interval=actor_update_interval,
                          use_huber=int(args.use_huber_loss), use_per=int(args.use_per), gamma=args.gamma, huber_delta=args.huber_delta,
                          per_nu=args.per_nu, per_eps=args.per_eps, lr=args.lr, adam_beta1=0.9, adam_beta2=0.999, adam_eps=args.opti_eps,
                          max_grad_norm=args.max_grad_norm, tau=args.tau, weight_decay=float(getattr(args, "weight_decay", 0) or 0),
                          target_noise=float(target_noise or 0.0), discrete=int(bool(discrete)),
                          no_feature_norm=0 if getattr(args, "use_feature_normalization", True) else 1,
                          use_tanh=0 if getattr(args, "use_ReLU", True) else 1, cent_act_dim=int(cent_act_dim), act_offset=int(act_offset), mlp=int(bool(mlp)),
                          n_act_seg=len(segs), act_seg=(C.c_int32 * capi.MAX_ACT_SEG)(*segs))


def maddpg_entries(cfg, which):
    lib = capi.lib()
    total = C.c_int64()
    n = lib.mx_maddpg_param_layout(C.byref(cfg), which, None, 0, C.byref(total))
    if n < 0:
        raise capi.MxError(lib.mx_last_error().decode())
    arr = (capi.ParamEntry * n)()
    lib.mx_maddpg_param_layout(C.byref(cfg), which, arr, n, C.byref(total))
    return [(e.name.decode(), int(e.offset), int(e.rows), int(e.cols)) for e in arr], int(total.value)


def _init_net(mod, in_dim, hidden, out_specs, gain, use_orthogonal, use_relu=True):
    """Reference construction order (RNNBase then the head, mlp.py:14-23, rnn.py:8-17, act.py / r_actor_critic.py:90-93)."""
    import torch.nn as nn
    init_w = nn.init.orthogonal_ if use_orthogonal else nn.init.xavier_uniform_
    relu_gain = nn.init.calculate_gain("relu" if use_relu else "tanh")
    sd = {}

    def linear(prefix, i, o, g):
        m = nn.Linear(i, o)
        init_w(m.weight.data, gain=g)
        m.bias.data.zero_()
        sd[prefix + ".weight"], sd[prefix + ".bias"] = m.weight.data, m.bias.data

    def lnorm(prefix, n):
        sd[prefix + ".weight"], sd[prefix + ".bias"] = torch.ones(n), torch.zeros(n)

    if "rnn.feature_norm.weight" in mod.views:      # absent with --use_feature_normalization off
        lnorm("rnn.feature_norm", in_dim)
    linear("rnn.mlp.fc1.0", in_dim, hidden, relu_gain); lnorm("rnn.mlp.fc1.2", hidden)
    linear("rnn.mlp.fc_h.0", hidden, hidden, relu_gain); lnorm("rnn.mlp.fc_h.2", hidden)
    for k in ("0.weight", "0.bias", "2.weight", "2.bias"):
        sd["rnn.mlp.fc2.0." + k] = sd["rnn.mlp.fc_h." + k].clone()
    gru = nn.GRU(hidden, hidden, num_layers=1)
    for name, p in gru.named_parameters():
        if "bias" in name:
            p.data.zero_()
        else:
            init_w(p.data)
        sd["rnn.rnn.rnn." + name] = p.data
    lnorm("rnn.rnn.norm", hidden)
    for prefix, o, g in out_specs:
        linear(prefix, hidden, o, g)
    mod.load_state_dict({k: v.reshape(mod.views[k].shape) for k, v in sd.items()})


class R_MADDPGPolicy(object):
    act_segs = None             # one action block (MultiDiscrete is not built)

    def __init__(self, config, policy_config, target_noise=None, td3=False, train=True):
        self.config = config
        self.device = config["device"]
        self.args = self.config["args"]
        self.tau, self.lr, self.opti_eps = self.args.tau, self.args.lr, self.args.opti_eps
        self.weight_decay = getattr(self.args, "weight_decay", 0)
        if getattr(self.args, "prev_act_inp", False):
            raise NotImplementedError("B200 R-MADDPG path: --prev_act_inp is not implemented")
        for flag, want in (("use_conv1d", False),):      # fail loudly, never approximate
            if getattr(self.args, flag, want) != want:
                raise NotImplementedError("B200 R-MADDPG path requires %s=%s" % (flag, want))
        if getattr(self.args, "layer_N", 1) != 1 or getattr(self.args, "hidden_size", 64) != 64 or getattr(self.args, "recurrent_N", 1) != 1:
            raise NotImplementedError("B200 R-MADDPG path requires layer_N=1, recurrent_N=1, hidden_size=64")
        self.central_obs_dim, self.central_act_dim = policy_config["cent_obs_dim"], policy_config["cent_act_dim"]
        self.obs_space, self.act_space = policy_config["obs_space"], policy_config["act_space"]
        self.obs_dim, self.act_dim = space_dim(self.obs_space), space_dim(self.act_space)
        self.output_dim = self.act_dim
        self.hidden_size = self.args.hidden_size
        self.discrete = is_discrete(self.act_space)
        self.multidiscrete = "MultiDiscrete" in self.act_space.__class__.__name__
        if self.multidiscrete:
            raise NotImplementedError("B200 R-MADDPG path: MultiDiscrete action spaces are not implemented (Box and Discrete are)")
        if self.discrete and train:
            self.exploration = LinearDecay(self.args.epsilon_start, self.args.epsilon_finish, self.args.epsilon_anneal_time)   # :57-60
        self.td3, self.target_noise = bool(td3), target_noise
        capi.lib()
        self.dev = capi.device()
        # parameter layouts only: the critic's input is [cent_obs | actions of ALL agents] whatever the number of policies
        cfg = maddpg_cfg_struct(self.args, 1, self.obs_dim, self.act_dim, self.central_obs_dim, 1, 1, td3, target_noise, 1, self.discrete,
                                cent_act_dim=self.central_act_dim)
        self._a_entries, self.Pa = maddpg_entries(cfg, 0)
        self._c_entries, self.Pc = maddpg_entries(cfg, 1)
        z = lambda n: torch.zeros(n, dtype=torch.float32, device=self.dev)
        self.actor_vecs = [z(self.Pa) for _ in range(4)]      # theta, target, adam m, adam v
        self.critic_vecs = [z(self.Pc) for _ in range(4)]
        self.actor = FlatModule(self.actor_vecs[0], self._a_entries, "")
        self.target_actor = FlatModule(self.actor_vecs[1], self._a_entries, "")
        self.critic = FlatModule(self.critic_vecs[0], self._c_entries, "")
        self.target_critic = FlatModule(self.critic_vecs[1], self._c_entries, "")
        relu = bool(getattr(self.args, "use_ReLU", True))
        _init_net(self.actor, self.obs_dim, self.hidden_size, [("act.action_out", self.act_dim, self.args.gain)], self.args.gain,
                  self.args.use_orthogonal, use_relu=relu)
        _init_net(self.critic, self.central_obs_dim + self.central_act_dim, self.hidden_size,
                  [("q_outs.%d" % k, 1, 1.0) for k in range(2 if td3 else 1)], 1.0, self.args.use_orthogonal, use_relu=relu)
        # the reference constructs the two target networks like the live ones (rMADDPGPolicy.py:45-46) before overwriting them with
        # the live weights (:49-50): their initialisation consumes torch's generator, so it is replayed here -- a seeded run then
        # draws the same warm-up / exploration actions as the reference
        _init_net(self.target_actor, self.obs_dim, self.hidden_size, [("act.action_out", self.act_dim, self.args.gain)], self.args.gain,
                  self.args.use_orthogonal, use_relu=relu)
        _init_net(self.target_critic, self.central_obs_dim + self.central_act_dim, self.hidden_size,
                  [("q_outs.%d" % k, 1, 1.0) for k in range(2 if td3 else 1)], 1.0, self.args.use_orthogonal, use_relu=relu)
        self.actor_vecs[1].copy_(self.actor_vecs[0])          # rMADDPGPolicy.py:49-50
        self.critic_vecs[1].copy_(self.critic_vecs[0])
        self._trainer = None
        self._handle = None          # this policy's mx_maddpg (created by the trainer)

    # -- rollout-time single step: ONE launch of k_policy_step (csrc/rollout.cu) per env step -----------------------------
    def _stepper(self):
        if getattr(self, "_roll", None) is None:
            from offpolicy._b200.rollout import PolicyStepper
            self._roll = PolicyStepper(self.obs_dim, self.act_dim, feature_norm=bool(getattr(self.args, "use_feature_normalization", True)),
                                       tanh=not getattr(self.args, "use_ReLU", True))
        return self._roll

    def get_actions(self, obs, prev_actions, rnn_states, available_actions=None, t_env=None, explore=False, use_target=False, use_gumbel=False):
        theta = self.actor_vecs[1] if use_target else self.actor_vecs[0]
        o = np.asarray(obs, dtype=np.float32)
        st = self._stepper()
        if o.ndim == 3:
            outs, h = [], rnn_states
            for t in range(o.shape[0]):
                a, h, _, _ = st.step(theta, o[t], h, want_greedy=False)
                outs.append(a)
            out = torch.from_numpy(np.stack(outs))
        else:
            a, h, _, _ = st.step(theta, o, rnn_states, want_greedy=False)
            out = torch.from_numpy(a)
        h = torch.from_numpy(h)
        eps = None
        if self.discrete:                                                                   # rMADDPGPolicy.py:104-120
            if use_gumbel or (use_target and self.target_noise is not None):
                out = gumbel_softmax_hard(out, available_actions)
            elif explore:
                assert o.ndim == 2, "Cannot do exploration on a sequence!"
                onehot_actions = gumbel_softmax_hard(out, available_actions)
                batch_size = o.shape[0]
                eps = self.exploration.eval(t_env)
                rand_numbers = np.random.rand(batch_size, 1)
                logits = torch.ones(batch_size, self.act_dim)
                if available_actions is not None:
                    logits[torch.as_tensor(np.asarray(available_actions), dtype=torch.float32) == 0] = -1e10     # avail_choose, util.py:297-302
                random_actions = torch.distributions.OneHotCategorical(logits=logits).sample().numpy()
                take_random = (rand_numbers < eps).astype(int)
                out = (1 - take_random) * onehot_actions.cpu().numpy() + take_random * random_actions
            else:
                out = onehot_from_logits(out, available_actions)
            return out, h, eps
        if explore:
            assert o.ndim == 2, "Cannot do exploration on a sequence!"
            out = torch.empty(out.shape).normal_(mean=0, std=self.args.act_noise_std).to(out.device) + out     # util.py:217-218
        elif use_target and self.target_noise is not None:
            out = torch.empty(out.shape).normal_(mean=0, std=self.target_noise).to(out.device) + out
        return out, h, None

    def get_random_actions(self, obs, available_actions=None):
        if self.discrete:                                                                   # rMADDPGPolicy.py:143-150
            logits = torch.ones(obs.shape[0], self.act_dim)
            if available_actions is not None:
                logits[torch.as_tensor(np.asarray(available_actions), dtype=torch.float32) == 0] = -1e10
            return torch.distributions.OneHotCategorical(logits=logits).sample().numpy()
        return np.random.uniform(self.act_space.low, self.act_space.high, size=(obs.shape[0], self.act_dim))

    def init_hidden(self, num_agents, batch_size):
        if num_agents == -1:
            return torch.zeros(batch_size, self.hidden_size)
        return torch.zeros(num_agents, batch_size, self.hidden_size)

    def soft_target_updates(self):
        if self._trainer is None:
            raise RuntimeError("soft_target_updates: no trainer attached")
        capi.check(capi.lib().mx_maddpg_soft_update(self._handle, capi.stream_ptr()))

    def hard_target_updates(self):
        self.actor_vecs[1].copy_(self.actor_vecs[0])
        self.critic_vecs[1].copy_(self.critic_vecs[0])
