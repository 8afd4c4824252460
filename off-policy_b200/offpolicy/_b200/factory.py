"""Construction helpers for the drop-in classes outside a runner: what the reference's runner does in
runner/rnn/base_runner.py:110-178 (argparse namespace -> policy_info -> Policy -> Trainer -> Buffer), for callers that hold a plain
description of the workload instead of a parsed command line.  Used by bench.py and by the parity tests; no test or oracle code here.

`LearnerConfig` carries the reference's config.py defaults for the fields the learner path reads; any object with the same attribute
names works (the tests pass the oracle's own config dataclass)."""
import types
from dataclasses import dataclass

import numpy as np


@dataclass
class LearnerConfig:
    n_agents: int = 3
    obs_dim: int = 30
    act_dim: int = 9
    state_dim: int = 48
    hidden: int = 64                # config.py:63 hidden_size
    layer_n: int = 1                # config.py:67 layer_N
    mixer_hidden: int = 32          # config.py:101 mixer_hidden_dim
    hyper_hidden: int = 64          # config.py:103 hypernet_hidden_dim
    hyper_layers: int = 2           # config.py:105 hypernet_layers
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
    relu: bool = True
    prev_act_inp: bool = False
    gain: float = 0.01


@dataclass
class MaddpgLearnerConfig:
    """What a bench / example needs to describe an R-MADDPG / R-MATD3 learner (attribute names = the oracle's MaddpgConfig, so the CPU
    arm can be built from the same values; nothing here imports the oracle)."""
    n_agents: int = 3
    obs_dim: int = 18
    act_dim: int = 2
    state_dim: int = 54
    hidden: int = 64
    layer_n: int = 1
    feature_norm: bool = True
    relu: bool = True
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
    discrete: bool = False


class Box(object):      # duck-typed gym.spaces.Box: what the policies read is .shape / .low / .high
    def __init__(self, d, low=-1.0, high=1.0):
        self.shape = (d,)
        self.low = np.full(d, low, np.float32)
        self.high = np.full(d, high, np.float32)


class Discrete(object):  # duck-typed gym.spaces.Discrete
    def __init__(self, n):
        self.n = n


class MultiDiscrete(object):     # duck-typed envs/mpe/multi_discrete.py: the policies read the class name and .low / .high
    def __init__(self, array_of_param_array):
        self.low = np.array([x[0] for x in array_of_param_array])
        self.high = np.array([x[1] for x in array_of_param_array])
        self.num_discrete_space = self.low.shape[0]


def act_space(act, discrete=True):
    """The action space for a width: an int -> Discrete(n) (Box(n) with discrete False); a list / tuple of sub-space widths ->
    MultiDiscrete([[0, n_0 - 1], [0, n_1 - 1], ...])."""
    if isinstance(act, (list, tuple, np.ndarray)):
        return MultiDiscrete([[0, int(n) - 1] for n in act])
    return Discrete(act) if discrete else Box(act)


def act_width(act):
    """Width of the action vector of an action description of act_space (the sum of the sub-space widths for MultiDiscrete)."""
    return int(np.sum(act)) if isinstance(act, (list, tuple, np.ndarray)) else int(act)


def pd(x, p_id="policy_0"):
    """{policy_id: array}: the per-policy dict every buffer / trainer entry point of the reference takes."""
    return {p_id: x}


def qmix_args(cfg, B, **over):
    """The argparse namespace fields QMixPolicy / QMix / M_QMix read (config.py names), from a LearnerConfig-like object."""
    a = types.SimpleNamespace(
        hidden_size=cfg.hidden, layer_N=1, use_ReLU=bool(getattr(cfg, "relu", True)), use_feature_normalization=bool(cfg.feature_norm), use_orthogonal=True, gain=cfg.gain,
        use_conv1d=False, stacked_frames=1, use_rnn_layer=True, recurrent_N=1, prev_act_inp=bool(getattr(cfg, "prev_act_inp", False)), use_double_q=cfg.double_q,
        hypernet_layers=cfg.hyper_layers, mixer_hidden_dim=cfg.mixer_hidden, hypernet_hidden_dim=cfg.hyper_hidden, gamma=cfg.gamma,
        use_per=cfg.use_per, per_nu=cfg.per_nu, per_eps=cfg.per_eps, per_alpha=0.6, use_huber_loss=cfg.huber,
        huber_delta=cfg.huber_delta, max_grad_norm=cfg.max_grad_norm, lr=cfg.lr, opti_eps=cfg.opti_eps, weight_decay=0, tau=cfg.tau,
        use_popart=False, use_value_active_masks=False, use_same_share_obs=True, batch_size=B, episode_length=0,
        epsilon_start=1.0, epsilon_finish=0.05, epsilon_anneal_time=50000, use_available_actions=True)
    for k, v in over.items():
        setattr(a, k, v)
    return a


def _policy_info(cfg):
    return dict(obs_space=[cfg.obs_dim], share_obs_space=[cfg.state_dim], act_space=Discrete(cfg.act_dim),
                cent_obs_dim=cfg.state_dim, cent_act_dim=cfg.act_dim * cfg.n_agents)


def build_qmix(cfg, B, T, vdn=False, debug=False, **over):
    """(args, QMixPolicy, QMix) for recurrent QMIX / VDN.  debug=True also materialises the per-action Q values (parity tests) and keeps
    k_qhead / k_mix_core / k_qhead_bwd as separate launches; debug=False is the product configuration (fused k_mid)."""
    from offpolicy.algorithms.qmix.algorithm.QMixPolicy import QMixPolicy
    from offpolicy.algorithms.qmix.qmix import QMix
    from offpolicy._b200 import capi
    args = qmix_args(cfg, B, **over)
    pol = QMixPolicy({"args": args, "device": capi.device()}, _policy_info(cfg))
    tr = QMix(args, cfg.n_agents, {"policy_0": pol}, lambda a: "policy_0", device=capi.device(), episode_length=T, vdn=vdn)
    capi.lib().mx_qmix_set_debug(tr.handle, 1 if debug else 0)
    return args, pol, tr


def build_mqmix(cfg, B, debug=False):
    """(args, M_QMixPolicy, M_QMix): the transition-level (MLP) learner."""
    from offpolicy.algorithms.mqmix.algorithm.mQMixPolicy import M_QMixPolicy
    from offpolicy.algorithms.mqmix.mqmix import M_QMix
    from offpolicy._b200 import capi
    args = qmix_args(cfg, B)
    pol = M_QMixPolicy({"args": args, "device": capi.device()}, _policy_info(cfg))
    tr = M_QMix(args, cfg.n_agents, {"policy_0": pol}, lambda a: "policy_0", device=capi.device())
    capi.lib().mx_qmix_set_debug(tr.handle, 1 if debug else 0)
    return args, pol, tr


def make_rec_buffers(N, O, A, S, T, E, per_alpha=None, norm=False, rng="numpy", max_batch=32, avail=True):
    """RecReplayBuffer / PrioritizedRecReplayBuffer for one shared policy over N agents (rec_buffer.py:9-61, 243-270)."""
    from offpolicy.utils.rec_buffer import RecReplayBuffer, PrioritizedRecReplayBuffer
    info = {"policy_0": dict(obs_space=[O], share_obs_space=[S], act_space=Discrete(A))}
    agents = {"policy_0": list(range(N))}
    if per_alpha is None:
        return RecReplayBuffer(info, agents, E, T, True, avail, use_reward_normalization=norm, rng=rng, max_batch=max_batch)
    return PrioritizedRecReplayBuffer(per_alpha, info, agents, E, T, True, avail, use_reward_normalization=norm, rng=rng,
                                      max_batch=max_batch)


def maddpg_args(cfg, B, **over):
    """Namespace fields R_MADDPGPolicy / R_MADDPG / R_MATD3 read, from a config object with the oracle's MaddpgConfig attribute names;
    `over` sets args fields."""
    args = types.SimpleNamespace(
        hidden_size=cfg.hidden, layer_N=1, use_ReLU=bool(cfg.relu), use_feature_normalization=bool(cfg.feature_norm), use_orthogonal=True, gain=cfg.gain,
        use_conv1d=False, stacked_frames=1, use_rnn_layer=True, recurrent_N=1, prev_act_inp=False, gamma=cfg.gamma, use_per=cfg.use_per,
        per_nu=cfg.per_nu, per_eps=cfg.per_eps, use_huber_loss=cfg.huber, huber_delta=cfg.huber_delta, max_grad_norm=cfg.max_grad_norm,
        lr=cfg.lr, opti_eps=cfg.opti_eps, weight_decay=cfg.weight_decay, tau=cfg.tau, use_popart=False, use_value_active_masks=False,
        use_same_share_obs=True, batch_size=B, episode_length=0, epsilon_start=1.0, epsilon_finish=0.05, epsilon_anneal_time=50000,
        act_noise_std=0.1, target_action_noise_std=cfg.target_noise)
    for k, v in over.items():
        setattr(args, k, v)
    return args


def build_maddpg(cfg, B, T, **over):
    """(args, policy, trainer) for R-MADDPG (cfg.td3 False) / R-MATD3 (True), one shared policy; `over` sets args fields."""
    from offpolicy._b200 import capi
    if cfg.td3:
        from offpolicy.algorithms.r_matd3.algorithm.rMATD3Policy import R_MATD3Policy as Policy
        from offpolicy.algorithms.r_matd3.r_matd3 import R_MATD3 as Trainer
    else:
        from offpolicy.algorithms.r_maddpg.algorithm.rMADDPGPolicy import R_MADDPGPolicy as Policy
        from offpolicy.algorithms.r_maddpg.r_maddpg import R_MADDPG as Trainer
    args = maddpg_args(cfg, B, **over)
    info = dict(obs_space=Box(cfg.obs_dim, -np.inf, np.inf), share_obs_space=Box(cfg.state_dim, -np.inf, np.inf),
                act_space=Discrete(cfg.act_dim) if cfg.discrete else Box(cfg.act_dim), cent_obs_dim=cfg.state_dim, cent_act_dim=cfg.act_dim * cfg.n_agents)
    pol = Policy({"args": args, "device": capi.device()}, info)
    tr = Trainer(args, cfg.n_agents, {"policy_0": pol}, lambda a: "policy_0", device=capi.device(), episode_length=T)
    return args, pol, tr


def _mlp_maddpg_classes(td3):
    if td3:
        from offpolicy.algorithms.matd3.algorithm.MATD3Policy import MATD3Policy as Policy
        from offpolicy.algorithms.matd3.matd3 import MATD3 as Trainer
    else:
        from offpolicy.algorithms.maddpg.algorithm.MADDPGPolicy import MADDPGPolicy as Policy
        from offpolicy.algorithms.maddpg.maddpg import MADDPG as Trainer
    return Policy, Trainer


def mlp_maddpg_args(B, **over):
    """Namespace fields MADDPGPolicy / MADDPG / MATD3 read (config.py defaults); `over` sets args fields."""
    args = types.SimpleNamespace(
        hidden_size=64, layer_N=1, use_ReLU=True, use_feature_normalization=True, use_orthogonal=True, gain=0.01, use_conv1d=False,
        stacked_frames=1, gamma=0.99, use_per=False, per_nu=0.9, per_eps=1e-6, use_huber_loss=False, huber_delta=10.0, max_grad_norm=10.0,
        lr=7e-4, opti_eps=1e-5, weight_decay=0.0, tau=0.005, use_popart=False, use_value_active_masks=False, use_same_share_obs=True,
        batch_size=B, epsilon_start=1.0, epsilon_finish=0.05, epsilon_anneal_time=50000, act_noise_std=0.1, target_action_noise_std=0.2)
    for k, v in over.items():
        setattr(args, k, v)
    return args


def build_mlp_maddpg(n_agents, obs_dim, act_dim, state_dim, B, discrete=True, td3=False, **over):
    """(args, policy, trainer) for the transition-level MADDPG (td3 False) / MATD3 (True), one shared policy; `over` sets args fields.
    act_dim: an int, or a list of sub-space widths for a MultiDiscrete action space (act_space)."""
    from offpolicy._b200 import capi
    Policy, Trainer = _mlp_maddpg_classes(td3)
    args = mlp_maddpg_args(B, **over)
    info = dict(obs_space=Box(obs_dim, -np.inf, np.inf), share_obs_space=Box(state_dim, -np.inf, np.inf),
                act_space=act_space(act_dim, discrete), cent_obs_dim=state_dim, cent_act_dim=act_width(act_dim) * n_agents)
    pol = Policy({"args": args, "device": capi.device()}, info)
    tr = Trainer(args, n_agents, {"policy_0": pol}, lambda a: "policy_0", device=capi.device())
    return args, pol, tr


def build_mlp_maddpg_multi(specs, state_dim, B, discrete=True, td3=False, **over):
    """(args, {policy_id: policy}, trainer, agents) for the transition-level MADDPG / MATD3 with several policies (share_policy off).
    specs: one (obs_dim, act_dim) or (obs_dim, act_dim, n_agents) per policy, act_dim as in act_space (a list of sub-space widths gives a
    MultiDiscrete policy, whatever `discrete` says); policy_i controls the next n_agents agents (1 by default),
    agents = {policy_id: [agent ids]}.  The policies are constructed in id order, as train_mpe.py:139-150 does."""
    from offpolicy._b200 import capi
    Policy, Trainer = _mlp_maddpg_classes(td3)
    args = mlp_maddpg_args(B, **over)
    specs = [tuple(s) + (1,) * (3 - len(s)) for s in specs]
    total = sum(act_width(a) * n for _, a, n in specs)
    pols, agents, mapping, nxt = {}, {}, {}, 0
    for i, (o, a, n) in enumerate(specs):
        p = "policy_%d" % i
        info = dict(obs_space=Box(o, -np.inf, np.inf), share_obs_space=Box(state_dim, -np.inf, np.inf),
                    act_space=act_space(a, discrete), cent_obs_dim=state_dim, cent_act_dim=total)
        pols[p] = Policy({"args": args, "device": capi.device()}, info)
        agents[p] = list(range(nxt, nxt + n))
        mapping.update({k: p for k in agents[p]})
        nxt += n
    tr = Trainer(args, nxt, pols, lambda k: mapping[k], device=capi.device())
    return args, pols, tr, agents
