"""Drop-in `MADDPGPolicy` (reference: offpolicy/algorithms/maddpg/algorithm/MADDPGPolicy.py) of the transition-level MADDPG / MATD3
for Box, Discrete and MultiDiscrete action spaces.  `actor`, `critic`, `target_actor`, `target_critic` are named views (reference state_dict keys) of
the flat device vectors the CUDA learner (mx_maddpg with cfg.mlp) updates in place; the two Adam states live beside them.

The critic's Q heads are a plain Python list in the reference (maddpg/algorithm/actor_critic.py:67): they are not parameters, so no
optimiser, clip, state_dict or target update ever touches them, and the target critic keeps the heads of its own construction
(SURVEY.md App. D-6).  Here they sit behind the trunk of each critic vector (`critic_heads` / `target_critic_heads`), outside the range
the learner trains and averages; `critic.state_dict()` holds the trunk only, with the reference's `mlp.*` keys.

Rollout-time `get_actions` is one launch of k_policy_step in its MLP mode; the exploration / Gumbel / Gaussian draws are made on the
host with the reference's calls, in its order (MADDPGPolicy.py:63-139).

MultiDiscrete actions (e.g. simple_reference: move and speak) are one one-hot block per sub-space, as in the reference: `act_dim` is the
ndarray of the sub-space widths (util.py:237, the runner takes `np.sum` of it) and `output_dim` their sum, the width of the action
vector.  The actor has one head per sub-space, `act.action_outs.i`, each initialised in order; the learner sees them as one head of
`output_dim` rows.  Arg-max, Gumbel draws and random actions are made block by block, and the available-action mask is ignored."""
import numpy as np
import torch

from offpolicy._b200 import capi
from offpolicy._b200.flat import FlatModule, mlp_init
from offpolicy._b200.host_util import space_dim, is_discrete, LinearDecay
from offpolicy.algorithms.r_maddpg.algorithm.rMADDPGPolicy import maddpg_cfg_struct, maddpg_entries, onehot_from_logits, gumbel_softmax_hard


def _load(mods, sd):
    for m in mods:
        m.load_state_dict({k: sd[k] for k in m.views}, strict=True)


class MADDPGPolicy(object):
    def __init__(self, config, policy_config, target_noise=None, td3=False, train=True):
        self.config = config
        self.device = config["device"]
        self.args = self.config["args"]
        self.tau, self.lr, self.opti_eps = self.args.tau, self.args.lr, self.args.opti_eps
        self.weight_decay = getattr(self.args, "weight_decay", 0)
        if getattr(self.args, "use_conv1d", False):
            raise NotImplementedError("B200 MADDPG path requires use_conv1d=False")
        if getattr(self.args, "layer_N", 1) != 1 or getattr(self.args, "hidden_size", 64) != 64:
            raise NotImplementedError("B200 MADDPG path requires layer_N=1, hidden_size=64")
        self.central_obs_dim, self.central_act_dim = policy_config["cent_obs_dim"], policy_config["cent_act_dim"]
        self.obs_space, self.act_space = policy_config["obs_space"], policy_config["act_space"]
        self.multidiscrete = "MultiDiscrete" in self.act_space.__class__.__name__
        self.obs_dim = space_dim(self.obs_space)
        if self.multidiscrete:          # util.py:237 get_dim_from_space: the sub-space widths, an ndarray
            self.act_dim = np.asarray(self.act_space.high) - np.asarray(self.act_space.low) + 1
            self.act_segs = [int(n) for n in self.act_dim]
            self.output_dim = int(sum(self.act_segs))
        else:
            self.act_dim = space_dim(self.act_space)
            self.act_segs = None
            self.output_dim = self.act_dim
        self.hidden_size = self.args.hidden_size
        self.discrete = is_discrete(self.act_space)
        self.td3, self.target_noise = bool(td3), target_noise
        if self.discrete and train:
            self.exploration = LinearDecay(self.args.epsilon_start, self.args.epsilon_finish, self.args.epsilon_anneal_time)   # :57-60
        capi.lib()
        self.dev = capi.device()
        self.num_q = 2 if td3 else 1
        cfg = maddpg_cfg_struct(self.args, 1, self.obs_dim, self.output_dim, self.central_obs_dim, 1, 1, td3, target_noise, 1, self.discrete,
                                mlp=True, act_segs=self.act_segs)
        # the critic input is [cent_obs | centralised action]: cent_act_dim = n_agents * output_dim with one shared policy, the total
        # action width of all agents with one policy per agent (which need not be a multiple of this policy's output_dim)
        cfg.n_agents = max(1, self.central_act_dim // self.output_dim)
        cfg.cent_act_dim = self.central_act_dim
        self._a_entries, self.Pa = maddpg_entries(cfg, 0)
        self._c_entries, self.Pc = maddpg_entries(cfg, 1)
        self._h_entries, _ = maddpg_entries(cfg, 2)
        z = lambda n: torch.zeros(n, dtype=torch.float32, device=self.dev)
        self.actor_vecs = [z(self.Pa) for _ in range(4)]      # theta, target, adam m, adam v
        self.critic_vecs = [z(self.Pc) for _ in range(4)]
        self.actor = FlatModule(self.actor_vecs[0], self._a_entries, "")
        self.target_actor = FlatModule(self.actor_vecs[1], self._a_entries, "")
        self.critic = FlatModule(self.critic_vecs[0], self._c_entries, "")
        self.target_critic = FlatModule(self.critic_vecs[1], self._c_entries, "")
        self.critic_heads = FlatModule(self.critic_vecs[0], self._h_entries, "")
        self.target_critic_heads = FlatModule(self.critic_vecs[1], self._h_entries, "")
        relu = bool(getattr(self.args, "use_ReLU", True))
        fn = bool(getattr(self.args, "use_feature_normalization", True))
        if self.multidiscrete:        # act.py:15-17: one Linear per sub-space, each with its own init call, in order
            a_heads = [("act.action_outs.%d" % i, n, self.args.gain) for i, n in enumerate(self.act_segs)]
        else:
            a_heads = [("act.action_out", self.act_dim, self.args.gain)]                              # act.py:18-19
        c_heads = [("q_outs.%d" % k, 1, 1.0) for k in range(self.num_q)]                              # actor_critic.py:64-67
        c_in = self.central_obs_dim + self.central_act_dim
        # construction order of MADDPGPolicy.py:43-51: actor, critic (trunk, heads), target actor, target critic, then the two syncs
        _load([self.actor], mlp_init(self.obs_dim, self.hidden_size, a_heads, self.args.use_orthogonal, relu, fn))
        _load([self.critic, self.critic_heads], mlp_init(c_in, self.hidden_size, c_heads, self.args.use_orthogonal, relu, fn))
        _load([self.target_actor], mlp_init(self.obs_dim, self.hidden_size, a_heads, self.args.use_orthogonal, relu, fn))
        _load([self.target_critic, self.target_critic_heads], mlp_init(c_in, self.hidden_size, c_heads, self.args.use_orthogonal, relu, fn))
        self.target_actor.load_state_dict(self.actor.state_dict())
        self.target_critic.load_state_dict(self.critic.state_dict())      # the trunk only: the target heads stay their own
        self._roll = None
        self._trainer = None
        self._handle = None          # this policy's mx_maddpg (created by the trainer)

    def _forward(self, theta, obs):
        if self._roll is None:
            from offpolicy._b200.rollout import PolicyStepper
            self._roll = PolicyStepper(self.obs_dim, self.output_dim, mlp=True, feature_norm=bool(getattr(self.args, "use_feature_normalization", True)),
                                       tanh=not getattr(self.args, "use_ReLU", True))
        out, _, _, _ = self._roll.step(theta, np.asarray(obs, dtype=np.float32), None, want_greedy=False)
        return torch.from_numpy(out)

    def get_actions(self, obs, available_actions=None, t_env=None, explore=False, use_target=False, use_gumbel=False):
        """MADDPGPolicy.py:63-119."""
        batch_size = obs.shape[0]
        eps = None
        actor_out = self._forward(self.actor_vecs[1] if use_target else self.actor_vecs[0], obs)
        if self.multidiscrete:            # :73-89, block by block in sub-space order; available_actions is not used
            blocks = actor_out.split(self.act_segs, dim=-1)
            if use_gumbel or (use_target and self.target_noise is not None):
                actions = torch.cat([gumbel_softmax_hard(a) for a in blocks], dim=-1)
            elif explore:
                onehot_actions = torch.cat([gumbel_softmax_hard(a) for a in blocks], dim=-1)
                eps = self.exploration.eval(t_env)
                rand_numbers = np.random.rand(batch_size, 1)
                take_random = (rand_numbers < eps).astype(int).reshape(-1, 1)
                random_actions = torch.cat([torch.distributions.OneHotCategorical(logits=torch.ones(batch_size, n)).sample()
                                            for n in self.act_segs], dim=1)
                actions = (1 - take_random) * onehot_actions.numpy() + take_random * random_actions.numpy()
            else:
                actions = torch.cat([onehot_from_logits(a) for a in blocks], dim=-1)
        elif self.discrete:
            if use_gumbel or (use_target and self.target_noise is not None):
                actions = gumbel_softmax_hard(actor_out, available_actions)
            elif explore:
                onehot_actions = gumbel_softmax_hard(actor_out, available_actions)
                eps = self.exploration.eval(t_env)
                rand_numbers = np.random.rand(batch_size, 1)
                logits = torch.ones(batch_size, self.act_dim)
                if available_actions is not None:
                    logits[torch.as_tensor(np.asarray(available_actions), dtype=torch.float32) == 0] = -1e10     # avail_choose
                random_actions = torch.distributions.OneHotCategorical(logits=logits).sample().numpy()
                take_random = (rand_numbers < eps).astype(int)
                actions = (1 - take_random) * onehot_actions.numpy() + take_random * random_actions
            else:
                actions = onehot_from_logits(actor_out, available_actions)
        elif explore:
            actions = torch.empty(actor_out.shape).normal_(mean=0, std=self.args.act_noise_std) + actor_out       # util.py:217-218
        elif use_target and self.target_noise is not None:
            actions = torch.empty(actor_out.shape).normal_(mean=0, std=float(self.target_noise)) + actor_out
        else:
            actions = actor_out
        return actions, eps

    def get_random_actions(self, obs, available_actions=None):
        """MADDPGPolicy.py:121-139."""
        batch_size = obs.shape[0]
        if self.multidiscrete:            # :126-129: one OneHotCategorical per sub-space
            return np.concatenate([torch.distributions.OneHotCategorical(logits=torch.ones(batch_size, n)).sample().numpy()
                                   for n in self.act_segs], axis=-1)
        if self.discrete:
            logits = torch.ones(batch_size, self.act_dim)
            if available_actions is not None:
                logits[torch.as_tensor(np.asarray(available_actions), dtype=torch.float32) == 0] = -1e10
            return torch.distributions.OneHotCategorical(logits=logits).sample().numpy()
        return np.random.uniform(self.act_space.low, self.act_space.high, size=(batch_size, self.act_dim))

    def soft_target_updates(self):
        """MADDPGPolicy.py:141-145: Polyak over the critic trunk and the whole actor."""
        if self._handle is None:
            raise RuntimeError("soft_target_updates: no trainer attached")
        capi.check(capi.lib().mx_maddpg_soft_update(self._handle, capi.stream_ptr()))

    def hard_target_updates(self):
        """MADDPGPolicy.py:147-151: copy the critic trunk and the whole actor."""
        self.target_critic.load_state_dict(self.critic.state_dict())
        self.actor_vecs[1].copy_(self.actor_vecs[0])
