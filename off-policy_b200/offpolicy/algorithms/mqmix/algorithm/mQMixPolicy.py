"""Drop-in `M_QMixPolicy` (reference: offpolicy/algorithms/mqmix/algorithm/mQMixPolicy.py): the non-recurrent agent Q-network
(MLPBase + Linear head, mqmix/algorithm/agent_q_function.py) as named views of the flat device vector the CUDA learner trains.

Update-time Q evaluation lives in the learner kernels (the head is the first act_dim rows of the otherwise empty weight_ih slot, so
the time-batched front kernels of the recurrent path compute it unchanged); the rollout-time `get_actions` is one launch of
k_policy_step in its MLP mode, with the epsilon-greedy draws on the host in the reference's order (mQMixPolicy.py:60-110).
"""
import numpy as np
import torch

from offpolicy._b200 import capi
from offpolicy._b200.flat import FlatModule, mlp_init
from offpolicy._b200.host_util import LinearDecay, space_dim, is_discrete, onehot
from offpolicy.algorithms.qmix.algorithm.QMixPolicy import qmix_cfg_struct, param_entries


def mlp_reference_style_init(entries, in_dim, hidden, act_dim, gain, use_orthogonal=True, use_relu=True):
    """Initial weights in the reference's construction order (MLPBase, mlp.py:14-29, then ACTLayer, act.py:10-20) so that a seeded run
    consumes torch's generator identically; keys of the q_network views."""
    fn = any(n.endswith("mlp.feature_norm.weight") for n, *_ in entries)      # absent with --use_feature_normalization off
    return mlp_init(in_dim, hidden, [("q.action_out", act_dim, gain)], use_orthogonal, use_relu, fn)


class M_QMixPolicy(object):
    def __init__(self, config, policy_config, train=True):
        self.args = config["args"]
        self.device = config["device"]
        self.obs_space = policy_config["obs_space"]
        self.obs_dim = space_dim(self.obs_space)
        self.act_space = policy_config["act_space"]
        self.act_dim = space_dim(self.act_space)
        self.output_dim = self.act_dim
        self.hidden_size = self.args.hidden_size
        self.central_obs_dim = policy_config["cent_obs_dim"]
        self.discrete = is_discrete(self.act_space)
        self.multidiscrete = "MultiDiscrete" in self.act_space.__class__.__name__
        if self.multidiscrete:
            raise NotImplementedError("B200 M-QMIX path: MultiDiscrete action spaces are not implemented")
        for flag, want in (("use_conv1d", False),):
            if getattr(self.args, flag, want) != want:
                raise NotImplementedError("B200 M-QMIX path requires %s=%s" % (flag, want))
        if getattr(self.args, "layer_N", 1) != 1:
            raise NotImplementedError("B200 M-QMIX path requires layer_N=1")
        capi.lib()
        self.dev = capi.device()
        cfg = qmix_cfg_struct(self.args, 1, self.obs_dim, self.act_dim, 1, 1, 1, vdn=True, mlp=True)
        entries, total = param_entries(cfg)
        self._entries = entries
        flat = torch.zeros(total, dtype=torch.float32, device=self.dev)
        self.q_network = FlatModule(flat, entries, "agent.")
        self.q_network.load_state_dict(mlp_reference_style_init(entries, self.obs_dim, self.hidden_size, self.act_dim, self.args.gain,
                                                                self.args.use_orthogonal, use_relu=bool(getattr(self.args, "use_ReLU", True))))
        self._roll = None
        if train:
            self.exploration = LinearDecay(self.args.epsilon_start, self.args.epsilon_finish, self.args.epsilon_anneal_time)

    # -- rollout-time surface ------------------------------------------------------------------------------------
    def _step(self, obs, available_actions=None):
        if self._roll is None:
            from offpolicy._b200.rollout import PolicyStepper
            self._roll = PolicyStepper(self.obs_dim, self.act_dim, mlp=True, feature_norm=bool(getattr(self.args, "use_feature_normalization", True)),
                                       tanh=not getattr(self.args, "use_ReLU", True))
        q, _, greedy, greedy_q = self._roll.step(self.q_network.flat, obs, None, available_actions)
        return q, greedy, greedy_q

    def get_q_values(self, obs_batch, action_batch=None):
        q, _, _ = self._step(np.asarray(obs_batch, dtype=np.float32))
        q = torch.from_numpy(q)
        if action_batch is not None:                                                     # mQMixPolicy.py:44-58
            a = torch.as_tensor(np.asarray(action_batch)).long()
            return torch.gather(q, 1, a.unsqueeze(dim=-1))
        return q

    def get_actions(self, obs_batch, available_actions=None, t_env=None, explore=False):
        obs = np.asarray(obs_batch, dtype=np.float32)
        batch = obs.shape[0]
        _, greedy, greedy_q = self._step(obs, available_actions)
        greedy_Qs = torch.from_numpy(greedy_q)
        if explore:
            eps = self.exploration.eval(t_env)
            rand = np.random.rand(batch)                                                  # mQMixPolicy.py:95
            logits = torch.ones(batch, self.act_dim)
            if available_actions is not None:
                logits[torch.as_tensor(np.asarray(available_actions)) == 0] = -1e10
            random_actions = torch.distributions.Categorical(logits=logits).sample().numpy()
            take = (rand < eps).astype(int)
            return onehot((1 - take) * greedy + take * random_actions, self.act_dim), greedy_Qs
        return onehot(greedy, self.act_dim), greedy_Qs.unsqueeze(-1)

    def get_random_actions(self, obs, available_actions=None):
        batch = obs.shape[0]
        logits = torch.ones(batch, self.act_dim)
        if available_actions is not None:
            logits[torch.as_tensor(np.asarray(available_actions)) == 0] = -1e10
        return torch.distributions.OneHotCategorical(logits=logits).sample().numpy()

    def parameters(self):
        return self.q_network.parameters()

    def load_state(self, source_policy):
        self.q_network.load_state_dict(source_policy.q_network.state_dict())
