"""Drop-in `offpolicy.utils.mlp_buffer` (reference: offpolicy/utils/mlp_buffer.py) on the HBM-resident replay of libmarl_b200.

A transition is stored as an EPISODE OF LENGTH 1 of the episode replay (csrc/replay.cu): step 0 = (obs, share_obs, avail_acts),
step 1 = (next_obs, next_share_obs, next_avail_acts), plus acts / rewards / dones / dones_env of the single step.  Insert, ring
wrap, uniform and prioritised sampling (device-side fp64 trees), running reward statistics and the 128-bit gather kernel are the ones
of the recurrent path; `sample()` returns the reference's 13-tuple (11 fields + importance weights + indices, the last two None for
uniform sampling) whose entries materialise the reference's NumPy layout
on access while the B200 trainers (algorithms/mqmix/mqmix.py, algorithms/maddpg/maddpg.py) read the device-side batch directly.
`valid_transition` is kept twice: a host array for `materialize`, and a device copy [buffer_size][N] (`valid_dev`) that the MADDPG /
MATD3 actor loss reads through the batch's sampled indices.

Several policies (`--share_policy` off, one policy per agent): one store per policy with its own observation / action widths, its own
`valid_dev` and its own PER trees.  A sample draws ONE index set and applies it to every store, as the reference does
(mlp_buffer.py:100-106 uniform, 285-296 prioritised from the updated policy's tree).
"""
import numpy as np
import torch

from offpolicy.utils.rec_buffer import PolicyStoresState, RecPolicyBuffer, _LazyField, sample_shared_uniform, share_indices

MLP_FIELDS = ("obs", "share_obs", "acts", "rewards", "next_obs", "next_share_obs", "dones", "dones_env", "valid_transition",
              "avail_acts", "next_avail_acts")


class MlpSampledBatch(object):
    """The reference's sample tuple (mlp_buffer.py:80-110 / :300-320) + a handle on the device-side batch."""

    __slots__ = ("buffers", "B", "serial", "_p_ids", "_items", "_n", "host_inds")

    def __init__(self, buffers, B, p_ids, weights=None, idxes=None, per=False, host_inds=None):
        self.buffers, self.B, self._p_ids = buffers, B, p_ids
        self.serial = {p: buffers[p].rep.sample_serial for p in p_ids}
        self._n = 13          # uniform sampling returns (..., None, None) like the reference (mlp_buffer.py:98)
        self._items = [None] * 11 + [weights, idxes]
        self.host_inds = host_inds

    def __len__(self):
        return self._n

    def __getitem__(self, i):
        if isinstance(i, slice):
            return tuple(self[k] for k in range(*i.indices(self._n)))
        if i < 0:
            i += self._n
        if i >= self._n:
            raise IndexError(i)
        v = self._items[i]
        if v is None and i < 11:
            v = self._items[i] = _LazyField(self, MLP_FIELDS[i], self._p_ids)
        return v

    def __iter__(self):
        return (self[k] for k in range(self._n))

    def materialize(self, p_id, field):
        buf = self.buffers[p_id]
        if buf.rep.sample_serial != self.serial[p_id]:
            raise RuntimeError("this sample was overwritten by a later sample() call (the device batch region is reused)")
        return buf.materialize(field, self.B, self.host_inds)


class MlpPolicyBuffer(object):
    """One policy's transition store (mlp_buffer.py:113-240) = an episode replay with episode_length 1."""

    def __init__(self, buffer_size, num_agents, obs_space, share_obs_space, act_space, use_same_share_obs, use_avail_acts,
                 use_reward_normalization=False, use_per=False, per_alpha=0.0, max_batch=None):
        self.buffer_size = int(buffer_size)
        self.num_agents = int(num_agents)
        self.use_avail_acts = bool(use_avail_acts)
        self.rep = RecPolicyBuffer(buffer_size, 1, num_agents, obs_space, share_obs_space, act_space, use_same_share_obs, use_avail_acts,
                                   use_reward_normalization, use_per=use_per, per_alpha=per_alpha, max_batch=max_batch or 1024)
        self.valid_transition = np.zeros((self.buffer_size, self.num_agents, 1), dtype=np.float32)      # mlp_buffer.py:156
        self.valid_dev = torch.zeros(self.buffer_size, self.num_agents, dtype=torch.float32, device=self.rep.dev)

    @property
    def filled_i(self):
        return self.rep.filled_i

    @property
    def current_i(self):
        return self.rep.current_i

    def __len__(self):
        return self.filled_i

    def insert(self, num_insert_steps, obs, share_obs, acts, rewards, next_obs, next_share_obs, dones, dones_env, valid_transition,
               avail_acts=None, next_avail_acts=None):
        n = int(num_insert_steps)
        obs, next_obs = np.asarray(obs, dtype=np.float32), np.asarray(next_obs, dtype=np.float32)
        assert obs.shape[0] == n, ("different size!")                                                   # mlp_buffer.py:175
        f32 = lambda x: np.asarray(x, dtype=np.float32)
        av = np.stack([f32(avail_acts), f32(next_avail_acts)], 0) if self.use_avail_acts else None
        idx = self.rep.insert(n, np.stack([obs, next_obs], 0), np.stack([f32(share_obs), f32(next_share_obs)], 0), f32(acts)[None],
                              f32(rewards)[None], f32(dones)[None], f32(dones_env).reshape(1, n, 1), av)
        self.valid_transition[idx] = f32(valid_transition).reshape(n, self.num_agents, 1)
        self.valid_dev[torch.from_numpy(np.asarray(idx, dtype=np.int64)).to(self.rep.dev)] = \
            torch.from_numpy(self.valid_transition[idx, :, 0]).to(self.rep.dev)
        return idx

    # -- reference layout of one sampled field (mlp_buffer.py:203-240: `_cast` = transpose(1, 0, 2)) ----------------
    def materialize(self, field, B, host_inds=None):
        rep = self.rep
        if field == "valid_transition":
            inds = host_inds if host_inds is not None else np.asarray(rep.sampled_indices(B))
            return self.valid_transition[np.asarray(inds)].transpose(1, 0, 2)
        if field in ("avail_acts", "next_avail_acts") and not self.use_avail_acts:
            return None
        step = 1 if field.startswith("next_") else 0
        base = {"next_obs": "obs", "next_share_obs": "share_obs", "next_avail_acts": "avail_acts"}.get(field, field)
        v = rep._field_view(base, True, B)
        if base in ("obs", "avail_acts"):
            out = v[:, step].permute(1, 0, 2)                       # (B, N, D) -> (N, B, D)
        elif base == "share_obs":
            out = v[:, step]                                        # (B, S)
        elif base == "acts":
            out = v[:, 0].permute(1, 0, 2)
        elif base in ("rewards", "dones"):
            out = v.reshape(B, self.num_agents).permute(1, 0).unsqueeze(-1)
        else:                                                       # dones_env
            out = v.reshape(B, 1)
        return out.contiguous().cpu().numpy()

    # -- checkpoint / resume: the episode replay's persistent part + valid_transition -------------------------------------
    def state_dict(self):
        return {"rep": self.rep.state_dict(), "valid_transition": self.valid_transition.copy()}

    def load_state_dict(self, sd):
        valid = np.asarray(sd["valid_transition"], dtype=np.float32)
        if valid.shape != self.valid_transition.shape:
            raise ValueError("replay checkpoint has valid_transition of shape %s, this buffer %s" % (valid.shape, self.valid_transition.shape))
        self.rep.load_state_dict(sd["rep"])          # checks capacity, agents and widths
        self.valid_transition[...] = valid
        self.valid_dev.copy_(torch.from_numpy(valid[:, :, 0]).to(self.valid_dev.device))     # in place: learners keep its pointer


class MlpReplayBuffer(PolicyStoresState):
    def __init__(self, policy_info, policy_agents, buffer_size, use_same_share_obs, use_avail_acts, use_reward_normalization=False,
                 rng="numpy", max_batch=None, _per_alpha=None):
        self.policy_info = policy_info
        self.rng = rng
        self.policy_buffers = {
            p_id: MlpPolicyBuffer(buffer_size, len(policy_agents[p_id]), policy_info[p_id]["obs_space"], policy_info[p_id]["share_obs_space"],
                                  policy_info[p_id]["act_space"], use_same_share_obs, use_avail_acts, use_reward_normalization,
                                  use_per=_per_alpha is not None, per_alpha=_per_alpha or 0.0, max_batch=max_batch)
            for p_id in policy_info.keys()}

    def _first(self):
        return self.policy_buffers["policy_0"] if "policy_0" in self.policy_buffers else next(iter(self.policy_buffers.values()))

    def __len__(self):
        return self._first().filled_i              # mlp_buffer.py:44-45: the length of policy_0's store

    def insert(self, num_insert_steps, obs, share_obs, acts, rewards, next_obs, next_share_obs, dones, dones_env, valid_transition,
               avail_acts, next_avail_acts):
        idx_range = None
        for p_id in self.policy_info.keys():
            av = None if avail_acts is None or avail_acts[p_id] is None else np.array(avail_acts[p_id])
            nav = None if next_avail_acts is None or next_avail_acts[p_id] is None else np.array(next_avail_acts[p_id])
            idx_range = self.policy_buffers[p_id].insert(num_insert_steps, np.array(obs[p_id]), np.array(share_obs[p_id]), np.array(acts[p_id]),
                                                         np.array(rewards[p_id]), np.array(next_obs[p_id]), np.array(next_share_obs[p_id]),
                                                         np.array(dones[p_id]), np.array(dones_env[p_id]), np.array(valid_transition[p_id]),
                                                         av, nav)
        return idx_range

    def seed_device_rng(self, seed):
        self.rng = "device"
        for b in self.policy_buffers.values():
            b.rep.seed_device_rng(seed)

    def sample(self, batch_size):
        inds = sample_shared_uniform([b.rep for b in self.policy_buffers.values()], self._first().rep, batch_size, self.rng,
                                     self.__len__())                                  # np.random.choice(len, B), mlp_buffer.py:100
        return MlpSampledBatch(self.policy_buffers, batch_size, list(self.policy_info.keys()), host_inds=inds)


class PrioritizedMlpReplayBuffer(MlpReplayBuffer):
    """Proportional prioritised transition replay (mlp_buffer.py:243-340); fp64 trees on the device."""

    def __init__(self, alpha, policy_info, policy_agents, buffer_size, use_same_share_obs, use_avail_acts, use_reward_normalization=False,
                 rng="numpy", max_batch=None):
        super().__init__(policy_info, policy_agents, buffer_size, use_same_share_obs, use_avail_acts, use_reward_normalization, rng=rng,
                         max_batch=max_batch, _per_alpha=float(alpha))
        self.alpha = alpha

    def sample(self, batch_size, beta=0, p_id=None):
        assert len(self) > batch_size, "Not enough samples in the buffer!"                    # mlp_buffer.py:297
        assert beta > 0                                                                        # mlp_buffer.py:298
        rep = (self.policy_buffers[p_id] if p_id else self._first()).rep
        if self.rng != "device":
            rep.adopt_numpy_rng()                 # masses come from NumPy's global stream like np.random.random (mlp_buffer.py:287)
            rep.sample_device_per(batch_size, beta)
            rep.export_rng_to_numpy()
        else:
            rep.sample_device_per(batch_size, beta)
        share_indices([b.rep for b in self.policy_buffers.values()], rep, batch_size)      # p_id's draw selects every store's rows
        return MlpSampledBatch(self.policy_buffers, batch_size, list(self.policy_info.keys()), weights=rep.sampled_weights(batch_size),
                               idxes=rep.sampled_indices(batch_size), per=True)

    def update_priorities(self, idxes, priorities, p_id=None):
        (self.policy_buffers[p_id] if p_id else self._first()).rep.update_priorities(idxes, priorities)     # p_id's tree only
