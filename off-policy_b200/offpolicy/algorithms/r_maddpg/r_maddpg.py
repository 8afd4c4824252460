"""Drop-in `R_MADDPG` trainer (reference: offpolicy/algorithms/r_maddpg/r_maddpg.py) on the sm_100a learner.

`shared_train_policy_on_batch(p_id, batch)` = one `mx_maddpg_step`: target-actor next actions, critic sequence + target
branch steps, TD target, critic loss/backward/Adam, then (every `actor_update_interval`-th call) the actor update through
the updated critic -- all on the device.  MATD3's Gaussian target-action noise is drawn on the host with the reference's
own call (`torch.empty(shape).normal_`, utils/util.py:217-218) so a seeded run consumes torch's CPU RNG identically; for
Discrete actors the Gumbel draws of the target actions (MATD3) and of the actor update (`use_gumbel=True`, r_maddpg.py:277) are
drawn the same way (utils/util.py:127-130), in the reference's order.  `use_device_noise(gen)` makes the same draws on the device instead
(offpolicy/_b200/torch_rng.py).
`cent_train_policy_on_batch` (per-agent centralised observations) is unusable in the reference (SURVEY.md App. D-7) and is not built."""
import numpy as np
import torch

from offpolicy._b200 import capi
from offpolicy._b200.maddpg_trainer import MaddpgTrainer
from offpolicy.algorithms.r_maddpg.algorithm.rMADDPGPolicy import maddpg_cfg_struct, sample_gumbel
from offpolicy.utils.rec_buffer import SampledBatch


class _HostBatchC(object):
    """Device copy of a reference-layout NumPy batch."""

    def __init__(self, cfg, dev):
        B, T, N = cfg.max_batch, cfg.episode_len, cfg.n_agents
        r4 = lambda v: (v + 3) // 4 * 4
        self.cfg = cfg
        self.obs_ld, self.share_ld, self.act_ld = r4(cfg.obs_dim), r4(cfg.state_dim), r4(cfg.act_dim)
        z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)
        self.obs, self.share, self.acts = z(B, T + 1, N, self.obs_ld), z(B, T + 1, self.share_ld), z(B, T, N, self.act_ld)
        self.rew, self.dones, self.dones_env, self.weights = z(B, T, N), z(B, T, N), z(B, T), z(B)
        self.avail = None
        self.dev = dev

    def pack(self, batch, p_id, use_per):
        obs, share, acts, rew, dones, dones_env, _avail, weights, _idx = batch
        c = self.cfg
        t = lambda x: torch.as_tensor(np.asarray(x), dtype=torch.float32).to(self.dev)
        o = t(obs[p_id])
        B = o.shape[2]
        self.obs[:B, :, :, :c.obs_dim] = o.permute(2, 1, 0, 3)
        self.share[:B, :, :c.state_dim] = t(share[p_id]).permute(1, 0, 2)
        self.acts[:B, :, :, :c.act_dim] = t(acts[p_id]).permute(2, 1, 0, 3)
        self.rew[:B] = t(rew[p_id])[..., 0].permute(2, 1, 0)
        self.dones[:B] = t(dones[p_id])[..., 0].permute(2, 1, 0)
        self.dones_env[:B] = t(dones_env[p_id])[..., 0].permute(1, 0)
        if use_per:
            self.weights[:B] = t(weights)
        has_avail = _avail is not None and _avail.get(p_id) is not None
        if has_avail:
            if self.avail is None:
                self.avail = torch.ones(c.max_batch, c.episode_len + 1, c.n_agents, self.act_ld, dtype=torch.float32, device=self.dev)
            self.avail[:B, :, :, :c.act_dim] = t(_avail[p_id]).permute(2, 1, 0, 3)
        b = capi.Batch()
        b.B, b.obs_ld, b.share_ld, b.act_ld = B, self.obs_ld, self.share_ld, self.act_ld
        b.obs, b.share, b.acts = self.obs.data_ptr(), self.share.data_ptr(), self.acts.data_ptr()
        b.rewards, b.dones, b.dones_env = self.rew.data_ptr(), self.dones.data_ptr(), self.dones_env.data_ptr()
        b.weights = self.weights.data_ptr() if use_per else None
        b.avail = self.avail.data_ptr() if has_avail else None
        return b


class R_MADDPG(MaddpgTrainer):
    _popart_msg = "B200 R-MADDPG path: --use_popart is not implemented (the reference's PopArt target is used only there)"
    _cent_msg = "cent_train_policy_on_batch is unusable in the reference (missing train_info['update_actor']) and is not built"
    _idx_field = 8

    def __init__(self, args, num_agents, policies, policy_mapping_fn, device=None, episode_length=None, actor_update_interval=1):
        self.episode_length = T = args.episode_length if episode_length is None else episode_length
        # noise rows [B][T+1][N][A]: the target actions' draws cover every step, the actor update's obs[:-1]
        self.noise_steps, self.noise_rows = T + 1, {"target": (0, T + 1), "actor": (0, T)}
        MaddpgTrainer.__init__(self, args, num_agents, policies, policy_mapping_fn, device, actor_update_interval)

    def _cfg(self, pol, n_agents, cent_act_dim, act_offset):
        return maddpg_cfg_struct(self.args, n_agents, pol.obs_dim, pol.act_dim, pol.central_obs_dim, self.episode_length, self.max_batch,
                                 pol.td3, pol.target_noise if pol.td3 else 0.0, self.actor_update_interval, pol.discrete,
                                 cent_act_dim=cent_act_dim, act_offset=act_offset)

    def _device_batch(self, batch, p_id="policy_0"):
        if isinstance(batch, SampledBatch):
            buf = batch.buffers[p_id]
            if buf.sample_serial != batch.serial[p_id]:
                raise RuntimeError("stale sample: the buffer has been sampled again since this batch was drawn")
            return buf.batch_struct(batch.B)
        e = self._eng[p_id]
        if e.host_batch is None:
            e.host_batch = _HostBatchC(e.cfg, self.dev)
        return e.host_batch.pack(batch, p_id, self.use_per)

    def draw_target_noise(self, B, p_id=None):
        """The draw the reference makes for the target actions of one policy in one update: (T+1, N_p*B, Ac), agent-major rows, CPU RNG."""
        e = self._eng[p_id or self.policy_ids[0]]
        pol = e.pol
        T, N, Ac = self.episode_length, e.n_agents, pol.act_dim
        if pol.discrete:
            return sample_gumbel((T + 1, N * B, Ac))                                               # util.py:137 via rMADDPGPolicy.py:105-106
        return torch.empty(T + 1, N * B, Ac).normal_(mean=0, std=float(pol.target_noise))          # util.py:217-218

    def draw_actor_noise(self, B, p_id=None):
        """Gumbel draws of the actor update's `get_actions(..., use_gumbel=True)` over obs[:-1] (r_maddpg.py:277): (T, N_p*B, Ac)."""
        e = self._eng[p_id or self.policy_ids[0]]
        return sample_gumbel((self.episode_length, e.n_agents * B, e.pol.act_dim))
