"""Drop-in `MADDPG` trainer (reference: offpolicy/algorithms/maddpg/maddpg.py) of the transition-level MADDPG / MATD3 on the CUDA
learner in its `mlp` mode (csrc/maddpg.cu, maddpg_step_mlp).

`shared_train_policy_on_batch(p_id, batch)` is one `mx_maddpg_step_ex`: target-actor next actions, critic update through the frozen
Q heads, then the actor update through head 0 of the updated critic, masked by `valid_transition` -- all on the device.  The random
draws are made on the host with the reference's own calls, in its order: the target actions' noise (MATD3: Gumbel for Discrete,
N(0, target_action_noise_std) for Box actions), then the actor update's Gumbel draws (Discrete actors).

The reference never increments `num_updates` here (maddpg.py:33, 100; compare r_maddpg.py:330), so `update_actor` is always True and
MATD3 updates its actor on every call despite `actor_update_interval = 2` (SURVEY.md App. D-14).  The learner is therefore
configured with an actor update interval of 1.

Several policies (`--share_policy` off, train_mpe.py:139-150: one policy per agent, possibly with different observation and action
spaces) get one learner each.  Every critic sees the actions of all agents: `cent_act_dim` is the total action width and each policy's
agents sit at `act_offset`, in sorted policy-id order (maddpg.py:55-79).  Before a policy's step, every policy q writes its buffer
actions and its target actor's next actions into the updated policy's centralised action vectors (`mx_maddpg_cent_contribute`), q by q
in id order, which is also the order of the reference's target-noise draws.  Only the shared-observation form is built:
`cent_train_policy_on_batch` and `--use_popart` raise.

MultiDiscrete policies (`act_dim` an ndarray of sub-space widths) occupy `output_dim` columns of every action vector; the learner gets
the sub-space widths (cfg.act_seg) and transforms each one-hot block on its own.  Their Gumbel draws are one `sample_gumbel` call per
sub-space, in sub-space order, as the reference's per-block `gumbel_softmax` calls make them (MADDPGPolicy.py:73-89).

`use_device_noise(gen)` makes the same torch calls on the device, one fill each, straight into the learner's noise rows
(offpolicy/_b200/torch_rng.py)."""
import numpy as np
import torch

from offpolicy._b200 import capi
from offpolicy._b200.maddpg_trainer import MaddpgTrainer
from offpolicy.algorithms.r_maddpg.algorithm.rMADDPGPolicy import maddpg_cfg_struct, sample_gumbel
from offpolicy.utils.mlp_buffer import MlpSampledBatch


def _gumbel_blocks(rows, pol):
    """Gumbel(0, 1) draws for `rows` actor rows of a Discrete policy: one sample_gumbel call per MultiDiscrete sub-space, in order (the
    reference's per-block gumbel_softmax calls), or one call over the whole action."""
    if pol.act_segs is None:
        return sample_gumbel((rows, pol.act_dim))
    return torch.cat([sample_gumbel((rows, n)) for n in pol.act_segs], -1)


class _HostTransitions(object):
    """Device copy of a batch handed over in the reference's NumPy layout (mlp_buffer.py:203-240): compatibility path."""

    def __init__(self, cfg, dev):
        B, N = cfg.max_batch, cfg.n_agents
        r4 = lambda v: (v + 3) // 4 * 4
        self.cfg, self.dev = cfg, dev
        self.obs_ld, self.share_ld, self.act_ld = r4(cfg.obs_dim), r4(cfg.state_dim), r4(cfg.act_dim)      # cfg.act_dim = output_dim
        z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)
        self.obs, self.share, self.acts, self.avail = z(B, 2, N, self.obs_ld), z(B, 2, self.share_ld), z(B, 1, N, self.act_ld), z(B, 2, N, self.act_ld)
        self.rew, self.dones, self.dones_env, self.weights, self.valid = z(B, 1, N), z(B, 1, N), z(B, 1), z(B), z(B, N)

    def pack(self, batch, p_id, use_per):
        obs, share, acts, rew, nobs, nshare, dones, dones_env, valid, avail, navail = batch[:11]
        weights = batch[11] if len(batch) > 11 else None
        c = self.cfg
        t = lambda x: torch.as_tensor(np.asarray(x), dtype=torch.float32).to(self.dev)
        o = t(obs[p_id])                                          # (N, B, O)
        B = o.shape[1]
        self.obs[:B, 0, :, :c.obs_dim] = o.permute(1, 0, 2)
        self.obs[:B, 1, :, :c.obs_dim] = t(nobs[p_id]).permute(1, 0, 2)
        self.share[:B, 0, :c.state_dim] = t(share[p_id])
        self.share[:B, 1, :c.state_dim] = t(nshare[p_id])
        self.acts[:B, 0, :, :c.act_dim] = t(acts[p_id]).permute(1, 0, 2)
        self.avail[:B] = 1.0
        have_avail = False
        for step, av in ((0, avail), (1, navail)):
            if av is not None and av[p_id] is not None:
                self.avail[:B, step, :, :c.act_dim] = t(av[p_id]).permute(1, 0, 2)
                have_avail = True
        self.rew[:B, 0] = t(rew[p_id])[..., 0].permute(1, 0)
        self.dones[:B, 0] = t(dones[p_id])[..., 0].permute(1, 0)
        self.dones_env[:B, 0] = t(dones_env[p_id]).reshape(B)
        self.valid[:B] = t(valid[p_id])[..., 0].permute(1, 0)
        if use_per:
            self.weights[:B] = t(weights)
        b = capi.Batch()
        b.B, b.obs_ld, b.share_ld, b.act_ld = B, self.obs_ld, self.share_ld, self.act_ld
        b.obs, b.share, b.acts = self.obs.data_ptr(), self.share.data_ptr(), self.acts.data_ptr()
        b.avail = self.avail.data_ptr() if have_avail else None
        b.rewards, b.dones, b.dones_env = self.rew.data_ptr(), self.dones.data_ptr(), self.dones_env.data_ptr()
        b.weights = self.weights.data_ptr() if use_per else None
        b.idx = None
        return b


class MADDPG(MaddpgTrainer):
    counts_updates = False            # like the reference (maddpg.py:33, 100)
    _popart_msg = "B200 MADDPG path: --use_popart is not implemented"
    _cent_msg = "B200 MADDPG path: cent_train_policy_on_batch (use_same_share_obs=False) is not implemented"
    _idx_field = 12
    # noise rows [B][2][N][A] (the transition's two steps): the target actions' draws at the next step, the actor update's at the first
    noise_steps, noise_rows = 2, {"target": (1, 1), "actor": (0, 1)}

    def _cfg(self, pol, n_agents, cent_act_dim, act_offset):
        if not self.multi and pol.central_act_dim != n_agents * pol.output_dim:
            raise NotImplementedError("B200 MADDPG path: cent_act_dim %d != n_agents * output_dim %d" % (pol.central_act_dim, n_agents * pol.output_dim))
        # cfg.target_noise > 0 tells the learner that target-action noise is passed.  MATD3 always smooths (MADDPGPolicy.py:93, 111 test
        # `target_noise is not None`): a Discrete actor takes Gumbel draws whatever the std, a Box actor N(0, std) draws, all-zero at std 0
        tnoise = (1.0 if pol.discrete else float(pol.target_noise)) if pol.td3 else 0.0
        return maddpg_cfg_struct(self.args, n_agents, pol.obs_dim, pol.output_dim, pol.central_obs_dim, 1, self.max_batch, pol.td3, tnoise, 1,
                                 pol.discrete, cent_act_dim=cent_act_dim, act_offset=act_offset, mlp=True, act_segs=pol.act_segs)

    def draw_target_noise(self, B, p_id=None):
        """The draw get_update_info makes through policy p_id's target policy (maddpg.py:71): (N_p*B, A_p) agent-major rows, or None."""
        e = self._eng[p_id or self.policy_ids[0]]
        pol = e.pol
        if not pol.td3:
            return None
        if pol.discrete:
            return _gumbel_blocks(e.n_agents * B, pol)                                              # util.py:178-181
        return torch.empty(e.n_agents * B, pol.act_dim).normal_(mean=0, std=float(pol.target_noise))       # util.py:217-218

    def draw_actor_noise(self, B, p_id=None):
        """Gumbel draws of policy p_id's actor update, get_actions(..., use_gumbel=True) (maddpg.py:209): (N_p*B, A_p), or None for Box
        actors."""
        e = self._eng[p_id or self.policy_ids[0]]
        return _gumbel_blocks(e.n_agents * B, e.pol) if e.pol.discrete else None

    def _device_batch(self, batch, p_id):
        lib = capi.lib()
        e = self._eng[p_id]
        if isinstance(batch, MlpSampledBatch):
            buf = batch.buffers[p_id]
            if buf.rep.sample_serial != batch.serial[p_id]:
                raise RuntimeError("stale sample: the buffer has been sampled again since this batch was drawn")
            capi.check(lib.mx_maddpg_set_valid(e.handle, capi.ptr(buf.valid_dev)))
            return buf.rep.batch_struct(batch.B)
        if e.host_batch is None:
            e.host_batch = _HostTransitions(e.cfg, self.dev)
        b = e.host_batch.pack(batch, p_id, self.use_per)
        capi.check(lib.mx_maddpg_set_valid(e.handle, capi.ptr(e.host_batch.valid)))
        return b
