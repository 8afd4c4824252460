"""Drop-in `MADDPG` trainer (reference: offpolicy/algorithms/maddpg/maddpg.py) of the transition-level MADDPG / MATD3 on the CUDA
learner in its `mlp` mode (csrc/maddpg.cu, maddpg_step_mlp).

`shared_train_policy_on_batch(p_id, batch)` is one `mx_maddpg_step_ex`: target-actor next actions, critic update through the frozen
Q heads, then the actor update through head 0 of the updated critic, masked by `valid_transition` -- all on the device.  The random
draws are made on the host with the reference's own calls, in its order: the target actions' noise (MATD3: Gumbel for Discrete,
N(0, target_action_noise_std) for Box actions), then the actor update's Gumbel draws (Discrete actors).

The reference never increments `num_updates` here (maddpg.py:33, 100; compare r_maddpg.py:330), so `update_actor` is always True and
MATD3 updates its actor on every call despite `actor_update_interval = 2` (SURVEY.md App. D-14).  The learner is therefore
configured with an actor update interval of 1.  Only the shared-policy, shared-observation form is built:
`cent_train_policy_on_batch`, several policies and `--use_popart` raise."""
import ctypes as C

import numpy as np
import torch

from offpolicy._b200 import capi
from offpolicy.algorithms.r_maddpg.algorithm.rMADDPGPolicy import maddpg_cfg_struct, sample_gumbel
from offpolicy.utils.mlp_buffer import MlpSampledBatch
from offpolicy.utils.rec_buffer import DeviceArray


class _HostTransitions(object):
    """Device copy of a batch handed over in the reference's NumPy layout (mlp_buffer.py:203-240): compatibility path."""

    def __init__(self, cfg, dev):
        B, N = cfg.max_batch, cfg.n_agents
        r4 = lambda v: (v + 3) // 4 * 4
        self.cfg, self.dev = cfg, dev
        self.obs_ld, self.share_ld, self.act_ld = r4(cfg.obs_dim), r4(cfg.state_dim), r4(cfg.act_dim)
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


class MADDPG(object):
    def __init__(self, args, num_agents, policies, policy_mapping_fn, device=None, actor_update_interval=1):
        self.args = args
        self.use_per = args.use_per
        if getattr(args, "use_popart", False):
            raise NotImplementedError("B200 MADDPG path: --use_popart is not implemented")
        if list(policies.keys()) != ["policy_0"]:
            raise NotImplementedError("B200 MADDPG path: only one shared policy is implemented (the transition replay is shared-policy only)")
        self.num_agents = num_agents
        self.policies = policies
        self.policy_mapping_fn = policy_mapping_fn
        self.policy_ids = sorted(list(self.policies.keys()))
        self.policy_agents = {p: sorted(a for a in range(num_agents) if policy_mapping_fn(a) == p) for p in self.policies}
        self.num_updates = {p: 0 for p in self.policy_ids}           # never incremented, like the reference
        self.use_same_share_obs = getattr(args, "use_same_share_obs", True)
        self.actor_update_interval = actor_update_interval
        self.max_batch = int(getattr(args, "batch_size", 32))
        self.dev = capi.device()
        pol = self.policies["policy_0"]
        self.pol = pol
        N = len(self.policy_agents["policy_0"])
        if pol.central_act_dim != N * pol.act_dim:
            raise NotImplementedError("B200 MADDPG path: cent_act_dim %d != n_agents * act_dim %d" % (pol.central_act_dim, N * pol.act_dim))
        lib = capi.lib()
        # cfg.target_noise > 0 tells the learner that target-action noise is passed.  MATD3 always smooths (MADDPGPolicy.py:93, 111 test
        # `target_noise is not None`): a Discrete actor takes Gumbel draws whatever the std, a Box actor N(0, std) draws, all-zero at std 0
        tnoise = (1.0 if pol.discrete else float(pol.target_noise)) if pol.td3 else 0.0
        self.cfg = maddpg_cfg_struct(args, N, pol.obs_dim, pol.act_dim, pol.central_obs_dim, 1, self.max_batch, pol.td3, tnoise, 1,
                                     pol.discrete, mlp=True)
        nbytes = int(lib.mx_maddpg_workspace_bytes(C.byref(self.cfg)))
        if nbytes < 0:
            raise capi.MxError(lib.mx_last_error().decode())
        self.workspace = torch.zeros(nbytes, dtype=torch.uint8, device=self.dev)
        av = (C.c_void_p * 4)(*[v.data_ptr() for v in pol.actor_vecs])
        cv = (C.c_void_p * 4)(*[v.data_ptr() for v in pol.critic_vecs])
        h = C.c_void_p()
        capi.check(lib.mx_maddpg_create(C.byref(self.cfg), av, cv, capi.ptr(self.workspace), nbytes, C.byref(h)))
        self.handle = h
        pol._trainer, pol._handle = self, h
        ip = lib.mx_maddpg_info(h) - self.workspace.data_ptr()
        self._info = self.workspace[ip:ip + 32].view(torch.float32)
        pp = lib.mx_maddpg_priorities(h) - self.workspace.data_ptr()
        self._prio = self.workspace[pp:pp + 4 * self.max_batch].view(torch.float32)
        self._host_batch = None
        self._noise_dev = self._actor_noise_dev = None

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                capi.lib().mx_maddpg_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    def grad_views(self):
        """Numerator gradients (actor, critic) as flat views, for the parity tests."""
        a, c = C.c_int64(), C.c_int64()
        capi.lib().mx_maddpg_grad_views(self.handle, C.byref(a), C.byref(c))
        return (self.workspace[a.value:a.value + 4 * (self.pol.Pa + 4)].view(torch.float32),
                self.workspace[c.value:c.value + 4 * (self.pol.Pc + 4)].view(torch.float32))

    def draw_target_noise(self, B):
        """The draw get_update_info makes through the target policy (maddpg.py:71): (N*B, A) agent-major rows, or None."""
        pol, N = self.pol, self.cfg.n_agents
        if not pol.td3:
            return None
        if pol.discrete:
            return sample_gumbel((N * B, pol.act_dim))                                             # util.py:178-181
        return torch.empty(N * B, pol.act_dim).normal_(mean=0, std=float(pol.target_noise))       # util.py:217-218

    def draw_actor_noise(self, B):
        """Gumbel draws of the actor update's get_actions(..., use_gumbel=True) (maddpg.py:209): (N*B, A), or None for Box actors."""
        return sample_gumbel((self.cfg.n_agents * B, self.pol.act_dim)) if self.pol.discrete else None

    def _rows(self, draw, B, step):
        """(N*B, A) agent-major draw -> [b][step][n][A] of the learner's transition rows (the other step zero)."""
        if draw is None:
            return None
        N, A = self.cfg.n_agents, self.pol.act_dim
        ours = torch.zeros(B, 2, N, A)
        ours[:, step] = draw.view(N, B, A).permute(1, 0, 2)
        return ours.to(self.dev, non_blocking=True)

    def _device_batch(self, batch):
        lib = capi.lib()
        if isinstance(batch, MlpSampledBatch):
            buf = batch.buffers["policy_0"]
            if buf.rep.sample_serial != batch.serial["policy_0"]:
                raise RuntimeError("stale sample: the buffer has been sampled again since this batch was drawn")
            capi.check(lib.mx_maddpg_set_valid(self.handle, capi.ptr(buf.valid_dev)))
            return buf.rep.batch_struct(batch.B)
        if self._host_batch is None:
            self._host_batch = _HostTransitions(self.cfg, self.dev)
        b = self._host_batch.pack(batch, "policy_0", self.use_per)
        capi.check(lib.mx_maddpg_set_valid(self.handle, capi.ptr(self._host_batch.valid)))
        return b

    def train_policy_on_batch(self, update_policy_id, batch):
        if self.use_same_share_obs:
            return self.shared_train_policy_on_batch(update_policy_id, batch)
        return self.cent_train_policy_on_batch(update_policy_id, batch)

    def cent_train_policy_on_batch(self, update_policy_id, batch):
        raise NotImplementedError("B200 MADDPG path: cent_train_policy_on_batch (use_same_share_obs=False) is not implemented")

    def shared_train_policy_on_batch(self, update_policy_id, batch):
        """maddpg.py:90-249."""
        if update_policy_id != "policy_0":
            raise NotImplementedError("B200 MADDPG path: one shared policy 'policy_0'")
        lib = capi.lib()
        b = self._device_batch(batch)
        self._noise_dev = self._rows(self.draw_target_noise(b.B), b.B, 1)
        self._actor_noise_dev = self._rows(self.draw_actor_noise(b.B), b.B, 0)
        upd = C.c_int32()
        capi.check(lib.mx_maddpg_step_ex(self.handle, C.byref(b), capi.ptr(self._noise_dev), capi.ptr(self._actor_noise_dev), C.byref(upd),
                                         capi.stream_ptr()))
        info = self._info
        train_info = {"critic_loss": info[0], "critic_grad_norm": info[1], "actor_loss": info[4], "actor_grad_norm": info[5],
                      "update_actor": True}
        new_priorities = DeviceArray(self._prio[:b.B]) if self.use_per else None
        return train_info, new_priorities, batch[12]

    def prep_training(self):
        pass

    def prep_rollout(self):
        pass
