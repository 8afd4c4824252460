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
import ctypes as C

import numpy as np
import torch

from offpolicy._b200 import capi
from offpolicy._b200.maddpg_state import MaddpgLearnerState
from offpolicy._b200.torch_rng import DeviceNoise, draw
from offpolicy.algorithms.r_maddpg.algorithm.rMADDPGPolicy import maddpg_cfg_struct, sample_gumbel
from offpolicy.utils.mlp_buffer import MlpSampledBatch
from offpolicy.utils.rec_buffer import DeviceArray


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


class _Engine(object):
    """One policy's learner: its mx_maddpg handle (cfg.mlp), the workspace views and the host-batch staging."""

    def __init__(self, args, pol, n_agents, max_batch, cent_act_dim, act_offset):
        lib = capi.lib()
        self.pol, self.n_agents = pol, n_agents
        # cfg.target_noise > 0 tells the learner that target-action noise is passed.  MATD3 always smooths (MADDPGPolicy.py:93, 111 test
        # `target_noise is not None`): a Discrete actor takes Gumbel draws whatever the std, a Box actor N(0, std) draws, all-zero at std 0
        tnoise = (1.0 if pol.discrete else float(pol.target_noise)) if pol.td3 else 0.0
        self.cfg = maddpg_cfg_struct(args, n_agents, pol.obs_dim, pol.output_dim, pol.central_obs_dim, 1, max_batch, pol.td3, tnoise, 1,
                                     pol.discrete, cent_act_dim=cent_act_dim, act_offset=act_offset, mlp=True, act_segs=pol.act_segs)
        nbytes = int(lib.mx_maddpg_workspace_bytes(C.byref(self.cfg)))
        if nbytes < 0:
            raise capi.MxError(lib.mx_last_error().decode())
        self.workspace = torch.zeros(nbytes, dtype=torch.uint8, device=capi.device())
        av = (C.c_void_p * 4)(*[v.data_ptr() for v in pol.actor_vecs])
        cv = (C.c_void_p * 4)(*[v.data_ptr() for v in pol.critic_vecs])
        h = C.c_void_p()
        capi.check(lib.mx_maddpg_create(C.byref(self.cfg), av, cv, capi.ptr(self.workspace), nbytes, C.byref(h)))
        self.handle = h
        ip = lib.mx_maddpg_info(h) - self.workspace.data_ptr()
        self.info = self.workspace[ip:ip + 32].view(torch.float32)
        pp = lib.mx_maddpg_priorities(h) - self.workspace.data_ptr()
        self.prio = self.workspace[pp:pp + 4 * max_batch].view(torch.float32)
        self.host_batch = None

    def close(self):
        if self.handle:
            capi.lib().mx_maddpg_destroy(self.handle)
            self.handle = None


class MADDPG(MaddpgLearnerState, DeviceNoise):
    def __init__(self, args, num_agents, policies, policy_mapping_fn, device=None, actor_update_interval=1):
        self.args = args
        self.use_per = args.use_per
        if getattr(args, "use_popart", False):
            raise NotImplementedError("B200 MADDPG path: --use_popart is not implemented")
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
        self.multi = len(self.policy_ids) > 1
        total = sum(len(self.policy_agents[p]) * self.policies[p].output_dim for p in self.policy_ids)
        self._eng = {}
        off = 0
        for p in self.policy_ids:                    # the centralised action vector: sorted ids, each policy's agents in order
            pol, n_p = self.policies[p], len(self.policy_agents[p])
            if self.multi and pol.central_act_dim != total:
                raise ValueError("policy %s: cent_act_dim %d != total action width %d of all agents" % (p, pol.central_act_dim, total))
            if not self.multi and pol.central_act_dim != n_p * pol.output_dim:
                raise NotImplementedError("B200 MADDPG path: cent_act_dim %d != n_agents * output_dim %d" % (pol.central_act_dim, n_p * pol.output_dim))
            self._eng[p] = _Engine(args, pol, n_p, self.max_batch, total if self.multi else 0, off if self.multi else 0)
            pol._trainer, pol._handle = self, self._eng[p].handle
            off += n_p * pol.output_dim
        first = self._eng[self.policy_ids[0]]
        # the first policy's learner under the single-policy names (graph helpers, tests)
        self.pol, self.cfg, self.workspace, self.handle, self._info, self._prio = first.pol, first.cfg, first.workspace, first.handle, first.info, first.prio
        self._noise_dev = self._actor_noise_dev = None
        self._keep = None

    def __del__(self):
        try:
            for e in getattr(self, "_eng", {}).values():
                e.close()
            self.handle = None
        except Exception:
            pass

    def grad_views(self, p_id=None):
        """Numerator gradients (actor, critic) of one policy's learner as flat views, for the parity tests."""
        e = self._eng[p_id or self.policy_ids[0]]
        a, c = C.c_int64(), C.c_int64()
        capi.lib().mx_maddpg_grad_views(e.handle, C.byref(a), C.byref(c))
        return (e.workspace[a.value:a.value + 4 * (e.pol.Pa + 4)].view(torch.float32),
                e.workspace[c.value:c.value + 4 * (e.pol.Pc + 4)].view(torch.float32))

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

    def _rows(self, draw, B, step, p_id=None):
        """(N*B, A) agent-major draw -> [b][step][n][A] of the learner's transition rows (the other step zero)."""
        if draw is None:
            return None
        e = self._eng[p_id or self.policy_ids[0]]
        N, A = e.n_agents, e.pol.output_dim
        ours = torch.zeros(B, 2, N, A)
        ours[:, step] = draw.view(N, B, A).permute(1, 0, 2)
        return ours.to(self.dev, non_blocking=True)

    _noise_steps = 2

    def _noise_cols(self, p_id):
        return self._eng[p_id].pol.output_dim

    def _noise_draws(self, B, p_id, which, buf):
        """Device mode: the torch calls of draw_target_noise (step 1) / draw_actor_noise (step 0) as fills into [b][step][n][A], one
        per MultiDiscrete sub-space at its columns."""
        e = self._eng[p_id]
        pol, N, A = e.pol, e.n_agents, e.pol.output_dim
        col = (1 if which == "target" else 0) * N * A
        ld = (0, A, 2 * N * A)
        if which == "target" and not pol.discrete:
            return [draw(capi.TRNG_NORMAL, 1, N, B, A, buf, col, *ld, std=float(pol.target_noise))]
        out = []
        for n in (pol.act_segs if pol.act_segs is not None else [pol.act_dim]):
            out.append(draw(capi.TRNG_GUMBEL, 1, N, B, int(n), buf, col, *ld))
            col += int(n)
        return out

    def _noise(self, B, p_id, which):
        """One policy's target ('target') or actor-update ('actor') noise rows on the device, or None when its update takes none."""
        pol = self._eng[p_id].pol
        if self.noise_gen is not None:
            return self._device_noise(B, p_id, which) if (pol.td3 if which == "target" else pol.discrete) else None
        if which == "target":
            return self._rows(self.draw_target_noise(B, p_id), B, 1, p_id)
        return self._rows(self.draw_actor_noise(B, p_id), B, 0, p_id)

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

    def train_policy_on_batch(self, update_policy_id, batch):
        if self.use_same_share_obs:
            return self.shared_train_policy_on_batch(update_policy_id, batch)
        return self.cent_train_policy_on_batch(update_policy_id, batch)

    def cent_train_policy_on_batch(self, update_policy_id, batch):
        raise NotImplementedError("B200 MADDPG path: cent_train_policy_on_batch (use_same_share_obs=False) is not implemented")

    def shared_train_policy_on_batch(self, update_policy_id, batch):
        """maddpg.py:90-249."""
        if update_policy_id not in self._eng:
            raise KeyError("unknown policy id %r" % (update_policy_id,))
        lib, stream = capi.lib(), capi.stream_ptr()
        e = self._eng[update_policy_id]
        b = self._device_batch(batch, update_policy_id)
        if self.multi:
            # maddpg.py:38-81 (get_update_info): every policy's buffer actions and TARGET-actor next actions, policy by policy in id
            # order -- the target-noise draws (MATD3) consume torch's CPU generator in that same order
            keep = []
            for q in self.policy_ids:
                bq = b if q == update_policy_id else self._device_batch(batch, q)
                nq = self._noise(b.B, q, "target")
                keep.append((bq, nq))
                if q == update_policy_id:
                    self._noise_dev = nq
                capi.check(lib.mx_maddpg_cent_contribute(self._eng[q].handle, C.byref(bq), capi.ptr(nq), e.handle, stream))
            self._keep = keep
        else:
            self._noise_dev = self._noise(b.B, update_policy_id, "target")
        self._actor_noise_dev = self._noise(b.B, update_policy_id, "actor")
        upd = C.c_int32()
        capi.check(lib.mx_maddpg_step_ex(e.handle, C.byref(b), capi.ptr(self._noise_dev), capi.ptr(self._actor_noise_dev), C.byref(upd),
                                         stream))
        info = e.info
        train_info = {"critic_loss": info[0], "critic_grad_norm": info[1], "actor_loss": info[4], "actor_grad_norm": info[5],
                      "update_actor": True}
        new_priorities = DeviceArray(e.prio[:b.B]) if self.use_per else None
        return train_info, new_priorities, batch[12]

    def prep_training(self):
        pass

    def prep_rollout(self):
        pass
