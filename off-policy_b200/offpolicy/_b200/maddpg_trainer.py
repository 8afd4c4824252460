"""The trainer core of the actor-critic learners: R_MADDPG / R_MATD3 (recurrent, whole episodes) and MADDPG / MATD3 (MLP,
transitions) derive from `MaddpgTrainer`.

It owns one mx_maddpg learner per policy, the policy / agent / centralised-action wiring, the update step, checkpoints
(`MaddpgLearnerState`) and the update noise in both modes.  The noise of one policy's update lives in a [B][steps][N][A] layout;
a subclass states its geometry: `noise_steps` and, per draw ('target': the target actions', 'actor': the actor update's Gumbel
draws), the first step and the number of steps the draw covers (`noise_rows`).  Host mode places the draws of
`draw_target_noise` / `draw_actor_noise` (torch's CPU generator) there with `place_noise` / `_rows`; device mode
(`use_device_noise(gen)`) makes the same torch calls as fills straight into fixed device buffers (offpolicy/_b200/torch_rng.py).

A subclass supplies its configuration struct (`_cfg`), its batch staging (`_device_batch`), its host draws, the index of the
sample indices in the reference's batch tuple (`_idx_field`), its refusal messages and whether it counts its updates
(`counts_updates`)."""
import ctypes as C

import torch

from offpolicy._b200 import capi
from offpolicy._b200.maddpg_state import MaddpgLearnerState
from offpolicy._b200.torch_rng import draw
from offpolicy.utils.rec_buffer import DeviceArray


class _Engine(object):
    """One policy's learner: its mx_maddpg handle, the workspace views and the host-batch staging."""

    def __init__(self, cfg, pol, n_agents, max_batch):
        lib = capi.lib()
        self.cfg, self.pol, self.n_agents = cfg, pol, n_agents
        nbytes = int(lib.mx_maddpg_workspace_bytes(C.byref(cfg)))
        if nbytes < 0:
            raise capi.MxError(lib.mx_last_error().decode())
        self.workspace = torch.zeros(nbytes, dtype=torch.uint8, device=capi.device())
        av = (C.c_void_p * 4)(*[v.data_ptr() for v in pol.actor_vecs])
        cv = (C.c_void_p * 4)(*[v.data_ptr() for v in pol.critic_vecs])
        h = C.c_void_p()
        capi.check(lib.mx_maddpg_create(C.byref(cfg), av, cv, capi.ptr(self.workspace), nbytes, C.byref(h)))
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


class MaddpgTrainer(MaddpgLearnerState):
    counts_updates = True          # num_updates[p] += 1 per update, and the actor updates every actor_update_interval-th one
    noise_gen = None               # a DeviceTorchGenerator in device noise mode

    def __init__(self, args, num_agents, policies, policy_mapping_fn, device=None, actor_update_interval=1):
        self.args = args
        self.use_per = args.use_per
        if getattr(args, "use_popart", False):
            raise NotImplementedError(self._popart_msg)
        self.num_agents = num_agents
        self.policies = policies
        self.policy_mapping_fn = policy_mapping_fn
        self.policy_ids = sorted(list(self.policies.keys()))
        self.policy_agents = {p: sorted(a for a in range(num_agents) if policy_mapping_fn(a) == p) for p in self.policies}
        self.actor_update_interval = actor_update_interval
        self.num_updates = {p: 0 for p in self.policy_ids}
        self.use_same_share_obs = getattr(args, "use_same_share_obs", True)
        self.max_batch = int(getattr(args, "batch_size", 32))
        self.dev = capi.device()
        self._noise_bufs = {}
        self._in_flight = None
        # one shared policy ('policy_0' for every agent): the single-learner layout; several policies (config.py:61 share_policy False,
        # train/train_mpe.py:139-150): one learner per policy, and every critic sees the actions of all agents: cent_act_dim is the
        # total action width and each policy's agents sit at act_offset, in sorted policy-id order (r_maddpg.py:62-105,
        # maddpg.py:55-79)
        self.multi = len(self.policy_ids) > 1
        total = sum(len(self.policy_agents[p]) * self.policies[p].output_dim for p in self.policy_ids)
        self._eng = {}
        off = 0
        for p in self.policy_ids:
            pol, n_p = self.policies[p], len(self.policy_agents[p])
            if self.multi and pol.central_act_dim != total:
                raise ValueError("policy %s: cent_act_dim %d != total action width %d of all agents" % (p, pol.central_act_dim, total))
            cfg = self._cfg(pol, n_p, total if self.multi else 0, off if self.multi else 0)
            self._eng[p] = _Engine(cfg, pol, n_p, self.max_batch)
            pol._trainer, pol._handle = self, self._eng[p].handle
            off += n_p * pol.output_dim
        first = self._eng[self.policy_ids[0]]
        # the first policy's learner under the single-policy names (graph helpers, tests)
        self.pol, self.cfg, self.workspace, self.handle, self._info, self._prio = first.pol, first.cfg, first.workspace, first.handle, first.info, first.prio

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

    # -- update noise ----------------------------------------------------------------------------------------------------
    def use_device_noise(self, gen):
        """Draw every update's noise from `gen` (a DeviceTorchGenerator) on the device instead of from torch's CPU generator; None
        goes back to the host draws."""
        self.noise_gen = gen

    def _takes_noise(self, p_id, which):
        pol = self._eng[p_id].pol
        return pol.td3 if which == "target" else pol.discrete

    def place_noise(self, draw, dst, first):
        """Write a host draw (torch's layout: its steps of N*B agent-major rows, or one step as (N*B, A)) into dst [B][steps][N][A]
        from step `first` on; the other steps are left as they are."""
        B, _, N, A = dst.shape
        count = draw.numel() // (N * B * A)
        dst[:, first:first + count] = draw.reshape(count, N, B, A).permute(2, 0, 1, 3)

    def _rows(self, draw, B, first, p_id=None):
        """A host draw placed from step `first` on in fresh noise rows on the device (zero elsewhere), or None without a draw."""
        if draw is None:
            return None
        e = self._eng[p_id or self.policy_ids[0]]
        x = torch.zeros(B, self.noise_steps, e.n_agents, e.pol.output_dim)
        self.place_noise(draw, x, first)
        return x.to(self.dev, non_blocking=True)

    def _noise_buffer(self, p_id, which, B):
        """The fixed device buffer a policy's device draws and whole-update graphs read, zero outside the draws."""
        key = (p_id, which, B)
        if key not in self._noise_bufs:
            e = self._eng[p_id]
            self._noise_bufs[key] = torch.zeros(B, self.noise_steps, e.n_agents, e.pol.output_dim, dtype=torch.float32, device=self.dev)
        return self._noise_bufs[key]

    def _noise_draws(self, B, p_id, which, buf=None):
        """Device mode: the torch calls of draw_target_noise / draw_actor_noise as fills into `buf` (by default the policy's noise
        buffer), one per MultiDiscrete sub-space at its columns; [] when the update takes no such noise."""
        if not self._takes_noise(p_id, which):
            return []
        e = self._eng[p_id]
        pol, N, A = e.pol, e.n_agents, e.pol.output_dim
        buf = self._noise_buffer(p_id, which, B) if buf is None else buf
        first, count = self.noise_rows[which]
        col, ld = first * N * A, (N * A, A, self.noise_steps * N * A)
        if which == "target" and not pol.discrete:
            return [draw(capi.TRNG_NORMAL, count, N, B, A, buf, col, *ld, std=float(pol.target_noise or 0.0))]
        out = []
        for n in pol.act_segs or [A]:
            out.append(draw(capi.TRNG_GUMBEL, count, N, B, n, buf, col, *ld))
            col += n
        return out

    def _device_noise(self, B, p_id, which):
        """Device mode: one policy's draws filled into its noise buffer."""
        for d in self._noise_draws(B, p_id, which):
            self.noise_gen.fill(d)
        return self._noise_buffer(p_id, which, B)

    def _noise(self, B, p_id, which):
        """One policy's target ('target') or actor-update ('actor') noise rows on the device, or None when its update takes none."""
        if not self._takes_noise(p_id, which):
            return None
        if self.noise_gen is not None:
            return self._device_noise(B, p_id, which)
        draw_fn = self.draw_target_noise if which == "target" else self.draw_actor_noise
        return self._rows(draw_fn(B, p_id), B, self.noise_rows[which][0], p_id)

    def _target_noise(self, B, p_id=None):
        return self._noise(B, p_id or self.policy_ids[0], "target")

    def _actor_noise(self, B, p_id=None):
        return self._noise(B, p_id or self.policy_ids[0], "actor")

    # -- the update --------------------------------------------------------------------------------------------------------
    def train_policy_on_batch(self, update_policy_id, batch):
        if self.use_same_share_obs:
            return self.shared_train_policy_on_batch(update_policy_id, batch)
        return self.cent_train_policy_on_batch(update_policy_id, batch)

    def cent_train_policy_on_batch(self, update_policy_id, batch):
        raise NotImplementedError(self._cent_msg)

    def shared_train_policy_on_batch(self, update_policy_id, batch):
        if update_policy_id not in self._eng:
            raise KeyError("unknown policy id %r" % (update_policy_id,))
        lib, stream = capi.lib(), capi.stream_ptr()
        e = self._eng[update_policy_id]
        b = self._device_batch(batch, update_policy_id)
        if self.multi:
            # get_update_info (r_maddpg.py:40-105, maddpg.py:38-81): every policy's buffer actions and TARGET-actor next actions,
            # policy by policy in id order -- the target-noise draws (MATD3) consume torch's CPU generator in that same order
            noises = []
            for q in self.policy_ids:
                bq = b if q == update_policy_id else self._device_batch(batch, q)
                nq = self._target_noise(b.B, q)
                noises.append(nq)
                if q == update_policy_id:
                    noise = nq
                capi.check(lib.mx_maddpg_cent_contribute(self._eng[q].handle, C.byref(bq), capi.ptr(nq), e.handle, stream))
        else:
            noise = self._target_noise(b.B, update_policy_id)
            noises = [noise]
        update_actor = self.num_updates[update_policy_id] % self.actor_update_interval == 0
        actor_noise = self._actor_noise(b.B, update_policy_id) if update_actor else None
        self._in_flight = (noises, actor_noise)        # the device copies: alive until the launches that read them have run
        upd = C.c_int32()
        capi.check(lib.mx_maddpg_step_ex(e.handle, C.byref(b), capi.ptr(noise), capi.ptr(actor_noise), C.byref(upd), stream))
        info = e.info
        train_info = {"critic_loss": info[0], "critic_grad_norm": info[1]}
        if upd.value:
            train_info["actor_loss"], train_info["actor_grad_norm"] = info[4], info[5]
        train_info["update_actor"] = bool(upd.value)
        if self.counts_updates:
            self.num_updates[update_policy_id] += 1
        new_priorities = DeviceArray(e.prio[:b.B]) if self.use_per else None
        return train_info, new_priorities, batch[self._idx_field]

    def prep_training(self):
        pass

    def prep_rollout(self):
        pass
