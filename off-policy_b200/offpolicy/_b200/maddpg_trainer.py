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
(`counts_updates`).

Data-parallel use (`torch.distributed` initialised, or `args.dp_world_size`, world size G > 1): one process per GPU, each rank samples
its own batch from its own replay shard (weak scaling: the global batch is G * B).  Per update every policy's learner sums two flat
buffers over the ranks, the critic's and then the actor's (the actor's backward reads the critic after its Adam step), so every rank
clips by the same global norm and applies bit-identical Adam and Polyak steps; the replicas never diverge.  The sums travel over NVLink
peer memory inside the step (csrc/p2p.cu), or, with MARL_B200_P2P=0 or without peer mappings, through `torch.distributed.all_reduce`
between the phases of the update (`update_phases`).  PER trees and the noise stay local: each rank draws the noise of its own rows from
its own generator (torch's CPU generator, or its own DeviceTorchGenerator), so a G-rank run does not reproduce a one-GPU run's noise
stream."""
import ctypes as C
import os
import sys

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
        off, n = C.c_int64(), C.c_int64()
        capi.check(lib.mx_maddpg_ws_lookup(h, b"p2p_abort", C.byref(off), C.byref(n)))
        self.abort = self.workspace[off.value:off.value + 4].view(torch.float32)      # sticky abort word of the data-parallel exchange
        self.host_batch = None

    def grad_buffer(self, net):
        """The flat buffer grad[P+4] one exchange of network `net` (capi.MADDPG_ACTOR / _CRITIC) sums over the ranks."""
        n = C.c_int64()
        off = capi.lib().mx_maddpg_grad_buffer(self.handle, net, C.byref(n)) - self.workspace.data_ptr()
        return self.workspace[off:off + 4 * n.value].view(torch.float32)

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
        dist = torch.distributed
        self.world_size = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        self.world_size = int(getattr(args, "dp_world_size", None) or self.world_size)     # (tests drive several "ranks" from one process)
        self._p2p = False
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
        if self.world_size > 1 and self.dev.type == "cuda" and os.environ.get("MARL_B200_P2P", "1") != "0" and \
                dist.is_available() and dist.is_initialized():
            try:
                self._setup_p2p()
            except Exception as ex:       # no peer access / symmetric memory on this box: the all-reduce path stays in use
                sys.stderr.write("marl_b200: peer-memory gradient exchange unavailable (%s); using torch.distributed.all_reduce\n" % (ex,))
            # every rank must use the same exchange: fall back everywhere if any rank could not map its peers
            agree = torch.tensor([1 if self._p2p else 0], dtype=torch.int32, device=self.dev)
            dist.all_reduce(agree, op=dist.ReduceOp.MIN)
            if int(agree) == 0:
                self._p2p = False

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

    # -- data-parallel gradient exchange over NVLink peer memory (csrc/p2p.cu) ------------------------------------------------
    def p2p_block_bytes(self, p_id, net):
        """Bytes of the symmetric block one rank allocates for network `net` of policy p_id's learner."""
        return int(capi.lib().mx_maddpg_p2p_block_bytes(self._eng[p_id].handle, net))

    def _setup_p2p(self):
        """One symmetric block per policy and network on every rank (torch.distributed._symmetric_memory: allocation + exchange of
        the peer mappings is plumbing), handed to the library; from then on `mx_maddpg_step_ex` contains both exchanges."""
        import torch.distributed._symmetric_memory as symm
        dist = torch.distributed
        ptrs, keep = {}, []
        for p in self.policy_ids:
            for net in (capi.MADDPG_ACTOR, capi.MADDPG_CRITIC):
                block = symm.empty(self.p2p_block_bytes(p, net) // 4, dtype=torch.float32, device=self.dev)
                block.zero_()
                hdl = symm.rendezvous(block, dist.group.WORLD.group_name)
                ptrs[(p, net)] = [int(x) for x in hdl.buffer_ptrs]
                keep.append((block, hdl))
        torch.cuda.synchronize(self.dev)
        dist.barrier()
        self.attach_peer_blocks(dist.get_rank(), ptrs, keep=keep)
        self._p2p = self._p2p_selftest([b for b, _ in keep])

    def _p2p_selftest(self, blocks):
        """One exchange of a known pattern on every block before the first real update: rank r publishes r + 1 in every element, the
        reduce must return G (G + 1) / 2 everywhere without a time-out.  Every rank always reaches both barriers (local failures are
        only recorded) and the caller combines the verdicts with an all-reduce, so a box on which peer loads misbehave falls back to
        the all-reduce exchange on ALL ranks instead of training on garbage."""
        dist = torch.distributed
        lib, stream = capi.lib(), capi.stream_ptr()
        rank, world = dist.get_rank(), dist.get_world_size()
        nets = [(p, net) for p in self.policy_ids for net in (capi.MADDPG_ACTOR, capi.MADDPG_CRITIC)]
        counts = {(p, net): self.ws_view("adam_ta" if net == capi.MADDPG_ACTOR else "adam_tc", p, torch.float64) for p, net in nets}
        saved = {k: v.clone() for k, v in counts.items()}
        ok = True
        try:
            for p, net in nets:
                self._eng[p].grad_buffer(net).fill_(float(rank + 1))
                self._eng[p].abort.zero_()
                counts[(p, net)][0] = 1.0                 # the kernels take the step number (slot parity, flag value) from here
                capi.check(lib.mx_maddpg_p2p_publish(self._eng[p].handle, net, stream))
            for p, net in nets:
                capi.check(lib.mx_maddpg_p2p_reduce(self._eng[p].handle, net, stream))
            torch.cuda.synchronize(self.dev)
            want = world * (world + 1) / 2.0
            ok = all(bool((self._eng[p].grad_buffer(net) == want).all().item()) for p, net in nets) and \
                all(float(e.abort[0]) == 0.0 for e in self._eng.values())
        except Exception as ex:
            sys.stderr.write("marl_b200: peer-memory self-test raised %s\n" % (ex,))
            ok = False
        for p, net in nets:
            counts[(p, net)].copy_(saved[(p, net)])
            self._eng[p].grad_buffer(net).zero_()
            self._eng[p].abort.zero_()
        self._reset_peer_flags(blocks)
        return ok

    def _reset_peer_flags(self, blocks):
        """Zero the symmetric blocks on every rank once nobody reads them any more: the flags start over, so the next exchange
        waits for the peers' next publish whatever step count the learners are at."""
        torch.cuda.synchronize(self.dev)
        torch.distributed.barrier()
        for b in blocks:
            b.zero_()
        torch.cuda.synchronize(self.dev)
        torch.distributed.barrier()

    def attach_peer_blocks(self, rank, block_ptrs, keep=None):
        """Hand every learner the world's blocks: block_ptrs[(p_id, net)] = the addresses of that network's block on ranks 0 .. G-1
        (net: capi.MADDPG_ACTOR / _CRITIC), one zeroed block per policy, network and rank.  `keep` holds the blocks alive."""
        lib = capi.lib()
        self._p2p_counters = []
        for p in self.policy_ids:
            for net in (capi.MADDPG_ACTOR, capi.MADDPG_CRITIC):
                ptrs = block_ptrs[(p, net)]
                if len(ptrs) != self.world_size:
                    raise ValueError("policy %s net %d: %d peer blocks for a world of %d ranks" % (p, net, len(ptrs), self.world_size))
                counter = torch.zeros(4, dtype=torch.int32, device=self.dev)
                arr = (C.c_void_p * len(ptrs))(*ptrs)
                capi.check(lib.mx_maddpg_set_peers(self._eng[p].handle, net, int(rank), len(ptrs), arr, capi.ptr(counter)))
                self._p2p_counters.append(counter)
        self._p2p_keep = keep
        self._p2p = True

    def _check_exchange(self):
        """Peer-memory exchange watchdog.  A rank that waits longer than the time-out for a peer sets its learner's abort word to -1
        on the device and applies NO update from then on (csrc/p2p.cu, csrc/optim.cu k_adam).  On the GPU the words are mirrored to
        pinned host memory after every update without a synchronisation and the copy of the PREVIOUS update is inspected here, so a
        dead peer turns into an exception one update later instead of silently diverging replicas."""
        if not self._p2p:
            return
        engines = [self._eng[p] for p in self.policy_ids]
        if self.dev.type != "cuda":
            if any(float(e.abort[0]) < 0.0 for e in engines):
                self._exchange_failed()
            return
        if getattr(self, "_xchg_host", None) is None:
            self._xchg_host = torch.zeros(len(engines), dtype=torch.float32).pin_memory()
            self._xchg_ev = torch.cuda.Event()
            self._xchg_pending = False
        if self._xchg_pending and self._xchg_ev.query():
            self._xchg_pending = False
            if float(self._xchg_host.min()) < 0.0:
                self._exchange_failed()
        if not self._xchg_pending:
            for i, e in enumerate(engines):
                self._xchg_host[i:i + 1].copy_(e.abort[0:1], non_blocking=True)
            self._xchg_ev.record(torch.cuda.current_stream(self.dev))
            self._xchg_pending = True

    def _exchange_failed(self):
        raise RuntimeError("marl_b200: a data-parallel peer did not deliver its gradient within the time-out; no update was applied "
                           "(replicas are still identical). Restart the job or set MARL_B200_P2P=0 for the all-reduce exchange.")

    def load_state_dict(self, sd):
        MaddpgLearnerState.load_state_dict(self, sd)
        if self._p2p and getattr(self, "_p2p_keep", None) and self.dev.type == "cuda" and torch.distributed.is_initialized():
            # the peers' "step reached" flags belong to the run that wrote them: start over (every rank restores the same step counts,
            # so the exchange resumes in lock-step)
            self._reset_peer_flags([b for b, _ in self._p2p_keep])

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

    def _stage_update(self, update_policy_id, batch):
        """The inputs of one update of policy update_policy_id on the device: its batch struct, its target noise and (on updates that
        train the actor) its actor noise; several policies: every policy's contribution to its centralised action vectors."""
        if update_policy_id not in self._eng:
            raise KeyError("unknown policy id %r" % (update_policy_id,))
        lib, stream = capi.lib(), capi.stream_ptr()
        e = self._eng[update_policy_id]
        b = self._device_batch(batch, update_policy_id)
        if self.multi:
            # get_update_info (r_maddpg.py:40-105, maddpg.py:38-81): every policy's buffer actions and TARGET-actor next actions,
            # policy by policy in id order -- the target-noise draws (MATD3) consume torch's CPU generator in that same order.  Row by
            # row: with data parallelism each rank contributes for its own rows only, so nothing is exchanged here
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
        return e, b, noise, actor_noise

    def _update_result(self, update_policy_id, e, b, updated, batch):
        info = e.info
        train_info = {"critic_loss": info[0], "critic_grad_norm": info[1]}
        if updated:
            train_info["actor_loss"], train_info["actor_grad_norm"] = info[4], info[5]
        train_info["update_actor"] = bool(updated)
        if self.counts_updates:
            self.num_updates[update_policy_id] += 1
        new_priorities = DeviceArray(e.prio[:b.B]) if self.use_per else None
        return train_info, new_priorities, batch[self._idx_field]

    def shared_train_policy_on_batch(self, update_policy_id, batch):
        if self.world_size > 1 and not self._p2p:
            result = self._allreduce_update(update_policy_id, batch)
        else:
            lib, stream = capi.lib(), capi.stream_ptr()
            e, b, noise, actor_noise = self._stage_update(update_policy_id, batch)
            upd = C.c_int32()
            capi.check(lib.mx_maddpg_step_ex(e.handle, C.byref(b), capi.ptr(noise), capi.ptr(actor_noise), C.byref(upd), stream))
            result = self._update_result(update_policy_id, e, b, upd.value, batch)
        self._check_exchange()
        return result

    def update_phases(self, update_policy_id, batch):
        """One update of policy update_policy_id as a generator split at its two exchanges (mx_maddpg_step_phase): it yields
        (engine, net) when network `net`'s buffer engine.grad_buffer(net) is ready to be summed over the ranks -- the critic's, then,
        on updates that train the actor, the actor's -- and returns shared_train_policy_on_batch's result.  The caller sums in
        between: `torch.distributed.all_reduce` (the fallback exchange), or, for several ranks driven from one process, every rank's
        mx_maddpg_p2p_publish before any rank's mx_maddpg_p2p_reduce."""
        lib, stream = capi.lib(), capi.stream_ptr()
        e, b, noise, actor_noise = self._stage_update(update_policy_id, batch)
        upd = C.c_int32()

        def phase(k):
            capi.check(lib.mx_maddpg_step_phase(e.handle, k, C.byref(b), capi.ptr(noise), capi.ptr(actor_noise), C.byref(upd), stream))
        phase(capi.MADDPG_CRITIC_GRADS)
        yield e, capi.MADDPG_CRITIC
        phase(capi.MADDPG_CRITIC_APPLY)
        if upd.value:
            phase(capi.MADDPG_ACTOR_GRADS)
            yield e, capi.MADDPG_ACTOR
            phase(capi.MADDPG_ACTOR_APPLY)
        return self._update_result(update_policy_id, e, b, upd.value, batch)

    def _allreduce_update(self, update_policy_id, batch):
        """The fallback exchange (MARL_B200_P2P=0 or no peer mappings): the phases of the update with an all-reduce of each buffer."""
        g = self.update_phases(update_policy_id, batch)
        try:
            while True:
                e, net = next(g)
                torch.distributed.all_reduce(e.grad_buffer(net))
        except StopIteration as stop:
            return stop.value

    def prep_training(self):
        pass

    def prep_rollout(self):
        pass
