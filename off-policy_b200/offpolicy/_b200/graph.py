"""Whole-step CUDA graph: [sample ->] QMIX step [-> PER write-back] [-> soft update] captured once, replayed per step.

`mx_graph_capture` records the library's own launch sequence on a dedicated (non-default) stream; after that a learner
step costs one `cudaGraphLaunch` and no host work at all (indices come from the device-resident MT19937 stream).
"""
import contextlib
import ctypes as C

import torch

from offpolicy._b200 import capi

SAMPLE_UNIFORM, SAMPLE_PER, SOFT_UPDATE, PER_WRITEBACK = 1, 2, 4, 8


def _grow_scratch(gen, draws):
    """The generator's scratch, which the captured fills share, grown to hold the largest of `draws`."""
    if draws:
        words = max(gen.words(d) for d in draws)
        if gen._scratch.numel() < words:
            gen._scratch = torch.zeros(words, dtype=torch.int32, device=capi.device())


class _Graph(object):
    """What the graph helpers share: the capture flags, the dedicated (non-default) stream the graphs run on and the annealed PER
    exponent."""

    def _open(self, rep, trainer, beta, soft_update):
        self.lib = capi.lib()
        self._rep, self._per, self._beta = rep, bool(getattr(trainer, "use_per", False)), float(beta)
        self.flags = (SAMPLE_PER | PER_WRITEBACK if self._per else SAMPLE_UNIFORM) | (SOFT_UPDATE if soft_update else 0)
        dev = capi.device()
        self.cuda = dev.type == "cuda"            # (the CPU-emulated unit-test build re-runs the sequence instead of a graph)
        self.stream = torch.cuda.Stream(device=dev) if self.cuda else None
        if self.cuda:
            self.stream.wait_stream(torch.cuda.current_stream(dev))
        self._sp = C.c_void_p(self.stream.cuda_stream if self.cuda else 0)

    def _set_beta(self, beta):
        """`beta`: PER importance-sampling exponent of this step (the runner anneals it every step, base_runner.py:159-160); it lives
        in a device scalar the captured draw reads, so changing it costs one tiny launch and no re-capture."""
        if beta is not None and self._per and float(beta) != self._beta:
            capi.check(self.lib.mx_replay_set_beta(self._rep.handle, float(beta), self._sp))
            self._beta = float(beta)

    def synchronize(self):
        if self.cuda:
            self.stream.synchronize()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class StepGraph(_Graph):
    """`buffer`: RecReplayBuffer / PrioritizedRecReplayBuffer with a recurrent trainer, or MlpReplayBuffer / PrioritizedMlpReplayBuffer with
    M_QMix / M_VDN (transitions are length-1 episodes of the same HBM replay, so the captured sequence is the same)."""

    def __init__(self, buffer, trainer, batch_size, beta=0.4, soft_update=True, p_id="policy_0"):
        pb = buffer.policy_buffers[p_id]
        self._open(getattr(pb, "rep", pb), trainer, beta, soft_update)          # MlpPolicyBuffer wraps the episode replay
        g = C.c_void_p()
        capi.check(self.lib.mx_graph_capture(self._rep.handle, trainer.handle, int(batch_size), float(beta), self.flags, self._sp,
                                             C.byref(g)))
        self.handle = g
        self.num_kernels = int(self.lib.mx_graph_num_kernels(g))
        self._keep = (buffer, trainer)

    def launch(self, beta=None):
        self._set_beta(beta)
        capi.check(self.lib.mx_graph_launch(self.handle, self._sp))

    def close(self):
        if self.handle:
            self.lib.mx_graph_destroy(self.handle)
            self.handle = None


def _refuse_data_parallel(who, trainer):
    """A data-parallel update is not captured: its exchanges must order every rank's publish before any rank's reduce, which two
    graphs on one device cannot promise; the eager update (shared_train_policy_on_batch) runs the exchanges."""
    if getattr(trainer, "world_size", 1) > 1:
        raise ValueError("%s: the trainer trains data-parallel over %d ranks; a data-parallel update is not captured as a CUDA graph, "
                         "call shared_train_policy_on_batch instead" % (who, trainer.world_size))


class MaddpgStepGraph(_Graph):
    """[sample ->] shared_train_policy_on_batch [-> PER write-back] [-> soft update] of one policy of an R_MADDPG / R_MATD3 or
    single-policy MADDPG / MATD3 trainer, as CUDA graphs: one per update_actor variant the trainer can ask for.

    Host noise mode (the default): per `launch()` the host draws the noise the reference would draw (torch's CPU generator, the
    trainer's draw_target_noise / draw_actor_noise, in its order) into a pinned staging slot, enqueues the copies on the graph's
    stream and replays the graph.  Device noise mode (`trainer.use_device_noise(gen)`): the noise fills are captured at the head of
    each graph, so `launch()` is one graph launch with no host draw and no copy, and torch's host generator is not touched.

    The learner of an MLP trainer is pointed at the replay's `valid_transition` store before the capture: the captured step masks
    its actor loss with the store the graph samples from."""

    RING = 4

    def __init__(self, buffer, trainer, batch_size, beta=0.4, soft_update=True, p_id="policy_0"):
        _refuse_data_parallel("MaddpgStepGraph", trainer)
        self.graphs = {}
        pb = buffer.policy_buffers[p_id]
        e = trainer._eng[p_id]
        self.trainer, self.B, self.p_id, self.pol = trainer, int(batch_size), p_id, e.pol
        if e.cfg.mlp:
            capi.check(capi.lib().mx_maddpg_set_valid(e.handle, capi.ptr(pb.valid_dev)))
        self.tnoise_dev = trainer._noise_buffer(p_id, "target", self.B) if e.pol.td3 else None
        self.anoise_dev = trainer._noise_buffer(p_id, "actor", self.B) if e.pol.discrete else None
        self._open(getattr(pb, "rep", pb), trainer, beta, soft_update)          # (after the buffers' zero fill)
        self._gen = gen = trainer.noise_gen
        if gen is None:
            # pinned staging ring: a slot is rewritten only after the H2D copy that last read it has completed (its event)
            ring = lambda d: None if d is None else [torch.zeros(d.shape).pin_memory() if self.cuda else torch.zeros(d.shape)
                                                     for _ in range(self.RING)]
            self.tnoise_host, self.anoise_host = ring(self.tnoise_dev), ring(self.anoise_dev)
            self._copied, self._slot = [None] * self.RING, 0
        self._draws = {}
        for upd in ((1, 0) if trainer.counts_updates and trainer.actor_update_interval > 1 else (1,)):
            draws = [] if gen is None else \
                trainer._noise_draws(self.B, p_id, "target") + (trainer._noise_draws(self.B, p_id, "actor") if upd else [])
            arr = (capi.TrngDraw * max(1, len(draws)))(*draws)
            _grow_scratch(gen, draws)
            g = C.c_void_p()
            capi.check(self.lib.mx_maddpg_graph_capture_ex(
                self._rep.handle, e.handle, self.B, float(beta), self.flags, capi.ptr(self.tnoise_dev), capi.ptr(self.anoise_dev), upd,
                capi.ptr(gen.state) if draws else None, arr, len(draws), capi.ptr(gen._scratch) if draws else None,
                gen._scratch.numel() if draws else 0, self._sp, C.byref(g)))
            self.graphs[upd], self._draws[upd] = g, arr
        self.num_kernels = {u: int(self.lib.mx_graph_num_kernels(g)) for u, g in self.graphs.items()}
        self._keep = (buffer, trainer, gen, gen and gen._scratch)      # the captured fills read this scratch: keep it alive

    def launch(self, beta=None):
        """One update; returns whether it updated the actor."""
        tr = self.trainer
        self._set_beta(beta)
        upd = 1 if tr.num_updates[self.p_id] % tr.actor_update_interval == 0 else 0
        if self._gen is None:
            self._stage_noise(upd)
        capi.check(self.lib.mx_graph_launch(self.graphs[upd], self._sp))
        if tr.counts_updates:
            tr.num_updates[self.p_id] += 1
        return bool(upd)

    def _stage_noise(self, upd):
        """Host noise mode: this update's draws into the next pinned slot, and their copies enqueued on the graph's stream."""
        tr, pol, B = self.trainer, self.pol, self.B
        k = self._slot
        self._slot = (k + 1) % self.RING
        if self._copied[k] is not None:
            self._copied[k].synchronize()
        with torch.cuda.stream(self.stream) if self.cuda else contextlib.nullcontext():
            if pol.td3:
                tr.place_noise(tr.draw_target_noise(B, self.p_id), self.tnoise_host[k], tr.noise_rows["target"][0])
                self.tnoise_dev.copy_(self.tnoise_host[k], non_blocking=True)
            if pol.discrete and upd:
                tr.place_noise(tr.draw_actor_noise(B, self.p_id), self.anoise_host[k], tr.noise_rows["actor"][0])
                self.anoise_dev.copy_(self.anoise_host[k], non_blocking=True)
            if self.cuda and (pol.td3 or pol.discrete):
                if self._copied[k] is None:
                    self._copied[k] = torch.cuda.Event()
                self._copied[k].record(self.stream)

    def close(self):
        for g in self.graphs.values():
            self.lib.mx_graph_destroy(g)
        self.graphs = {}


class MaddpgBatchTrainGraph(_Graph):
    """One `batch_train` of the runner (runner/{rnn,mlp}/base_runner.py) for a trainer with one policy per agent (share_policy off):
    R_MADDPG / R_MATD3 over a RecReplayBuffer / PrioritizedRecReplayBuffer, or MADDPG / MATD3 over an MlpReplayBuffer /
    PrioritizedMlpReplayBuffer, as CUDA graphs: one per update_actor variant the trainer can ask for.  A launch updates every
    policy in id order -- sample (uniform: one index set from the store `buffer.sample` draws from; PER: from the policy's own tree),
    every policy's centralised-action contribution, the step, the PER write-back to the policy's tree -- then soft-updates every
    policy when the actor was updated, as the eager runner does with `shared_train_policy_on_batch` per policy.  The indices come
    from the stores' device MT19937 streams, so the buffer must be in device RNG mode (`seed_device_rng` / `adopt_numpy_rng`).

    Noise modes as in MaddpgStepGraph.  Host mode: per `launch()` the host makes every draw of the whole batch_train in the eager
    order (per updated policy p: the target noise of every policy q in id order, then p's actor draws) into one pinned staging slot
    and enqueues their copies, one device buffer per draw.  Device mode: the fills sit in the graph before each policy's update.

    After a launch each policy's train_info and priorities are in its engine's `info` / `prio` views (trainer._eng[p_id])."""

    RING = 4

    def __init__(self, buffer, trainer, batch_size, beta=0.4, soft_update=True):
        _refuse_data_parallel("MaddpgBatchTrainGraph", trainer)
        if not getattr(trainer, "multi", False):
            raise ValueError("MaddpgBatchTrainGraph: the trainer has one shared policy; its update is captured by MaddpgStepGraph")
        ids = list(trainer.policy_ids)
        if sorted(buffer.policy_buffers) != ids:
            raise ValueError("MaddpgBatchTrainGraph: the buffer holds policies %s, the trainer %s" % (sorted(buffer.policy_buffers), ids))
        if getattr(buffer, "rng", None) != "device":
            raise ValueError("MaddpgBatchTrainGraph: the graph draws its indices from the stores' device RNG streams; put the buffer in "
                             "device RNG mode first (seed_device_rng / adopt_numpy_rng)")
        self.graphs = {}
        self.trainer, self.B, self.ids = trainer, int(batch_size), ids
        self._update_actor()                      # refuses update counts that differ modulo the interval
        B, P = self.B, len(ids)
        pbs = [buffer.policy_buffers[p] for p in ids]
        reps = [getattr(pb, "rep", pb) for pb in pbs]   # MlpPolicyBuffer wraps the episode replay
        first = buffer._first()
        uniform_store = reps.index(getattr(first, "rep", first))
        lib = capi.lib()
        for p, pb in zip(ids, pbs):
            if trainer._eng[p].cfg.mlp:
                capi.check(lib.mx_maddpg_set_valid(trainer._eng[p].handle, capi.ptr(pb.valid_dev)))
        self._gen = gen = trainer.noise_gen
        takes = trainer._takes_noise
        # device mode: the fills write each policy's own buffers inside the graph, update by update; host mode: every draw of the
        # batch_train is copied in before the launch, so each (updated policy, drawing policy) pair has a buffer of its own
        buf = (lambda p, q, w: trainer._noise_buffer(q, w, B)) if gen is not None else \
            (lambda p, q, w: torch.zeros_like(trainer._noise_buffer(q, w, B)))
        self.tnoise_dev = {(p, q): buf(p, q, "target") if takes(q, "target") else None for p in ids for q in ids}
        self.anoise_dev = {p: buf(p, p, "actor") if takes(p, "actor") else None for p in ids}
        self._open(reps[0], trainer, beta, soft_update)          # (after the buffers' zero fill)
        self._reps = reps
        if gen is None:
            # pinned staging ring: a slot is rewritten only after the H2D copies that last read it have completed (its event)
            host = lambda d: None if d is None else (torch.zeros(d.shape).pin_memory() if self.cuda else torch.zeros(d.shape))
            self._ring = [({k: host(d) for k, d in self.tnoise_dev.items()}, {k: host(d) for k, d in self.anoise_dev.items()})
                          for _ in range(self.RING)]
            self._copied, self._slot = [None] * self.RING, 0
        stores = (C.c_void_p * P)(*[r.handle for r in reps])
        learners = (C.c_void_p * P)(*[trainer._eng[p].handle for p in ids])
        tptr = (C.c_void_p * (P * P))(*[capi.ptr(self.tnoise_dev[p, q]) for p in ids for q in ids])
        aptr = (C.c_void_p * P)(*[capi.ptr(self.anoise_dev[p]) for p in ids])
        self._draws = {}
        for upd in ((1, 0) if trainer.counts_updates and trainer.actor_update_interval > 1 else (1,)):
            per_policy = [[] if gen is None else
                          sum((trainer._noise_draws(B, q, "target", self.tnoise_dev[p, q]) for q in ids), []) +
                          (trainer._noise_draws(B, p, "actor", self.anoise_dev[p]) if upd else []) for p in ids]
            draws = sum(per_policy, [])
            arr = (capi.TrngDraw * max(1, len(draws)))(*draws)
            counts = (C.c_int32 * P)(*[len(d) for d in per_policy])
            _grow_scratch(gen, draws)
            g = C.c_void_p()
            capi.check(self.lib.mx_maddpg_batch_graph_capture(
                stores, learners, P, uniform_store, B, float(beta), self.flags, tptr, aptr, upd, capi.ptr(gen.state) if draws else None,
                arr, counts, capi.ptr(gen._scratch) if draws else None, gen._scratch.numel() if draws else 0, self._sp, C.byref(g)))
            self.graphs[upd], self._draws[upd] = g, (arr, counts)
        self.num_kernels = {u: int(self.lib.mx_graph_num_kernels(g)) for u, g in self.graphs.items()}
        self._keep = (buffer, trainer, gen, gen and gen._scratch, stores, learners, tptr, aptr)   # the captured fills read this scratch

    def _update_actor(self):
        """Whether this batch_train updates the actors; the policies' update counts must agree modulo the interval (one variant per
        graph)."""
        tr = self.trainer
        upd = {tr.num_updates[p] % tr.actor_update_interval == 0 for p in self.ids}
        if len(upd) > 1:
            raise ValueError("MaddpgBatchTrainGraph: the policies' update counts %s differ modulo the actor update interval %d"
                             % ([tr.num_updates[p] for p in self.ids], tr.actor_update_interval))
        return 1 if upd.pop() else 0

    def _set_beta(self, beta):
        """PER: every store draws (each policy samples from its own tree), so each keeps the exponent."""
        if beta is not None and self._per and float(beta) != self._beta:
            for r in self._reps:
                capi.check(self.lib.mx_replay_set_beta(r.handle, float(beta), self._sp))
            self._beta = float(beta)

    def launch(self, beta=None):
        """One batch_train; returns whether it updated the actors."""
        tr = self.trainer
        upd = self._update_actor()
        self._set_beta(beta)
        if self._gen is None:
            self._stage_noise(upd)
        capi.check(self.lib.mx_graph_launch(self.graphs[upd], self._sp))
        if tr.counts_updates:
            for p in self.ids:
                tr.num_updates[p] += 1
        return bool(upd)

    def _stage_noise(self, upd):
        """Host noise mode: the batch_train's draws, in the eager order, into the next pinned slot, and their copies enqueued on the
        graph's stream."""
        tr, B = self.trainer, self.B
        k = self._slot
        self._slot = (k + 1) % self.RING
        if self._copied[k] is not None:
            self._copied[k].synchronize()
        th, ah = self._ring[k]
        copied = False
        with torch.cuda.stream(self.stream) if self.cuda else contextlib.nullcontext():
            for p in self.ids:
                for q in self.ids:
                    if th[p, q] is not None:
                        tr.place_noise(tr.draw_target_noise(B, q), th[p, q], tr.noise_rows["target"][0])
                        self.tnoise_dev[p, q].copy_(th[p, q], non_blocking=True)
                        copied = True
                if upd and ah[p] is not None:
                    tr.place_noise(tr.draw_actor_noise(B, p), ah[p], tr.noise_rows["actor"][0])
                    self.anoise_dev[p].copy_(ah[p], non_blocking=True)
                    copied = True
            if self.cuda and copied:
                if self._copied[k] is None:
                    self._copied[k] = torch.cuda.Event()
                self._copied[k].record(self.stream)

    def close(self):
        for g in self.graphs.values():
            self.lib.mx_graph_destroy(g)
        self.graphs = {}
