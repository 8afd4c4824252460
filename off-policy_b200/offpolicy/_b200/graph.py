"""Whole-step CUDA graph: [sample ->] QMIX step [-> PER write-back] [-> soft update] captured once, replayed per step.

`mx_graph_capture` records the library's own launch sequence on a dedicated (non-default) stream; after that a learner
step costs one `cudaGraphLaunch` and no host work at all (indices come from the device-resident MT19937 stream).
"""
import contextlib
import ctypes as C

import torch

from offpolicy._b200 import capi

SAMPLE_UNIFORM, SAMPLE_PER, SOFT_UPDATE, PER_WRITEBACK = 1, 2, 4, 8


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
            if draws:
                words = max(gen.words(d) for d in draws)
                if gen._scratch.numel() < words:
                    gen._scratch = torch.zeros(words, dtype=torch.int32, device=capi.device())
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
