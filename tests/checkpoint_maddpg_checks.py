"""Checkpoint / resume of the MADDPG-family learners (R-MADDPG / R-MATD3, MADDPG / MATD3) and of the transition replays
(MlpReplayBuffer / PrioritizedMlpReplayBuffer, also under M-QMIX): a run restored from `save_checkpoint` into fresh objects continues
bit-identically.  Shared by the emulated and the GPU test modules; same pattern as checkpoint_checks.check_resume.

A `Case` describes one trainer + replay configuration.  One round = insert a few episodes / transitions (so the ring wraps after the
checkpoint), sample, train every policy, write PER priorities back, soft-update; it returns what a caller can see of that round:
sampled indices, every train_info scalar, the new priorities."""
import contextlib
import os
import tempfile

import numpy as np
import torch

from offpolicy._b200 import capi
from offpolicy._b200 import factory as fx
from offpolicy._b200.checkpoint import save_checkpoint, load_checkpoint


class Case(object):
    """kind: "rec" (R_MADDPG / R_MATD3 over a RecReplayBuffer), "mlp" (MADDPG / MATD3 over an MlpReplayBuffer) or "mqmix" (M_QMix over
    an MlpReplayBuffer).  specs: one (n_agents, obs_dim, act) per policy, act an int or a list of MultiDiscrete sub-space widths."""

    def __init__(self, kind, specs, S, B, E, T=1, td3=False, discrete=True, per=False, rng="numpy", norm=False, avail=False,
                 interval=None, insert=2):
        self.kind, self.specs, self.S, self.B, self.E, self.T = kind, [tuple(s) for s in specs], S, B, E, T
        self.td3, self.discrete, self.per, self.rng, self.norm, self.avail = td3, discrete, per, rng, norm, avail
        self.interval, self.insert = interval, insert
        self.ids = ["policy_%d" % i for i in range(len(specs))]
        nxt, self.agents = 0, {}
        for p, (n, _, _) in zip(self.ids, self.specs):
            self.agents[p] = list(range(nxt, nxt + n))
            nxt += n
        self.n_agents = nxt
        self.max_batch = max(B, insert, 8)

    # -- construction -----------------------------------------------------------------------------------------------
    def build(self, seed):
        """(trainer, buffer, {p_id: policy}) constructed from scratch; `seed` sets the initial weights and the device RNG."""
        torch.manual_seed(seed)
        np.random.seed(seed)
        tr, pols = self._trainer()
        buf = self._buffer()
        if self.rng == "device":
            buf.seed_device_rng(seed)
        return tr, buf, pols

    def _trainer(self):
        dev = capi.device()
        if self.kind == "mqmix":
            n, o, a = self.specs[0]
            cfg = fx.LearnerConfig(n_agents=n, obs_dim=o, act_dim=a, state_dim=self.S, use_per=self.per, gain=1.0)
            _, pol, tr = fx.build_mqmix(cfg, self.B)
            return tr, {"policy_0": pol}
        if self.kind == "mlp":
            if len(self.specs) == 1:
                n, o, a = self.specs[0]
                _, pol, tr = fx.build_mlp_maddpg(n, o, a, self.S, self.B, discrete=self.discrete, td3=self.td3, use_per=self.per)
                return tr, {"policy_0": pol}
            _, pols, tr, _ = fx.build_mlp_maddpg_multi([(o, a, n) for n, o, a in self.specs], self.S, self.B, discrete=self.discrete,
                                                        td3=self.td3, use_per=self.per)
            return tr, pols
        if self.td3:
            from offpolicy.algorithms.r_matd3.algorithm.rMATD3Policy import R_MATD3Policy as Policy
            from offpolicy.algorithms.r_matd3.r_matd3 import R_MATD3 as Trainer
        else:
            from offpolicy.algorithms.r_maddpg.algorithm.rMADDPGPolicy import R_MADDPGPolicy as Policy
            from offpolicy.algorithms.r_maddpg.r_maddpg import R_MADDPG as Trainer
        args = fx.maddpg_args(fx.MaddpgLearnerConfig(use_per=self.per, td3=self.td3, discrete=self.discrete, gain=1.0), self.B)
        cent_act = sum(n * a for n, _, a in self.specs)
        pols = {}
        for p, (n, o, a) in zip(self.ids, self.specs):
            info = dict(obs_space=fx.Box(o, -np.inf, np.inf), share_obs_space=fx.Box(self.S, -np.inf, np.inf),
                        act_space=fx.Discrete(a) if self.discrete else fx.Box(a), cent_obs_dim=self.S, cent_act_dim=cent_act)
            pols[p] = Policy({"args": args, "device": dev}, info)
        owner = {k: p for p, ks in self.agents.items() for k in ks}
        kw = {"actor_update_interval": self.interval} if self.interval else {}
        tr = Trainer(args, self.n_agents, pols, lambda k: owner[k], device=dev, episode_length=self.T, **kw)
        return tr, pols

    def _spaces(self):
        return {p: dict(obs_space=[o], share_obs_space=[self.S], act_space=fx.act_space(a, self.discrete))
                for p, (_, o, a) in zip(self.ids, self.specs)}

    def _buffer(self):
        from offpolicy.utils.rec_buffer import RecReplayBuffer, PrioritizedRecReplayBuffer
        from offpolicy.utils.mlp_buffer import MlpReplayBuffer, PrioritizedMlpReplayBuffer
        info, mb = self._spaces(), self.max_batch
        if self.kind == "rec":
            if self.per:
                return PrioritizedRecReplayBuffer(0.6, info, self.agents, self.E, self.T, True, self.avail, self.norm, rng=self.rng, max_batch=mb)
            return RecReplayBuffer(info, self.agents, self.E, self.T, True, self.avail, self.norm, rng=self.rng, max_batch=mb)
        if self.per:
            return PrioritizedMlpReplayBuffer(0.6, info, self.agents, self.E, True, self.avail, self.norm, rng=self.rng, max_batch=mb)
        return MlpReplayBuffer(info, self.agents, self.E, True, self.avail, self.norm, rng=self.rng, max_batch=mb)

    # -- data -------------------------------------------------------------------------------------------------------
    def _acts(self, rs, lead, a):
        if isinstance(a, (list, tuple)):
            return np.concatenate([np.eye(k, dtype=np.float32)[rs.randint(0, k, lead)] for k in a], -1)
        if self.discrete:
            return np.eye(a, dtype=np.float32)[rs.randint(0, a, lead)]
        return rs.uniform(-1, 1, lead + (a,)).astype(np.float32)

    def _avail(self, rs, lead, a):
        if not self.avail:
            return None
        w = fx.act_width(a)
        m = (rs.rand(*(lead + (w,))) < 0.7).astype(np.float32)
        m[..., 0] = 1.0
        return m

    def fill(self, buf, rs, n):
        while n > 0:
            k = min(n, self.max_batch)
            self.put(buf, rs, k)
            n -= k

    def put(self, buf, rs, n):
        """n random episodes (kind "rec") or transitions into every policy's store."""
        f32 = lambda x: np.asarray(x, dtype=np.float32)
        if self.kind == "rec":
            T = self.T
            share = rs.randn(T + 1, n, self.S)
            rew = rs.randn(T, n, 1, 1)
            de = np.maximum.accumulate((rs.rand(T, n, 1) < 0.15).astype(np.float32), axis=0)
            obs, acts, rews, dones, share_d, de_d, av = {}, {}, {}, {}, {}, {}, {}
            for p, (N, o, a) in zip(self.ids, self.specs):
                obs[p] = f32(rs.randn(T + 1, n, N, o))
                acts[p] = self._acts(rs, (T, n, N), a)
                rews[p], dones[p] = f32(np.repeat(rew, N, 2)), f32(np.repeat(de[:, :, None], N, 2))
                share_d[p], de_d[p] = f32(share), de
                av[p] = self._avail(rs, (T + 1, n, N), a)
            buf.insert(n, obs, share_d, acts, rews, dones, de_d, av if self.avail else None)
            return
        share, nshare = rs.randn(n, self.S), rs.randn(n, self.S)
        rew, de = rs.randn(n, 1, 1), (rs.rand(n, 1) < 0.2).astype(np.float32)
        d = {k: {} for k in ("obs", "acts", "rew", "nobs", "dones", "valid", "av", "nav", "share", "nshare", "de")}
        for p, (N, o, a) in zip(self.ids, self.specs):
            d["obs"][p], d["nobs"][p] = f32(rs.randn(n, N, o)), f32(rs.randn(n, N, o))
            d["acts"][p] = self._acts(rs, (n, N), a)
            d["rew"][p], d["dones"][p] = f32(np.repeat(rew, N, 1)), f32(np.repeat(de[:, :, None], N, 1))
            d["valid"][p] = (rs.rand(n, N, 1) < 0.9).astype(np.float32)
            d["av"][p], d["nav"][p] = self._avail(rs, (n, N), a), self._avail(rs, (n, N), a)
            d["share"][p], d["nshare"][p], d["de"][p] = f32(share), f32(nshare), de
        buf.insert(n, d["obs"], d["share"], d["acts"], d["rew"], d["nobs"], d["nshare"], d["dones"], d["de"], d["valid"],
                   d["av"] if self.avail else None, d["nav"] if self.avail else None)

    # -- one round ----------------------------------------------------------------------------------------------------
    def first_store(self, buf):
        pb = buf.policy_buffers["policy_0"]
        return getattr(pb, "rep", pb)

    def round(self, tr, buf, pols, rs, insert=True):
        if insert and self.insert:
            self.put(buf, rs, self.insert)
        smp = buf.sample(self.B, 0.5, "policy_0") if self.per else buf.sample(self.B)
        out = [np.asarray(self.first_store(buf).sampled_indices(self.B)).tolist()]
        if self.kind == "mqmix":
            info, prio, idx = tr.train_policy_on_batch(smp, True)
            out.append([float(info[k]) for k in ("loss", "grad_norm", "Q_tot")])
            if self.per:
                out.append(np.asarray(prio).tolist())
                buf.update_priorities(idx, prio, "policy_0")
            tr.soft_target_updates()
            return out
        upd_any = False
        for p in self.ids:
            info, prio, idx = tr.train_policy_on_batch(p, smp)
            out.append(sorted((k, float(v) if torch.is_tensor(v) else v) for k, v in info.items()))
            if self.per:
                out.append(np.asarray(prio).tolist())
                buf.update_priorities(idx, prio, p)
            upd_any = upd_any or bool(info["update_actor"])
        if upd_any:
            for p in self.ids:
                pols[p].soft_target_updates()
        return out


def snapshot(tr, buf):
    """Everything the learner and the replay hold that the next rounds depend on and a caller can read."""
    if capi.device().type == "cuda":
        torch.cuda.synchronize()
    snap = {"len": len(buf)}
    if hasattr(tr, "_eng"):
        lib = capi.lib()
        for p in tr.policy_ids:
            e = tr._eng[p]
            snap[p] = {"vecs": [v.cpu().clone() for v in e.pol.actor_vecs + e.pol.critic_vecs],
                       "adam": [tr.ws_view(n, p, torch.float64).cpu().clone() for n in ("adam_ta", "adam_tc")],
                       "num_updates": tr.num_updates[p], "engine_updates": int(lib.mx_maddpg_num_updates(e.handle))}
    else:
        snap["qmix"] = [v.cpu().clone() for v in (tr.theta, tr.theta_tgt, tr.adam_m, tr.adam_v, tr.ws_view("adam_t", torch.float64))]
    return snap


def assert_same(a, b, where="state"):
    if torch.is_tensor(a):
        assert torch.equal(a, b), where
    elif isinstance(a, dict):
        assert sorted(a) == sorted(b), where
        for k in a:
            assert_same(a[k], b[k], "%s.%s" % (where, k))
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            assert_same(x, y, "%s[%d]" % (where, i))
    else:
        assert a == b, (where, a, b)


def _prefix(case, k):
    """A run that has done k rounds, the last of them filling the ring: (trainer, buffer, policies, data stream)."""
    tr, buf, pols = case.build(1)
    rs = np.random.RandomState(5)
    case.fill(buf, rs, case.E - k * case.insert)         # the rounds after the checkpoint wrap the ring
    np.random.seed(11)
    torch.manual_seed(11)
    for _ in range(k):
        case.round(tr, buf, pols, rs)
    return tr, buf, pols, rs


def check_resume(case, k=2):
    """k rounds, save, k more (the ring wraps) = the uninterrupted run; fresh objects under other seeds, load, the same k rounds: every
    train_info scalar, the sampled indices, the PER priorities, all eight vectors of every policy, the Adam counters, num_updates and
    len(buffer) bit-identical."""
    tr, buf, pols, rs = _prefix(case, k)
    with tempfile.TemporaryDirectory() as d:
        path = save_checkpoint(os.path.join(d, "ck.pt"), tr, buf, extra={"round": k})
        rs_state = rs.get_state()
        want = [case.round(tr, buf, pols, rs) for _ in range(k)]
        want_snap = snapshot(tr, buf)
        del tr, buf, pols
        tr2, buf2, pols2 = case.build(2)
        np.random.seed(999)
        torch.manual_seed(999)
        assert load_checkpoint(path, tr2, buf2) == {"round": k}
    rs.set_state(rs_state)
    got = [case.round(tr2, buf2, pols2, rs) for _ in range(k)]
    assert_same(got, want, "rounds")
    assert_same(snapshot(tr2, buf2), want_snap)
    return tr2, pols2


def _stream_ctx():
    if capi.device().type != "cuda":
        return contextlib.nullcontext(), None
    side = torch.cuda.Stream()                 # a capture needs a non-default stream
    side.wait_stream(torch.cuda.current_stream())
    return torch.cuda.stream(side), side


def _info_record(case, tr, buf, upd):
    if capi.device().type == "cuda":
        torch.cuda.synchronize()
    info = tr._eng["policy_0"].info
    return [np.asarray(case.first_store(buf).sampled_indices(case.B)).tolist(), float(info[0]), float(info[1])] + \
        ([float(info[4]), float(info[5])] if upd else []) + [bool(upd)]


def check_graph_resume(case, k=3):
    """As check_resume, but the restored objects run the k rounds through the captured whole-update graph (MaddpgStepGraph), against
    the uninterrupted run's eager rounds.  The graph samples from the device RNG and inserts nothing, so neither do the rounds after the
    checkpoint here."""
    assert case.rng == "device" and not case.per and len(case.specs) == 1
    tr, buf, pols, rs = _prefix(case, k)
    with tempfile.TemporaryDirectory() as d:
        path = save_checkpoint(os.path.join(d, "ck.pt"), tr, buf)
        want = []
        for _ in range(k):
            r = case.round(tr, buf, pols, rs, insert=False)
            want.append(_info_record(case, tr, buf, dict(r[1])["update_actor"]))
        want_snap = snapshot(tr, buf)
        del tr, buf, pols
        tr2, buf2, pols2 = case.build(2)
        np.random.seed(999)
        torch.manual_seed(999)
        load_checkpoint(path, tr2, buf2)
    got = []
    ctx, side = _stream_ctx()
    with ctx:
        from offpolicy._b200.graph import MaddpgStepGraph
        g = MaddpgStepGraph(buf2, tr2, case.B)
        for _ in range(k):
            upd = g.launch()
            g.synchronize()
            got.append(_info_record(case, tr2, buf2, upd))
        g.close()
    assert_same(got, want, "rounds")
    assert_same(snapshot(tr2, buf2), want_snap)


# ---- host fences: a process that keeps building fresh replays (every resume does) must not run out -----------------------------
def check_fence_pool_reuses_released_ids():
    lib = capi.lib()
    held = []
    while True:
        f = lib.mx_host_fence_alloc()
        if f < 0:
            break
        held.append(f)
    assert held and b"out of fences" in lib.mx_last_error()
    try:
        assert lib.mx_host_fence_release(held[-1]) == 0
        assert lib.mx_host_fence_record(held[-1], None) != 0 and lib.mx_host_fence_wait(held[-1]) != 0      # a released id is dead
        assert lib.mx_host_fence_release(held[-1]) != 0 and b"bad fence" in lib.mx_last_error()
        assert lib.mx_host_fence_alloc() == held[-1]
        assert lib.mx_host_fence_record(held[-1], None) == 0 and lib.mx_host_fence_wait(held[-1]) == 0
    finally:
        for f in held:
            lib.mx_host_fence_release(f)


def check_dropped_buffers_release_their_fences(n=60):
    """Each store holds up to six fences (insert staging, host-drawn index ring); n built, used and dropped stores need more than the
    process-wide pool of 256 unless a dropped store gives its fences back."""
    import gc
    case = Case("rec", [(2, 6, 2)], S=8, B=4, E=8, T=4, discrete=False)
    rs = np.random.RandomState(0)
    for _ in range(n):
        buf = case._buffer()
        case.fill(buf, rs, case.E)
        buf.sample(case.B)
        del buf
        gc.collect()
    buf = case._buffer()
    case.fill(buf, rs, case.E)
    buf.sample(case.B)


# ---- configurations of another shape are refused -----------------------------------------------------------------------------
def check_rejected(case_a, case_b, trainer=True, buffer=False, a_objects=None):
    """A checkpoint of case_a does not load into case_b's trainer / buffer: ValueError, and nothing of case_b was overwritten."""
    tr, buf, _ = a_objects if a_objects is not None else case_a.build(1)
    tr2, buf2, _ = case_b.build(2)
    before = snapshot(tr2, buf2)
    with tempfile.TemporaryDirectory() as d:
        path = save_checkpoint(os.path.join(d, "ck.pt"), tr if trainer else None, buf if buffer else None)
        try:
            load_checkpoint(path, tr2 if trainer else None, buf2 if buffer else None, restore_host_rng=False)
        except ValueError:
            pass
        else:
            raise AssertionError("a checkpoint of another configuration was accepted")
    assert_same(snapshot(tr2, buf2), before, "after a refused load")
