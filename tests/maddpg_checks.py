"""R-MADDPG / R-MATD3 learner parity checks (emulated CPU build and real GPU): reference goldens + the pinned oracle in lock-step."""
import types

import numpy as np
import torch

from helpers import load_golden, sub, rel_err
from qmix_checks import close
from test_oracle_maddpg import maddpg_from_golden, maddpg_batch, actor_noise


from offpolicy._b200.factory import Box, Discrete, maddpg_args as make_args, build_maddpg as build  # noqa: E402,F401


def ref_tuple(b):
    d = lambda x: {"policy_0": x}
    return tuple(d(x) for x in b[:7]) + (b[7], b[8])


def named_views(flat, entries):
    out = {}
    for name, off, rows, cols in entries:
        n = rows * (cols if cols else 1)
        out[name] = flat[off:off + n].view(rows, cols) if cols else flat[off:off + n]
    return out


def check_golden(name):
    g = load_golden(name)
    L, cfg, B, T, steps = maddpg_from_golden(g)
    args, pol, tr = build(cfg, B, T)
    for tag, mod in (("actor", pol.actor), ("critic", pol.critic), ("tgt_actor", pol.target_actor), ("tgt_critic", pol.target_critic)):
        mod.load_state_dict(sub(g, "init.%s." % tag))
    problems = []
    for s in range(steps):
        batch, noise = maddpg_batch(g, s)
        torch.manual_seed(1000 + s)                         # the trainer draws the MATD3 / Gumbel noise from torch's CPU RNG like the reference
        info, prio, _ = tr.shared_train_policy_on_batch("policy_0", ref_tuple(batch))
        ref, rprio = L.step(batch, noise, actor_noise(g, s))
        ga, gc = tr.grad_views()
        for key in ("critic_loss", "critic_grad_norm"):
            e = rel_err(info[key].cpu(), g["s%d.%s" % (s, key)])
            if e > 1e-4:
                problems.append("step %d %s rel err %.3e (got %r want %r)" % (s, key, e, float(info[key]), float(g["s%d.%s" % (s, key)])))
        coef = min(1.0, cfg.max_grad_norm / (float(ref["critic_grad_norm"]) + 1e-6))
        cviews = named_views(gc, pol._c_entries)
        for k, gr in L.critic_grads.items():
            ok, err, lim = close(cviews[k] / gc[pol.Pc] * coef, gr, 1e-4)
            if not ok:
                problems.append("step %d critic grad %s err %.3e > %.3e" % (s, k, err, lim))
        assert bool(info["update_actor"]) == bool(int(g["s%d.update_actor" % s]))
        if info["update_actor"]:
            for key in ("actor_loss", "actor_grad_norm"):
                e = rel_err(info[key].cpu(), g["s%d.%s" % (s, key)])
                if e > 1e-4:
                    problems.append("step %d %s rel err %.3e (got %r want %r)" % (s, key, e, float(info[key]), float(g["s%d.%s" % (s, key)])))
            coef = min(1.0, cfg.max_grad_norm / (float(g["s%d.actor_grad_norm" % s]) + 1e-6))
            aviews = named_views(ga, pol._a_entries)
            for k, v in aviews.items():
                key = "s%d.grad.actor.%s" % (s, k)
                if key in g:
                    ok, err, lim = close(v / ga[pol.Pa] * coef, g[key], 1e-4)
                    if not ok:
                        problems.append("step %d actor grad %s err %.3e > %.3e" % (s, k, err, lim))
            pol.soft_target_updates()
            L.soft_update()
        if cfg.use_per:
            ok, err, lim = close(np.asarray(prio), g["s%d.prio" % s], 1e-4)
            if not ok:
                problems.append("step %d priorities err %.3e" % (s, err))
    for tag, mod in (("actor", pol.actor), ("critic", pol.critic), ("tgt_actor", pol.target_actor), ("tgt_critic", pol.target_critic)):
        for k, v in mod.state_dict().items():
            want = g["final.%s.%s" % (tag, k)]
            err = np.abs(v.cpu().numpy() - want).max()
            if err > 5e-3 * cfg.lr * steps + 1e-7:
                problems.append("final %s.%s err %.3e" % (tag, k, err))
    assert not problems, "\n".join(problems[:40])


def check_get_actions(name):
    """Rollout-time `get_actions` / `get_random_actions` against the reference (seeded), rMADDPGPolicy.py:62-160."""
    g = load_golden(name)
    L, cfg, B, T, steps = maddpg_from_golden(g)
    args, pol, tr = build(cfg, B, T)
    pol.actor.load_state_dict(sub(g, "init.actor."))
    obs, h = g["act.in.obs"], torch.from_numpy(g["act.in.h"])
    a, h2, _ = pol.get_actions(obs, None, h, explore=False)
    a = a.cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    if cfg.discrete:
        assert np.array_equal(a, g["act.greedy"])
    else:
        assert np.abs(a - g["act.greedy"]).max() < 1e-5
    assert np.abs(h2.cpu().numpy() - g["act.new_h"]).max() < 1e-5
    torch.manual_seed(5); np.random.seed(5)
    a, _, eps = pol.get_actions(obs, None, h, t_env=20000, explore=True)
    a = a.cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
    if cfg.discrete:
        assert abs(eps - float(g["act.eps"])) < 1e-12
        assert np.array_equal(a.astype(np.float32), g["act.explore"])
    else:
        assert np.abs(a - g["act.explore"]).max() < 1e-5
    torch.manual_seed(6); np.random.seed(6)
    r = np.asarray(pol.get_random_actions(obs), dtype=np.float32)
    assert np.array_equal(r, g["act.random"])


def check_graph_matches_eager(td3, disc, B=4, T=6, E=16, steps=4):
    """sample -> shared_train_policy_on_batch -> soft update through the drop-in classes, eager vs the captured whole-update
    CUDA graphs (one per update_actor variant): same device RNG stream, same torch CPU noise stream -> same parameters."""
    import replay_checks as rc
    from offpolicy.utils.rec_buffer import RecReplayBuffer
    from offpolicy._b200.graph import MaddpgStepGraph
    from oracle.maddpg import MaddpgConfig
    from oracle.qmix import randomize_all
    cfg = MaddpgConfig(act_dim=5 if disc else 2, discrete=disc, td3=td3, actor_update_interval=2 if td3 else 1, gain=1.0)
    n, o, a, sdim = cfg.n_agents, cfg.obs_dim, cfg.act_dim, cfg.state_dim
    results = []
    for mode in ("eager", "graph"):
        rs = np.random.RandomState(3)
        info = {"policy_0": dict(obs_space=[o], share_obs_space=[sdim], act_space=Discrete(a) if disc else Box(a))}
        buf = RecReplayBuffer(info, {"policy_0": list(range(n))}, E, T, True, False, rng="device", max_batch=max(B, E))
        acts = np.eye(a, dtype=np.float32)[rs.randint(0, a, (T, E, n))] if disc else rs.uniform(-1, 1, (T, E, n, a)).astype(np.float32)
        ep = [rs.randn(T + 1, E, n, o).astype(np.float32), np.repeat(rs.randn(T + 1, E, 1, sdim).astype(np.float32), n, 2), acts,
              np.repeat(rs.randn(T, E, 1, 1).astype(np.float32), n, 2), np.zeros((T, E, n, 1), np.float32), np.zeros((T, E, 1), np.float32)]
        buf.insert(E, *[rc.d(x) for x in ep], None)
        torch.manual_seed(1)
        args, pol, tr = build(cfg, B, T)
        init = torch.Generator().manual_seed(11)
        for vec in (pol.actor_vecs[0], pol.critic_vecs[0]):
            vec.add_((0.05 * torch.randn(vec.shape, generator=init)).to(vec.device))
        pol.hard_target_updates()
        buf.seed_device_rng(5)
        torch.manual_seed(99)
        upds = []
        if mode == "eager":
            for s in range(steps):
                smp = buf.sample(B)
                info_t, _, _ = tr.shared_train_policy_on_batch("policy_0", smp)
                upds.append(bool(info_t["update_actor"]))
                if info_t["update_actor"]:
                    pol.soft_target_updates()
        else:
            g = MaddpgStepGraph(buf, tr, B)
            for s in range(steps):
                upds.append(g.launch())
            g.synchronize()
            g.close()
        results.append(([v.clone().cpu() for v in pol.actor_vecs + pol.critic_vecs], upds))
    assert results[0][1] == results[1][1]
    for x, y in zip(results[0][0], results[1][0]):
        assert float((x - y).abs().max()) <= 1e-6 * float(x.abs().max()) + 1e-7


def check_replay_batch_equals_host_batch(T=5, B=4, E=9):
    """The replay's batch region pads every episode row of the per-step fields (rewards / dones / dones_env) to 16 bytes; the
    learner must index them with the reported episode strides.  T * N = 15 and T = 5 are not multiples of 4 here: training on the
    device-side sample and on the same sample handed over as NumPy arrays (dense host layout) must give the same update."""
    import replay_checks as rc
    from offpolicy.utils.rec_buffer import RecReplayBuffer
    from oracle.maddpg import MaddpgConfig
    cfg = MaddpgConfig(act_dim=2, discrete=False, td3=False, actor_update_interval=1, gain=1.0)
    n, o, a, sdim = cfg.n_agents, cfg.obs_dim, cfg.act_dim, cfg.state_dim
    rs = np.random.RandomState(3)
    info = {"policy_0": dict(obs_space=[o], share_obs_space=[sdim], act_space=Box(a))}
    buf = RecReplayBuffer(info, {"policy_0": list(range(n))}, E, T, True, False, rng="numpy", max_batch=max(B, E))
    de = np.maximum.accumulate((rs.rand(T, E, 1) < 0.2).astype(np.float32), axis=0)
    ep = [rs.randn(T + 1, E, n, o).astype(np.float32), np.repeat(rs.randn(T + 1, E, 1, sdim).astype(np.float32), n, 2),
          rs.uniform(-1, 1, (T, E, n, a)).astype(np.float32), np.repeat(rs.randn(T, E, 1, 1).astype(np.float32), n, 2),
          np.repeat(de[:, :, None], n, 2), de]
    buf.insert(E, *[rc.d(x) for x in ep], None)
    outs = []
    for mode in ("device", "host"):
        torch.manual_seed(1)
        args, pol, tr = build(cfg, B, T)
        init = torch.Generator().manual_seed(11)
        for vec in (pol.actor_vecs[0], pol.critic_vecs[0]):
            vec.add_((0.05 * torch.randn(vec.shape, generator=init)).to(vec.device))
        pol.hard_target_updates()
        np.random.seed(7)
        smp = buf.sample(B)
        if mode == "host":
            smp = tuple({"policy_0": smp[i]["policy_0"]} for i in range(6)) + (None, None, None)
        info_t, _, _ = tr.shared_train_policy_on_batch("policy_0", smp)
        outs.append(([float(info_t["critic_loss"]), float(info_t["actor_loss"])], [v.clone().cpu() for v in pol.actor_vecs[:1] + pol.critic_vecs[:1]]))
    assert outs[0][0] == outs[1][0], (outs[0][0], outs[1][0])
    for x, y in zip(outs[0][1], outs[1][1]):
        assert torch.equal(x, y)


# ---- several policies (share_policy = False) -------------------------------------------------------------------------------------------
def build_multi(specs, state_dim, td3, discrete, B, T, args_from):
    """One drop-in policy per agent + ONE trainer over all of them, like train/train_mpe.py:139-150 + runner/rnn/base_runner.py:110-150."""
    from offpolicy._b200 import capi, factory
    if td3:
        from offpolicy.algorithms.r_matd3.algorithm.rMATD3Policy import R_MATD3Policy as Policy
        from offpolicy.algorithms.r_matd3.r_matd3 import R_MATD3 as Trainer
    else:
        from offpolicy.algorithms.r_maddpg.algorithm.rMADDPGPolicy import R_MADDPGPolicy as Policy
        from offpolicy.algorithms.r_maddpg.r_maddpg import R_MADDPG as Trainer
    args = factory.maddpg_args(args_from, B)
    CA = sum(a for _, a in specs)
    pols = {}
    for i, (o, a) in enumerate(specs):
        info = dict(obs_space=Box(o, -np.inf, np.inf), share_obs_space=Box(state_dim, -np.inf, np.inf), act_space=Discrete(a) if discrete else Box(a),
                    cent_obs_dim=state_dim, cent_act_dim=CA)
        pols["policy_%d" % i] = Policy({"args": args, "device": capi.device()}, info)
    tr = Trainer(args, len(specs), pols, lambda a: "policy_%d" % a, device=capi.device(), episode_length=T)
    return args, pols, tr


def check_multi_golden(name, through_buffer=False):
    """Engine vs the reference's own outputs for one-policy-per-agent training (tests/golden/*_multi_*.npz, make_goldens.py multi): every
    policy updated from the same sample in id order, soft updates of all policies after a round that updated the actors.  With
    through_buffer the episodes go through a multi-policy RecReplayBuffer (insert -> sample with fixed indices) instead of host batches."""
    from test_oracle_maddpg import multi_from_golden, multi_round_inputs
    g = load_golden(name)
    L, specs, B, T, rounds, td3, disc = multi_from_golden(g)
    N = len(specs)
    S = int(g["meta.cfg"][1])
    args, pols, tr = build_multi(specs, S, td3, disc, B, T, L.cfgs[0])
    for i in range(N):
        pol = pols["policy_%d" % i]
        for tag, mod in (("actor", pol.actor), ("critic", pol.critic), ("tgt_actor", pol.target_actor), ("tgt_critic", pol.target_critic)):
            mod.load_state_dict(sub(g, "init.p%d.%s." % (i, tag)))
    problems = []
    pd = lambda v: {"policy_%d" % i: v for i in range(N)}
    lr = L.cfgs[0].lr
    for r in range(rounds):
        obs, share, acts, rew, dones, de = multi_round_inputs(g, r, N)
        batch = ({"policy_%d" % i: obs[i] for i in range(N)}, pd(share), {"policy_%d" % i: acts[i] for i in range(N)}, pd(rew[None]),
                 {"policy_%d" % i: dones[i] for i in range(N)}, pd(de), pd(None), None, None)
        if through_buffer:
            from offpolicy.utils.rec_buffer import RecReplayBuffer
            info = {"policy_%d" % i: dict(obs_space=[o], share_obs_space=[S], act_space=Discrete(a) if disc else Box(a)) for i, (o, a) in enumerate(specs)}
            buf = RecReplayBuffer(info, {"policy_%d" % i: [i] for i in range(N)}, B, T, True, False, rng="numpy", max_batch=max(B, 8))
            ep = lambda d_: {k: np.swapaxes(v, 0, 1) if v.ndim == 4 else v for k, v in d_.items()}       # (N_p,T,B,D) -> (T,B,N_p,D) insert layout
            buf.insert(B, ep(batch[0]), {k: np.repeat(share[:, :, None], 1, 2) for k in batch[1]}, ep(batch[2]), ep(batch[3]), ep(batch[4]), batch[5], None)
            for pb in buf.policy_buffers.values():
                pb.gather(np.arange(B))                    # fixed indices: the sample IS the golden batch
            from offpolicy.utils.rec_buffer import SampledBatch
            batch = SampledBatch(buf.policy_buffers, B, None, None, list(info.keys()))
        upd_any = False
        for i in range(N):
            p = "policy_%d" % i
            pol = pols[p]
            noises = {q: g["r%d.u%d.noise.p%d" % (r, i, q)] for q in range(N)} if td3 else None
            torch.manual_seed(2000 + 10 * r + i)            # the trainer draws the MATD3 / Gumbel noise from torch's CPU RNG in the reference's order
            info_t, _, _ = tr.shared_train_policy_on_batch(p, batch)
            ref = L.step(i, obs, share, acts, rew, dones, de, noises, g.get("r%d.u%d.actor_noise" % (r, i)))
            ga, gc = tr.grad_views(p)
            for key in ("critic_loss", "critic_grad_norm"):
                e = rel_err(info_t[key].cpu(), g["r%d.u%d.%s" % (r, i, key)])
                if e > 1e-4:
                    problems.append("round %d policy %d %s rel err %.3e (got %r want %r)" % (r, i, key, e, float(info_t[key]), float(g["r%d.u%d.%s" % (r, i, key)])))
            coef = min(1.0, L.cfgs[i].max_grad_norm / (float(ref["critic_grad_norm"]) + 1e-6))
            cviews = named_views(gc, pol._c_entries)
            for k, gr in L.critic_grads.items():
                ok, err, lim = close(cviews[k] / gc[pol.Pc] * coef, gr, 1e-4)
                if not ok:
                    problems.append("round %d policy %d critic grad %s err %.3e > %.3e" % (r, i, k, err, lim))
            assert bool(info_t["update_actor"]) == bool(int(g["r%d.u%d.update_actor" % (r, i)]))
            if info_t["update_actor"]:
                upd_any = True
                for key in ("actor_loss", "actor_grad_norm"):
                    e = rel_err(info_t[key].cpu(), g["r%d.u%d.%s" % (r, i, key)])
                    if e > 1e-4:
                        problems.append("round %d policy %d %s rel err %.3e (got %r want %r)" % (r, i, key, e, float(info_t[key]), float(g["r%d.u%d.%s" % (r, i, key)])))
                coef = min(1.0, L.cfgs[i].max_grad_norm / (float(g["r%d.u%d.actor_grad_norm" % (r, i)]) + 1e-6))
                aviews = named_views(ga, pol._a_entries)
                for k, v in aviews.items():
                    key = "r%d.u%d.grad.actor.%s" % (r, i, k)
                    if key in g:
                        ok, err, lim = close(v / ga[pol.Pa] * coef, g[key], 1e-4)
                        if not ok:
                            problems.append("round %d policy %d actor grad %s err %.3e > %.3e" % (r, i, k, err, lim))
        if upd_any:
            for i in range(N):
                pols["policy_%d" % i].soft_target_updates()
            L.soft_update_all()
    for i in range(N):
        pol = pols["policy_%d" % i]
        for tag, mod in (("actor", pol.actor), ("critic", pol.critic), ("tgt_actor", pol.target_actor), ("tgt_critic", pol.target_critic)):
            for k, v in mod.state_dict().items():
                want = g["final.p%d.%s.%s" % (i, tag, k)]
                err = np.abs(v.cpu().numpy() - want).max()
                if err > 5e-3 * lr * rounds + 1e-7:
                    problems.append("final p%d %s.%s err %.3e" % (i, tag, k, err))
    assert not problems, "\n".join(problems[:40])


def check_oracle_lockstep(cfg, B, T, steps=3, seed=40):
    """R-MADDPG / R-MATD3 whole updates at (B, T) in lock-step with the fp32 oracle, from the randomised state of
    row_coverage_checks.maddpg_pair: per update the losses, grad norms and every clipped critic / actor gradient tensor within 1e-4,
    the draws taken from torch's CPU generator in the trainer's order (R-MATD3's target noise, then the Discrete actor's Gumbel draws on
    the updates that train the actor), soft updates after each actor update; the parameters after the last one within 5e-3 lr per
    update.  Returns the worst gradient error relative to its bound."""
    import row_coverage_checks as rc
    from oracle.maddpg import MaddpgLearner, sample_gumbel, synth_batch_cont, synth_batch_disc
    L64, pol, tr = rc.maddpg_pair(cfg, B, T)
    L = MaddpgLearner(cfg, dtype=torch.float32)
    for dst, src in ((L.actor, pol.actor), (L.critic, pol.critic), (L.tgt_actor, pol.target_actor), (L.tgt_critic, pol.target_critic)):
        dst.load_state_dict({k: v.cpu() for k, v in src.state_dict().items()})
    N, problems, worst = cfg.n_agents, [], 0.0
    for s in range(steps):
        batch = (synth_batch_disc if cfg.discrete else synth_batch_cont)(cfg, B, T, seed=seed + s)
        w = np.random.RandomState(seed + 100 + s).rand(B).astype(np.float32) * 0.9 + 0.1
        batch = tuple(batch) + (w if cfg.use_per else None, np.arange(B) if cfg.use_per else None)
        update = tr.num_updates["policy_0"] % tr.actor_update_interval == 0
        torch.manual_seed(1000 + s)
        tnoise = tr.draw_target_noise(B).numpy() if cfg.td3 else None
        anoise = sample_gumbel((T, N * B, cfg.act_dim)).numpy() if cfg.discrete and update else None
        torch.manual_seed(1000 + s)
        info, _, _ = tr.shared_train_policy_on_batch("policy_0", ref_tuple(batch))
        ref, _ = L.step(batch, tnoise, anoise)
        ga, gc = tr.grad_views()
        assert bool(info["update_actor"]) == bool(ref["update_actor"]) == update, (s, info["update_actor"], ref["update_actor"])
        keys = ("critic_loss", "critic_grad_norm") + (("actor_loss", "actor_grad_norm") if update else ())
        for key in keys:
            e = rel_err(info[key].cpu(), ref[key])
            if e > 1e-4:
                problems.append("step %d %s rel err %.3e" % (s, key, e))
        nets = [(gc, pol.Pc, pol._c_entries, L.critic_grads, ref["critic_grad_norm"])]
        if update:
            nets.append((ga, pol.Pa, pol._a_entries, L.actor_grads, ref["actor_grad_norm"]))
        for flat, P, entries, grads, gn in nets:
            coef = min(1.0, cfg.max_grad_norm / (float(gn) + 1e-6))
            views = named_views(flat, entries)
            for k, gr in grads.items():
                ok, err, lim = close(views[k] / flat[P] * coef, gr, 1e-4)
                worst = max(worst, err / lim)
                if not ok:
                    problems.append("step %d grad %s err %.3e > %.3e" % (s, k, err, lim))
        if update:
            pol.soft_target_updates()
            L.soft_update()
    for mod, ref_mod in ((pol.actor, L.actor), (pol.critic, L.critic), (pol.target_actor, L.tgt_actor), (pol.target_critic, L.tgt_critic)):
        for k, v in mod.state_dict().items():
            err = float((v.cpu() - ref_mod.state_dict()[k]).abs().max())
            if err > 5e-3 * cfg.lr * steps + 1e-7:
                problems.append("final %s err %.3e" % (k, err))
    assert not problems, "\n".join(problems[:40])
    return worst
