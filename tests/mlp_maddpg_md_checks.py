"""Shared checks of the transition-level MADDPG / MATD3 with MultiDiscrete action spaces (csrc/maddpg.cu cfg.act_seg,
algorithms/maddpg with `act_dim` an ndarray of sub-space widths) against oracle/maddpg_mlp_md.py: synthetic batches, the lock-step
comparison and the fixtures of tests/golden/make_goldens_mlp_maddpg_md.py.  The emulated tests and the GPU tests run the same checks at
different sizes.

A policy spec is (obs_dim, act, n_agents) with act an int (Discrete(act)) or a list of sub-space widths (MultiDiscrete)."""
import numpy as np
import torch

from helpers import load_golden, rel_err
from mlp_maddpg_checks import assert_actor_tail_unchanged, actor_tail_params, clipped_engine_grads, engine_grads, grad_errors
from mlp_maddpg_multi_checks import FIELDS, golden_batch_multi, golden_draws, golden_expected, golden_rng_before, golden_sd

from oracle.maddpg_mlp_md import MlpMaddpgMD, draw_noise_multi_md, step_multi_md

# simple_reference (scripts/train_mpe_matd3.sh): 2 agents, obs 21, MultiDiscrete([[0,4],[0,9]]) = move 5 + speak 10, shared obs 42
N, O, S, SEGS = 2, 21, 42, [5, 10]
REFERENCE_SPEC = [(O, SEGS, N)]


def width(act):
    return int(np.sum(act)) if isinstance(act, (list, tuple)) else int(act)


def norm_specs(specs):
    """[(obs_dim, act[, n_agents])] -> {policy_i: (obs_dim, act, n_agents)}."""
    out = {}
    for i, s in enumerate(specs):
        o, a = int(s[0]), s[1]
        a = [int(n) for n in a] if isinstance(a, (list, tuple, np.ndarray)) else int(a)
        out["policy_%d" % i] = (o, a, int(s[2]) if len(s) > 2 else 1)
    return out


def onehot_acts(rng, act, N, B):
    """Buffer actions of N agents: one one-hot block per sub-space (the runner stores np.concatenate of the blocks)."""
    segs = act if isinstance(act, list) else [act]
    return np.concatenate([np.eye(n, dtype=np.float32)[rng.integers(0, n, (N, B))] for n in segs], -1)


def synth_batch_md(rng, specs, B, S, per=False, avail=False):
    """A sample of every policy's store in the reference's layout (mlp_buffer.py:80-110): the 13-tuple of {policy_id: array}.  The
    stores hold the same transitions, so the shared observation and dones_env are one array.  avail: masks with zeros for every policy
    (a MultiDiscrete policy must ignore them)."""
    f = lambda *s: rng.standard_normal(s).astype(np.float32)
    share, nshare = f(B, S), f(B, S)
    dones_env = (rng.random((B, 1)) < 0.1).astype(np.float32)
    out = [dict() for _ in range(11)]
    for p, (o, a, n) in norm_specs(specs).items():
        A = width(a)
        av = nav = None
        if avail:
            av = (rng.random((n, B, A)) < 0.6).astype(np.float32)
            nav = (rng.random((n, B, A)) < 0.6).astype(np.float32)
        valid = (rng.random((n, B, 1)) < 0.8).astype(np.float32)
        valid[:, 0] = 1.0
        vals = (f(n, B, o), share, onehot_acts(rng, a, n, B), f(n, B, 1), f(n, B, o), nshare, (rng.random((n, B, 1)) < 0.1).astype(np.float32),
                dones_env, valid, av, nav)
        for d, v in zip(out, vals):
            d[p] = v
    w = (0.2 + rng.random(B)).astype(np.float32) if per else None
    return tuple(out) + (w, np.arange(B) if per else None)


def noise_shapes(tr):
    """{policy_id: (n_agents, act, discrete, td3, target_std)} of a trainer, for draw_noise_multi_md."""
    return {p: (e.n_agents, list(e.pol.act_segs) if e.pol.act_segs is not None else e.pol.act_dim, e.pol.discrete, e.pol.td3, e.pol.target_noise)
            for p, e in tr._eng.items()}


def oracle_from(args, pol):
    cpu = lambda m: {k: v.cpu() for k, v in m.state_dict().items()}
    return MlpMaddpgMD(cpu(pol.actor), cpu(pol.critic), cpu(pol.critic_heads), cpu(pol.target_actor), cpu(pol.target_critic),
                       cpu(pol.target_critic_heads), pol.discrete, pol.td3, gamma=args.gamma, lr=args.lr, eps=args.opti_eps,
                       weight_decay=args.weight_decay, max_grad_norm=args.max_grad_norm, tau=args.tau, huber=args.use_huber_loss,
                       huber_delta=args.huber_delta, use_per=args.use_per, per_eps=args.per_eps, relu=bool(args.use_ReLU),
                       feature_norm=bool(args.use_feature_normalization), segs=pol.act_segs)


def lockstep(args, pols, tr, batches, rtol=1e-4, ptol=2e-5):
    """Engine and oracle step through `batches`: per batch, every policy in id order (the runner's batch_train), then the soft target
    updates.  The engine's draws are replayed from the same RNG state for the oracle; returns the max deviations seen."""
    learners = {p: oracle_from(args, pol) for p, pol in pols.items()}
    heads0 = {p: ({k: v.clone() for k, v in pol.critic_heads.state_dict().items()},
                  {k: v.clone() for k, v in pol.target_critic_heads.state_dict().items()}) for p, pol in pols.items()}
    shapes = noise_shapes(tr)
    worst = {"info": 0.0, "param": 0.0, "prio": 0.0, "grad": 0.0}
    for s, batch in enumerate(batches):
        B = np.asarray(batch[0]["policy_0"]).shape[1]
        for p in sorted(pols):
            tail0 = actor_tail_params(pols[p])
            rng_before = torch.get_rng_state()
            info, prio, _ = tr.shared_train_policy_on_batch(p, batch)
            rng_after = torch.get_rng_state()
            torch.set_rng_state(rng_before)
            tn, an = draw_noise_multi_md(shapes, p, B)
            assert torch.equal(torch.get_rng_state(), rng_after), p
            ref, rprio, grads = step_multi_md(learners, p, batch, tn, an)
            assert info["update_actor"] is True
            assert_actor_tail_unchanged(pols[p], tail0)
            errs = grad_errors(clipped_engine_grads(tr, pols[p], ref, args.max_grad_norm, p), grads, rtol, "step %d %s" % (s, p))
            worst["grad"] = max([worst["grad"]] + list(errs.values()))
            for k, v in ref.items():
                d = abs(float(info[k]) - v) / max(1.0, abs(v))
                worst["info"] = max(worst["info"], d)
                assert d <= rtol, (p, k, float(info[k]), v)
            if rprio is not None:
                d = float(np.max(np.abs(np.asarray(prio) - rprio) / np.maximum(1.0, np.abs(rprio))))
                worst["prio"] = max(worst["prio"], d)
                assert d <= rtol, (p, d)
        for p in sorted(pols):
            pols[p].soft_target_updates()
            learners[p].soft_update()
        for p, pol in pols.items():
            L = learners[p]
            for mod, ref_sd in ((pol.actor, L.actor), (pol.critic, L.critic), (pol.target_actor, L.target_actor), (pol.target_critic, L.target_critic)):
                for k, v in mod.state_dict().items():
                    if ".fc_h." in k and args.weight_decay:
                        continue      # fc_h is in no forward pass: the reference's Adam skips it (no grad), the engine's decays it
                    d = float((v.cpu() - ref_sd[k].detach()).abs().max())
                    worst["param"] = max(worst["param"], d)
                    assert d <= ptol, (p, k, d)
    for p, pol in pols.items():                       # the heads are not parameters: byte-identical throughout
        for k, v in pol.critic_heads.state_dict().items():
            assert torch.equal(v, heads0[p][0][k]), (p, k)
        for k, v in pol.target_critic_heads.state_dict().items():
            assert torch.equal(v, heads0[p][1][k]), (p, k)
    return worst


# ---- fixtures of the unmodified reference (tests/golden/make_goldens_mlp_maddpg_md.py) ---------------------------------------------
GOLDENS_MD = ["mlp_matd3_md", "mlp_maddpg_md", "mlp_maddpg_md_ties", "mlp_maddpg_md_per_huber", "mlp_matd3_multi_md"]
TGT_SEG_ZEROED = "meta.zero_tgt_seg"       # (policy index, sub-space) whose target-actor head weights were zeroed before the first update


def golden_meta(g):
    S, B, steps, td3, per, huber = [int(v) for v in g["meta.cfg"]]
    n_pol = len(g["meta.obs"])
    specs = []
    for i in range(n_pol):
        segs = [int(v) for v in g["meta.act.policy_%d" % i]]
        specs.append((int(g["meta.obs"][i]), segs if g["meta.md"][i] else segs[0], int(g["meta.agents"][i])))
    gamma, lr, eps, mgn, tau, hd, per_eps, tstd, wd, gain = [float(v) for v in g["meta.hparams"]]
    over = dict(gamma=gamma, lr=lr, opti_eps=eps, max_grad_norm=mgn, tau=tau, huber_delta=hd, per_eps=per_eps, target_action_noise_std=tstd,
                weight_decay=wd, gain=gain, use_per=bool(per), use_huber_loss=bool(huber))
    return (specs, S, B, steps, bool(td3)), over


def zero_target_segment(tgt_sd, seg):
    """The ties fixtures' edit: sub-space `seg` of the target actor's head gets zero weights, so its logits all equal the (zero) bias."""
    k = "act.action_outs.%d.weight" % seg
    tgt_sd[k] = torch.zeros_like(tgt_sd[k])
    return tgt_sd


def init_sd(g, p, tag):
    """Initial state_dict of one network; a target network not stored is the live one (the construction's hard update)."""
    sd = golden_sd(g, "%s.init.%s." % (p, tag))
    return sd if sd or not tag.startswith("tgt_") else golden_sd(g, "%s.init.%s." % (p, tag[4:]))


def oracle_against_golden(name):
    """The oracle from the fixture's initial weights: losses 1e-6, tensors 2e-5, its own draws equal to the stored ones."""
    torch.set_num_threads(1)
    g = load_golden(name)
    (specs, S, B, steps, td3), over = golden_meta(g)
    shapes = norm_specs(specs)
    p_ids = sorted(shapes)
    learners = {}
    for p in p_ids:
        sd = lambda tag: init_sd(g, p, tag)
        segs = shapes[p][1] if isinstance(shapes[p][1], list) else None
        learners[p] = MlpMaddpgMD(sd("actor"), sd("critic"), sd("heads"), sd("tgt_actor"), sd("tgt_critic"), sd("tgt_heads"), True, td3,
                                  gamma=over["gamma"], lr=over["lr"], eps=over["opti_eps"], weight_decay=over["weight_decay"],
                                  max_grad_norm=over["max_grad_norm"], tau=over["tau"], huber=over["use_huber_loss"],
                                  huber_delta=over["huber_delta"], use_per=over["use_per"], per_eps=over["per_eps"], segs=segs)
    noise = {p: (n, a, True, td3, over["target_action_noise_std"]) for p, (o, a, n) in shapes.items()}
    for s in range(steps):
        for p in p_ids:
            torch.set_rng_state(torch.from_numpy(golden_rng_before(g, s, p, p_ids)))
            tn, an = draw_noise_multi_md(noise, p, B)
            assert np.array_equal(torch.get_rng_state().numpy(), g["s%d.%s.rng_after" % (s, p)])
            mine = [tn[q] for q in p_ids if tn[q] is not None] + [an]
            ref = golden_draws(g, s, p)
            # the reference draws one sample_gumbel per sub-space: the stored draws are the blocks, in call order
            segs_of = lambda q: shapes[q][1] if isinstance(shapes[q][1], list) else [shapes[q][1]]
            blocks = [x for q in p_ids if tn[q] is not None for x in tn[q].split(segs_of(q), -1)] + list(an.split(segs_of(p), -1))
            assert len(blocks) == len(ref), (len(blocks), len(ref))
            for a, b in zip(blocks, ref):
                assert np.array_equal(a.numpy(), b)
            assert len(mine) == (len(p_ids) if td3 else 0) + 1
            info, prio, grads = step_multi_md(learners, p, golden_batch_multi(g, s, p, p_ids), tn, an)
            assert rel_err(info["critic_loss"], g["s%d.%s.critic_loss" % (s, p)]) < 1e-6
            assert rel_err(info["actor_loss"], g["s%d.%s.actor_loss" % (s, p)]) < 1e-6
            for k in ("critic_grad_norm", "actor_grad_norm"):
                assert rel_err(info[k], g["s%d.%s.%s" % (s, p, k)]) < 1e-5, k
            if prio is not None:
                assert rel_err(prio, g["s%d.%s.prio" % (s, p)]) < 1e-5
            if s == 0:
                for net in ("critic", "actor"):
                    for k, v in grads[net].items():
                        key = "s0.%s.grad.%s.%s" % (p, net, k)
                        if key in g:
                            assert rel_err(v, g[key]) < 2e-5, key
                for tag, d in (("actor", learners[p].actor), ("critic", learners[p].critic)):
                    for k, v in d.items():
                        assert rel_err(v.detach(), golden_expected(g, "s0.%s.post.%s.%s" % (p, tag, k), p, tag)) < 2e-5, (p, tag, k)
        for p in p_ids:
            learners[p].soft_update()
    for p in p_ids:
        L = learners[p]
        for tag, d in (("actor", L.actor), ("critic", L.critic), ("tgt_actor", L.target_actor), ("tgt_critic", L.target_critic)):
            for k, v in d.items():
                key = "final.%s.%s.%s" % (p, tag, k)
                if key in g:
                    assert rel_err(v.detach(), g[key]) < 2e-5, (p, tag, k)
        for tag, d in (("heads", L.heads), ("tgt_heads", L.target_heads)):
            for k, v in d.items():
                assert np.array_equal(v.numpy(), g["final.%s.%s.%s" % (p, tag, k)])


def engine_against_golden(name, ptol_lr=5e-3):
    """The drop-in policies + trainer built under the fixture's seed, each policy stepped on its fixture batch from the stored RNG state.
    Construction bit for bit (with the `act.action_outs.i` keys); the RNG state after, losses and grad norms of every update; parameters
    after every policy's first update and every network after the last step within 5e-3 lr per update (DESIGN.md section 2); the head
    sets byte-identical."""
    from offpolicy._b200.factory import build_mlp_maddpg_multi
    torch.set_num_threads(1)          # as the fixtures were made: orthogonal_ init rounds with the thread count
    g = load_golden(name)
    (specs, S, B, steps, td3), over = golden_meta(g)
    torch.manual_seed(3)
    args, pols, tr, _ = build_mlp_maddpg_multi(specs, S, B, discrete=True, td3=td3, **over)
    p_ids = sorted(pols)
    assert np.array_equal(torch.get_rng_state().numpy(), g["construct.rng"])
    if TGT_SEG_ZEROED in g:
        i, seg = [int(v) for v in g[TGT_SEG_ZEROED]]
        pol = pols[p_ids[i]]
        pol.target_actor.load_state_dict(zero_target_segment(pol.target_actor.state_dict(), seg))
    mods = lambda pol: (("actor", pol.actor), ("critic", pol.critic), ("tgt_actor", pol.target_actor), ("tgt_critic", pol.target_critic),
                        ("heads", pol.critic_heads), ("tgt_heads", pol.target_critic_heads))
    for p in p_ids:
        for tag, mod in mods(pols[p]):
            ref = init_sd(g, p, tag)
            sd = mod.state_dict()
            assert set(sd) == set(ref), (p, tag, sorted(sd), sorted(ref))
            for k, v in sd.items():
                assert np.array_equal(v.cpu().numpy(), ref[k].numpy().reshape(v.shape)), (p, tag, k)
    tol = lambda n: ptol_lr * args.lr * n + 1e-7
    for s in range(steps):
        for p in p_ids:
            torch.set_rng_state(torch.from_numpy(golden_rng_before(g, s, p, p_ids)))
            tail0 = actor_tail_params(pols[p])
            info, prio, _ = tr.shared_train_policy_on_batch(p, golden_batch_multi(g, s, p, p_ids))
            assert np.array_equal(torch.get_rng_state().numpy(), g["s%d.%s.rng_after" % (s, p)]), (s, p)
            for k in ("critic_loss", "critic_grad_norm", "actor_loss", "actor_grad_norm"):
                assert rel_err(float(info[k]), g["s%d.%s.%s" % (s, p, k)]) < 1e-4, (s, p, k)
            assert_actor_tail_unchanged(pols[p], tail0)
            # every clipped gradient tensor the fixture records (each policy's first update), 1e-4 x max|ref| each
            key = lambda net, k: "s%d.%s.grad.%s.%s" % (s, p, net, k)
            ref = {net: {k: g[key(net, k)] for k in ours if key(net, k) in g} for net, ours in engine_grads(tr, pols[p], p).items()}
            if s == 0:
                assert ref["critic"] and ref["actor"], p
            norms = {k: g["s%d.%s.%s" % (s, p, k)] for k in ("critic_grad_norm", "actor_grad_norm")}
            grad_errors(clipped_engine_grads(tr, pols[p], norms, args.max_grad_norm, p), ref, 1e-4, "step %d %s" % (s, p))
            if prio is not None:
                assert rel_err(np.asarray(prio), g["s%d.%s.prio" % (s, p)]) < 1e-4, (s, p)
            if s == 0:
                for tag, mod in (("actor", pols[p].actor), ("critic", pols[p].critic)):
                    for k, v in mod.state_dict().items():
                        ref = golden_expected(g, "s0.%s.post.%s.%s" % (p, tag, k), p, tag)
                        assert np.abs(v.cpu().numpy() - ref).max() <= tol(1), (s, p, tag, k)
        for p in p_ids:
            pols[p].soft_target_updates()
    for p in p_ids:
        for tag, mod in mods(pols[p])[:4]:
            for k, v in mod.state_dict().items():
                key = "final.%s.%s.%s" % (p, tag, k)
                if key in g:
                    assert np.abs(v.cpu().numpy() - g[key]).max() <= tol(steps), (p, tag, k)
        for tag, mod in mods(pols[p])[4:]:
            for k, v in mod.state_dict().items():
                assert np.array_equal(v.cpu().numpy(), g["final.%s.%s.%s" % (p, tag, k)].reshape(v.shape)), (p, tag, k)
