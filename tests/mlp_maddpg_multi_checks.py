"""Shared checks of the transition-level MADDPG / MATD3 with several policies (share_policy off): synthetic multi-policy batches, the
lock-step comparison against oracle/maddpg_mlp_multi.py and the runner for the fixtures of make_goldens_mlp_maddpg_multi.py.  The
emulated tests and the GPU tests run the same checks at different sizes."""
import numpy as np
import torch

from helpers import load_golden, rel_err
from mlp_maddpg_checks import assert_actor_tail_unchanged, actor_tail_params, clipped_engine_grads, engine_grads, grad_errors, oracle_from

from oracle.maddpg_mlp import MlpMaddpg
from oracle.maddpg_mlp_multi import draw_noise_multi, step_multi

FIELDS = ("obs", "share_obs", "acts", "rewards", "next_obs", "next_share_obs", "dones", "dones_env", "valid_transition", "avail_acts",
          "next_avail_acts")


def norm_specs(specs):
    """(obs_dim, act_dim[, n_agents]) per policy -> {policy_i: (obs_dim, act_dim, n_agents)}."""
    return {"policy_%d" % i: tuple(int(v) for v in s) + (1,) * (3 - len(s)) for i, s in enumerate(specs)}


def synth_batch_multi(rng, specs, B, S, discrete, avail=False, ties=False, per=False):
    """A sample of several policies' stores in the reference's layout (mlp_buffer.py:80-110): the 13-tuple of {policy_id: array}.
    The stores hold the same transitions, so the shared observation and dones_env are one array for every policy."""
    f = lambda *s: rng.standard_normal(s).astype(np.float32)
    share, nshare = f(B, S), f(B, S)
    dones_env = (rng.random((B, 1)) < 0.1).astype(np.float32)
    out = [dict() for _ in range(11)]
    for p, (O, A, N) in norm_specs(specs).items():
        acts = np.eye(A, dtype=np.float32)[rng.integers(0, A, (N, B))] if discrete else np.tanh(f(N, B, A))
        av = nav = None
        if avail:
            av = (rng.random((N, B, A)) < 0.7).astype(np.float32)
            nav = (rng.random((N, B, A)) < 0.7).astype(np.float32)
            av[..., 0] = nav[..., 0] = 1.0
            if ties:      # every action but the first masked: -1e10 ties -> onehot_from_logits is multi-hot on those rows
                nav[:, : B // 4] = 0.0
                nav[:, : B // 8, 0] = 1.0
        valid = (rng.random((N, B, 1)) < 0.8).astype(np.float32)
        valid[:, 0] = 1.0
        vals = (f(N, B, O), share, acts, f(N, B, 1), f(N, B, O), nshare, (rng.random((N, B, 1)) < 0.1).astype(np.float32), dones_env,
                valid, av, nav)
        for d, v in zip(out, vals):
            d[p] = v
    w = (0.2 + rng.random(B)).astype(np.float32) if per else None
    return tuple(out) + (w, np.arange(B) if per else None)


def noise_shapes(tr):
    """{policy_id: (n_agents, act_dim, discrete, td3, target_std)} of a trainer, for draw_noise_multi."""
    return {p: (e.n_agents, e.pol.act_dim, e.pol.discrete, e.pol.td3, e.pol.target_noise) for p, e in tr._eng.items()}


def check_params(pols, learners, ptol, skip_fc_h=False):
    worst = 0.0
    for p, pol in pols.items():
        L = learners[p]
        for mod, ref_sd in ((pol.actor, L.actor), (pol.critic, L.critic), (pol.target_actor, L.target_actor), (pol.target_critic, L.target_critic)):
            for k, v in mod.state_dict().items():
                if skip_fc_h and ".fc_h." in k:
                    continue
                d = float((v.cpu() - ref_sd[k].detach()).abs().max())
                worst = max(worst, d)
                assert d <= ptol, (p, k, d)
    return worst


def lockstep_multi(args, pols, tr, batches, rtol=1e-4, ptol=2e-5):
    """Engine and oracle step through `batches`: per batch, every policy in id order (the runner's batch_train, base_runner.py:187-217),
    then the soft target updates of all policies.  The engine's draws are replayed from the same RNG state for the oracle."""
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
            tn, an = draw_noise_multi(shapes, p, B)
            assert torch.equal(torch.get_rng_state(), rng_after), p
            ref, rprio, grads = step_multi(learners, p, batch, tn, an)
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
        worst["param"] = max(worst["param"], check_params(pols, learners, ptol, skip_fc_h=bool(args.weight_decay)))
    for p, pol in pols.items():                       # the heads are not parameters: byte-identical throughout
        for k, v in pol.critic_heads.state_dict().items():
            assert torch.equal(v, heads0[p][0][k]), (p, k)
        for k, v in pol.target_critic_heads.state_dict().items():
            assert torch.equal(v, heads0[p][1][k]), (p, k)
    return worst


# ---- fixtures of the unmodified reference (tests/golden/make_goldens_mlp_maddpg_multi.py) ------------------------------------------
GOLDENS_MULTI = ["mlp_maddpg_multi_disc", "mlp_matd3_multi_disc", "mlp_matd3_multi_box", "mlp_maddpg_multi_per_huber"]


def golden_meta_multi(g):
    S, B, steps, td3, discrete, per, huber = [int(v) for v in g["meta.cfg"]]
    specs = [tuple(int(v) for v in row) for row in g["meta.specs"]]
    gamma, lr, eps, mgn, tau, hd, per_eps, tstd, wd, gain = [float(v) for v in g["meta.hparams"]]
    over = dict(gamma=gamma, lr=lr, opti_eps=eps, max_grad_norm=mgn, tau=tau, huber_delta=hd, per_eps=per_eps, target_action_noise_std=tstd,
                weight_decay=wd, gain=gain, use_per=bool(per), use_huber_loss=bool(huber))
    return (specs, S, B, steps, bool(td3), bool(discrete)), over


def golden_batch_multi(g, s, p, p_ids):
    f = lambda k: {q: g.get("s%d.%s.in.%s.%s" % (s, p, q, k)) for q in p_ids}
    w = g.get("s%d.%s.in.weights" % (s, p))
    return tuple(f(k) for k in FIELDS) + (w, None if w is None else np.arange(len(w)))


def golden_sd(g, prefix):
    return {k[len(prefix):]: torch.from_numpy(v) for k, v in g.items() if k.startswith(prefix)}


def golden_draws(g, s, p):
    pre = "s%d.%s.draw" % (s, p)
    return [g[k] for k in sorted((k for k in g if k.startswith(pre)), key=lambda k: int(k[len(pre):]))]


def golden_rng_before(g, s, p, p_ids):
    """The torch RNG state before update (s, p): the previous update's state after it, or the construction state (nothing draws in
    between; make_goldens_mlp_maddpg_multi.py asserts it)."""
    i = s * len(p_ids) + p_ids.index(p)
    if i == 0:
        return g["construct.rng"]
    ps, pp = divmod(i - 1, len(p_ids))
    return g["s%d.%s.rng_after" % (ps, p_ids[pp])]


def golden_expected(g, key, p, tag):
    """A stored network value; the `fc_h` block (in no forward pass, not stored after construction) is expected at its initial value,
    the live copy exactly and the target copy up to the round-off of the soft updates."""
    if key in g:
        return g[key]
    k = key.split(".%s." % tag, 1)[1]
    assert ".fc_h." in k, key
    return g["%s.init.%s.%s" % (p, tag.replace("tgt_", ""), k)]


def _init_sd(g, p, tag):
    """Initial state_dict of one network; the target trunks were the live ones at construction (stored once)."""
    return golden_sd(g, "%s.init.%s." % (p, tag.replace("tgt_", "") if tag in ("tgt_actor", "tgt_critic") else tag))


def oracle_against_golden(name):
    """The oracle from the fixture's initial weights: losses 1e-6, tensors 2e-5, its own draws equal to the stored ones."""
    torch.set_num_threads(1)
    g = load_golden(name)
    (specs, S, B, steps, td3, discrete), over = golden_meta_multi(g)
    p_ids = sorted(norm_specs(specs))
    learners = {}
    for p in p_ids:
        sd = lambda tag: _init_sd(g, p, tag)
        learners[p] = MlpMaddpg(sd("actor"), sd("critic"), sd("heads"), sd("tgt_actor"), sd("tgt_critic"), sd("tgt_heads"), discrete, td3,
                                gamma=over["gamma"], lr=over["lr"], eps=over["opti_eps"], weight_decay=over["weight_decay"],
                                max_grad_norm=over["max_grad_norm"], tau=over["tau"], huber=over["use_huber_loss"],
                                huber_delta=over["huber_delta"], use_per=over["use_per"], per_eps=over["per_eps"])
    shapes = {p: (n, a, discrete, td3, over["target_action_noise_std"]) for p, (o, a, n) in norm_specs(specs).items()}
    for s in range(steps):
        for p in p_ids:
            torch.set_rng_state(torch.from_numpy(golden_rng_before(g, s, p, p_ids)))
            tn, an = draw_noise_multi(shapes, p, B)
            assert np.array_equal(torch.get_rng_state().numpy(), g["s%d.%s.rng_after" % (s, p)])
            mine = [tn[q] for q in p_ids if tn[q] is not None] + ([an] if an is not None else [])
            ref = golden_draws(g, s, p)
            assert len(mine) == len(ref)
            for a, b in zip(mine, ref):
                assert np.array_equal(a.numpy(), b)
            info, prio, grads = step_multi(learners, p, golden_batch_multi(g, s, p, p_ids), tn, an)
            assert rel_err(info["critic_loss"], g["s%d.%s.critic_loss" % (s, p)]) < 1e-6
            assert rel_err(info["actor_loss"], g["s%d.%s.actor_loss" % (s, p)]) < 1e-6
            for k in ("critic_grad_norm", "actor_grad_norm"):
                assert rel_err(info[k], g["s%d.%s.%s" % (s, p, k)]) < 1e-5, k
            if prio is not None:
                assert rel_err(prio, g["s%d.%s.prio" % (s, p)]) < 1e-5
            if s == 0:                                # gradients and post-Adam parameters of every policy's first update
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
    for p in p_ids:                                   # every network and head set after the last step's soft updates
        L = learners[p]
        for tag, d in (("actor", L.actor), ("critic", L.critic), ("tgt_actor", L.target_actor), ("tgt_critic", L.target_critic)):
            for k, v in d.items():
                assert rel_err(v.detach(), golden_expected(g, "final.%s.%s.%s" % (p, tag, k), p, tag)) < 2e-5, (p, tag, k)
        for tag, d in (("heads", L.heads), ("tgt_heads", L.target_heads)):
            for k, v in d.items():
                assert np.array_equal(v.numpy(), g["final.%s.%s.%s" % (p, tag, k)])


def engine_against_golden(name, ptol_lr=5e-3):
    """The drop-in policies + trainer built under the fixture's seed, each policy stepped on its fixture batch from the stored RNG state.
    Construction bit for bit; the RNG state after, losses and grad norms of every update; parameters after every policy's first update
    and every network after the last step within 5e-3 lr per update (DESIGN.md section 2); the head sets byte-identical."""
    from offpolicy._b200.factory import build_mlp_maddpg_multi
    torch.set_num_threads(1)          # as the fixtures were made: orthogonal_ init rounds with the thread count
    g = load_golden(name)
    (specs, S, B, steps, td3, discrete), over = golden_meta_multi(g)
    torch.manual_seed(3)
    args, pols, tr, _ = build_mlp_maddpg_multi(specs, S, B, discrete=discrete, td3=td3, **over)
    p_ids = sorted(pols)
    assert np.array_equal(torch.get_rng_state().numpy(), g["construct.rng"])
    mods = lambda pol: (("actor", pol.actor), ("critic", pol.critic), ("tgt_actor", pol.target_actor), ("tgt_critic", pol.target_critic),
                        ("heads", pol.critic_heads), ("tgt_heads", pol.target_critic_heads))
    for p in p_ids:
        for tag, mod in mods(pols[p]):
            ref = _init_sd(g, p, tag)
            sd = mod.state_dict()
            assert set(sd) == set(ref), (p, tag)
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
                ref = golden_expected(g, "final.%s.%s.%s" % (p, tag, k), p, tag)
                assert np.abs(v.cpu().numpy() - ref).max() <= tol(steps), (p, tag, k)
        for tag, mod in mods(pols[p])[4:]:
            for k, v in mod.state_dict().items():
                assert np.array_equal(v.cpu().numpy(), g["final.%s.%s.%s" % (p, tag, k)].reshape(v.shape)), (p, tag, k)
