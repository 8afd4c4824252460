"""Shared checks of the transition-level MADDPG / MATD3 learner (algorithms/maddpg, csrc/maddpg.cu cfg.mlp) against
oracle/maddpg_mlp.py: the emulated tests and the GPU tests run the same lock-step comparison at different sizes."""
import numpy as np
import torch

from helpers import load_golden, rel_err
from maddpg_checks import named_views

from oracle.maddpg_mlp import MlpMaddpg


def synth_batch(rng, N, B, O, S, A, discrete, avail=False, ties=False, per=False):
    """A batch in the reference's sample layout (mlp_buffer.py:80-110): the 13-tuple of {policy_0: array} entries."""
    f = lambda *s: rng.standard_normal(s).astype(np.float32)
    if discrete:
        acts = np.eye(A, dtype=np.float32)[rng.integers(0, A, (N, B))]
    else:
        acts = np.tanh(f(N, B, A))
    av = nav = None
    if avail:
        av = (rng.random((N, B, A)) < 0.7).astype(np.float32)
        nav = (rng.random((N, B, A)) < 0.7).astype(np.float32)
        av[..., 0] = nav[..., 0] = 1.0
        if ties:          # every action but the first masked: -1e10 ties -> onehot_from_logits is multi-hot on those rows
            nav[:, : B // 4] = 0.0
            nav[:, : B // 8, 0] = 1.0
    share = f(B, S)
    valid = (rng.random((N, B, 1)) < 0.8).astype(np.float32)
    valid[:, 0] = 1.0
    w = (0.2 + rng.random(B)).astype(np.float32) if per else None
    d = lambda: {"policy_0": None}
    pd = lambda x: {"policy_0": x}
    return (pd(f(N, B, O)), pd(share), pd(acts), pd(f(N, B, 1)), pd(f(N, B, O)), pd(f(B, S)),
            pd((rng.random((N, B, 1)) < 0.1).astype(np.float32)), pd((rng.random((B, 1)) < 0.1).astype(np.float32)), pd(valid),
            pd(av) if avail else d(), pd(nav) if avail else d(), w, np.arange(B) if per else None)


def oracle_from(args, pol):
    cpu = lambda m: {k: v.cpu() for k, v in m.state_dict().items()}
    return MlpMaddpg(cpu(pol.actor), cpu(pol.critic), cpu(pol.critic_heads), cpu(pol.target_actor), cpu(pol.target_critic),
                     cpu(pol.target_critic_heads), pol.discrete, pol.td3, gamma=args.gamma, lr=args.lr, eps=args.opti_eps,
                     weight_decay=args.weight_decay, max_grad_norm=args.max_grad_norm, tau=args.tau, huber=args.use_huber_loss,
                     huber_delta=args.huber_delta, use_per=args.use_per, per_eps=args.per_eps, relu=bool(args.use_ReLU),
                     feature_norm=bool(args.use_feature_normalization))


def actor_tail(pol):
    """First float of the actor vector past its trained range: the learner's net layout (qmix.cu mx_net_layout) puts the head in the
    weight_ih slot (bias at bias_ih), then bias_hh, then the output LayerNorm, which optimise() takes as the end of the actor's range."""
    bih = min(off for name, off, _, _ in pol._a_entries if name.startswith("act.") and name.endswith(".bias"))
    return bih + 2 * 3 * 64


def engine_grads(tr, pol, p_id=None):
    """The engine's unclipped gradients of its last step, {"critic": {key: tensor}, "actor": {key: tensor}} in float64: numerator over
    denominator.  The critic's range stops at its weight_ih slot (the frozen heads sit there), so its four scalars are at the first head's
    offset; the actor's are at Pa, and every float of its vector past the trained range carries an exactly zero gradient."""
    ga, gc = (v.detach().cpu().double() for v in tr.grad_views(p_id))
    c_den = float(gc[pol._h_entries[0][1]])
    a_den = float(ga[pol.Pa])
    tail = ga[actor_tail(pol):pol.Pa]
    assert int((tail != 0).sum()) == 0, ("actor gradient past its trained range", int((tail != 0).sum()))
    return {"critic": {k: v / c_den for k, v in named_views(gc, pol._c_entries).items()},
            "actor": {k: v / a_den for k, v in named_views(ga, pol._a_entries).items()}}


def clipped_engine_grads(tr, pol, ref_info, max_grad_norm, p_id=None):
    """engine_grads scaled by torch.nn.utils.clip_grad_norm_'s factor at the reference's grad norms: comparable with the oracle's
    (clipped) gradients and the fixtures'."""
    coef = lambda k: min(1.0, max_grad_norm / (float(ref_info[k]) + 1e-6))
    g = engine_grads(tr, pol, p_id)
    return {net: {k: v * coef(net + "_grad_norm") for k, v in d.items()} for net, d in g.items()}


def actor_tail_params(pol):
    """The actor's floats past its trained range (live, target, Adam m, v): no update may touch them."""
    t = actor_tail(pol)
    return [v[t:].clone() for v in pol.actor_vecs]


def assert_actor_tail_unchanged(pol, before):
    for i, (v, v0) in enumerate(zip(pol.actor_vecs, before)):
        assert torch.equal(v[actor_tail(pol):], v0), ("actor vector %d changed past the trained range" % i)


def grad_errors(ours, ref, rtol=1e-4, tag=""):
    """{net.key: max |ours - ref| / max |ref|} over every tensor of `ref` ({net: {key: tensor}}); raises listing every tensor beyond
    rtol x max|ref| (a tensor whose reference is zero must be exactly zero)."""
    errs, bad = {}, []
    for net, d in ref.items():
        for k, r in d.items():
            r = torch.as_tensor(r).double().reshape(ours[net][k].shape)
            diff, scale = float((ours[net][k] - r).abs().max()), float(r.abs().max())
            errs[net + "." + k] = diff / scale if scale > 0 else (0.0 if diff == 0.0 else float("inf"))
            if diff > rtol * scale:
                bad.append("%s %s.%s: err %.3e > %.1e x max|ref| %.3e" % (tag, net, k, diff, rtol, scale))
    assert not bad, "\n".join(bad)
    return errs


def lockstep(args, pol, tr, batches, rtol=1e-4, ptol=2e-5, soft=True):
    """Engine and oracle step through `batches` (soft target update after each); returns the max deviations seen."""
    L = oracle_from(args, pol)
    heads0 = {k: v.clone() for k, v in pol.critic_heads.state_dict().items()}
    theads0 = {k: v.clone() for k, v in pol.target_critic_heads.state_dict().items()}
    worst = {"info": 0.0, "param": 0.0, "prio": 0.0, "grad": 0.0}
    for s, batch in enumerate(batches):
        B = np.asarray(batch[0]["policy_0"]).shape[1]
        tail0 = actor_tail_params(pol)
        rng_before = torch.get_rng_state()
        info, prio, _ = tr.shared_train_policy_on_batch("policy_0", batch)
        rng_after = torch.get_rng_state()
        torch.set_rng_state(rng_before)
        tn, an = tr.draw_target_noise(B), tr.draw_actor_noise(B)          # the same calls, the same draws
        assert torch.equal(torch.get_rng_state(), rng_after)
        ref, rprio, grads = L.step(batch, tn, an)
        assert info["update_actor"] is True
        errs = grad_errors(clipped_engine_grads(tr, pol, ref, args.max_grad_norm), grads, rtol, "step %d" % s)
        worst["grad"] = max([worst["grad"]] + list(errs.values()))
        for k, v in ref.items():
            d = abs(float(info[k]) - v) / max(1.0, abs(v))
            worst["info"] = max(worst["info"], d)
            assert d <= rtol, (k, float(info[k]), v)
        if rprio is not None:
            p = np.asarray(prio)
            d = float(np.max(np.abs(p - rprio) / np.maximum(1.0, np.abs(rprio))))
            worst["prio"] = max(worst["prio"], d)
            assert d <= rtol, d
        if soft:
            pol.soft_target_updates()
            L.soft_update()
        for mod, ref_sd in ((pol.actor, L.actor), (pol.critic, L.critic), (pol.target_actor, L.target_actor), (pol.target_critic, L.target_critic)):
            for k, v in mod.state_dict().items():
                if ".fc_h." in k and args.weight_decay:
                    continue      # fc_h is in no forward pass: the reference's Adam skips it (no grad), the engine's decays it
                d = float((v.cpu() - ref_sd[k].detach()).abs().max())
                worst["param"] = max(worst["param"], d)
                assert d <= ptol, (k, d)
        assert_actor_tail_unchanged(pol, tail0)
    # the heads are not parameters: byte-identical after every update and target update
    for k, v in pol.critic_heads.state_dict().items():
        assert torch.equal(v, heads0[k]), k
    for k, v in pol.target_critic_heads.state_dict().items():
        assert torch.equal(v, theads0[k]), k
    return worst


# ---- fixtures of the unmodified reference (tests/golden/make_goldens_mlp_maddpg.py) --------------------------------------------------
GOLDENS = ["mlp_maddpg_disc", "mlp_matd3_disc", "mlp_maddpg_box", "mlp_matd3_box", "mlp_maddpg_disc_avail", "mlp_maddpg_per_huber"]
_FIELDS = ("obs", "share_obs", "acts", "rewards", "next_obs", "next_share_obs", "dones", "dones_env", "valid_transition", "avail_acts",
           "next_avail_acts")


def golden_meta(g):
    N, O, A, S, B, steps, td3, discrete, per, huber = [int(v) for v in g["meta.cfg"]]
    gamma, lr, eps, mgn, tau, hd, per_eps, tstd, wd, gain = [float(v) for v in g["meta.hparams"]]
    over = dict(gamma=gamma, lr=lr, opti_eps=eps, max_grad_norm=mgn, tau=tau, huber_delta=hd, per_eps=per_eps, target_action_noise_std=tstd,
                weight_decay=wd, gain=gain, use_per=bool(per), use_huber_loss=bool(huber))
    return (N, O, A, S, B, steps, bool(td3), bool(discrete)), over


def golden_batch(g, s):
    f = lambda k: {"policy_0": g.get("s%d.in.%s" % (s, k))}
    w = g.get("s%d.in.weights" % s)
    return tuple(f(k) for k in _FIELDS) + (w, None if w is None else np.arange(len(w)))


def golden_sd(g, prefix):
    return {k[len(prefix):]: torch.from_numpy(v) for k, v in g.items() if k.startswith(prefix)}


def golden_draws(g, s):
    return [g[k] for k in sorted((k for k in g if k.startswith("s%d.draw" % s)), key=lambda k: int(k.split("draw")[1]))]


def engine_against_golden(name, ptol_lr=5e-3):
    """The drop-in policy + trainer built under the golden's seed, stepped on the golden batches from the golden RNG states."""
    from offpolicy._b200.factory import build_mlp_maddpg
    torch.set_num_threads(1)          # as the fixtures were made: orthogonal_ init rounds with the thread count
    g = load_golden(name)
    (N, O, A, S, B, steps, td3, discrete), over = golden_meta(g)
    torch.manual_seed(3)
    args, pol, tr = build_mlp_maddpg(N, O, A, S, B, discrete=discrete, td3=td3, **over)
    # construction: the reference's order and generator consumption, bit for bit
    assert np.array_equal(torch.get_rng_state().numpy(), g["construct.rng"])
    for tag, mod in (("actor", pol.actor), ("critic", pol.critic), ("tgt_actor", pol.target_actor), ("tgt_critic", pol.target_critic),
                     ("heads", pol.critic_heads), ("tgt_heads", pol.target_critic_heads)):
        sd = mod.state_dict()
        assert set(sd) == {k[len("init.%s." % tag):] for k in g if k.startswith("init.%s." % tag)}, tag
        for k, v in sd.items():
            assert np.array_equal(v.cpu().numpy(), g["init.%s.%s" % (tag, k)].reshape(v.shape)), (tag, k)
    for s in range(steps):
        torch.set_rng_state(torch.from_numpy(g["s%d.rng_before" % s]))
        tail0 = actor_tail_params(pol)
        info, prio, _ = tr.shared_train_policy_on_batch("policy_0", golden_batch(g, s))
        assert np.array_equal(torch.get_rng_state().numpy(), g["s%d.rng_after" % s])
        for k in ("critic_loss", "critic_grad_norm", "actor_loss", "actor_grad_norm"):
            assert rel_err(float(info[k]), g["s%d.%s" % (s, k)]) < 1e-4, (s, k)
        assert_actor_tail_unchanged(pol, tail0)
        # every clipped gradient tensor the fixture records, 1e-4 x max|ref| each
        ref = {net: {k: g["s%d.grad.%s.%s" % (s, net, k)] for k in ours if "s%d.grad.%s.%s" % (s, net, k) in g}
               for net, ours in engine_grads(tr, pol).items()}
        assert ref["critic"] and ref["actor"], s
        grad_errors(clipped_engine_grads(tr, pol, {k: g["s%d.%s" % (s, k)] for k in ("critic_grad_norm", "actor_grad_norm")},
                                         args.max_grad_norm), ref, 1e-4, "step %d" % s)
        if prio is not None:
            assert rel_err(np.asarray(prio), g["s%d.prio" % s]) < 1e-4
        for tag, mod in (("actor", pol.actor), ("critic", pol.critic)):
            for k, v in mod.state_dict().items():
                ref_new = g["s%d.post.%s.%s" % (s, tag, k)]
                # the update within 5e-3 lr per element per step (DESIGN.md section 2)
                assert np.abs(v.cpu().numpy() - ref_new).max() <= ptol_lr * args.lr * (s + 1) + 1e-7, (s, tag, k)
        pol.soft_target_updates()
        for tag, mod in (("tgt_actor", pol.target_actor), ("tgt_critic", pol.target_critic)):
            for k, v in mod.state_dict().items():
                assert np.abs(v.cpu().numpy() - g["s%d.post.%s.%s" % (s, tag, k)]).max() <= ptol_lr * args.lr * (s + 1) + 1e-7, (s, tag, k)
        for tag, mod in (("heads", pol.critic_heads), ("tgt_heads", pol.target_critic_heads)):
            for k, v in mod.state_dict().items():
                assert np.array_equal(v.cpu().numpy(), g["s%d.post.%s.%s" % (s, tag, k)].reshape(v.shape)), (s, tag, k)
