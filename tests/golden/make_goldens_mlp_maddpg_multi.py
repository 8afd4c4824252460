"""Generate tests/golden/mlp_{maddpg,matd3}_multi_*.npz by running the UNMODIFIED reference's transition-level MADDPG / MATD3 with one
policy per agent (share_policy off; offpolicy/algorithms/{maddpg,matd3}) in the build container:

    python tests/golden/make_goldens_mlp_maddpg_multi.py

The update loop is the MLP runner's batch_train (runner/mlp/base_runner.py:187-217): at each step, every policy in id order trains on
its own sample (all policies' stores hold the same transitions), then every policy's targets are soft-updated.

A fixture stores the torch RNG state after construction, every policy's initial weights and both head sets.  Per update it stores the
inputs, the noise draws the reference made (in call order), train_info, the priorities and the torch RNG state after the update (the
state before it is the previous update's, or the construction state: nothing else draws in between, which is asserted here).  The
clipped gradients and the post-Adam parameters are stored for the first update of every policy, and every network and head set after
the last step's soft updates.  So that a fixture stays small, values that equal stored ones are not repeated, and each equality is
asserted here: the target trunks at construction (a copy of the live ones), and the `fc_h` block, which no forward pass uses (layer_N
= 1), so it keeps its initial values (the targets' copy up to the round-off of the soft updates, FC_H_POLYAK_TOL).  The single-policy fixtures come from make_goldens_mlp_maddpg.py.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [HERE, os.path.join(ROOT, "tests"), ROOT]

import ref_harness as rh  # noqa: E402
from make_goldens_mlp_maddpg import FIELDS, heads_np, sd_np  # noqa: E402
from mlp_maddpg_multi_checks import norm_specs, synth_batch_multi  # noqa: E402

SPEAKER_LISTENER = [(3, 3), (11, 5)]          # simple_speaker_listener: speaker obs 3, Discrete(3); listener obs 11, Discrete(5)
SPEAKER_LISTENER_S = 14
FC_H_POLYAK_TOL = 1e-6          # |target fc_h - initial fc_h| after the soft updates: fp32 round-off of (1 - tau) x + tau x


def gen_multi(name, td3, discrete, specs, S, flags=(), B=16, steps=3, per=False, seed=41):
    rh.import_reference()
    sp = rh.gym_spaces()
    import offpolicy.utils.util as util
    import offpolicy.algorithms.maddpg.algorithm.MADDPGPolicy as polmod
    args = rh.make_args(["--algorithm_name", "matd3" if td3 else "maddpg"] + list(flags))
    if td3:
        from offpolicy.algorithms.matd3.algorithm.MATD3Policy import MATD3Policy as Policy
        from offpolicy.algorithms.matd3.matd3 import MATD3 as Trainer
    else:
        from offpolicy.algorithms.maddpg.algorithm.MADDPGPolicy import MADDPGPolicy as Policy
        from offpolicy.algorithms.maddpg.maddpg import MADDPG as Trainer
    shapes = norm_specs(specs)
    p_ids = sorted(shapes)
    total = sum(a * n for _, a, n in shapes.values())
    dev = torch.device("cpu")
    torch.manual_seed(3)
    pols, mapping, nxt = {}, {}, 0
    for p in p_ids:                                       # train_mpe.py:139-150: the policies in id order
        O, A, N = shapes[p]
        info = dict(obs_space=sp.Box(-np.inf, np.inf, (O,)), share_obs_space=sp.Box(-np.inf, np.inf, (S,)),
                    act_space=sp.Discrete(A) if discrete else sp.Box(-1.0, 1.0, (A,)), cent_obs_dim=S, cent_act_dim=total)
        pols[p] = Policy({"args": args, "device": dev}, info)
        mapping.update({k: p for k in range(nxt, nxt + N)})
        nxt += N
    out = {"construct.rng": torch.get_rng_state().numpy().copy()}
    tr = Trainer(args, nxt, pols, lambda a: mapping[a], device=dev)
    for p, pol in pols.items():
        for live, tgt in ((pol.actor, pol.target_actor), (pol.critic, pol.target_critic)):
            for k, v in live.state_dict().items():
                assert torch.equal(v, tgt.state_dict()[k]), (p, k)          # the construction's hard update: stored once
        out.update(sd_np("%s.init.actor." % p, pol.actor))
        out.update(sd_np("%s.init.critic." % p, pol.critic))
        out.update(heads_np("%s.init.heads." % p, pol.critic))
        out.update(heads_np("%s.init.tgt_heads." % p, pol.target_critic))
    trunk = lambda prefix, mod: {k: v for k, v in sd_np(prefix, mod).items() if ".fc_h." not in k}

    draws = []
    real_gumbel, real_gauss = util.sample_gumbel, polmod.gaussian_noise

    def gumbel(*a, **k):
        g = real_gumbel(*a, **k)
        draws.append(g.detach().numpy().copy())
        return g

    def gauss(*a, **k):
        g = real_gauss(*a, **k)
        draws.append(g.detach().numpy().copy())
        return g
    util.sample_gumbel, polmod.gaussian_noise = gumbel, gauss
    grads = {}
    for pol in pols.values():
        for tag, opt, mod in (("critic", pol.critic_optimizer, pol.critic), ("actor", pol.actor_optimizer, pol.actor)):
            step = opt.step

            def recording_step(*a, _step=step, _tag=tag, _mod=mod, **k):
                for n, prm in _mod.named_parameters():
                    if prm.grad is not None:
                        grads["%s.%s" % (_tag, n)] = prm.grad.detach().numpy().copy()
                return _step(*a, **k)
            opt.step = recording_step
    rng = np.random.default_rng(seed)
    rng_state = torch.get_rng_state().clone()
    try:
        for s in range(steps):
            for p in p_ids:
                b = synth_batch_multi(rng, specs, B, S, discrete, per=per)
                for f, v in zip(FIELDS, b[:11]):
                    for q in p_ids:
                        if v[q] is not None:
                            out["s%d.%s.in.%s.%s" % (s, p, q, f)] = v[q]
                if per:
                    out["s%d.%s.in.weights" % (s, p)] = b[11]
                draws.clear()
                grads.clear()
                assert torch.equal(torch.get_rng_state(), rng_state)          # the RNG state before = the one last stored
                info_t, prio, _ = tr.shared_train_policy_on_batch(p, b)
                rng_state = torch.get_rng_state().clone()
                out["s%d.%s.rng_after" % (s, p)] = rng_state.numpy().copy()
                for i, d in enumerate(draws):
                    out["s%d.%s.draw%d" % (s, p, i)] = d
                for k in ("critic_loss", "critic_grad_norm", "actor_loss", "actor_grad_norm"):
                    out["s%d.%s.%s" % (s, p, k)] = np.asarray(float(info_t[k]), np.float64)
                assert info_t["update_actor"]
                if prio is not None:
                    out["s%d.%s.prio" % (s, p)] = np.asarray(prio, np.float32)
                if s == 0:                                # the first update of every policy: gradients and post-Adam parameters
                    for k, v in grads.items():
                        out["s0.%s.grad.%s" % (p, k)] = v
                    for tag, mod in (("actor", pols[p].actor), ("critic", pols[p].critic)):
                        out.update(trunk("s0.%s.post.%s." % (p, tag), mod))
            for p in p_ids:                               # base_runner.py:209-211
                pols[p].soft_target_updates()
        for p, pol in pols.items():                       # every network after the last step's soft updates
            for tag, mod in (("actor", pol.actor), ("critic", pol.critic), ("tgt_actor", pol.target_actor), ("tgt_critic", pol.target_critic)):
                out.update(trunk("final.%s.%s." % (p, tag), mod))
                init = "%s.init.%s." % (p, tag.replace("tgt_", ""))
                for k, v in mod.state_dict().items():
                    if ".fc_h." in k:     # in no forward pass: no gradient, no Adam step; Polyak of equal values moves it by round-off only
                        d = np.abs(v.detach().numpy() - out[init + k]).max()
                        assert d <= (FC_H_POLYAK_TOL if tag.startswith("tgt_") else 0.0), (p, tag, k, d)
            out.update(heads_np("final.%s.heads." % p, pol.critic))
            out.update(heads_np("final.%s.tgt_heads." % p, pol.target_critic))
    finally:
        util.sample_gumbel, polmod.gaussian_noise = real_gumbel, real_gauss
    out["meta.cfg"] = np.array([S, B, steps, int(td3), int(discrete), int(per), int(args.use_huber_loss)])
    out["meta.specs"] = np.array([shapes[p] for p in p_ids], dtype=np.int64)
    out["meta.hparams"] = np.array([args.gamma, args.lr, args.opti_eps, args.max_grad_norm, args.tau, args.huber_delta, args.per_eps,
                                    float(args.target_action_noise_std), args.weight_decay, args.gain], dtype=np.float64)
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, **out)
    print(name, "->", path, "%.1f KB" % (os.path.getsize(path) / 1024), "critic_loss", float(out["s0.policy_0.critic_loss"]))


if __name__ == "__main__":
    torch.set_num_threads(1)          # orthogonal_ (a QR) rounds differently with the thread count: the tests replay it on one thread
    gen_multi("mlp_maddpg_multi_disc", False, True, SPEAKER_LISTENER, SPEAKER_LISTENER_S)
    gen_multi("mlp_matd3_multi_disc", True, True, SPEAKER_LISTENER, SPEAKER_LISTENER_S)
    # three policies with different observation and Box action widths (a smaller batch keeps the fixture small)
    gen_multi("mlp_matd3_multi_box", True, False, [(6, 2), (9, 3), (4, 1)], 19, B=8)
    gen_multi("mlp_maddpg_multi_per_huber", False, True, SPEAKER_LISTENER, SPEAKER_LISTENER_S,
              flags=["--use_per", "--use_huber_loss", "--huber_delta", "1.0"], per=True, seed=43)
