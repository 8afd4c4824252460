"""Generate tests/golden/mlp_{maddpg,matd3}_*md*.npz by running the UNMODIFIED reference's transition-level MADDPG / MATD3
(offpolicy/algorithms/{maddpg,matd3}) with MultiDiscrete action spaces (offpolicy/envs/mpe/multi_discrete.py) in the build container:

    python tests/golden/make_goldens_mlp_maddpg_md.py

The shapes are simple_reference's (scripts/train_mpe_matd3.sh): 2 agents, obs 21, shared obs 42, MultiDiscrete([[0,4],[0,9]]).  The
update loop is the MLP runner's batch_train (runner/mlp/base_runner.py:187-217), as in make_goldens_mlp_maddpg_multi.py: at each step,
every policy in id order trains on its own sample, then every policy's targets are soft-updated.  With one shared policy this is the
runner's loop too.

A fixture stores the torch RNG state after construction and every policy's initial networks and both head sets; an initial target
network is stored only where it is not a copy of the live one (the ties fixture's edit).  Per
update it stores the inputs, the noise draws the reference made (one per sample_gumbel call, so one per sub-space, in call order),
train_info, the priorities and the torch RNG state after the update (the state before it is the previous update's, or the construction
state; asserted here).  The clipped gradients and the post-Adam parameters are stored for the first update of every policy, and every
network and head set after the last step's soft updates.  The `fc_h` block, which no forward pass uses, is stored at construction only
(its later values are asserted here, as in make_goldens_mlp_maddpg_multi.py).
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
from make_goldens_mlp_maddpg_multi import FC_H_POLYAK_TOL  # noqa: E402
from mlp_maddpg_md_checks import REFERENCE_SPEC, S, TGT_SEG_ZEROED, norm_specs, synth_batch_md, width, zero_target_segment  # noqa: E402

WORLD_COMM_LEADER = [(34, 5), (34, [5, 4])]     # a Discrete(5) policy beside a MultiDiscrete([5, 4]) one (simple_world_comm's leader)
WORLD_COMM_S = 68
LOSS_FLOOR = 1e-2          # smallest |loss| / grad norm a fixture may hold (see gen)


def gen(name, td3, specs, S, flags=(), B=16, steps=3, per=False, seed=44, zero_tgt_seg=None):
    rh.import_reference()
    sp = rh.gym_spaces()
    import offpolicy.utils.util as util
    import offpolicy.algorithms.maddpg.algorithm.MADDPGPolicy as polmod
    from offpolicy.envs.mpe.multi_discrete import MultiDiscrete
    args = rh.make_args(["--algorithm_name", "matd3" if td3 else "maddpg"] + list(flags))
    if td3:
        from offpolicy.algorithms.matd3.algorithm.MATD3Policy import MATD3Policy as Policy
        from offpolicy.algorithms.matd3.matd3 import MATD3 as Trainer
    else:
        from offpolicy.algorithms.maddpg.algorithm.MADDPGPolicy import MADDPGPolicy as Policy
        from offpolicy.algorithms.maddpg.maddpg import MADDPG as Trainer
    shapes = norm_specs(specs)
    p_ids = sorted(shapes)
    total = sum(width(a) * n for _, a, n in shapes.values())
    dev = torch.device("cpu")
    torch.manual_seed(3)
    pols, mapping, nxt = {}, {}, 0
    for p in p_ids:                                       # train_mpe.py:139-150: the policies in id order
        o, a, n = shapes[p]
        act = MultiDiscrete([[0, k - 1] for k in a]) if isinstance(a, list) else sp.Discrete(a)
        info = dict(obs_space=sp.Box(-np.inf, np.inf, (o,)), share_obs_space=sp.Box(-np.inf, np.inf, (S,)), act_space=act,
                    cent_obs_dim=S, cent_act_dim=total)
        pols[p] = Policy({"args": args, "device": dev}, info)
        mapping.update({k: p for k in range(nxt, nxt + n)})
        nxt += n
    out = {"construct.rng": torch.get_rng_state().numpy().copy()}
    tr = Trainer(args, nxt, pols, lambda a: mapping[a], device=dev)
    if zero_tgt_seg is not None:                          # that sub-space of the target actor ties on every row
        i, seg = zero_tgt_seg
        pol = pols[p_ids[i]]
        pol.target_actor.load_state_dict(zero_target_segment(pol.target_actor.state_dict(), seg))
        out[TGT_SEG_ZEROED] = np.array([i, seg])
    for p, pol in pols.items():
        for tag, live, tgt in (("actor", pol.actor, pol.target_actor), ("critic", pol.critic, pol.target_critic)):
            out.update(sd_np("%s.init.%s." % (p, tag), live))
            if any(not torch.equal(v, tgt.state_dict()[k]) for k, v in live.state_dict().items()):
                out.update(sd_np("%s.init.tgt_%s." % (p, tag), tgt))       # the ties edit; otherwise a copy of the live net, stored once
        out.update(heads_np("%s.init.heads." % p, pol.critic))
        out.update(heads_np("%s.init.tgt_heads." % p, pol.target_critic))
    trunk = lambda prefix, mod: {k: v for k, v in sd_np(prefix, mod).items() if ".fc_h." not in k}

    draws = []
    real_gumbel = util.sample_gumbel

    def gumbel(*a, **k):
        g = real_gumbel(*a, **k)
        draws.append(g.detach().numpy().copy())
        return g
    util.sample_gumbel = gumbel
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
                b = synth_batch_md(rng, specs, B, S, per=per)
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
                    # the tests compare these relative to their own size: a loss that is a near-cancellation of O(1) terms would ask
                    # for agreement far below fp32 summation-order round-off, so such a draw is not used as a fixture
                    assert abs(float(info_t[k])) > LOSS_FLOOR, (name, s, p, k, float(info_t[k]))
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
                for k, v in mod.state_dict().items():
                    if ".fc_h." in k:     # in no forward pass: no gradient, no Adam step; Polyak of equal values moves it by round-off only
                        d = np.abs(v.detach().numpy() - out["%s.init.%s.%s" % (p, tag.replace("tgt_", ""), k)]).max()
                        assert d <= (FC_H_POLYAK_TOL if tag.startswith("tgt_") else 0.0), (p, tag, k, d)
            out.update(heads_np("final.%s.heads." % p, pol.critic))
            out.update(heads_np("final.%s.tgt_heads." % p, pol.target_critic))
    finally:
        util.sample_gumbel = real_gumbel
    out["meta.cfg"] = np.array([S, B, steps, int(td3), int(per), int(args.use_huber_loss)])
    out["meta.obs"] = np.array([shapes[p][0] for p in p_ids], dtype=np.int64)
    out["meta.agents"] = np.array([shapes[p][2] for p in p_ids], dtype=np.int64)
    out["meta.md"] = np.array([int(isinstance(shapes[p][1], list)) for p in p_ids], dtype=np.int64)
    for i, p in enumerate(p_ids):
        a = shapes[p][1]
        out["meta.act.policy_%d" % i] = np.array(a if isinstance(a, list) else [a], dtype=np.int64)
    out["meta.hparams"] = np.array([args.gamma, args.lr, args.opti_eps, args.max_grad_norm, args.tau, args.huber_delta, args.per_eps,
                                    float(args.target_action_noise_std), args.weight_decay, args.gain], dtype=np.float64)
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, **out)
    kb = os.path.getsize(path) / 1024
    assert kb < 1024, (name, kb)
    print(name, "->", path, "%.1f KB" % kb, "critic_loss", float(out["s0.policy_0.critic_loss"]))


if __name__ == "__main__":
    torch.set_num_threads(1)          # orthogonal_ (a QR) rounds differently with the thread count: the tests replay it on one thread
    gen("mlp_matd3_md", True, REFERENCE_SPEC, S)
    gen("mlp_maddpg_md", False, REFERENCE_SPEC, S, seed=49)
    gen("mlp_maddpg_md_ties", False, REFERENCE_SPEC, S, seed=46, zero_tgt_seg=(0, 1))
    gen("mlp_maddpg_md_per_huber", False, REFERENCE_SPEC, S, flags=["--use_per", "--use_huber_loss", "--huber_delta", "1.0"], per=True,
        seed=47)
    gen("mlp_matd3_multi_md", True, WORLD_COMM_LEADER, WORLD_COMM_S, B=8, seed=48)
