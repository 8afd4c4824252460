"""Generate tests/golden/mlp_{maddpg,matd3}_*.npz by running the UNMODIFIED reference's transition-level MADDPG / MATD3
(offpolicy/algorithms/{maddpg,matd3}) in the build container:

    python tests/golden/make_goldens_mlp_maddpg.py

Weights are the reference's own construction under torch.manual_seed, so a fixture also pins the construction order (the torch RNG
state after construction is stored).  Per update it stores the inputs, every noise draw the reference made (captured by wrapping its
sample_gumbel / gaussian_noise, in call order), train_info, the clipped gradients each optimiser stepped with, the post-Adam
parameters, the post-Polyak targets, both Q-head sets, the PER priorities and the torch RNG state before and after the update.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [HERE, os.path.join(ROOT, "tests"), ROOT]

import ref_harness as rh  # noqa: E402
from mlp_maddpg_checks import synth_batch  # noqa: E402

N, O, A, S = 3, 18, 5, 54          # simple_spread (scripts/train_mpe_maddpg.sh)
FIELDS = ("obs", "share_obs", "acts", "rewards", "next_obs", "next_share_obs", "dones", "dones_env", "valid_transition", "avail_acts",
          "next_avail_acts")


def sd_np(prefix, module):
    return {prefix + k: v.detach().numpy().copy() for k, v in module.state_dict().items()}


def heads_np(prefix, critic):
    out = {}
    for k, q in enumerate(critic.q_outs):
        out["%sq_outs.%d.weight" % (prefix, k)] = q.weight.detach().numpy().copy()
        out["%sq_outs.%d.bias" % (prefix, k)] = q.bias.detach().numpy().copy()
    return out


def gen(name, td3, discrete, flags=(), B=16, steps=3, avail=False, ties=False, per=False):
    rh.import_reference()
    sp = rh.gym_spaces()
    import offpolicy.utils.util as util
    args = rh.make_args(["--algorithm_name", "matd3" if td3 else "maddpg"] + list(flags))
    if td3:
        import offpolicy.algorithms.maddpg.algorithm.MADDPGPolicy as polmod
        from offpolicy.algorithms.matd3.algorithm.MATD3Policy import MATD3Policy as Policy
        from offpolicy.algorithms.matd3.matd3 import MATD3 as Trainer
    else:
        import offpolicy.algorithms.maddpg.algorithm.MADDPGPolicy as polmod
        from offpolicy.algorithms.maddpg.algorithm.MADDPGPolicy import MADDPGPolicy as Policy
        from offpolicy.algorithms.maddpg.maddpg import MADDPG as Trainer
    info = dict(obs_space=sp.Box(-np.inf, np.inf, (O,)), share_obs_space=sp.Box(-np.inf, np.inf, (S,)),
                act_space=sp.Discrete(A) if discrete else sp.Box(-1.0, 1.0, (A,)), cent_obs_dim=S, cent_act_dim=A * N)
    dev = torch.device("cpu")
    torch.manual_seed(3)
    pol = Policy({"args": args, "device": dev}, info)
    out = {"construct.rng": torch.get_rng_state().numpy().copy()}
    tr = Trainer(args, N, {"policy_0": pol}, lambda a: "policy_0", device=dev)
    for tag, mod in (("actor", pol.actor), ("critic", pol.critic), ("tgt_actor", pol.target_actor), ("tgt_critic", pol.target_critic)):
        out.update(sd_np("init.%s." % tag, mod))
    out.update(heads_np("init.heads.", pol.critic))
    out.update(heads_np("init.tgt_heads.", pol.target_critic))

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
    for tag, opt, mod in (("critic", pol.critic_optimizer, pol.critic), ("actor", pol.actor_optimizer, pol.actor)):
        step = opt.step

        def recording_step(*a, _step=step, _tag=tag, _mod=mod, **k):
            for n, p in _mod.named_parameters():
                if p.grad is not None:
                    grads["%s.%s" % (_tag, n)] = p.grad.detach().numpy().copy()
            return _step(*a, **k)
        opt.step = recording_step
    rng = np.random.default_rng(40)
    try:
        for s in range(steps):
            b = synth_batch(rng, N, B, O, S, A, discrete, avail=avail, ties=ties, per=per)
            for f, v in zip(FIELDS, b[:11]):
                if v["policy_0"] is not None:
                    out["s%d.in.%s" % (s, f)] = v["policy_0"]
            if per:
                out["s%d.in.weights" % s] = b[11]
            draws.clear()
            grads.clear()
            out["s%d.rng_before" % s] = torch.get_rng_state().numpy().copy()
            info_t, prio, _ = tr.shared_train_policy_on_batch("policy_0", b)
            out["s%d.rng_after" % s] = torch.get_rng_state().numpy().copy()
            for i, d in enumerate(draws):
                out["s%d.draw%d" % (s, i)] = d
            for k in ("critic_loss", "critic_grad_norm", "actor_loss", "actor_grad_norm"):
                out["s%d.%s" % (s, k)] = np.asarray(float(info_t[k]), np.float64)
            assert info_t["update_actor"]
            for k, v in grads.items():
                out["s%d.grad.%s" % (s, k)] = v
            if prio is not None:
                out["s%d.prio" % s] = np.asarray(prio, np.float32)
            for tag, mod in (("actor", pol.actor), ("critic", pol.critic)):
                out.update(sd_np("s%d.post.%s." % (s, tag), mod))
            pol.soft_target_updates()
            for tag, mod in (("tgt_actor", pol.target_actor), ("tgt_critic", pol.target_critic)):
                out.update(sd_np("s%d.post.%s." % (s, tag), mod))
            out.update(heads_np("s%d.post.heads." % s, pol.critic))
            out.update(heads_np("s%d.post.tgt_heads." % s, pol.target_critic))
    finally:
        util.sample_gumbel, polmod.gaussian_noise = real_gumbel, real_gauss
    out["meta.cfg"] = np.array([N, O, A, S, B, steps, int(td3), int(discrete), int(per), int(args.use_huber_loss)])
    out["meta.hparams"] = np.array([args.gamma, args.lr, args.opti_eps, args.max_grad_norm, args.tau, args.huber_delta, args.per_eps,
                                    float(args.target_action_noise_std), args.weight_decay, args.gain], dtype=np.float64)
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, **out)
    print(name, "->", path, "%.1f KB" % (os.path.getsize(path) / 1024), "critic_loss", float(out["s0.critic_loss"]))


if __name__ == "__main__":
    torch.set_num_threads(1)          # orthogonal_ (a QR) rounds differently with the thread count: the tests replay it on one thread
    gen("mlp_maddpg_disc", False, True)
    gen("mlp_matd3_disc", True, True)
    gen("mlp_maddpg_box", False, False)
    gen("mlp_matd3_box", True, False)
    gen("mlp_maddpg_disc_avail", False, True, avail=True, ties=True)
    gen("mlp_maddpg_per_huber", False, True, flags=["--use_per", "--use_huber_loss", "--huber_delta", "1.0"], per=True)
