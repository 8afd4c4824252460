"""Generate the QMIX / M-QMIX fixtures with more than 32 actions by running the UNMODIFIED reference (build container only).

    python tests/golden/make_goldens_qmix_many_actions.py

SMAC's action count is 6 + the number of enemies, so 27m_vs_30m has 36 actions: past the 32 that one warp lane per action covers.
Five fixtures, in the format of the other QMIX fixtures (tests/golden/make_goldens.py):
  qmix_a36_ties          recurrent QMIX, 5 agents, 36 actions, double Q, avail masks; the live head's rows 35 / 3 and 33 / 32 are
                         equal and lead the others, so the greedy choice is mostly a tie, which must resolve to the lower action
                         (across a lane's pair of actions and across lanes)
  qmix_a64_hyper1        64 actions, 1-layer hypernets, Huber loss, no double Q
  qmix_a33_prev_act      33 actions with --prev_act_inp (network input obs + 33)
  mqmix_a36              M-QMIX, 36 actions, avail and next-step avail masks
  qmix_rollout_a36       the rollout surface at 36 actions: greedy chain, sequence form, exploring and random actions
The recurrent QMIX fixtures store their initial weights as four seeds (tests/qmix_wide_fixture.py) plus, for qmix_a36_ties, the tied
live head (tests/qmix_many_actions_fixture.py), and hold one step each, so that each stays under 1 MB.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]

import make_goldens as mg  # noqa: E402
from oracle.qmix import QmixConfig  # noqa: E402

SEEDS = np.array([31, 32, 33, 34], np.int64)
TIES = ((3, 35), (32, 33))      # (kept row, row made equal to it): the lower index must win on equal Q


def tie_head_rows(q_network, pairs=TIES):
    """Make head rows equal (weight and bias) so that their Q values are bit-equal for every input, and raise their biases above
    the others so that a tied pair is the greedy choice wherever one of its actions is available."""
    with torch.no_grad():
        out = q_network.q.action_out
        top = float(out.bias.max())
        for i, (src, dst) in enumerate(pairs):
            out.bias[src] = top + 4.0 / (i + 1)
            out.weight[dst].copy_(out.weight[src])
            out.bias[dst].copy_(out.bias[src])


def gen_qmix_seeded(name, cfg, flags=(), B=3, T=6, ties=False):
    """One reference step from seeded initial weights (tests/qmix_wide_fixture.py), as make_goldens.py's gen_qmix stores it.  ties:
    the live agent's tied head rows are applied after the seeds are loaded and stored as `init_head.*` (the targets keep distinct rows,
    so which of two tied actions is greedy changes the double-Q target)."""
    import qmix_wide_fixture as wf
    from oracle.qmix import synth_batch
    flags = ["--mixer_hidden_dim", str(cfg.mixer_hidden), "--hypernet_hidden_dim", str(cfg.hyper_hidden)] + list(flags)
    args, pol, tr = mg.build_reference_qmix(cfg, flags, T)
    nets = {"agent": pol.q_network, "mixer": tr.mixer, "tgt_agent": tr.target_policies["policy_0"].q_network, "tgt_mixer": tr.target_mixer}
    sds = wf.init_state({"agent": pol.q_network.state_dict(), "mixer": tr.mixer.state_dict()}, SEEDS)
    for role, net in nets.items():
        net.load_state_dict(sds[role])
    out = {"meta.init_seeds": SEEDS}
    if ties:
        tie_head_rows(pol.q_network)
        out["init_head.weight"] = pol.q_network.q.action_out.weight.detach().numpy().copy()
        out["init_head.bias"] = pol.q_network.q.action_out.bias.detach().numpy().copy()
    b = synth_batch(cfg, B, T, seed=100, avail_p=0.7, var_len=True)
    for k, v in zip(["obs", "share", "acts", "rew", "dones", "dones_env", "avail"], b):
        out["s0.in.%s" % k] = v
    info, prio, _ = tr.train_policy_on_batch(mg.to_ref_batch(b))
    out["s0.loss"] = info["loss"].detach().numpy()
    out["s0.grad_norm"] = np.asarray(float(info["grad_norm"]), np.float32)
    out["s0.Q_tot"] = info["Q_tot"].detach().numpy()
    for k, p in pol.q_network.named_parameters():
        if p.grad is not None:
            out["s0.grad.agent.%s" % k] = p.grad.numpy().copy()
    for k, p in tr.mixer.named_parameters():
        out["s0.grad.mixer.%s" % k] = p.grad.numpy().copy()
    tr.soft_target_updates()
    for role, net in nets.items():
        out.update(mg.sd_np("s0.%s." % role, net))
    out["meta.cfg"] = np.array([cfg.n_agents, cfg.obs_dim, cfg.act_dim, cfg.state_dim, cfg.hidden, cfg.mixer_hidden,
                                cfg.hyper_hidden, cfg.hyper_layers, B, T, 1])
    out["meta.flags"] = np.array([args.use_double_q, args.use_huber_loss, False, bool(args.prev_act_inp), not args.use_feature_normalization,
                                  not args.use_ReLU], dtype=np.int64)
    out["meta.hparams"] = np.array([args.gamma, args.lr, args.opti_eps, args.max_grad_norm, args.tau, args.huber_delta,
                                    args.per_nu, args.per_eps], dtype=np.float64)
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, **out)
    print(name, "->", path, "%.1f KB" % (os.path.getsize(path) / 1024), "loss", out["s0.loss"])


def gen_rollout(name, cfg, steps=4):
    """The reference QMixPolicy's rollout surface, as tests/golden/make_goldens.py's qmix_rollout, at `cfg`."""
    args, pol, tr = mg.build_reference_qmix(cfg, (), 8)
    tie_head_rows(pol.q_network)
    out = {}
    out.update(mg.sd_np("init.agent.", pol.q_network))
    rs = np.random.RandomState(93)
    R = cfg.n_agents
    obs = rs.randn(steps, R, cfg.obs_dim).astype(np.float32)
    avail = (rs.rand(steps, R, cfg.act_dim) < 0.6).astype(np.float32)
    avail[:, :, 0] = 1.0
    out["in.obs"], out["in.avail"] = obs, avail
    with torch.no_grad():
        h = np.zeros((R, cfg.hidden), np.float32)
        for t in range(steps):
            a, h2, gq = pol.get_actions(obs[t], None, h, avail[t])
            out["greedy%d.actions" % t], out["greedy%d.h" % t], out["greedy%d.q" % t] = np.asarray(a, np.float32), h2.numpy().copy(), gq.numpy().copy()
            h = h2.numpy()
        q_seq, h_seq = pol.get_q_values(obs, None, torch.zeros(R, cfg.hidden))
        out["seq.q"], out["seq.h"] = q_seq.numpy().copy(), h_seq.numpy().copy()
        for tag, av in (("explore", avail[0]), ("explore_noavail", None)):
            torch.manual_seed(5); np.random.seed(5)
            a, h2, gq = pol.get_actions(obs[0], None, np.zeros((R, cfg.hidden), np.float32), av, t_env=20000, explore=True)
            out[tag + ".actions"], out[tag + ".q"] = np.asarray(a, np.float32), gq.numpy().copy()
        torch.manual_seed(6); np.random.seed(6)
        out["random.actions"] = np.asarray(pol.get_random_actions(obs[0], avail[0]), np.float32)
        torch.manual_seed(6); np.random.seed(6)
        out["random_noavail.actions"] = np.asarray(pol.get_random_actions(obs[0]), np.float32)
    out["meta.cfg"] = np.array([cfg.n_agents, cfg.obs_dim, cfg.act_dim, cfg.hidden, steps])
    out["meta.eps"] = np.array([args.epsilon_start, args.epsilon_finish, args.epsilon_anneal_time], np.float64)
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, **out)
    print(name, "->", path, "%.1f KB" % (os.path.getsize(path) / 1024))


if __name__ == "__main__":
    torch.set_num_threads(1)
    gen_qmix_seeded("qmix_a36_ties", QmixConfig(n_agents=5, obs_dim=30, act_dim=36, state_dim=48), ties=True)
    gen_qmix_seeded("qmix_a64_hyper1", QmixConfig(n_agents=3, obs_dim=30, act_dim=64, state_dim=48, hyper_layers=1),
                    flags=["--use_huber_loss", "--use_double_q"])
    gen_qmix_seeded("qmix_a33_prev_act", QmixConfig(n_agents=3, obs_dim=30, act_dim=33, state_dim=48), flags=["--prev_act_inp"])
    mg.gen_mqmix("mqmix_a36", QmixConfig(n_agents=3, obs_dim=18, act_dim=36, state_dim=54), steps=1)
    gen_rollout("qmix_rollout_a36", QmixConfig(n_agents=5, obs_dim=30, act_dim=36, state_dim=48))
