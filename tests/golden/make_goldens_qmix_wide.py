"""Generate the wide-state QMIX fixtures by running the UNMODIFIED reference QMix (build container only).

    python tests/golden/make_goldens_qmix_wide.py

State 448 with 3 agents is just past the point where the hypernet tile of the shared-memory mixer kernels no longer fits an SM, so the
engine takes its wide-state path (tensor-core state layers).  Two fixtures:
  qmix_wide_s448          2-layer hypernets, double Q, availability masks
  qmix_wide_s448_hyper1   1-layer hypernets, Huber loss
Each holds the step's inputs, loss, grad_norm, Q_tot, every clipped gradient, the post-Adam parameters and the post-Polyak targets.
The initial weights are stored as four seeds (tests/qmix_wide_fixture.py) and loaded into the reference's networks before the step.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]

from make_goldens import build_reference_qmix, sd_np, to_ref_batch  # noqa: E402
from oracle.qmix import QmixConfig, synth_batch  # noqa: E402
import qmix_wide_fixture as wf  # noqa: E402

SEEDS = np.array([21, 22, 23, 24], np.int64)


def gen(name, cfg, flags=(), B=3, T=5):
    flags = ["--mixer_hidden_dim", str(cfg.mixer_hidden), "--hypernet_hidden_dim", str(cfg.hyper_hidden)] + list(flags)
    args, pol, tr = build_reference_qmix(cfg, flags, T)
    nets = {"agent": pol.q_network, "mixer": tr.mixer, "tgt_agent": tr.target_policies["policy_0"].q_network, "tgt_mixer": tr.target_mixer}
    sds = wf.init_state({"agent": pol.q_network.state_dict(), "mixer": tr.mixer.state_dict()}, SEEDS)
    for role, net in nets.items():
        net.load_state_dict(sds[role])
    out = {"meta.init_seeds": SEEDS}
    b = synth_batch(cfg, B, T, seed=300, avail_p=0.7, var_len=True)
    for k, v in zip(["obs", "share", "acts", "rew", "dones", "dones_env", "avail"], b):
        out["s0.in.%s" % k] = v
    info, prio, _ = tr.train_policy_on_batch(to_ref_batch(b))
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
        out.update(sd_np("s0.%s." % role, net))
    out["meta.cfg"] = np.array([cfg.n_agents, cfg.obs_dim, cfg.act_dim, cfg.state_dim, cfg.hidden, cfg.mixer_hidden,
                                cfg.hyper_hidden, cfg.hyper_layers, B, T, 1])
    out["meta.flags"] = np.array([args.use_double_q, args.use_huber_loss, False, bool(args.prev_act_inp), not args.use_feature_normalization,
                                  not args.use_ReLU], dtype=np.int64)
    out["meta.hparams"] = np.array([args.gamma, args.lr, args.opti_eps, args.max_grad_norm, args.tau, args.huber_delta,
                                    args.per_nu, args.per_eps], dtype=np.float64)
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, **out)
    print(name, "->", path, "%.1f KB" % (os.path.getsize(path) / 1024), "loss", out["s0.loss"])


if __name__ == "__main__":
    torch.set_num_threads(1)
    gen("qmix_wide_s448", QmixConfig(n_agents=3, obs_dim=30, act_dim=9, state_dim=448, mixer_hidden=16, hyper_hidden=16))
    gen("qmix_wide_s448_hyper1", QmixConfig(n_agents=3, obs_dim=30, act_dim=9, state_dim=448, mixer_hidden=16, hyper_hidden=16,
                                            hyper_layers=1), flags=["--use_huber_loss"])
