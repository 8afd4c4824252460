"""The transition-level MADDPG / MATD3 against outputs of the unmodified reference (tests/golden/mlp_*.npz, made by
make_goldens_mlp_maddpg.py): the oracle (oracle/maddpg_mlp.py) to fp32 round-off, the engine on the CPU-emulated kernels to the
DESIGN.md section 2 tolerances, both from the reference's own construction and torch RNG stream."""
import numpy as np
import pytest
import torch

import mlp_maddpg_checks as mc
from helpers import load_golden, rel_err
from oracle.maddpg_mlp import MlpMaddpg, draw_noise


@pytest.mark.parametrize("name", mc.GOLDENS)
def test_oracle_reproduces_reference(name):
    """Loss 1e-6, tensors 2e-5 (relative to their max-abs), the reference's draws from the same RNG state, both head sets unchanged."""
    torch.set_num_threads(1)
    g = load_golden(name)
    (N, O, A, S, B, steps, td3, discrete), over = mc.golden_meta(g)
    L = MlpMaddpg(mc.golden_sd(g, "init.actor."), mc.golden_sd(g, "init.critic."), mc.golden_sd(g, "init.heads."),
                  mc.golden_sd(g, "init.tgt_actor."), mc.golden_sd(g, "init.tgt_critic."), mc.golden_sd(g, "init.tgt_heads."),
                  discrete, td3, gamma=over["gamma"], lr=over["lr"], eps=over["opti_eps"], weight_decay=over["weight_decay"],
                  max_grad_norm=over["max_grad_norm"], tau=over["tau"], huber=over["use_huber_loss"], huber_delta=over["huber_delta"],
                  use_per=over["use_per"], per_eps=over["per_eps"])
    for s in range(steps):
        torch.set_rng_state(torch.from_numpy(g["s%d.rng_before" % s]))
        tn, an = draw_noise(N, B, A, discrete, td3, over["target_action_noise_std"])
        assert np.array_equal(torch.get_rng_state().numpy(), g["s%d.rng_after" % s])
        assert len([d for d in (tn, an) if d is not None]) == len(mc.golden_draws(g, s))
        for mine, ref in zip([d for d in (tn, an) if d is not None], mc.golden_draws(g, s)):
            assert np.array_equal(mine.numpy(), ref)
        info, prio, grads = L.step(mc.golden_batch(g, s), tn, an)
        assert rel_err(info["critic_loss"], g["s%d.critic_loss" % s]) < 1e-6
        assert rel_err(info["actor_loss"], g["s%d.actor_loss" % s]) < 1e-6
        for k in ("critic_grad_norm", "actor_grad_norm"):
            assert rel_err(info[k], g["s%d.%s" % (s, k)]) < 1e-5, k
        if prio is not None:
            assert rel_err(prio, g["s%d.prio" % s]) < 1e-5
        for net in ("critic", "actor"):
            for k, v in grads[net].items():
                key = "s%d.grad.%s.%s" % (s, net, k)
                if key in g:
                    assert rel_err(v, g[key]) < 2e-5, key
        L.soft_update()
        for tag, d in (("actor", L.actor), ("critic", L.critic), ("tgt_actor", L.target_actor), ("tgt_critic", L.target_critic)):
            for k, v in d.items():
                assert rel_err(v.detach(), g["s%d.post.%s.%s" % (s, tag, k)]) < 2e-5, (tag, k)
        for tag, d in (("heads", L.heads), ("tgt_heads", L.target_heads)):
            for k, v in d.items():
                assert np.array_equal(v.numpy(), g["s%d.post.%s.%s" % (s, tag, k)])


@pytest.mark.parametrize("name", mc.GOLDENS)
def test_engine_reproduces_reference(emu_engine, name):
    mc.engine_against_golden(name)
