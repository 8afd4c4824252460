"""QMIX learner kernels' logic on the CPU fiber emulator vs the reference goldens (and the oracle's trace)."""
import numpy as np
import pytest
import torch

import qmix_checks as qc
from helpers import rel_err


@pytest.mark.parametrize("name", ["qmix_small", "qmix_small_huber_nodq", "qmix_small_per", "qmix_small_hyper1", "qmix_5ag"])
def test_step_matches_reference_golden(emu_engine, name):
    qc.check_step_against(None, name)


@pytest.mark.parametrize("n_agents,B,T", [(3, 8, 7), (4, 8, 7), (3, 12, 7)])
def test_front_bwd_tile_heights_vs_oracle(emu_engine, n_agents, B, T):
    """The backward front kernel picks 32-, 48- or 64-row tiles from the row count and the SM count (4 in the emulator):
    M = B (T+1) N = 192 -> 48-row tiles, 256 -> 64-row tiles, 288 -> 48-row tiles in two waves."""
    from oracle.qmix import QmixConfig, synth_batch
    cfg = QmixConfig(n_agents=n_agents, obs_dim=11, act_dim=5, state_dim=13, gain=1.0)
    L, args, pol, tr = qc.oracle_and_trainer(cfg, B, T)
    batch = synth_batch(cfg, B, T, seed=5, avail_p=0.8, var_len=True) + (None, None)
    qc.compare_step(L, pol, tr, batch, cfg, steps=2)


@pytest.mark.parametrize("name", ["qmix_small", "qmix_small_per", "qmix_small_hyper1"])
def test_fused_mixer_kernel_matches_reference_golden(emu_engine, name):
    """`mixer_split=0` selects the single fused k_mixer instead of the default hyper_fwd / core / hyper_bwd pipeline: both must
    reproduce the reference."""
    lib = emu_engine.lib()
    lib.mx_set_option(b"mixer_split", 0)
    try:
        c0 = lib.mx_launch_count()
        qc.check_step_against(None, name)
        fused = lib.mx_launch_count() - c0
    finally:
        lib.mx_set_option(b"mixer_split", 1)
    c0 = lib.mx_launch_count()
    qc.check_step_against(None, name)
    split = lib.mx_launch_count() - c0
    g = qc.load_golden(name)
    steps = int(g["meta.steps"]) if "meta.steps" in g else None
    assert split > fused and (split - fused) % 2 == 0, (split, fused, steps)      # two extra launches per learner step


@pytest.mark.parametrize("split", [1, 0])
@pytest.mark.parametrize("mixer_hidden,hyper_hidden,n_agents,layers", [(48, 40, 4, 2), (64, 64, 2, 1), (20, 64, 3, 2)])
def test_mixer_shapes_vs_oracle(emu_engine, split, mixer_hidden, hyper_hidden, n_agents, layers):
    """Mixer widths that are not the defaults (mixer_hidden not a multiple of 32 / equal to 64 = two units per lane in k_mix_core,
    hypernet_hidden != 64, one hypernet layer), split and fused kernels, PER weights + Huber, against the oracle in lock-step."""
    from oracle.qmix import QmixConfig, synth_batch
    lib = emu_engine.lib()
    cfg = QmixConfig(n_agents=n_agents, obs_dim=7, act_dim=4, state_dim=10, mixer_hidden=mixer_hidden, hyper_hidden=hyper_hidden,
                     hyper_layers=layers, gain=1.0, use_per=True, huber=True, huber_delta=0.7)
    B, T = 5, 6
    lib.mx_set_option(b"mixer_split", split)
    try:
        L, args, pol, tr = qc.oracle_and_trainer(cfg, B, T)
        w = np.random.RandomState(3).rand(B) * 0.9 + 0.1
        batch = synth_batch(cfg, B, T, seed=9, avail_p=0.8, var_len=True) + (w, np.arange(B))
        qc.compare_step(L, pol, tr, batch, cfg, steps=2)
    finally:
        lib.mx_set_option(b"mixer_split", 1)


def test_fused_mid_kernel_eight_warp_variant_vs_oracle(emu_engine):
    """SMAC 8m widths (8 agents x 14 actions): the per-warp operand slices of k_mid no longer fit 16 warps into shared memory, so the
    launcher takes the 8-warp instantiation (mid.cu mid_pick_warps).  Product configuration (debug outputs off), PER + Huber."""
    from oracle.qmix import QmixConfig, synth_batch
    lib = emu_engine.lib()
    cfg = QmixConfig(n_agents=8, obs_dim=9, act_dim=14, state_dim=11, gain=1.0, use_per=True, huber=True, huber_delta=0.8)
    B, T = 4, 5
    L, args, pol, tr = qc.oracle_and_trainer(cfg, B, T, debug=False)
    w = np.random.RandomState(4).rand(B) * 0.9 + 0.1
    batch = synth_batch(cfg, B, T, seed=11, avail_p=0.7, var_len=True) + (w, np.arange(B))
    # gradients are held to 1e-4 as everywhere; some fc2 gradient entries here are ~6e-6, the size of Adam's eps, where the first
    # Adam step amplifies fp32 round-off of the gradient -- hence the wider bound on the PARAMETERS only
    c0 = lib.mx_launch_count()
    qc.compare_step(L, pol, tr, batch, cfg, steps=2, param_tol=3e-2)
    with_mid = lib.mx_launch_count() - c0
    lib.mx_set_option(b"mid_fused", 0)
    try:
        L2, args2, pol2, tr2 = qc.oracle_and_trainer(cfg, B, T, debug=False)
        c0 = lib.mx_launch_count()
        qc.compare_step(L2, pol2, tr2, batch, cfg, steps=2, param_tol=3e-2)
        separate = lib.mx_launch_count() - c0
    finally:
        lib.mx_set_option(b"mid_fused", 1)
    assert separate > with_mid, (separate, with_mid)          # k_mid really was the kernel that ran


@pytest.mark.parametrize("name", ["qmix_small", "qmix_small_huber_nodq", "qmix_small_per", "qmix_small_hyper1", "qmix_5ag"])
def test_product_configuration_matches_reference_golden(emu_engine, name):
    """debug outputs off = what bench.py / the runner execute: k_qhead + k_mix_core + k_qhead_bwd run as the single k_mid."""
    lib = emu_engine.lib()
    c0 = lib.mx_launch_count()
    qc.check_step_against(None, name, debug=False)
    fused = lib.mx_launch_count() - c0
    lib.mx_set_option(b"mid_fused", 0)
    try:
        c0 = lib.mx_launch_count()
        qc.check_step_against(None, name, debug=False)
        separate = lib.mx_launch_count() - c0
    finally:
        lib.mx_set_option(b"mid_fused", 1)
    assert separate > fused and (separate - fused) % 2 == 0, (separate, fused)      # two launches fewer per learner step


@pytest.mark.parametrize("mixer_hidden,hyper_hidden,n_agents,act_dim", [(48, 40, 4, 4), (64, 64, 2, 20), (20, 64, 8, 17)])
def test_product_configuration_shapes_vs_oracle(emu_engine, mixer_hidden, hyper_hidden, n_agents, act_dim):
    """k_mid at other widths: more than 16 actions (one lane per action instead of two half dot products), 8 agents, wide mixer."""
    from oracle.qmix import QmixConfig, synth_batch
    cfg = QmixConfig(n_agents=n_agents, obs_dim=7, act_dim=act_dim, state_dim=10, mixer_hidden=mixer_hidden, hyper_hidden=hyper_hidden,
                     gain=1.0, use_per=True, huber=True, huber_delta=0.7)
    B, T = 5, 6
    L, args, pol, tr = qc.oracle_and_trainer(cfg, B, T, debug=False)
    w = np.random.RandomState(3).rand(B) * 0.9 + 0.1
    batch = synth_batch(cfg, B, T, seed=9, avail_p=0.6, var_len=True) + (w, np.arange(B))
    qc.compare_step(L, pol, tr, batch, cfg, steps=2)


def test_mpe_shapes_without_avail_masks(emu_engine):
    qc.check_mpe_shapes_without_avail_masks(steps=1, B=8)       # (the GPU test runs the script's batch of 32, two steps)


@pytest.mark.parametrize("debug", [True, False])
def test_prev_act_inp_matches_reference_golden(emu_engine, debug):
    """--prev_act_inp (config.py:81): the agent net reads [obs | previous one-hot action]; golden made by the reference with the flag."""
    qc.check_step_against(None, "qmix_small_prev_act", intermediates=False, debug=debug)


@pytest.mark.parametrize("opts", [dict(), dict(front_tc=0), dict(wgrad_tc=2)], ids=["default", "ffma_front", "tc_backward"])
def test_feature_normalization_off_matches_reference_golden(emu_engine, opts):
    """--use_feature_normalization (a store_false flag): no input LayerNorm, its two tensors absent from the state_dict."""
    lib = emu_engine.lib()
    for k, v in opts.items():
        lib.mx_set_option(k.encode(), v)
    try:
        qc.check_step_against(None, "qmix_small_nofn", intermediates=False, debug=False)
    finally:
        lib.mx_set_option(b"front_tc", 1)
        lib.mx_set_option(b"wgrad_tc", -1)


@pytest.mark.parametrize("opts", [dict(), dict(front_tc=0), dict(wgrad_tc=2)], ids=["default", "ffma_front", "tc_backward"])
def test_tanh_networks_match_reference_golden(emu_engine, opts):
    """--use_ReLU (a store_false flag): Linear -> Tanh -> LayerNorm blocks (mlp.py:12,19-22); the backward uses tanh' = 1 - u^2 on the saved
    activation outputs."""
    lib = emu_engine.lib()
    for k, v in opts.items():
        lib.mx_set_option(k.encode(), v)
    try:
        qc.check_step_against(None, "qmix_small_tanh", intermediates=True, debug="wgrad_tc" not in opts)
    finally:
        lib.mx_set_option(b"front_tc", 1)
        lib.mx_set_option(b"wgrad_tc", -1)


@pytest.mark.parametrize("B,N,T", [(2, 2, 5), (4, 2, 5), (5, 3, 5), (8, 3, 5), (2, 2, 9), (4, 2, 9), (5, 3, 9), (8, 3, 9)])
def test_recurrence_kernel_families_vs_oracle(emu_engine, B, N, T):
    """Both CTA widths of the GRU recurrences, picked by sequence length.  T = 5: the 256-thread k_gru_fwd / k_gru_bwd with 1, 2 or 4 rows
    per CTA from the row count (R = B N = 4, 8, 15, 24 on the emulator's 4 SMs: forward 1 / 2 / 4 / 4, backward 1 / 1 / 2 / 4).  T = 9: the
    128-thread k_gru_fwd2 / k_gru_bwd2, one row per CTA.  Forward intermediates, then two steps in lock-step with the oracle."""
    from oracle.qmix import QmixConfig, synth_batch
    cfg = QmixConfig(n_agents=N, obs_dim=11, act_dim=5, state_dim=13, gain=1.0)
    L, args, pol, tr = qc.oracle_and_trainer(cfg, B, T)
    batch = synth_batch(cfg, B, T, seed=21, avail_p=0.8, var_len=True) + (None, None)
    for s in range(2):
        info, prio, _ = tr.train_policy_on_batch(qc.ref_tuple(batch))
        if s == 0:
            bad = qc.check_forward_intermediates(tr, L, batch, cfg, B, T)
            assert not bad, bad
        qc.check_engine_step(L, pol, tr, batch, cfg, info, prio, {k: v.clone() for k, v in tr.grad_views().items()}, s)


@pytest.mark.parametrize("td3,disc", [(False, False), (True, True)])
def test_recurrence_kernel_128_threads_maddpg(emu_engine, td3, disc):
    """R-MADDPG / R-MATD3 at T = 9: the 128-thread recurrences run the actor (T1 = T + 1) and the critic over the buffer sequence, whose
    backward stores T1 = T steps per sequence (the one-step branch rows with an initial state stay on the 256-thread kernels).  Three
    updates against the oracle: losses, grad norms, every critic gradient tensor, all four networks."""
    import maddpg_checks as mc
    from oracle.maddpg import MaddpgConfig, MaddpgLearner, synth_batch_cont, synth_batch_disc, sample_gumbel
    from oracle.qmix import randomize_all
    cfg = MaddpgConfig(act_dim=5 if disc else 2, discrete=disc, td3=td3, actor_update_interval=2 if td3 else 1, gain=1.0)
    B, T = 4, 9
    L = MaddpgLearner(cfg, seed=5)
    randomize_all(L.actor, 1); randomize_all(L.critic, 2)
    L.sync_targets()
    randomize_all(L.tgt_actor, 3, 0.05); randomize_all(L.tgt_critic, 4, 0.05)
    args, pol, tr = mc.build(cfg, B, T)
    for ours, ref in ((pol.actor, L.actor), (pol.critic, L.critic), (pol.target_actor, L.tgt_actor), (pol.target_critic, L.tgt_critic)):
        ours.load_state_dict(ref.state_dict())
    for s in range(3):
        batch = (synth_batch_disc if disc else synth_batch_cont)(cfg, B, T, seed=40 + s) + (None, None)
        upd = s % cfg.actor_update_interval == 0
        torch.manual_seed(77 + s)
        if disc:
            noise = sample_gumbel((T + 1, cfg.n_agents * B, cfg.act_dim)).numpy() if td3 else None
            anoise = sample_gumbel((T, cfg.n_agents * B, cfg.act_dim)).numpy() if upd else None
        else:
            noise = torch.empty(T + 1, cfg.n_agents * B, cfg.act_dim).normal_(mean=0, std=cfg.target_noise).numpy() if td3 else None
            anoise = None
        torch.manual_seed(77 + s)
        info, _, _ = tr.shared_train_policy_on_batch("policy_0", mc.ref_tuple(batch))
        ref, _ = L.step(batch, noise, anoise)
        assert rel_err(info["critic_loss"].cpu(), ref["critic_loss"]) < 1e-4
        assert rel_err(info["critic_grad_norm"].cpu(), ref["critic_grad_norm"]) < 1e-4
        ga, gc = tr.grad_views()
        coef = min(1.0, cfg.max_grad_norm / (float(ref["critic_grad_norm"]) + 1e-6))
        cviews = mc.named_views(gc, pol._c_entries)
        for k, gr in L.critic_grads.items():
            ok, err, lim = qc.close(cviews[k] / gc[pol.Pc] * coef, gr, 1e-4)
            assert ok, (s, k, err, lim)
        assert bool(info["update_actor"]) == bool(ref["update_actor"]) == upd
        if ref["update_actor"]:
            assert rel_err(info["actor_loss"].cpu(), ref["actor_loss"]) < 1e-4
            assert rel_err(info["actor_grad_norm"].cpu(), ref["actor_grad_norm"]) < 2e-4
            pol.soft_target_updates()
            L.soft_update()
    for ours, ref in ((pol.actor, L.actor), (pol.critic, L.critic), (pol.target_actor, L.tgt_actor), (pol.target_critic, L.tgt_critic)):
        for k, v in ours.state_dict().items():
            assert float((v.cpu() - ref.state_dict()[k]).abs().max()) <= 5e-3 * cfg.lr * 3 + 1e-7, k


@pytest.mark.parametrize("obs,prev,relu", [(57, False, True), (60, False, False), (64, False, True), (64, False, False), (50, True, True),
                                           (55, True, False)])
def test_one_thread_per_row_front_kernel_vs_oracle(emu_engine, obs, prev, relu):
    """Input widths 57 .. 64 (with --prev_act_inp: observation + 9 actions) fill the shared memory with operand tiles, so the pair-exchange
    buffer of k_front_fwd_tc2 no longer fits and the launcher takes k_front_fwd_tc (one thread per accumulator row); ReLU and tanh blocks.
    Forward intermediates (without the previous-action input, which the oracle's trace does not stack), then two steps in lock-step."""
    from oracle.qmix import QmixConfig, synth_batch
    cfg = QmixConfig(n_agents=3, obs_dim=obs, act_dim=9, state_dim=20, gain=1.0, prev_act_inp=prev, relu=relu)
    B, T = 5, 6
    L, args, pol, tr = qc.oracle_and_trainer(cfg, B, T)
    batch = synth_batch(cfg, B, T, seed=8, avail_p=0.8, var_len=True) + (None, None)
    for s in range(2):
        info, prio, _ = tr.train_policy_on_batch(qc.ref_tuple(batch))
        if s == 0 and not prev:
            bad = qc.check_forward_intermediates(tr, L, batch, cfg, B, T)
            assert not bad, bad
        qc.check_engine_step(L, pol, tr, batch, cfg, info, prio, {k: v.clone() for k, v in tr.grad_views().items()}, s)
