"""QMIX learner kernels' logic on the CPU fiber emulator vs the reference goldens (and the oracle's trace)."""
import numpy as np
import pytest

import qmix_checks as qc


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


@pytest.mark.parametrize("threads", [128, 256])
@pytest.mark.parametrize("name,debug", [("qmix_small", True), ("qmix_small", False), ("qmix_5ag", False), ("qmix_small_per", False)])
def test_recurrence_kernel_variants_match_reference_golden(emu_engine, name, debug, threads):
    """Both CTA widths of the GRU recurrences (option gru_threads: the 128-thread kernels k_gru_fwd2 / k_gru_bwd2 are picked when all rows
    are resident at once, the 256-thread ones otherwise) against the reference goldens, intermediates included."""
    lib = emu_engine.lib()
    lib.mx_set_option(b"gru_threads", threads)
    try:
        qc.check_step_against(None, name, intermediates=True, debug=debug)
    finally:
        lib.mx_set_option(b"gru_threads", 0)


@pytest.mark.parametrize("name,debug", [("qmix_small", True), ("qmix_5ag", False), ("qmix_small_per", False), ("qmix_small_tanh", True)])
def test_two_rows_per_cta_recurrences_match_reference_golden(emu_engine, name, debug):
    """Option gru_rows = 2: k_gru_fwd2<2> / k_gru_bwd2<2> carry two sequence rows per CTA through the same register-resident W_hh slice (picked
    automatically when there are more row-CTAs than two per SM hold at once: SMAC 8m).  Intermediates included; odd row counts leave
    the last CTA with one empty slot."""
    lib = emu_engine.lib()
    lib.mx_set_option(b"gru_rows", 2)
    try:
        qc.check_step_against(None, name, intermediates=True, debug=debug)
    finally:
        lib.mx_set_option(b"gru_rows", 0)


def test_two_rows_per_cta_recurrences_odd_row_count_vs_oracle(emu_engine):
    from oracle.qmix import QmixConfig, synth_batch
    lib = emu_engine.lib()
    cfg = QmixConfig(n_agents=3, obs_dim=9, act_dim=5, state_dim=11, gain=1.0)
    B, T = 5, 9            # 15 rows: the eighth CTA of each net has one row and one empty slot
    lib.mx_set_option(b"gru_rows", 2)
    try:
        L, args, pol, tr = qc.oracle_and_trainer(cfg, B, T)
        batch = synth_batch(cfg, B, T, seed=21, avail_p=0.8, var_len=True) + (None, None)
        qc.compare_step(L, pol, tr, batch, cfg, steps=2)
    finally:
        lib.mx_set_option(b"gru_rows", 0)


@pytest.mark.parametrize("name", ["maddpg_box", "matd3_disc_avail"])
def test_recurrence_kernel_128_threads_maddpg(emu_engine, name):
    """R-MADDPG uses the recurrences with an initial state (branch steps, h0) and T1 != T + 1: the 128-thread kernels on those paths."""
    import maddpg_checks as mdc
    lib = emu_engine.lib()
    lib.mx_set_option(b"gru_threads", 128)
    try:
        mdc.check_golden(name)
        lib.mx_set_option(b"gru_rows", 2)          # two rows per CTA on the same paths (initial state h0, T1 != T + 1)
        mdc.check_golden(name)
    finally:
        lib.mx_set_option(b"gru_threads", 0)
        lib.mx_set_option(b"gru_rows", 0)


@pytest.mark.parametrize("threads", [128, 256])
@pytest.mark.parametrize("name", ["qmix_small", "qmix_small_prev_act", "qmix_small_tanh"])
def test_front_tensor_core_kernel_variants_match_reference_golden(emu_engine, name, threads):
    """k_front_fwd_tc (one thread per accumulator row) and k_front_fwd_tc2 (two threads per row, pair-wise LayerNorm statistics): option
    front_tc_threads, default 256."""
    lib = emu_engine.lib()
    lib.mx_set_option(b"front_tc_threads", threads)
    try:
        qc.check_step_against(None, name, intermediates=(name != "qmix_small_prev_act"), debug=True)
    finally:
        lib.mx_set_option(b"front_tc_threads", 256)


@pytest.mark.parametrize("split", [0, 1])
@pytest.mark.parametrize("name", ["qmix_small", "qmix_5ag", "qmix_small_per", "qmix_small_tanh"])
def test_gru_weight_gradient_kernel_split_matches_reference_golden(emu_engine, name, split):
    """Option gru_wgrad_split: dW_ih / dW_hh / db_ih / db_hh from k_gru_wgrad (its own kernel, launched beside k_front_bwd on the GPU;
    default) or from inside k_front_bwd (0).  Same gradient partial rows either way; one more launch per step with the split."""
    lib = emu_engine.lib()
    lib.mx_set_option(b"gru_wgrad_split", split)
    lib.mx_set_option(b"wgrad_tc", 0)
    try:
        c0 = lib.mx_launch_count()
        qc.check_step_against(None, name, intermediates=False, debug=False)
        n = lib.mx_launch_count() - c0
    finally:
        lib.mx_set_option(b"gru_wgrad_split", 1)
        lib.mx_set_option(b"wgrad_tc", -1)
    test_gru_weight_gradient_kernel_split_matches_reference_golden.counts[(name, split)] = n
    both = test_gru_weight_gradient_kernel_split_matches_reference_golden.counts
    if (name, 0) in both and (name, 1) in both:
        assert both[(name, 1)] > both[(name, 0)], both


test_gru_weight_gradient_kernel_split_matches_reference_golden.counts = {}


@pytest.mark.parametrize("mma", [0, 1])
@pytest.mark.parametrize("name", ["qmix_small", "qmix_5ag", "qmix_small_nofn"])
def test_front_backward_gemm_variants_match_reference_golden(emu_engine, name, mma):
    """k_front_bwd with its GEMMs on mma.sync 3xTF32 tiles (csrc/mx_mma.cuh, default) and on the FFMA micro-kernels (option front_bwd_mma)."""
    lib = emu_engine.lib()
    lib.mx_set_option(b"front_bwd_mma", mma)
    lib.mx_set_option(b"wgrad_tc", 0)
    try:
        qc.check_step_against(None, name, intermediates=False, debug=False)
    finally:
        lib.mx_set_option(b"front_bwd_mma", 0)
        lib.mx_set_option(b"wgrad_tc", -1)
