"""Tensor-core (wgmma) kernels on the CPU emulator (tests/emu + csrc/mx_tc.cuh's restated instructions): the emulated wgmma decodes
shared-memory descriptors with the convention the GPU runs validated (tests/test_gpu_tc.py) and fills each thread's own fragment registers,
so these tests run the kernels' INDEXING -- operand tiles, descriptor strides, the warpgroups' tile dealing, fragment placement in the
per-CTA accumulator slices, mbarrier arrivals -- without a GPU.  Async-proxy ordering is outside what an emulator can see."""
import numpy as np
import pytest
import torch

import qmix_checks as qc


def probe(capi, M, N, K, passes, swap):
    lib = capi.lib()
    g = torch.Generator().manual_seed(M * 7 + N)
    X = torch.randn(M, K, generator=g)
    W = torch.randn(N, K, generator=g) * 0.3
    Y = torch.full((M, N), float("nan"))
    capi.check(lib.mx_tc_linear_probe(capi.ptr(X), capi.ptr(W), capi.ptr(Y), M, N, K, passes, swap, None))
    ref = X.double() @ W.double().t()
    return float((Y.double() - ref).abs().max() / ref.abs().max())


def test_3xtf32_building_block_matches_fp64(emu_engine):
    for (M, N, K) in [(128, 16, 8), (300, 64, 64), (100, 256, 64), (130, 192, 64)]:
        e3 = probe(emu_engine, M, N, K, 3, 0)
        e1 = probe(emu_engine, M, N, K, 1, 0)
        assert e3 < 2e-6, (M, N, K, e3)
        assert 1e-5 < e1 < 5e-3, (M, N, K, e1)
    assert probe(emu_engine, 128, 64, 64, 3, 1) > 1e-2          # the other stride assignment reads the wrong core matrices


@pytest.mark.parametrize("front_tc", [1, 0])
def test_qmix_step_front_paths_match_reference_golden(emu_engine, front_tc):
    lib = emu_engine.lib()
    lib.mx_set_option(b"front_tc", front_tc)
    try:
        qc.check_step_against(None, "qmix_5ag")
    finally:
        lib.mx_set_option(b"front_tc", 1)


@pytest.mark.parametrize("obs_dim", [65, 80, 100, 128])
def test_wide_input_front_kernel_vs_oracle(emu_engine, obs_dim):
    """64 < obs_dim <= 128 (SMAC 8m / 2s3z observations are 80 wide): fc1's K dimension fed to the tensor core in two chunks that
    accumulate in the accumulator (k_front_fwd_tc_wide2).  More than 128 rows so a CTA runs several tiles."""
    from oracle.qmix import QmixConfig, synth_batch
    cfg = QmixConfig(n_agents=5, obs_dim=obs_dim, act_dim=6, state_dim=20, gain=1.0)
    B, T = 12, 5           # 12 * 6 * 5 = 360 rows: 3 tiles for the 2 CTAs per net of the emulator's 4 "SMs"
    L, args, pol, tr = qc.oracle_and_trainer(cfg, B, T, debug=False)
    batch = synth_batch(cfg, B, T, seed=4, avail_p=0.7, var_len=True) + (None, None)
    # parameter bound 1e-2 * lr: an element with |g| ~ eps sees Adam amplify a 1e-6-relative gradient difference (measured 5.3e-3 * lr
    # at obs 100, with the gradients themselves equal to 9e-7 of their maximum)
    qc.compare_step(L, pol, tr, batch, cfg, steps=2, param_tol=1e-2)


def test_front_tc_selects_the_wide_tensor_core_kernel(emu_engine):
    from oracle.qmix import QmixConfig, synth_batch
    lib = emu_engine.lib()
    cfg = QmixConfig(n_agents=2, obs_dim=80, act_dim=4, state_dim=10, gain=1.0)
    names = {}
    for opt in (0, 1):
        lib.mx_set_option(b"front_tc", opt)
        try:
            L, args, pol, tr = qc.oracle_and_trainer(cfg, 3, 2, debug=False)
            import ctypes as C
            lib.mx_profile_begin(None)
            tr.train_policy_on_batch(qc.ref_tuple(synth_batch(cfg, 3, 2, seed=1) + (None, None)))
            buf = C.create_string_buffer(8192)
            ms = (C.c_float * 128)()
            n = lib.mx_profile_end(None, buf, 8192, ms, 128)
            names[opt] = buf.value.decode().split(";")[:n]
        finally:
            lib.mx_set_option(b"front_tc", 1)
    assert "k_front_fwd" in names[0] and "k_front_fwd_tc_wide" not in names[0]
    assert "k_front_fwd_tc_wide" in names[1] and "k_front_fwd" not in names[1] and "k_tc_prep_weights" in names[1]


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("name", ["qmix_small", "qmix_5ag", "qmix_small_prev_act", "qmix_small_per", "qmix_small_huber_nodq", "qmix_small_hyper1"])
def test_tensor_core_weight_gradients_match_reference_golden(emu_engine, name, mode):
    """Option wgrad_tc.  1: k_wgrad_tc produces every dW / db of the front layers and the GRU matrices, the LayerNorm gradients and the
    data-gradient chain still come from k_front_bwd.  2: k_front_bwd_tc (data-gradient chain + LayerNorm gradients on the tensor cores) replaces
    k_front_bwd altogether.  All gradient tensors against the reference's."""
    lib = emu_engine.lib()
    lib.mx_set_option(b"wgrad_tc", mode)
    try:
        qc.check_step_against(None, name, intermediates=False, debug=False)
    finally:
        lib.mx_set_option(b"wgrad_tc", -1)


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("B,T,N,obs", [(24, 5, 5, 30), (7, 9, 3, 64), (3, 2, 2, 17), (32, 12, 3, 30)])
def test_tensor_core_weight_gradients_vs_oracle(emu_engine, B, T, N, obs, mode):
    """Row counts that are not multiples of the 64-row chunks, more chunks than CTAs (several accumulation rounds per CTA) and fewer
    (CTAs without rows write zero partials), input widths up to 64."""
    from oracle.qmix import QmixConfig, synth_batch
    lib = emu_engine.lib()
    cfg = QmixConfig(n_agents=N, obs_dim=obs, act_dim=6, state_dim=20, gain=1.0)
    lib.mx_set_option(b"wgrad_tc", mode)
    try:
        L, args, pol, tr = qc.oracle_and_trainer(cfg, B, T, debug=False)
        batch = synth_batch(cfg, B, T, seed=4, avail_p=0.7, var_len=True) + (None, None)
        qc.compare_step(L, pol, tr, batch, cfg, steps=2, param_tol=1e-2)
    finally:
        lib.mx_set_option(b"wgrad_tc", -1)


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("name", ["mqmix_small", "mqmix_small_per_huber_nodq", "mqmix_small_noavail"])
def test_tensor_core_backward_mlp_variant_matches_reference_golden(emu_engine, name, mode):
    """The MLP (transition-level) learner through the tensor-core backward: no recurrent matrix -- its slots of the gradient partials are
    never written and stay zero (mqmix_checks asserts that the unused slots of the parameter vector do not move)."""
    import mqmix_checks as mc
    lib = emu_engine.lib()
    lib.mx_set_option(b"wgrad_tc", mode)
    try:
        mc.check_golden(name, debug=False)
        mc.check_vs_oracle(B=200, steps=1, avail=True)        # 1 200 rows: more 64-row chunks than the emulator's 4 "SMs"
    finally:
        lib.mx_set_option(b"wgrad_tc", -1)


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("obs_dim", [65, 80, 96, 112, 128])
def test_tensor_core_backward_wide_inputs_vs_oracle(emu_engine, obs_dim, mode):
    """64 < obs_dim <= 128 through the tensor-core backward (fc1's transposed weight image takes turns with fc2's in shared memory, the
    feature LayerNorm's gradients are summed in two 64-column rounds, dW1 is read from two 64-column blocks of the accumulator), together with the
    wide forward kernel."""
    from oracle.qmix import QmixConfig, synth_batch
    lib = emu_engine.lib()
    cfg = QmixConfig(n_agents=5, obs_dim=obs_dim, act_dim=6, state_dim=20, gain=1.0)
    B, T = 24, 5           # 720 rows: 6 tiles / 12 chunks on the emulator's 4 "SMs"
    lib.mx_set_option(b"wgrad_tc", mode)
    try:
        L, args, pol, tr = qc.oracle_and_trainer(cfg, B, T, debug=False)
        batch = synth_batch(cfg, B, T, seed=4, avail_p=0.7, var_len=True) + (None, None)
        qc.compare_step(L, pol, tr, batch, cfg, steps=2, param_tol=1e-2)
    finally:
        lib.mx_set_option(b"wgrad_tc", -1)


def test_config2_full_size_all_tensor_core_kernels_vs_oracle(emu_engine):
    """BASELINE config 2 at its real size (B = 32, T = 60, N = 3: 5 856 agent-net rows = 46 tiles / 92 chunks) with every tensor-core
    kernel on: k_front_fwd_tc, k_front_bwd_tc, k_wgrad_tc."""
    from oracle.qmix import QmixConfig, synth_batch
    import torch
    lib = emu_engine.lib()
    torch.set_num_threads(4)
    cfg = QmixConfig(gain=1.0)
    lib.mx_set_option(b"wgrad_tc", 2)
    try:
        L, args, pol, tr = qc.oracle_and_trainer(cfg, 32, 60, debug=False)
        batch = synth_batch(cfg, 32, 60, seed=5, avail_p=0.8, var_len=True) + (None, None)
        qc.compare_step(L, pol, tr, batch, cfg, steps=1, param_tol=1e-2)
    finally:
        lib.mx_set_option(b"wgrad_tc", -1)
        torch.set_num_threads(1)


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("name", ["maddpg_box", "matd3_box", "maddpg_disc", "matd3_disc_avail", "maddpg_box_per", "matd3_disc_nofn", "maddpg_box_tanh"])
def test_maddpg_updates_through_the_tensor_core_backward(emu_engine, name, mode):
    """R-MADDPG / R-MATD3: the critic's (input 60 / 69 wide) and the actor's (18 wide) weight-gradient passes on k_wgrad_tc /
    k_front_bwd_tc; the frozen-critic pass that only needs the action gradient stays on k_front_bwd.  R-MADDPG passes no side array for
    the LayerNorm sums, so mode 2 runs k_front_bwd_tc with resident weights for inputs up to 64 (actor, Box critic) and 65 .. 128
    (Discrete critic)."""
    import maddpg_checks as mc
    lib = emu_engine.lib()
    lib.mx_set_option(b"wgrad_tc", mode)
    try:
        mc.check_golden(name)
    finally:
        lib.mx_set_option(b"wgrad_tc", -1)
