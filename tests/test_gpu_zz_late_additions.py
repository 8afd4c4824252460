"""GPU parity tests for features that were finished after the round's last GPU visit (emulator-verified only so far).  The file
name sorts last on purpose: `pytest -x` reaches these after every test that has already been seen green on a B200."""
import pytest

import qmix_checks as qc

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("debug", [True, False])
def test_prev_act_inp_matches_reference_golden(gpu_engine, debug):
    """--prev_act_inp: input width 30 + 9 = 39 (tensor-core front kernel with K padded to 40)."""
    qc.check_step_against(None, "qmix_small_prev_act", intermediates=False, debug=debug)


@pytest.mark.parametrize("debug", [True, False])
@pytest.mark.parametrize("name", ["mqmix_small", "mqmix_small_per_huber_nodq", "mqmix_small_noavail"])
def test_mqmix_matches_reference_golden(gpu_engine, name, debug):
    """MLP (transition-level) QMIX, SURVEY.md section 8(f).4 first slice."""
    import mqmix_checks as mc
    mc.check_golden(name, debug)


def test_mlp_buffer_sample_layout(gpu_engine):
    import mqmix_checks as mc
    mc.check_buffer_vs_reference_layout()


@pytest.mark.parametrize("kw", [dict(B=1000), dict(B=1000, avail=True, per=True, huber=True), dict(B=256, avail=True, double_q=False), dict(B=1000, vdn=True),
                                dict(B=320, hyper_layers=1, N=5, O=80, A=11, S=120)],
                         ids=["mpe_b1000", "avail_per_huber", "avail_nodq", "vdn", "hyper1_2s3z_shapes"])
def test_mlp_learner_vs_oracle(gpu_engine, kw):
    """scripts/train_mpe_mqmix.sh sizes (batch 1000 transitions) in lock-step with the pinned oracle (oracle/mqmix.py); obs 80 takes the
    FFMA front kernel (obs_dim > 64), obs 18 the tensor-core one."""
    import mqmix_checks as mc
    mc.check_vs_oracle(steps=2, **kw)


def test_mlp_buffer_vs_reference_golden(gpu_engine):
    import mqmix_checks as mc
    mc.check_buffer_vs_reference_golden()


@pytest.mark.parametrize("per", [False, True], ids=["uniform", "per"])
def test_mlp_step_graph_vs_eager(gpu_engine, per):
    import mqmix_checks as mc
    mc.check_step_graph_vs_eager(per=per, B=1000, E=4096)


def test_c_host_example_runs(gpu_engine, tmp_path):
    """examples/c_host.c: the C-ABI driven from plain C (cudaMalloc'd buffers, no Python / torch in the process)."""
    import subprocess
    from test_c_host_example import build_c_host
    exe = build_c_host(str(tmp_path / "c_host"))
    r = subprocess.run([exe, "4"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("step ")]
    assert len(lines) == 4 and r.stdout.strip().splitlines()[-1].startswith("ok"), r.stdout


@pytest.mark.parametrize("front_tc", [1, 0])
@pytest.mark.parametrize("name", ["qmix_small_nofn", "qmix_small_tanh"])
def test_network_structure_flags_match_reference_golden(gpu_engine, name, front_tc):
    """--use_feature_normalization / --use_ReLU switched off (store_false flags): no input LayerNorm, tanh blocks -- tensor-core and FFMA front."""
    lib = gpu_engine.lib()
    lib.mx_set_option(b"front_tc", front_tc)
    try:
        qc.check_step_against(None, name, intermediates=True, debug=True)
        qc.check_step_against(None, name, intermediates=False, debug=False)
    finally:
        lib.mx_set_option(b"front_tc", 1)


@pytest.mark.parametrize("name", ["mqmix_small_nofn", "mqmix_small_tanh"])
def test_network_structure_flags_mlp(gpu_engine, name):
    import mqmix_checks as mc
    mc.check_golden(name, debug=False)          # includes the rollout surface (k_policy_step with the same flags)


@pytest.mark.parametrize("name", ["matd3_disc_nofn", "maddpg_box_tanh"])
def test_network_structure_flags_maddpg(gpu_engine, name):
    import maddpg_checks as mdc
    mdc.check_golden(name)
    mdc.check_get_actions(name)


# ---- option-gated tensor-core kernels written without a GPU (off by default): last, so that a failure here hides nothing else ----

@pytest.mark.parametrize("obs_dim,n_agents,B,T", [(80, 8, 8, 20), (128, 3, 16, 12), (72, 5, 32, 10)])
def test_wide_input_tensor_core_front_kernel_vs_oracle(gpu_engine, obs_dim, n_agents, B, T):
    """k_front_fwd_tc_wide (64 < obs_dim <= 128, option front_tc_wide, off by default until timed): emulator-verified indexing; this is its
    first run on real tensor cores.  Runs under a launch-count check that the wide kernel, not the FFMA one, executed."""
    import ctypes as C
    import numpy as np
    from oracle.qmix import QmixConfig, synth_batch
    lib = gpu_engine.lib()
    cfg = QmixConfig(n_agents=n_agents, obs_dim=obs_dim, act_dim=7, state_dim=40, gain=1.0)
    lib.mx_set_option(b"front_tc_wide", 1)
    try:
        L, args, pol, tr = qc.oracle_and_trainer(cfg, B, T, debug=False)
        tr.use_step_graph = False
        batch = synth_batch(cfg, B, T, seed=4, avail_p=0.7, var_len=True) + (None, None)
        lib.mx_profile_begin(gpu_engine.stream_ptr())
        qc.compare_step(L, pol, tr, batch, cfg, steps=1, param_tol=1e-2)
        buf = C.create_string_buffer(8192)
        ms = (C.c_float * 256)()
        n = lib.mx_profile_end(gpu_engine.stream_ptr(), buf, 8192, ms, 256)
        assert "k_front_fwd_tc_wide" in buf.value.decode().split(";")[:n]
        qc.compare_step(L, pol, tr, batch, cfg, steps=2, param_tol=1e-2)
    finally:
        lib.mx_set_option(b"front_tc_wide", 1)


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("name", ["qmix_small", "qmix_5ag", "qmix_small_per"])
def test_tensor_core_weight_gradients_match_reference_golden(gpu_engine, name, mode):
    """Option wgrad_tc (off by default until timed).  1: k_wgrad_tc -- dW / db of the front layers and the GRU matrices on the tensor cores with
    transposed operand staging, beside k_front_bwd's data-gradient chain.  2: k_front_bwd_tc replaces k_front_bwd as well.
    Emulator-verified indexing; first run on real tensor cores here."""
    lib = gpu_engine.lib()
    lib.mx_set_option(b"wgrad_tc", mode)
    try:
        qc.check_step_against(None, name, intermediates=False, debug=False)
    finally:
        lib.mx_set_option(b"wgrad_tc", -1)


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("B,T,N,obs", [(32, 60, 3, 30), (24, 5, 5, 30), (3, 2, 2, 17)])
def test_tensor_core_weight_gradients_vs_oracle(gpu_engine, B, T, N, obs, mode):
    """BASELINE config-2 size (5 856 rows = 92 chunks on 122 CTAs), several chunks per CTA, fewer chunks than CTAs."""
    from oracle.qmix import QmixConfig, synth_batch
    lib = gpu_engine.lib()
    cfg = QmixConfig(n_agents=N, obs_dim=obs, act_dim=9, state_dim=48, gain=1.0)
    lib.mx_set_option(b"wgrad_tc", mode)
    try:
        L, args, pol, tr = qc.oracle_and_trainer(cfg, B, T, debug=False)
        tr.use_step_graph = False
        batch = synth_batch(cfg, B, T, seed=4, avail_p=0.7, var_len=True) + (None, None)
        qc.compare_step(L, pol, tr, batch, cfg, steps=2, param_tol=1e-2)
    finally:
        lib.mx_set_option(b"wgrad_tc", -1)


@pytest.mark.parametrize("mode", [1, 2])
def test_tensor_core_backward_mlp_variant(gpu_engine, mode):
    """M_QMix (1 000 transitions = 6 000 agent-net rows) through k_wgrad_tc / k_front_bwd_tc."""
    import mqmix_checks as mc
    lib = gpu_engine.lib()
    lib.mx_set_option(b"wgrad_tc", mode)
    try:
        mc.check_golden("mqmix_small", debug=False)
        mc.check_vs_oracle(B=1000, steps=2, avail=True)
    finally:
        lib.mx_set_option(b"wgrad_tc", -1)


@pytest.mark.parametrize("obs_dim,n_agents,B,T,mode", [(80, 8, 8, 20, 2), (80, 5, 32, 30, 1), (128, 3, 16, 12, 2)])
def test_tensor_core_backward_wide_inputs_vs_oracle(gpu_engine, obs_dim, n_agents, B, T, mode):
    """SMAC-sized observations (8m / 2s3z: 80) through the wide tensor-core forward AND backward kernels."""
    from oracle.qmix import QmixConfig, synth_batch
    lib = gpu_engine.lib()
    cfg = QmixConfig(n_agents=n_agents, obs_dim=obs_dim, act_dim=11, state_dim=60, gain=1.0)
    lib.mx_set_option(b"front_tc_wide", 1)
    lib.mx_set_option(b"wgrad_tc", mode)
    try:
        L, args, pol, tr = qc.oracle_and_trainer(cfg, B, T, debug=False)
        tr.use_step_graph = False
        batch = synth_batch(cfg, B, T, seed=4, avail_p=0.7, var_len=True) + (None, None)
        qc.compare_step(L, pol, tr, batch, cfg, steps=2, param_tol=1e-2)
    finally:
        lib.mx_set_option(b"wgrad_tc", -1)
        lib.mx_set_option(b"front_tc_wide", 1)


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("name", ["maddpg_box", "matd3_disc_avail"])
def test_maddpg_updates_through_the_tensor_core_backward(gpu_engine, name, mode):
    import maddpg_checks as mc
    lib = gpu_engine.lib()
    lib.mx_set_option(b"front_tc_wide", 1)
    lib.mx_set_option(b"wgrad_tc", mode)
    try:
        mc.check_golden(name)
    finally:
        lib.mx_set_option(b"wgrad_tc", -1)
        lib.mx_set_option(b"front_tc_wide", 1)


@pytest.mark.parametrize("name", ["maddpg_multi_disc", "matd3_multi_box", "matd3_multi_disc"])
def test_per_agent_policies_match_reference_golden(gpu_engine, name):
    """share_policy = False (scripts/train_mpe_rmaddpg.sh:14 -> train/train_mpe.py:139-150): one policy per agent with its own observation /
    action widths; every policy's target actor feeds the centralised action vectors (mx_maddpg_cent_contribute)."""
    import maddpg_checks as mdc
    mdc.check_multi_golden(name)


def test_per_agent_policies_through_the_multi_policy_buffer(gpu_engine):
    import maddpg_checks as mdc
    mdc.check_multi_golden("maddpg_multi_disc", through_buffer=True)


@pytest.mark.parametrize("ll", [1, 0])
def test_dead_peer_aborts_the_update_and_the_host_raises(gpu_engine, ll):
    """ADVICE (round 1): a rank whose peer never delivers must not apply an update from stale or partial sums.  One GPU is enough to
    show it: a world-2 learner is given its own symmetric block plus a second local block that nobody ever writes (the "peer" that
    died).  With the wait shortened to 30 ms (option p2p_timeout_ms; 10 s in production) the step must end with info[7] = -1,
    parameters, targets and Adam state untouched, and the NEXT train call must raise (QMix._check_exchange).  Both exchange protocols."""
    import time
    import torch
    from helpers import load_golden, oracle_from_golden, golden_batch, sub
    capi = gpu_engine
    lib = capi.lib()
    g = load_golden("qmix_small")
    L, cfg, B, T, steps = oracle_from_golden(g)
    lib.mx_set_option(b"p2p_timeout_ms", 30)
    lib.mx_set_option(b"p2p_ll", ll)
    try:
        args, pol, tr = qc.build_trainer(cfg, B, T, debug=False, dp_world_size=2)
        qc.load_state(pol, tr, sub(g, "init.agent."), sub(g, "init.mixer."), sub(g, "init.tgt_agent."), sub(g, "init.tgt_mixer."))
        n = int(lib.mx_qmix_p2p_block_bytes(tr.handle)) // 4
        blocks = [torch.zeros(n, dtype=torch.float32, device=tr.dev) for _ in range(2)]
        tr.attach_peer_blocks(0, [b.data_ptr() for b in blocks], keep=blocks)
        tr.use_step_graph = False
        before = [t.clone() for t in (tr.theta, tr.theta_tgt, tr.adam_m, tr.adam_v)]
        t_before = tr.ws_view("adam_t", torch.float64).clone()
        batch = golden_batch(g, 0)
        t0 = time.time()
        tr.train_policy_on_batch(qc.ref_tuple(batch))
        torch.cuda.synchronize()
        assert time.time() - t0 < 5.0                                        # the shortened wait, not the 10 s default
        assert float(tr._info[7]) == -1.0
        for a, b in zip(before, (tr.theta, tr.theta_tgt, tr.adam_m, tr.adam_v)):
            assert torch.equal(a, b)                                          # nothing was applied
        assert torch.equal(t_before, tr.ws_view("adam_t", torch.float64))
        with pytest.raises(RuntimeError, match="did not deliver"):
            for _ in range(3):                                                # the mirrored flag is read one step late, without a sync
                tr.train_policy_on_batch(qc.ref_tuple(batch))
                torch.cuda.synchronize()
    finally:
        lib.mx_set_option(b"p2p_timeout_ms", 10000)
        lib.mx_set_option(b"p2p_ll", 1)
