"""QMIX learner parity on the real sm_100a kernels through the C-ABI: reference goldens, the oracle at the
BASELINE.json sizes, CUDA-graph replay, and size-independent properties."""
import ctypes as C

import numpy as np
import pytest
import torch

import qmix_checks as qc
import replay_checks as rc
from helpers import rel_err

pytestmark = pytest.mark.gpu

GOLDENS = ["qmix_small", "qmix_small_huber_nodq", "qmix_small_per", "qmix_small_hyper1", "qmix_5ag"]


@pytest.mark.parametrize("name", GOLDENS)
def test_step_matches_reference_golden(gpu_engine, name):
    qc.check_step_against(None, name)


@pytest.mark.parametrize("name", GOLDENS)
def test_product_configuration_matches_reference_golden(gpu_engine, name):
    """debug outputs off = what bench.py / the runner execute (k_mid between the recurrences, forked hypernet branch)."""
    qc.check_step_against(None, name, debug=False)


@pytest.mark.parametrize("mixer_hidden,hyper_hidden,n_agents,act_dim", [(48, 40, 4, 4), (64, 64, 2, 20), (20, 64, 8, 17)])
def test_product_configuration_shapes_vs_oracle(gpu_engine, mixer_hidden, hyper_hidden, n_agents, act_dim):
    from oracle.qmix import QmixConfig, synth_batch
    cfg = QmixConfig(n_agents=n_agents, obs_dim=7, act_dim=act_dim, state_dim=10, mixer_hidden=mixer_hidden, hyper_hidden=hyper_hidden,
                     gain=1.0, use_per=True, huber=True, huber_delta=0.7)
    B, T = 5, 6
    L, args, pol, tr = qc.oracle_and_trainer(cfg, B, T, debug=False)
    w = np.random.RandomState(3).rand(B) * 0.9 + 0.1
    batch = synth_batch(cfg, B, T, seed=9, avail_p=0.6, var_len=True) + (w, np.arange(B))
    qc.compare_step(L, pol, tr, batch, cfg, steps=2)


def test_config2_3m_full_size_product_configuration_vs_oracle(gpu_engine):
    """BASELINE config 2 exactly as benchmarked: 14-launch two-branch step with k_mid, three consecutive steps."""
    from oracle.qmix import QmixConfig, synth_batch
    torch.set_num_threads(8)
    cfg = QmixConfig(gain=1.0)
    L, args, pol, tr = qc.oracle_and_trainer(cfg, 32, 60, debug=False)
    batch = synth_batch(cfg, 32, 60, seed=5, avail_p=0.8, var_len=True) + (None, None)
    qc.compare_step(L, pol, tr, batch, cfg, steps=3)


_oracle_and_trainer = qc.oracle_and_trainer
_compare_step = qc.compare_step


def test_config2_3m_full_size_vs_oracle(gpu_engine):
    """BASELINE config 2: QMIX 3m shapes, B=32, T=60 -- three consecutive steps (Adam state, Polyak)."""
    from oracle.qmix import QmixConfig, synth_batch
    torch.set_num_threads(8)
    cfg = QmixConfig(gain=1.0)
    L, args, pol, tr = _oracle_and_trainer(cfg, 32, 60)
    batch = synth_batch(cfg, 32, 60, seed=5, avail_p=0.8, var_len=True) + (None, None)
    _compare_step(L, pol, tr, batch, cfg, steps=3)


def test_config4_8m_per_full_size_vs_oracle(gpu_engine):
    """BASELINE config 4: 8 agents, obs 80, A=14, S=168, T=120, B=64 with PER weights and priorities."""
    from oracle.qmix import QmixConfig, synth_batch
    torch.set_num_threads(8)
    cfg = QmixConfig(n_agents=8, obs_dim=80, act_dim=14, state_dim=168, use_per=True)
    L, args, pol, tr = _oracle_and_trainer(cfg, 64, 120)
    w = (np.random.RandomState(2).rand(64) * 0.9 + 0.1)
    batch = synth_batch(cfg, 64, 120, seed=6, avail_p=0.8, var_len=True) + (w, np.arange(64))
    _compare_step(L, pol, tr, batch, cfg, steps=1)


def test_config5_2s3z_vs_oracle(gpu_engine):
    from oracle.qmix import QmixConfig, synth_batch
    torch.set_num_threads(8)
    cfg = QmixConfig(n_agents=5, obs_dim=80, act_dim=11, state_dim=120)
    L, args, pol, tr = _oracle_and_trainer(cfg, 32, 120)
    batch = synth_batch(cfg, 32, 120, seed=7, avail_p=0.8, var_len=False) + (None, None)
    _compare_step(L, pol, tr, batch, cfg, steps=1)


def test_two_learners_on_two_streams_vs_oracle(gpu_engine):
    """Two learners whose steps run at the same time on two streams (2s3z sizes: every tensor-core kernel of the forward, the
    data-gradient chain and the weight gradients): each handle's accumulators are its own, both match their oracle."""
    from oracle.qmix import QmixConfig, synth_batch
    torch.set_num_threads(8)
    cfg = QmixConfig(n_agents=5, obs_dim=80, act_dim=11, state_dim=120)
    runs = []
    for seed in (7, 6):          # two different batches, each within the one-step Adam parameter tolerance on its own
        L, args, pol, tr = _oracle_and_trainer(cfg, 32, 120)
        runs.append((L, pol, tr, synth_batch(cfg, 32, 120, seed=seed, avail_p=0.8, var_len=False) + (None, None)))
    dev = torch.device("cuda", 0)
    streams = [torch.cuda.Stream(device=dev) for _ in runs]
    for st in streams:
        st.wait_stream(torch.cuda.current_stream(dev))
    outs = []
    for (L, pol, tr, batch), st in zip(runs, streams):
        with torch.cuda.stream(st):
            outs.append(tr.train_policy_on_batch(qc.ref_tuple(batch)))
    torch.cuda.synchronize()
    for (L, pol, tr, batch), (info, prio, _) in zip(runs, outs):
        gv = {k: v.clone() for k, v in tr.grad_views().items()}
        qc.check_engine_step(L, pol, tr, batch, cfg, info, prio, gv)


@pytest.mark.parametrize("mode", ["forked", "fused"])
def test_config5_2s3z_branch_modes_vs_oracle(gpu_engine, mode):
    """2s3z sizes with the forked branch forced on (split mixer beside the agent nets; the default at this size is the in-line
    fused k_mixer) and forced off: both against the oracle."""
    from oracle.qmix import QmixConfig, synth_batch
    torch.set_num_threads(8)
    lib = gpu_engine.lib()
    lib.mx_set_option(b"overlap", 2 if mode == "forked" else 0)
    try:
        cfg = QmixConfig(n_agents=5, obs_dim=80, act_dim=11, state_dim=120)
        L, args, pol, tr = _oracle_and_trainer(cfg, 32, 120)
        batch = synth_batch(cfg, 32, 120, seed=7, avail_p=0.8, var_len=False) + (None, None)
        _compare_step(L, pol, tr, batch, cfg, steps=1)      # (a second step would compare gradients at parameters that already differ by the Adam-step tolerance)
    finally:
        lib.mx_set_option(b"overlap", 1)


@pytest.mark.parametrize("mode", ["forked", "fused"])
@pytest.mark.parametrize("mixer_hidden,hyper_hidden,n_agents,layers", [(48, 40, 4, 2), (64, 64, 2, 1), (20, 64, 3, 2)])
def test_mixer_shapes_vs_oracle(gpu_engine, mode, mixer_hidden, hyper_hidden, n_agents, layers):
    from oracle.qmix import QmixConfig, synth_batch
    lib = gpu_engine.lib()
    cfg = QmixConfig(n_agents=n_agents, obs_dim=7, act_dim=4, state_dim=10, mixer_hidden=mixer_hidden, hyper_hidden=hyper_hidden,
                     hyper_layers=layers, gain=1.0, use_per=True, huber=True, huber_delta=0.7)
    B, T = 5, 6
    lib.mx_set_option(b"overlap", 2 if mode == "forked" else 0)
    try:
        L, args, pol, tr = _oracle_and_trainer(cfg, B, T)
        w = np.random.RandomState(3).rand(B) * 0.9 + 0.1
        batch = synth_batch(cfg, B, T, seed=9, avail_p=0.8, var_len=True) + (w, np.arange(B))
        _compare_step(L, pol, tr, batch, cfg, steps=2)
    finally:
        lib.mx_set_option(b"overlap", 1)


def test_vdn_vs_oracle(gpu_engine):
    """VDN = sum mixer (reference is shape-broken, App. D-1: pinned against the oracle's intent restatement)."""
    from oracle.qmix import QmixConfig, synth_batch
    cfg = QmixConfig(vdn=True)
    L, args, pol, tr = _oracle_and_trainer(cfg, 8, 20, vdn=True)
    batch = synth_batch(cfg, 8, 20, seed=8, avail_p=0.7, var_len=True) + (None, None)
    _compare_step(L, pol, tr, batch, cfg, steps=2)


def _filled_buffer(cfg, T, E, B, per=False, seed=0):
    rs = np.random.RandomState(seed)
    N, O, A, S = cfg.n_agents, cfg.obs_dim, cfg.act_dim, cfg.state_dim
    buf = rc.make_buffers(N, O, A, S, T, E, per_alpha=0.6 if per else None, rng="device", max_batch=max(B, 64))
    for c in range(0, E, 64):
        n = min(64, E - c)
        ep = [rs.randn(T + 1, n, N, O), np.repeat(rs.randn(T + 1, n, 1, S), N, 2), np.eye(A)[rs.randint(0, A, (T, n, N))],
              np.repeat(rs.randn(T, n, 1, 1), N, 2), np.zeros((T, n, N, 1)), np.zeros((T, n, 1)), np.ones((T + 1, n, N, A))]
        buf.insert(n, *[rc.d(x.astype(np.float32)) for x in ep])
    return buf


def test_sample_train_end_to_end_and_graph_replay(gpu_engine):
    """sample (device MT19937) -> train -> soft update through the drop-in classes equals the oracle fed with the same
    indices; then the same sequence replayed from ONE captured CUDA graph gives the same parameters."""
    from oracle.qmix import QmixConfig
    capi = gpu_engine
    lib = capi.lib()
    cfg = QmixConfig(gain=1.0)
    B, T, E = 32, 60, 256
    results = []
    for mode in ("eager", "graph"):
        torch.manual_seed(0)
        buf = _filled_buffer(cfg, T, E, B)
        L, args, pol, tr = _oracle_and_trainer(cfg, B, T)
        buf.seed_device_rng(123)
        np.random.seed(123)
        pb = buf.policy_buffers["policy_0"]
        if mode == "eager":
            for s in range(4):
                smp = buf.sample(B)
                idx = np.asarray(pb.sampled_indices(B))
                assert np.array_equal(idx, np.random.choice(E, B))
                info, _, _ = tr.train_policy_on_batch(smp)
                tr.soft_target_updates()
                host = tuple(smp[i]["policy_0"] for i in range(7)) + (None, None)
                ref, _, _ = L.step(host)
                L.soft_update()
                assert rel_err(info["loss"].cpu(), ref["loss"]) < 1e-4
                assert rel_err(info["grad_norm"].cpu(), ref["grad_norm"]) < 1e-4
        else:
            from offpolicy._b200.graph import StepGraph
            torch.cuda.synchronize()
            g = StepGraph(buf, tr, B)
            assert g.num_kernels >= 10
            for s in range(4):
                g.launch()
            g.synchronize()
            g.close()
        results.append((tr.theta.clone(), tr.theta_tgt.clone(), tr.adam_m.clone()))
    # same kernels, same order (the step is deterministic since r01m; the bound predates that and is kept loose on purpose)
    for a, b in zip(results[0], results[1]):
        assert float((a - b).abs().max()) <= 1e-6 * float(a.abs().max()) + 1e-7


def test_size_independent_properties_full_size(gpu_engine):
    """At config-2 size: (1) permuting the episodes of a batch leaves loss / grad_norm unchanged (summation order only);
    (2) soft update with tau=1 equals a hard update; (3) hard update is idempotent; (4) lr=0 leaves parameters bit-identical."""
    from oracle.qmix import QmixConfig, synth_batch
    cfg = QmixConfig(gain=1.0)
    B, T = 32, 60
    batch = synth_batch(cfg, B, T, seed=21, avail_p=0.8, var_len=True)
    perm = np.random.RandomState(0).permutation(B)
    pbatch = tuple(x[..., perm, :] if x.ndim == 4 else x[:, perm] for x in batch)
    outs = []
    for bt in (batch, pbatch):
        L, args, pol, tr = _oracle_and_trainer(cfg, B, T)
        info, _, _ = tr.train_policy_on_batch(qc.ref_tuple(bt + (None, None)))
        outs.append((float(info["loss"]), float(info["grad_norm"]), float(info["Q_tot"])))
    for a, b in zip(*outs):
        assert abs(a - b) <= 2e-5 * abs(a)
    L, args, pol, tr = _oracle_and_trainer(cfg, B, T, tau=1.0)
    tr.soft_target_updates()
    assert torch.equal(tr.theta, tr.theta_tgt)
    tr.hard_target_updates()
    tr.hard_target_updates()
    assert torch.equal(tr.theta, tr.theta_tgt)
    L, args, pol, tr = _oracle_and_trainer(cfg, B, T, lr=0.0)
    before = tr.theta.clone()
    tr.train_policy_on_batch(qc.ref_tuple(batch + (None, None)))
    assert torch.equal(before, tr.theta)


def test_error_behaviour(gpu_engine):
    """Errors surface as exceptions like the reference's asserts (rec_buffer.py:287-289; qmix needs H=64)."""
    from oracle.qmix import QmixConfig
    from offpolicy._b200.capi import MxError
    cfg = QmixConfig()
    buf = _filled_buffer(cfg, 4, 8, 4, per=True)
    with pytest.raises(AssertionError):
        buf.sample(8, 0.4, "policy_0")          # len(self) > batch_size
    with pytest.raises(AssertionError):
        buf.sample(4, 0.0, "policy_0")          # beta > 0
    with pytest.raises(AssertionError):
        buf.update_priorities(np.array([0, 1]), np.array([1.0, -1.0], np.float32), "policy_0")
    with pytest.raises(MxError):
        qc.build_trainer(QmixConfig(hidden=128), 4, 4)


# ---------------------------------------------------------------------------------------------------------------
# recurrent MADDPG / MATD3 (BASELINE config 3)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["maddpg_box", "matd3_box", "maddpg_box_per", "maddpg_disc", "matd3_disc", "matd3_disc_avail"])
def test_maddpg_matches_reference_golden(gpu_engine, name):
    import maddpg_checks as mc
    mc.check_golden(name)


@pytest.mark.parametrize("td3", [False, True])
def test_config3_maddpg_spread_full_size_vs_oracle(gpu_engine, td3):
    """BASELINE config 3: R-MADDPG / R-MATD3, MPE simple_spread shapes (N=3, obs 18, state 54, T=25, B=32), Box(2) actions;
    three consecutive updates against the pinned oracle (critic + actor losses, grad norms, all four networks)."""
    import maddpg_checks as mc
    from oracle.maddpg import MaddpgConfig, MaddpgLearner, synth_batch_cont
    from oracle.qmix import randomize_all
    torch.set_num_threads(8)
    cfg = MaddpgConfig(td3=td3, actor_update_interval=2 if td3 else 1, gain=1.0)
    B, T = 32, 25
    L = MaddpgLearner(cfg, seed=5)
    randomize_all(L.actor, 1); randomize_all(L.critic, 2)
    L.sync_targets()
    randomize_all(L.tgt_actor, 3, 0.05); randomize_all(L.tgt_critic, 4, 0.05)
    args, pol, tr = mc.build(cfg, B, T)
    for ours, ref in ((pol.actor, L.actor), (pol.critic, L.critic), (pol.target_actor, L.tgt_actor), (pol.target_critic, L.tgt_critic)):
        ours.load_state_dict(ref.state_dict())
    for s in range(3):
        batch = synth_batch_cont(cfg, B, T, seed=40 + s) + (None, None)
        torch.manual_seed(77 + s)
        noise = torch.empty(T + 1, cfg.n_agents * B, cfg.act_dim).normal_(mean=0, std=cfg.target_noise).numpy() if td3 else None
        torch.manual_seed(77 + s)
        info, _, _ = tr.shared_train_policy_on_batch("policy_0", mc.ref_tuple(batch))
        ref, _ = L.step(batch, noise)
        assert rel_err(info["critic_loss"].cpu(), ref["critic_loss"]) < 1e-4
        assert rel_err(info["critic_grad_norm"].cpu(), ref["critic_grad_norm"]) < 1e-4
        assert bool(info["update_actor"]) == bool(ref["update_actor"])
        if ref["update_actor"]:
            assert rel_err(info["actor_loss"].cpu(), ref["actor_loss"]) < 1e-4
            assert rel_err(info["actor_grad_norm"].cpu(), ref["actor_grad_norm"]) < 2e-4
            pol.soft_target_updates()
            L.soft_update()
    for ours, ref in ((pol.actor, L.actor), (pol.critic, L.critic), (pol.target_actor, L.tgt_actor), (pol.target_critic, L.tgt_critic)):
        for k, v in ours.state_dict().items():
            assert float((v.cpu() - ref.state_dict()[k]).abs().max()) <= 5e-3 * cfg.lr * 3 + 1e-7, k


@pytest.mark.parametrize("td3", [False, True])
def test_config3_maddpg_spread_discrete_full_size_vs_oracle(gpu_engine, td3):
    """MPE simple_spread's real action space is Discrete(5) (envs/mpe/environment.py:62-63): arg-max one-hot / hard Gumbel-softmax
    target actions and the straight-through Gumbel-softmax actor update, full size (N=3, T=25, B=32), vs the pinned oracle."""
    import maddpg_checks as mc
    from oracle.maddpg import MaddpgConfig, MaddpgLearner, synth_batch_disc, sample_gumbel
    from oracle.qmix import randomize_all
    torch.set_num_threads(8)
    cfg = MaddpgConfig(act_dim=5, discrete=True, td3=td3, actor_update_interval=2 if td3 else 1, gain=1.0)
    B, T = 32, 25
    L = MaddpgLearner(cfg, seed=5)
    randomize_all(L.actor, 1); randomize_all(L.critic, 2)
    L.sync_targets()
    randomize_all(L.tgt_actor, 3, 0.05); randomize_all(L.tgt_critic, 4, 0.05)
    args, pol, tr = mc.build(cfg, B, T)
    for ours, ref in ((pol.actor, L.actor), (pol.critic, L.critic), (pol.target_actor, L.tgt_actor), (pol.target_critic, L.tgt_critic)):
        ours.load_state_dict(ref.state_dict())
    for s in range(3):
        batch = synth_batch_disc(cfg, B, T, seed=40 + s) + (None, None)
        upd = s % cfg.actor_update_interval == 0
        torch.manual_seed(77 + s)
        noise = sample_gumbel((T + 1, cfg.n_agents * B, cfg.act_dim)).numpy() if td3 else None
        anoise = sample_gumbel((T, cfg.n_agents * B, cfg.act_dim)).numpy() if upd else None
        torch.manual_seed(77 + s)
        info, _, _ = tr.shared_train_policy_on_batch("policy_0", mc.ref_tuple(batch))
        ref, _ = L.step(batch, noise, anoise)
        assert rel_err(info["critic_loss"].cpu(), ref["critic_loss"]) < 1e-4
        assert rel_err(info["critic_grad_norm"].cpu(), ref["critic_grad_norm"]) < 1e-4
        assert bool(info["update_actor"]) == bool(ref["update_actor"]) == upd
        if ref["update_actor"]:
            assert rel_err(info["actor_loss"].cpu(), ref["actor_loss"]) < 1e-4
            assert rel_err(info["actor_grad_norm"].cpu(), ref["actor_grad_norm"]) < 2e-4
            pol.soft_target_updates()
            L.soft_update()
    for ours, ref in ((pol.actor, L.actor), (pol.critic, L.critic), (pol.target_actor, L.tgt_actor), (pol.target_critic, L.tgt_critic)):
        for k, v in ours.state_dict().items():
            assert float((v.cpu() - ref.state_dict()[k]).abs().max()) <= 5e-3 * cfg.lr * 3 + 1e-7, k


@pytest.mark.parametrize("name", ["maddpg_box", "maddpg_disc", "matd3_disc"])
def test_maddpg_rollout_actions_match_reference(gpu_engine, name):
    import maddpg_checks as mc
    mc.check_get_actions(name)


@pytest.mark.parametrize("td3,disc", [(False, False), (True, False), (False, True), (True, True)])
def test_maddpg_whole_update_graph_matches_eager(gpu_engine, td3, disc):
    import maddpg_checks as mc
    mc.check_graph_matches_eager(td3, disc, B=32, T=25, E=64, steps=4)


def test_maddpg_replay_batch_equals_host_batch_odd_episode_length(gpu_engine):
    import maddpg_checks as mc
    mc.check_replay_batch_equals_host_batch()


def test_mpe_shapes_without_avail_masks(gpu_engine):
    """BASELINE configs[0] shapes (train_mpe_qmix.sh): T = 25, 3 agents -> padded episode rows in the batch region, no avail masks,
    reward normalisation."""
    qc.check_mpe_shapes_without_avail_masks()
