"""Wide-state QMIX mixer on the H100 at SMAC global-all-local shapes (every agent's observation appended to the global state).

train_smac_qmix.sh runs 3s5z_vs_3s6z with --use_global_all_local_state: N = 8, obs 268, 15 actions, state 230 + 8 x 268 = 2 374,
episode length 170, batch 32.  The shared-memory hypernet tile cannot hold such a state; the learner takes the wide-state path
(tensor-core state layers, csrc/mixer_wide.cu).  Checked against the oracle in lock-step, and graph replay against eager steps."""
import numpy as np
import pytest
import torch

import mqmix_checks as mc
import qmix_checks as qc
import qmix_wide_fixture as wf
import replay_checks as rc
from helpers import rel_err

pytestmark = pytest.mark.gpu

SHAPES = {      # N, obs, actions, state, episode length (get_obs_size / get_state_size of the SMAC env with this fork's defaults)
    "3s5z_vs_3s6z_global": (8, 268, 15, 2374, 170),
    "8m_global": (8, 204, 14, 1800, 120),
}


@pytest.mark.parametrize("debug", [True, False])
@pytest.mark.parametrize("name", ["qmix_wide_s448", "qmix_wide_s448_hyper1"])
def test_step_matches_wide_reference_fixture(gpu_engine, monkeypatch, name, debug):
    """The unmodified reference QMix at S = 448 (tests/golden/make_goldens_qmix_wide.py), in the debug configuration (separate
    head / core kernels, forward intermediates checked) and in the product configuration."""
    monkeypatch.setattr(qc, "load_golden", wf.load)
    qc.check_step_against(None, name, debug=debug)


def _cfg(name, **over):
    from oracle.qmix import QmixConfig
    N, O, A, S, _ = SHAPES[name]
    return QmixConfig(n_agents=N, obs_dim=O, act_dim=A, state_dim=S, gain=1.0, **over)


@pytest.mark.parametrize("name,steps", [("3s5z_vs_3s6z_global", 3), ("8m_global", 2)])
def test_smac_global_state_vs_oracle(gpu_engine, name, steps):
    """B = 32 with avail masks and variable episode lengths, consecutive steps (Adam state, soft update) in the product configuration."""
    from oracle.qmix import synth_batch
    torch.set_num_threads(8)
    cfg = _cfg(name)
    T = SHAPES[name][4]
    L, args, pol, tr = qc.oracle_and_trainer(cfg, 32, T, debug=False)
    assert tr.ws_view("hyp_pre").numel() > 0
    batch = synth_batch(cfg, 32, T, seed=5, avail_p=0.8, var_len=True) + (None, None)
    qc.compare_step(L, pol, tr, batch, cfg, steps=steps)


def test_smac_global_state_hyper1_per_huber_vs_oracle(gpu_engine):
    """1-layer hypernets (state -> N x mixer_hidden directly: 352 stacked GEMM columns per net), PER weights and Huber loss."""
    from oracle.qmix import synth_batch
    torch.set_num_threads(8)
    cfg = _cfg("8m_global", hyper_layers=1, use_per=True, huber=True, huber_delta=0.7)
    B, T = 16, 60
    L, args, pol, tr = qc.oracle_and_trainer(cfg, B, T, debug=False)
    w = np.random.RandomState(3).rand(B) * 0.9 + 0.1
    batch = synth_batch(cfg, B, T, seed=9, avail_p=0.7, var_len=True) + (w, np.arange(B))
    qc.compare_step(L, pol, tr, batch, cfg, steps=2)


def _filled_buffer(cfg, T, E, B, seed=0):
    rs = np.random.RandomState(seed)
    N, O, A, S = cfg.n_agents, cfg.obs_dim, cfg.act_dim, cfg.state_dim
    buf = rc.make_buffers(N, O, A, S, T, E, rng="device", max_batch=max(B, 64))
    for c in range(0, E, 8):
        n = min(8, E - c)
        av = (rs.rand(T + 1, n, N, A) < 0.7) * 1.0
        av[..., 0] = 1.0
        ep = [rs.randn(T + 1, n, N, O), np.repeat(rs.randn(T + 1, n, 1, S), N, 2), np.eye(A)[rs.randint(0, A, (T, n, N))],
              np.repeat(rs.randn(T, n, 1, 1), N, 2), np.zeros((T, n, N, 1)), np.zeros((T, n, 1)), av]
        buf.insert(n, *[rc.d(x.astype(np.float32)) for x in ep])
    return buf


def test_train_smac_qmix_shape_graph_replay_equals_eager(gpu_engine):
    """sample (device MT19937) -> step -> soft update at the train_smac_qmix.sh shape: eager drop-in calls against the oracle fed the same
    episodes, then the same sequence replayed from one captured CUDA graph leaves the same parameters."""
    from offpolicy._b200.graph import StepGraph
    torch.set_num_threads(8)
    cfg = _cfg("3s5z_vs_3s6z_global")
    T = SHAPES["3s5z_vs_3s6z_global"][4]
    B, E = 32, 48
    results = []
    for mode in ("eager", "graph"):
        torch.manual_seed(0)
        buf = _filled_buffer(cfg, T, E, B)
        L, args, pol, tr = qc.oracle_and_trainer(cfg, B, T, debug=False)
        buf.seed_device_rng(123)
        if mode == "eager":
            for s in range(3):
                smp = buf.sample(B)
                info, _, _ = tr.train_policy_on_batch(smp)
                tr.soft_target_updates()
                host = tuple(smp[i]["policy_0"] for i in range(7)) + (None, None)
                ref, _, _ = L.step(host)
                L.soft_update()
                assert rel_err(info["loss"].cpu(), ref["loss"]) < 1e-4
                assert rel_err(info["grad_norm"].cpu(), ref["grad_norm"]) < 1e-4
        else:
            torch.cuda.synchronize()
            g = StepGraph(buf, tr, B)
            for s in range(3):
                g.launch()
            g.synchronize()
            g.close()
        results.append((tr.theta.clone(), tr.theta_tgt.clone(), tr.adam_m.clone()))
    for a, b in zip(results[0], results[1]):
        assert float((a - b).abs().max()) <= 1e-6 * float(a.abs().max()) + 1e-7


def test_mqmix_wide_state_b1000_vs_oracle(gpu_engine):
    """Transition-level M-QMIX shares the mixer: B = 1 000 transitions at the 3s5z_vs_3s6z global-all-local state.  The state-layer
    pre-activations of the live net match fp64 to fp32 level with no sign flip; loss, grad_norm and Q_tot match the oracle to 1e-4 and
    every gradient tensor to 1e-3 relative L2.  (Element-wise the oracle's own fp32 rounding decides the side of a hypernet ReLU unit
    that lies within ~1e-5 of zero: at 192 000 hypernet units per step one such unit moves a few elements of its rows.)"""
    from oracle.qmix import QmixConfig, randomize_all
    from oracle.mqmix import MqmixLearner, synth_transitions
    from offpolicy._b200 import capi
    from offpolicy.algorithms.mqmix.algorithm.mQMixPolicy import M_QMixPolicy as Pol
    from offpolicy.algorithms.mqmix.mqmix import M_QMix as Tr
    torch.set_num_threads(8)
    N, O, A, S, B = 8, 268, 15, 2374, 1000
    cfg = QmixConfig(n_agents=N, obs_dim=O, act_dim=A, state_dim=S, gain=1.0)
    L = MqmixLearner(cfg, seed=3)
    randomize_all(L.agent, 1); randomize_all(L.mixer, 2)
    L.sync_targets()
    randomize_all(L.tgt_agent, 3, 0.05); randomize_all(L.tgt_mixer, 4, 0.05)
    args = qc.make_args(cfg, B)
    info = dict(obs_space=[O], share_obs_space=[S], act_space=rc.Discrete(A), cent_obs_dim=S, cent_act_dim=A * N)
    pol = Pol({"args": args, "device": capi.device()}, info)
    tr = Tr(args, N, {"policy_0": pol}, lambda a: "policy_0", device=capi.device())
    pol.q_network.load_state_dict(L.agent.state_dict()); tr.target_q_network.load_state_dict(L.tgt_agent.state_dict())
    tr.mixer.load_state_dict(L.mixer.state_dict()); tr.target_mixer.load_state_dict(L.tgt_mixer.state_dict())
    sd = {k: v.detach().double() for k, v in L.mixer.state_dict().items()}
    b = synth_transitions(cfg, B, seed=50, avail=True)
    info_t, _, _ = tr.train_policy_on_batch(mc._to_dicts(b, None), True)
    gv = {k: v.clone() for k, v in tr.grad_views().items()}
    pre = tr.ws_view("hyp_pre").double().cpu()
    pre = pre.view(2, B * 2, pre.numel() // (4 * B))
    X = torch.as_tensor(b[1], dtype=torch.float64)          # live rows: transition b = engine row 2 b
    col = 0
    for wk in ("hyper_w1.0", "hyper_w2.0", "hyper_b2.0", "hyper_b1"):
        W, bias = sd[wk + ".weight"], sd[wk + ".bias"]
        ref = X @ W.T + bias
        got = pre[0, 0::2, col:col + W.shape[0]]
        assert float((got - ref).abs().max()) < 2e-6 * float(ref.abs().max()), wk
        assert int(((got > 0) != (ref > 0)).sum()) == 0, wk
        col += (W.shape[0] + 3) // 4 * 4
    ref, _, _ = L.step(b + (None, None))
    for k in ("loss", "grad_norm", "Q_tot"):
        assert rel_err(info_t[k].cpu(), ref[k]) < 1e-4, (k, float(info_t[k]), float(ref[k]))
    coef = min(1.0, cfg.max_grad_norm / (float(ref["grad_norm"]) + 1e-6))
    named = dict(("agent." + k, p) for k, p in L.agent.named_parameters())
    named.update(("mixer." + k, p) for k, p in L.mixer.named_parameters())
    for k, p in named.items():
        if p.grad is None:
            continue
        a, r = (gv[k] * coef).detach().cpu().double().flatten(), p.grad.detach().double().flatten()
        if float(r.norm()) > 1e-6:
            assert float((a - r).norm() / r.norm()) < 1e-3, k
