"""The QMIX learner at SMAC's real widths on the H100's own grid, against the float64 oracle: the same checks as
tests/test_emu_smac_widths.py (inputs above 128 columns, 9 to 32 agents, the input width refused at creation), with the edge shapes taken
from this device's SM count, and the 27m_vs_30m shape over two steps."""
import ctypes as C

import numpy as np
import pytest
import torch

import kink
import row_coverage_checks as rc
import test_emu_smac_widths as ew

pytestmark = pytest.mark.gpu


@pytest.fixture
def oracle_threads():
    n = torch.get_num_threads()
    torch.set_num_threads(8)
    yield
    torch.set_num_threads(n)


def _rules():
    return rc.TileRules(torch.cuda.get_device_properties(0).multi_processor_count)


@pytest.mark.parametrize("case", ew._boundary_cases(), ids=lambda c: c[0])
def test_kernels_on_each_side_of_each_boundary(gpu_engine, case):
    """As on the emulator, through the device launchers (whose shared-memory checks the emulator skips): 384 columns launch."""
    name, kw, B, T, debug, want, not_want = case
    kw = dict(kw)
    cfg = ew.cfg_of(kw.pop("obs"), kw.pop("act"), kw.pop("N"), **kw)
    names = ew.step_kernels(gpu_engine, cfg, B, T, debug, stream=gpu_engine.stream_ptr())
    rc.assert_kernels_ran(names, want)
    assert not [k for k in not_want if k in names], (name, not_want, names)


@pytest.mark.parametrize("N,A", [(6, 14), (7, 14), (17, 18), (18, 18), (10, 36), (11, 36)])
def test_mid_warps_on_each_side_of_each_boundary(gpu_engine, N, A):
    """k_mid's warp count (template argument W of k_mid<W, actions per lane>) in one captured product step, against mid_warps: 16 warps
    at N 6 and 8 at N 7 with 14 actions, 8 at N 17 and none at N 18 with 18 actions, 8 at N 10 and none at N 11 with 36."""
    import contextlib
    import io
    from oracle.qmix import synth_batch
    from offpolicy._b200 import capi, factory
    import qmix_checks as qc
    from test_gpu_qmix_schedule import graph_structure
    B, T = 2, 9
    cfg = ew.cfg_of(11, A, N)
    with contextlib.redirect_stdout(io.StringIO()):
        args, pol, tr = factory.build_qmix(cfg, B, T, debug=False)
    batch = list(qc.ref_tuple(synth_batch(cfg, B, T, seed=5, avail_p=0.8, var_len=True) + (np.ones(B, np.float32), np.arange(B))))
    tr.train_policy_on_batch(batch)          # first launches (module loading, shared-memory attributes) outside the capture
    b = tr._device_batch(batch)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph(keep_graph=True)
    with torch.cuda.graph(g):
        capi.check(capi.lib().mx_qmix_step(tr.handle, C.byref(b), capi.stream_ptr()))
    try:
        nodes, _ = graph_structure(g.raw_cuda_graph())
    finally:
        g.reset()
        torch.cuda.synchronize()
    W = rc.mid_warps(N, A)
    mids = [n for n in nodes if n.startswith("k_mid")]
    want = ["k_mid<%d,%d>" % (W, 2 if A > 32 else 1)] if W else []
    print("N %d A %d: restated %d warps, captured %s" % (N, A, W, mids))
    assert mids == want, (N, A, mids, want)


def test_input_width_limit_refused_at_creation(gpu_engine):
    ew.test_input_width_limit_refused_at_creation(gpu_engine)


# every edge at the first FFMA width and at the widest; the tail and CTA edges at the SMAC widths
GPU_TARGETS = {129: None, 384: None}


def _wide_cases():
    if not torch.cuda.is_available():
        return [pytest.param(129, 1, 1, 1, "", id="no-device")]
    R = _rules()
    out = []
    for width in ew.WIDE:
        tgts = GPU_TARGETS.get(width, ew.TAIL_TARGETS)
        for tg, (B, T, N), lay, note in rc.pick_shapes(R, width, Ns=(3, 5, 8), Ts=range(8, 65), Bs=range(1, 130), targets=tgts):
            out.append(pytest.param(width, B, T, N, note, id="in%d-B%d-T%d-N%d-%s" % (width, B, T, N, "_".join(ew.TAGS[t] for t in tg))))
    return out


@pytest.mark.parametrize("width,B,T,N,note", _wide_cases())
def test_wide_input_isolated_episodes_and_rows(gpu_engine, oracle_threads, width, B, T, N, note):
    ew.run_wide(gpu_engine, width, B, T, N, note, stream=gpu_engine.stream_ptr(), rules=_rules(), every_up_to=8)


@pytest.mark.parametrize("obs,B", [(129, 65), (320, 65), (320, 2113)])
def test_mqmix_wide_input_isolated_transitions(gpu_engine, oracle_threads, obs, B):
    """M-QMIX at 129 and 320 columns; B = 2 113 is one past the mixer's 16 sms transitions on 132 SMs."""
    from oracle.mqmix import synth_transitions
    R = _rules()
    N = 3
    cfg = ew.cfg_of(obs, 6, N, S=14)
    L64, pol, tr = rc.mqmix_pair(cfg, B)
    batch = synth_transitions(cfg, B, seed=7, avail=True) + (None, None)
    TM, _, grid = R.agent_rows(2 * N * B, obs, gru_ext=False)["k_front_bwd"]
    eps = rc.sample_episodes(B, 1, N, TM, grid, every_up_to=8)
    names = rc.kernels_run(gpu_engine.lib(), gpu_engine.stream_ptr(), lambda: rc.isolated_episode_gradients(L64, tr, batch, eps[:1], B, 1, N, mlp=True,
                                                                                          ulps=rc.td_ulps(obs)))
    rc.assert_kernels_ran(names, ["k_front_fwd", "k_front_bwd", "k_mlp_dgi"])
    assert "k_gru_wgrad" not in names and not [n for n in names if "_tc" in n], names
    worst = rc.isolated_episode_gradients(L64, tr, batch, eps, B, 1, N, mlp=True, ulps=rc.td_ulps(obs))
    print("M-QMIX in_dim %d B %d: %d transitions isolated; worst gradient %.2e (bound %.0e)" % (obs, B, len(eps), max(worst.values()), rc.GRAD_TOL))


@pytest.mark.parametrize("key", list(ew.MANY))
def test_many_agents_isolated_rows_and_transitions(gpu_engine, oracle_threads, key):
    ew.run_many(gpu_engine, key, 4, 12, stream=gpu_engine.stream_ptr())


@pytest.mark.parametrize("N,S", [(27, 129), (32, 65), (32, 1170)])
def test_many_agents_wide_state(gpu_engine, oracle_threads, N, S):
    """The first wide state at 27 and 32 agents, and 32 agents with 1-layer hypernets at state 1 170 (stacked state layers of 32 x 32 +
    ... columns: k_mixw_fwd runs 9 column blocks)."""
    from oracle.qmix import synth_batch
    B, T = 4, 12
    cfg = ew.cfg_of(11, 31, N, S=S, hyper_layers=1 if S == 1170 else 2)
    L64, pol, tr = rc.qmix_pair(cfg, B, T, debug=True)
    batch = rc.last_episode_full_length(synth_batch(cfg, B, T, seed=5, avail_p=0.8, var_len=True) + (np.ones(B, np.float32), np.arange(B)))
    names = rc.kernels_run(gpu_engine.lib(), gpu_engine.stream_ptr(), lambda: rc.isolated_episode_gradients(L64, tr, batch, [0], B, T, N))
    rc.assert_kernels_ran(names, ["k_mixw_fwd", "k_mixw_wgrad"])
    worst = rc.isolated_episode_gradients(L64, tr, batch, list(range(B)), B, T, N)
    worst_t = rc.per_transition(L64, tr, batch, B, T, N, True)
    print("N %d S %d: worst gradient %.2e, worst transition %.2e" % (N, S, max(worst.values()), max(v for k, v in worst_t.items() if k != "greedy decided rows")))


@pytest.mark.parametrize("vdn", [False, True])
def test_mqmix_32_agents_isolated_transitions(gpu_engine, oracle_threads, vdn):
    from oracle.mqmix import synth_transitions
    N, B = 32, 40
    cfg = ew.cfg_of(20, 15, N, S=14, vdn=vdn)
    L64, pol, tr = rc.mqmix_pair(cfg, B)
    batch = synth_transitions(cfg, B, seed=7, avail=True) + (None, None)
    worst = rc.isolated_episode_gradients(L64, tr, batch, [0, 17, B - 1], B, 1, N, mlp=True)
    print("M-%s N 32 B %d: worst gradient %.2e (bound %.0e)" % ("VDN" if vdn else "QMIX", B, max(worst.values()), rc.GRAD_TOL))


@pytest.mark.parametrize("N,layers,S,B,T", ew.GEMM_CASES + [(32, 1, 1170, 3, 44), (8, 2, 2374, 40, 53)])
def test_state_gemms_every_block_vs_float64(gpu_engine, oracle_threads, N, layers, S, B, T):
    """As on the emulator, plus 32 agents with 1-layer hypernets at state 1 170 (1 024 + 32 + 64 + 32 stacked columns: nine full 128-column
    blocks) and 3s5z_vs_3s6z's global state at N 8 (S 2 374, 2 160 state rows, 2 120 elements)."""
    from oracle.qmix import synth_batch
    cfg = ew.cfg_of(11, 5, N, S=S, hyper_layers=layers)
    L64, pol, tr = rc.qmix_pair(cfg, B, T, debug=True)
    batch = synth_batch(cfg, B, T, seed=4, avail_p=0.8, var_len=True) + (np.ones(B, np.float32), np.arange(B))
    names = rc.kernels_run(gpu_engine.lib(), gpu_engine.stream_ptr(), lambda: tr.train_policy_on_batch(rc.qc.ref_tuple(batch)))
    rc.assert_kernels_ran(names, ["k_mixw_fwd", "k_mixw_wgrad"])
    worst = rc.state_gemm_blocks(L64, tr, batch, B, T)
    k = max(worst, key=worst.get)
    print("N %d layers %d S %d rows %d elements %d: worst %s %.2e (bound %.0e)" % (N, layers, S, B * (T + 1), B * T, k, worst[k], rc.GEMM_TOL))


def _rel_l2(a, b):
    return float((a - b).norm() / (b.norm() + 1e-300))


def test_27m_vs_30m_two_steps_against_float64(gpu_engine, oracle_threads):
    """27m_vs_30m (N 27, obs 285, 36 actions, state 1 170, T 180, B 32), product configuration, two steps on the same batch.  Each
    step's unclipped gradients are judged against float64 beside the fp32 oracle's; both oracles start each step from the engine's
    parameters, so the comparison is of one step's arithmetic, not of drift.  Per tensor the engine's relative L2 error against float64
    must stay within RATIO times the fp32 oracle's, or under FLOOR.

    Measured on an H100 SXM (132 SMs, default power limit), before resolving kinks: at step 2 mixer.hyper_w1.* were off by 2.1e-4 / 1.2e-4
    / 7.2e-5 (first weight / second weight / second bias), 170-280 times the fp32 oracle's error, every other tensor within 2.6x of it or
    under 2e-6.  The cause is one |.| kink: hyper_w1's output at (t 2, b 14, column 765) is 6.1e-9, 2.5e-9 of that transition's largest,
    and the engine's fp32 value has the other sign (tests/kink.py resolve_abs_kinks); flipping it in float64 moves the bias gradient at column 765 by 0.5024, the
    engine's difference there is 0.5022.  The agent's feature_norm / fc1 gradients at step 2 (7.1e-5, 3.8e-5 against float64) are the
    fp32 oracle's error to two digits: round-off of sums that cancel.  Every engine tensor also carries a common offset of about 1.3e-6
    at both steps, which FLOOR covers."""
    import qmix_checks as qc
    from oracle.qmix import QmixLearner, synth_batch
    from test_gpu_qmix_many_actions import _cfg27, T27
    RATIO, FLOOR = 4.0, 5e-6
    cfg = _cfg27()
    B = 32
    L, args, pol, tr = qc.oracle_and_trainer(cfg, B, T27, debug=False)
    tr.use_step_graph = False
    batch = synth_batch(cfg, B, T27, seed=5, avail_p=0.8, var_len=True) + (None, None)
    rows = []
    for s in range(2):
        nets = (pol.q_network, tr.mixer, tr.target_q_network, tr.target_mixer)
        L32, L64 = QmixLearner(cfg), QmixLearner(cfg, dtype=torch.float64)
        for LL in (L32, L64):
            for dst, src in zip((LL.agent, LL.mixer, LL.tgt_agent, LL.tgt_mixer), nets):
                dst.load_state_dict({k: v.detach().cpu() for k, v in src.state_dict().items()})
        tr.train_policy_on_batch(qc.ref_tuple(batch))
        gv = {k: v.detach().cpu().double() for k, v in tr.grad_views().items()}
        tr.soft_target_updates()
        L32.grads(batch)
        L64.grads(batch)
        g32 = dict(("agent." + k, p.grad) for k, p in L32.agent.named_parameters())
        g32.update(("mixer." + k, p.grad) for k, p in L32.mixer.named_parameters())
        g64 = dict(("agent." + k, p.grad) for k, p in L64.agent.named_parameters())
        g64.update(("mixer." + k, p.grad) for k, p in L64.mixer.named_parameters())
        g64 = {k: (None if v is None else v.clone()) for k, v in g64.items()}
        raw = {k: (None if v is None else _rel_l2(gv[k], v)) for k, v in g64.items()}
        e32 = {k: (None if v is None else _rel_l2(g32[k].double(), v)) for k, v in g64.items()}     # the fp32 oracle keeps float64's signs
        flips = kink.resolve_abs_kinks(L64, batch, gv, g64)
        print("step %d: %d |.| kink(s) resolved: %s" % (s + 1, len(flips), flips))
        for k in g64:
            if g64[k] is None:          # the agent net's unused fc_h layer
                assert float(gv[k].abs().max()) == 0.0, k
                continue
            rows.append((s, k, raw[k], _rel_l2(gv[k], g64[k]), e32[k]))
    print("step tensor  engine-vs-float64 (before / after kinks)  fp32-oracle-vs-float64  ratio")
    for s, k, e_raw, e_eng, e_32 in rows:
        print("%d %-36s %.2e %.2e %.2e %.2f" % (s + 1, k, e_raw, e_eng, e_32, e_eng / max(e_32, 1e-300)))
    bad = [(s + 1, k, e_eng, e_32) for s, k, e_raw, e_eng, e_32 in rows if e_eng > RATIO * e_32 and e_eng > FLOOR]
    assert not bad, bad
