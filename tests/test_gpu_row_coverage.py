"""Row and tile coverage of the QMIX / M-QMIX learner kernels on the GPU's own grid, against the float64 oracle.

The same checks as tests/test_emu_row_coverage.py, with the edge shapes derived from this device's SM count (132 on an H100 SXM): one
tile with every other CTA idle, last tiles holding one row or one short of full, a CTA running a second / third tile, k_front_bwd_tc one
tile past its CTAs, the mixer's 16 sms / 16 sms + 1 transitions.  Large shapes isolate the first and last episode and the ones holding
a CTA's next tile; two further shapes: the config-2 batch (3m, B 32, T 60) with every episode isolated in turn, and 8m at full size
(M = 30 976 rows, several tiles per CTA)."""
import numpy as np
import pytest
import torch

import row_coverage_checks as rc
import test_emu_row_coverage as ec


@pytest.fixture
def oracle_threads():
    """The float64 oracle runs on 8 host threads; the process-wide setting is restored afterwards."""
    n = torch.get_num_threads()
    yield
    torch.set_num_threads(n)


def _rules():
    return rc.TileRules(torch.cuda.get_device_properties(0).multi_processor_count)


def _gpu_cases():
    if not torch.cuda.is_available():
        return [pytest.param("none", 1, 1, 1, "", id="no-device")]
    R = _rules()
    out = []
    for path in ("obs11_debug", "obs60_a36_product", "prev_act_product", "obs80_debug", "obs120_a64_product"):
        for tg, (B, T, N), lay, note in rc.pick_shapes(R, ec._in_dim(path), Ns=(3, 5, 8), Ts=range(8, 65), Bs=range(1, 130)):
            out.append(pytest.param(path, B, T, N, note, id="%s-B%d-T%d-N%d-%s" % (path, B, T, N, "_".join(ec.TAGS[t] for t in tg))))
    for tg, (B, T, N), lay, note in rc.pick_mixer_shapes(R, Ns=(3,), Ts=range(2, 161), Bs=range(1, 200)):
        for path in ("obs11_debug", "obs60_a36_product"):
            out.append(pytest.param(path, B, T, N, note, id="%s-B%d-T%d-N%d-%s" % (path, B, T, N, ec.TAGS[tg[0]])))
    return out


def _run(gpu_engine, path, B, T, N, note, S=13, cfg=None, every_up_to=16, extra_kernels=()):
    from oracle.qmix import synth_batch
    R = _rules()
    obs, act, prev, debug, kernels = ec.PATHS[path]
    if note:
        print("shape note:", note)
    cfg = cfg or ec._cfg(obs, act, prev, N, S=S)
    ind = cfg.obs_dim + (cfg.act_dim if cfg.prev_act_inp else 0)
    L64, pol, tr = rc.qmix_pair(cfg, B, T, debug=debug)
    batch = rc.last_episode_full_length(synth_batch(cfg, B, T, seed=5, avail_p=0.8, var_len=True) + (np.ones(B, np.float32), np.arange(B)))
    TM, _, grid = R.agent_rows(B * (T + 1) * N, ind)[R.row_kernel(ind)]
    eps = rc.sample_episodes(B, T, N, TM, grid, every_up_to=every_up_to)
    lib = gpu_engine.lib()
    names = rc.kernels_run(lib, gpu_engine.stream_ptr(), lambda: rc.isolated_episode_gradients(L64, tr, batch, eps[:1], B, T, N))
    rc.assert_kernels_ran(names, list(kernels) + list(extra_kernels))
    worst_g = rc.isolated_episode_gradients(L64, tr, batch, eps, B, T, N)
    worst_f = rc.per_row_forward(L64, tr, batch, B, T, N, debug)
    gk, fk = max(worst_g, key=worst_g.get), max(worst_f, key=worst_f.get)
    print("sms %d B %d T %d N %d M %d: %d episodes isolated; worst gradient %s %.2e (bound %.0e); worst row %s %.2e (bound %.0e)"
          % (R.sms, B, T, N, B * (T + 1) * N, len(eps), gk, worst_g[gk], rc.GRAD_TOL, fk, worst_f[fk], rc.ROW_TOL))


@pytest.mark.gpu
@pytest.mark.parametrize("path,B,T,N,note", _gpu_cases())
def test_isolated_episode_gradients_and_rows(gpu_engine, oracle_threads, path, B, T, N, note):
    _run(gpu_engine, path, B, T, N, note)


@pytest.mark.gpu
def test_config2_every_episode_isolated(gpu_engine, oracle_threads):
    """The config-2 batch (3m: B 32, T 60, N 3, obs 30, seed 5): its last 64 agent-net rows carry no gradient in the whole-batch step;
    here each of the 32 episodes is the whole gradient once."""
    from oracle.qmix import QmixConfig
    cfg = QmixConfig(gain=1.0, use_per=True)
    _run(gpu_engine, "obs11_debug", 32, 60, 3, "", cfg=cfg, every_up_to=32)


@pytest.mark.gpu
def test_8m_full_size_sampled_episodes(gpu_engine, oracle_threads):
    """8m at full size (B 32, T 120, N 8, obs 80: M = 30 976 rows, several 64-row chunks per CTA): the first and the last episode and
    the ones holding a CTA's next chunk."""
    from oracle.qmix import QmixConfig
    cfg = QmixConfig(n_agents=8, obs_dim=80, act_dim=14, state_dim=168, gain=1.0, use_per=True)
    _run(gpu_engine, "obs80_debug", 32, 120, 8, "", cfg=cfg, every_up_to=0)


@pytest.mark.gpu
@pytest.mark.parametrize("S,B,T", [(449, 3, 11), (449, 40, 53)])
def test_wide_state_mixer_isolated(gpu_engine, oracle_threads, S, B, T):
    _run(gpu_engine, "obs11_debug", B, T, 3, "", S=S, extra_kernels=("k_mixw_fwd", "k_mixw_wgrad"))


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 65, 2112, 2113])
def test_mqmix_isolated_transitions(gpu_engine, oracle_threads, B):
    """M-QMIX at the mixer's 16 sms / 16 sms + 1 transitions (2 112 / 2 113 on 132 SMs) and around the first chunk edge."""
    from oracle.qmix import QmixConfig
    from oracle.mqmix import synth_transitions
    R = _rules()
    N = 3
    cfg = QmixConfig(n_agents=N, obs_dim=20, act_dim=6, state_dim=14, gain=1.0, use_per=True)
    L64, pol, tr = rc.mqmix_pair(cfg, B)
    batch = synth_transitions(cfg, B, seed=7, avail=True) + (None, None)
    TM, _, grid = R.agent_rows(2 * N * B, 20)["k_front_bwd"]
    eps = rc.sample_episodes(B, 1, N, TM, grid)
    names = rc.kernels_run(gpu_engine.lib(), gpu_engine.stream_ptr(),
                           lambda: rc.isolated_episode_gradients(L64, tr, batch, eps[:1], B, 1, N, mlp=True))
    rc.assert_kernels_ran(names, ["k_front_fwd_tc", "k_mlp_qselect", "k_mlp_dgi", "k_front_bwd", "k_mix_core"])
    worst = rc.isolated_episode_gradients(L64, tr, batch, eps, B, 1, N, mlp=True)
    print("M-QMIX B %d: worst gradient %.2e (bound %.0e)" % (B, max(worst.values()), rc.GRAD_TOL))


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["obs11_debug", "obs80_debug"])
def test_batch_size_changes_on_one_learner(gpu_engine, oracle_threads, path):
    R = _rules()
    obs, act, prev, debug, kernels = ec.PATHS[path]
    ind = ec._in_dim(path)
    (tg, (Bmax, T, N), lay, note), = rc.pick_shapes(R, ind, Ns=(3, 5, 8), Ts=range(8, 65), Bs=range(1, 130), targets=["tiles = sms+1"])
    kern = R.row_kernel(ind)
    tiles = lambda B: R.agent_rows(B * (T + 1) * N, ind)[kern][1]
    fewer = [B for B in range(1, Bmax) if tiles(B) < tiles(Bmax)]
    Bs = [Bmax, 1, max(fewer, key=lambda B: (tiles(B), B))]
    print("batch sizes", Bs, "tiles", [tiles(B) for B in Bs])
    cfg = ec._cfg(obs, act, prev, N)
    L64, pol, tr = rc.qmix_pair(cfg, Bmax, T, debug=debug)
    worst = rc.batch_size_sequence(L64, pol, tr, cfg, Bs, T)
    print("worst gradient %.2e (bound %.0e)" % (max(worst.values()), rc.GRAD_TOL))


@pytest.mark.gpu
@pytest.mark.parametrize("act", [36, 64])
def test_two_actions_per_lane_in_the_fused_mid_kernel(gpu_engine, oracle_threads, act):
    """k_mid itself with two actions per lane (A = 36 / 64) at a small batch, where the step runs the split mixer and k_mid."""
    from oracle.qmix import synth_batch
    B, T, N = 3, 9, 3
    cfg = ec._cfg(11, act, False, N)
    L64, pol, tr = rc.qmix_pair(cfg, B, T, debug=False)
    batch = rc.last_episode_full_length(synth_batch(cfg, B, T, seed=6, avail_p=0.8, var_len=True) + (np.ones(B, np.float32), np.arange(B)))
    names = rc.kernels_run(gpu_engine.lib(), gpu_engine.stream_ptr(), lambda: rc.isolated_episode_gradients(L64, tr, batch, [0], B, T, N))
    assert "k_mid" in names and "k_front_fwd_tc" in names and "k_front_fwd_tc1" not in names, names
    rc.isolated_episode_gradients(L64, tr, batch, list(range(B)), B, T, N)
    rc.per_row_forward(L64, tr, batch, B, T, N, False)


def _maddpg_gpu_cases():
    if not torch.cuda.is_available():
        return [pytest.param(False, 1, 8, 3, id="no-device")]
    return [pytest.param(disc, B, T, N, id="%s-B%d-T%d-%s" % ("disc" if disc else "box", B, T, "_".join(t.replace(" ", "").replace("=", "").replace("+", "p")
                                                                                                          for t in tg)))
            for tg, (B, T, N), lay, note in rc.pick_maddpg_shapes(_rules()) for disc in (False, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("disc,B,T,N", _maddpg_gpu_cases())
def test_maddpg_isolated_episode_gradients(gpu_engine, oracle_threads, disc, B, T, N):
    """R-MADDPG critic and actor, Box and Discrete, T >= 8, on the edges of k_head_bwd's 32-row tiles at this device's SM count."""
    ec.run_maddpg(gpu_engine, disc, B, T, N, stream=gpu_engine.stream_ptr(), rules=_rules())


def _maddpg_wide_gpu_cases():
    if not torch.cuda.is_available():
        return [pytest.param("none", 1, 8, id="no-device")]
    return ec.maddpg_wide_params(_rules())


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,T", _maddpg_wide_gpu_cases())
def test_maddpg_isolated_episodes_above_128_columns(gpu_engine, oracle_threads, name, B, T):
    """R-MADDPG / R-MATD3 above 128 critic columns (tests/test_emu_row_coverage.py MADDPG_WIDE) on every k_head_bwd and k_front_bwd edge
    of the critic's, the actor's and the copies' row spaces at this device's SM count, episodes shorter than 8 steps and longer."""
    N, obs, S, disc, td3 = ec.MADDPG_WIDE[name]
    ec.run_maddpg(gpu_engine, disc, B, T, N, stream=gpu_engine.stream_ptr(), rules=_rules(), td3=td3, obs=obs, S=S)


@pytest.mark.gpu
@pytest.mark.parametrize("disc", [True, False], ids=["disc", "box"])
def test_rmatd3_oracle_lockstep_simple_spread5(gpu_engine, oracle_threads, disc):
    """R-MATD3 whole updates at simple_spread N = 5 (critic 150 + 5 x act columns) and the script's B 32, T 25, three in a row against
    the fp32 oracle."""
    import maddpg_checks as mdc
    from oracle.maddpg import MaddpgConfig
    cfg = MaddpgConfig(n_agents=5, obs_dim=30, act_dim=5 if disc else 2, state_dim=150, discrete=disc, td3=True, actor_update_interval=2,
                       gain=1.0, use_per=True)
    print("worst gradient / bound %.2f" % mdc.check_oracle_lockstep(cfg, 32, 25))


@pytest.mark.gpu
def test_maddpg_wide_launches_match_the_tile_rules(gpu_engine):
    """Every k_front_bwd launch of one captured R-MADDPG update at simple_spread N = 5 (critic 175) has the tile height, grid and dynamic
    shared memory that maddpg_front_spaces restates -- the critic's B T and the copies' N B T rows at 175 columns, the actor's B (T+1) N
    at 30, no k_gru_wgrad beside it -- at the shapes of the wide cases' edges, so those edges are the ones the device runs; and the
    critic's launches run no tensor-core kernel."""
    from checkpoint_maddpg_checks import Case
    from offpolicy._b200.torch_rng import DeviceTorchGenerator
    from test_gpu_launch_config import graph_configs
    R = _rules()
    N, obs, S = 5, 30, 150
    cin = S + 5 * N
    shapes = sorted({(B, T) for tg, (B, T, _), _, _ in rc.pick_maddpg_shapes(R, N=N, Ts=range(4, 40), Bs=range(1, 200), obs=obs, cin=cin)})
    for B, T in shapes:
        case = Case(kind="rec", specs=[(N, obs, 5)], S=S, B=B, E=max(64, 2 * B), T=T, rng="device")
        tr, buf, pols = case.build(1)
        case.fill(buf, np.random.RandomState(5), case.E)
        torch.manual_seed(11)
        tr.use_device_noise(DeviceTorchGenerator(seed=3))
        smp = buf.sample(B)
        for _ in range(2):
            tr.train_policy_on_batch("policy_0", smp)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph(keep_graph=True)
        with torch.cuda.graph(g):
            tr.train_policy_on_batch("policy_0", smp)
        try:
            nodes, _ = graph_configs(g.raw_cuda_graph())
        finally:
            g.reset()
            torch.cuda.synchronize()
        sp = rc.maddpg_front_spaces(R, B, T, N, obs, cin)
        want = ["k_front_bwd<%d> grid=(%d, 1, 1) block=(256, 1, 1) smem=%d" % R.front_bwd_launch(M, cin if name != "actor" else obs)
                for name, (M, TM, nt) in sp.items()]
        got = [n for n in nodes if n.startswith("k_front_bwd<")]
        assert sorted(got) == sorted(want), (B, T, got, want)
        assert not any(n.split(" ")[0] in ("k_front_bwd_tc", "k_wgrad_tc", "k_gru_wgrad<2>", "k_gru_wgrad<3>", "k_gru_wgrad<4>")
                       for n in nodes), (B, T, nodes)
        print("B %d T %d:" % (B, T), got)
