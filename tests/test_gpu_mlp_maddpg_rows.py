"""Transition-level coverage of the MLP MADDPG / MATD3 learner on the device, at its SM count: isolated critic transitions and actor
rows, per-transition priorities and a changing batch size against the float64 oracle, at batch sizes on the tile edges of the step's
three row spaces (tests/mlp_maddpg_row_checks.py), the script's B = 1 000 among them."""
import numpy as np
import pytest
import torch

import mlp_maddpg_row_checks as rk

pytestmark = pytest.mark.gpu
SPREAD = [(18, 5, 3)]


def _rules():
    return rk.TileRules(torch.cuda.get_device_properties(0).multi_processor_count)


def _check(worst, stats):
    assert worst["grad"] <= rk.GRAD_TOL and worst["td_ulps"] <= rk.TD_ULPS
    print("worst", worst, "redraws", stats["redraws"], "of them ill-conditioned", stats.get("ill_conditioned", 0),
          "smallest margin kept %.2e" % stats.get("min_margin", float("inf")))


def test_simple_spread_matd3_edges(gpu_engine):
    """MATD3, Discrete, simple_spread: every edge of the critic (69 columns), the actor (18) and the copies (69), and B = 1 000."""
    R = _rules()
    edges = rk.pick_batches(R, 3, 18, 69)
    for B, tg, note in edges:
        print(B, tg, note)
    _check(*rk.run_case(gpu_engine, gpu_engine.stream_ptr(), R, SPREAD, 54, True, True, sorted({B for B, _, _ in edges} | {1000})))


@pytest.mark.parametrize("name,specs,S,disc,td3,avail,over", [
    ("maddpg_disc_next_avail", SPREAD, 54, True, False, True, {}),
    ("maddpg_box", SPREAD, 54, False, False, False, {}),
    ("matd3_box", SPREAD, 54, False, True, False, {}),
    ("matd3_disc_tanh", SPREAD, 54, True, True, False, {"use_ReLU": False}),
    ("narrow_critic", [(10, 5, 2)], 20, True, False, False, {}),
    ("obs60", [(60, 5, 2)], 20, True, True, False, {}),
    ("obs100", [(100, 5, 2)], 20, True, False, False, {}),
    ("md_5_10", [(21, [5, 10], 2)], 42, True, True, False, {}),
    ("md_three_blocks", [(16, [3, 4, 2], 3)], 30, True, False, False, {}),
])
def test_isolated_transitions_at_the_edges(gpu_engine, name, specs, S, disc, td3, avail, over):
    """Each configuration at the batch sizes on its own row spaces' edges.  The narrow critic runs every edge (its sms / sms + 1 tiles
    need B 4 193 / 8 449); the other configurations skip the edges above B = 1 100, which the simple_spread case and the narrow critic
    run with the same kernels."""
    R = _rules()
    N, O, cin = rk.geometry(specs, S, "policy_0")
    edges = rk.pick_batches(R, N, O, cin)
    Bs = sorted({B for B, _, _ in edges if B <= 1100 or name == "narrow_critic"})
    print("skipped:", [(B, tg) for B, tg, _ in edges if B not in Bs])
    _check(*rk.run_case(gpu_engine, gpu_engine.stream_ptr(), R, specs, S, disc, td3, Bs, avail=avail, **over))


@pytest.mark.parametrize("specs,S,p,td3", [
    ([(3, 3, 1), (11, 5, 1)], 14, "policy_0", True),
    ([(3, 3, 1), (11, 5, 1)], 14, "policy_1", True),
    ([(8, 4, 1), (10, 5, 2)], 16, "policy_1", False),
    ([(8, 4, 1), (12, [3, 5], 2)], 16, "policy_1", True),
], ids=["speaker", "listener", "two_agent_policy_at_offset", "md_beside_discrete"])
def test_isolated_transitions_several_policies(gpu_engine, specs, S, p, td3):
    R = _rules()
    N, O, cin = rk.geometry(specs, S, p)
    Bs = sorted({B for B, _, _ in rk.pick_batches(R, N, O, cin) if B <= 1100})
    _check(*rk.run_case(gpu_engine, gpu_engine.stream_ptr(), R, specs, S, True, td3, Bs, p=p))


@pytest.mark.parametrize("td3", [False, True])
def test_batch_size_changes_on_one_learner(gpu_engine, td3):
    """max_batch = the actor's nearest edge to sms + 1 tiles, then B = 1, then one 64-row critic chunk smaller."""
    R = _rules()
    Bmax = max(B for B, tg, _ in rk.pick_batches(R, 3, 18, 69) if "actor tiles = sms+1" in tg)
    args, pols, tr, L64 = rk.build_pair(SPREAD, 54, Bmax, True, td3, use_per=True)
    stats = {"redraws": 0}
    worst = rk.batch_size_sequence(args, tr, pols, L64, "policy_0", rk.make_batches(SPREAD, 54, True), [Bmax, 1, Bmax - 64], 5,
                                   np.random.default_rng(5), stats, R, gpu_engine, gpu_engine.stream_ptr())
    assert worst <= rk.GRAD_TOL
    print("worst", worst, "redraws", stats["redraws"])


def _wide_params():
    """Every edge of simple_spread N = 5 MATD3 and of the 320-column critic (the critic's sms / sms + 1 tiles need B 4 193 / 4 225 at
    132 SMs); the other wide cases up to B 1 100; and B = 1 000 for every case."""
    import test_emu_mlp_maddpg_rows as er
    if not torch.cuda.is_available():
        return [pytest.param("none", "policy_0", 1, id="no-device")]
    every = ("spread5_matd3_disc", "critic320_matd3_disc")
    out = er.wide_params(_rules(), lambda name: 10 ** 9 if name in every else 1100)
    for name, v in er.WIDE.items():
        for p in v[5]:
            out.append(pytest.param(name, p, 1000, id="%s-%s-B1000" % (name, p)))
    return out


@pytest.mark.parametrize("name,p,B", _wide_params())
def test_isolated_transitions_above_128_columns(gpu_engine, name, p, B):
    """Critic (and one actor) inputs above 128 columns: FFMA k_front_fwd / k_front_bwd on 32-row tiles of 162-211 KB, every isolated
    pair in its space's last tile on the device's own grid (tests/test_emu_mlp_maddpg_rows.py WIDE)."""
    import test_emu_mlp_maddpg_rows as er
    specs, S, disc, td3, avail, _ = er.WIDE[name]
    worst, stats = rk.run_case(gpu_engine, gpu_engine.stream_ptr(), _rules(), specs, S, disc, td3, [B], p=p, avail=avail)
    print("%s %s B %d:" % (name, p, B), end=" ")
    _check(worst, stats)


@pytest.mark.parametrize("N,S,td3,disc", [(5, 150, True, True), (6, 216, False, True), (5, 295, True, True)],
                         ids=["spread5_matd3_critic175", "spread6_maddpg_critic246", "critic320_matd3"])
def test_wide_launches_match_the_tile_rules(gpu_engine, N, S, td3, disc):
    """Every k_front_bwd launch of one captured MLP update at the batch sizes of the wide edges has the tile height, grid and dynamic
    shared memory the Python tile rules restate (front_bwd_pick_rm / front_bwd_smem without k_gru_wgrad): critic B rows and the
    agent-replaced copies N B rows at the critic's width, the actor's 2 B N rows at its own -- so the edges the isolated checks pick are
    the ones the device runs."""
    from checkpoint_maddpg_checks import Case
    from offpolicy._b200.torch_rng import DeviceTorchGenerator
    from test_gpu_launch_config import graph_configs
    R = _rules()
    O, cin = 6 * N, S + 5 * N
    for B in sorted({B for B, _, _ in rk.pick_batches(R, N, O, cin) if B <= 1024}):      # the replay samples at most 1 024
        case = Case(kind="mlp", specs=[(N, O, 5)], S=S, B=B, E=B + 64, td3=td3, discrete=disc, rng="device")
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
        # critic above 128 columns, actor below 65: all three spaces on k_front_bwd
        want = ["k_front_bwd<%d> grid=(%d, 1, 1) block=(256, 1, 1) smem=%d" % R.front_bwd_launch(M, w)
                for M, w in ((B, cin), (N * B, cin), (2 * B * N, O))]
        got = [n for n in nodes if n.startswith("k_front_bwd<")]
        assert sorted(got) == sorted(want), (B, got, want)
        assert not any(n.split(" ")[0] in ("k_front_bwd_tc", "k_wgrad_tc") for n in nodes), (B, nodes)
        print("B %d:" % B, got)
