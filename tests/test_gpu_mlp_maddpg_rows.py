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
    print("worst", worst, "redraws", stats["redraws"], "smallest margin kept %.2e" % stats.get("min_margin", float("inf")))


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
