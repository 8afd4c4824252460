"""MaddpgBatchTrainGraph on the H100 at the shapes the reference's several-policy scripts train: whole batch_trains replayed through the
captured graph equal eager batch_trains bit for bit, and a graph replays exactly the kernels one eager batch_train launches."""
import pytest

from maddpg_batch_graph_checks import BatchCase, check_graph_equals_eager, eager_launches

pytestmark = pytest.mark.gpu

SL = [(1, 3, 3), (1, 11, 5)]                 # simple_speaker_listener: speaker obs 3 / Discrete(3), listener obs 11 / Discrete(5)
SPREAD = [(1, 18, 5)] * 3                    # simple_spread, one policy per agent
SPREAD5 = [(1, 30, 5)] * 5                   # simple_spread with 5 agents and 5 landmarks, one policy per agent
# (case, device noise): train_mpe_rmaddpg.sh shapes (episode 25, batch 32, 5 000-episode store); MLP at batch 1 000 from 100 000
# transitions
CASES = {
    "rmaddpg_speaker_listener": (BatchCase("rec", SL, S=14, B=32, E=5000, T=25, rng="device"), False),
    "rmatd3_speaker_listener_per": (BatchCase("rec", SL, S=14, B=32, E=5000, T=25, td3=True, per=True, rng="device"), True),
    "maddpg_speaker_listener_per": (BatchCase("mlp", SL, S=14, B=1000, E=100000, per=True, rng="device"), True),
    "matd3_speaker_listener_per": (BatchCase("mlp", SL, S=14, B=1000, E=100000, td3=True, per=True, rng="device"), True),
    "maddpg_spread_per": (BatchCase("mlp", SPREAD, S=54, B=1000, E=100000, per=True, rng="device"), True),
    "matd3_spread_per": (BatchCase("mlp", SPREAD, S=54, B=1000, E=100000, td3=True, per=True, rng="device"), True),
    # simple_spread with 5 agents and 5 landmarks, one policy per agent: critic input 150 + 25 = 175 (FFMA k_front_fwd / k_front_bwd)
    "matd3_spread5_per_agent_per": (BatchCase("mlp", SPREAD5, S=150, B=1000, E=100000, td3=True, per=True, rng="device"), True),
    "rmatd3_spread5_per_agent": (BatchCase("rec", SPREAD5, S=150, B=32, E=5000, T=25, td3=True, rng="device"), True),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_batch_graph_launches_equal_eager_batch_trains_h100(gpu_engine, name):
    case, device_noise = CASES[name]
    rec = check_graph_equals_eager(case, k=3, device_noise=device_noise)
    if name.startswith("rmatd3"):
        assert [r["update_actor"] for r in rec] == [True, False, True]


@pytest.mark.parametrize("name", sorted(CASES))
def test_batch_graph_replays_the_kernels_of_one_eager_batch_train(gpu_engine, name):
    case, device_noise = CASES[name]
    for upd in ((True, False) if name.startswith("rmatd3") else (True,)):
        n_eager, n_graph = eager_launches(case, device_noise, upd)
        assert n_graph == n_eager > 0, (upd, n_graph, n_eager)
