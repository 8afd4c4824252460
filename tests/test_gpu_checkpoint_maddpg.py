"""Checkpoint / resume (SURVEY.md 8(f).3) of R-MADDPG / R-MATD3, MADDPG / MATD3 and the transition replays on the H100 at working
sizes: the restored run continues bit-identically, eagerly and through the captured whole-update graphs."""
import pytest

import checkpoint_maddpg_checks as cm
from checkpoint_maddpg_checks import Case

pytestmark = pytest.mark.gpu

SPREAD = dict(S=54, B=1000, E=100_000, insert=250)          # simple_spread: 3 agents, obs 18, Discrete(5); B = 1000 from 100 000 transitions


@pytest.mark.parametrize("case", [Case("mlp", [(3, 18, 5)], **SPREAD), Case("mlp", [(3, 18, 5)], td3=True, **SPREAD),
                                  Case("mlp", [(3, 18, 5)], per=True, rng="device", norm=True, **SPREAD)],
                         ids=["maddpg", "matd3", "maddpg_per_device_rng_norm"])
def test_mlp_resume_at_train_mpe_sizes(gpu_engine, case):
    cm.check_resume(case, 3)


@pytest.mark.parametrize("case", [Case("mlp", [(1, 3, 3), (1, 11, 5)], S=14, B=1000, E=100_000, insert=250),
                                  Case("rec", [(1, 3, 3), (1, 11, 5)], S=14, B=32, E=5000, T=25, insert=8)],
                         ids=["maddpg", "rmaddpg"])
def test_speaker_listener_one_policy_per_agent(gpu_engine, case):
    cm.check_resume(case, 3)


@pytest.mark.parametrize("case", [Case("rec", [(3, 18, 2)], S=54, B=32, E=5000, T=25, td3=True, discrete=False, rng="device", insert=8),
                                  Case("mlp", [(3, 18, 5)], td3=True, rng="device", **SPREAD)],
                         ids=["rmatd3_spread", "matd3_spread"])
def test_graph_on_restored_objects_equals_eager(gpu_engine, case):
    cm.check_graph_resume(case, 3)


def test_dropped_buffers_release_their_host_fences(gpu_engine):
    """A run that is resumed again and again in one process builds a fresh replay each time: the dropped ones must give their host
    fences back to the bounded pool."""
    cm.check_dropped_buffers_release_their_fences()
    cm.check_fence_pool_reuses_released_ids()


def test_checkpoint_of_another_configuration_is_rejected(gpu_engine):
    cm.check_rejected(Case("rec", [(3, 18, 2)], S=54, B=32, E=64, T=25, discrete=False),
                      Case("rec", [(3, 18, 2)], S=54, B=32, E=64, T=25, discrete=False, td3=True))
    cm.check_rejected(Case("mlp", [(3, 18, 5)], S=54, B=64, E=256), Case("mlp", [(3, 17, 5)], S=54, B=64, E=256), trainer=False, buffer=True)
