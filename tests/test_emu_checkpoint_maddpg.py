"""Checkpoint / resume (SURVEY.md 8(f).3) of R-MADDPG / R-MATD3, MADDPG / MATD3 and the transition replays on the CPU fiber
emulator: the restored run continues bit-identically, and a checkpoint of another configuration is refused."""
import pytest

import checkpoint_maddpg_checks as cm
from checkpoint_maddpg_checks import Case

RESUME = {
    "rmaddpg_box": (Case("rec", [(2, 6, 2)], S=8, B=4, E=8, T=4, discrete=False), 2),
    # an odd number of updates before the checkpoint: the restored learner must resume in the critic-only phase
    "rmatd3_disc_avail": (Case("rec", [(2, 6, 4)], S=8, B=4, E=9, T=4, td3=True, avail=True, insert=1), 3),
    "rmaddpg_speaker_listener": (Case("rec", [(1, 3, 3), (1, 11, 5)], S=14, B=4, E=8, T=4), 2),
    "maddpg_disc_per_device_rng_norm": (Case("mlp", [(3, 6, 5)], S=10, B=8, E=40, per=True, rng="device", norm=True, insert=4), 2),
    "matd3_multidiscrete": (Case("mlp", [(2, 8, [3, 4])], S=10, B=8, E=40, td3=True, insert=4), 2),
    "maddpg_several_policies": (Case("mlp", [(1, 4, 3), (2, 6, 5)], S=10, B=8, E=40, insert=4), 2),
    "mqmix_per": (Case("mqmix", [(3, 6, 4)], S=10, B=8, E=40, per=True, insert=4), 2),
}


@pytest.mark.parametrize("name", sorted(RESUME))
def test_resume_is_bit_identical(emu_engine, name):
    case, k = RESUME[name]
    cm.check_resume(case, k)


@pytest.mark.parametrize("case", [Case("rec", [(2, 6, 3)], S=8, B=4, E=9, T=4, td3=True, rng="device", insert=1),
                                  Case("mlp", [(3, 6, 5)], S=10, B=8, E=40, td3=True, rng="device", insert=4)],
                         ids=["rmatd3", "matd3"])
def test_graph_on_restored_objects_equals_eager(emu_engine, case):
    cm.check_graph_resume(case, 3)


REC = Case("rec", [(2, 6, 2)], S=8, B=4, E=8, T=4, discrete=False)
MLP = Case("mlp", [(2, 6, 5)], S=10, B=8, E=16)
REJECT = {
    "layout": (REC, Case("rec", [(2, 7, 2)], S=8, B=4, E=8, T=4, discrete=False)),
    "recurrent_vs_mlp": (REC, Case("mlp", [(2, 6, 2)], S=8, B=4, E=8, discrete=False)),
    "td3": (MLP, Case("mlp", [(2, 6, 5)], S=10, B=8, E=16, td3=True)),
    "rtd3": (REC, Case("rec", [(2, 6, 2)], S=8, B=4, E=8, T=4, discrete=False, td3=True)),
    "actor_update_interval": (REC, Case("rec", [(2, 6, 2)], S=8, B=4, E=8, T=4, discrete=False, interval=3)),
    "policy_set": (MLP, Case("mlp", [(1, 6, 5), (1, 6, 5)], S=10, B=8, E=16)),
    "qmix_checkpoint": (Case("mqmix", [(2, 6, 5)], S=10, B=8, E=16), MLP),
}


@pytest.mark.parametrize("name", sorted(REJECT))
def test_learner_checkpoint_of_another_configuration_is_rejected(emu_engine, name):
    a, b = REJECT[name]
    cm.check_rejected(a, b)


def test_replay_checkpoint_of_another_width_is_rejected(emu_engine):
    cm.check_rejected(MLP, Case("mlp", [(2, 7, 5)], S=10, B=8, E=16), trainer=False, buffer=True)


def test_learner_state_calls_refuse_bad_arguments(emu_engine):
    import ctypes as C
    tr, _, _ = REC.build(1)
    lib, off, n = emu_engine.lib(), C.c_int64(), C.c_int64()
    assert lib.mx_maddpg_ws_lookup(tr.handle, b"adam_ta", C.byref(off), C.byref(n)) == 0 and n.value == 8
    assert lib.mx_maddpg_ws_lookup(tr.handle, b"no_such_region", C.byref(off), C.byref(n)) != 0
    assert b"no_such_region" in lib.mx_last_error()
    assert lib.mx_maddpg_set_num_updates(tr.handle, -1) != 0 and b"< 0" in lib.mx_last_error()
    assert lib.mx_maddpg_set_num_updates(tr.handle, 7) == 0 and lib.mx_maddpg_num_updates(tr.handle) == 7


def test_fence_pool_reuses_released_ids(emu_engine):
    cm.check_fence_pool_reuses_released_ids()


def test_per_network_state_dict_keys_are_unchanged(emu_engine):
    """The per-network state_dicts keep the reference's key names (App. E), so its .pt files still load into the drop-in classes."""
    _, _, pols = REC.build(1)
    pol = pols["policy_0"]
    assert list(pol.actor.state_dict()) == [e[0] for e in pol._a_entries]
    assert list(pol.actor.state_dict())[:2] == ["rnn.feature_norm.weight", "rnn.feature_norm.bias"]
    assert "act.action_out.weight" in pol.actor.state_dict() and "rnn.rnn.rnn.weight_hh_l0" in pol.target_actor.state_dict()
    assert [k for k in pol.critic.state_dict() if k.startswith("q_outs")] == ["q_outs.0.weight", "q_outs.0.bias"]
    _, _, pols = MLP.build(1)
    pol = pols["policy_0"]
    assert list(pol.actor.state_dict())[:2] == ["mlp.feature_norm.weight", "mlp.feature_norm.bias"]
    assert "act.action_out.weight" in pol.actor.state_dict()
    assert all(k.startswith("mlp.") for k in pol.critic.state_dict()) and list(pol.critic.state_dict()) == list(pol.target_critic.state_dict())
    assert list(pol.critic_heads.state_dict()) == ["q_outs.0.weight", "q_outs.0.bias"]
