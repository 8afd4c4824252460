"""MaddpgBatchTrainGraph on the CPU fiber emulator (the emulated build re-runs the captured sequence): whole batch_trains of trainers
with one policy per agent against the eager runner, in both noise modes and after a checkpoint resume; the refusals of the new entry
point and of the single-policy one."""
import ctypes as C

import numpy as np
import pytest
import torch

from maddpg_batch_graph_checks import BatchCase, check_graph_equals_eager, check_resume_through_graph

# simple_speaker_listener: speaker obs 3 / Discrete(3), listener obs 11 / Discrete(5), shared observation 14
SL = [(1, 3, 3), (1, 11, 5)]
CASES = {
    "rmaddpg_speaker_listener": BatchCase("rec", SL, S=14, B=4, E=9, T=4, rng="device"),
    "rmatd3_three_box_per": BatchCase("rec", [(1, 4, 2), (2, 5, 3), (1, 3, 2)], S=9, B=4, E=9, T=3, td3=True, discrete=False, per=True,
                                      rng="device"),
    "maddpg_speaker_listener_per_huber": BatchCase("mlp", SL, S=14, B=8, E=40, per=True, rng="device", over={"use_huber_loss": True}),
    "matd3_discrete_multidiscrete": BatchCase("mlp", [(1, 6, 5), (1, 7, [5, 4])], S=10, B=8, E=40, td3=True, rng="device"),
}


@pytest.mark.parametrize("device_noise", [False, True], ids=["host_noise", "device_noise"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_batch_graph_launches_equal_eager_batch_trains(emu_engine, name, device_noise):
    """5 launches (the host staging ring of 4 slots wraps; inserts between them wrap the replay's ring) = 5 eager batch_trains:
    train_info, priorities, sampled indices and trees of every policy, all vectors, Adam counters, update counts, the stores' device
    RNG, the device and the CPU torch generators."""
    rec = check_graph_equals_eager(CASES[name], k=5, device_noise=device_noise)
    if name.startswith("rmatd3"):          # the actor every 2nd batch_train: both graph variants ran
        assert [r["update_actor"] for r in rec] == [True, False, True, False, True]


def test_batch_graph_continues_a_resumed_run(emu_engine):
    check_resume_through_graph(CASES["rmatd3_three_box_per"], k=3, device_noise=True)


def test_batch_graph_continues_a_resumed_host_noise_run(emu_engine):
    check_resume_through_graph(CASES["matd3_discrete_multidiscrete"], k=2, device_noise=False)


# ---- refusals --------------------------------------------------------------------------------------------------------------------
def _objects(name="rmaddpg_speaker_listener"):
    case = CASES[name]
    tr, buf, pols = case.build(1)
    case.fill(buf, np.random.RandomState(5), case.E)
    return case, tr, buf


def _capture(tr, buf, order, B, flags=1):
    from offpolicy._b200 import capi
    lib = capi.lib()
    P = len(order)
    stores = (C.c_void_p * P)(*[getattr(buf.policy_buffers[p], "rep", buf.policy_buffers[p]).handle for p in order])
    learners = (C.c_void_p * P)(*[tr._eng[p].handle for p in order])
    noise = (C.c_void_p * (P * P))()
    g = C.c_void_p()
    rc = lib.mx_maddpg_batch_graph_capture(stores, learners, P, 0, B, 0.4, flags, noise, (C.c_void_p * P)(), 1, None, None, None, None, 0,
                                           None, C.byref(g))
    if rc == 0:
        lib.mx_graph_destroy(g)
    return rc, lib.mx_last_error().decode()


def test_batch_capture_refuses_misordered_or_mismatched_learners(emu_engine):
    case, tr, buf = _objects()
    rc, err = _capture(tr, buf, ["policy_1", "policy_0"], case.B)
    assert rc != 0 and "act_offset" in err and "policy-id order" in err
    # the stores of the other policy under the right learners: the store does not hold that learner's batches
    from offpolicy._b200 import capi
    lib, P = capi.lib(), 2
    stores = (C.c_void_p * P)(*[buf.policy_buffers[p].handle for p in ("policy_1", "policy_0")])
    learners = (C.c_void_p * P)(*[tr._eng[p].handle for p in ("policy_0", "policy_1")])
    g = C.c_void_p()
    assert lib.mx_maddpg_batch_graph_capture(stores, learners, P, 0, case.B, 0.4, 1, (C.c_void_p * 4)(), (C.c_void_p * 2)(), 1, None, None,
                                             None, None, 0, None, C.byref(g)) != 0
    assert "does not hold the batches of learner 0" in lib.mx_last_error().decode()
    # learners of two different policy sets
    _, tr2, _ = _objects("matd3_discrete_multidiscrete")
    learners = (C.c_void_p * P)(tr._eng["policy_0"].handle, tr2._eng["policy_1"].handle)
    stores = (C.c_void_p * P)(*[buf.policy_buffers[p].handle for p in ("policy_0", "policy_1")])
    assert lib.mx_maddpg_batch_graph_capture(stores, learners, P, 0, case.B, 0.4, 1, (C.c_void_p * 4)(), (C.c_void_p * 2)(), 1, None, None,
                                             None, None, 0, None, C.byref(g)) != 0
    assert "not of one policy set" in lib.mx_last_error().decode()
    # one learner alone
    rc, err = _capture(tr, buf, ["policy_0"], case.B)
    assert rc != 0 and "mx_maddpg_graph_capture_ex" in err


def test_batch_capture_refuses_a_batch_over_max_batch(emu_engine):
    case, tr, buf = _objects()
    rc, err = _capture(tr, buf, ["policy_0", "policy_1"], case.max_batch + 1)
    assert rc != 0 and "max_batch" in err
    from offpolicy._b200 import capi
    from offpolicy._b200.graph import MaddpgBatchTrainGraph
    with pytest.raises(capi.MxError, match="max_batch"):
        MaddpgBatchTrainGraph(buf, tr, case.max_batch + 1)


def test_batch_capture_refuses_fills_the_scratch_cannot_hold(emu_engine):
    from offpolicy._b200 import capi
    from offpolicy._b200.torch_rng import DeviceTorchGenerator
    case, tr, buf = _objects()
    gen = DeviceTorchGenerator(seed=3)
    tr.use_device_noise(gen)
    draws = tr._noise_draws(case.B, "policy_0", "actor")
    lib, P = capi.lib(), 2
    arr = (capi.TrngDraw * len(draws))(*draws)
    counts = (C.c_int32 * P)(len(draws), 0)
    stores = (C.c_void_p * P)(*[buf.policy_buffers[p].handle for p in case.ids])
    learners = (C.c_void_p * P)(*[tr._eng[p].handle for p in case.ids])
    scratch = torch.zeros(1, dtype=torch.int32)
    g = C.c_void_p()
    assert lib.mx_maddpg_batch_graph_capture(stores, learners, P, 0, case.B, 0.4, 1, (C.c_void_p * 4)(), (C.c_void_p * 2)(), 1,
                                             capi.ptr(gen.state), arr, counts, capi.ptr(scratch), 1, None, C.byref(g)) != 0
    assert "scratch of 1 words" in lib.mx_last_error().decode()


def test_batch_graph_refuses_unequal_update_counts(emu_engine):
    from offpolicy._b200.graph import MaddpgBatchTrainGraph
    case, tr, buf = _objects("rmatd3_three_box_per")
    tr.num_updates["policy_1"] += 1
    with pytest.raises(ValueError, match="differ modulo the actor update interval"):
        MaddpgBatchTrainGraph(buf, tr, case.B)


def test_batch_graph_refuses_a_shared_policy_trainer(emu_engine):
    from offpolicy._b200.graph import MaddpgBatchTrainGraph
    case = BatchCase("rec", [(2, 6, 3)], S=8, B=4, E=9, T=4, rng="device")
    tr, buf, _ = case.build(1)
    with pytest.raises(ValueError, match="MaddpgStepGraph"):
        MaddpgBatchTrainGraph(buf, tr, case.B)


def test_batch_graph_refuses_a_host_rng_buffer(emu_engine):
    from offpolicy._b200.graph import MaddpgBatchTrainGraph
    case = BatchCase("rec", SL, S=14, B=4, E=9, T=4)
    tr, buf, _ = case.build(1)
    with pytest.raises(ValueError, match="device RNG"):
        MaddpgBatchTrainGraph(buf, tr, case.B)


def test_single_policy_capture_refuses_a_recurrent_learner_of_several_policies(emu_engine):
    """The recurrent learner of a several-policy trainer was captured, and its graph stepped on stale centralised action vectors."""
    from offpolicy._b200 import capi
    from offpolicy._b200.graph import MaddpgStepGraph
    case, tr, buf = _objects()
    lib = capi.lib()
    g = C.c_void_p()
    rc = lib.mx_maddpg_graph_capture(buf.policy_buffers["policy_0"].handle, tr._eng["policy_0"].handle, case.B, 0.0, 1, None, None, 1,
                                     None, C.byref(g))
    assert rc != 0
    err = lib.mx_last_error().decode()
    assert "several policies" in err and "mx_maddpg_batch_graph_capture" in err
    with pytest.raises(capi.MxError, match="several policies"):
        MaddpgStepGraph(buf, tr, case.B)
