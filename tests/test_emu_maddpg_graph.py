"""MaddpgStepGraph on the CPU fiber emulator: the whole-update graph of R-MADDPG / R-MATD3 and of single-policy MADDPG / MATD3, in
host and device noise mode, against eager updates; the learner's `valid_transition` pointer; the graph variants; the refusal of
several policies."""
import numpy as np
import pytest
import torch

from checkpoint_maddpg_checks import Case, _info_record, _stream_ctx, assert_same, snapshot

# (case, graphs captured): R-MATD3 updates its actor every 2nd call, so it needs the update_actor = 0 variant too
CASES = {
    "maddpg_discrete": (Case("mlp", [(3, 6, 5)], S=10, B=8, E=40, rng="device"), 1),
    "matd3_box": (Case("mlp", [(2, 6, 2)], S=10, B=8, E=40, td3=True, discrete=False, rng="device"), 1),
    "matd3_multidiscrete": (Case("mlp", [(2, 8, [3, 4])], S=10, B=8, E=40, td3=True, rng="device"), 1),
    "rmatd3_discrete": (Case("rec", [(2, 6, 3)], S=8, B=4, E=9, T=4, td3=True, rng="device"), 2),
    "rmaddpg_box": (Case("rec", [(2, 6, 2)], S=8, B=4, E=9, T=4, discrete=False, rng="device"), 1),
}


def _run(case, mode, n, device_noise=False, on_insert=None):
    """n updates of a freshly built trainer, eager or through MaddpgStepGraph: (rounds, learner state, torch's generator state,
    graphs captured)."""
    from offpolicy._b200.graph import MaddpgStepGraph
    from offpolicy._b200.torch_rng import DeviceTorchGenerator
    tr, buf, pols = case.build(1)
    if on_insert is not None:
        insert = buf.insert
        buf.insert = lambda k, *a: on_insert(*a) or insert(k, *a)
    case.fill(buf, np.random.RandomState(5), case.E)
    torch.manual_seed(11)
    if device_noise:
        tr.use_device_noise(DeviceTorchGenerator(seed=3))
    rec, graphs = [], None
    ctx, _ = _stream_ctx()
    with ctx:
        if mode == "eager":
            for _ in range(n):
                r = case.round(tr, buf, pols, None, insert=False)
                rec.append(_info_record(case, tr, buf, dict(r[1])["update_actor"]))
        else:
            g = MaddpgStepGraph(buf, tr, case.B)
            graphs = len(g.graphs)
            for _ in range(n):
                upd = g.launch()
                g.synchronize()
                rec.append(_info_record(case, tr, buf, upd))
            g.close()
    return rec, snapshot(tr, buf), torch.get_rng_state().clone(), graphs


@pytest.mark.parametrize("name", sorted(CASES))
def test_host_noise_graph_launches_equal_eager_updates(emu_engine, name):
    """n host-mode launches = n eager updates, bit for bit: sampled indices, train_info, every vector, update counts and torch's
    generator afterwards; and the graph variants the trainer needs, no more."""
    case, n_graphs = CASES[name]
    rec_e, snap_e, rng_e, _ = _run(case, "eager", 4)
    rec_g, snap_g, rng_g, graphs = _run(case, "graph", 4)
    assert_same(rec_g, rec_e, "rounds")
    assert_same(snap_g, snap_e)
    assert torch.equal(rng_g, rng_e), "torch's generator after the updates"
    assert graphs == n_graphs


@pytest.mark.parametrize("device_noise", [False, True], ids=["host_noise", "device_noise"])
def test_graph_masks_the_actor_with_the_replays_valid_transition(emu_engine, device_noise):
    """A graph built on a freshly built MLP trainer (no eager step has pointed its learner at a valid_transition store) masks the
    actor loss with the replay's valid_transition, not with 1 - done: its launches equal eager updates on a replay where the two
    masks differ."""
    case = Case("mlp", [(3, 6, 5)], S=10, B=8, E=40, td3=True, rng="device")
    differ = []

    def seen(obs, share, acts, rew, nobs, nshare, dones, de, valid, *avail):
        differ.append(bool(((np.asarray(valid["policy_0"]) == 0) & (np.asarray(dones["policy_0"]) == 0)).any()))

    rec_e, snap_e, _, _ = _run(case, "eager", 3, device_noise)
    rec_g, snap_g, _, _ = _run(case, "graph", 3, device_noise, on_insert=seen)
    assert any(differ), "the replay holds no valid_transition 0 where done is 0"
    assert_same(rec_g, rec_e, "rounds")
    assert_same(snap_g, snap_e)


def test_graph_of_several_policies_is_refused(emu_engine):
    from offpolicy._b200 import capi
    from offpolicy._b200.graph import MaddpgStepGraph
    case = Case("mlp", [(1, 3, 3), (1, 11, 5)], S=14, B=8, E=40, td3=True, rng="device")
    tr, buf, _ = case.build(1)
    with pytest.raises(capi.MxError, match="several policies"):
        MaddpgStepGraph(buf, tr, case.B)
