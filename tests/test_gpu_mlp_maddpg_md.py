"""Transition-level MADDPG / MATD3 with MultiDiscrete action spaces on the real sm_90a kernels: the fixtures of the unmodified reference,
lock-step against oracle/maddpg_mlp_md.py at small sizes and at simple_reference shapes (B = 1000 drawn from a replay of 100 000
transitions), and the captured whole-update graph of a shared MultiDiscrete learner against eager steps."""

import numpy as np
import pytest
import torch

import mlp_maddpg_md_checks as mdc
from mlp_maddpg_multi_checks import FIELDS

pytestmark = pytest.mark.gpu
N, O, S, SEGS = mdc.N, mdc.O, mdc.S, mdc.SEGS


@pytest.mark.parametrize("name", mdc.GOLDENS_MD)
def test_engine_reproduces_reference(gpu_engine, name):
    mdc.engine_against_golden(name)


@pytest.mark.parametrize("specs,td3,over", [(mdc.REFERENCE_SPEC, False, {}), (mdc.REFERENCE_SPEC, True, {}),
                                            (mdc.REFERENCE_SPEC, False, {"use_per": True, "use_huber_loss": True, "huber_delta": 1.0}),
                                            ([(11, 5), (9, [5, 4])], True, {})])
def test_lockstep_small(gpu_engine, specs, td3, over):
    from offpolicy._b200.factory import build_mlp_maddpg_multi
    torch.manual_seed(3)
    args, pols, tr, _ = build_mlp_maddpg_multi(specs, S, 32, discrete=True, td3=td3, **over)
    rng = np.random.default_rng(4)
    avail = len(specs) == 1              # masks with zeros: a MultiDiscrete policy ignores them
    mdc.lockstep(args, pols, tr, [mdc.synth_batch_md(rng, specs, 32, S, per=args.use_per, avail=avail) for _ in range(3)])


def _filled_buffer(B, size, seed):
    from offpolicy._b200.factory import Box, MultiDiscrete
    from offpolicy.utils.mlp_buffer import MlpReplayBuffer
    info = {"policy_0": dict(obs_space=Box(O), share_obs_space=Box(S), act_space=MultiDiscrete([[0, n - 1] for n in SEGS]))}
    buf = MlpReplayBuffer(info, {"policy_0": list(range(N))}, size, True, False, max_batch=B)
    rng = np.random.default_rng(seed)
    tr = lambda x: np.asarray(x["policy_0"]).transpose(1, 0, 2)          # (N, B, .) -> the runner's (B, N, .)
    for _ in range(size // B):
        b = mdc.synth_batch_md(rng, mdc.REFERENCE_SPEC, B, S)
        buf.insert(B, {"policy_0": tr(b[0])}, {"policy_0": b[1]["policy_0"]}, {"policy_0": tr(b[2])}, {"policy_0": tr(b[3])},
                   {"policy_0": tr(b[4])}, {"policy_0": b[5]["policy_0"]}, {"policy_0": tr(b[6])}, {"policy_0": b[7]["policy_0"]},
                   {"policy_0": tr(b[8])}, None, None)
    return buf


@pytest.mark.parametrize("td3", [False, True])
def test_lockstep_simple_reference_sizes(gpu_engine, td3):
    """B = 1000 from 100 000 stored transitions; the batch is the replay's device batch (valid_transition read through its indices).
    Losses to 1e-3; parameters to two Adam steps of lr (a gradient element within round-off of zero may take either sign)."""
    from offpolicy._b200.factory import build_mlp_maddpg
    B = 1000
    torch.manual_seed(8)
    args, pol, tr = build_mlp_maddpg(N, O, SEGS, S, B, td3=td3)
    buf = _filled_buffer(B, 100_000, 9)
    np.random.seed(10)
    L = mdc.oracle_from(args, pol)
    for k in range(3):
        s = buf.sample(B)
        host = tuple({"policy_0": s.materialize("policy_0", f)} for f in FIELDS[:9]) + ({"policy_0": None}, {"policy_0": None}, None, None)
        before = torch.get_rng_state()
        info, _, _ = tr.shared_train_policy_on_batch("policy_0", s)
        torch.set_rng_state(before)
        ref, _, _ = L.step(host, tr.draw_target_noise(B), tr.draw_actor_noise(B))
        for key, v in ref.items():
            d = abs(float(info[key]) - v) / max(1.0, abs(v))
            assert d <= 1e-3, (k, key, float(info[key]), v)
        pol.soft_target_updates()
        L.soft_update()
        for mod, ref_sd in ((pol.actor, L.actor), (pol.critic, L.critic)):
            for key, v in mod.state_dict().items():
                assert float((v.cpu() - ref_sd[key].detach()).abs().max()) <= 2 * args.lr + 1e-6, key


@pytest.mark.parametrize("td3", [False, True])
def test_graph_replay_equals_eager(gpu_engine, td3):
    """MaddpgStepGraph (device uniform sample -> step -> soft update) of a shared MultiDiscrete learner replayed = the same
    updates run eagerly, bit for bit."""
    from offpolicy._b200.factory import build_mlp_maddpg
    from offpolicy._b200.graph import MaddpgStepGraph
    B = 256
    runs = []
    side = torch.cuda.Stream()                 # a capture needs a non-default stream; eager steps run on the same one
    for mode in ("eager", "graph"):
        with torch.cuda.stream(side):
            torch.manual_seed(21)
            args, pol, tr = build_mlp_maddpg(N, O, SEGS, S, B, td3=td3)
            buf = _filled_buffer(B, 4096, 22)
            buf.seed_device_rng(23)
            if mode == "graph":
                g = MaddpgStepGraph(buf, tr, B)
            infos = []
            for k in range(3):
                torch.manual_seed(100 + k)
                if mode == "eager":
                    info, _, _ = tr.shared_train_policy_on_batch("policy_0", buf.sample(B))
                    pol.soft_target_updates()
                    torch.cuda.synchronize()
                    infos.append([float(info[i]) for i in ("critic_loss", "critic_grad_norm", "actor_loss", "actor_grad_norm")])
                else:
                    g.launch()
                    torch.cuda.synchronize()
                    infos.append([float(tr._info[i]) for i in (0, 1, 4, 5)])
            runs.append((infos, [v.clone() for v in pol.actor_vecs + pol.critic_vecs]))
    assert runs[0][0] == runs[1][0]
    for a, b in zip(runs[0][1], runs[1][1]):
        assert torch.equal(a, b)


def test_rollout_forward_matches_independent_actor(gpu_engine):
    """The rollout forward (k_policy_step, 15 outputs) against the oracle's actor on the same weights, live and target."""
    from offpolicy._b200.factory import build_mlp_maddpg
    torch.manual_seed(6)
    args, pol, tr = build_mlp_maddpg(N, O, SEGS, S, 8)
    rng = np.random.default_rng(0)
    with torch.no_grad():
        for v in pol.actor_vecs[:2]:
            v.add_(torch.from_numpy(rng.standard_normal(v.numel()).astype(np.float32) * 0.05).to(v.device))      # heads away from gain 0.01
    L = mdc.oracle_from(args, pol)
    obs = rng.standard_normal((500, O)).astype(np.float32)
    for theta, net in ((pol.actor_vecs[0], L.actor), (pol.actor_vecs[1], L.target_actor)):
        got = pol._forward(theta, obs).numpy()
        want = L.actor_out(net, torch.from_numpy(obs)).detach().numpy()
        assert got.shape == (500, 15)
        assert np.abs(got - want).max() <= 1e-4 * max(1.0, np.abs(want).max())


@pytest.mark.parametrize("discrete", [True, False])
def test_wide_single_block_actions_lockstep(gpu_engine, discrete):
    """The MLP learner takes one block wider than 8 (Discrete(12), Box(12)), against oracle/maddpg_mlp.py."""
    import mlp_maddpg_checks as mc
    from offpolicy._b200.factory import build_mlp_maddpg
    torch.manual_seed(5)
    n, o, a, s2, B = 2, 10, 12, 20, 32
    for td3 in (False, True):
        args, pol, tr = build_mlp_maddpg(n, o, a, s2, B, discrete=discrete, td3=td3)
        rng = np.random.default_rng(7)
        mc.lockstep(args, pol, tr, [mc.synth_batch(rng, n, B, o, s2, a, discrete) for _ in range(3)])
