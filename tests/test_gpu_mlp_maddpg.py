"""Transition-level MADDPG / MATD3 on the real sm_90a kernels: lock-step against oracle/maddpg_mlp.py at small and at
scripts/train_mpe_maddpg.sh sizes (B = 1000 drawn from a replay of 100 000 transitions), and the captured whole-update graph against
eager steps."""

import numpy as np
import pytest
import torch

import mlp_maddpg_checks as mc

pytestmark = pytest.mark.gpu
N, O, A, S = 3, 18, 5, 54


@pytest.mark.parametrize("name", mc.GOLDENS)
def test_engine_reproduces_reference(gpu_engine, name):
    """The fixtures of the unmodified reference (tests/golden/mlp_*.npz), as on the emulator."""
    mc.engine_against_golden(name)


@pytest.mark.parametrize("discrete,td3,avail,over", [(True, False, True, {}), (True, True, False, {}), (False, False, False, {}),
                                                     (False, True, False, {}),
                                                     (True, False, False, {"use_per": True, "use_huber_loss": True, "huber_delta": 1.0})])
def test_lockstep_small(gpu_engine, discrete, td3, avail, over):
    from offpolicy._b200.factory import build_mlp_maddpg
    torch.manual_seed(3)
    args, pol, tr = build_mlp_maddpg(N, O, A, S, 32, discrete=discrete, td3=td3, **over)
    rng = np.random.default_rng(4)
    mc.lockstep(args, pol, tr, [mc.synth_batch(rng, N, 32, O, S, A, discrete, avail=avail, ties=avail, per=args.use_per) for _ in range(3)])


def _filled_buffer(B, size, discrete, seed, N=N, O=O, S=S, A=A):
    from offpolicy._b200.factory import Box, Discrete
    from offpolicy.utils.mlp_buffer import MlpReplayBuffer
    info = {"policy_0": dict(obs_space=Box(O), share_obs_space=Box(S), act_space=Discrete(A) if discrete else Box(A))}
    buf = MlpReplayBuffer(info, {"policy_0": list(range(N))}, size, True, False, max_batch=B)
    rng = np.random.default_rng(seed)
    for _ in range(size // B):
        b = mc.synth_batch(rng, N, B, O, S, A, discrete)
        tr = lambda x: np.asarray(x["policy_0"]).transpose(1, 0, 2)         # (N, B, .) -> the runner's (B, N, .)
        buf.insert(B, {"policy_0": tr(b[0])}, {"policy_0": b[1]["policy_0"]}, {"policy_0": tr(b[2])}, {"policy_0": tr(b[3])},
                   {"policy_0": tr(b[4])}, {"policy_0": b[5]["policy_0"]}, {"policy_0": tr(b[6])}, {"policy_0": b[7]["policy_0"]},
                   {"policy_0": tr(b[8])}, None, None)
    return buf


@pytest.mark.parametrize("discrete,td3", [(True, False), (True, True), (False, False), (False, True)])
def test_lockstep_train_mpe_maddpg_sizes(gpu_engine, discrete, td3):
    """B = 1000 from 100 000 stored transitions; the batch is the replay's device batch (valid_transition read through its indices).
    Losses to 1e-3; parameters to two Adam steps of lr (a gradient element within round-off of zero may take either sign)."""
    _lockstep_b1000(discrete, td3, N, O, S)


# simple_spread with N agents and N landmarks: observation 6 N, shared observation 6 N^2, critic input 6 N^2 + 5 N = 175 at N = 5 and 246
# at N = 6 -- FFMA k_front_fwd / k_front_bwd on 32-row tiles for the critic and the agent-replaced copies
@pytest.mark.parametrize("n_agents", [5, 6], ids=["spread5_critic175", "spread6_critic246"])
@pytest.mark.parametrize("td3", [False, True], ids=["maddpg", "matd3"])
def test_lockstep_simple_spread_above_128_columns(gpu_engine, n_agents, td3):
    """Three whole updates at B = 1 000 from 100 000 stored transitions against the fp32 oracle, as at simple_spread's 3 agents."""
    _lockstep_b1000(True, td3, n_agents, 6 * n_agents, 6 * n_agents * n_agents)


def _lockstep_b1000(discrete, td3, N, O, S):
    from offpolicy._b200.factory import build_mlp_maddpg
    B = 1000
    torch.manual_seed(8)
    args, pol, tr = build_mlp_maddpg(N, O, A, S, B, discrete=discrete, td3=td3)
    buf = _filled_buffer(B, 100_000, discrete, 9, N, O, S)
    np.random.seed(10)
    L = mc.oracle_from(args, pol)
    # one device batch at a time: a later sample() reuses the batch region
    worst = 0.0
    for k in range(3):
        s = buf.sample(B)
        host = tuple({"policy_0": s.materialize("policy_0", f)} for f in
                     ("obs", "share_obs", "acts", "rewards", "next_obs", "next_share_obs", "dones", "dones_env", "valid_transition")) + \
            ({"policy_0": None}, {"policy_0": None}, None, None)
        before = torch.get_rng_state()
        info, _, _ = tr.shared_train_policy_on_batch("policy_0", s)
        torch.set_rng_state(before)
        ref, _, _ = L.step(host, tr.draw_target_noise(B), tr.draw_actor_noise(B))
        for key, v in ref.items():
            d = abs(float(info[key]) - v) / max(1.0, abs(v))
            worst = max(worst, d)
            assert d <= 1e-3, (k, key, float(info[key]), v)
        pol.soft_target_updates()
        L.soft_update()
        for mod, ref_sd in ((pol.actor, L.actor), (pol.critic, L.critic)):
            for key, v in mod.state_dict().items():
                assert float((v.cpu() - ref_sd[key].detach()).abs().max()) <= 2 * args.lr + 1e-6, key


@pytest.mark.parametrize("discrete,td3", [(True, False), (True, True), (False, False), (False, True)])
def test_graph_replay_equals_eager(gpu_engine, discrete, td3):
    """MaddpgStepGraph (device uniform sample -> step -> soft update) replayed = the same updates run eagerly, bit for bit."""
    from offpolicy._b200.factory import build_mlp_maddpg
    from offpolicy._b200.graph import MaddpgStepGraph
    B = 256
    runs = []
    side = torch.cuda.Stream()                 # a capture needs a non-default stream; eager steps run on the same one
    for mode in ("eager", "graph"):
        with torch.cuda.stream(side):
            torch.manual_seed(21)
            args, pol, tr = build_mlp_maddpg(N, O, A, S, B, discrete=discrete, td3=td3)
            buf = _filled_buffer(B, 4096, discrete, 22)
            buf.seed_device_rng(23)
            if mode == "graph":
                g = MaddpgStepGraph(buf, tr, B)
            infos = []
            for k in range(3):
                torch.manual_seed(100 + k)
                if mode == "eager":
                    batch = buf.sample(B)
                    info, _, _ = tr.shared_train_policy_on_batch("policy_0", batch)
                    pol.soft_target_updates()
                else:
                    g.launch()
                    info = tr._info
                torch.cuda.synchronize()
                infos.append([float(info[i]) for i in ("critic_loss", "critic_grad_norm", "actor_loss", "actor_grad_norm")] if mode == "eager"
                             else [float(tr._info[i]) for i in (0, 1, 4, 5)])
            runs.append((infos, [v.clone() for v in pol.actor_vecs + pol.critic_vecs]))
    assert runs[0][0] == runs[1][0]
    for a, b in zip(runs[0][1], runs[1][1]):
        assert torch.equal(a, b)
