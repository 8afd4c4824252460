"""Transition-level MADDPG / MATD3 with one policy per agent on the real sm_90a kernels: the fixtures of the unmodified reference,
lock-step against oracle/maddpg_mlp_multi.py at small batches, and at B = 1000 drawn from a 100 000-transition multi-policy replay
(simple_speaker_listener and 3-agent simple_spread shapes, one policy per agent) with the replay's device batch."""
import numpy as np
import pytest
import torch

import mlp_maddpg_multi_checks as mm
from mlp_maddpg_checks import oracle_from
from oracle.maddpg_mlp_multi import draw_noise_multi, step_multi

pytestmark = pytest.mark.gpu
SL, SL_S = [(3, 3), (11, 5)], 14                  # simple_speaker_listener
SPREAD, SPREAD_S = [(18, 5)] * 3, 54              # simple_spread, one policy per agent


@pytest.mark.parametrize("name", mm.GOLDENS_MULTI)
def test_engine_reproduces_reference_multi(gpu_engine, name):
    mm.engine_against_golden(name)


@pytest.mark.parametrize("specs,S,discrete,td3,avail,over", [
    (SL, SL_S, True, False, True, {}),
    (SL, SL_S, True, True, False, {}),
    ([(6, 2), (9, 3, 2), (4, 1)], 19, False, False, False, {}),
    ([(6, 2), (9, 3, 2), (4, 1)], 19, False, True, False, {}),
    (SL, SL_S, True, False, False, {"use_per": True, "use_huber_loss": True, "huber_delta": 1.0}),
])
def test_lockstep_multi_small(gpu_engine, specs, S, discrete, td3, avail, over):
    from offpolicy._b200.factory import build_mlp_maddpg_multi
    torch.manual_seed(3)
    B = 32
    args, pols, tr, _ = build_mlp_maddpg_multi(specs, S, B, discrete=discrete, td3=td3, **over)
    rng = np.random.default_rng(4)
    mm.lockstep_multi(args, pols, tr, [mm.synth_batch_multi(rng, specs, B, S, discrete, avail=avail, ties=avail, per=args.use_per)
                                       for _ in range(2)])


_BUFFERS = {}


def _filled_multi_buffer(specs, S, B, size, discrete, seed):
    """One filled replay per shape, shared by the tests of this module (a store's host fences are process-wide and never freed)."""
    key = (tuple(specs), S, B, size, discrete, seed)
    if key not in _BUFFERS:
        _BUFFERS[key] = _fill_multi_buffer(specs, S, B, size, discrete, seed)
    return _BUFFERS[key]


def _fill_multi_buffer(specs, S, B, size, discrete, seed):
    from offpolicy._b200.factory import Box, Discrete
    from offpolicy.utils.mlp_buffer import MlpReplayBuffer
    shapes = mm.norm_specs(specs)
    info = {p: dict(obs_space=Box(o), share_obs_space=Box(S), act_space=Discrete(a) if discrete else Box(a)) for p, (o, a, n) in shapes.items()}
    agents, nxt = {}, 0
    for p, (o, a, n) in shapes.items():
        agents[p] = list(range(nxt, nxt + n))
        nxt += n
    buf = MlpReplayBuffer(info, agents, size, True, False, max_batch=B)
    rng = np.random.default_rng(seed)
    tr = lambda x: np.asarray(x).transpose(1, 0, 2)
    for _ in range(size // B):
        b = mm.synth_batch_multi(rng, specs, B, S, discrete)
        per_p = lambda i, t=True: {p: (tr(b[i][p]) if t else b[i][p]) for p in shapes}
        buf.insert(B, per_p(0), per_p(1, False), per_p(2), per_p(3), per_p(4), per_p(5, False), per_p(6), per_p(7, False), per_p(8), None, None)
    buf.seed_device_rng(seed)          # the index set is drawn on the first store and gathered into the others on the device
    return buf


@pytest.mark.parametrize("specs,S", [(SL, SL_S), (SPREAD, SPREAD_S)], ids=["speaker_listener", "spread_per_agent"])
@pytest.mark.parametrize("discrete,td3", [(True, False), (True, True), (False, False), (False, True)])
def test_lockstep_multi_train_sizes(gpu_engine, specs, S, discrete, td3):
    """B = 1000 from 100 000 stored transitions, one sample per policy update (the runner's batch_train) as the replay's device batch.
    Losses to 1e-3; parameters to two Adam steps of lr (a gradient element within round-off of zero may take either sign)."""
    from offpolicy._b200.factory import build_mlp_maddpg_multi
    B = 1000
    torch.manual_seed(8)
    args, pols, tr, _ = build_mlp_maddpg_multi(specs, S, B, discrete=discrete, td3=td3)
    buf = _filled_multi_buffer(specs, S, B, 100_000, discrete, 9)
    learners = {p: oracle_from(args, pol) for p, pol in pols.items()}
    shapes = mm.noise_shapes(tr)
    for k in range(2):
        for p in sorted(pols):
            s = buf.sample(B)          # one device batch at a time: a later sample() reuses the batch region
            host = tuple({q: s.materialize(q, f) for q in pols} for f in mm.FIELDS[:9]) + \
                ({q: None for q in pols}, {q: None for q in pols}, None, None)
            before = torch.get_rng_state()
            info, _, _ = tr.shared_train_policy_on_batch(p, s)
            torch.set_rng_state(before)
            tn, an = draw_noise_multi(shapes, p, B)
            ref, _, _ = step_multi(learners, p, host, tn, an)
            for key, v in ref.items():
                d = abs(float(info[key]) - v) / max(1.0, abs(v))
                assert d <= 1e-3, (k, p, key, float(info[key]), v)
        for p in sorted(pols):
            pols[p].soft_target_updates()
            learners[p].soft_update()
        for p, pol in pols.items():
            for mod, ref_sd in ((pol.actor, learners[p].actor), (pol.critic, learners[p].critic)):
                for key, v in mod.state_dict().items():
                    assert float((v.cpu() - ref_sd[key].detach()).abs().max()) <= 2 * args.lr + 1e-6, (p, key)
