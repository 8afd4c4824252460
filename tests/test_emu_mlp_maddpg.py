"""Transition-level MADDPG / MATD3 (algorithms/maddpg, algorithms/matd3) on the CPU-emulated kernels: lock-step against
oracle/maddpg_mlp.py and the frozen critic heads (construction, keys and RNG consumption against the reference: test_mlp_maddpg_goldens.py); and, where the reference checkout
is present, the unmodified MLP runner (runner/mlp/mpe_runner.py) with the script's reward normalisation against the pure reference."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import mlp_maddpg_checks as mc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("OFFPOLICY_REFERENCE_ROOT", "/root/reference")
# simple_spread shapes (scripts/train_mpe_maddpg.sh): 3 agents, obs 18, Discrete(5), shared observation 54
N, O, A, S = 3, 18, 5, 54

CASES = {
    # name: (discrete, td3, avail, ties, args overrides)
    "maddpg_disc": (True, False, False, False, {}),
    "matd3_disc": (True, True, False, False, {}),
    "maddpg_box": (False, False, False, False, {}),
    "matd3_box": (False, True, False, False, {}),
    "maddpg_disc_avail": (True, False, True, True, {}),
    "matd3_disc_avail": (True, True, True, False, {}),
    "maddpg_per_huber": (True, False, False, False, {"use_per": True, "use_huber_loss": True, "huber_delta": 1.0}),
    "maddpg_box_tanh_wd": (False, False, False, False, {"use_ReLU": False, "weight_decay": 1e-3}),
}


@pytest.mark.parametrize("name", list(CASES))
def test_lockstep_against_oracle(emu_engine, name):
    from offpolicy._b200.factory import build_mlp_maddpg
    discrete, td3, avail, ties, over = CASES[name]
    torch.manual_seed(5)
    B = 24
    args, pol, tr = build_mlp_maddpg(N, O, A, S, B, discrete=discrete, td3=td3, **over)
    rng = np.random.default_rng(7)
    batches = [mc.synth_batch(rng, N, B, O, S, A, discrete, avail=avail, ties=ties, per=args.use_per) for _ in range(3)]
    mc.lockstep(args, pol, tr, batches)


def test_hard_update_keeps_the_heads(emu_engine):
    from offpolicy._b200.factory import build_mlp_maddpg
    torch.manual_seed(2)
    args, pol, tr = build_mlp_maddpg(N, O, A, S, 16, discrete=True, td3=True)
    rng = np.random.default_rng(1)
    L = mc.oracle_from(args, pol)
    th = {k: v.clone() for k, v in pol.target_critic_heads.state_dict().items()}
    tr.shared_train_policy_on_batch("policy_0", mc.synth_batch(rng, N, 16, O, S, A, True))
    pol.hard_target_updates()
    for k, v in pol.target_critic.state_dict().items():
        assert torch.equal(v, pol.critic.state_dict()[k]), k
    for k, v in pol.target_critic_heads.state_dict().items():
        assert torch.equal(v, th[k]), k
    assert torch.equal(pol.actor_vecs[1], pol.actor_vecs[0])
    del L


def test_unsupported_configurations_raise(emu_engine):
    from offpolicy._b200.factory import build_mlp_maddpg
    with pytest.raises(NotImplementedError):
        build_mlp_maddpg(N, O, A, S, 8, use_popart=True)
    args, pol, tr = build_mlp_maddpg(N, O, A, S, 8)
    with pytest.raises(NotImplementedError):
        tr.cent_train_policy_on_batch("policy_0", None)


def test_drop_in_modules_resolve_to_this_repository():
    sys.path.insert(0, os.path.join(ROOT, "off-policy_b200"))
    import offpolicy.algorithms.maddpg.maddpg as m1
    import offpolicy.algorithms.matd3.matd3 as m2
    import offpolicy.algorithms.maddpg.algorithm.MADDPGPolicy as p1
    import offpolicy.algorithms.matd3.algorithm.MATD3Policy as p2
    for m in (m1, m2, p1, p2):
        assert os.path.realpath(m.__file__).startswith(os.path.realpath(os.path.join(ROOT, "off-policy_b200"))), m.__file__


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "offpolicy", "runner")), reason="reference checkout not present")
@pytest.mark.parametrize("algo", ["maddpg", "matd3"])
def test_mlp_runner_with_reward_normalization(emu_engine, algo):
    """scripts/train_mpe_maddpg.sh's flags on the unmodified runner: identical episodes, train_info to fp32 round-off."""
    out = {}
    procs = {}
    for eng in ("b200", "reference"):
        cmd = [sys.executable, os.path.join(ROOT, "tests", "integration", "run_mpe.py"), "--engine", eng, "--algo", algo, "--steps", "150",
               "--runner", "mlp", "--use_reward_normalization"]
        procs[eng] = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=dict(os.environ, OMP_NUM_THREADS="1"))
    for eng, p in procs.items():
        so, se = p.communicate(timeout=1500)
        assert p.returncode == 0, se.decode()[-3000:]
        out[eng] = json.loads(so.decode().strip().splitlines()[-1])
    ours, ref = out["b200"], out["reference"]
    assert ours["trainer"] == "offpolicy.algorithms.%s.%s" % (algo, algo) and "off-policy_b200" in ours["buffer"]
    assert ours["train_steps"] == ref["train_steps"] > 0
    assert ours["rewards"] == ref["rewards"]
    assert len(ours["train"]) == len(ref["train"]) > 0
    for a, b in zip(ours["train"], ref["train"]):
        assert set(a) == set(b)
        for k in a:
            assert abs(a[k] - b[k]) <= 2e-5 * max(1.0, abs(b[k])), (k, a[k], b[k])
