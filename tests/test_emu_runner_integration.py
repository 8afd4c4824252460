"""Drop-in claim, end to end (SURVEY.md section 8(b)): the UNMODIFIED reference runners -- offpolicy/runner/rnn/mpe_runner.py on MPE
simple_spread (what scripts/train_mpe_{qmix,vdn,rmaddpg,rmatd3}.sh start) and offpolicy/runner/rnn/smac_runner.py on a synthetic
environment with the SMAC 3m interface (StarCraft II is not installable here) -- are run twice with the same seed: once on the
reference's own buffer / policy / trainer classes, once with this repository's `offpolicy` package shadowing them (kernels on the
CPU fiber emulator).  Warm-up, epsilon-greedy / Gumbel exploration, episode insertion, sampling, training and target updates all
go through the runner's own code.  The two runs must collect IDENTICAL episodes (bit-equal rewards: same generator draws in the same
order, same actions) and report the same train_info to fp32 round-off.

Needs the reference checkout (it is the thing being run); skipped where it is absent (the GPU box).
"""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("OFFPOLICY_REFERENCE_ROOT", "/root/reference")
pytestmark = pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "offpolicy", "runner")), reason="reference checkout not present")

RUNS = {
    # name: (algorithm, env steps, extra reference flags, compare against the pure reference?)   [name smac_*: run_smac_like.py]
    # also exercises the runner's periodic evaluation (greedy rollouts) and checkpoint saving (state_dict -> torch.save)
    "qmix": ("qmix", 125, ["--save_interval", "50", "--use_eval", "--eval_interval", "75", "--num_eval_episodes", "2"], True),
    # scripts/train_mpe_qmix.sh:14 normalises rewards; `--use_soft_update` is a store_false flag, i.e. HARD target updates every
    # hard_update_interval_episode episodes like the shipped train_smac_qmix.sh (SURVEY.md App. D-12)
    "qmix_reward_norm": ("qmix", 125, ["--use_reward_normalization", "--use_soft_update", "--hard_update_interval_episode", "2"], True),
    # network input [obs | previous action]; the reference's own rollout path raises with this flag (QMixPolicy.py:54-58 concatenates a
    # NumPy observation with a tensor), so only its learner is pinned (golden qmix_small_prev_act) and the runner runs on the drop-in
    "qmix_prev_act": ("qmix", 100, ["--prev_act_inp"], False),
    "rmaddpg": ("rmaddpg", 125, ["--actor_train_interval_step", "1", "--save_interval", "50"], True),
    "rmatd3": ("rmatd3", 125, ["--actor_train_interval_step", "1"], True),
    # scripts/train_mpe_rmaddpg.sh passes `--share_policy` (store_false: ONE POLICY PER AGENT, train/train_mpe.py:139-150) and
    # --use_reward_normalization.  Its scenario (simple_speaker_listener: different observation widths per agent) cannot be stepped by the
    # reference's own DummyVecEnv under NumPy >= 1.24 (np.array of ragged observations raises, envs/env_wrappers.py), so the runner runs
    # simple_spread with three per-agent policies; the heterogeneous shapes are pinned by the *_multi_* goldens (tests/test_emu_maddpg.py)
    "rmaddpg_per_agent": ("rmaddpg", 125, ["--actor_train_interval_step", "1", "--share_policy", "--use_reward_normalization"], True),
    "rmatd3_per_agent": ("rmatd3", 125, ["--actor_train_interval_step", "1", "--share_policy"], True),
    "qmix_per": ("qmix", 100, ["--use_per"], False),   # the reference's PER insert raises IndexError for 1-episode inserts (App. D-2): drop-in only
    "vdn": ("vdn", 100, [], False),          # the reference's recurrent VDN mixer is shape-broken (SURVEY.md App. D-1): drop-in only
    # offpolicy/runner/rnn/smac_runner.py (scripts/train_smac_qmix.sh) on a synthetic env with the 3m interface: availability masks
    # that change every step (the env asserts no unavailable action is ever chosen), early termination, episode limit 60
    "smac_qmix": ("qmix", 220, [], True),
    "smac_qmix_per_hard": ("qmix", 200, ["--use_per", "--use_soft_update", "--hard_update_interval_episode", "2"], False),
    # offpolicy/runner/mlp/mpe_runner.py (the transition-level algorithms, SURVEY.md section 8(f).4): M_QMix on MlpReplayBuffer
    "mlp_mqmix": ("mqmix", 150, ["--runner", "mlp"], True),
    "mlp_mqmix_reward_norm": ("mqmix", 125, ["--runner", "mlp", "--use_reward_normalization"], True),
    "mlp_mqmix_per": ("mqmix", 100, ["--runner", "mlp", "--use_per"], False),       # reference PER insert bug (mlp_buffer.py:282)
    "mlp_mvdn": ("mvdn", 100, ["--runner", "mlp"], False),                         # reference M_VDNMixer is broken (App. D-5)
    # MLP MADDPG / MATD3 have no B200 learner (SURVEY.md App. D-6): the shadow package lets them fall through to the reference's own
    # trainer, which then trains from the HBM transition replay (its sample materialises the reference's 13-tuple) -- same run, bit for bit
    # --use_feature_normalization is a store_false flag: the networks lose their input LayerNorm (rollout kernel + learner)
    "qmix_no_feature_norm": ("qmix", 100, ["--use_feature_normalization"], True),
    "mlp_mqmix_no_feature_norm": ("mqmix", 100, ["--runner", "mlp", "--use_feature_normalization"], True),
    # --use_ReLU is a store_false flag too: tanh networks (different init gain, mlp.py:12), rollout kernel + learner
    "qmix_tanh": ("qmix", 100, ["--use_ReLU"], True),
    "rmaddpg_tanh": ("rmaddpg", 100, ["--actor_train_interval_step", "1", "--use_ReLU"], True),
    "rmatd3_no_feature_norm": ("rmatd3", 100, ["--actor_train_interval_step", "1", "--use_feature_normalization"], True),
    "mlp_maddpg": ("maddpg", 100, ["--runner", "mlp"], True),
    "mlp_matd3": ("matd3", 100, ["--runner", "mlp"], True),
    # simple_spread with 5 agents (3 landmarks): observation 26, shared observation 130, critic input 130 + 5 x 5 = 155 -- above 128
    # columns, FFMA k_front_fwd / k_front_bwd on 32-row tiles for the critic and its agent-replaced copies
    "mlp_maddpg_5_agents": ("maddpg", 100, ["--runner", "mlp", "--agents", "5"], True),
}


def _start(engine, algo, steps, extra, script):
    cmd = [sys.executable, os.path.join(ROOT, "tests", "integration", script), "--engine", engine, "--algo", algo, "--steps", str(steps)] + extra
    return subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=dict(os.environ, OMP_NUM_THREADS="1"))


@pytest.fixture(scope="module")
def results(emu_engine):
    procs = {}
    for name, (algo, steps, extra, vs_ref) in RUNS.items():
        script = "run_smac_like.py" if name.startswith("smac_") else "run_mpe.py"
        procs[(name, "b200")] = _start("b200", algo, steps, extra, script)
        if vs_ref:
            procs[(name, "reference")] = _start("reference", algo, steps, extra, script)
    out = {}
    for key, p in procs.items():
        so, se = p.communicate(timeout=1500)
        assert p.returncode == 0, "%s failed:\n%s" % (key, se.decode()[-3000:])
        out[key] = json.loads(so.decode().strip().splitlines()[-1])
    return out


@pytest.mark.parametrize("name", list(RUNS))
def test_reference_runner_on_the_drop_in_engine(results, name):
    algo, steps, extra, vs_ref = RUNS[name]
    ours = results[(name, "b200")]
    assert "off-policy_b200" in ours["buffer"], ours["buffer"]                     # the shadow package really was the one in use
    assert ours["env_steps"] >= steps and ours["train_steps"] > 0 and len(ours["rewards"]) >= 2
    for info in ours["train"]:
        assert all(v == v and abs(v) < 1e9 for v in info.values()), info            # finite
    if not vs_ref:
        return
    ref = results[(name, "reference")]
    assert REF in ref["buffer"]
    assert ours["train_steps"] == ref["train_steps"]
    assert ours["rewards"] == ref["rewards"], (ours["rewards"], ref["rewards"])      # identical episodes, bit for bit
    assert len(ours["train"]) == len(ref["train"]) > 0
    for a, b in zip(ours["train"], ref["train"]):
        assert set(a) == set(b)
        for k in a:
            assert abs(a[k] - b[k]) <= 2e-5 * max(1.0, abs(b[k])), (name, k, a[k], b[k])
