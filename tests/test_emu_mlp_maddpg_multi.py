"""Transition-level MADDPG / MATD3 with one policy per agent (share_policy off) on the CPU-emulated kernels: the fixtures of the
unmodified reference (tests/golden/mlp_*_multi_*.npz), lock-step against oracle/maddpg_mlp_multi.py, the multi-policy transition
replay, the configurations that still raise and, where the reference checkout is present, the unmodified MLP runner with
`--share_policy` against the pure reference."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import mlp_maddpg_multi_checks as mm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("OFFPOLICY_REFERENCE_ROOT", "/root/reference")
SL = [(3, 3), (11, 5)]           # simple_speaker_listener: speaker obs 3, Discrete(3); listener obs 11, Discrete(5); share 14
SL_S = 14


@pytest.mark.parametrize("name", mm.GOLDENS_MULTI)
def test_oracle_reproduces_reference_multi(name):
    """Losses 1e-6, tensors 2e-5, the oracle's own draws equal to the reference's from the same RNG states."""
    mm.oracle_against_golden(name)


@pytest.mark.parametrize("name", mm.GOLDENS_MULTI)
def test_engine_reproduces_reference_multi(emu_engine, name):
    mm.engine_against_golden(name)


LOCKSTEP = {
    # name: (specs, S, discrete, td3, avail, ties, args overrides)
    "maddpg_disc_sl": (SL, SL_S, True, False, False, False, {}),
    "matd3_disc_sl": (SL, SL_S, True, True, False, False, {}),
    "maddpg_box_3pol": ([(6, 2), (9, 3), (4, 1)], 19, False, False, False, False, {}),
    "matd3_box_3pol": ([(6, 2), (9, 3), (4, 1)], 19, False, True, False, False, {}),
    "maddpg_disc_avail_ties": (SL, SL_S, True, False, True, True, {}),
    "matd3_disc_avail": (SL, SL_S, True, True, True, False, {}),
    "maddpg_per_huber": (SL, SL_S, True, False, False, False, {"use_per": True, "use_huber_loss": True, "huber_delta": 1.0}),
    # one policy with two agents: its agents sit at a non-zero act_offset, one after the other
    "maddpg_disc_two_agent_policy": ([(5, 3), (7, 4, 2), (6, 2)], 16, True, False, True, False, {}),
    "matd3_box_two_agent_policy": ([(5, 2, 2), (7, 3), (6, 1, 2)], 16, False, True, False, False, {}),
}


@pytest.mark.parametrize("name", list(LOCKSTEP))
def test_lockstep_multi_against_oracle(emu_engine, name):
    from offpolicy._b200.factory import build_mlp_maddpg_multi
    specs, S, discrete, td3, avail, ties, over = LOCKSTEP[name]
    torch.manual_seed(5)
    B = 24
    args, pols, tr, _ = build_mlp_maddpg_multi(specs, S, B, discrete=discrete, td3=td3, **over)
    rng = np.random.default_rng(7)
    batches = [mm.synth_batch_multi(rng, specs, B, S, discrete, avail=avail, ties=ties, per=args.use_per) for _ in range(2)]
    mm.lockstep_multi(args, pols, tr, batches)


def test_single_policy_calls_unchanged(emu_engine):
    """With one policy the per-policy helpers default to it: the draws and views of the shared-policy trainer."""
    from offpolicy._b200.factory import build_mlp_maddpg
    torch.manual_seed(1)
    args, pol, tr = build_mlp_maddpg(3, 18, 5, 54, 8, discrete=True, td3=True)
    st = torch.get_rng_state()
    a = tr.draw_target_noise(8)
    torch.set_rng_state(st)
    b = tr.draw_target_noise(8, "policy_0")
    assert a.shape == (24, 5) and torch.equal(a, b)
    assert tr.draw_actor_noise(8).shape == (24, 5)
    ga, gc = tr.grad_views()
    assert ga.numel() == pol.Pa + 4 and gc.numel() == pol.Pc + 4


def test_cent_act_dim_mismatch_raises(emu_engine):
    from offpolicy._b200.factory import Discrete, Box, mlp_maddpg_args
    from offpolicy._b200 import capi
    from offpolicy.algorithms.maddpg.algorithm.MADDPGPolicy import MADDPGPolicy
    from offpolicy.algorithms.maddpg.maddpg import MADDPG
    args = mlp_maddpg_args(8)
    mk = lambda o, a, ca: MADDPGPolicy({"args": args, "device": capi.device()}, dict(obs_space=Box(o), share_obs_space=Box(6),
                                                                                   act_space=Discrete(a), cent_obs_dim=6, cent_act_dim=ca))
    pols = {"policy_0": mk(3, 3, 8), "policy_1": mk(4, 5, 7)}
    with pytest.raises(ValueError):
        MADDPG(args, 2, pols, lambda k: "policy_%d" % k)


def test_unsupported_multi_configurations_raise(emu_engine):
    from offpolicy._b200.factory import build_mlp_maddpg_multi, LearnerConfig, qmix_args, _policy_info
    from offpolicy._b200 import capi
    with pytest.raises(NotImplementedError):
        build_mlp_maddpg_multi(SL, SL_S, 8, use_popart=True)
    args, pols, tr, _ = build_mlp_maddpg_multi(SL, SL_S, 8)
    with pytest.raises(NotImplementedError):
        tr.cent_train_policy_on_batch("policy_0", None)
    # M-QMIX / M-VDN with several policies: the buffer accepts them, the trainer does not
    from offpolicy.algorithms.mqmix.algorithm.mQMixPolicy import M_QMixPolicy
    from offpolicy.algorithms.mqmix.mqmix import M_QMix
    cfg = LearnerConfig()
    qa = qmix_args(cfg, 8)
    qp = {"policy_%d" % i: M_QMixPolicy({"args": qa, "device": capi.device()}, _policy_info(cfg)) for i in range(3)}
    for vdn in (False, True):
        with pytest.raises(NotImplementedError):
            M_QMix(qa, 3, qp, lambda k: "policy_%d" % k, device=capi.device(), vdn=vdn)


def test_graph_capture_of_multi_policy_learner_fails(emu_engine):
    from offpolicy._b200 import capi
    from offpolicy._b200.factory import build_mlp_maddpg_multi
    B = 8
    args, pols, tr, agents = build_mlp_maddpg_multi(SL, SL_S, B)
    buf = _multi_buffer(SL, SL_S, B, 64, True, 3)
    lib = capi.lib()
    e = tr._eng["policy_0"]
    g = C.c_void_p()
    rc = lib.mx_maddpg_graph_capture(buf.policy_buffers["policy_0"].rep.handle, e.handle, B, 0.0, 1, None, None, 1, capi.stream_ptr(),
                                     C.byref(g))
    assert rc != 0
    assert b"several policies" in lib.mx_last_error()


# ---- the multi-policy transition replay ---------------------------------------------------------------------------------------------
def _multi_buffer(specs, S, B, size, discrete, seed, per_alpha=None, rng="numpy", avail=False):
    from offpolicy._b200.factory import Box, Discrete
    from offpolicy.utils.mlp_buffer import MlpReplayBuffer, PrioritizedMlpReplayBuffer
    shapes = mm.norm_specs(specs)
    info = {p: dict(obs_space=Box(o), share_obs_space=Box(S), act_space=Discrete(a) if discrete else Box(a)) for p, (o, a, n) in shapes.items()}
    agents, nxt = {}, 0
    for p, (o, a, n) in shapes.items():
        agents[p] = list(range(nxt, nxt + n))
        nxt += n
    if per_alpha is None:
        buf = MlpReplayBuffer(info, agents, size, True, avail, max_batch=B, rng=rng)
    else:
        buf = PrioritizedMlpReplayBuffer(per_alpha, info, agents, size, True, avail, max_batch=B, rng=rng)
    r = np.random.default_rng(seed)
    tr = lambda x: np.asarray(x).transpose(1, 0, 2)                     # (N, B, .) -> the runner's (B, N, .)
    stored = []
    for _ in range(size // B):
        b = mm.synth_batch_multi(r, specs, B, S, discrete, avail=avail)
        per_p = lambda i, t=True: {p: (tr(b[i][p]) if t else b[i][p]) for p in shapes}
        buf.insert(B, per_p(0), per_p(1, False), per_p(2), per_p(3), per_p(4), per_p(5, False), per_p(6), per_p(7, False), per_p(8),
                   per_p(9) if avail else None, per_p(10) if avail else None)
        stored.append(b)
    return buf if not stored else _Stored(buf, stored, shapes)


class _Stored(object):
    """The buffer plus what was inserted, row-major per policy: the NumPy restatement materialize is checked against."""

    def __init__(self, buf, batches, shapes):
        self.buf, self.shapes = buf, shapes
        cat = lambda i, p, axis: np.concatenate([b[i][p] for b in batches], axis)
        self.rows = {p: {f: (cat(i, p, 0) if f in ("share_obs", "next_share_obs", "dones_env") else cat(i, p, 1))
                         for i, f in enumerate(mm.FIELDS) if batches[0][i][p] is not None} for p in shapes}

    def __getattr__(self, k):
        return getattr(self.buf, k)

    def expect(self, p, f, inds):
        v = self.rows[p][f]
        if f in ("share_obs", "next_share_obs", "dones_env"):
            return v[inds]
        return v[:, inds]


SPECS3 = [(5, 3), (7, 4, 2), (6, 2)]


@pytest.mark.parametrize("rng", ["numpy", "device"])
def test_multi_buffer_shares_one_index_set(emu_engine, rng):
    B, S = 16, 12
    st = _multi_buffer(SPECS3, S, B, 128, True, 4, rng=rng, avail=True)
    if rng == "device":
        st.buf.seed_device_rng(11)
    np.random.seed(2)
    expect_inds = np.random.randint(0, 128, B) if rng == "numpy" else None
    np.random.seed(2)
    s = st.buf.sample(B)
    inds = [np.asarray(st.buf.policy_buffers[p].rep.sampled_indices(B)) for p in sorted(st.shapes)]
    for i in inds[1:]:
        assert np.array_equal(i, inds[0])
    if expect_inds is not None:
        assert np.array_equal(inds[0], expect_inds)          # one np.random.randint(0, len, B) call
    assert len(st.buf) == 128
    for p in sorted(st.shapes):
        for f in mm.FIELDS:
            got = s.materialize(p, f)
            want = st.expect(p, f, inds[0])
            assert got.shape == want.shape, (p, f)
            assert np.array_equal(got, want), (p, f)
        # the device valid_transition store of each policy has that policy's width
        assert tuple(st.buf.policy_buffers[p].valid_dev.shape) == (128, st.shapes[p][2])


@pytest.mark.parametrize("rng", ["numpy", "device"])
def test_multi_buffer_per_uses_the_updated_policys_tree(emu_engine, rng):
    B, S = 8, 12
    st = _multi_buffer(SPECS3, S, B, 64, True, 5, per_alpha=0.6, rng=rng)
    buf = st.buf
    if rng == "device":
        buf.seed_device_rng(3)
    np.random.seed(1)
    trees0 = {p: [t.copy() for t in buf.policy_buffers[p].rep.tree_values()] for p in st.shapes}
    # make policy_1's tree very different: everything but row 7 at a tiny priority
    idx = np.arange(64)
    pr = np.full(64, 1e-9, np.float32)
    pr[7] = 100.0
    buf.update_priorities(idx, pr, "policy_1")
    for p in ("policy_0", "policy_2"):                          # written back to p's tree only
        for a, b in zip(buf.policy_buffers[p].rep.tree_values(), trees0[p]):
            assert np.array_equal(a, b), p
    assert not np.array_equal(buf.policy_buffers["policy_1"].rep.tree_values()[0], trees0["policy_1"][0])
    s = buf.sample(B, 0.4, "policy_1")
    got = np.asarray(s[12])
    assert np.all(got == 7)                                     # drawn from policy_1's tree
    for p in st.shapes:
        assert np.array_equal(np.asarray(buf.policy_buffers[p].rep.sampled_indices(B)), got), p
        assert np.array_equal(s.materialize(p, "obs"), st.expect(p, "obs", got)), p
    s0 = buf.sample(B, 0.4, "policy_0")                         # policy_0's tree is still uniform
    assert len(set(np.asarray(s0[12]).tolist())) > 1


def test_multi_buffer_device_batch_trains_like_host_batch(emu_engine):
    """The trainer on the replay's device batch (valid_transition through the sampled indices) = the same sample materialised."""
    from offpolicy._b200.factory import build_mlp_maddpg_multi
    B, S = 16, 16
    specs = [(5, 3), (7, 4, 2), (6, 2)]
    st = _multi_buffer(specs, S, B, 128, True, 8)
    res = []
    for mode in ("device", "host"):
        torch.manual_seed(4)
        args, pols, tr, _ = build_mlp_maddpg_multi(specs, S, B, discrete=True, td3=True)
        np.random.seed(6)
        out = []
        for p in sorted(pols):
            s = st.buf.sample(B)
            batch = s if mode == "device" else \
                tuple({q: s.materialize(q, f) for q in pols} for f in mm.FIELDS[:9]) + ({q: None for q in pols}, {q: None for q in pols}, None, None)
            info, _, _ = tr.shared_train_policy_on_batch(p, batch)
            out.append([float(info[k]) for k in ("critic_loss", "critic_grad_norm", "actor_loss", "actor_grad_norm")])
        res.append((out, [v.clone() for q in sorted(pols) for v in pols[q].actor_vecs[:1] + pols[q].critic_vecs[:1]]))
    assert res[0][0] == res[1][0]
    for a, b in zip(res[0][1], res[1][1]):
        assert torch.equal(a, b)


# ---- the unmodified reference runner with --share_policy ----------------------------------------------------------------------------
@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "offpolicy", "runner")), reason="reference checkout not present")
@pytest.mark.parametrize("norm", [False, True])
@pytest.mark.parametrize("algo", ["maddpg", "matd3"])
def test_mlp_runner_share_policy(emu_engine, algo, norm):
    """runner/mlp with one policy per agent (separated_collect_rollout, batch_train over every policy): identical episodes, train_info
    of every policy's every update to fp32 round-off."""
    out, procs = {}, {}
    for eng in ("b200", "reference"):
        cmd = [sys.executable, os.path.join(ROOT, "tests", "integration", "run_mpe.py"), "--engine", eng, "--algo", algo, "--steps", "150",
               "--runner", "mlp", "--share_policy"] + (["--use_reward_normalization"] if norm else [])
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
