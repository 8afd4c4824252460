"""Transition-level MADDPG / MATD3 with MultiDiscrete action spaces (simple_reference: move Discrete(5) + speak Discrete(10)) on the
CPU-emulated kernels: the engine against the fixtures of the unmodified reference, lock-step against oracle/maddpg_mlp_md.py,
get_actions / get_random_actions against the reference's per-sub-space calls, the replay storing the concatenated one-hot blocks, the
learner's refusal of bad segment lists and, where the reference checkout is present, the unmodified MLP runner on simple_reference."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import mlp_maddpg_md_checks as mdc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("OFFPOLICY_REFERENCE_ROOT", "/root/reference")
N, O, S, SEGS = mdc.N, mdc.O, mdc.S, mdc.SEGS


@pytest.mark.parametrize("name", mdc.GOLDENS_MD)
def test_engine_reproduces_reference(emu_engine, name):
    mdc.engine_against_golden(name)


LOCKSTEP = {
    # name: (specs, td3, avail, args overrides)
    "maddpg": (mdc.REFERENCE_SPEC, False, False, {}),
    "matd3": (mdc.REFERENCE_SPEC, True, False, {}),
    "maddpg_per_huber": (mdc.REFERENCE_SPEC, False, False, {"use_per": True, "use_huber_loss": True, "huber_delta": 1.0}),
    "matd3_tanh_wd": (mdc.REFERENCE_SPEC, True, False, {"use_ReLU": False, "weight_decay": 1e-3}),
    "maddpg_avail_ignored": (mdc.REFERENCE_SPEC, False, True, {}),
    "matd3_avail_ignored": (mdc.REFERENCE_SPEC, True, True, {}),
    "matd3_three_segments": ([(9, [3, 4, 2], 3)], True, False, {}),
    "matd3_mixed_policies": ([(11, 5), (9, [5, 4]), (7, [2, 3, 2], 2)], True, False, {}),
    "maddpg_mixed_policies": ([(11, 5), (9, [5, 4])], False, False, {}),
}


@pytest.mark.parametrize("name", list(LOCKSTEP))
def test_lockstep_against_oracle(emu_engine, name):
    """The oracle ignores the available-action masks of MultiDiscrete policies, so the *_avail_ignored cases check the engine does too."""
    from offpolicy._b200.factory import build_mlp_maddpg_multi
    specs, td3, avail, over = LOCKSTEP[name]
    torch.manual_seed(5)
    B, S2 = 24, 30
    args, pols, tr, _ = build_mlp_maddpg_multi(specs, S2, B, discrete=True, td3=td3, **over)
    rng = np.random.default_rng(7)
    batches = [mdc.synth_batch_md(rng, specs, B, S2, per=args.use_per, avail=avail) for _ in range(3)]
    mdc.lockstep(args, pols, tr, batches)


def test_avail_batch_trains_like_no_avail(emu_engine):
    """A batch whose masks are full of zeros trains a MultiDiscrete learner exactly as the same batch without masks."""
    from offpolicy._b200.factory import build_mlp_maddpg
    res = []
    for with_avail in (True, False):
        torch.manual_seed(9)
        args, pol, tr = build_mlp_maddpg(N, O, SEGS, S, 16, td3=True)
        rng = np.random.default_rng(3)
        out = []
        for _ in range(2):
            b = list(mdc.synth_batch_md(rng, mdc.REFERENCE_SPEC, 16, S, avail=True))
            if not with_avail:
                b[9], b[10] = {"policy_0": None}, {"policy_0": None}
            info, _, _ = tr.shared_train_policy_on_batch("policy_0", tuple(b))
            out.append([float(info[k]) for k in ("critic_loss", "critic_grad_norm", "actor_loss", "actor_grad_norm")])
        res.append((out, [v.clone() for v in pol.actor_vecs + pol.critic_vecs]))
    assert res[0][0] == res[1][0]
    for a, b in zip(res[0][1], res[1][1]):
        assert torch.equal(a, b)


def test_policy_exposes_reference_dims(emu_engine):
    """act_dim is the ndarray of sub-space widths (the MLP runner takes np.sum of it), output_dim the int sum; the actor's head keys are
    act.action_outs.i, consecutive row blocks of one head in the flat vector."""
    from offpolicy._b200.factory import build_mlp_maddpg
    torch.manual_seed(1)
    args, pol, tr = build_mlp_maddpg(N, O, SEGS, S, 8)
    assert isinstance(pol.act_dim, np.ndarray) and pol.act_dim.tolist() == SEGS and int(np.sum(pol.act_dim)) == 15
    assert pol.output_dim == 15 and isinstance(pol.output_dim, int) and pol.multidiscrete and pol.discrete
    sd = pol.actor.state_dict()
    assert [k for k in sd if k.startswith("act.")] == ["act.action_outs.0.weight", "act.action_outs.0.bias", "act.action_outs.1.weight",
                                                       "act.action_outs.1.bias"]
    assert tuple(sd["act.action_outs.0.weight"].shape) == (5, 64) and tuple(sd["act.action_outs.1.weight"].shape) == (10, 64)
    ent = {name: (off, rows) for name, off, rows, cols in pol._a_entries}
    assert ent["act.action_outs.1.weight"][0] == ent["act.action_outs.0.weight"][0] + 5 * 64
    assert ent["act.action_outs.1.bias"][0] == ent["act.action_outs.0.bias"][0] + 5


# ---- rollout-time actions against the reference's per-sub-space calls (MADDPGPolicy.py:73-89, 126-129) --------------------------------
def _ref_sample_gumbel(shape, eps=1e-20):               # util.py:127-130
    u = torch.FloatTensor(*shape).uniform_()
    return -torch.log(-torch.log(u + eps) + eps)


def _ref_onehot(logits):                                # util.py:106-118, eps = 0
    return (logits == logits.max(-1, keepdim=True)[0]).float()


def _ref_gumbel_hard(logits):                           # util.py:133-166, hard = True
    y = F.softmax(logits + _ref_sample_gumbel(logits.shape), dim=-1)
    return (_ref_onehot(y) - y).detach() + y


def _ref_get_actions(actor_out, segs, mode, eps, B):
    blocks = actor_out.split(segs, -1)
    if mode == "gumbel":
        return torch.cat(list(map(_ref_gumbel_hard, blocks)), dim=-1)
    if mode == "explore":
        onehot = torch.cat(list(map(_ref_gumbel_hard, blocks)), dim=-1)
        take = (np.random.rand(B, 1) < eps).astype(int).reshape(-1, 1)
        rnd = torch.cat([torch.distributions.OneHotCategorical(logits=torch.ones(B, n)).sample() for n in segs], dim=1)
        return (1 - take) * onehot.numpy() + take * rnd.numpy()
    return torch.cat(list(map(_ref_onehot, blocks)), dim=-1)


@pytest.mark.parametrize("mode", ["greedy", "gumbel", "target", "explore"])
def test_get_actions_match_reference_calls(emu_engine, mode):
    from offpolicy._b200.factory import build_mlp_maddpg
    torch.manual_seed(4)
    args, pol, tr = build_mlp_maddpg(N, O, SEGS, S, 8, td3=(mode == "target"))
    B = 64
    obs = np.random.default_rng(2).standard_normal((B, O)).astype(np.float32)
    theta = pol.actor_vecs[1] if mode == "target" else pol.actor_vecs[0]
    actor_out = pol._forward(theta, obs)
    kw = dict(greedy={}, gumbel=dict(use_gumbel=True), target=dict(use_target=True), explore=dict(explore=True, t_env=20000))[mode]
    avail = np.zeros((B, 15), np.float32)                # ignored by MultiDiscrete policies
    torch.manual_seed(11)
    np.random.seed(12)
    got, eps = pol.get_actions(obs, avail, **kw)
    rng_t, rng_n = torch.get_rng_state(), np.random.get_state()
    torch.manual_seed(11)
    np.random.seed(12)
    want = _ref_get_actions(actor_out, SEGS, "gumbel" if mode == "target" else mode, pol.exploration.eval(20000), B)
    assert torch.equal(torch.get_rng_state(), rng_t)
    assert np.array_equal(np.random.get_state()[1], rng_n[1])
    assert np.array_equal(np.asarray(got), np.asarray(want))
    assert (eps is None) == (mode != "explore")
    hard = np.asarray(got)
    assert np.allclose(hard[:, :5].sum(-1), 1.0, atol=1e-5) and np.allclose(hard[:, 5:].sum(-1), 1.0, atol=1e-5)


def test_get_random_actions_match_reference_calls(emu_engine):
    from offpolicy._b200.factory import build_mlp_maddpg
    torch.manual_seed(4)
    args, pol, tr = build_mlp_maddpg(N, O, SEGS, S, 8)
    obs = np.zeros((32, O), np.float32)
    torch.manual_seed(13)
    got = pol.get_random_actions(obs, np.zeros((32, 15), np.float32))
    after = torch.get_rng_state()
    torch.manual_seed(13)
    want = np.concatenate([torch.distributions.OneHotCategorical(logits=torch.ones(32, n)).sample().numpy() for n in SEGS], axis=-1)
    assert torch.equal(torch.get_rng_state(), after)
    assert got.shape == (32, 15) and np.array_equal(got, want)


# ---- the replay: MultiDiscrete actions are stored as the concatenated blocks -------------------------------------------------------
@pytest.mark.parametrize("rng", ["numpy", "device"])
def test_mlp_replay_stores_concatenated_blocks(emu_engine, rng):
    from offpolicy._b200.factory import Box, MultiDiscrete
    from offpolicy.utils.mlp_buffer import MlpReplayBuffer
    B, size = 16, 64
    info = {"policy_0": dict(obs_space=Box(O), share_obs_space=Box(S), act_space=MultiDiscrete([[0, 4], [0, 9]]))}
    buf = MlpReplayBuffer(info, {"policy_0": list(range(N))}, size, True, False, max_batch=B, rng=rng)
    r = np.random.default_rng(4)
    tr = lambda x: np.asarray(x["policy_0"]).transpose(1, 0, 2)
    stored = []
    for _ in range(size // B):
        b = mdc.synth_batch_md(r, mdc.REFERENCE_SPEC, B, S)
        buf.insert(B, {"policy_0": tr(b[0])}, {"policy_0": b[1]["policy_0"]}, {"policy_0": tr(b[2])}, {"policy_0": tr(b[3])},
                   {"policy_0": tr(b[4])}, {"policy_0": b[5]["policy_0"]}, {"policy_0": tr(b[6])}, {"policy_0": b[7]["policy_0"]},
                   {"policy_0": tr(b[8])}, None, None)
        stored.append(b)
    if rng == "device":
        buf.seed_device_rng(5)
    np.random.seed(3)
    s = buf.sample(B)
    inds = np.asarray(buf.policy_buffers["policy_0"].rep.sampled_indices(B))
    acts = np.concatenate([b[2]["policy_0"] for b in stored], 1)          # (N, rows, 15)
    got = s.materialize("policy_0", "acts")
    assert got.shape == (N, B, 15)
    assert np.array_equal(got, acts[:, inds])
    assert np.allclose(got[..., :5].sum(-1), 1.0) and np.allclose(got[..., 5:].sum(-1), 1.0)


# ---- the learner refuses bad segment lists -----------------------------------------------------------------------------------------
def _cfg(lib_capi, act_dim, segs, discrete=1, mlp=1, episode_len=1):
    c = lib_capi.MaddpgCfg(n_agents=2, obs_dim=O, act_dim=act_dim, state_dim=S, hidden=64, episode_len=episode_len, max_batch=8, num_q=1,
                           actor_update_interval=1, gamma=0.99, lr=1e-3, adam_beta1=0.9, adam_beta2=0.999, adam_eps=1e-5, max_grad_norm=10.0,
                           tau=0.005, discrete=discrete, mlp=mlp)
    c.n_act_seg = len(segs)
    for i, n in enumerate(segs[:lib_capi.MAX_ACT_SEG]):
        c.act_seg[i] = n
    return c


@pytest.mark.parametrize("act_dim,segs,discrete,mlp,msg", [
    (16, [5, 10], 1, 1, b"sum to 15"),
    (15, [5, 10, 0], 1, 1, b"width 0"),
    (10, [2, 2, 2, 2, 2], 1, 1, b"n_act_seg 5"),
    (15, [5, 10], 0, 1, b"need discrete"),
    (6, [2, 4], 1, 0, b"recurrent learner takes no action segments"),
    (5, [5], 1, 0, b"recurrent learner takes no action segments"),
    (33, [], 1, 1, b"act_dim 33 > 32"),
    (9, [], 1, 0, b"act_dim 9 > 8"),
])
def test_create_rejects_bad_segments(emu_engine, act_dim, segs, discrete, mlp, msg):
    lib = emu_engine.lib()
    c = _cfg(emu_engine, act_dim, segs, discrete, mlp, episode_len=1 if mlp else 4)
    assert lib.mx_maddpg_workspace_bytes(C.byref(c)) == -1
    assert msg in lib.mx_last_error(), lib.mx_last_error()
    h = C.c_void_p()
    assert lib.mx_maddpg_create(C.byref(c), None, None, None, 0, C.byref(h)) != 0


def test_segment_lists_accepted(emu_engine):
    lib = emu_engine.lib()
    for act_dim, segs, mlp in ((15, [5, 10], 1), (32, [8, 8, 8, 8], 1), (5, [5], 1), (5, [], 0)):
        c = _cfg(emu_engine, act_dim, segs, 1, mlp, episode_len=1 if mlp else 4)
        assert lib.mx_maddpg_workspace_bytes(C.byref(c)) > 0, lib.mx_last_error()


def test_recurrent_and_qmix_policies_still_raise(emu_engine):
    from offpolicy._b200.factory import MultiDiscrete, mlp_maddpg_args, Box
    from offpolicy.algorithms.r_maddpg.algorithm.rMADDPGPolicy import R_MADDPGPolicy
    from offpolicy.algorithms.mqmix.algorithm.mQMixPolicy import M_QMixPolicy
    args = mlp_maddpg_args(8)
    info = dict(obs_space=Box(O), share_obs_space=Box(S), act_space=MultiDiscrete([[0, 4], [0, 9]]), cent_obs_dim=S, cent_act_dim=30)
    for cls in (R_MADDPGPolicy, M_QMixPolicy):
        with pytest.raises(NotImplementedError):
            cls({"args": args, "device": emu_engine.device()}, info)


# ---- the unmodified MLP runner on simple_reference ---------------------------------------------------------------------------------
@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "offpolicy", "runner")), reason="reference checkout not present")
@pytest.mark.parametrize("algo,share", [("matd3", False), ("maddpg", False), ("matd3", True)])
def test_mlp_runner_simple_reference(emu_engine, algo, share):
    """scripts/train_mpe_matd3.sh's scenario on runner/mlp/mpe_runner.py (one shared policy, or one per agent with --share_policy):
    identical episodes, train_info to fp32 round-off."""
    out, procs = {}, {}
    for eng in ("b200", "reference"):
        cmd = [sys.executable, os.path.join(ROOT, "tests", "integration", "run_mpe.py"), "--engine", eng, "--algo", algo, "--steps", "200",
               "--runner", "mlp", "--scenario", "simple_reference", "--agents", "2"] + (["--share_policy"] if share else [])
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


# ---- the same policy calls composed from the reference's own util.py functions (MADDPGPolicy.py:73-89) ------------------------------
def _reference_util():
    """utils/util.py of the reference checkout, loaded as a module of its own (the drop-in `offpolicy` package stays imported)."""
    import importlib.util
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import ref_harness as rh
    rh._install_gym_shim()
    spec = importlib.util.spec_from_file_location("reference_offpolicy_util", os.path.join(REF, "offpolicy", "utils", "util.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.skipif(not os.path.isfile(os.path.join(REF, "offpolicy", "utils", "util.py")), reason="reference checkout not present")
@pytest.mark.parametrize("mode", ["greedy", "gumbel", "target", "explore"])
def test_get_actions_match_reference_functions(emu_engine, mode):
    """get_actions against MADDPGPolicy.py:73-89 composed from the reference's own gumbel_softmax / onehot_from_logits, on the logits of
    an independent actor (oracle/maddpg_mlp_md.py) from the same weights: identical actions, the same torch and NumPy RNG states after."""
    from offpolicy._b200.factory import build_mlp_maddpg
    from torch.distributions import OneHotCategorical
    util = _reference_util()
    torch.manual_seed(4)
    args, pol, tr = build_mlp_maddpg(N, O, SEGS, S, 8, td3=(mode == "target"))
    B = 64
    obs = np.random.default_rng(2).standard_normal((B, O)).astype(np.float32)
    L = mdc.oracle_from(args, pol)
    actor_out = L.actor_out(L.target_actor if mode == "target" else L.actor, torch.from_numpy(obs)).detach()
    kw = dict(greedy={}, gumbel=dict(use_gumbel=True), target=dict(use_target=True), explore=dict(explore=True, t_env=20000))[mode]
    torch.manual_seed(11)
    np.random.seed(12)
    got, _ = pol.get_actions(obs, np.zeros((B, 15), np.float32), **kw)
    rng_t, rng_n = torch.get_rng_state(), np.random.get_state()
    torch.manual_seed(11)
    np.random.seed(12)
    blocks = list(actor_out.split(SEGS, -1))
    if mode in ("gumbel", "target"):
        want = torch.cat(list(map(lambda a: util.gumbel_softmax(a, hard=True), blocks)), dim=-1)
    elif mode == "explore":
        onehot = torch.cat(list(map(lambda a: util.gumbel_softmax(a, hard=True), blocks)), dim=-1)
        take = (np.random.rand(B, 1) < pol.exploration.eval(20000)).astype(int).reshape(-1, 1)
        rnd = torch.cat([OneHotCategorical(logits=torch.ones(B, n)).sample() for n in SEGS], dim=1)
        want = (1 - take) * util.to_numpy(onehot) + take * util.to_numpy(rnd)
    else:
        want = torch.cat(list(map(util.onehot_from_logits, blocks)), dim=-1)
    assert torch.equal(torch.get_rng_state(), rng_t)
    assert np.array_equal(np.random.get_state()[1], rng_n[1])
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    hard = lambda x: np.concatenate([(b == b.max(-1, keepdims=True)) for b in np.split(x, [5], -1)], -1)
    assert np.array_equal(hard(got), hard(want))              # the same one-hot choices in every block
    assert np.abs(got - want).max() <= 1e-5                   # the straight-through values to fp32 round-off of the two forwards


def test_rollout_forward_matches_independent_actor(emu_engine):
    """The rollout forward (k_policy_step, 15 outputs) against the oracle's actor on the same weights, live and target."""
    from offpolicy._b200.factory import build_mlp_maddpg
    torch.manual_seed(6)
    args, pol, tr = build_mlp_maddpg(N, O, SEGS, S, 8)
    rng = np.random.default_rng(0)
    with torch.no_grad():
        for v in pol.actor_vecs[:2]:
            v.add_(torch.from_numpy(rng.standard_normal(v.numel()).astype(np.float32) * 0.05).to(v.device))      # heads away from gain 0.01
    L = mdc.oracle_from(args, pol)
    obs = rng.standard_normal((200, O)).astype(np.float32)
    for theta, net in ((pol.actor_vecs[0], L.actor), (pol.actor_vecs[1], L.target_actor)):
        got = pol._forward(theta, obs).numpy()
        want = L.actor_out(net, torch.from_numpy(obs)).detach().numpy()
        assert got.shape == (200, 15)
        assert np.abs(got - want).max() <= 1e-4 * max(1.0, np.abs(want).max())


@pytest.mark.parametrize("discrete", [True, False])
def test_wide_single_block_actions_lockstep(emu_engine, discrete):
    """The MLP learner takes one block wider than 8 (Discrete(12), Box(12)), against oracle/maddpg_mlp.py."""
    import mlp_maddpg_checks as mc
    from offpolicy._b200.factory import build_mlp_maddpg
    torch.manual_seed(5)
    n, o, a, s2, B = 2, 10, 12, 20, 16
    for td3 in (False, True):
        args, pol, tr = build_mlp_maddpg(n, o, a, s2, B, discrete=discrete, td3=td3)
        rng = np.random.default_rng(7)
        mc.lockstep(args, pol, tr, [mc.synth_batch(rng, n, B, o, s2, a, discrete) for _ in range(3)])
