"""QMIX / VDN / M-QMIX / M-VDN with more than 32 actions (up to 64) on the CPU fiber emulator.

SMAC's action count is 6 + the number of enemies (27m_vs_30m: 36).  Past 32 the Q-head kernels hold two actions per lane
(k_mid, k_qhead, k_qhead_bwd take an actions-per-lane parameter of 2); these tests pin that instantiation against the reference
fixtures made by tests/golden/make_goldens_qmix_many_actions.py and against the oracle in lock-step."""
import os
import subprocess
import sys

import numpy as np
import pytest

import qmix_checks as qc
import mqmix_checks as mc
import rollout_checks as rc
import qmix_many_actions_fixture as mf
from helpers import load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))


def _cfg(A, N=3, O=20, S=30, **over):
    from oracle.qmix import QmixConfig
    return QmixConfig(n_agents=N, obs_dim=O, act_dim=A, state_dim=S, gain=1.0, **over)


def _lockstep(cfg, B=3, T=5, steps=2, per=False, vdn=False, debug=False, seed=9, param_tol=5e-3):
    from oracle.qmix import synth_batch
    L, args, pol, tr = qc.oracle_and_trainer(cfg, B, T, vdn=vdn, debug=debug)
    extra = (np.random.RandomState(3).rand(B) * 0.9 + 0.1, np.arange(B)) if per else (None, None)
    batch = synth_batch(cfg, B, T, seed=seed, avail_p=0.6, var_len=True) + extra
    qc.compare_step(L, pol, tr, batch, cfg, steps=steps, param_tol=param_tol)


# debug=True keeps k_qhead / k_mix_core / k_qhead_bwd as separate launches and checks every per-action Q value and the greedy actions;
# debug=False runs the product configuration, the fused k_mid
@pytest.mark.parametrize("debug", [True, False], ids=["qhead", "mid"])
@pytest.mark.parametrize("name", ["qmix_a36_ties", "qmix_a64_hyper1"])
def test_engine_matches_many_action_reference_fixture(emu_engine, monkeypatch, name, debug):
    monkeypatch.setattr(qc, "load_golden", mf.load)
    qc.check_step_against(None, name, intermediates=True, debug=debug)


@pytest.mark.parametrize("debug", [True, False], ids=["qhead", "mid"])
def test_prev_act_inp_many_actions_matches_reference_fixture(emu_engine, monkeypatch, debug):
    """--prev_act_inp at 33 actions: the network input is obs + 33 one-hot columns (k_pack_prev_act)."""
    monkeypatch.setattr(qc, "load_golden", mf.load)
    qc.check_step_against(None, "qmix_a33_prev_act", intermediates=False, debug=debug)


@pytest.mark.parametrize("debug", [True, False])
def test_mqmix_many_actions_matches_reference_fixture(emu_engine, debug):
    """M-QMIX at 36 actions, avail and next-step avail masks (k_mlp_qselect), and its rollout surface."""
    mc.check_golden("mqmix_a36", debug=debug)


def test_rollout_many_actions_matches_reference_fixture(emu_engine, monkeypatch):
    """k_policy_step at 36 actions: greedy chain with tied Q values (equal head rows 3 / 35 and 32 / 33), sequence form, exploring and
    random actions under the reference's seeds."""
    monkeypatch.setattr(rc, "load_golden", lambda name: load_golden("qmix_rollout_a36"))
    rc.check_rollout()


@pytest.mark.parametrize("A", [33, 36, 48, 64])
@pytest.mark.parametrize("debug", [False, True], ids=["mid", "qhead"])
def test_many_actions_vs_oracle(emu_engine, A, debug):
    _lockstep(_cfg(A), debug=debug)


@pytest.mark.parametrize("A", [36, 64])
@pytest.mark.parametrize("huber", [False, True])
def test_many_actions_per_vs_oracle(emu_engine, A, huber):
    # param_tol: at A = 36 one head-weight gradient element is -6.4e-7 (eps / 16), where Adam's lr * g / (|g| + eps) turns its fp32
    # round-off (7e-8 absolute, 1e-7 of the tensor's largest entry) into 0.6 % of lr; the gradients themselves pass at 1e-4
    _lockstep(_cfg(A, use_per=True, huber=huber, huber_delta=0.7), B=4, T=4, per=True, param_tol=1e-2)


@pytest.mark.parametrize("A", [36, 64])
def test_many_actions_no_double_q_vs_oracle(emu_engine, A):
    _lockstep(_cfg(A, double_q=False, hyper_layers=1))


@pytest.mark.parametrize("A", [36, 64])
def test_vdn_many_actions_vs_oracle(emu_engine, A):
    _lockstep(_cfg(A, vdn=True), vdn=True)


@pytest.mark.parametrize("A", [33, 36, 48, 64])
def test_mqmix_many_actions_vs_oracle(emu_engine, A):
    mc.check_vs_oracle(N=3, O=18, A=A, S=54, B=24, steps=2, avail=True)


@pytest.mark.parametrize("kw", [dict(per=True), dict(per=True, huber=True), dict(double_q=False), dict(vdn=True)],
                         ids=["per", "per_huber", "nodq", "vdn"])
def test_mqmix_many_actions_variants_vs_oracle(emu_engine, kw):
    mc.check_vs_oracle(N=3, O=18, A=36, S=54, B=24, steps=2, avail=True, **kw)


def test_act_dim_limit(emu_engine):
    """64 actions is the learner's limit; 65 is refused at creation with a message that names it."""
    import ctypes as C
    from offpolicy._b200 import capi
    lib = capi.lib()
    total = C.c_int64()
    for A, ok in ((64, True), (65, False)):
        cfg = capi.QmixCfg(n_agents=3, obs_dim=8, act_dim=A, state_dim=5, hidden=64, mixer_hidden=32, hyper_hidden=64, hyper_layers=2,
                           episode_len=4, max_batch=2)
        n = lib.mx_qmix_param_layout(C.byref(cfg), None, 0, C.byref(total))
        assert (n > 0) == ok, A
        if not ok:
            assert b"act_dim must be <= 64" in lib.mx_last_error()


@pytest.mark.parametrize("order", ["reverse", "random"])
def test_many_actions_thread_orders(order):
    """The fixture and lock-step checks with the emulator's threads run in reverse / pseudo-random order (missing barriers)."""
    env = dict(os.environ, EMU_ORDER=order)
    code = ("import sys; sys.path[:0] = [%r, %r, %r]\n"
            "import pytest\n"
            "sys.exit(pytest.main(['-q', '-x', '-p', 'no:cacheprovider', %r, '-k', "
            "'test_engine_matches_many_action_reference_fixture and qmix_a36_ties or test_many_actions_vs_oracle and 64']))\n"
            % (ROOT, os.path.join(ROOT, "off-policy_b200"), HERE, os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
