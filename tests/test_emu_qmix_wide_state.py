"""Wide-state QMIX mixer (SMAC's global-all-local state) on the CPU fiber emulator.

A state too wide for the shared-memory hypernet tile sends the learner down the wide-state path: the hypernetworks' state-reading
layers run as tensor-core GEMMs (csrc/mixer_wide.cu) and the hypernet kernels work from their pre-activations.  These tests pin that
path against the oracle in lock-step, pin the path decision, and pin the GEMMs' 3xTF32 accuracy against fp64."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import qmix_checks as qc
import mqmix_checks as mc
import qmix_wide_fixture as wf
from helpers import oracle_from_golden, golden_batch, rel_err

FIXTURES = ["qmix_wide_s448", "qmix_wide_s448_hyper1"]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))


def _cfg(S, N=3, O=30, A=9, layers=2, **over):
    from oracle.qmix import QmixConfig
    return QmixConfig(n_agents=N, obs_dim=O, act_dim=A, state_dim=S, hyper_layers=layers, gain=1.0, **over)


def _lockstep(cfg, B, T, steps=2, per=False, seed=9):
    from oracle.qmix import synth_batch
    L, args, pol, tr = qc.oracle_and_trainer(cfg, B, T)
    extra = (np.random.RandomState(3).rand(B) * 0.9 + 0.1, np.arange(B)) if per else (None, None)
    batch = synth_batch(cfg, B, T, seed=seed, avail_p=0.8, var_len=True) + extra
    qc.compare_step(L, pol, tr, batch, cfg, steps=steps)
    return tr


def _ws_region(tr, name):
    from offpolicy._b200 import capi
    lib = capi.lib()
    off, n = ctypes.c_int64(), ctypes.c_int64()
    assert lib.mx_qmix_ws_lookup(tr.handle, name.encode(), ctypes.byref(off), ctypes.byref(n)) == 0
    return int(off.value), int(n.value)


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_reproduces_wide_reference_fixture(name):
    """The oracle against the unmodified reference QMix at S = 448 (2-layer hypernets with double Q and avail masks; 1-layer
    hypernets with Huber loss): loss, grad_norm, Q_tot, every gradient, post-Adam parameters, post-Polyak targets."""
    torch.set_num_threads(1)
    g = wf.load(name)
    L, cfg, B, T, steps = oracle_from_golden(g)
    info, _, _ = L.step(golden_batch(g, 0))
    assert rel_err(info["loss"], g["s0.loss"]) < 1e-6
    assert rel_err(info["grad_norm"], g["s0.grad_norm"]) < 1e-5
    assert rel_err(info["Q_tot"], g["s0.Q_tot"]) < 1e-5
    for role, mod in (("agent", L.agent), ("mixer", L.mixer)):
        for k, p in mod.named_parameters():
            key = "s0.grad.%s.%s" % (role, k)
            if key in g:
                assert rel_err(p.grad, g[key]) < 2e-5, key
            else:
                assert p.grad is None and "fc_h" in k
    L.soft_update()
    for tag, mod in (("agent", L.agent), ("mixer", L.mixer), ("tgt_agent", L.tgt_agent), ("tgt_mixer", L.tgt_mixer)):
        for k, v in mod.state_dict().items():
            assert rel_err(v, g["s0.%s.%s" % (tag, k)]) < 2e-6, (tag, k)


@pytest.mark.parametrize("name", FIXTURES)
def test_engine_matches_wide_reference_fixture(emu_engine, monkeypatch, name):
    """The engine's wide-state path against the same fixtures (the checks of the other QMIX fixtures, incl. the forward
    intermediates of the debug mode)."""
    monkeypatch.setattr(qc, "load_golden", wf.load)
    qc.check_step_against(None, name)


@pytest.mark.parametrize("S,layers", [(448, 2), (448, 1), (1000, 2), (1000, 1)])
def test_wide_state_vs_oracle(emu_engine, S, layers):
    """S = 448 is the first multiple of 64 past the shared-memory limit at N = 3 (the tile needs 242 KB), 1 000 far past it; both
    hypernet depths, avail masks, double Q, variable episode lengths, two steps with Adam and the soft update in between."""
    tr = _lockstep(_cfg(S, layers=layers), B=3, T=5)
    off, n = _ws_region(tr, "hyp_pre")
    assert n > 0


def test_wide_state_per_huber_vs_oracle(emu_engine):
    tr = _lockstep(_cfg(520, use_per=True, huber=True, huber_delta=0.7), B=4, T=4, per=True)
    assert _ws_region(tr, "d_pre")[1] > 0


def test_wide_state_mqmix_vs_oracle(emu_engine):
    """Transition-level M-QMIX (cfg.mlp) shares the mixer, so it takes the same path."""
    mc.check_vs_oracle(N=3, O=20, A=6, S=640, B=24, steps=2, avail=True)


@pytest.mark.parametrize("order", ["reverse", "random"])
def test_wide_state_thread_orders(order):
    """The same lock-step comparison with the emulator's threads run in reverse / pseudo-random order (missing barriers)."""
    env = dict(os.environ, EMU_ORDER=order)
    code = ("import sys; sys.path[:0] = [%r, %r, %r]\n"
            "import pytest\n"
            "sys.exit(pytest.main(['-q', '-x', '-p', 'no:cacheprovider', %r, '-k', 'test_wide_state_vs_oracle and 448-2']))\n"
            % (ROOT, os.path.join(ROOT, "off-policy_b200"), HERE, os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]


def test_path_decision_and_workspace(emu_engine):
    """Just below the limit the wide-state regions are empty and sit at the very end of the workspace, so the workspace is the one
    the learner always had; just above, they are appended.  VDN never takes the path."""
    def regions(S, layers=2, vdn=False):
        _, _, _, tr = qc.oracle_and_trainer(_cfg(S, layers=layers), 3, 5, vdn=vdn) if not vdn else \
            (None, None, None, qc.build_trainer(_cfg(S, layers=layers, vdn=True), 3, 5, vdn=True)[2])
        off, n = _ws_region(tr, "hyp_pre")
        return n, off, tr.workspace.numel()

    for layers in (2, 1):
        n, off, total = regions(384, layers)
        assert n == 0 and off == total
        n, off, total = regions(448, layers)
        assert n > 0 and off < total
    n, off, total = regions(3000, vdn=True)
    assert n == 0 and off == total


def test_below_threshold_keeps_shared_memory_kernels(emu_engine):
    """S = 384 (just below the limit) runs the shared-memory mixer kernels and matches the oracle; S = 448 adds exactly the three
    wide-state launches (weight images, state-layer GEMM, state-layer weight gradient)."""
    lib = emu_engine.lib()
    c0 = lib.mx_launch_count()
    _lockstep(_cfg(384), B=3, T=5, steps=1)
    below = lib.mx_launch_count() - c0
    c0 = lib.mx_launch_count()
    _lockstep(_cfg(448), B=3, T=5, steps=1)
    above = lib.mx_launch_count() - c0
    assert above == below + 3


def test_state_gemm_3xtf32_vs_fp64(emu_engine):
    """The state-layer GEMMs at K >= 2 000: the forward's pre-activations (K = S = 2 048) and the weight gradient (gradient
    partial 0 = d_pre^T X over the live elements) agree with fp64 to fp32 level, far below single-pass TF32 error (~1e-3)."""
    from oracle.qmix import synth_batch
    cfg = _cfg(2048, N=2, O=8, A=4)
    B, T = 2, 3
    L, args, pol, tr = qc.oracle_and_trainer(cfg, B, T)
    sd = {k: v.detach().double() for k, v in L.mixer.state_dict().items()}
    batch = synth_batch(cfg, B, T, seed=4, avail_p=1.0, var_len=False) + (None, None)
    tr.train_policy_on_batch(qc.ref_tuple(batch))
    X = torch.as_tensor(batch[1], dtype=torch.float64).permute(1, 0, 2).reshape(B * (T + 1), -1)     # engine row b (T+1) + t
    pre_all = tr.ws_view("hyp_pre").double()
    Cp = pre_all.numel() // (2 * B * (T + 1))
    pre = pre_all.view(2, B * (T + 1), Cp)
    W, b = sd["hyper_w1.0.weight"], sd["hyper_w1.0.bias"]          # block 0 of the live net
    ref = X @ W.T + b
    err = float((pre[0, :, :W.shape[0]] - ref).abs().max() / ref.abs().max())
    assert err < 2e-6, err
    # weight gradient: rows t < T of every episode, d_pre block 0
    d_pre = tr.ws_view("d_pre").double().view(B * T, Cp)[:, :W.shape[0]]
    Xl = X.view(B, T + 1, -1)[:, :T].reshape(B * T, -1)
    gref = d_pre.T @ Xl
    off = dict((n, o) for n, o, r, c in tr.entries)["mixer.hyper_w1.0.weight"]
    g = tr.ws_view("gpart").double()[off:off + W.numel()].view_as(W)
    gerr = float((g - gref).abs().max() / gref.abs().max())
    assert gerr < 2e-6, gerr
    bref = d_pre.sum(0)
    boff = dict((n, o) for n, o, r, c in tr.entries)["mixer.hyper_w1.0.bias"]
    assert float((tr.ws_view("gpart").double()[boff:boff + b.numel()] - bref).abs().max() / bref.abs().max()) < 2e-6
