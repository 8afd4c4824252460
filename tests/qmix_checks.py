"""QMIX learner parity checks shared by the emulated (CPU) and real (GPU) test modules.

Tolerances (north_star: "within 1e-4 rel on fp32 losses/grads"): scalars 1e-4 relative; every gradient tensor
max-abs error <= 1e-4 x max-abs of the reference tensor (+1e-7 abs); parameters after Adam: the UPDATE
(new - old) within 5e-3 x lr per element (Adam normalises the step to ~lr; for near-zero gradients the step is
lr*g/eps, i.e. an ABSOLUTE gradient error of 1e-8 already moves the step by 1e-3 x lr -- the reference run with a
different thread count shows the same spread); Polyak targets 1e-6.
"""
import types

import numpy as np
import torch

from helpers import load_golden, golden_cfg, oracle_from_golden, golden_batch, sub, rel_err
from replay_checks import Discrete


def make_args(cfg, B, **over):
    from offpolicy._b200 import factory
    return factory.qmix_args(cfg, B, **over)


def build_trainer(cfg, B, T, vdn=False, debug=True, **over):
    # debug: also materialise per-action Q values for the intermediate checks (and keep k_qhead / k_mix_core / k_qhead_bwd as
    # separate launches); debug=False runs the product configuration (the fused k_mid between the recurrences)
    from offpolicy._b200 import factory
    return factory.build_qmix(cfg, B, T, vdn=vdn, debug=debug, **over)


def load_state(pol, tr, agent_sd, mixer_sd, tgt_agent_sd, tgt_mixer_sd):
    pol.q_network.load_state_dict(agent_sd)
    tr.target_q_network.load_state_dict(tgt_agent_sd)
    if mixer_sd is not None:
        tr.mixer.load_state_dict(mixer_sd)
        tr.target_mixer.load_state_dict(tgt_mixer_sd)


def ref_tuple(b):
    d = lambda x: {"policy_0": x}
    return tuple(d(x) for x in b[:7]) + (b[7], b[8])


def to_rows(x, N, B):
    """oracle (T+1, N*B, D) with row = n*B + b  ->  ours [M][D] with m = (b*(T+1)+t)*N + n"""
    T1, _, D = x.shape
    return x.reshape(T1, N, B, D).permute(2, 0, 1, 3).reshape(-1, D)


def close(a, b, rtol, atol=1e-7):
    a = np.asarray(torch.as_tensor(a).detach().cpu(), dtype=np.float64)
    b = np.asarray(torch.as_tensor(b).detach().cpu(), dtype=np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    err = np.abs(a - b).max()
    lim = rtol * np.abs(b).max() + atol
    return err <= lim, err, lim


def check_forward_intermediates(tr, L, batch, cfg, B, T):
    """Localise a kernel bug: every materialised activation vs the oracle's cell-by-cell trace."""
    from oracle.qmix import agent_trace
    N = cfg.n_agents
    M = B * (T + 1) * N
    E = B * T
    x = L.stack_agents(batch[0])
    bad = []

    def cmp(name, ours, want, rtol=2e-5):
        ok, err, lim = close(ours, want, rtol, 1e-6)
        if not ok:
            bad.append("%s: err %.3e > %.3e" % (name, err, lim))

    for tag, net in (("live", L.agent), ("tgt", L.tgt_agent)):
        trc = agent_trace(net, x)
        cmp("gi_" + tag, tr.ws_view("gi_" + tag)[:M * 192].view(M, 192), to_rows(trc["gi"], N, B))
        cmp("h_" + tag, tr.ws_view("h_" + tag)[:M * 64].view(M, 64), to_rows(trc["h"], N, B))
        cmp("q_" + tag, tr.ws_view("q_" + tag)[:M * cfg.act_dim].view(M, cfg.act_dim), to_rows(trc["q"], N, B), 1e-4)
        if tag == "live":
            cmp("u1", tr.ws_view("u1")[:M * 64].view(M, 64), to_rows(trc["u1"], N, B))
            cmp("u2", tr.ws_view("u2")[:M * 64].view(M, 64), to_rows(trc["u2"], N, B))
            g = tr.ws_view("gates")[:M * 192].view(M, 192)
            cmp("r", g[:, :64], to_rows(trc["r"], N, B))
            cmp("z", g[:, 64:128], to_rows(trc["z"], N, B))
            cmp("n", g[:, 128:], to_rows(trc["n"], N, B))
            cmp("hn", tr.ws_view("hn")[:M * 64].view(M, 64), to_rows(trc["hn"], N, B))
    loss, prio, aux = L.loss_terms(batch)
    tb = lambda v: v.permute(1, 0, 2).reshape(E, -1)            # oracle (T,B,k) -> ours [b*T+t][k]
    cmp("q_taken", tr.ws_view("q_taken")[:E * N].view(E, N), tb(aux["q_taken"].detach()), 1e-4)
    cmp("q_next", tr.ws_view("q_next")[:E * N].view(E, N), tb(aux["tq_next"]), 1e-4)
    cmp("qtot", tr.ws_view("qtot")[:E].view(E, 1), tb(aux["q_tot"].detach()), 1e-4)
    cmp("qtot_next", tr.ws_view("qtot_next")[:E].view(E, 1), tb(aux["q_tot_next"]), 1e-4)
    cmp("err", tr.ws_view("err")[:E].view(E, 1), tb(aux["err"].detach()), 1e-4)
    return bad


def check_step_against(g_or_none, name=None, intermediates=True, debug=True):
    g = load_golden(name)
    L, cfg, B, T, steps = oracle_from_golden(g)
    args, pol, tr = build_trainer(cfg, B, T, debug=debug)
    intermediates = intermediates and debug
    load_state(pol, tr, sub(g, "init.agent."), sub(g, "init.mixer."), sub(g, "init.tgt_agent."), sub(g, "init.tgt_mixer."))
    problems = []
    for s in range(steps):
        batch = golden_batch(g, s)
        prev = {k: v.clone() for k, v in list(pol.q_network.state_dict().items())}
        prev_m = {k: v.clone() for k, v in list(tr.mixer.state_dict().items())}
        info, prio, idx = tr.train_policy_on_batch(ref_tuple(batch))
        if intermediates and s == 0:
            problems += check_forward_intermediates(tr, L, batch, cfg, B, T)
        for key, want in (("loss", g["s%d.loss" % s]), ("grad_norm", g["s%d.grad_norm" % s]), ("Q_tot", g["s%d.Q_tot" % s])):
            e = rel_err(info[key].cpu(), want)
            if e > 1e-4:
                problems.append("step %d %s: rel err %.3e (got %r want %r)" % (s, key, e, float(info[key]), float(want)))
        if cfg.use_per:
            ok, err, lim = close(np.asarray(prio), g["s%d.prio" % s], 1e-4)
            if not ok:
                problems.append("step %d priorities err %.3e" % (s, err))
        # gradients: golden holds clipped grads
        gn = float(g["s%d.grad_norm" % s])
        coef = min(1.0, cfg.max_grad_norm / (gn + 1e-6))
        gv = tr.grad_views()
        for full, ours in gv.items():
            role, pname = full.split(".", 1)
            key = "s%d.grad.%s.%s" % (s, role, pname)
            if key not in g:
                if float(ours.abs().max()) != 0.0:
                    problems.append("step %d grad %s should be zero (unused parameter)" % (s, full))
                continue
            ok, err, lim = close(ours * coef, g[key], 1e-4)
            if not ok:
                problems.append("step %d grad %s: err %.3e > %.3e" % (s, full, err, lim))
        tr.soft_target_updates()
        for role, mod, prv in (("agent", pol.q_network, prev), ("mixer", tr.mixer, prev_m)):
            for k, v in mod.state_dict().items():
                want = g["s%d.%s.%s" % (s, role, k)]
                d_ours = (v.cpu() - prv[k].cpu()).numpy()
                d_want = want - prv[k].cpu().numpy()
                err = np.abs(d_ours - d_want).max()
                # Adam's step is lr * m_hat / (sqrt(v_hat) + eps): an absolute gradient error d moves it by up to lr * d / eps, so the
                # 1e-4 gradient budget (relative to the tensor's largest entry) is propagated through that sensitivity.
                gkey = "s%d.grad.%s.%s" % (s, role, k)
                gmax = float(np.abs(g[gkey]).max()) if gkey in g else 0.0
                lim = cfg.lr * min(2.0, 5e-3 + 1e-4 * gmax / cfg.opti_eps)
                if err > lim + 1e-9:
                    problems.append("step %d param %s.%s: update err %.3e" % (s, role, k, err))
        for role, mod in (("tgt_agent", tr.target_q_network), ("tgt_mixer", tr.target_mixer)):
            for k, v in mod.state_dict().items():
                ok, err, lim = close(v, g["s%d.%s.%s" % (s, role, k)], 1e-6, 1e-7)
                if not ok:
                    problems.append("step %d %s.%s: err %.3e" % (s, role, k, err))
        # keep the oracle in lock-step for the next step's intermediates
        L.step(batch)
        L.soft_update()
    assert not problems, "\n".join(problems[:40])


# ---- oracle in lock-step (any size) ----------------------------------------------------------------------------
def oracle_and_trainer(cfg, B, T, seed=3, vdn=False, **over):
    from oracle.qmix import QmixLearner, randomize_all
    L = QmixLearner(cfg, seed=seed)
    randomize_all(L.agent, 1)
    if not vdn:
        randomize_all(L.mixer, 2)
    L.sync_targets()
    randomize_all(L.tgt_agent, 3, 0.05)
    if not vdn:
        randomize_all(L.tgt_mixer, 4, 0.05)
    args, pol, tr = build_trainer(cfg, B, T, vdn=vdn, **over)
    load_state(pol, tr, L.agent.state_dict(), None if vdn else L.mixer.state_dict(), L.tgt_agent.state_dict(),
                  None if vdn else L.tgt_mixer.state_dict())
    return L, args, pol, tr


def grad_failures(gv, coef, L, cfg, tol):
    """Names of gradient tensors outside `tol` (max-norm, see the module docstring) or `10 * tol` relative L2."""
    named = dict(("agent." + k, p) for k, p in L.agent.named_parameters())
    if not cfg.vdn:
        named.update(("mixer." + k, p) for k, p in L.mixer.named_parameters())
    bad = []
    for k, p in named.items():
        if p.grad is None:
            assert float(gv[k].abs().max()) == 0.0, k
            continue
        ok, err, lim = close(gv[k] * coef, p.grad, tol)
        a = (gv[k] * coef).detach().cpu().double().flatten()
        b = p.grad.detach().cpu().double().flatten()
        l2 = float((a - b).norm() / (b.norm() + 1e-30))
        if not ok or (l2 > 10 * tol and float(b.norm()) > 1e-6):
            bad.append((k, err, lim, l2))
    return bad


def compare_step(L, pol, tr, batch, cfg, steps=1, tol=1e-4, param_tol=5e-3, mlp=False):
    for s in range(steps):
        info, prio, _ = tr.train_policy_on_batch(ref_tuple(batch))
        gv = {k: v.clone() for k, v in tr.grad_views().items()}
        check_engine_step(L, pol, tr, batch, cfg, info, prio, gv, s, tol, param_tol)


def check_engine_step(L, pol, tr, batch, cfg, info, prio, gv, s=0, tol=1e-4, param_tol=5e-3):
    """Step `s` of compare_step after the engine ran it (train_info `info`, priorities `prio`, gradient views `gv`): the oracle
    steps on the same batch and both are compared; then both apply the soft target update."""
    import kink
    B, T = (batch[0].shape[2], batch[2].shape[1])
    L0 = kink.snapshot(L) if getattr(cfg, "relu", True) else None
    ref, rprio, _ = L.step(batch)
    coef = min(1.0, cfg.max_grad_norm / (float(ref["grad_norm"]) + 1e-6))
    bad = grad_failures(gv, coef, L, cfg, tol)
    if bad and L0 is not None:
        # ReLU kink? re-run the oracle step with the engine's ReLU masks (tests/kink.py): only units within round-off of zero may differ
        masks = kink.engine_masks(tr, B, T, cfg.n_agents, mlp=False)
        (ref, rprio, _), flips, max_pre = kink.redo_with_engine_masks(L0, lambda LL: LL.step(batch), masks)
        assert flips > 0 and max_pre < kink.KINK_TOL, (s, "gradient mismatch not explained by ReLU kinks", flips, max_pre, bad[:3])
        kink.adopt(L, L0)
        coef = min(1.0, cfg.max_grad_norm / (float(ref["grad_norm"]) + 1e-6))
        bad = grad_failures(gv, coef, L, cfg, tol)
        print("kink-aware comparison: %d ReLU unit(s) within %.1e of zero flipped" % (flips, max_pre))
    assert not bad, (s, bad[:4])
    tr.soft_target_updates()
    L.soft_update()
    for k in ("loss", "grad_norm", "Q_tot"):
        assert rel_err(info[k].cpu(), ref[k]) < tol, (s, k, float(info[k]), float(ref[k]))
    if rprio is not None:
        assert rel_err(np.asarray(prio), rprio) < tol
    for k, v in pol.q_network.state_dict().items():
        assert float((v.cpu() - L.agent.state_dict()[k]).abs().max()) <= param_tol * cfg.lr * (s + 1) + 1e-7, (s, k)
    for k, v in tr.target_q_network.state_dict().items():
        assert float((v.cpu() - L.tgt_agent.state_dict()[k]).abs().max()) <= 1e-6, (s, k)


def check_mpe_shapes_without_avail_masks(steps=2, B=32):
    """BASELINE configs[0]: scripts/train_mpe_qmix.sh = recurrent QMIX on MPE simple_spread (3 agents, obs 18, Discrete(5), state 54,
    episode_length 25, batch 32, --use_reward_normalization) -- no available-action masks (runner/rnn/mpe_runner.py:62 passes
    avail_acts = None).  Replay (reward normalisation on, use_avail_acts False) -> sample -> train, against the oracle replay +
    oracle learner fed the same episodes and the same NumPy index stream."""
    import replay_checks as rc
    from oracle.qmix import QmixConfig, QmixLearner, randomize_all
    from oracle.replay import UniformReplay
    N, O, A, S, T, E = 3, 18, 5, 54, 25, 48
    cfg = QmixConfig(n_agents=N, obs_dim=O, act_dim=A, state_dim=S, gain=1.0)
    L, args, pol, tr = oracle_and_trainer(cfg, B, T, debug=False)
    buf = rc.make_buffers(N, O, A, S, T, E, norm=True, rng="numpy", max_batch=max(B, 32), avail=False)
    ora = UniformReplay(E, T, N, O, S, A, use_avail=False, reward_norm=True, rng=None)
    rs = np.random.RandomState(4)
    for n in (30, 10, 20):                      # the third insert wraps the ring: running reward statistics evict
        de = np.maximum.accumulate((rs.rand(T, n, 1) < 0.05).astype(np.float32), axis=0)
        ep = [rs.randn(T + 1, n, N, O), np.repeat(rs.randn(T + 1, n, 1, S), N, 2), np.eye(A)[rs.randint(0, A, (T, n, N))],
              np.repeat(2.0 + rs.randn(T, n, 1, 1), N, 2), np.repeat(de[:, :, None], N, 2), de]
        ep = [x.astype(np.float32) for x in ep]
        buf.insert(n, *[rc.d(x) for x in ep], None)
        ora.insert(n, *ep, None)
    np.random.seed(21)
    for s in range(steps):
        st = np.random.get_state()
        smp = buf.sample(B)
        np.random.set_state(st)
        out, inds = ora.sample(B)
        assert smp[6]["policy_0"] is None and out[6] is None
        info, _, _ = tr.train_policy_on_batch(smp)
        tr.soft_target_updates()
        ref, _, _ = L.step(tuple(out))
        L.soft_update()
        for k in ("loss", "grad_norm", "Q_tot"):
            assert rel_err(info[k].cpu(), ref[k]) < 1e-4, (s, k, float(info[k]), float(ref[k]))
    for k, v in pol.q_network.state_dict().items():
        assert float((v.cpu() - L.agent.state_dict()[k]).abs().max()) <= 5e-3 * cfg.lr * steps + 1e-7, k
