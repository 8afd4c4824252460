"""The QMIX learner at SMAC's real widths on the CPU fiber emulator (4 SMs), against the float64 oracle: agent inputs wider than 128
columns (the FFMA k_front_fwd / k_front_bwd / k_gru_wgrad path), 9 to 32 agents (k_mid's warp count, the mixer's N-wide tiles, the
wide-state threshold), and the input width the learners refuse at creation.

SMAC observation widths with the reference env's defaults (obs_last_action, obs_agent_id): 8m 204, 3s5z_vs_3s6z 268, 1c3s5z 310, MMM2
370; 27m_vs_30m's 285 plus 36 previous actions is 321.  tests/row_coverage_checks.py restates the launchers' rules; the first tests pin
that restatement, the others run the isolated-episode gradients, the per-row forward and the per-transition mixer values on its edges."""
import numpy as np
import pytest
import torch

import row_coverage_checks as rc

EMU_SMS = 4
RULES = rc.TileRules(EMU_SMS)
FFMA_WIDE = ["k_front_fwd", "k_front_bwd", "k_gru_wgrad"]

# width: (obs_dim, act_dim, prev_act_inp, debug): the forward, k_front_bwd and k_gru_wgrad run FFMA, and no tensor-core agent kernel
WIDE = {
    129: (129, 5, False, True),       # the first FFMA width, 1 mod 64
    204: (204, 14, False, False),     # 8m
    268: (268, 15, False, True),      # 3s5z_vs_3s6z
    310: (310, 15, False, False),     # 1c3s5z
    321: (285, 36, True, False),      # 27m_vs_30m's observation + its 36 previous actions (k_pack_prev_act)
    370: (370, 18, False, True),      # MMM2
    384: (384, 9, False, False),      # the widest input the recurrent step accepts
}


def cfg_of(obs, act, N, S=13, prev=False, **over):
    from oracle.qmix import QmixConfig
    return QmixConfig(n_agents=N, obs_dim=obs, act_dim=act, state_dim=S, gain=1.0, prev_act_inp=prev, use_per=True, **over)


def step_kernels(engine, cfg, B, T, debug, stream=None, mlp=False):
    """Kernel names of one step of a fresh learner at cfg."""
    from oracle.qmix import synth_batch
    if mlp:
        from oracle.mqmix import synth_transitions
        L64, pol, tr = rc.mqmix_pair(cfg, B, debug=debug)
        batch = synth_transitions(cfg, B, seed=7, avail=True) + (None, None)
        return rc.kernels_run(engine.lib(), stream, lambda: rc.isolated_episode_gradients(L64, tr, batch, [0], B, 1, cfg.n_agents, mlp=True))
    L64, pol, tr = rc.qmix_pair(cfg, B, T, debug=debug)
    batch = synth_batch(cfg, B, T, seed=5, avail_p=0.8, var_len=True) + (np.ones(B, np.float32), np.arange(B))
    return rc.kernels_run(engine.lib(), stream, lambda: tr.train_policy_on_batch(rc.qc.ref_tuple(batch)))


def assert_ffma_wide(names):
    rc.assert_kernels_ran(names, FFMA_WIDE)
    tc = [n for n in names if "_tc" in n]
    assert not tc, ("a tensor-core agent kernel ran above 128 input columns", tc)


def test_launcher_rules_restatement():
    """The restated limits and thresholds, as numbers: the widest k_front_bwd input (384 with k_gru_wgrad beside it, 320 without); the
    FFMA tiles above 128 columns (32-row forward tiles on half the SMs per net, k_front_bwd and k_gru_wgrad on the same tiles); k_mid's
    warp count per (N, A); the first wide state per N."""
    assert rc.front_bwd_max_in_dim(True) == 384 and rc.front_bwd_max_in_dim(False) == 320
    lay = rc.TileRules(132).agent_rows(5856, 204)
    assert lay["k_front_fwd"] == (32, 183, 66) and lay["k_front_bwd"] == lay["k_gru_wgrad"]
    assert "k_gru_wgrad" not in rc.TileRules(132).agent_rows(5856, 204, gru_ext=False)
    assert RULES.row_kernel(128) == "k_wgrad_tc" and RULES.row_kernel(129) == "k_front_bwd"
    # the input tiles are round_up(in_dim, 64) wide: up to 192 columns 48-row tiles still fit (3m's rows take them on 132 SMs), above
    # only 32-row tiles
    assert rc.TileRules(132).front_bwd_rm(5856, 192, True) == 3
    assert {RULES.front_bwd_rm(M, w, True) for M in range(1, 2000, 7) for w in (193, 384)} == {2}
    # k_mid: 16 warps, then 8, then not at all
    assert [rc.mid_warps(N, 14) for N in (6, 7, 18, 19)] == [16, 8, 8, 0]
    assert [rc.mid_warps(N, 18) for N in (6, 7, 17, 18)] == [16, 8, 8, 0]
    assert [rc.mid_warps(N, 36) for N in (1, 10, 11)] == [8, 8, 0]
    assert [rc.mid_warps(N, 64) for N in (4, 5)] == [8, 0]
    assert {N: rc.min_wide_state(N) for N in (3, 8, 24, 27, 32)} == {3: 385, 8: 321, 24: 193, 27: 129, 32: 65}


def _boundary_cases():
    # (id, cfg kwargs, B, T, debug, kernels that must run, kernels that must not)
    return [
        ("in128", dict(obs=128, act=5, N=2), 2, 4, True, ["k_front_fwd_tc_wide", "k_front_bwd_tc", "k_wgrad_tc"], ["k_gru_wgrad"]),
        ("in129", dict(obs=129, act=5, N=2), 2, 4, True, FFMA_WIDE, ["k_front_bwd_tc", "k_wgrad_tc", "k_front_fwd_tc_wide"]),
        ("in384", dict(obs=384, act=5, N=2), 2, 4, True, FFMA_WIDE, []),
        ("mid16_N6_A14", dict(obs=11, act=14, N=6), 2, 3, False, ["k_mid"], ["k_qhead"]),
        ("mid8_N7_A14", dict(obs=11, act=14, N=7), 2, 3, False, ["k_mid"], ["k_qhead"]),
        ("mid8_N17_A18", dict(obs=11, act=18, N=17), 1, 3, False, ["k_mid"], ["k_qhead"]),
        ("nomid_N18_A18", dict(obs=11, act=18, N=18), 1, 3, False, ["k_qhead", "k_mix_core", "k_qhead_bwd"], ["k_mid"]),
        ("mid8_N10_A36", dict(obs=11, act=36, N=10), 1, 3, False, ["k_mid"], ["k_qhead"]),
        ("nomid_N11_A36", dict(obs=11, act=36, N=11), 1, 3, False, ["k_qhead", "k_qhead_bwd"], ["k_mid"]),
    ] + [("state%d_N%d" % (S, N), dict(obs=11, act=5, N=N, S=S), 1, 2, True, ["k_mixw_fwd", "k_mixw_wgrad"] if wide else ["k_mix_hyper_fwd"],
          [] if wide else ["k_mixw_fwd"])
         for N in (3, 27, 32) for S, wide in ((rc.min_wide_state(N) - 1, False), (rc.min_wide_state(N), True))]


@pytest.mark.parametrize("case", _boundary_cases(), ids=lambda c: c[0])
def test_kernels_on_each_side_of_each_boundary(emu_engine, case):
    """One step on each side of every restated boundary, kernels asserted by name: input width 128 / 129 (tensor cores / FFMA) and 384
    (the widest accepted, 385 is refused below); k_mid at 16 warps, at 8 and not at all (k_qhead + mixer core + k_qhead_bwd); the
    mixer's state one below and at the first wide state for N = 3, 27, 32.  The emulator marks k_mid's 16- and 8-warp launches with
    one name: tests/test_gpu_smac_widths.py reads the warp count from the captured graph's k_mid<W, APL> on each side."""
    name, kw, B, T, debug, want, not_want = case
    kw = dict(kw)
    cfg = cfg_of(kw.pop("obs"), kw.pop("act"), kw.pop("N"), **kw)
    names = step_kernels(emu_engine, cfg, B, T, debug)
    rc.assert_kernels_ran(names, want)
    assert not [k for k in not_want if k in names], (name, not_want, names)


# ---- refusals at creation ---------------------------------------------------------------------------------------------------
def _refused(engine, build, width, limit):
    with pytest.raises(engine.MxError) as ei:
        build()
    msg = str(ei.value)
    assert ("%d" % width) in msg and ("%d" % limit) in msg and "k_front_bwd" in msg, msg


def test_input_width_limit_refused_at_creation(emu_engine):
    """The recurrent QMIX step takes 384 input columns and refuses 385 (MMM2's 370 + 18 previous actions is 388); M-QMIX takes 320 and
    refuses 321; R-MADDPG refuses a critic input (state + every agent's actions) and an actor input over 320.  The message names the width
    and the limit."""
    import qmix_checks as qc
    import mqmix_checks as mc
    import maddpg_checks as mdc
    from oracle.maddpg import MaddpgConfig
    qc.build_trainer(cfg_of(384, 5, 2), 2, 3)
    _refused(emu_engine, lambda: qc.build_trainer(cfg_of(385, 5, 2), 2, 3), 385, 384)
    _refused(emu_engine, lambda: qc.build_trainer(cfg_of(370, 18, 10, prev=True), 2, 3), 388, 384)
    qc.build_trainer(cfg_of(370, 14, 10, prev=True), 2, 3)
    mc.build(cfg_of(320, 5, 2), 4, False)
    _refused(emu_engine, lambda: mc.build(cfg_of(321, 5, 2), 4, False), 321, 320)
    mdc.build(MaddpgConfig(n_agents=3, obs_dim=20, act_dim=5, state_dim=305, discrete=True), 2, 8)
    _refused(emu_engine, lambda: mdc.build(MaddpgConfig(n_agents=3, obs_dim=20, act_dim=5, state_dim=306, discrete=True), 2, 8), 321, 320)
    _refused(emu_engine, lambda: mdc.build(MaddpgConfig(n_agents=3, obs_dim=321, act_dim=5, state_dim=30, discrete=True), 2, 8), 321, 320)
    # MLP MADDPG / MATD3 at simple_spread with N agents and N landmarks: critic input 6 N^2 + 5 N -- N = 7 gives 294 + 35 = 329, refused;
    # the 320-column critic (295 + 5 x 5) builds and takes a step
    import mlp_maddpg_checks as mlc
    from offpolicy._b200.factory import build_mlp_maddpg
    for td3 in (False, True):
        _refused(emu_engine, lambda: build_mlp_maddpg(7, 42, 5, 294, 4, discrete=True, td3=td3), 329, 320)
        torch.manual_seed(2)
        args, pol, tr = build_mlp_maddpg(5, 30, 5, 295, 4, discrete=True, td3=td3)
        info, _, _ = tr.shared_train_policy_on_batch("policy_0", mlc.synth_batch(np.random.default_rng(3), 5, 4, 30, 295, 5, True))
        assert all(np.isfinite(float(info[k])) for k in ("critic_loss", "actor_loss")), info


# ---- wide inputs -------------------------------------------------------------------------------------------------------------
def run_wide(engine, width, B, T, N, note, stream=None, rules=RULES, every_up_to=16):
    from oracle.qmix import synth_batch
    obs, act, prev, debug = WIDE[width]
    if note:
        print("shape note:", note)
    cfg = cfg_of(obs, act, N, prev=prev)
    L64, pol, tr = rc.qmix_pair(cfg, B, T, debug=debug)
    batch = rc.last_episode_full_length(synth_batch(cfg, B, T, seed=5, avail_p=0.8, var_len=True) + (np.ones(B, np.float32), np.arange(B)))
    TM, _, grid = rules.agent_rows(B * (T + 1) * N, width)["k_front_bwd"]
    eps = rc.sample_episodes(B, T, N, TM, grid, every_up_to=every_up_to)
    names = rc.kernels_run(engine.lib(), stream, lambda: rc.isolated_episode_gradients(L64, tr, batch, eps[:1], B, T, N))
    assert_ffma_wide(names)
    if prev:
        rc.assert_kernels_ran(names, ["k_pack_prev_act"])
    worst_g = rc.isolated_episode_gradients(L64, tr, batch, eps, B, T, N)
    worst_f = rc.per_row_forward(L64, tr, batch, B, T, N, debug)
    gk, fk = max(worst_g, key=worst_g.get), max(worst_f, key=worst_f.get)
    print("sms %d in_dim %d B %d T %d N %d M %d (tiles of %d): %d episodes isolated; worst gradient %s %.2e (bound %.0e); worst row %s %.2e "
          "(bound %.0e)" % (rules.sms, width, B, T, N, B * (T + 1) * N, TM, len(eps), gk, worst_g[gk], rc.GRAD_TOL, fk, worst_f[fk], rc.ROW_TOL))


TAGS = {"one tile": "one", "tail 1": "tail1", "tail TM-1": "tailTMm1", "tiles = sms": "sms", "tiles = sms+1": "smsp1", "tiles = 2 sms+1": "2smsp1",
        "episode inside one tile": "epin1", "episode spans three tiles": "epspan3"}
# the emulator runs every edge at the first FFMA width and at the widest; the SMAC widths take the tail edges
EMU_TARGETS = {129: None, 384: None}
TAIL_TARGETS = ["tail 1", "tail TM-1", "tiles = sms+1"]


def _wide_cases():
    out = []
    for width in WIDE:
        tgts = EMU_TARGETS.get(width, TAIL_TARGETS)
        for tg, (B, T, N), lay, note in rc.pick_shapes(RULES, width, Ns=(2, 3, 5), Ts=range(2, 25), Bs=range(1, 65), targets=tgts):
            out.append(pytest.param(width, B, T, N, note, id="in%d-B%d-T%d-N%d-%s" % (width, B, T, N, "_".join(TAGS[t] for t in tg))))
    return out


@pytest.mark.parametrize("width,B,T,N,note", _wide_cases())
def test_wide_input_isolated_episodes_and_rows(emu_engine, width, B, T, N, note):
    run_wide(emu_engine, width, B, T, N, note)


@pytest.mark.parametrize("obs,B", [(129, 5), (129, 11), (320, 5), (320, 11)])
def test_mqmix_wide_input_isolated_transitions(emu_engine, obs, B):
    """Transition-level M-QMIX above 128 columns: FFMA k_front_fwd / k_front_bwd without k_gru_wgrad (no GRU), up to its 320-column
    limit; B = 5 / 11 put 30 / 66 rows on the 32-row tiles (a tail of 30 and of 2)."""
    from oracle.mqmix import synth_transitions
    N = 3
    cfg = cfg_of(obs, 6, N, S=14)
    L64, pol, tr = rc.mqmix_pair(cfg, B)
    batch = synth_transitions(cfg, B, seed=7, avail=True) + (None, None)
    TM, _, grid = RULES.agent_rows(2 * N * B, obs, gru_ext=False)["k_front_bwd"]
    eps = rc.sample_episodes(B, 1, N, TM, grid)
    names = rc.kernels_run(emu_engine.lib(), None, lambda: rc.isolated_episode_gradients(L64, tr, batch, eps[:1], B, 1, N, mlp=True,
                                                                                          ulps=rc.td_ulps(obs)))
    rc.assert_kernels_ran(names, ["k_front_fwd", "k_front_bwd", "k_mlp_dgi"])
    assert "k_gru_wgrad" not in names and not [n for n in names if "_tc" in n], names
    worst = rc.isolated_episode_gradients(L64, tr, batch, eps, B, 1, N, mlp=True, ulps=rc.td_ulps(obs))
    print("M-QMIX in_dim %d B %d: worst gradient %.2e (bound %.0e)" % (obs, B, max(worst.values()), rc.GRAD_TOL))


# ---- many agents -------------------------------------------------------------------------------------------------------------
# (N, A, extra cfg, debug, kernels): SMAC's 9 / 10 agents (MMM, 10m_vs_11m), the k_mid limit at 18 actions and one past it, 24 / 27 / 32
# agents with their action counts, both hypernet depths and VDN at 32
MANY = {
    "N9_A15_product": (9, 15, {}, False, ["k_mid"]),
    "N10_A17_debug": (10, 17, {}, True, ["k_qhead", "k_mix_core", "k_qhead_bwd"]),
    "N17_A18_product": (17, 18, {}, False, ["k_mid"]),
    "N18_A18_product": (18, 18, {}, False, ["k_qhead", "k_qhead_bwd"]),
    "N24_A30_debug": (24, 30, {}, True, ["k_qhead", "k_mix_core"]),
    "N27_A36_product": (27, 36, {}, False, ["k_qhead", "k_qhead_bwd"]),
    "N32_A31_hyper1_debug": (32, 31, dict(hyper_layers=1), True, ["k_qhead", "k_mix_core"]),
    "N32_A64_hyper2_product": (32, 64, {}, False, ["k_qhead", "k_qhead_bwd"]),
    "N32_A36_vdn_debug": (32, 36, dict(vdn=True), True, ["k_qhead", "k_qhead_bwd"]),
}


def run_many(engine, key, B, T, stream=None, obs=11, S=13):
    from oracle.qmix import synth_batch
    N, A, over, debug, kernels = MANY[key]
    cfg = cfg_of(obs, A, N, S=S, **over)
    L64, pol, tr = rc.qmix_pair(cfg, B, T, debug=debug)
    batch = rc.last_episode_full_length(synth_batch(cfg, B, T, seed=5, avail_p=0.8, var_len=True) + (np.ones(B, np.float32), np.arange(B)))
    names = rc.kernels_run(engine.lib(), stream, lambda: rc.isolated_episode_gradients(L64, tr, batch, [B - 1], B, T, N))
    rc.assert_kernels_ran(names, kernels)
    worst_g = rc.isolated_episode_gradients(L64, tr, batch, list(range(B)), B, T, N)
    worst_f = rc.per_row_forward(L64, tr, batch, B, T, N, debug)
    worst_t = rc.per_transition(L64, tr, batch, B, T, N, debug, agent_values="k_mid" not in names)
    gk, tk = max(worst_g, key=worst_g.get), max((k for k in worst_t if k != "greedy decided rows"), key=worst_t.get)
    print("N %d A %d B %d T %d S %d: worst gradient %s %.2e (bound %.0e); worst row %.2e; worst transition %s %.2e (bound %.0e)%s"
          % (N, A, B, T, S, gk, worst_g[gk], rc.GRAD_TOL, max(worst_f.values()), tk, worst_t[tk], rc.ROW_TOL,
             "; greedy checked on %d rows" % worst_t["greedy decided rows"] if debug else ""))


@pytest.mark.parametrize("key", list(MANY))
def test_many_agents_isolated_rows_and_transitions(emu_engine, key):
    run_many(emu_engine, key, 2, 3)


@pytest.mark.parametrize("N,S", [(27, 129), (32, 65)])
def test_many_agents_wide_state(emu_engine, N, S):
    """The first wide state at 27 and 32 agents (the mixer's tile holds N 32 columns of hypernet output): the state GEMMs beside k_mid's
    fallback, isolated episodes and every transition."""
    from oracle.qmix import synth_batch
    B, T = 2, 3
    cfg = cfg_of(11, 31, N, S=S)
    L64, pol, tr = rc.qmix_pair(cfg, B, T, debug=True)
    batch = rc.last_episode_full_length(synth_batch(cfg, B, T, seed=5, avail_p=0.8, var_len=True) + (np.ones(B, np.float32), np.arange(B)))
    names = rc.kernels_run(emu_engine.lib(), None, lambda: rc.isolated_episode_gradients(L64, tr, batch, [0], B, T, N))
    rc.assert_kernels_ran(names, ["k_mixw_fwd", "k_mixw_wgrad"])
    worst = rc.isolated_episode_gradients(L64, tr, batch, list(range(B)), B, T, N)
    worst_t = rc.per_transition(L64, tr, batch, B, T, N, True)
    gk, tk = max(worst, key=worst.get), max((k for k in worst_t if k != "greedy decided rows"), key=worst_t.get)
    print("N %d S %d: worst gradient %s %.2e (bound %.0e); worst transition %s %.2e (bound %.0e)"
          % (N, S, gk, worst[gk], rc.GRAD_TOL, tk, worst_t[tk], rc.ROW_TOL))


@pytest.mark.parametrize("vdn", [False, True])
def test_mqmix_32_agents_isolated_transitions(emu_engine, vdn):
    """M-QMIX / M-VDN with 32 agents: 2 N B rows, each transition's gradient alone."""
    from oracle.mqmix import synth_transitions
    N, B = 32, 3
    cfg = cfg_of(20, 15, N, S=14, vdn=vdn)
    L64, pol, tr = rc.mqmix_pair(cfg, B)
    batch = synth_transitions(cfg, B, seed=7, avail=True) + (None, None)
    worst = rc.isolated_episode_gradients(L64, tr, batch, list(range(B)), B, 1, N, mlp=True)
    print("M-%s N 32 B %d: worst gradient %.2e (bound %.0e)" % ("VDN" if vdn else "QMIX", B, max(worst.values()), rc.GRAD_TOL))


# ---- the wide-state GEMMs, block by block ----------------------------------------------------------------------------------------
# (N, hypernet layers, S, B, T): more than 128 state rows ending in a partial 128-row tile (B (T+1) = 135), E = B T = 132 elements (not a
# multiple of the 32-element K chunk of the weight gradient), S = 449 = 7 x 64 + 1 (a last state chunk and feature tile of one column);
# stacked columns 160 + 32 + 64 + 32 = 288 (1-layer hypernets at N 5: two full 128-column blocks and a partial one of 32) and
# 64 + 64 + 64 + 32 = 224 (2-layer: one full block and a partial one of 96)
GEMM_CASES = [(5, 1, 449, 3, 44), (5, 2, 449, 3, 44)]


@pytest.mark.parametrize("N,layers,S,B,T", GEMM_CASES)
def test_state_gemms_every_block_vs_float64(emu_engine, N, layers, S, B, T):
    from oracle.qmix import synth_batch
    cfg = cfg_of(11, 5, N, S=S, hyper_layers=layers)
    L64, pol, tr = rc.qmix_pair(cfg, B, T, debug=True)
    batch = synth_batch(cfg, B, T, seed=4, avail_p=0.8, var_len=True) + (np.ones(B, np.float32), np.arange(B))
    names = rc.kernels_run(emu_engine.lib(), None, lambda: tr.train_policy_on_batch(rc.qc.ref_tuple(batch)))
    rc.assert_kernels_ran(names, ["k_mixw_fwd", "k_mixw_wgrad"])
    worst = rc.state_gemm_blocks(L64, tr, batch, B, T)
    k = max(worst, key=worst.get)
    print("N %d layers %d S %d rows %d elements %d: worst %s %.2e (bound %.0e)" % (N, layers, S, B * (T + 1), B * T, k, worst[k], rc.GEMM_TOL))
