"""Row and tile coverage of the QMIX / M-QMIX learner kernels on the CPU fiber emulator (4 SMs), against the float64 oracle.

Shapes come from tests/row_coverage_checks.py's restatement of the launchers' tile rules: one tile with every other CTA idle, a last tile
holding one row or one row short of full, one CTA running a second (third) tile, an episode inside one tile and one across three,
the mixer's 16 sms / 16 sms + 1 transitions.  Each shape isolates every episode's gradient in turn and checks every row of the forward;
each test also asserts that the kernel it means to pin actually ran."""
import os
import subprocess
import sys

import numpy as np
import pytest

import row_coverage_checks as rc

EMU_SMS = 4
RULES = rc.TileRules(EMU_SMS)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))

# path: (obs_dim, act_dim, prev_act_inp, debug, kernels that must run)
PATHS = {
    # obs <= 56: k_front_fwd_tc2 (marked k_front_fwd_tc), FFMA k_front_bwd + k_gru_wgrad; debug: k_qhead / k_mix_core / k_qhead_bwd
    "obs11_debug": (11, 5, False, True, ["k_front_fwd_tc", "k_front_bwd", "k_gru_wgrad", "k_qhead", "k_mix_core", "k_qhead_bwd"]),
    # obs 57..64: the one-thread-per-row k_front_fwd_tc (marked k_front_fwd_tc1); two actions per lane (A = 36); product configuration: k_mid
    "obs60_a36_product": (60, 36, False, False, ["k_front_fwd_tc1", "k_front_bwd", "k_gru_wgrad", "k_mid"]),
    # --prev_act_inp: [obs | previous action] packed per step
    "prev_act_product": (11, 9, True, False, ["k_pack_prev_act", "k_front_bwd", "k_mid"]),
    # obs 65..128: k_front_fwd_tc_wide2 + k_front_bwd_tc (two CTAs per SM) + k_wgrad_tc
    "obs80_debug": (80, 9, False, True, ["k_front_fwd_tc_wide", "k_front_bwd_tc", "k_wgrad_tc", "k_qhead_bwd"]),
    # in_dim 81..128: k_front_bwd_tc at one CTA per SM; A = 64 (two actions per lane at the limit), product configuration (k_mid
    # where its operands fit, k_qhead / k_qhead_bwd at N = 5)
    "obs120_a64_product": (120, 64, False, False, ["k_front_fwd_tc_wide", "k_front_bwd_tc", "k_wgrad_tc", "k_mid"]),
}


def _cfg(obs, act, prev, N, S=13, **over):
    from oracle.qmix import QmixConfig
    return QmixConfig(n_agents=N, obs_dim=obs, act_dim=act, state_dim=S, gain=1.0, prev_act_inp=prev, use_per=True, **over)


def _in_dim(path):
    obs, act, prev = PATHS[path][:3]
    return obs + (act if prev else 0)


TAGS = {"one tile": "one", "tail 1": "tail1", "tail TM-1": "tailTMm1", "tiles = sms": "sms", "tiles = sms+1": "smsp1", "tiles = 2 sms+1": "2smsp1",
        "episode inside one tile": "epin1", "episode spans three tiles": "epspan3", "front_bwd_tc tiles = CTAs+1": "bwdtcp1",
        "E = 16 sms": "E16sms", "E = 16 sms+1": "E16smsp1"}


def _cases():
    out = []
    for path in PATHS:
        for tg, (B, T, N), lay, note in rc.pick_shapes(RULES, _in_dim(path), Ns=(2, 3, 5), Ts=range(2, 25), Bs=range(1, 65)):
            out.append(pytest.param(path, B, T, N, note, id="%s-B%d-T%d-N%d-%s" % (path, B, T, N, "_".join(TAGS[t] for t in tg))))
    for tg, (B, T, N), lay, note in rc.pick_mixer_shapes(RULES):
        for path in ("obs11_debug", "obs60_a36_product"):
            out.append(pytest.param(path, B, T, N, note, id="%s-B%d-T%d-N%d-%s" % (path, B, T, N, TAGS[tg[0]])))
    return out


def run_isolated(engine, path, B, T, N, note, S=13, extra_kernels=()):
    from oracle.qmix import synth_batch
    obs, act, prev, debug, kernels = PATHS[path]
    if note:
        print("shape note:", note)
    cfg = _cfg(obs, act, prev, N, S=S)
    L64, pol, tr = rc.qmix_pair(cfg, B, T, debug=debug)
    batch = rc.last_episode_full_length(synth_batch(cfg, B, T, seed=5, avail_p=0.8, var_len=True) + (np.ones(B, np.float32), np.arange(B)))
    lib = engine.lib()
    lay = RULES.agent_rows(B * (T + 1) * N, _in_dim(path))
    TM, _, grid = lay[RULES.row_kernel(_in_dim(path))]
    eps = rc.sample_episodes(B, T, N, TM, grid)
    names = rc.kernels_run(lib, None, lambda: rc.isolated_episode_gradients(L64, tr, batch, eps[:1], B, T, N))
    rc.assert_kernels_ran(names, list(kernels) + list(extra_kernels))
    worst_g = rc.isolated_episode_gradients(L64, tr, batch, eps, B, T, N)
    # the workspace holds the forward of the last isolated step, taken from the restored state: every row against float64
    worst_f = rc.per_row_forward(L64, tr, batch, B, T, N, debug)
    gk = max(worst_g, key=worst_g.get)
    fk = max(worst_f, key=worst_f.get)
    print("B %d T %d N %d M %d: %d episodes isolated; worst gradient %s %.2e (bound %.0e); worst row %s %.2e (bound %.0e)"
          % (B, T, N, B * (T + 1) * N, len(eps), gk, worst_g[gk], rc.GRAD_TOL, fk, worst_f[fk], rc.ROW_TOL))
    return worst_g, worst_f


def test_tile_rules_restatement():
    """The Python tile rules reproduce the launchers' documented choices: 3m (5 856 rows) takes 48-row tiles on the H100 (one wave of
    122, not two of 183); the emulator's 192 / 256 / 288 rows take 48 / 64 / 48 (tests/test_emu_qmix.py); the mixer switches to 32-row
    tiles above 16 sms transitions; k_front_bwd_tc runs two CTAs per SM up to 80 input columns."""
    assert rc.TileRules(132).front_bwd_rm(5856, 30, True) == 3
    assert [RULES.front_bwd_rm(M, 11, True) for M in (192, 256, 288)] == [3, 4, 3]
    assert RULES.mixer_rows(64)[0] == 16 and RULES.mixer_rows(65)[0] == 32
    assert RULES.bwd_tc_ctas_per_sm(80) == 2 and RULES.bwd_tc_ctas_per_sm(81) == 1
    for sms in (4, 132):
        R = rc.TileRules(sms)
        for ind in (11, 80):
            got = rc.pick_shapes(R, ind, Ns=(2, 3, 5, 8), Ts=range(2, 65), Bs=range(1, 130))
            hit = set(t for tg, _, _, _ in got for t in tg)
            assert set(rc.AGENT_TARGETS) <= hit, (sms, ind, hit)


@pytest.mark.parametrize("name", ["qmix_small", "qmix_small_per", "qmix_small_prev_act"])
def test_float64_oracle_reproduces_reference_golden(name):
    """The float64 learner is the same step: built from the golden's state with .double(), its first step's loss and clipped gradients
    agree with the reference's float32 ones to float32 round-off."""
    import torch
    from helpers import load_golden, oracle_from_golden, golden_batch, rel_err
    g = load_golden(name)
    L, cfg, B, T, steps = oracle_from_golden(g)
    L64 = rc.float64_twin(L)
    assert all(p.dtype == torch.float64 for p in L64.params)
    info, _, _ = L64.step(golden_batch(g, 0))
    assert rel_err(info["loss"], g["s0.loss"]) < 1e-5
    for role, mod in (("agent", L64.agent), ("mixer", L64.mixer)):
        for k, p in mod.named_parameters():
            key = "s0.grad.%s.%s" % (role, k)
            if key in g:
                assert p.grad.dtype == torch.float64 and rel_err(p.grad, g[key]) < 1e-4, key


@pytest.mark.parametrize("path,B,T,N,note", _cases())
def test_isolated_episode_gradients_and_rows(emu_engine, path, B, T, N, note):
    run_isolated(emu_engine, path, B, T, N, note)


@pytest.mark.parametrize("S,B,T", [(449, 3, 11), (449, 2, 16), (481, 1, 5)])
def test_wide_state_mixer_isolated(emu_engine, S, B, T):
    """The wide-state mixer (k_mixw_fwd / k_mixw_wgrad): S = 449 and 481 are one past a multiple of its 32-feature K chunk (the state
    switches to this path between 384 and 448 at N = 3); E = 33 / 32 / 5 transitions against its 32-element K chunk of the weight
    gradient."""
    run_isolated(emu_engine, "obs11_debug", B, T, 3, "", S=S, extra_kernels=("k_mixw_fwd", "k_mixw_wgrad"))


@pytest.mark.parametrize("B", [1, 5, 11, 64, 65])
def test_mqmix_isolated_transitions(emu_engine, B):
    """Transition-level M-QMIX: M = 2 N B rows (observation and next observation), E = B transitions; B = 64 / 65 are the mixer's
    16 sms / 16 sms + 1 transitions.  Each transition's gradient alone (first, last and CTA-boundary ones above 16)."""
    from oracle.qmix import QmixConfig
    from oracle.mqmix import synth_transitions
    N = 3
    cfg = QmixConfig(n_agents=N, obs_dim=20, act_dim=6, state_dim=14, gain=1.0, use_per=True)
    L64, pol, tr = rc.mqmix_pair(cfg, B)
    batch = synth_transitions(cfg, B, seed=7, avail=True) + (None, None)
    TM, _, grid = RULES.agent_rows(2 * N * B, 20)["k_front_bwd"]
    eps = rc.sample_episodes(B, 1, N, TM, grid)
    names = rc.kernels_run(emu_engine.lib(), None, lambda: rc.isolated_episode_gradients(L64, tr, batch, eps[:1], B, 1, N, mlp=True))
    assert "k_front_bwd" in names and "k_mlp_dgi" in names, names
    worst = rc.isolated_episode_gradients(L64, tr, batch, eps, B, 1, N, mlp=True)
    print("M-QMIX B %d: worst gradient %.2e (bound %.0e)" % (B, max(worst.values()), rc.GRAD_TOL))


@pytest.mark.parametrize("path", ["obs11_debug", "obs80_debug"])
def test_batch_size_changes_on_one_learner(emu_engine, path):
    """One learner (max_batch = the batch of the 2 sms + 1 tile edge): a step at max_batch, one at B = 1, one at the largest B that
    needs one tile fewer than max_batch; each against float64 (gradients, loss, priorities, Adam update, soft update)."""
    obs, act, prev, debug, kernels = PATHS[path]
    ind = _in_dim(path)
    (tg, (Bmax, T, N), lay, note), = [s for s in rc.pick_shapes(RULES, ind, Ns=(2, 3, 5), Ts=range(2, 25), Bs=range(1, 65),
                                                               targets=["tiles = 2 sms+1"])]
    kern = RULES.row_kernel(ind)
    tiles = lambda B: RULES.agent_rows(B * (T + 1) * N, ind)[kern][1]
    fewer = [B for B in range(1, Bmax) if tiles(B) < tiles(Bmax)]
    Bs = [Bmax, 1, max(fewer, key=lambda B: (tiles(B), B))]
    print("batch sizes", Bs, "tiles", [tiles(B) for B in Bs])
    cfg = _cfg(obs, act, prev, N)
    L64, pol, tr = rc.qmix_pair(cfg, Bmax, T, debug=debug)
    worst = rc.batch_size_sequence(L64, pol, tr, cfg, Bs, T)
    print("worst gradient %.2e (bound %.0e)" % (max(worst.values()), rc.GRAD_TOL))


@pytest.mark.parametrize("path", ["obs11_debug", "obs80_debug"])
def test_isolated_gradients_reverse_thread_order(path):
    """The isolated-gradient checks of the tile-tail shapes with the emulator's threads run in reverse order (missing barriers)."""
    env = dict(os.environ, EMU_ORDER="reverse")
    code = ("import sys; sys.path[:0] = [%r, %r, %r]\n"
            "import pytest\n"
            "sys.exit(pytest.main(['-q', '-x', '-p', 'no:cacheprovider', %r, '-k', "
            "'test_isolated_episode_gradients_and_rows and %s and (tail1 or tailTMm1 or smsp1)']))\n"
            % (ROOT, os.path.join(ROOT, "off-policy_b200"), HERE, os.path.abspath(__file__), path))
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]


def _maddpg_cases():
    return [pytest.param(disc, B, T, N, id="%s-B%d-T%d-%s" % ("disc" if disc else "box", B, T, "_".join(t.replace(" ", "").replace("=", "").replace("+", "p")
                                                                                                          for t in tg)))
            for tg, (B, T, N), lay, note in rc.pick_maddpg_shapes(RULES) for disc in (False, True)]


def run_maddpg(engine, disc, B, T, N, stream=None, every_up_to=16, rules=RULES, td3=False, obs=None, S=None):
    from oracle.maddpg import MaddpgConfig, synth_batch_cont, synth_batch_disc
    kw = {} if obs is None else dict(obs_dim=obs, state_dim=S)
    cfg = MaddpgConfig(n_agents=N, act_dim=5 if disc else 2, discrete=disc, td3=td3, actor_update_interval=2 if td3 else 1, gain=1.0,
                       use_per=True, **kw)      # R_MATD3 trains the actor on every second update
    L64, pol, tr = rc.maddpg_pair(cfg, B, T)
    batch = (synth_batch_disc if disc else synth_batch_cont)(cfg, B, T, seed=40) + (None, None)
    batch = rc.last_episode_full_length(batch)
    _, _, grid = rules.head_rows(B * T)
    eps = rc.sample_episodes(B, T - 1, 1, 32, grid, every_up_to=every_up_to)       # critic rows: T per episode
    names = rc.kernels_run(engine.lib(), stream, lambda: rc.maddpg_isolated_episodes(L64, pol, tr, batch, eps[:1], B, T))
    rc.assert_kernels_ran(names, ["k_head_bwd", "k_gru_bwd", "k_front_bwd"])
    cin = cfg.state_dim + N * cfg.act_dim
    if cin > 128:          # FFMA forward and backward for the critic and its copies; the actor (<= 64 or > 128 here) on k_front_bwd too
        assert "k_front_fwd" in names and not {"k_front_bwd_tc", "k_wgrad_tc"} & set(names), names
    if cin > 128 and cfg.obs_dim > 128:     # every net above 128 columns: no tensor-core forward anywhere in the step
        assert not [k for k in names if k.startswith("k_front_fwd_tc")], names
    worst = rc.maddpg_isolated_episodes(L64, pol, tr, batch, eps, B, T)
    k = max(worst, key=worst.get)
    print("R-%s %s obs %d critic %d B %d T %d N %d (critic rows %d, actor rows %d): %d episodes isolated; worst gradient %s %.2e (bound %.0e)"
          % ("MATD3" if td3 else "MADDPG", "Discrete" if disc else "Box", cfg.obs_dim, cin, B, T, N, B * T, B * (T + 1) * N, len(eps), k,
             worst[k], rc.GRAD_TOL))
    return worst


# R-MADDPG / R-MATD3 above 128 critic columns (FFMA k_front_fwd / k_front_bwd on 32-row tiles, the GRU weight gradients inside
# k_front_bwd, the copies' data gradient through the critic's input LayerNorm): name: (N, obs, S, Discrete, TD3)
MADDPG_WIDE = {
    "spread5_rmaddpg_disc_critic175": (5, 30, 150, True, False),
    "spread6_rmatd3_box_critic228": (6, 36, 216, False, True),
    "actor140_critic316_rmaddpg_disc": (3, 140, 301, True, False),
    "critic320_rmatd3_disc": (5, 30, 295, True, True),
}


def maddpg_wide_params(rules, keep=lambda B, T: True):
    """(case, B, T) per shape on the k_head_bwd and k_front_bwd edges of the case's row spaces (episodes of 4 to 39 steps: T < 8 runs
    k_gru_bwd's short-sequence variant, T >= 8 k_gru_bwd2), the id naming the edges."""
    out = []
    short = lambda t: t.replace("front ", "").replace("tiles = sms+1", "smsp1").replace("tiles = sms", "sms").replace("tail TM-1", "tailTMm1") \
        .replace("one tile", "one").replace(" ", "")
    for name, (N, obs, S, disc, td3) in MADDPG_WIDE.items():
        cin = S + N * (5 if disc else 2)
        for tg, (B, T, _), lay, note in rc.pick_maddpg_shapes(rules, N=N, Ts=range(4, 40), Bs=range(1, 200), obs=obs, cin=cin):
            if keep(B, T):
                out.append(pytest.param(name, B, T, id="%s-B%d-T%d-%s" % (name, B, T, "_".join(sorted({short(t) for t in tg})))))
    return out


def test_maddpg_wide_shapes_cover_every_edge():
    """Each wide case has shapes on every k_front_bwd edge of its three spaces (an edge that cannot occur -- the odd tails of the actor's
    and the copies' rows at an even agent count, a tile count the tile rule skips -- on the nearest one, named in the note), episodes
    shorter than 8 among them, and 32-row tiles wherever a space is above 128 columns."""
    for name, (N, obs, S, disc, td3) in MADDPG_WIDE.items():
        cin = S + N * (5 if disc else 2)
        shapes = rc.pick_maddpg_shapes(RULES, N=N, Ts=range(4, 40), Bs=range(1, 200), obs=obs, cin=cin)
        got = {t for tg, _, _, _ in shapes for t in tg}
        notes = " ".join(n for _, _, _, n in shapes)
        assert "T < 8" in got, name
        for space in ("critic", "actor", "copies"):
            for e in rc.FRONT_TARGETS:
                assert "%s front %s" % (space, e) in got, (name, space, e)
        for space in ("actor", "copies"):
            for e in ("tail 1", "tail TM-1"):
                assert ("%s front %s cannot occur (an even row count)" % (space, e) in notes) == (N % 2 == 0), (name, space, e, notes)
        for space, (M, TM, nt) in rc.maddpg_front_spaces(RULES, 3, 9, N, obs, cin).items():
            assert TM == 32 or (space == "actor" and obs <= 64), (name, space, TM)


@pytest.mark.parametrize("name,B,T", maddpg_wide_params(RULES, keep=lambda B, T: B == 1 and T <= 20))
def test_maddpg_isolated_episodes_above_128_columns(emu_engine, name, B, T):
    """Emulated: the one-episode shapes up to T 20 (one tile, the tails, T < 8); the multi-tile edges run on the device."""
    N, obs, S, disc, td3 = MADDPG_WIDE[name]
    run_maddpg(emu_engine, disc, B, T, N, td3=td3, obs=obs, S=S)


@pytest.mark.parametrize("disc,B,T,N", _maddpg_cases())
def test_maddpg_isolated_episode_gradients(emu_engine, disc, B, T, N):
    """R-MADDPG critic and actor, Box and Discrete, T >= 8 (k_gru_bwd2's T1 = T branch for the critic sequences), on the edges of
    k_head_bwd's 32-row tiles for the critic's B T rows and the actor's B (T+1) N rows."""
    run_maddpg(emu_engine, disc, B, T, N)


@pytest.mark.parametrize("act", [36, 64])
def test_two_actions_per_lane_in_the_fused_mid_kernel(emu_engine, act):
    """k_mid itself (no fallback accepted) with two actions per lane, A = 36 and 64, at a shape whose operands fit it (N = 3): isolated
    episodes and every row, and k_front_fwd_tc2 (not the one-thread-per-row variant) at obs 11."""
    from oracle.qmix import synth_batch
    B, T, N = 3, 9, 3
    cfg = _cfg(11, act, False, N)
    L64, pol, tr = rc.qmix_pair(cfg, B, T, debug=False)
    batch = rc.last_episode_full_length(synth_batch(cfg, B, T, seed=6, avail_p=0.8, var_len=True) + (np.ones(B, np.float32), np.arange(B)))
    names = rc.kernels_run(emu_engine.lib(), None, lambda: rc.isolated_episode_gradients(L64, tr, batch, [0], B, T, N))
    assert "k_mid" in names and "k_front_fwd_tc" in names and "k_front_fwd_tc1" not in names, names
    rc.isolated_episode_gradients(L64, tr, batch, list(range(B)), B, T, N)
    rc.per_row_forward(L64, tr, batch, B, T, N, False)


@pytest.mark.parametrize("td3", [False, True], ids=["rmaddpg", "rmatd3"])
def test_maddpg_oracle_lockstep_above_128_columns(emu_engine, td3):
    """Whole R-MADDPG / R-MATD3 updates at simple_spread N = 5 (critic 175), three in a row, against the fp32 oracle (the H100 runs
    the script's B 32, T 25)."""
    import maddpg_checks as mdc
    from oracle.maddpg import MaddpgConfig
    cfg = MaddpgConfig(n_agents=5, obs_dim=30, act_dim=5, state_dim=150, discrete=True, td3=td3, actor_update_interval=2 if td3 else 1,
                       gain=1.0, use_per=True)
    print("worst gradient / bound %.2f" % mdc.check_oracle_lockstep(cfg, 3, 9))
