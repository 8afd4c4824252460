"""Transition-level coverage of the MLP MADDPG / MATD3 learner on the CPU-emulated kernels (4 SMs): isolated critic transitions and
actor rows, per-transition priorities and a changing batch size against the float64 oracle, at batch sizes on the tile edges of the
step's three row spaces (tests/mlp_maddpg_row_checks.py)."""
import numpy as np
import pytest

import mlp_maddpg_row_checks as rk

EMU_SMS = 4
RULES = rk.TileRules(EMU_SMS)
# simple_spread (scripts/train_mpe_maddpg.sh): 3 agents, obs 18, Discrete(5), shared observation 54 -> critic input 69 (> 64: the
# tensor-core backward k_front_bwd_tc + k_wgrad_tc); the actor's 18 columns take k_front_bwd
SPREAD = [(18, 5, 3)]


def _check(worst, stats):
    assert worst["grad"] <= rk.GRAD_TOL and worst["td_ulps"] <= rk.TD_ULPS
    print("worst", worst, "redraws", stats["redraws"], "of them ill-conditioned", stats.get("ill_conditioned", 0),
          "smallest margin kept %.2e" % stats.get("min_margin", float("inf")))


EDGES = rk.pick_batches(RULES, 3, 18, 69)
# Not run here: the copies' nearest edge to sms + 1 tiles (B 86) and the wide critic's sms / sms + 1 chunks (B 193, 257), which take
# 86 to 257 emulated transitions; test_gpu_mlp_maddpg_rows.py runs every edge at the device's SM count
EMU_EDGES = [e for e in EDGES if e[0] <= 65]


def test_edge_batches_cover_every_row_space():
    """Every (row space, edge) has a batch size; the edges the tile rules cannot produce say so."""
    got = {t for _, tg, _ in EDGES for t in tg}
    assert got == {sp + " " + e for sp in ("critic", "actor", "copies") for e in rk.EDGE_TARGETS}
    notes = [n for _, _, n in EDGES if n]
    assert any(n.startswith("actor tail 1 cannot occur") for n in notes), notes


@pytest.mark.parametrize("B,edges,note", EMU_EDGES, ids=["B%d" % B for B, _, _ in EMU_EDGES])
def test_simple_spread_matd3_edges(emu_engine, B, edges, note):
    """MATD3, Discrete: the tile edges of the critic (69 columns), the actor (18) and the agent-replaced copies (69)."""
    _check(*rk.run_case(emu_engine, None, RULES, SPREAD, 54, True, True, [B]))


# (specs, S, discrete, td3, avail, batch sizes, overrides): batch sizes on an edge of the path's row kernels at 4 SMs.  The narrow critic
# (FFMA k_front_bwd on its B rows) runs at its sms-tile edge (B 97) and its TM-1 tail (B 31); its nearest edge to sms + 1 tiles (B 257)
# runs on the device only
CASES = {
    "maddpg_disc_next_avail": (SPREAD, 54, True, False, True, [11], {}),
    "maddpg_box": (SPREAD, 54, False, False, False, [5], {}),
    "matd3_box": (SPREAD, 54, False, True, False, [21], {}),
    "matd3_disc_tanh": (SPREAD, 54, True, True, False, [5], {"use_ReLU": False}),
    # critic input 20 + 2 x 5 = 30 <= 64: the FFMA k_front_bwd on all three row spaces
    "narrow_critic_maddpg": ([(10, 5, 2)], 20, True, False, False, [97], {}),
    "narrow_critic_matd3_box": ([(10, 5, 2)], 20, False, True, False, [31], {}),
    # actor observation widths 57-64 and 65-128
    "obs60": ([(60, 5, 2)], 20, True, True, False, [9], {}),
    "obs100": ([(100, 5, 2)], 20, True, False, False, [9], {}),
    # MultiDiscrete: simple_reference's [5, 10], and three blocks
    "md_5_10": ([(21, [5, 10], 2)], 42, True, True, False, [9], {}),
    "md_three_blocks": ([(16, [3, 4, 2], 3)], 30, True, False, False, [7], {}),
}


@pytest.mark.parametrize("name", list(CASES))
def test_isolated_transitions(emu_engine, name):
    specs, S, disc, td3, avail, Bs, over = CASES[name]
    _check(*rk.run_case(emu_engine, None, RULES, specs, S, disc, td3, Bs, avail=avail, **over))


# several policies: simple_speaker_listener (speaker obs 3 / Discrete(3), listener obs 11 / Discrete(5)), and a two-agent policy at
# act_offset 4 behind a one-agent one; every updated policy's transitions isolated after every policy's cent_contribute
MULTI = {
    "speaker": ([(3, 3, 1), (11, 5, 1)], 14, "policy_0", True),
    "listener": ([(3, 3, 1), (11, 5, 1)], 14, "policy_1", True),
    "two_agent_policy_at_offset": ([(8, 4, 1), (10, 5, 2)], 16, "policy_1", False),
    "md_beside_discrete": ([(8, 4, 1), (12, [3, 5], 2)], 16, "policy_1", True),
}


@pytest.mark.parametrize("name", list(MULTI))
def test_isolated_transitions_several_policies(emu_engine, name):
    specs, S, p, td3 = MULTI[name]
    _check(*rk.run_case(emu_engine, None, RULES, specs, S, True, td3, [7], p=p))


# Above 128 input columns (tc_bwd.cu WG_MAX_IN) a net runs FFMA k_front_fwd forward and FFMA k_front_bwd backward on 32-row tiles of
# round_up(in, 64)-wide shared-memory rows (162 KB at 155-192 columns, 186 KB up to 256, 211 KB up to 320, the widest the learner takes).
# simple_spread with N agents and N landmarks (--num_agents / --num_landmarks): observation 6 N, shared observation 6 N^2, critic input
# 6 N^2 + 5 N -- 175 at N = 5, 246 at N = 6 (329 at N = 7 is refused).  Every batch size on an edge of the case's three row spaces.
# (specs, S, discrete, td3, avail, policies isolated)
WIDE = {
    "spread5_matd3_disc": ([(30, 5, 5)], 150, True, True, False, ["policy_0"]),
    "spread6_maddpg_disc_next_avail": ([(36, 5, 6)], 216, True, False, True, ["policy_0"]),
    "spread5_maddpg_box": ([(30, 5, 5)], 150, False, False, False, ["policy_0"]),
    "critic320_matd3_disc": ([(30, 5, 5)], 295, True, True, False, ["policy_0"]),
    "actor132_maddpg_disc": ([(132, 5, 2)], 20, True, False, False, ["policy_0"]),
    # one policy per agent: policy_0 writes the first action columns, policy_4 the last (act_offset 20)
    "spread5_per_agent_matd3_disc": ([(30, 5, 1)] * 5, 150, True, True, False, ["policy_0", "policy_4"]),
}


def edge_tag(edges):
    tag = {"one tile": "one", "tail 1": "tail1", "tail TM-1": "tailTMm1", "tiles = sms": "sms", "tiles = sms+1": "smsp1"}
    return "_".join(e.split(" ", 1)[0] + "_" + tag[e.split(" ", 1)[1]] for e in edges)


def wide_params(rules, Bmax=None):
    """(case, policy, B) per batch size on an edge of that policy's row spaces (B <= Bmax(case), every edge when Bmax is None), the id
    naming the edges."""
    out = []
    for name, (specs, S, disc, td3, avail, ps) in WIDE.items():
        for p in ps:
            for B, tg, note in rk.pick_batches(rules, *rk.geometry(specs, S, p)):
                if Bmax is None or B <= Bmax(name):
                    out.append(pytest.param(name, p, B, id="%s-%s-B%d-%s" % (name, p, B, edge_tag(tg))))
    return out


def test_wide_edges_cover_every_row_space():
    """Above 128 columns the critic's and the copies' row kernel is k_front_bwd on 32-row tiles, and every (row space, edge) of each
    wide case has a batch size.  At the parent commit row_tiles looked up k_wgrad_tc there and raised KeyError."""
    for name, (specs, S, disc, td3, avail, ps) in WIDE.items():
        for p in ps:
            N, O, cin = rk.geometry(specs, S, p)
            for B in (1, 31, 97, 129):
                sp = rk.spaces(RULES, B, N, O, cin)
                for space, w in (("critic", cin), ("copies", cin), ("actor", O)):
                    if w > 128:
                        assert sp[space][1:3] == ("k_front_bwd", 32), (name, space, B, sp[space])
            got = {t for _, tg, _ in rk.pick_batches(RULES, N, O, cin) for t in tg}
            assert got == {s + " " + e for s in ("critic", "actor", "copies") for e in rk.EDGE_TARGETS}, (name, p, got)


# Emulated: simple_spread N = 5 MATD3 at every edge up to B 31 (the copies' and the actor's sms / sms + 1 tiles, the critic's 31-row
# tail); the other cases up to B 11.  The critic's sms / sms + 1 tiles (B 97 / 129 here) and every other edge run on the device.
@pytest.mark.parametrize("name,p,B", wide_params(RULES, lambda name: 31 if name == "spread5_matd3_disc" else 11))
def test_isolated_transitions_above_128_columns(emu_engine, name, p, B):
    specs, S, disc, td3, avail, _ = WIDE[name]
    worst, stats = rk.run_case(emu_engine, None, RULES, specs, S, disc, td3, [B], p=p, avail=avail)
    _check(worst, stats)


@pytest.mark.parametrize("td3", [False, True])
def test_batch_size_changes_on_one_learner(emu_engine, td3):
    """max_batch = the actor's nearest edge to sms + 1 tiles (B 43), then B = 1, then one 48-row actor tile smaller (8 transitions)."""
    Bmax = max(B for B, tg, _ in EDGES if "actor tiles = sms+1" in tg)
    args, pols, tr, L64 = rk.build_pair(SPREAD, 54, Bmax, True, td3, use_per=True)
    stats = {"redraws": 0}
    worst = rk.batch_size_sequence(args, tr, pols, L64, "policy_0", rk.make_batches(SPREAD, 54, True), [Bmax, 1, Bmax - 8], 5,
                                   np.random.default_rng(5), stats, RULES, emu_engine)
    print("worst", worst, "redraws", stats["redraws"])
