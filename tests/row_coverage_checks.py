"""Row and tile coverage of the QMIX / M-QMIX learners against a float64 oracle: shared by the emulated (CPU) and the GPU test modules.

The lock-step checks (qmix_checks.check_engine_step) compare whole-batch gradients per tensor.  Rows whose gradient is zero -- the
last N rows of every episode (step T+1 only picks the double-Q arg-max) and the padded tail of a short episode -- and rows whose share of
a tensor is below that budget are invisible there, and those rows sit exactly at the tail of the row space, where a tile kernel that
drops, double-counts or mis-addresses its last partial tile goes wrong.  The checks here make every row count:

* isolated episodes: PER on, importance weights one-hot on episode b.  The loss is linear in the weights, so the step's gradient is
  exactly episode b's (T+1) N agent-net rows and T mixer rows; losing one of them moves it by ~1 / (T N), not 1 / rows.
* per-row forward: every materialised activation of every row (masked rows included), live and target net, against the float64
  trace, bounded relative to the row's own largest magnitude.
* batch size changing on one learner: max_batch, then 1, then a batch one tile smaller, each step against float64 (the optimiser
  must read only the gradient partials this step wrote).

`TileRules` restates the launchers' tile rules (csrc/agent_bwd.cu front_bwd_pick_rm, csrc/tc_bwd.cu, csrc/tc_linear.cu,
csrc/mixer.cu) for an SM count, and `pick_shapes` searches (B, T, N) that put the row / transition counts on the tile edges.
"""
import ctypes as C
import itertools

import numpy as np
import torch

import kink
import qmix_checks as qc
from helpers import rel_err

# Isolated-episode gradients: max |engine - float64| <= GRAD_TOL x max |float64| per tensor.  Measured worst case on the emulator
# (3xTF32 tensor-core layers, FFMA elsewhere) over every shape of tests/test_emu_row_coverage.py: 3.2e-6; on an H100 SXM (132 SMs, default
# power limit) over tests/test_gpu_row_coverage.py: 4.9e-6 (R-MADDPG 4.6e-6).
GRAD_TOL = 2e-5
# Tensors whose gradient is a fixed linear image of ONE sum over the episode's rows of dL/d(output) -- the QMIX mixer's hyper_b2 output
# bias (sum over the T transitions of dL/dQ_tot), the R-MADDPG critic's output biases and output-LayerNorm bias (sum over the T rows of
# dL/dQ) -- lose relative precision when those terms cancel: the fp32 sum keeps an absolute error of order eps sum |term| while the
# result shrinks (measured 3.8e-5 of |sum| on the QMIX bias at S 481, B 1, T 5, and 3.9e-5 on the R-MADDPG critic's at B 1, T 10).  Their
# bound is GRAD_TOL x max|ref| x sum |term| / |sum term|, the cancellation ratio taken from the float64 TD errors; it equals GRAD_TOL
# wherever the terms share a sign.
SUM_OF_OUTPUT_GRADS = ("mixer.hyper_b2.2.bias", "critic.q_outs.0.bias", "critic.q_outs.1.bias", "critic.rnn.rnn.norm.bias")


def _cancellation(terms):
    """sum |t| / |sum t| over a float64 tensor of per-row output gradients (1 where nothing cancels)."""
    t = terms.double().flatten()
    s = float(t.sum().abs())
    a = float(t.abs().sum())
    return a / s if s > 0.0 else (1.0 if a == 0.0 else float("inf"))


# Per-row forward: |engine - float64| <= ROW_TOL x max_j |float64[row, j]| + ROW_ATOL for every row; the recurrent state h (and the gates /
# Q values computed from it) carry the round-off of up to T + 1 cell steps.  Measured worst: 2.6e-6 on the emulator (T <= 24); 1.3e-5 on
# an H100 SXM, q_tgt at T = 151 (the mixer's 16 sms + 1 edge), 5.4e-6 at T <= 64.
ROW_TOL = 2e-5
# M-QMIX: the engine's TD error of a transition within this many fp32 ulps of max(|Q_tot|, |y|) of the float64 one.
TD_ULPS = 16
ROW_ATOL = 1e-6


def td_ulps(in_dim):
    """TD_ULPS up to 32 input columns, in proportion above: the input LayerNorm and fc1 sum over in_dim terms, and one transition's fp32
    TD error carries that round-off.  Measured on the emulator (N 3, B 11), worst over the transitions, in ulps of max(|Q_tot|, |y|): obs 20
    engine 5, fp32 oracle 7; obs 129 engine 30, fp32 oracle 37; obs 320 engine 114, fp32 oracle 68."""
    return TD_ULPS * max(1, _cdiv(in_dim, 32))


# ---- the launchers' tile rules -------------------------------------------------------------------------------------------
def _cdiv(a, b):
    return -(-a // b)


def _round_up(a, b):
    return _cdiv(a, b) * b


def _ld(k):                 # mx_tile.cuh mx_ld: padded leading dimension of a shared-memory tile
    return _round_up(k, 8) + 4


def _front_bwd_smem_floats(in_dim, TM, gru_ext):         # agent_bwd.cu front_bwd_smem
    I64, ld64, ldg, ldi = _round_up(in_dim, 64), _ld(64), _ld(192), _ld(_round_up(in_dim, 64))
    o = TM * ldg + (0 if gru_ext else TM * ld64) + TM * ld64 + (0 if gru_ext else TM * ld64) + 2 * TM * ld64 + 3 * TM * ldi
    return o + 64 * ld64 + 2 * I64 + 4 * 64 + 3 * TM * 2 + 4 * 64


SMEM_BYTES = 227 * 1024


def front_bwd_smem(in_dim, TM, gru_ext=False):
    """k_front_bwd's dynamic shared memory in bytes (front_bwd_launch: front_bwd_smem's floats + 16).  gru_ext: k_gru_wgrad beside it
    (the recurrent QMIX step).  The actor-critic learners run it without (the GRU's h_{t-1} / dgi_n * r tiles here): above 128 columns
    only the 32-row tile fits, 162 KB at 155-192 columns, 186 KB up to 256, 211 KB up to 320."""
    return _front_bwd_smem_floats(in_dim, TM, gru_ext) * 4 + 16


def front_bwd_pick_rm(M, in_dim, sms, gru_ext=False):
    """agent_bwd.cu front_bwd_pick_rm: 16 RM rows per tile, RM in 2..4, minimising waves x (1 + RM) over the heights that fit 227 KB."""
    best, best_cost = 2, 1e30
    for rm in (2, 3, 4):
        if front_bwd_smem(in_dim, 16 * rm, gru_ext) > SMEM_BYTES:
            continue
        cost = _cdiv(_cdiv(M, 16 * rm), sms) * (1.0 + rm)
        if cost < best_cost - 1e-9:
            best, best_cost = rm, cost
    return best


def front_bwd_max_in_dim(gru_ext):
    """agent_bwd.cu mx_front_bwd_max_in_dim: the widest input whose 32-row k_front_bwd tile fits (384 with k_gru_wgrad beside it, as in
    the recurrent QMIX step; 320 without, as in M-QMIX and both MADDPG learners).  The learners refuse wider inputs at creation."""
    w = 0
    while _front_bwd_smem_floats(w + 64, 32, gru_ext) * 4 + 16 <= SMEM_BYTES:
        w += 64
    return w


def mid_warps(N, A, ME=32):
    """mid.cu mid_pick_warps / mx_mid_supported: k_mid's warps per CTA (16 or 8), 0 where its per-warp operand staging does not fit in
    220 KB even with 8 warps (the step then runs k_qhead + the mixer core + k_qhead_bwd)."""
    if not (ME <= 64 and A <= 64 and N <= 32):
        return 0
    AR = 64 if A > 32 else 32
    gP, gM = _round_up(N * ME, 4), _round_up(ME, 4)
    for W in (16, 8):
        total = 2 * AR * 66 + 2 * AR + 4 * 64 + W * 66 + W * A * 64 + W * AR + 2 * W * 64
        total += W * ((3 * N * 64 + 2 * gP + 4 * gM + N * AR + 3) & ~3)
        if total * 4 + 16 <= 220 * 1024:
            return W
    return 0


def mix_wide_state(S, N, ME=32, HY=64):
    """mixer.cu mx_mix_wide_state: the state moves to the tensor-core GEMMs (k_mixw_fwd / k_mixw_wgrad) when a 32-transition mixer tile
    of round_up(S, 64) state columns no longer fits beside the hypernet tiles (N ME columns of them)."""
    S64, H64, P64, M64 = _round_up(S, 64), _round_up(HY, 64), _round_up(N * ME, 64), _round_up(ME, 64)
    TE = 32
    total = TE * _ld(S64) + 3 * TE * _ld(H64) + TE * _ld(P64) + 3 * TE * _ld(M64) + TE * 32 + 8 * TE + 64 * _ld(max(S64, H64))
    return total * 4 + 16 > SMEM_BYTES


def min_wide_state(N, ME=32, HY=64):
    """The narrowest state that takes the wide-state path at N agents."""
    S = 1
    while not mix_wide_state(S, N, ME, HY):
        S += 1
    return S


class TileRules(object):
    """Row tiling of one learner step on `sms` SMs (4 in the emulator, multi_processor_count on a GPU)."""

    def __init__(self, sms):
        self.sms = int(sms)

    def front_bwd_rm(self, M, in_dim, gru_ext):
        return front_bwd_pick_rm(M, in_dim, self.sms, gru_ext)

    def front_bwd_launch(self, M, in_dim, gru_ext=False):
        """One k_front_bwd launch over M rows of width in_dim: (RM, grid, dynamic shared memory in bytes), as a captured graph node
        shows it ("k_front_bwd<RM> grid=(grid, 1, 1) ... smem=bytes")."""
        rm = self.front_bwd_rm(M, in_dim, gru_ext)
        return rm, min(self.sms, _cdiv(M, 16 * rm)), front_bwd_smem(in_dim, 16 * rm, gru_ext)

    def bwd_tc_ctas_per_sm(self, in_dim):
        """k_front_bwd_tc streams its weight operands through one buffer; two CTAs per SM when twice that fits."""
        kp16 = _round_up(in_dim, 16)
        total = 2 * 128 * 64 * 4 + 2 * max(kp16, 64) * 64 * 4
        return 2 if 2 * (total + 2048) <= 227 * 1024 else 1

    def agent_rows(self, M, in_dim, gru_ext=True):
        """The row tiling {kernel: (rows per tile, tiles, grid)} of the backward's row kernels and of the forward (its grid per net).
        gru_ext: the recurrent QMIX step, whose k_gru_wgrad runs beside k_front_bwd; False for M-QMIX (no GRU) and for both actor-critic
        learners, whose k_front_bwd computes the GRU weight gradients itself (R-MADDPG / R-MATD3) or has none (MLP MADDPG / MATD3)."""
        sms = self.sms
        out = {}
        if in_dim > 128:           # FFMA throughout: k_front_fwd<2> (32-row tiles, the two nets share the SMs); k_front_bwd and
            # k_gru_wgrad (recurrent step) on front_bwd_pick_rm's tiles, their heights filtered by round_up(in_dim, 64)-wide smem tiles
            TM = 16 * self.front_bwd_rm(M, in_dim, gru_ext)
            nt = _cdiv(M, TM)
            out["k_front_bwd"] = (TM, nt, min(sms, nt))
            if gru_ext:
                out["k_gru_wgrad"] = out["k_front_bwd"]
            nf = _cdiv(M, 32)
            out["k_front_fwd"] = (32, nf, min(max(sms // 2, 1), nf))
        elif in_dim > 64:          # k_front_bwd_tc (128-row tiles) + k_wgrad_tc (64-row chunks, one persistent CTA per SM)
            nt = _cdiv(M, 128)
            out["k_front_bwd_tc"] = (128, nt, min(self.bwd_tc_ctas_per_sm(in_dim) * sms, nt))
            nc = _cdiv(M, 64)
            out["k_wgrad_tc"] = (64, nc, min(sms, nc))
            out["k_front_fwd_tc_wide"] = (128, nt, min(sms, nt))
        else:                      # k_front_bwd (+ k_gru_wgrad in the recurrent QMIX step: same tile height and grid)
            TM = 16 * self.front_bwd_rm(M, in_dim, gru_ext)
            nt = _cdiv(M, TM)
            out["k_front_bwd"] = (TM, nt, min(sms, nt))
            if gru_ext:
                out["k_gru_wgrad"] = out["k_front_bwd"]
            nf = _cdiv(M, 128)
            out["k_front_fwd_tc"] = (128, nf, min(max(sms // 2, 1), nf))
        return out

    def mixer_rows(self, E):
        """k_mixer / k_mix_hyper_fwd / k_mix_hyper_bwd: 16 RM transitions per tile, RM = 2 above 16 sms transitions."""
        TE = 32 if E > 16 * self.sms else 16
        nt = _cdiv(E, TE)
        return (TE, nt, min(self.sms, nt))

    def head_rows(self, M):
        """R-MADDPG's k_head_bwd: 32-row tiles, grid min(sms, tiles) (critic rows B T, actor rows B (T+1) N)."""
        nt = _cdiv(M, 32)
        return (32, nt, min(self.sms, nt))

    def row_kernel(self, in_dim):
        """The kernel whose tiles define the agent-net row edges of a path."""
        return "k_wgrad_tc" if 64 < in_dim <= 128 else "k_front_bwd"


def _edges(rules, in_dim, N, T, B):
    """Which row / transition edges the shape (B, T, N) hits."""
    r = (T + 1) * N
    M, E = B * r, B * T
    kern = rules.row_kernel(in_dim)
    rows = rules.agent_rows(M, in_dim)
    TM, nt, grid = rows[kern]
    hits = set()
    if nt == 1:
        hits.add("one tile")
    if M % TM == 1:
        hits.add("tail 1")
    if M % TM == TM - 1:
        hits.add("tail TM-1")
    for k, name in ((rules.sms, "tiles = sms"), (rules.sms + 1, "tiles = sms+1"), (2 * rules.sms + 1, "tiles = 2 sms+1")):
        if nt == k:
            hits.add(name)
    if "k_front_bwd_tc" in rows:
        _, nt2, _ = rows["k_front_bwd_tc"]
        if nt2 == rules.bwd_tc_ctas_per_sm(in_dim) * rules.sms + 1:
            hits.add("front_bwd_tc tiles = CTAs+1")
    firsts = [(b * r) // TM for b in range(B)]
    lasts = [((b + 1) * r - 1) // TM for b in range(B)]
    if any(f == l for f, l in zip(firsts, lasts)):
        hits.add("episode inside one tile")
    if any(l - f >= 2 for f, l in zip(firsts, lasts)):
        hits.add("episode spans three tiles")
    if E == 16 * rules.sms:
        hits.add("E = 16 sms")
    if E == 16 * rules.sms + 1:
        hits.add("E = 16 sms+1")
    return hits, dict(M=M, E=E, TM=TM, tiles=nt, grid=grid)


AGENT_TARGETS = ["one tile", "tail 1", "tail TM-1", "tiles = sms", "tiles = sms+1", "tiles = 2 sms+1", "episode inside one tile",
                 "episode spans three tiles"]
MIXER_TARGETS = ["E = 16 sms", "E = 16 sms+1"]


def pick_shapes(rules, in_dim, Ns=(2, 3), Ts=range(2, 17), Bs=range(1, 65), targets=None, max_rows=None):
    """(B, T, N) per edge, the cheapest (fewest isolated rows B M) that hits it.  Some edges cannot occur on a path (the tile-height rule
    minimises waves, so just above `sms` tiles it may take a taller tile): then the nearest tile count that occurs is taken, and the
    returned note says so.  Returns [(targets hit, (B, T, N), layout, note)], one entry per distinct shape."""
    targets = list(targets or AGENT_TARGETS + (["front_bwd_tc tiles = CTAs+1"] if 64 < in_dim <= 128 else []))
    best, notes = {}, {}
    cands = []
    for N, T, B in itertools.product(Ns, Ts, Bs):
        hits, lay = _edges(rules, in_dim, N, T, B)
        if max_rows and lay["M"] > max_rows:
            continue
        cands.append((B * lay["M"], (B, T, N), hits, lay))
    cands.sort(key=lambda c: c[0])
    for tgt in targets:
        for cost, shape, hits, lay in cands:
            if tgt in hits:
                best[tgt] = shape
                break
        else:
            want = {"tiles = sms": rules.sms, "tiles = sms+1": rules.sms + 1, "tiles = 2 sms+1": 2 * rules.sms + 1}.get(tgt)
            if want is None:
                raise AssertionError("no shape in the search space hits %r" % tgt)
            # the nearest count at or above: some CTA still runs one more tile than the others
            near = min((c for c in cands if c[3]["tiles"] >= want), key=lambda c: (c[3]["tiles"] - want, c[0]))
            best[tgt] = near[1]
            notes[tgt] = "%s cannot occur on this path (tile rule); nearest: %d tiles of %d rows" % (tgt, near[3]["tiles"], near[3]["TM"])
    out = {}
    for tgt, shape in best.items():
        out.setdefault(shape, []).append(tgt)
    res = []
    for shape, tg in sorted(out.items()):
        B, T, N = shape
        res.append((tg, shape, _edges(rules, in_dim, N, T, B)[1], "; ".join(notes[t] for t in tg if t in notes)))
    return res


def pick_mixer_shapes(rules, Ns=(2, 3), Ts=range(1, 40), Bs=range(1, 80)):
    """(B, T, N) with E = B T = 16 sms and 16 sms + 1 transitions (the mixer's tile height switch), fewest rows."""
    res = []
    for tgt, E0 in (("E = 16 sms", 16 * rules.sms), ("E = 16 sms+1", 16 * rules.sms + 1)):
        for E in range(E0, E0 + 64):      # E0 may be prime beyond the search space: the next count that occurs, still on the same side
            c = [(B * (T + 1) * N * B, (B, T, N)) for N, T, B in itertools.product(Ns, Ts, Bs) if B * T == E]
            if c:
                break
        assert c, "no shape with %d transitions in the search space" % E0
        B, T, N = min(c)[1]
        note = "" if E == E0 else "%s: %d has no factor pair in the search space; %d transitions instead" % (tgt, E0, E)
        res.append(([tgt], (B, T, N), dict(E=E, tiles=rules.mixer_rows(E)), note))
    return res


MADDPG_TARGETS = ["critic one tile", "critic tail 1", "critic tail 31", "critic tiles = sms+1", "actor tail 1", "actor tail 31"]


FRONT_TARGETS = ["one tile", "tail 1", "tail TM-1", "tiles = sms", "tiles = sms+1"]


def maddpg_front_spaces(rules, B, T, N, obs, cin):
    """R-MADDPG / R-MATD3's k_front_bwd row spaces {space: (rows, rows per tile, tiles)}: the critic's B T rows and the agent-replaced
    copies' N B T rows at the critic's width, the actor's B (T+1) N rows at its own.  No k_gru_wgrad beside it (gru_ext False): the kernel
    computes the GRU weight gradients itself.  Above 128 columns FFMA k_front_bwd on 32-row tiles; at 65-128 the actor's and critic's
    weight gradients run on k_wgrad_tc instead, so only widths outside that band are k_front_bwd edges (the copies' at every width)."""
    out = {}
    for name, M, w in (("critic", B * T, cin), ("copies", N * B * T, cin), ("actor", B * (T + 1) * N, obs)):
        if name == "copies" or not 64 < w <= 128:
            TM = 16 * rules.front_bwd_rm(M, w, False)
            out[name] = (M, TM, _cdiv(M, TM))
    return out


def _front_edges(rules, M, TM, nt):
    """The k_front_bwd edges (FRONT_TARGETS) one row space of M rows in nt tiles of TM hits."""
    return {e for e, ok in (("one tile", nt == 1), ("tail 1", M % TM == 1), ("tail TM-1", M % TM == TM - 1),
                            ("tiles = sms", nt == rules.sms), ("tiles = sms+1", nt == rules.sms + 1)) if ok}


def _head_edges(rules, B, T, N):
    """The k_head_bwd edges (MADDPG_TARGETS) of the critic's B T and the actor's B (T+1) N rows."""
    Mc, Ma = B * T, B * (T + 1) * N
    _, ntc, _ = rules.head_rows(Mc)
    return {t for t, ok in (("critic one tile", ntc == 1), ("critic tail 1", Mc % 32 == 1), ("critic tail 31", Mc % 32 == 31),
                            ("critic tiles = sms+1", ntc == rules.sms + 1), ("actor tail 1", Ma % 32 == 1), ("actor tail 31", Ma % 32 == 31))
            if ok}


def pick_maddpg_shapes(rules, N=3, Ts=range(8, 40), Bs=range(1, 200), obs=None, cin=None):
    """R-MADDPG (B, T) on the edges of k_head_bwd's 32-row tiles, with T >= 8 (the critic's k_gru_bwd2 stores T1 = T steps per
    sequence): critic rows Mc = B T and actor rows Ma = B (T+1) N.  With the widths obs / cin also on the k_front_bwd edges of each
    space of maddpg_front_spaces (labelled "critic front tail 1", ...), and one shape with episodes shorter than 8 (k_gru_bwd's
    short-sequence variant).  An edge no shape hits takes the nearest one that occurs, and the note says so: a tile count the tile rule
    skips (the nearest count above), or an odd tail of a space whose row count is always even (the actor's and the copies' at even N:
    the nearest tail).  Returns [(targets, (B, T, N), layout, note)], fewest rows first."""
    cands = sorted(((B * B * (T + 1) * N, (B, T)) for T in Ts for B in Bs))
    front = lambda B, T: maddpg_front_spaces(rules, B, T, N, obs, cin)
    out, notes = {}, {}

    def place(shape, label, note=None):
        out.setdefault((shape[0], shape[1], N), []).append(label)
        if note:
            notes[label] = note

    for tgt in MADDPG_TARGETS:
        hit = next((bt for _, bt in cands if bt[1] >= 8 and tgt in _head_edges(rules, bt[0], bt[1], N)), None)
        if hit is None and tgt.startswith("actor tail") and N % 2 == 0:
            continue                      # B (T+1) N rows at even N: no odd tail; the k_front_bwd tails of the actor cover its last tile
        assert hit is not None, "no R-MADDPG shape in the search space hits %r" % tgt
        place(hit, tgt)
    if cin is None:
        return [(tg, shape, dict(Mc=shape[0] * shape[1], Ma=shape[0] * (shape[1] + 1) * N), "") for shape, tg in sorted(out.items())]
    short = next((bt for _, bt in cands if bt[1] < 8), None)
    assert short is not None, "no R-MADDPG shape with episodes shorter than 8 in the search space"
    place(short, "T < 8")
    for space in front(1, 8):
        for e in FRONT_TARGETS:
            label = "%s front %s" % (space, e)
            lay = lambda bt: front(bt[0], bt[1])[space]
            hit = next((bt for _, bt in cands if e in _front_edges(rules, *lay(bt))), None)
            if hit is not None:
                place(hit, label)
            elif e.startswith("tail"):
                tail = lambda bt: lay(bt)[0] % lay(bt)[1]
                ok = [bt for _, bt in cands if tail(bt)]
                hit = min(ok, key=(lambda bt: tail(bt)) if e == "tail 1" else (lambda bt: lay(bt)[1] - tail(bt)))
                place(hit, label, "%s cannot occur (an even row count); nearest: a last tile of %d of %d rows at B %d T %d"
                      % (label, tail(hit), lay(hit)[1], hit[0], hit[1]))
            else:
                want = rules.sms + (e == "tiles = sms+1")
                hit = min((bt for _, bt in cands if lay(bt)[2] >= want), key=lambda bt: (lay(bt)[2] - want, bt[0] * bt[0] * (bt[1] + 1)))
                place(hit, label, "%s cannot occur (tile rule); nearest: %d tiles" % (label, lay(hit)[2]))
    return [(tg, shape, dict(Mc=shape[0] * shape[1], Ma=shape[0] * (shape[1] + 1) * N), "; ".join(notes[t] for t in tg if t in notes))
            for shape, tg in sorted(out.items())]


def sample_episodes(B, T, N, TM, grid, every_up_to=16):
    """Every episode up to `every_up_to`; above, the first, the last and the ones that hold a row where a CTA's next tile starts
    (the tile boundaries k grid TM) or the last tile starts."""
    if B <= every_up_to:
        return list(range(B))
    r = (T + 1) * N
    M = B * r
    rows = {0, M - 1, ((M - 1) // TM) * TM}
    k = 1
    while k * grid * TM < M:
        rows.add(k * grid * TM)
        rows.add(k * grid * TM - 1)
        k += 1
    return sorted({row // r for row in rows})


# ---- learners --------------------------------------------------------------------------------------------------------------
def float64_twin(L):
    """The float64 learner holding L's state: same networks, same targets, Adam state fresh (as L's before its first step)."""
    from oracle.qmix import QmixLearner
    from oracle.mqmix import MqmixLearner
    cls = MqmixLearner if isinstance(L, MqmixLearner) else QmixLearner
    L64 = cls(L.cfg, dtype=torch.float64)
    for dst, src in ((L64.agent, L.agent), (L64.mixer, L.mixer), (L64.tgt_agent, L.tgt_agent), (L64.tgt_mixer, L.tgt_mixer)):
        dst.load_state_dict(src.state_dict())
    return L64


def qmix_pair(cfg, B, T, debug=True):
    """(float64 oracle, policy, trainer) with the randomised state of qmix_checks.oracle_and_trainer; trainer max_batch = B."""
    L, args, pol, tr = qc.oracle_and_trainer(cfg, B, T, debug=debug, vdn=cfg.vdn)
    tr.use_step_graph = False
    return float64_twin(L), pol, tr


def mqmix_pair(cfg, B, debug=False):
    """(float64 oracle, policy, trainer) of M-QMIX, or M-VDN when cfg.vdn, with every tensor randomised; trainer max_batch = B."""
    from oracle.mqmix import MqmixLearner
    from oracle.qmix import randomize_all
    import mqmix_checks as mc
    L = MqmixLearner(cfg, seed=3)
    randomize_all(L.agent, 1)
    if not cfg.vdn:
        randomize_all(L.mixer, 2)
    L.sync_targets()
    randomize_all(L.tgt_agent, 3, 0.05)
    if not cfg.vdn:
        randomize_all(L.tgt_mixer, 4, 0.05)
    if cfg.vdn:
        from offpolicy._b200 import capi
        from offpolicy.algorithms.mvdn.algorithm.mVDNPolicy import M_VDNPolicy
        from offpolicy.algorithms.mvdn.mvdn import M_VDN
        args = qc.make_args(cfg, B)
        info = dict(obs_space=[cfg.obs_dim], share_obs_space=[cfg.state_dim], act_space=qc.Discrete(cfg.act_dim), cent_obs_dim=cfg.state_dim,
                    cent_act_dim=cfg.act_dim * cfg.n_agents)
        pol = M_VDNPolicy({"args": args, "device": capi.device()}, info)
        tr = M_VDN(args, cfg.n_agents, {"policy_0": pol}, lambda a: "policy_0", device=capi.device())
        capi.lib().mx_qmix_set_debug(tr.handle, 1 if debug else 0)
    else:
        args, pol, tr = mc.build(cfg, B, debug)
        tr.mixer.load_state_dict(L.mixer.state_dict())
        tr.target_mixer.load_state_dict(L.tgt_mixer.state_dict())
    pol.q_network.load_state_dict(L.agent.state_dict())
    tr.target_q_network.load_state_dict(L.tgt_agent.state_dict())
    return float64_twin(L), pol, tr


def last_episode_full_length(batch):
    """synth_batch(var_len=True) ends every episode at a length in [T/2, T]; make the LAST one run all T steps, so the tail of the row
    space (all but the final N step-(T+1) rows) and of the transition space carries gradient in its isolated run."""
    obs, share, acts, rew, dones, dones_env = batch[:6]
    dones_env = dones_env.copy()
    dones_env[:, -1, 0] = 0.0
    dones_env[-1, -1, 0] = 1.0
    dones = np.repeat(dones_env[None], dones.shape[0], axis=0)
    return (obs, share, acts, rew, dones, dones_env) + tuple(batch[6:])


def maddpg_pair(cfg, B, T):
    """(float64 oracle, policy, trainer) of R-MADDPG / R-MATD3 with every tensor randomised, trainer max_batch = B."""
    import maddpg_checks as mc
    from oracle.maddpg import MaddpgLearner
    from oracle.qmix import randomize_all
    L = MaddpgLearner(cfg, seed=5)
    randomize_all(L.actor, 1)
    randomize_all(L.critic, 2)
    L.sync_targets()
    randomize_all(L.tgt_actor, 3, 0.05)
    randomize_all(L.tgt_critic, 4, 0.05)
    args, pol, tr = mc.build(cfg, B, T)
    L64 = MaddpgLearner(cfg, dtype=torch.float64)
    for ours, ref, ref64 in ((pol.actor, L.actor, L64.actor), (pol.critic, L.critic, L64.critic), (pol.target_actor, L.tgt_actor, L64.tgt_actor),
                             (pol.target_critic, L.tgt_critic, L64.tgt_critic)):
        ours.load_state_dict(ref.state_dict())
        ref64.load_state_dict(ref.state_dict())
    return L64, pol, tr


def maddpg_isolated_episodes(L64, pol, tr, batch, episodes, B, T, tol=None):
    """R-MADDPG / R-MATD3 with one episode isolated per run, from the same state each time (R-MATD3: both critic heads, the target-action
    noise drawn in the trainer's order, the actor only on the updates actor_update_interval selects).  Critic: PER weights one-hot on episode b, so the
    critic gradient is exactly episode b's T rows.  Actor: every agent of every other episode is done from its first step, so the actor
    loss keeps episode b's (T N) rows plus only the first step of the others (the per-agent mask lags the done flag by one step, the first
    step is always live).  Both clipped gradients against the float64 update.  Returns the worst relative error per tensor."""
    import copy
    import maddpg_checks as mc
    from offpolicy._b200 import capi
    from oracle.maddpg import sample_gumbel
    tol = GRAD_TOL if tol is None else tol
    cfg, N = L64.cfg, L64.cfg.n_agents
    ws0 = tr.workspace.clone()
    vec0 = [v.clone() for v in pol.actor_vecs + pol.critic_vecs]
    L0 = copy.deepcopy(L64)
    worst = {}
    for b in episodes:
        tr.workspace.copy_(ws0)
        for v, v0 in zip(pol.actor_vecs + pol.critic_vecs, vec0):
            v.copy_(v0)
        tr.num_updates["policy_0"] = 0
        capi.check(capi.lib().mx_maddpg_set_num_updates(tr._eng["policy_0"].handle, 0))     # the handle's own count picks the actor update
        L = copy.deepcopy(L0)
        w = np.zeros(B, np.float32)
        w[b] = 1.0
        dones = batch[4].copy()
        dones[:, :, [x for x in range(B) if x != b], :] = 1.0
        bt = tuple(batch[:4]) + (dones,) + tuple(batch[5:7]) + (w, np.arange(B))
        # the trainer's draws from torch's CPU generator, in its order: R-MATD3's target-action noise over the T+1 steps, then (when
        # this update trains the actor) the Discrete actor's Gumbel draws over the first T
        update = tr.num_updates["policy_0"] % tr.actor_update_interval == 0
        torch.manual_seed(77 + b)
        tnoise = tr.draw_target_noise(B).numpy() if cfg.td3 else None
        anoise = sample_gumbel((T, N * B, cfg.act_dim)).numpy() if cfg.discrete and update else None
        torch.manual_seed(77 + b)
        info, _, _ = tr.shared_train_policy_on_batch("policy_0", mc.ref_tuple(bt))
        ga, gc = tr.grad_views()
        ref, _ = L.step(bt, tnoise, anoise)
        assert bool(info["update_actor"]) == bool(ref["update_actor"]) == update, (info["update_actor"], ref["update_actor"], update)
        errs = {}
        nets = [("critic", gc, pol.Pc, pol._c_entries, L.critic_grads, ref["critic_grad_norm"])]
        if update:
            nets.append(("actor", ga, pol.Pa, pol._a_entries, L.actor_grads, ref["actor_grad_norm"]))
        for tag, flat, P, entries, grads, gn in nets:
            coef = min(1.0, cfg.max_grad_norm / (float(gn) + 1e-6))
            views = mc.named_views(flat.detach().cpu().double(), entries)
            den = float(flat[P])
            for k, gr in grads.items():
                ref_k = gr.detach().double()
                name = tag + "." + k
                c = 1.0
                if name in SUM_OF_OUTPUT_GRADS:      # critic output head(s): sums over the episode's T rows of the TD errors (one per head)
                    c = max(_cancellation(e[:, b]) for e in L.critic_errs)
                errs[name] = float((views[k] / den * coef - ref_k).abs().max() / (ref_k.abs().max() + 1e-30)) / c
        bad = {k: e for k, e in errs.items() if e > tol}
        assert not bad, ("episode %d of %d isolated: gradients off the float64 oracle (bound %.1e x max|ref|)" % (b, B, tol),
                         sorted(bad.items(), key=lambda kv: -kv[1])[:6])
        for k, e in errs.items():
            worst[k] = max(worst.get(k, 0.0), e)
    tr.workspace.copy_(ws0)
    for v, v0 in zip(pol.actor_vecs + pol.critic_vecs, vec0):
        v.copy_(v0)
    return worst


def kernels_run(lib, stream, fn):
    """Names of the kernels `fn()` launched (mx_profile_begin / mx_profile_end)."""
    lib.mx_profile_begin(stream)
    try:
        fn()
    finally:
        buf = C.create_string_buffer(65536)
        ms = (C.c_float * 2048)()
        n = lib.mx_profile_end(stream, buf, 65536, ms, 2048)
    return buf.value.decode().split(";")[:n]


# Kernels a test means to pin, and what the launcher runs instead where that kernel does not apply: above the overlap row limit the
# GPU step runs serially with the fused k_mixer, and k_mid takes only the widths whose per-warp operands fit its shared memory
# (mid.cu mid_pick_warps / mx_mid_supported) -- otherwise k_qhead + the mixer + k_qhead_bwd run separately.
KERNEL_ALTERNATIVES = {"k_mix_core": ["k_mixer"], "k_mid": ["k_qhead", "k_qhead_bwd"]}


def assert_kernels_ran(names, kernels):
    for k in kernels:
        alt = KERNEL_ALTERNATIVES.get(k)
        assert k in names or (alt and all(a in names for a in alt)), (k, "did not run", names)


# ---- the checks ---------------------------------------------------------------------------------------------------------------
def _grad_errors(gv, L64, ref_scale=1.0, cancel=1.0):
    """{tensor: max |engine - float64 x ref_scale| / max |float64 x ref_scale|} over the learner's parameters (unused ones must be exactly
    zero); for SUM_OF_OUTPUT_GRADS the error is further divided by the cancellation ratio `cancel`."""
    named = dict(("agent." + k, p) for k, p in L64.agent.named_parameters())
    if not L64.cfg.vdn:
        named.update(("mixer." + k, p) for k, p in L64.mixer.named_parameters())
    out = {}
    for k, p in named.items():
        ours = gv[k].detach().cpu().double()
        if p.grad is None:
            assert float(ours.abs().max()) == 0.0, (k, "unused parameter has a gradient")
            continue
        ref = p.grad.detach().double() * ref_scale
        out[k] = float((ours - ref).abs().max() / (ref.abs().max() + 1e-30)) / (cancel if k in SUM_OF_OUTPUT_GRADS else 1.0)
    return out


def isolated_episode_gradients(L64, tr, batch, episodes, B, T, N, mlp=False, tol=GRAD_TOL, ulps=TD_ULPS):
    """For each b in `episodes`: one engine step with importance weights e_b from the same state, its unclipped gradient against the
    float64 oracle's.  ReLU units within round-off of zero may pick the other side (tests/kink.py): a failing comparison is re-run with the
    engine's ReLU masks forced and must then pass.  Returns the worst relative error per tensor."""
    sd0 = tr.state_dict()
    worst = {}
    for b in episodes:
        w = np.zeros(B, np.float32)
        w[b] = 1.0
        bt = tuple(batch[:-2]) + (w, np.arange(B))
        tr.load_state_dict(sd0)
        if mlp:
            import mqmix_checks as mc
            tr.train_policy_on_batch(mc._to_dicts(tuple(batch[:-2]), w), True)
        else:
            tr.train_policy_on_batch(qc.ref_tuple(bt))
        gv = {k: v.detach().cpu().clone() for k, v in tr.grad_views().items()}
        _, _, aux = L64.grads(bt)
        scale, cancel = 1.0, 1.0
        if mlp:
            # one transition: its whole gradient is its TD error times d Q_tot / d theta.  Where Q_tot and the target nearly cancel, the
            # fp32 TD error carries an error of a few ulps of max(|Q_tot|, |y|) -- relative to the error itself, eps |Q| / |err|, into EVERY
            # tensor alike (measured 7.2e-5 on an H100 for one of 2 112 transitions).  The engine's TD error must be within TD_ULPS ulps of
            # that magnitude; the row coverage is then judged against the float64 gradient taken at the engine's TD error
            e_ref = float(aux["err"].detach()[b])
            e_eng = float(tr.ws_view("err")[b])
            mag = max(abs(float(aux["q_tot"].detach().flatten()[b])), abs(float(aux["target"].detach().flatten()[b])))
            assert abs(e_eng - e_ref) <= ulps * 2.0 ** -23 * mag, ("transition %d: TD error %r vs float64 %r (|Q| %.3e)" % (b, e_eng, e_ref, mag))
            scale = e_eng / e_ref if e_ref != 0.0 else 1.0
        else:
            cancel = _cancellation(aux["err"].detach()[:, b])
        errs = _grad_errors(gv, L64, scale, cancel)
        bad = {k: e for k, e in errs.items() if e > tol}
        if bad and getattr(L64.cfg, "relu", True):
            masks = [m.double() for m in kink.engine_masks(tr, B, T, N, mlp=mlp)]
            _, flips, max_pre = kink.redo_with_engine_masks(L64, lambda LL: LL.grads(bt), masks)
            assert flips > 0 and max_pre < kink.KINK_TOL, ("episode %d: gradient mismatch not explained by ReLU kinks" % b, flips, max_pre,
                                                           sorted(bad.items(), key=lambda kv: -kv[1])[:4])
            errs = _grad_errors(gv, L64, scale, cancel)
            bad = {k: e for k, e in errs.items() if e > tol}
        assert not bad, ("episode %d of %d isolated: gradients off the float64 oracle (bound %.1e x max|ref|)" % (b, B, tol),
                         sorted(bad.items(), key=lambda kv: -kv[1])[:6])
        for k, e in errs.items():
            worst[k] = max(worst.get(k, 0.0), e)
    tr.load_state_dict(sd0)
    return worst


def _rows_close(name, ours, want, rtol, atol, bad, worst):
    ours = torch.as_tensor(ours).detach().cpu().double()
    want = torch.as_tensor(want).detach().cpu().double()
    assert ours.shape == want.shape, (name, ours.shape, want.shape)
    err = (ours - want).abs().amax(dim=1)
    scale = want.abs().amax(dim=1)
    ratio = err / (rtol * scale + atol)
    worst[name] = max(worst.get(name, 0.0), float((err / (scale + atol / rtol)).max()))
    if float(ratio.max()) > 1.0:
        r = int(ratio.argmax())
        bad.append("%s: row %d of %d off by %.3e (row max %.3e, bound %.3e); %d row(s) out of bound"
                   % (name, r, ours.shape[0], float(err[r]), float(scale[r]), rtol * float(scale[r]) + atol, int((ratio > 1.0).sum())))


def agent_input(L64, batch):
    """The agent net's input rows as the oracle builds them, (T+1, N B, in_dim) in float64."""
    x = L64.stack_agents(batch[0])
    if L64.cfg.prev_act_inp:
        a = L64.stack_agents(batch[2])
        x = torch.cat((x, torch.cat((torch.zeros(1, a.shape[1], a.shape[2], dtype=a.dtype), a), 0)), -1)
    return x


def per_row_forward(L64, tr, batch, B, T, N, debug, rtol=ROW_TOL, atol=ROW_ATOL):
    """Every materialised activation of all M rows (masked ones included) of the live and the target net against the float64 trace
    of the step the engine just ran; each row bounded relative to its own largest magnitude.  Returns {region: worst err / row max}."""
    from oracle.qmix import agent_trace
    M = B * (T + 1) * N
    A = L64.cfg.act_dim
    x = agent_input(L64, batch)
    bad, worst = [], {}
    rows = lambda v: qc.to_rows(v, N, B)
    # the input LayerNorm's (mean, rstd) per row: above 128 columns k_front_fwd computes them in its own strided loop
    if L64.cfg.feature_norm:
        xr = rows(x)
        mean = xr.mean(1, keepdim=True)
        rstd = 1.0 / torch.sqrt(((xr - mean) ** 2).mean(1, keepdim=True) + 1e-5)
        _rows_close("st0", tr.ws_view("st0")[:M * 2].view(M, 2), torch.cat([mean, rstd], 1), rtol, atol, bad, worst)
    for tag, net in (("live", L64.agent), ("tgt", L64.tgt_agent)):
        trc = agent_trace(net, x)
        _rows_close("gi_" + tag, tr.ws_view("gi_" + tag)[:M * 192].view(M, 192), rows(trc["gi"]), rtol, atol, bad, worst)
        _rows_close("h_" + tag, tr.ws_view("h_" + tag)[:M * 64].view(M, 64), rows(trc["h"]), rtol, atol, bad, worst)
        if debug:
            _rows_close("q_" + tag, tr.ws_view("q_" + tag)[:M * A].view(M, A), rows(trc["q"]), rtol, atol, bad, worst)
        if tag == "live":
            _rows_close("u1", tr.ws_view("u1")[:M * 64].view(M, 64), rows(trc["u1"]), rtol, atol, bad, worst)
            _rows_close("u2", tr.ws_view("u2")[:M * 64].view(M, 64), rows(trc["u2"]), rtol, atol, bad, worst)
            g = tr.ws_view("gates")[:M * 192].view(M, 192)
            want = torch.cat([rows(trc["r"]), rows(trc["z"]), rows(trc["n"])], 1)
            _rows_close("gates", g, want, rtol, atol, bad, worst)
            _rows_close("hn", tr.ws_view("hn")[:M * 64].view(M, 64), rows(trc["hn"]), rtol, atol, bad, worst)
    assert not bad, "\n".join(bad)
    return worst


GREEDY_MARGIN = 1e-3


def per_transition(L64, tr, batch, B, T, N, debug, agent_values=True, rtol=ROW_TOL, atol=ROW_ATOL):
    """One engine step with every importance weight 1 from the trainer's current state (restored afterwards), then every transition
    (b, t) against float64: q_taken / q_next per agent, Q_tot, the target net's Q_tot at t+1 and the TD error, and dq_taken per
    (transition, agent) -- agent N-1 included, the last lane of the mixer's agent loop.  Each transition is bounded relative to its own
    largest value; Q_tot also by how far its agents' round-off reaches it; the TD error relative to the larger of those scales of Q_tot
    and y (it is their difference), and dq_taken (the TD error times d Q_tot / dq)
    against the float64 one taken at the engine's TD error.  In debug mode also the greedy action of every row whose float64 arg-max
    leads the runner-up available action by more than GREEDY_MARGIN.  agent_values=False where k_mid ran: it keeps q_taken, q_next and
    dq_taken in registers and writes only the per-transition values.  Returns {field: worst err / scale}."""
    sd0 = tr.state_dict()
    w = np.ones(B, np.float32)
    bt = tuple(batch[:-2]) + (w, np.arange(B))
    tr.train_policy_on_batch(qc.ref_tuple(bt))
    E = B * T
    ws = lambda name, n: tr.ws_view(name)[:n].detach().cpu().double()
    _, _, aux = L64.loss_terms(bt)
    q_taken = aux["q_taken"]
    numer = (L64._huber(aux["err"]) if L64.cfg.huber else aux["err"] ** 2).sum()
    dq = torch.autograd.grad(numer, q_taken)[0].detach()                       # d (sum of per-transition losses) / dq, (T, B, N)
    per_e = lambda v: v.detach().permute(1, 0, 2).reshape(E, -1)               # (T, B, X) -> [b T + t][X]
    bad, worst = [], {}
    if agent_values:
        _rows_close("q_taken", ws("q_taken", E * N).view(E, N), per_e(q_taken), rtol, atol, bad, worst)
        _rows_close("q_next", ws("q_next", E * N).view(E, N), per_e(aux["tq_next"]), rtol, atol, bad, worst)
    qt, qn, y = per_e(aux["q_tot"]), per_e(aux["q_tot_next"]), per_e(aux["target"])
    # Q_tot sums N agent terms that cancel: the agents' Q values carry their rows' round-off (within rtol of each), which reaches Q_tot
    # as sum_n |dQ_tot/dq_n| |q_n|, not as |Q_tot| (measured on an H100 at N 32, T 12: 9.4e-5 of |Q_tot|).  Each transition's scale is
    # that first-order propagation, or |Q_tot| where it is larger
    share = torch.as_tensor(batch[1], dtype=torch.float64)
    prop = []
    for mixer, q_in, s_in in ((L64.mixer, q_taken.detach(), share[:-1]), (L64.tgt_mixer, aux["tq_next"].detach(), share[1:])):
        q_in = q_in.clone().requires_grad_(True)
        jac = torch.autograd.grad(mixer(q_in, s_in).sum(), q_in)[0]
        prop.append(per_e((jac * q_in).detach().abs()).sum(1, keepdim=True))
    _rows_close("qtot", torch.cat([ws("qtot", E).view(E, 1), prop[0]], 1), torch.cat([qt, prop[0]], 1), rtol, atol, bad, worst)
    _rows_close("qtot_next", torch.cat([ws("qtot_next", E).view(E, 1), prop[1]], 1), torch.cat([qn, prop[1]], 1), rtol, atol, bad, worst)
    live = 1.0 - per_e(aux["bad"])
    err_ref = per_e(aux["err"])
    err_eng = ws("err", E).view(E, 1)
    mag = torch.maximum(torch.maximum(qt.abs(), y.abs()), prop[0] + L64.cfg.gamma * prop[1]) * live
    _rows_close("err", torch.cat([err_eng, mag], 1), torch.cat([err_ref, mag], 1), rtol, atol, bad, worst)
    if agent_values:
        ratio = torch.where(err_ref != 0, err_eng / torch.where(err_ref != 0, err_ref, torch.ones_like(err_ref)), torch.ones_like(err_ref))
        dq_eng = ws("dq_taken", E * N).view(E, N)
        dq_ref = per_e(dq) * ratio
        # the engine keeps gradient numerators: dq_taken is d(sum of losses)/dq up to one constant factor of the loss convention
        s = float((dq_eng * dq_ref).sum() / max(float((dq_ref * dq_ref).sum()), 1e-300))
        assert abs(s - round(s)) < 1e-3 and round(s) != 0, ("dq_taken is not an integer multiple of d(sum of losses)/dq", s)
        _rows_close("dq_taken", dq_eng, dq_ref * round(s), rtol, atol, bad, worst)
    if debug:
        from oracle.qmix import masked_argmax
        M = B * (T + 1) * N
        q_all = aux["q_all"].detach()
        av = L64.stack_agents(batch[6]) if batch[6] is not None else None
        qm = q_all.clone()
        if av is not None:
            qm[av == 0] = -1e300
        top2 = qm.topk(2, dim=-1)[0]
        margin = qc.to_rows((top2[..., 0] - top2[..., 1]).unsqueeze(-1), N, B).flatten()
        want = qc.to_rows(masked_argmax(q_all, av).unsqueeze(-1).double(), N, B).flatten()
        got = tr.ws_view("greedy", torch.int32)[:M].detach().cpu().double()
        sure = margin > GREEDY_MARGIN
        wrong = (got != want) & sure
        assert not bool(wrong.any()), ("greedy action off the float64 arg-max on %d of %d decided rows" % (int(wrong.sum()), int(sure.sum())),
                                       int(wrong.nonzero()[0]))
        worst["greedy decided rows"] = float(sure.sum())
    tr.load_state_dict(sd0)
    assert not bad, "\n".join(bad)
    return worst


# The wide-state GEMMs (3xTF32 on the tensor cores) against float64 on the engine's own operands: max |engine - float64| per block
# within GEMM_TOL x max |float64| of that block (the whole-K fp32 round-off; single-pass TF32 would be ~1e-3).
GEMM_TOL = 2e-6


def wide_state_blocks(cfg):
    """mixer.cu mx_mix_wide_layout: the four stacked state-reading layers [(parameter prefix, first column, rows)] and Cp, the stacked
    columns per net padded to 16.  Block 0 / 1: hyper_w1 / hyper_w2's first (or only) layer, 2: hyper_b2's first layer, 3: hyper_b1."""
    N, ME, HY = cfg.n_agents, cfg.mixer_hidden, cfg.hyper_hidden
    two = cfg.hyper_layers == 2
    spec = [("hyper_w1.0" if two else "hyper_w1", HY if two else N * ME), ("hyper_w2.0" if two else "hyper_w2", HY if two else ME),
            ("hyper_b2.0", HY), ("hyper_b1", ME)]
    out, c = [], 0
    for name, rows in spec:
        out.append((name, c, rows))
        c += _round_up(rows, 4)
    return out, _round_up(c, 16)


def state_gemm_blocks(L64, tr, batch, B, T, tol=GEMM_TOL):
    """After one engine step on `batch` (max_batch = B): every stacked block of the state GEMMs against float64.
    k_mixw_fwd: pre[net][row][c] = share[row] . W_net[c] + b_net[c] over all B (T+1) state rows, live and target net.
    k_mixw_wgrad: gradient partial 0 of each block's weight and bias = d_pre[e]^T share[row(e)] summed over the B T elements, d_pre
    being the engine's own (the hypernet backward's output).  Returns {block / quantity: worst err / max |ref|}."""
    blocks, Cp = wide_state_blocks(L64.cfg)
    R, E = B * (T + 1), B * T
    X = torch.as_tensor(batch[1], dtype=torch.float64).permute(1, 0, 2).reshape(R, -1)        # engine row b (T+1) + t
    Xl = X.view(B, T + 1, -1)[:, :T].reshape(E, -1)                                            # element b T + t reads row b (T+1) + t
    pre = tr.ws_view("hyp_pre").detach().cpu().double()
    assert pre.numel() == 2 * R * Cp, (pre.numel(), 2 * R * Cp)
    pre = pre.view(2, R, Cp)
    d_pre = tr.ws_view("d_pre").detach().cpu().double().view(E, Cp)
    gpart = tr.ws_view("gpart").detach().cpu().double()
    offs = dict((n, o) for n, o, r, c in tr.entries)
    worst, bad = {}, []

    def close(tag, ours, ref):
        e = float((ours - ref).abs().max() / (ref.abs().max() + 1e-300))
        worst[tag] = e
        if e > tol:
            bad.append((tag, e))

    for name, c0, rows in blocks:
        for net, mixer in ((0, L64.mixer), (1, L64.tgt_mixer)):
            sd = mixer.state_dict()
            W, b = sd[name + ".weight"].double(), sd[name + ".bias"].double()
            close("%s fwd net %d" % (name, net), pre[net, :, c0:c0 + rows], X @ W.T + b)
        dp = d_pre[:, c0:c0 + rows]
        W = L64.mixer.state_dict()[name + ".weight"]
        o = offs["mixer." + name + ".weight"]
        close("%s dW" % name, gpart[o:o + W.numel()].view(W.shape), dp.T @ Xl)
        o = offs["mixer." + name + ".bias"]
        close("%s db" % name, gpart[o:o + rows], dp.sum(0))
    assert not bad, bad
    return worst


def batch_size_sequence(L64, pol, tr, cfg, Bs, T, seed=30, tol=GRAD_TOL, param_tol=5e-3):
    """Steps at the batch sizes `Bs` on ONE learner (max_batch = Bs[0]), each in lock-step with the float64 oracle: gradients, loss,
    parameters after Adam, targets after the soft update."""
    from oracle.qmix import synth_batch
    worst = {}
    for s, B in enumerate(Bs):
        w = np.random.RandomState(seed + 100 + s).rand(B).astype(np.float32) * 0.9 + 0.1
        batch = synth_batch(cfg, B, T, seed=seed + s, avail_p=0.8, var_len=True) + (w, np.arange(B))
        info, prio, _ = tr.train_policy_on_batch(qc.ref_tuple(batch))
        gv = {k: v.detach().cpu().clone() for k, v in tr.grad_views().items()}
        L0 = kink.snapshot(L64) if getattr(cfg, "relu", True) else None
        ref, rprio, _ = L64.step(batch)
        # the oracle's step leaves the CLIPPED gradients in .grad; the engine's views are the unclipped ones
        clip = lambda r: min(1.0, cfg.max_grad_norm / (float(r["grad_norm"]) + 1e-6))
        errs = _grad_errors({k: v * clip(ref) for k, v in gv.items()}, L64)
        bad = {k: e for k, e in errs.items() if e > tol}
        if bad and L0 is not None:
            masks = [m.double() for m in kink.engine_masks(tr, B, T, cfg.n_agents, mlp=False)]
            (ref, rprio, _), flips, max_pre = kink.redo_with_engine_masks(L0, lambda LL: LL.step(batch), masks)
            assert flips > 0 and max_pre < kink.KINK_TOL, (s, B, "gradient mismatch not explained by ReLU kinks", flips, max_pre, bad)
            kink.adopt(L64, L0)
            errs = _grad_errors({k: v * clip(ref) for k, v in gv.items()}, L64)
            bad = {k: e for k, e in errs.items() if e > tol}
        assert not bad, ("step %d at B = %d" % (s, B), sorted(bad.items(), key=lambda kv: -kv[1])[:6])
        for k, e in errs.items():
            worst[k] = max(worst.get(k, 0.0), e)
        for k in ("loss", "grad_norm", "Q_tot"):
            assert rel_err(info[k].cpu(), ref[k]) < tol, (s, B, k, float(info[k]), float(ref[k]))
        assert rel_err(np.asarray(prio), rprio) < 1e-4, (s, B, "priorities")
        tr.soft_target_updates()
        L64.soft_update()
        for mod, ref_mod in ((pol.q_network, L64.agent), (tr.mixer, L64.mixer)):
            for k, v in mod.state_dict().items():
                d = float((v.cpu().double() - ref_mod.state_dict()[k]).abs().max())
                assert d <= param_tol * cfg.lr * (s + 1) + 1e-7, (s, B, k, d)
        for mod, ref_mod in ((tr.target_q_network, L64.tgt_agent), (tr.target_mixer, L64.tgt_mixer)):
            for k, v in mod.state_dict().items():
                assert float((v.cpu().double() - ref_mod.state_dict()[k]).abs().max()) <= 1e-6, (s, B, k)
    return worst
