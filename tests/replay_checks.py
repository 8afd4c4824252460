"""Replay parity checks shared by the emulated (CPU) and the real (GPU) test modules.
Bit-exact against the reference goldens and against oracle/replay.py."""
import numpy as np
import torch

from helpers import load_golden, FIELDS
from oracle.mt19937 import LegacyMT19937
from oracle.replay import UniformReplay, PrioritizedReplay

REF_FIELDS = ["obs", "share_obs", "acts", "rewards", "dones", "dones_env", "avail_acts"]


from offpolicy._b200.factory import Discrete, make_rec_buffers as make_buffers, pd as d  # noqa: E402,F401


class Box(object):      # duck-typed gym.spaces.Box for the constructor
    def __init__(self, d):
        self.shape = (d,)


def golden_insert(g, tag, j):
    f = [g["%s.ins%d.%s" % (tag, j, k)] for k in FIELDS]
    return [d(x) for x in f]


def check_uniform_golden():
    g = load_golden("replay_small")
    N, O, A, S, T, E = [int(v) for v in g["meta"]]
    for tag, norm in (("plain", False), ("norm", True)):
        buf = make_buffers(N, O, A, S, T, E, norm=norm)
        for j, n_ep in enumerate((5, 7, 9)):
            r = buf.insert(n_ep, *golden_insert(g, tag, j))
            assert np.array_equal(r, g["%s.idx_range%d" % (tag, j + 1)]), (tag, j)
        assert len(buf) == E
        np.random.seed(123)
        for k in range(3):
            smp = buf.sample(6)
            assert smp[7] is None and smp[8] is None
            idx = np.asarray(buf.policy_buffers["policy_0"].sampled_indices(6))
            assert np.array_equal(idx, g["%s.inds" % tag][k])
            for name, f in zip(FIELDS, smp[:7]):
                got, want = f["policy_0"], g["%s.draw%d.%s" % (tag, k, name)]
                assert got.shape == want.shape and got.dtype == want.dtype, (name, got.shape, want.shape)
                if name == "rew" and norm:
                    assert np.allclose(got, want, rtol=2e-6, atol=2e-6)   # fp32 mean/std summation order differs
                else:
                    assert np.array_equal(got, want), (tag, k, name)


def check_device_rng_stream(seed=321, E=37, B=16, rounds=45, starts=(None,), dims=(2, 5, 3, 6, 3)):
    """Device MT19937 == np.random.seed(seed); np.random.choice(...) across several state regenerations.

    B may be a tuple of batch sizes and `starts` a tuple of stream positions; every (B, start) pair restarts the stream.  A start of
    None seeds the device generator; an integer p draws a p-word prefix from NumPy's stream (one word per uint32 value, past the first
    twist) and hands that state to the device, so the first device draw begins at word p.  k_draw's uniform fast path reads the 256 words
    from the position on, so p + 256 = 623, 624, 625 sit on either side of its limit."""
    N, O, A, S, T = dims
    Bs = (B,) if np.isscalar(B) else tuple(B)
    mb = max(max(Bs), min(E, 1024))
    buf = make_buffers(N, O, A, S, T, E, rng="device", max_batch=mb)
    rs = np.random.RandomState(0)
    ep = lambda n: [d(rs.randn(T + 1, n, N, O)), d(rs.randn(T + 1, n, N, S)), d(np.eye(A)[rs.randint(0, A, (T, n, N))]),
                    d(rs.randn(T, n, N, 1)), d(np.zeros((T, n, N, 1))), d(np.zeros((T, n, 1))), d(np.ones((T + 1, n, N, A)))]
    left = E
    while left > 0:
        n = min(mb, left)
        buf.insert(n, *ep(n))
        left -= n
    assert len(buf) == E
    pb = buf.policy_buffers["policy_0"]
    for b in Bs:
        for p in starts:
            np.random.seed(seed)
            if p is None:
                buf.seed_device_rng(seed)
            else:
                np.random.randint(0, 2 ** 32, size=p, dtype=np.uint32)
                assert np.random.get_state()[2] == p
                buf.adopt_numpy_rng()
            for k in range(rounds):      # 45 x ~20 words > 624: crosses the twist at least once
                buf.sample(b)
                got = np.asarray(pb.sampled_indices(b))
                want = np.random.choice(E, b)
                assert np.array_equal(got, want), (b, p, k)
    # n == 1 consumes nothing; adopt / export of NumPy's own state round-trips
    one = make_buffers(N, O, A, S, T, 4, rng="device", max_batch=4)
    one.insert(1, *ep(1))
    np.random.seed(5)
    np.random.random(size=11)
    one.adopt_numpy_rng()
    one.sample(3)
    assert np.array_equal(np.asarray(one.policy_buffers["policy_0"].sampled_indices(3)), np.zeros(3, np.int64))
    one.policy_buffers["policy_0"].export_rng_to_numpy()
    a = np.random.random(size=4)
    np.random.seed(5)
    np.random.random(size=11)
    assert np.array_equal(a, np.random.random(size=4))


def check_per_golden():
    g = load_golden("replay_small")
    N, O, A, S, T, E = [int(v) for v in g["meta"]]
    buf = make_buffers(N, O, A, S, T, E, per_alpha=0.6)
    z = lambda *s: np.zeros(s, np.float32)
    dummy = [d(z(T + 1, 6, N, O)), d(z(T + 1, 6, N, S)), d(z(T, 6, N, A)), d(z(T, 6, N, 1)), d(z(T, 6, N, 1)), d(z(T, 6, 1)),
             d(z(T + 1, 6, N, A))]
    buf.insert(6, *dummy)
    buf.insert(6, *dummy)
    pb = buf.policy_buffers["policy_0"]
    # leaves handed over pre-powered in fp64 (NumPy's float32 pow is platform SIMD code; exactness of the
    # *tree arithmetic and indices* is what is pinned here; the on-device pow path is checked to 1 ulp below)
    leaves0 = g["per.prio0"] ** 0.6
    pb.update_priorities(np.arange(12), leaves=leaves0.astype(np.float64))
    s, m = pb.tree_values()
    assert np.array_equal(s, g["per.leaves0"]) and np.array_equal(m, g["per.minleaves0"])
    np.random.seed(77)
    smp = buf.sample(5, 0.4, "policy_0")
    assert np.array_equal(np.asarray(smp[8]), g["per.idx0"])
    assert np.allclose(np.asarray(smp[7]), g["per.w0"], rtol=1e-13, atol=0)
    # duplicate indices: last write wins
    pb.update_priorities(g["per.upd_idx"], leaves=(g["per.upd_prio"] ** 0.6).astype(np.float64))
    s, m = pb.tree_values()
    assert np.array_equal(s, g["per.leaves1"]) and np.array_equal(m, g["per.minleaves1"])
    smp = buf.sample(8, 0.7, "policy_0")
    assert np.array_equal(np.asarray(smp[8]), g["per.idx1"])
    assert np.allclose(np.asarray(smp[7]), g["per.w1"], rtol=1e-13, atol=0)
    # on-device fp32 pow path (what the trainer's priorities take): <= 1 ulp of NumPy's float32 power
    buf2 = make_buffers(N, O, A, S, T, E, per_alpha=0.6)
    buf2.insert(6, *dummy)
    buf2.insert(6, *dummy)
    buf2.update_priorities(np.arange(12), g["per.prio0"], "policy_0")
    s2, _ = buf2.policy_buffers["policy_0"].tree_values()
    cap = len(s2) // 2
    got = s2[cap:cap + 12].astype(np.float32)
    want = (g["per.prio0"] ** 0.6).astype(np.float32)
    assert np.all(np.abs(got.view(np.int32) - want.view(np.int32)) <= 1)


def check_per_vs_oracle_random(seed=5, E=50, B=8, steps=6):
    """Insert priming (intent of the reference's broken loop), sampling, write-back with duplicates, vs oracle."""
    N, O, A, S, T = 2, 4, 3, 5, 3
    rs = np.random.RandomState(seed)
    buf = make_buffers(N, O, A, S, T, E, per_alpha=0.6, rng="device", max_batch=16)
    ora = PrioritizedReplay(0.6, E, T, N, O, S, A, rng=LegacyMT19937(99), prime_leaves=True)
    pb = buf.policy_buffers["policy_0"]
    buf.seed_device_rng(99)

    def ep(n):
        f = [rs.randn(T + 1, n, N, O), np.repeat(rs.randn(T + 1, n, 1, S), N, 2), np.eye(A)[rs.randint(0, A, (T, n, N))],
             rs.randn(T, n, N, 1), np.zeros((T, n, N, 1)), np.zeros((T, n, 1)), np.ones((T + 1, n, N, A))]
        return [x.astype(np.float32) for x in f]

    for n in (16, 16, 9):
        e = ep(n)
        buf.insert(n, *[d(x) for x in e])
        ora.insert(n, *e)
    for k in range(steps):
        smp = buf.sample(B, 0.5, "policy_0")
        out, inds = ora.sample(B, 0.5)
        assert np.array_equal(np.asarray(smp[8]), inds), k
        assert np.allclose(np.asarray(smp[7]), out[7], rtol=1e-13)
        for name, ref in zip(REF_FIELDS, out[:7]):
            assert np.array_equal(smp[REF_FIELDS.index(name)]["policy_0"], ref), name
        pr = (rs.rand(B) * 2 + 0.01).astype(np.float32)
        leaves = (pr ** 0.6).astype(np.float64)
        pb.update_priorities(inds, leaves=leaves)
        ora.sum_tree.set(inds, leaves)
        ora.min_tree.set(inds, leaves)
        if k == 2:       # wrap the ring, which also re-primes overwritten slots with max_priority ** alpha
            e = ep(7)
            buf.insert(7, *[d(x) for x in e])
            ora.insert(7, *e)
        s, m = pb.tree_values()
        assert np.array_equal(s, ora.sum_tree.v) and np.array_equal(m, ora.min_tree.v), k


def check_uniform_vs_oracle_shapes(shape, seed=0):
    """Random insert/sample sequence at a given (N,O,A,S,T,E,B) vs oracle, including ring wrap and avail=None."""
    N, O, A, S, T, E, B, use_avail = shape
    rs = np.random.RandomState(seed)
    buf = make_buffers(N, O, A, S, T, E, rng="numpy", max_batch=max(B, 8), avail=use_avail)
    ora = UniformReplay(E, T, N, O, S, A, use_avail=use_avail, rng=None)

    def ep(n):
        f = [rs.randn(T + 1, n, N, O), np.repeat(rs.randn(T + 1, n, 1, S), N, 2), np.eye(A)[rs.randint(0, A, (T, n, N))],
             rs.randn(T, n, N, 1), (rs.rand(T, n, N, 1) < 0.3) * 1.0, (rs.rand(T, n, 1) < 0.3) * 1.0]
        f.append((rs.rand(T + 1, n, N, A) < 0.5) * 1.0 if use_avail else None)
        return [x.astype(np.float32) if x is not None else None for x in f]

    total = 0
    while total < 2 * E + 3:
        n = int(rs.randint(1, min(8, E + 1)))
        e = ep(n)
        r1 = buf.insert(n, *[d(x) for x in e])
        r2 = ora.insert(n, *[x for x in e])
        assert np.array_equal(r1, r2)
        total += n
        assert len(buf) == len(ora)
        assert buf.policy_buffers["policy_0"].current_i == ora.store.cursor
        st = np.random.get_state()
        smp = buf.sample(B)
        np.random.set_state(st)
        out, inds = ora.sample(B)
        for i, name in enumerate(REF_FIELDS):
            got = smp[i]["policy_0"]
            if out[i] is None:
                assert got is None
            else:
                assert np.array_equal(got, out[i]), name


def check_reward_norm_running_stats(seed=3, E=7, B=5, inserts=40):
    """Running reward statistics (updated at insert, evicted episodes subtracted) vs the oracle's full rescan
    (rec_buffer.py:209-223) over many ring wraps: single-episode inserts like the RNN runners, a few multi-episode ones, episodes
    that terminate early (masked steps), sampled rewards compared after every insert."""
    N, O, A, S, T = 3, 4, 3, 5, 6
    rs = np.random.RandomState(seed)
    buf = make_buffers(N, O, A, S, T, E, norm=True, rng="numpy", max_batch=max(B, 8))
    ora = UniformReplay(E, T, N, O, S, A, reward_norm=True, rng=None)

    def ep(n):
        de = np.maximum.accumulate((rs.rand(T, n, 1) < 0.15).astype(np.float32), axis=0)
        f = [rs.randn(T + 1, n, N, O), np.repeat(rs.randn(T + 1, n, 1, S), N, 2), np.eye(A)[rs.randint(0, A, (T, n, N))],
             np.repeat(3.0 + 2.0 * rs.randn(T, n, 1, 1), N, 2), np.repeat(de[:, :, None], N, 2), de, np.ones((T + 1, n, N, A))]
        return [x.astype(np.float32) for x in f]

    for k in range(inserts):
        n = 1 if k % 7 else int(rs.randint(2, 5))
        e = ep(n)
        buf.insert(n, *[d(x) for x in e])
        ora.insert(n, *e)
        st = np.random.get_state()
        smp = buf.sample(B)
        np.random.set_state(st)
        out, inds = ora.sample(B)
        got, want = smp[3]["policy_0"], out[3]
        assert np.abs(got - want).max() <= 2e-5 * max(1.0, np.abs(want).max()), (k, np.abs(got - want).max())


# ---- training-scale replays ----------------------------------------------------------------------------------------------------
STATE_MEAN_AT = 24       # byte offset of MxReplayState.reward_mean (csrc/mx_internal.h); reward_std follows it
TMA_GATHER_LIMIT = 96 << 20   # mx_launch_gather_tma: batches of more bytes than this take the vectorised k_gather


def episode_bytes(pb):
    """Bytes one episode occupies in the store and in the batch region (every padded field, mx_replay_layout_query)."""
    L = pb.L
    return 4 * sum(int(getattr(L, f)) for f in ("ep_obs", "ep_share", "ep_acts", "ep_avail", "ep_rew", "ep_dones", "ep_dones_env",
                                                 "ep_actidx"))


def smac_episodes(g, n, N, O, A, S, T):
    """n episodes of a SMAC-like shape: buffer fields (share_obs once per step) and oracle fields (share_obs with an agent axis of 1),
    one-hot actions, avail masks, a team reward, episodes that end before T."""
    f32 = np.float32
    end = g.integers(T // 2, T + 3, n)
    de = (np.arange(T)[:, None] >= end[None, :]).astype(f32)[:, :, None]                        # (T, n, 1)
    obs = g.standard_normal((T + 1, n, N, O), dtype=f32)
    share = g.standard_normal((T + 1, n, S), dtype=f32)
    acts = np.eye(A, dtype=f32)[g.integers(0, A, (T, n, N))]
    rew = np.repeat((0.4 + g.standard_normal((T, n, 1, 1), dtype=f32)).astype(f32), N, 2)
    dones = np.repeat(de[:, :, None, :], N, 2)
    avail = (g.random((T + 1, n, N, A), dtype=f32) < 0.7).astype(f32)
    buf_f = [obs, share, acts, rew, dones, de, avail]
    return buf_f, [obs, share[:, :, None, :], acts, rew, dones, de, avail]


def fill_smac_replay(shape, E, max_batch, chunk=8, seed=0):
    """Uniform replay (avail masks, reward normalisation) and the oracle, filled with E + E // 4 + 1 episodes: the ring wraps once."""
    N, O, A, S, T = shape
    buf = make_buffers(N, O, A, S, T, E, norm=True, rng="numpy", max_batch=max_batch)
    ora = UniformReplay(E, T, N, O, S, A, reward_norm=True, rng=None)
    g = np.random.default_rng(seed)
    left = E + E // 4 + 1
    while left > 0:
        n = min(chunk, left)
        bf, of = smac_episodes(g, n, N, O, A, S, T)
        assert np.array_equal(buf.insert(n, *[d(x) for x in bf]), ora.insert(n, *of))
        left -= n
    assert len(buf) == E and buf.policy_buffers["policy_0"].current_i == ora.store.cursor
    return buf, ora


def check_sample_vs_oracle(buf, ora, B, seed):
    """One host-drawn sample of B episodes against the oracle's gather: every field byte for byte (normalised rewards to 2e-6, the
    oracle's statistics being fp32 sums), and the action-index field the learners read (first maximum of the one-hot action), which is
    the last field of every episode in the batch region.  Returns the sampled rewards."""
    pb = buf.policy_buffers["policy_0"]
    np.random.seed(seed)
    smp = buf.sample(B)
    np.random.seed(seed)
    out, inds = ora.sample(B)
    assert np.array_equal(np.asarray(pb.sampled_indices(B)), inds)
    for i, name in enumerate(REF_FIELDS):
        got = smp[i]["policy_0"]
        assert got.shape == out[i].shape and got.dtype == out[i].dtype, (name, got.shape, out[i].shape)
        if name == "rewards":
            assert np.allclose(got, out[i], rtol=2e-6, atol=2e-6), np.abs(got - out[i]).max()
        else:
            assert np.array_equal(got, out[i]), name
    T, N = ora.store.T, ora.store.N
    ai = pb._view(pb.L.off_b_actidx, B * int(pb.L.ep_actidx), torch.int32).view(B, -1)[:, :T * N].cpu().numpy()
    assert np.array_equal(ai.reshape(B, T, N), np.argmax(out[2], -1).transpose(2, 1, 0))
    return smp[3]["policy_0"]


def device_reward_stats(pb):
    """(mean, std) the gather normalises with: the fp32 values the insert keeps in the replay's state block."""
    at = int(pb.L.off_state) + STATE_MEAN_AT
    m, s = pb.blob[at:at + 16].view(torch.float64).cpu().numpy()
    return float(m), float(s)


def rescan_reward_stats(store):
    """float64 mean / population std of every unmasked filled reward (rec_buffer.py:209-220), two passes."""
    F = store.filled
    de = store.dones_env[:, :F, 0]
    keep = np.concatenate([np.ones_like(de[:1], bool), de[:-1] != 1.0], 0)                   # step t counts unless done at t - 1
    r = store.rewards[:, :F, :, 0]
    r = r[np.broadcast_to(keep[:, :, None], r.shape)].astype(np.float64)
    m = r.mean()
    return m, float(np.sqrt(np.mean((r - m) ** 2)))


def f32_ulps(got, want):
    """|got - want| in units of the fp32 spacing at want."""
    return abs(got - want) / float(np.spacing(np.float32(abs(want))))


def check_reward_stats_long_run(loc, scale, E=5000, inserts=20000, every=500, seed=12, T=25, N=3, B=32, vs_oracle=True):
    """Running reward statistics over a long run of single-episode inserts (MPE-like: T 25, 3 agents, some episodes end early, the
    ring wraps inserts // E times).  Every `every` inserts: the device mean and std are within 4 fp32 ulps of a float64 rescan of
    every filled reward, and a sample's rewards are (r - mean) / std in fp32 with exactly those statistics.  vs_oracle: the statistics
    are also within 2e-5 of the oracle's and the sampled rewards within 2e-5 of its normalised rewards.  The oracle sums in fp32 like
    the reference, so that holds only while its mean's error is small against the spread: at mean 1e3, std 1e-2 one ulp of the mean
    is 6e-3 std, and the float64 rescan is the yardstick.  Returns the worst (mean, std) error in ulps."""
    O, A, S = 2, 2, 3
    rs = np.random.RandomState(seed)
    buf = make_buffers(N, O, A, S, T, E, norm=True, rng="numpy", max_batch=B)
    ora = UniformReplay(E, T, N, O, S, A, reward_norm=True, rng=None)
    pb = buf.policy_buffers["policy_0"]
    f32 = np.float32
    obs, share = np.zeros((T + 1, 1, N, O), f32), np.zeros((T + 1, 1, S), f32)
    acts, avail = np.zeros((T, 1, N, A), f32), np.ones((T + 1, 1, N, A), f32)
    worst = [0.0, 0.0]
    for k in range(inserts):
        de = (np.arange(T) >= rs.randint(T // 2, 2 * T)).astype(f32)[:, None, None]          # half the episodes end early
        rew = (loc + scale * rs.randn(T, 1, N, 1)).astype(f32)
        dones = np.repeat(de[:, :, None, :], N, 2)
        buf.insert(1, d(obs), d(share), d(acts), d(rew), d(dones), d(de), d(avail))
        ora.insert(1, obs, share[:, :, None, :], acts, rew, dones, de, avail)
        if (k + 1) % every:
            continue
        m64, s64 = rescan_reward_stats(ora.store)
        dm, ds = device_reward_stats(pb)
        um, us = f32_ulps(dm, m64), f32_ulps(ds, s64)
        worst = [max(worst[0], um), max(worst[1], us)]
        assert um <= 4 and us <= 4, (k, dm, m64, um, ds, s64, us)
        if vs_oracle:
            om, osd = ora.store.reward_stats()
            assert abs(dm - om) <= 2e-5 * max(1.0, abs(om)) and abs(ds - osd) <= 2e-5 * osd, (k, dm, om, ds, osd)
        st = np.random.get_state()
        smp = buf.sample(B)
        np.random.set_state(st)
        out, inds = ora.sample(B)
        got = smp[3]["policy_0"]
        raw = ora.store.rewards[:, inds].transpose(2, 0, 1, 3)
        assert np.array_equal(got, (raw - f32(dm)) / f32(ds)), k
        if vs_oracle:
            assert np.abs(got - out[3]).max() <= 2e-5 * max(1.0, np.abs(out[3]).max()), (k, np.abs(got - out[3]).max())
    return worst


# ---- transition PER at the MLP runners' sizes -----------------------------------------------------------------------------------
def transition_replay(specs, E, rng, max_batch=1024):
    """PrioritizedMlpReplayBuffer (alpha 0.6, no avail masks) with one policy per (n_agents, obs, share_obs, actions) of `specs`."""
    from offpolicy.utils.mlp_buffer import PrioritizedMlpReplayBuffer
    info = {"policy_%d" % i: dict(obs_space=[o], share_obs_space=[s], act_space=Discrete(a)) for i, (n, o, s, a) in enumerate(specs)}
    agents = {"policy_%d" % i: list(range(n)) for i, (n, o, s, a) in enumerate(specs)}
    return PrioritizedMlpReplayBuffer(0.6, info, agents, E, True, False, rng=rng, max_batch=max_batch)


def transitions(rs, n, spec):
    """n random transitions of one policy: the buffer's insert arguments and the oracle's (an episode of length 1)."""
    N, O, S, A = spec
    f = lambda *s: rs.randn(*s).astype(np.float32)
    obs, nobs, share, nshare, rew = f(n, N, O), f(n, N, O), f(n, S), f(n, S), f(n, N, 1)
    acts = np.eye(A, dtype=np.float32)[rs.randint(0, A, (n, N))]
    dones, de, valid = np.zeros((n, N, 1), np.float32), np.zeros((n, 1), np.float32), np.ones((n, N, 1), np.float32)
    mine = [obs, share, acts, rew, nobs, nshare, dones, de, valid]
    theirs = [np.stack([obs, nobs]), np.stack([share, nshare])[:, :, None], acts[None], rew[None], dones[None], de.reshape(1, n, 1)]
    return mine, theirs


def _last_writes(idx):
    """Unique indices of a write-back and the position of each one's last occurrence (last write wins)."""
    u, first_rev = np.unique(idx[::-1], return_index=True)
    return u, len(idx) - 1 - first_rev


def check_per_transitions_vs_oracle(E, spec=(1, 1, 1, 1), rounds=100, B=1000, rng="device", seed=3, gap=2500):
    """PrioritizedMlpReplayBuffer at the MLP runners' sizes against oracle/replay.py, bit for bit.

    Fill to E - gap with inserts of max_batch (1 024); run `rounds` rounds of sample(B, beta) with beta annealed 0.4 -> 1.0 and a
    write-back of B pre-powered fp64 leaves to the drawn indices (some rounds plant hot leaves, so later draws repeat indices and the
    write-backs hold duplicates); halfway, insert gap + 1 600 transitions, which wraps the ring and re-primes written-back leaves
    with max_priority ** alpha in a call that crosses the end.  Every round: indices bit-equal, IS weights within rtol 1e-13, the
    sampled rows equal the oracle's, the whole sum and min trees bit-equal.  Every few rounds one word (rng "device": a uniform draw
    of one index; rng "numpy": a uint32 from NumPy's stream, as the environment would) shifts the stream's parity, so PER draws of
    2 B words hold a half-drawn double across the generator's twists.  Last, one write-back through the trainer's fp32 priority path
    (the device powers them): leaves within 1 ulp of NumPy's float32 power.  Returns (worst weight error, largest duplicate count)."""
    from oracle.replay import PrioritizedReplay
    N, O, S, A = spec
    rs = np.random.RandomState(seed)
    buf = transition_replay([spec], E, "numpy" if rng == "numpy" else "device")
    host = np.random.RandomState(seed)
    if rng == "device":
        buf.seed_device_rng(seed)
    ora = PrioritizedReplay(0.6, E, 1, N, O, S, A, use_avail=False, rng=host if rng == "device" else None, prime_leaves=True)
    pb = buf.policy_buffers["policy_0"]

    def put(total):
        while total > 0:
            n = min(1024, total)
            mine, theirs = transitions(rs, n, spec)
            assert np.array_equal(buf.insert(n, *[d(x) for x in mine], None, None), ora.insert(n, *theirs))
            total -= n

    def draw(beta):
        st = np.random.get_state()
        smp = buf.sample(B, beta)
        idx, w = np.asarray(smp[12]), np.asarray(smp[11])
        if rng == "numpy":
            after = np.random.get_state()
            np.random.set_state(st)
        out, inds = ora.sample(B, beta)
        if rng == "numpy":       # the exported stream continues where NumPy's own draw left it
            now = np.random.get_state()
            assert np.array_equal(now[1], after[1]) and now[2] == after[2]
        assert np.array_equal(idx, inds)
        assert np.array_equal(smp[0]["policy_0"], out[0][:, 0]) and np.array_equal(smp[4]["policy_0"], out[0][:, 1])
        err = float(np.max(np.abs(w - out[7]) / out[7]))
        assert err <= 1e-13, err
        return idx, err

    put(E - gap)
    cap = ora.sum_tree.cap
    worst, dup = 0.0, 1
    for k in range(rounds):
        if k == rounds // 2:
            put(gap + 1600)
            assert len(buf) == E and pb.current_i == ora.store.cursor == 1600
        if k % 7 == 3:
            if rng == "device":
                pb.rep.sample_device_uniform(1)
                assert np.array_equal(np.asarray(pb.rep.sampled_indices(1)), host.randint(0, len(ora), 1))
            else:
                np.random.randint(0, 2 ** 32, size=1, dtype=np.uint32)
        idx, err = draw(0.4 + 0.6 * k / max(rounds - 1, 1))
        worst = max(worst, err)
        dup = max(dup, int(np.unique(idx, return_counts=True)[1].max()))
        leaves = (rs.rand(B) * 2 + 0.01) ** 0.6
        if k % 5 == 0:
            leaves[rs.randint(0, B, 3)] = 0.1 * E        # each holds several % of the mass: drawn tens of times next round
        pb.rep.update_priorities(idx, leaves=leaves)
        ora.sum_tree.set(idx, leaves)
        ora.min_tree.set(idx, leaves)
        s, m = pb.rep.tree_values()
        assert np.array_equal(s, ora.sum_tree.v) and np.array_equal(m, ora.min_tree.v), k
    assert dup > 1
    # the trainer's path: fp32 priorities, powered on the device
    idx, err = draw(1.0)
    prio = (rs.rand(B) * 2 + 0.01).astype(np.float32)
    prio[rs.randint(0, B, 3)] = 40.0
    buf.update_priorities(idx, prio)
    s, m = pb.rep.tree_values()
    u, last = _last_writes(idx)
    got = s[cap + u].astype(np.float32)
    assert np.array_equal(got.astype(np.float64), s[cap + u])
    want = prio[last] ** 0.6
    assert want.dtype == np.float32 and np.all(np.abs(got.view(np.int32) - want.view(np.int32)) <= 1)
    ora.sum_tree.set(u, s[cap + u])
    ora.min_tree.set(u, s[cap + u])
    ora.max_priority = max(ora.max_priority, float(prio.max()))
    assert np.array_equal(s, ora.sum_tree.v) and np.array_equal(m, ora.min_tree.v)
    idx, err = draw(1.0)
    return max(worst, err), dup


def check_per_transition_policies(E, rounds=8, B=1000, seed=4):
    """Several policies (simple_speaker_listener: speaker obs 3 / 3 actions, listener obs 11 / 5 actions, shared obs 14): sample(B, beta,
    "policy_1") draws from policy_1's tree (bit-equal to the oracle) and the drawn indices select the rows of BOTH stores;
    update_priorities(..., "policy_1") changes policy_1's tree only (fp32 path: leaves within 1 ulp of NumPy's float32 power, trees
    bit-equal to the oracle given those leaves) while policy_0's tree stays bit-unchanged."""
    from oracle.replay import PrioritizedReplay
    specs = [(1, 3, 14, 3), (1, 11, 14, 5)]
    rs = np.random.RandomState(seed)
    buf = transition_replay(specs, E, "device")
    buf.seed_device_rng(seed)
    ora = PrioritizedReplay(0.6, E, 1, *specs[1], use_avail=False, rng=np.random.RandomState(seed), prime_leaves=True)
    host = [np.zeros((E, n, o), np.float32) for n, o, s, a in specs]
    left = E - 7
    while left > 0:
        n = min(1024, left)
        fields = [transitions(rs, n, sp) for sp in specs]
        slots = buf.insert(n, *[{"policy_%d" % p: fields[p][0][i] for p in range(2)} for i in range(9)], None, None)
        assert np.array_equal(slots, ora.insert(n, *fields[1][1]))
        for p in range(2):
            host[p][slots] = fields[p][0][0]
        left -= n
    b0, b1 = buf.policy_buffers["policy_0"].rep, buf.policy_buffers["policy_1"].rep
    tree0 = b0.tree_values()
    cap = ora.sum_tree.cap
    for k in range(rounds):
        beta = 0.4 + 0.6 * k / max(rounds - 1, 1)
        smp = buf.sample(B, beta, "policy_1")
        idx = np.asarray(smp[12])
        out, inds = ora.sample(B, beta)
        assert np.array_equal(idx, inds), k
        assert np.allclose(np.asarray(smp[11]), out[7], rtol=1e-13, atol=0)
        for p in range(2):
            assert np.array_equal(smp[0]["policy_%d" % p], host[p][idx].transpose(1, 0, 2)), (k, p)
        prio = (rs.rand(B) * 2 + 0.01).astype(np.float32)
        prio[rs.randint(0, B, 2)] = 0.05 * E
        buf.update_priorities(idx, prio, "policy_1")
        s, m = b1.tree_values()
        u, last = _last_writes(idx)
        got = s[cap + u].astype(np.float32)
        assert np.all(np.abs(got.view(np.int32) - (prio[last] ** 0.6).view(np.int32)) <= 1)
        ora.sum_tree.set(u, s[cap + u])
        ora.min_tree.set(u, s[cap + u])
        assert np.array_equal(s, ora.sum_tree.v) and np.array_equal(m, ora.min_tree.v), k
        t0 = b0.tree_values()
        assert np.array_equal(t0[0], tree0[0]) and np.array_equal(t0[1], tree0[1]), k
