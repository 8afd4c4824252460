"""Data-parallel R-MATD3 and MADDPG / MATD3 on the H100: two ranks in one process on one device, driven through the update's phases with
their symmetric blocks in device memory (every rank publishes before any rank reduces, so no kernel waits on a peer).  Each update must
equal one learner stepping the full batch: train_info within 1e-5, the summed gradient buffers within the row-coverage checks'
reorder tolerance, the parameters within the Adam-step bound, the two replicas bit-identical and each rank's PER priorities the single
learner's for its rows.  A two-process variant over real peer memory needs two GPUs."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

import maddpg_dp_checks as dc
from helpers import load_golden, rel_err

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
GRAD_TOL = 2e-5          # row_coverage_checks.GRAD_TOL: the same sums in another order


def shard_batch(batch, r, Bl):
    """Rank r's rows of a batch tuple ({policy: array} entries, then the PER weights and the sample indices)."""
    cut = lambda x: {k: dc.shard(v, r, Bl) for k, v in x.items()} if isinstance(x, dict) else dc.shard(x, r, Bl)
    return tuple(cut(x) for x in batch[:-1]) + (None if batch[-1] is None else np.arange(Bl),)


def dp_vs_single(make, batch_fn, B, steps, world=2):
    """make(B, world) -> ({policy: policy}, trainer) from the current torch seed; batch_fn(s) -> the full batch of update round s."""
    from offpolicy._b200 import capi
    torch.manual_seed(7)
    pols1, tr1 = make(B, 1)
    ranks = []
    for r in range(world):
        torch.manual_seed(7)
        ranks.append(make(B // world, world))
    trs, rank_pols = [tr for _, tr in ranks], [p for p, _ in ranks]
    blocks = dc.host_blocks(trs, device=capi.device())
    Bl, lr = B // world, trs[0].args.lr
    n_upd = 0
    for s in range(steps):
        batch = batch_fn(s)
        shards = [shard_batch(batch, r, Bl) for r in range(world)]
        any_actor = False
        for p in tr1.policy_ids:
            torch.manual_seed(100 + s)
            tn, an = dc.global_draws(tr1, B, p)
            dc.feed_draws([tr1], tn, an, B)
            dc.feed_draws(trs, tn, an, Bl)
            info1, prio1, _ = tr1.shared_train_policy_on_batch(p, batch)
            res = dc.lockstep_update(trs, p, shards, capi.stream_ptr())
            if torch.cuda.is_available():
                torch.cuda.synchronize()
            upd = info1["update_actor"]
            any_actor |= upd
            keys = ("critic_loss", "critic_grad_norm") + (("actor_loss", "actor_grad_norm") if upd else ())
            for r, (info, prio, _) in enumerate(res):
                assert info["update_actor"] == upd
                for k in keys:
                    assert rel_err(float(info[k]), float(info1[k])) <= 1e-5, (s, p, r, k, float(info[k]), float(info1[k]))
                if prio1 is not None:
                    want = np.asarray(prio1)[r * Bl:(r + 1) * Bl]
                    assert rel_err(np.asarray(prio), want) <= 1e-5, (s, p, r)
            for net in (capi.MADDPG_CRITIC,) + ((capi.MADDPG_ACTOR,) if upd else ()):
                want = tr1._eng[p].grad_buffer(net)
                for tr in trs:
                    got = tr._eng[p].grad_buffer(net)
                    err = float((got - want).abs().max())
                    assert err <= GRAD_TOL * float(want.abs().max()), (s, p, net, err)
        if any_actor:
            for pols in [pols1] + rank_pols:
                for pol in pols.values():
                    pol.soft_target_updates()
        n_upd += 1
        dc.assert_replicas_identical(rank_pols)
        for a, b in zip(dc.vecs(pols1)[::4], dc.vecs(rank_pols[0])[::4]):      # live parameters: the Adam-step bound per update
            assert float((a - b).abs().max()) <= 5e-3 * lr * n_upd + 1e-7, s
    dc.assert_flags(trs, blocks, world)
    for tr in trs:
        assert all(float(e.abort[0]) == 0.0 for e in tr._eng.values())


def _rmatd3(B, world):
    from offpolicy._b200.factory import build_maddpg
    from oracle.maddpg import MaddpgConfig
    cfg = MaddpgConfig(n_agents=3, obs_dim=18, act_dim=2, state_dim=54, discrete=False, td3=True, actor_update_interval=2, gain=1.0)
    args, pol, tr = build_maddpg(cfg, B, 25, dp_world_size=world)
    return {"policy_0": pol}, tr


def test_rmatd3_spread_two_ranks_equal_full_batch(gpu_engine):
    """bench.py's rmatd3_spread shape (3 agents, obs 18, Box(2), state 54, episodes of 25) at B = 2 x 16: three updates, so both slot
    parities are used and the second update trains the critic only."""
    from maddpg_checks import ref_tuple
    from oracle.maddpg import MaddpgConfig, synth_batch_cont
    cfg = MaddpgConfig(n_agents=3, obs_dim=18, act_dim=2, state_dim=54, discrete=False, td3=True, actor_update_interval=2, gain=1.0)
    dp_vs_single(_rmatd3, lambda s: ref_tuple(tuple(synth_batch_cont(cfg, 32, 25, seed=50 + s)) + (None, None)), 32, 3)


@pytest.mark.parametrize("td3", [False, True])
def test_mlp_spread_per_two_ranks_equal_full_batch(gpu_engine, td3):
    """MLP MADDPG / MATD3 at simple_spread's widths, B = 2 x 500 drawn from 100 000 transitions, with PER weights and priorities."""
    from offpolicy._b200.factory import build_mlp_maddpg
    from mlp_maddpg_checks import synth_batch
    store = synth_batch(np.random.default_rng(1), 3, 100_000, 18, 54, 5, True, per=True)
    rng = np.random.default_rng(2)

    def batch(s):
        idx = np.sort(rng.choice(100_000, 1000, replace=False))
        take = lambda x: None if x is None else np.ascontiguousarray(np.take(x, idx, axis=max(x.ndim - 2, 0)))
        return tuple({k: take(v) for k, v in d.items()} for d in store[:11]) + ((0.2 + rng.random(1000)).astype(np.float32), idx)

    def make(B, world):
        args, pol, tr = build_mlp_maddpg(3, 18, 5, 54, B, discrete=True, td3=td3, use_per=True, dp_world_size=world)
        return {"policy_0": pol}, tr
    dp_vs_single(make, batch, 1000, 2)


def test_mlp_speaker_listener_two_ranks_equal_full_batch(gpu_engine):
    """simple_speaker_listener with one policy per agent (obs 3 / 11, Discrete(3) / Discrete(5), shared observation 14): every policy's
    learner exchanges its own two buffers, its contributions to the centralised actions are row by row."""
    from offpolicy._b200.factory import build_mlp_maddpg_multi
    from mlp_maddpg_multi_checks import synth_batch_multi
    specs = [(3, 3), (11, 5)]

    def make(B, world):
        args, pols, tr, _ = build_mlp_maddpg_multi(specs, 14, B, discrete=True, td3=False, dp_world_size=world)
        return pols, tr
    dp_vs_single(make, lambda s: synth_batch_multi(np.random.default_rng(10 + s), specs, 512, 14, True), 512, 2)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("p2p", [True, False])
def test_two_gpu_rmaddpg_peer_memory_and_nccl(p2p):
    """Two processes, one GPU each: the exchange over real peer memory inside mx_maddpg_step_ex, and the NCCL fallback."""
    g = load_golden("maddpg_box")
    with tempfile.TemporaryDirectory() as td:
        port = 29700 + os.getpid() % 200 + (50 if p2p else 0)
        procs = []
        for r in range(2):
            env = dict(os.environ, RANK=str(r), WORLD_SIZE="2", LOCAL_RANK=str(r), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port),
                       MARL_B200_P2P="1" if p2p else "0")
            procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "dp_worker_maddpg.py"), td, "maddpg_box", "gpu"],
                                          env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT))
        outs = [p.communicate(timeout=300)[0].decode() for p in procs]
        assert all(p.returncode == 0 for p in procs), "\n".join(outs)
        r0, r1 = [dict(np.load(os.path.join(td, "rank%d.npz" % r))) for r in range(2)]
    assert int(r0["p2p"]) == int(p2p) == int(r1["p2p"]), "\n".join(outs)
    assert float(r0["abort"]) == 0.0 and float(r1["abort"]) == 0.0
    for k in r0:
        if k.startswith("s") and not k.endswith("update_actor"):
            assert float(r0[k]) == float(r1[k]), k
            assert rel_err(float(r0[k]), float(g[k])) <= 1e-4, (k, float(r0[k]), float(g[k]))
        if k.startswith("vec"):
            assert np.array_equal(r0[k], r1[k]), k
