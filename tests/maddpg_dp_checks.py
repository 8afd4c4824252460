"""Data-parallel R-MADDPG / R-MATD3 and MADDPG / MATD3 (the learners' two gradient exchanges, csrc/p2p.cu + csrc/maddpg.cu): several
"ranks" driven from one process, each training on its slice of one batch.  Every rank steps through `update_phases` in turn; at each
exchange every rank publishes before any rank reduces, so nothing ever waits on a peer.  The noise of an update is one global draw
taken from torch's CPU generator as the single learner would take it, each rank reading its own rows of it."""
import ctypes as C

import numpy as np
import torch

from helpers import load_golden, rel_err, sub


def shard(x, r, Bl):
    """Rank r's rows of a batch array: the batch axis is the second-to-last one of every (..., B, D) field (and axis 0 of a 1-D one)."""
    if x is None:
        return None
    x = np.asarray(x)
    ax = max(x.ndim - 2, 0)
    idx = [slice(None)] * x.ndim
    idx[ax] = slice(r * Bl, (r + 1) * Bl)
    return np.ascontiguousarray(x[tuple(idx)])


def shard_draw(d, r, Bl, world):
    """Rank r's rows of a draw in torch's agent-major layout (..., N * B, A), row = n * B + b."""
    lead, NB, A = d.shape[:-2], d.shape[-2], d.shape[-1]
    N = NB // (Bl * world)
    return d.reshape(*lead, N, Bl * world, A)[..., r * Bl:(r + 1) * Bl, :].reshape(*lead, N * Bl, A).contiguous()


def global_draws(tr, B, p_id):
    """The draws one update of policy p_id takes from torch's CPU generator at the full batch B, in the trainer's order: every
    policy's target noise (MATD3), then the actor update's Gumbel draws.  Returns ({q: target draw or None}, actor draw or None)."""
    cls = type(tr)
    tn = {q: (cls.draw_target_noise(tr, B, q) if tr._takes_noise(q, "target") else None)
          for q in (tr.policy_ids if tr.multi else [p_id])}
    upd = tr.num_updates[p_id] % tr.actor_update_interval == 0
    an = cls.draw_actor_noise(tr, B, p_id) if upd and tr._takes_noise(p_id, "actor") else None
    return tn, an


def feed_draws(ranks, tn, an, Bl):
    """Point every rank's host draws at its rows of the global draws."""
    world = len(ranks)
    for r, tr in enumerate(ranks):
        tr.draw_target_noise = lambda B, p_id=None, r=r, tr=tr: shard_draw(tn[p_id or tr.policy_ids[0]], r, Bl, world)
        tr.draw_actor_noise = lambda B, p_id=None, r=r: shard_draw(an, r, Bl, world)


def host_blocks(ranks, device="cpu"):
    """One zeroed block per rank, policy and network, attached to every rank; returns {(p_id, net): [block of rank 0, ...]}."""
    from offpolicy._b200 import capi
    tr0 = ranks[0]
    blocks = {(p, net): [torch.zeros(tr0.p2p_block_bytes(p, net) // 4, dtype=torch.float32, device=device) for _ in ranks]
              for p in tr0.policy_ids for net in (capi.MADDPG_ACTOR, capi.MADDPG_CRITIC)}
    ptrs = {k: [b.data_ptr() for b in v] for k, v in blocks.items()}
    for r, tr in enumerate(ranks):
        tr.attach_peer_blocks(r, ptrs, keep=blocks)
    return blocks


def lockstep_update(ranks, p_id, batches, stream=None):
    """One update of policy p_id on every rank: the phases of all ranks in turn, every publish before any reduce."""
    from offpolicy._b200 import capi
    lib = capi.lib()
    gens = [tr.update_phases(p_id, b) for tr, b in zip(ranks, batches)]
    results = [None] * len(gens)
    while True:
        points = []
        for i, g in enumerate(gens):
            try:
                points.append(next(g))
            except StopIteration as stop:
                results[i] = stop.value
                points.append(None)
        if all(pt is None for pt in points):
            return results
        assert all(pt is not None for pt in points), "the ranks disagree on whether this update trains the actor"
        for e, net in points:
            capi.check(lib.mx_maddpg_p2p_publish(e.handle, net, stream))
        for e, net in points:
            capi.check(lib.mx_maddpg_p2p_reduce(e.handle, net, stream))


def vecs(pols):
    return [v for p in sorted(pols) for v in list(pols[p].actor_vecs) + list(pols[p].critic_vecs)]


def assert_replicas_identical(rank_pols):
    ref = vecs(rank_pols[0])
    for pols in rank_pols[1:]:
        for a, b in zip(ref, vecs(pols)):
            assert torch.equal(a.cpu(), b.cpu()), "replicas diverged"


def flag_words(tr, p, net, block, world):
    """The flag words of one symmetric block (mx_maddpg_p2p_block_bytes: slots of both parities for 16 ranks, then the flags)."""
    P = tr._eng[p].grad_buffer(net).numel() - 4
    slot = -(-(P + 8) // 64) * 64
    return block[2 * 16 * slot:2 * 16 * slot + world].view(torch.int32)


def assert_flags(ranks, blocks, world):
    """Every block's flag words: writer r raised the step count of that network's Adam counter on every rank."""
    from offpolicy._b200 import capi
    tr0 = ranks[0]
    for (p, net), bl in blocks.items():
        count = float(tr0.ws_view("adam_ta" if net == capi.MADDPG_ACTOR else "adam_tc", p, torch.float64)[0])
        for b in bl:
            flags = flag_words(tr0, p, net, b, world).cpu()
            assert [int(f) for f in flags] == [int(count)] * world, (p, net, flags, count)


def _check_info(info, want, keys, tol, tag):
    for k in keys:
        e = rel_err(float(info[k]), want[k])
        assert e <= tol, (tag, k, float(info[k]), want[k], e)


# ---- the goldens: one builder and one check per kind ----------------------------------------------------------------------------------
def golden_dp(name, world=2, tol=1e-4):
    """Each of `world` ranks trains on its slice of the golden's batches; train_info within `tol` of the reference's, parameters within
    the Adam-step bound of the golden checks, live and target replicas bit-identical, flags equal to the step counts, and each rank's
    PER priorities equal to the golden's for its rows."""
    g = load_golden(name)
    if "meta.specs" in g or "meta.md" in g:
        return _golden_dp_policies(g, world, tol)
    if "construct.rng" in g:
        return _golden_dp_mlp(g, world, tol)
    return _golden_dp_rnn(g, world, tol)


def _golden_dp_rnn(g, world, tol):
    from maddpg_checks import build, ref_tuple
    from test_oracle_maddpg import maddpg_from_golden, maddpg_batch
    L, cfg, B, T, steps = maddpg_from_golden(g)
    Bl = B // world
    ranks, rank_pols = [], []
    for r in range(world):
        args, pol, tr = build(cfg, Bl, T, dp_world_size=world)
        assert tr.world_size == world and not tr._p2p
        for tag, mod in (("actor", pol.actor), ("critic", pol.critic), ("tgt_actor", pol.target_actor), ("tgt_critic", pol.target_critic)):
            mod.load_state_dict(sub(g, "init.%s." % tag))
        ranks.append(tr)
        rank_pols.append({"policy_0": pol})
    blocks = host_blocks(ranks)
    for s in range(steps):
        batch, _ = maddpg_batch(g, s)
        torch.manual_seed(1000 + s)                       # the draws of the single learner (check_golden)
        tn, an = global_draws(ranks[0], B, "policy_0")
        feed_draws(ranks, tn, an, Bl)
        shards = [ref_tuple(tuple(shard(x, r, Bl) for x in batch[:8]) + (np.arange(Bl),)) for r in range(world)]
        res = lockstep_update(ranks, "policy_0", shards)
        want = {k: float(g["s%d.%s" % (s, k)]) for k in ("critic_loss", "critic_grad_norm", "actor_loss", "actor_grad_norm") if "s%d.%s" % (s, k) in g}
        upd = bool(int(g["s%d.update_actor" % s]))
        for r, (info, prio, _) in enumerate(res):
            assert info["update_actor"] == upd, (s, r)
            _check_info(info, want, ("critic_loss", "critic_grad_norm") + (("actor_loss", "actor_grad_norm") if upd else ()), tol, (s, r))
            if cfg.use_per:
                assert rel_err(np.asarray(prio), g["s%d.prio" % s][r * Bl:(r + 1) * Bl]) < 1e-4, (s, r)
        if upd:
            for pols in rank_pols:
                pols["policy_0"].soft_target_updates()
        assert_replicas_identical(rank_pols)
        assert_flags(ranks, blocks, world)
    pol = rank_pols[0]["policy_0"]
    for tag, mod in (("actor", pol.actor), ("critic", pol.critic), ("tgt_actor", pol.target_actor), ("tgt_critic", pol.target_critic)):
        for k, v in mod.state_dict().items():
            assert np.abs(v.cpu().numpy() - g["final.%s.%s" % (tag, k)]).max() <= 5e-3 * cfg.lr * steps + 1e-7, (tag, k)
    return ranks


def _golden_dp_mlp(g, world, tol):
    from offpolicy._b200.factory import build_mlp_maddpg
    from mlp_maddpg_checks import golden_meta, golden_batch
    torch.set_num_threads(1)
    (N, O, A, S, B, steps, td3, discrete), over = golden_meta(g)
    Bl = B // world
    ranks, rank_pols = [], []
    for r in range(world):
        torch.manual_seed(3)                              # the golden's construction: every rank starts from the same replica
        args, pol, tr = build_mlp_maddpg(N, O, A, S, Bl, discrete=discrete, td3=td3, dp_world_size=world, **over)
        ranks.append(tr)
        rank_pols.append({"policy_0": pol})
    blocks = host_blocks(ranks)
    for s in range(steps):
        torch.set_rng_state(torch.from_numpy(g["s%d.rng_before" % s]))
        tn, an = global_draws(ranks[0], B, "policy_0")
        assert np.array_equal(torch.get_rng_state().numpy(), g["s%d.rng_after" % s])
        feed_draws(ranks, tn, an, Bl)
        full = golden_batch(g, s)
        shards = [tuple({"policy_0": shard(d["policy_0"], r, Bl)} for d in full[:11]) + (shard(full[11], r, Bl), None if full[12] is None else np.arange(Bl))
                  for r in range(world)]
        res = lockstep_update(ranks, "policy_0", shards)
        want = {k: float(g["s%d.%s" % (s, k)]) for k in ("critic_loss", "critic_grad_norm", "actor_loss", "actor_grad_norm")}
        for r, (info, prio, _) in enumerate(res):
            _check_info(info, want, tuple(want), tol, (s, r))
            if prio is not None:
                assert rel_err(np.asarray(prio), g["s%d.prio" % s][r * Bl:(r + 1) * Bl]) < 1e-4, (s, r)
        pol = rank_pols[0]["policy_0"]
        for tag, mod in (("actor", pol.actor), ("critic", pol.critic)):
            for k, v in mod.state_dict().items():
                assert np.abs(v.cpu().numpy() - g["s%d.post.%s.%s" % (s, tag, k)]).max() <= 5e-3 * args.lr * (s + 1) + 1e-7, (s, tag, k)
        for pols in rank_pols:
            pols["policy_0"].soft_target_updates()
        for tag, mod in (("tgt_actor", pol.target_actor), ("tgt_critic", pol.target_critic)):
            for k, v in mod.state_dict().items():
                assert np.abs(v.cpu().numpy() - g["s%d.post.%s.%s" % (s, tag, k)]).max() <= 5e-3 * args.lr * (s + 1) + 1e-7, (s, tag, k)
        assert_replicas_identical(rank_pols)
        assert_flags(ranks, blocks, world)
    return ranks


def _golden_dp_policies(g, world, tol):
    """The fixtures of make_goldens_mlp_maddpg_multi / _md: one or several policies, each updated on its own fixture batch."""
    from offpolicy._b200.factory import build_mlp_maddpg_multi
    from mlp_maddpg_multi_checks import golden_batch_multi, golden_rng_before, golden_expected
    torch.set_num_threads(1)
    if "meta.md" in g:
        from mlp_maddpg_md_checks import golden_meta
        (specs, S, B, steps, td3), over = golden_meta(g)
        discrete = True
    else:
        from mlp_maddpg_multi_checks import golden_meta_multi
        (specs, S, B, steps, td3, discrete), over = golden_meta_multi(g)
    Bl = B // world
    ranks, rank_pols = [], []
    for r in range(world):
        torch.manual_seed(3)
        args, pols, tr, _ = build_mlp_maddpg_multi(specs, S, Bl, discrete=discrete, td3=td3, dp_world_size=world, **over)
        ranks.append(tr)
        rank_pols.append(pols)
    p_ids = ranks[0].policy_ids
    blocks = host_blocks(ranks)
    tol_p = lambda n: 5e-3 * args.lr * n + 1e-7
    for s in range(steps):
        for p in p_ids:
            torch.set_rng_state(torch.from_numpy(golden_rng_before(g, s, p, p_ids)))
            tn, an = global_draws(ranks[0], B, p)
            assert np.array_equal(torch.get_rng_state().numpy(), g["s%d.%s.rng_after" % (s, p)]), (s, p)
            feed_draws(ranks, tn, an, Bl)
            full = golden_batch_multi(g, s, p, p_ids)
            shards = [tuple({q: shard(d[q], r, Bl) for q in d} for d in full[:-2]) + (shard(full[-2], r, Bl), None if full[-1] is None else np.arange(Bl))
                      for r in range(world)]
            res = lockstep_update(ranks, p, shards)
            want = {k: float(g["s%d.%s.%s" % (s, p, k)]) for k in ("critic_loss", "critic_grad_norm", "actor_loss", "actor_grad_norm")}
            for r, (info, prio, _) in enumerate(res):
                _check_info(info, want, tuple(want), tol, (s, p, r))
                if prio is not None:
                    assert rel_err(np.asarray(prio), g["s%d.%s.prio" % (s, p)][r * Bl:(r + 1) * Bl]) < 1e-4, (s, p, r)
            if s == 0:
                pol = rank_pols[0][p]
                for tag, mod in (("actor", pol.actor), ("critic", pol.critic)):
                    for k, v in mod.state_dict().items():
                        ref = golden_expected(g, "s0.%s.post.%s.%s" % (p, tag, k), p, tag)
                        assert np.abs(v.cpu().numpy() - ref).max() <= tol_p(1), (s, p, tag, k)
        for pols in rank_pols:
            for p in p_ids:
                pols[p].soft_target_updates()
        assert_replicas_identical(rank_pols)
        assert_flags(ranks, blocks, world)
    for p in p_ids:
        pol = rank_pols[0][p]
        for tag, mod in (("actor", pol.actor), ("critic", pol.critic), ("tgt_actor", pol.target_actor), ("tgt_critic", pol.target_critic)):
            for k, v in mod.state_dict().items():
                ref = golden_expected(g, "final.%s.%s.%s" % (p, tag, k), p, tag)
                assert np.abs(v.cpu().numpy() - ref).max() <= tol_p(steps), (p, tag, k)
    return ranks
