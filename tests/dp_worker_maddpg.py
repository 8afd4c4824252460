"""Worker for test_dp_gloo_maddpg.py and test_gpu_maddpg_dp.py: one data-parallel rank of R-MADDPG / MLP MATD3.  On the CPU (gloo,
emulated kernels) there is no peer memory, so the trainer takes the fallback exchange: the phases of each update with an all-reduce of
each gradient buffer.  With `gpu` each rank owns one GPU (NCCL) and exchanges over peer memory unless MARL_B200_P2P=0."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "off-policy_b200"), os.path.join(ROOT, "tests", "emu")):
    sys.path.insert(0, p)


def main():
    out_dir, name = sys.argv[1], sys.argv[2]
    gpu = len(sys.argv) > 3 and sys.argv[3] == "gpu"       # one rank per GPU: NCCL, peer memory unless MARL_B200_P2P=0
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    from offpolicy._b200 import capi
    if gpu:
        torch.cuda.set_device(rank)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
        capi.lib()
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world)
        from build_emu import LIB
        capi._install_for_tests(LIB)
    import maddpg_dp_checks as dc
    from helpers import load_golden, sub
    torch.set_num_threads(1)
    g = load_golden(name)
    out = {}
    if "construct.rng" in g:
        from offpolicy._b200.factory import build_mlp_maddpg
        from mlp_maddpg_checks import golden_meta, golden_batch
        (N, O, A, S, B, steps, td3, discrete), over = golden_meta(g)
        Bl = B // world
        torch.manual_seed(3)
        args, pol, tr = build_mlp_maddpg(N, O, A, S, Bl, discrete=discrete, td3=td3, **over)
        for s in range(steps):
            torch.set_rng_state(torch.from_numpy(g["s%d.rng_before" % s]))
            tn, an = dc.global_draws(tr, B, "policy_0")
            _feed(tr, tn, an, rank, Bl, world, dc)
            full = golden_batch(g, s)
            batch = tuple({"policy_0": dc.shard(d["policy_0"], rank, Bl)} for d in full[:11]) + (dc.shard(full[11], rank, Bl), None)
            info, _, _ = tr.train_policy_on_batch("policy_0", batch)
            pol.soft_target_updates()
            _record(out, s, info)
    else:
        from maddpg_checks import build, ref_tuple
        from test_oracle_maddpg import maddpg_from_golden, maddpg_batch
        L, cfg, B, T, steps = maddpg_from_golden(g)
        Bl = B // world
        args, pol, tr = build(cfg, Bl, T)
        for tag, mod in (("actor", pol.actor), ("critic", pol.critic), ("tgt_actor", pol.target_actor), ("tgt_critic", pol.target_critic)):
            mod.load_state_dict(sub(g, "init.%s." % tag))
        for s in range(steps):
            batch, _ = maddpg_batch(g, s)
            torch.manual_seed(1000 + s)
            tn, an = dc.global_draws(tr, B, "policy_0")
            _feed(tr, tn, an, rank, Bl, world, dc)
            info, _, _ = tr.train_policy_on_batch("policy_0", ref_tuple(tuple(dc.shard(x, rank, Bl) for x in batch[:8]) + (None,)))
            if info["update_actor"]:
                pol.soft_target_updates()
            _record(out, s, info)
    assert tr.world_size == world and (gpu or not tr._p2p)
    out["p2p"] = int(tr._p2p)
    out["abort"] = float(tr._eng["policy_0"].abort[0])
    for i, v in enumerate(dc.vecs({"policy_0": pol})):
        out["vec%d" % i] = v.cpu().numpy()
    np.savez(os.path.join(out_dir, "rank%d.npz" % rank), **out)
    dist.destroy_process_group()


def _feed(tr, tn, an, rank, Bl, world, dc):
    """This rank's rows of the update's global draws."""
    tr.draw_target_noise = lambda B, p_id=None: dc.shard_draw(tn[p_id or "policy_0"], rank, Bl, world)
    tr.draw_actor_noise = lambda B, p_id=None: dc.shard_draw(an, rank, Bl, world)


def _record(out, s, info):
    for k in ("critic_loss", "critic_grad_norm", "actor_loss", "actor_grad_norm"):
        if k in info:
            out["s%d.%s" % (s, k)] = float(info[k])
    out["s%d.update_actor" % s] = int(info["update_actor"])


if __name__ == "__main__":
    main()
