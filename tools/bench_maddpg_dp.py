"""Data-parallel rate of the actor-critic learners: one process per GPU, each rank sampling B per update from its own replay shard
(weak scaling: the global batch is G * B), both gradient exchanges per update inside the step (peer memory) or, with MARL_B200_P2P=0,
through torch.distributed.all_reduce.  Shapes: bench.py's rmaddpg_spread / rmatd3_spread (3 agents, obs 18, Box(2), shared observation
54, episodes of 25) and the MLP simple_spread learner (obs 18, Discrete(5), MADDPG / MATD3).

Per shape it times `--steps` eager updates (sample -> shared_train_policy_on_batch -> soft target update) after `--warmup`, ending in
a device synchronise, and reports G x updates/s.  With G > 1 it then times the exchanges alone over `--steps` more updates: CUDA events
around the critic's and the actor's exchange of each update (driven through update_phases), summed per update.  At G = 1 there is no
exchange and its time is reported as null.  Prints one JSON line per shape.  Needs a CUDA device.

    python tools/bench_maddpg_dp.py --steps 200 --warmup 20                                  # G = 1
    torchrun --nproc_per_node 8 tools/bench_maddpg_dp.py --steps 200 --warmup 20             # G = 8
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "off-policy_b200"), os.path.join(ROOT, "tests")]

SHAPES = {"rmaddpg_spread": (False, 32), "rmatd3_spread": (True, 32), "mlp_maddpg_spread": (False, 1000), "mlp_matd3_spread": (True, 1000)}


def recurrent(td3, B, episodes, seed):
    from offpolicy._b200.factory import Box, build_maddpg
    from offpolicy.utils.rec_buffer import RecReplayBuffer
    from oracle.maddpg import MaddpgConfig
    import replay_checks as rc
    T = 25
    cfg = MaddpgConfig(n_agents=3, obs_dim=18, act_dim=2, state_dim=54, discrete=False, td3=td3, actor_update_interval=2 if td3 else 1,
                       gain=1.0)
    torch.manual_seed(1)                  # every rank starts from the same replica
    args, pol, tr = build_maddpg(cfg, B, T)
    n, o, a, s = cfg.n_agents, cfg.obs_dim, cfg.act_dim, cfg.state_dim
    info = {"policy_0": dict(obs_space=[o], share_obs_space=[s], act_space=Box(a))}
    buf = RecReplayBuffer(info, {"policy_0": list(range(n))}, episodes, T, True, False, rng="device", max_batch=max(B, 64))
    rs = np.random.RandomState(seed)      # each rank its own shard
    for _ in range(episodes // 64):
        E = 64
        ep = [rs.randn(T + 1, E, n, o).astype(np.float32), np.repeat(rs.randn(T + 1, E, 1, s).astype(np.float32), n, 2),
              rs.uniform(-1, 1, (T, E, n, a)).astype(np.float32), np.repeat(rs.randn(T, E, 1, 1).astype(np.float32), n, 2),
              np.zeros((T, E, n, 1), np.float32), np.zeros((T, E, 1), np.float32)]
        buf.insert(E, *[rc.d(x) for x in ep], None)
    buf.seed_device_rng(seed)
    return pol, tr, buf


def mlp(td3, B, size, seed):
    from offpolicy._b200.factory import Box, act_space, build_mlp_maddpg
    from offpolicy.utils.mlp_buffer import MlpReplayBuffer
    from mlp_maddpg_checks import synth_batch
    N, O, A, S = 3, 18, 5, 54
    torch.manual_seed(1)
    args, pol, tr = build_mlp_maddpg(N, O, A, S, B, discrete=True, td3=td3)
    info = {"policy_0": dict(obs_space=Box(O), share_obs_space=Box(S), act_space=act_space(A))}
    buf = MlpReplayBuffer(info, {"policy_0": list(range(N))}, size, True, False, max_batch=B)
    rng = np.random.default_rng(seed)
    t = lambda x: np.asarray(x["policy_0"]).transpose(1, 0, 2)
    for _ in range(size // B):
        b = synth_batch(rng, N, B, O, S, A, True)
        buf.insert(B, {"policy_0": t(b[0])}, {"policy_0": b[1]["policy_0"]}, {"policy_0": t(b[2])}, {"policy_0": t(b[3])},
                   {"policy_0": t(b[4])}, {"policy_0": b[5]["policy_0"]}, {"policy_0": t(b[6])}, {"policy_0": b[7]["policy_0"]},
                   {"policy_0": t(b[8])}, None, None)
    buf.seed_device_rng(seed)
    return pol, tr, buf


def update(pol, tr, buf, B):
    info, _, _ = tr.shared_train_policy_on_batch("policy_0", buf.sample(B))
    if info["update_actor"]:
        pol.soft_target_updates()


def exchange_ms(pol, tr, buf, B, steps):
    """Mean device time per update of its exchanges (CUDA events around each one)."""
    from offpolicy._b200 import capi
    lib, total = capi.lib(), 0.0
    for _ in range(steps):
        g = tr.update_phases("policy_0", buf.sample(B))
        evs = []
        try:
            while True:
                e, net = next(g)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                if tr._p2p:
                    capi.check(lib.mx_maddpg_p2p_publish(e.handle, net, capi.stream_ptr()))
                    capi.check(lib.mx_maddpg_p2p_reduce(e.handle, net, capi.stream_ptr()))
                else:
                    torch.distributed.all_reduce(e.grad_buffer(net))
                b.record()
                evs.append((a, b))
        except StopIteration as stop:
            if stop.value[0]["update_actor"]:
                pol.soft_target_updates()
        torch.cuda.synchronize()
        total += sum(a.elapsed_time(b) for a, b in evs)
    return total / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--episodes", type=int, default=2048, help="episodes per rank's shard (recurrent shapes)")
    ap.add_argument("--buffer", type=int, default=100_000, help="transitions per rank's shard (MLP shapes)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_maddpg_dp: needs a CUDA device")
    dist = torch.distributed
    if "WORLD_SIZE" in os.environ and int(os.environ["WORLD_SIZE"]) > 1:
        rank = int(os.environ["RANK"])
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
        dist.init_process_group("nccl", device_id=torch.device("cuda", torch.cuda.current_device()))
    rank = dist.get_rank() if dist.is_initialized() else 0
    world = dist.get_world_size() if dist.is_initialized() else 1
    for name in a.shapes.split(","):
        td3, B = SHAPES[name]
        pol, tr, buf = (mlp(td3, B, a.buffer, 10 + rank) if name.startswith("mlp") else recurrent(td3, B, a.episodes, 10 + rank))
        for _ in range(a.warmup):
            update(pol, tr, buf, B)
        torch.cuda.synchronize()
        if dist.is_initialized():
            dist.barrier()
        t0 = time.perf_counter()
        for _ in range(a.steps):
            update(pol, tr, buf, B)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        xms = exchange_ms(pol, tr, buf, B, a.steps) if world > 1 else None
        if rank == 0:
            print(json.dumps({"shape": name, "world": world, "batch_per_gpu": B, "global_batch": world * B, "steps": a.steps,
                              "updates_per_s_per_gpu": a.steps / dt, "samples_per_s": world * B * a.steps / dt,
                              "world_x_updates_per_s": world * a.steps / dt, "exchange": ("peer memory" if tr._p2p else "all_reduce") if world > 1 else None,
                              "exchange_ms_per_update": xms, "critic_loss": float(tr._info[0]),
                              "gpu": torch.cuda.get_device_name(), "n_gpus": world}), flush=True)
    if dist.is_initialized():
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
