"""Grad-steps/s of the transition-level MADDPG / MATD3 learner at the shapes of scripts/train_mpe_maddpg.sh: simple_spread (3 agents,
obs 18, Discrete(5), shared observation 54), B = 1 000 transitions drawn from a replay of 500 000.  `--shape reference` runs the shapes of
scripts/train_mpe_matd3.sh instead: simple_reference (2 agents, obs 21, shared observation 42, MultiDiscrete actions of sub-spaces 5 and
10).

GPU arm: the whole-update CUDA graph (MaddpgStepGraph: device uniform draw + gather -> mx_maddpg step -> soft target update), the
per-update noise drawn on the host from torch's CPU generator exactly as the reference draws it and copied into the graph's fixed
buffers through its pinned staging ring before each replay;
timed over `--steps` replays after `--warmup`, ending in a device synchronise.  CPU arm: oracle/maddpg_mlp.py (the reference's
update restated in eager PyTorch) on the same host and shapes, with its thread count and the host's core count.
Prints one JSON line per algorithm.  Needs a CUDA device; it never falls back to the CPU for the GPU arm.

    python tools/bench_mlp_maddpg.py --steps 500 --warmup 50
    python tools/bench_mlp_maddpg.py --shape reference --steps 500 --warmup 50
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "off-policy_b200"), os.path.join(ROOT, "tests")]

N, O, A, S = 3, 18, 5, 54
SEGS = None          # the MultiDiscrete sub-space widths of --shape reference; A is then their sum


def set_shape(shape):
    global N, O, A, S, SEGS
    if shape == "reference":
        N, O, S, SEGS = 2, 21, 42, [5, 10]
        A = sum(SEGS)


def synth(rng, B):
    if SEGS is None:
        from mlp_maddpg_checks import synth_batch
        return synth_batch(rng, N, B, O, S, A, True)
    from mlp_maddpg_md_checks import synth_batch_md
    return synth_batch_md(rng, [(O, SEGS, N)], B, S)


def fill(buf, B, size, rng):
    tr = lambda x: np.asarray(x["policy_0"]).transpose(1, 0, 2)
    for _ in range(size // B):
        b = synth(rng, B)
        buf.insert(B, {"policy_0": tr(b[0])}, {"policy_0": b[1]["policy_0"]}, {"policy_0": tr(b[2])}, {"policy_0": tr(b[3])},
                   {"policy_0": tr(b[4])}, {"policy_0": b[5]["policy_0"]}, {"policy_0": tr(b[6])}, {"policy_0": b[7]["policy_0"]},
                   {"policy_0": tr(b[8])}, None, None)


def gpu_arm(td3, B, size, steps, warmup):
    from offpolicy._b200.factory import build_mlp_maddpg, act_space, Box
    from offpolicy._b200.graph import MaddpgStepGraph
    from offpolicy.utils.mlp_buffer import MlpReplayBuffer
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.manual_seed(1)
        act = A if SEGS is None else SEGS
        args, pol, tr = build_mlp_maddpg(N, O, act, S, B, discrete=True, td3=td3)
        info = {"policy_0": dict(obs_space=Box(O), share_obs_space=Box(S), act_space=act_space(act))}
        buf = MlpReplayBuffer(info, {"policy_0": list(range(N))}, size, True, False, max_batch=B)
        fill(buf, B, size, np.random.default_rng(2))
        buf.seed_device_rng(3)
        g = MaddpgStepGraph(buf, tr, B)
        for _ in range(warmup):
            g.launch()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            g.launch()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        loss = float(tr._info[0])
    assert np.isfinite(loss)
    return steps / dt, loss


def cpu_arm(td3, B, steps):
    from oracle.maddpg_mlp import MlpMaddpg, draw_noise
    from oracle.maddpg_mlp_md import MlpMaddpgMD, draw_noise_md
    from offpolicy._b200.flat import mlp_init
    torch.manual_seed(1)
    heads = [("q_outs.%d" % k, 1, 1.0) for k in range(2 if td3 else 1)]
    a_heads = [("act.action_out", A, 0.01)] if SEGS is None else [("act.action_outs.%d" % i, n, 0.01) for i, n in enumerate(SEGS)]
    a = mlp_init(O, 64, a_heads, True)
    c = mlp_init(S + N * A, 64, heads, True)
    ct = mlp_init(S + N * A, 64, heads, True)
    split = lambda d, head: {k: v for k, v in d.items() if k.startswith("q_outs") == head}
    nets = (a, split(c, False), split(c, True), a, split(c, False), split(ct, True), True, td3)
    L = MlpMaddpg(*nets, lr=5e-4) if SEGS is None else MlpMaddpgMD(*nets, lr=5e-4, segs=SEGS)
    noise = (lambda: draw_noise(N, B, A, True, td3, 0.2)) if SEGS is None else (lambda: draw_noise_md(N, B, SEGS, td3))
    rng = np.random.default_rng(4)
    batches = [synth(rng, B) for _ in range(4)]
    L.step(batches[0], *noise())
    t0 = time.perf_counter()
    for i in range(steps):
        L.step(batches[i % 4], *noise())
        L.soft_update()
    return steps / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=500)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--batch", type=int, default=1000)
    ap.add_argument("--buffer", type=int, default=500_000)
    ap.add_argument("--cpu-steps", type=int, default=20)
    ap.add_argument("--algo", choices=["maddpg", "matd3", "both"], default="both")
    ap.add_argument("--shape", choices=["spread", "reference"], default="spread",
                    help="simple_spread (Discrete, train_mpe_maddpg.sh) or simple_reference (MultiDiscrete, train_mpe_matd3.sh)")
    a = ap.parse_args()
    set_shape(a.shape)
    if not torch.cuda.is_available():
        raise SystemExit("bench_mlp_maddpg: needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    for algo in (["maddpg", "matd3"] if a.algo == "both" else [a.algo]):
        td3 = algo == "matd3"
        rate, loss = gpu_arm(td3, a.batch, a.buffer, a.steps, a.warmup)
        cpu = cpu_arm(td3, a.batch, a.cpu_steps)
        rec = {"metric": "grad-steps/s", "algo": algo, "value": rate, "unit": "steps/s", "batch": a.batch, "buffer": a.buffer,
               "steps": a.steps, "warmup": a.warmup, "path": "CUDA graph: device draw + gather + mx_maddpg step (mlp) + soft update; "
               "host noise draws copied in per step through a pinned ring", "last_critic_loss": loss, "gpu": q,
               "cpu_oracle": {"value": cpu, "unit": "steps/s", "torch_threads": torch.get_num_threads(), "host_cores": os.cpu_count(),
                              "steps": a.cpu_steps, "kind": "oracle/maddpg_mlp.py (eager PyTorch restatement of the reference update)"},
               "speedup_vs_cpu_oracle": rate / cpu}
        if SEGS is not None:
            rec["shape"] = {"scenario": "simple_reference", "n_agents": N, "obs_dim": O, "state_dim": S, "act_segs": SEGS}
            rec["cpu_oracle"]["kind"] = "oracle/maddpg_mlp_md.py (eager PyTorch restatement of the reference update)"
        print(json.dumps(rec))


if __name__ == "__main__":
    main()
