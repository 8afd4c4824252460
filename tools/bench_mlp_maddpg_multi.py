"""Runner updates/s of the transition-level MADDPG / MATD3 with one policy per agent (share_policy off), B = 1 000 transitions drawn
from a replay of 500 000, at two shapes: simple_speaker_listener (obs 3 / 11, Discrete(3) / Discrete(5), shared observation 14) and
simple_spread with one policy per agent (3 x obs 18, Discrete(5), shared observation 54).

One timed iteration is the MLP runner's batch_train (runner/mlp/base_runner.py:187-217): for each policy, `sample(B)` (the host's NumPy
draw, one index set gathered into every policy's store) and `shared_train_policy_on_batch` (every policy's target actions into the
updated policy's centralised action vectors, then its mx_maddpg step), then the soft target updates of all policies.  It runs eagerly
(a multi-policy update is not captured as a graph); the noise draws come from torch's CPU generator as the reference makes them.
Timed over `--steps` iterations after `--warmup`, ending in a device synchronise.  CPU arm: oracle/maddpg_mlp_multi.py (the reference's
update restated in eager PyTorch) on the same shapes and host.  Prints one JSON line with a result per (shape, algorithm); needs a CUDA
device and never falls back to the CPU for the GPU arm.

    python tools/bench_mlp_maddpg_multi.py --steps 200 --warmup 20
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

SHAPES = {"speaker_listener": ([(3, 3), (11, 5)], 14), "spread_per_agent": ([(18, 5)] * 3, 54)}


def fill(buf, specs, S, B, size, rng):
    from mlp_maddpg_multi_checks import norm_specs, synth_batch_multi
    shapes = norm_specs(specs)
    tr = lambda x: np.asarray(x).transpose(1, 0, 2)                     # (N, B, .) -> the runner's (B, N, .)
    for _ in range(size // B):
        b = synth_batch_multi(rng, specs, B, S, True)
        per_p = lambda i, t=True: {p: (tr(b[i][p]) if t else b[i][p]) for p in shapes}
        buf.insert(B, per_p(0), per_p(1, False), per_p(2), per_p(3), per_p(4), per_p(5, False), per_p(6), per_p(7, False), per_p(8), None, None)


def gpu_arm(specs, S, td3, B, size, steps, warmup):
    from offpolicy._b200.factory import build_mlp_maddpg_multi, Discrete, Box
    from offpolicy.utils.mlp_buffer import MlpReplayBuffer
    from mlp_maddpg_multi_checks import norm_specs
    torch.manual_seed(1)
    args, pols, tr, agents = build_mlp_maddpg_multi(specs, S, B, discrete=True, td3=td3)
    info = {p: dict(obs_space=Box(o), share_obs_space=Box(S), act_space=Discrete(a)) for p, (o, a, n) in norm_specs(specs).items()}
    buf = MlpReplayBuffer(info, agents, size, True, False, max_batch=B)
    fill(buf, specs, S, B, size, np.random.default_rng(2))
    np.random.seed(3)
    ids = sorted(pols)

    def batch_train():
        out = None
        for p in ids:
            out, _, _ = tr.shared_train_policy_on_batch(p, buf.sample(B))
        for p in ids:
            pols[p].soft_target_updates()
        return out
    for _ in range(warmup):
        batch_train()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        info_t = batch_train()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    loss = float(info_t["critic_loss"])
    assert np.isfinite(loss)
    return steps / dt, loss


def cpu_arm(specs, S, td3, B, steps):
    from mlp_maddpg_multi_checks import norm_specs, synth_batch_multi
    from oracle.maddpg_mlp import MlpMaddpg
    from oracle.maddpg_mlp_multi import draw_noise_multi, step_multi
    from offpolicy._b200.flat import mlp_init
    torch.manual_seed(1)
    shapes = norm_specs(specs)
    total = sum(a * n for _, a, n in shapes.values())
    heads = [("q_outs.%d" % k, 1, 1.0) for k in range(2 if td3 else 1)]
    split = lambda d, head: {k: v for k, v in d.items() if k.startswith("q_outs") == head}
    learners = {}
    for p, (o, a, n) in shapes.items():
        act = mlp_init(o, 64, [("act.action_out", a, 0.01)], True)
        c, ct = mlp_init(S + total, 64, heads, True), mlp_init(S + total, 64, heads, True)
        learners[p] = MlpMaddpg(act, split(c, False), split(c, True), act, split(c, False), split(ct, True), True, td3, lr=5e-4)
    noise = {p: (n, a, True, td3, 0.2) for p, (o, a, n) in shapes.items()}
    rng = np.random.default_rng(4)
    batches = [synth_batch_multi(rng, specs, B, S, True) for _ in range(4)]

    def batch_train(i):
        for j, p in enumerate(sorted(learners)):
            tn, an = draw_noise_multi(noise, p, B)
            step_multi(learners, p, batches[(i + j) % 4], tn, an)
        for L in learners.values():
            L.soft_update()
    batch_train(0)
    t0 = time.perf_counter()
    for i in range(steps):
        batch_train(i)
    return steps / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--batch", type=int, default=1000)
    ap.add_argument("--buffer", type=int, default=500_000)
    ap.add_argument("--cpu-steps", type=int, default=10)
    ap.add_argument("--algo", choices=["maddpg", "matd3", "both"], default="both")
    ap.add_argument("--shape", choices=list(SHAPES) + ["both"], default="both")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mlp_maddpg_multi: needs a CUDA device")
    from offpolicy._b200 import capi
    capi.lib()
    results = []
    for shape in (list(SHAPES) if a.shape == "both" else [a.shape]):
        specs, S = SHAPES[shape]
        for algo in (["maddpg", "matd3"] if a.algo == "both" else [a.algo]):
            td3 = algo == "matd3"
            rate, loss = gpu_arm(specs, S, td3, a.batch, a.buffer, a.steps, a.warmup)
            cpu = cpu_arm(specs, S, td3, a.batch, a.cpu_steps)
            results.append({"shape": shape, "policies": len(specs), "algo": algo, "value": rate, "grad_steps_per_s": rate * len(specs),
                            "last_critic_loss": loss, "cpu_oracle": cpu, "speedup_vs_cpu_oracle": rate / cpu})
    # the card and its power limit, read in the same call as the measurement
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"metric": "runner updates/s", "unit": "batch_train/s", "batch": a.batch, "buffer": a.buffer, "steps": a.steps,
                      "warmup": a.warmup, "gpu": q,
                      "path": "eager: per policy host sample + gather, cent_contribute x policies + mx_maddpg step (mlp); soft updates",
                      "cpu_oracle_kind": "oracle/maddpg_mlp_multi.py (eager PyTorch restatement of the reference update)",
                      "cpu_oracle_steps": a.cpu_steps, "torch_threads": torch.get_num_threads(), "host_cores": os.cpu_count(),
                      "results": results}))


if __name__ == "__main__":
    main()
