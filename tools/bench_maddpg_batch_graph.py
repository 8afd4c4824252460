"""batch_train/s of MADDPG / MATD3 with one policy per agent (share_policy off): the runner's eager batch_train against the same
batch_train replayed as one CUDA graph (MaddpgBatchTrainGraph), both with the update noise drawn on the device
(trainer.use_device_noise) and the indices from the stores' device RNG.  Shapes:

    rmaddpg_speaker_listener / rmatd3_speaker_listener   R-MADDPG / R-MATD3 at train_mpe_rmaddpg.sh shapes: simple_speaker_listener
                                                         (obs 3 / 11, Discrete(3) / Discrete(5), shared observation 14), episode 25,
                                                         B = 32 episodes from a 5 000-episode store
    maddpg_speaker_listener / matd3_speaker_listener     MLP MADDPG / MATD3, the same spaces, B = 1 000 transitions from --buffer
    maddpg_spread_per_agent / matd3_spread_per_agent     MLP MADDPG / MATD3, simple_spread with three policies (obs 18, Discrete(5),
                                                         shared observation 54), B = 1 000 from --buffer

One eager batch_train is runner/{rnn,mlp}/base_runner.py's: per policy `sample` + `train_policy_on_batch`, then the soft updates of
every policy (tests/maddpg_batch_graph_checks.py: eager_batch_train).  One graph batch_train is one `launch()`.  Both arms run on the
same trainer and replay, alternating, --reps windows each; a window is --steps batch_trains after --warmup, between two device
synchronisations.  torch runs one host thread, the reference's default (config.py:17-18).  Prints one JSON line per shape with the
graph's kernel count, and the card's name, power limit and maximum SM clock read in the same call.  Needs a CUDA device.

    python tools/bench_maddpg_batch_graph.py --steps 200 --warmup 20 --reps 3
"""
import argparse
import contextlib
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "off-policy_b200"), os.path.join(ROOT, "tests")]

SL = [(1, 3, 3), (1, 11, 5)]
SPREAD = [(1, 18, 5)] * 3
SHAPES = {
    "rmaddpg_speaker_listener": dict(kind="rec", specs=SL, S=14, B=32, T=25, E=5000, td3=False),
    "rmatd3_speaker_listener": dict(kind="rec", specs=SL, S=14, B=32, T=25, E=5000, td3=True),
    "maddpg_speaker_listener": dict(kind="mlp", specs=SL, S=14, B=1000, td3=False),
    "matd3_speaker_listener": dict(kind="mlp", specs=SL, S=14, B=1000, td3=True),
    "maddpg_spread_per_agent": dict(kind="mlp", specs=SPREAD, S=54, B=1000, td3=False),
    "matd3_spread_per_agent": dict(kind="mlp", specs=SPREAD, S=54, B=1000, td3=True),
}


def case_of(name, buffer):
    from maddpg_batch_graph_checks import BatchCase
    s = dict(SHAPES[name])
    E = s.pop("E", buffer)
    return BatchCase(s.pop("kind"), s.pop("specs"), S=s.pop("S"), B=s.pop("B"), E=E, rng="device", insert=0, **s)


def timed(one, steps, warmup):
    for _ in range(warmup):
        one()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        one()
    torch.cuda.synchronize()
    return steps / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--buffer", type=int, default=500_000)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_maddpg_batch_graph: needs a CUDA device")
    torch.set_num_threads(1)
    from maddpg_batch_graph_checks import eager_batch_train
    from offpolicy._b200 import capi
    from offpolicy._b200.graph import MaddpgBatchTrainGraph
    from offpolicy._b200.torch_rng import DeviceTorchGenerator
    capi.lib()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    for name in a.shapes.split(","):
        case = case_of(name, a.buffer)
        with contextlib.redirect_stdout(sys.stderr):
            tr, buf, pols = case.build(1)
            case.fill(buf, np.random.RandomState(2), case.E)
            tr.use_device_noise(DeviceTorchGenerator(seed=3))
            g = MaddpgBatchTrainGraph(buf, tr, case.B)
            arms = {"eager": lambda: eager_batch_train(case, tr, buf, pols), "graph": g.launch}
            rates = {"eager": [], "graph": []}
            for _ in range(a.reps):
                for arm in ("eager", "graph"):
                    rates[arm].append(timed(arms[arm], a.steps, a.warmup))
            loss = {p: float(tr._eng[p].info[0]) for p in case.ids}
            kernels = g.num_kernels
            g.close()
        assert all(np.isfinite(v) for v in loss.values()), loss
        rec = {"metric": "batch_train/s", "shape": name, "policies": len(case.specs), "unit": "batch_train/s", "batch": case.B,
               "buffer": case.E, "steps": a.steps, "warmup": a.warmup, "eager": rates["eager"], "graph": rates["graph"],
               "median_graph_over_eager": float(np.median(rates["graph"]) / np.median(rates["eager"])),
               "graph_kernels": {str(u): n for u, n in kernels.items()}, "noise": "device", "torch_threads": torch.get_num_threads(),
               "gpu": card, "last_critic_loss": loss}
        print(json.dumps(rec), flush=True)
        del g, arms, tr, buf, pols
        torch.cuda.synchronize()


if __name__ == "__main__":
    main()
