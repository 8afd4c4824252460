"""Grad-steps/s of the MADDPG-family whole-update graphs (MaddpgStepGraph) with the update noise drawn on the host (torch's CPU
generator, placed in the graph's pinned staging ring and copied in before every replay) against drawn on the device
(trainer.use_device_noise: the fills at the head of the graph, one launch per update).  Shapes:

    maddpg_spread / matd3_spread        MLP MADDPG / MATD3, simple_spread (3 agents, obs 18, Discrete(5), shared observation 54)
    maddpg_reference / matd3_reference  MLP MADDPG / MATD3, simple_reference (2 agents, obs 21, MultiDiscrete 5 + 10, shared obs 42)
    rmatd3_spread                       R-MATD3 at bench.py's rmatd3_spread shapes (3 agents, obs 18, Box(2), state 54, T 25, B 32)

The MLP shapes take B = 1 000 transitions from a replay of --buffer (500 000) random transitions, R-MATD3 B = 32 episodes from 5 000.
Host and device arms alternate, --reps times each, in one process; each timed window is --steps updates after --warmup, between two
device synchronisations.  The fills' device time per update comes from CUDA events around --fill-reps eager rounds of the same fills.
torch runs one host thread, the reference's default (config.py:17-18).  Prints one JSON line per shape, with the card's name, power
limit and maximum SM clock read in the same call.  Needs a CUDA device.

    python tools/bench_maddpg_device_noise.py --steps 500 --warmup 50 --reps 3
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

SHAPES = {
    "maddpg_spread": dict(kind="mlp", specs=[(3, 18, 5)], S=54, B=1000, td3=False),
    "matd3_spread": dict(kind="mlp", specs=[(3, 18, 5)], S=54, B=1000, td3=True),
    "maddpg_reference": dict(kind="mlp", specs=[(2, 21, [5, 10])], S=42, B=1000, td3=False),
    "matd3_reference": dict(kind="mlp", specs=[(2, 21, [5, 10])], S=42, B=1000, td3=True),
    "rmatd3_spread": dict(kind="rec", specs=[(3, 18, 2)], S=54, B=32, td3=True, discrete=False, T=25, E=5000),
}


def case_of(name, buffer):
    from checkpoint_maddpg_checks import Case
    s = dict(SHAPES[name])
    E = s.pop("E", buffer)
    return Case(s.pop("kind"), s.pop("specs"), S=s.pop("S"), B=s.pop("B"), E=E, rng="device", insert=0, **s)


def timed(one, steps, warmup):
    for _ in range(warmup):
        one()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        one()
    torch.cuda.synchronize()
    return steps / (time.perf_counter() - t0)


def graph_arm(tr, buf, B):
    """The whole-update graph (MaddpgStepGraph): in host noise mode the host draws the noise and copies it in through the graph's
    pinned ring before every replay; in device noise mode the fills run at the head of the graph."""
    from offpolicy._b200.graph import MaddpgStepGraph
    g = MaddpgStepGraph(buf, tr, B)
    return g.launch, g


def fill_ms(tr, B, reps):
    """Device time of one update's fills (every draw of an actor-updating update), from CUDA events; and the MT19937 words they use."""
    draws = tr._noise_draws(B, "policy_0", "target") + tr._noise_draws(B, "policy_0", "actor")
    gen = tr.noise_gen
    for d in draws:
        gen.fill(d)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        for d in draws:
            gen.fill(d)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps, sum(gen.words(d) for d in draws), len(draws)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=500)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--buffer", type=int, default=500_000)
    ap.add_argument("--fill-reps", type=int, default=200)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_maddpg_device_noise: needs a CUDA device")
    torch.set_num_threads(1)
    from offpolicy._b200 import capi
    from offpolicy._b200.torch_rng import DeviceTorchGenerator
    capi.lib()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    for name in a.shapes.split(","):
        case = case_of(name, a.buffer)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side), contextlib.redirect_stdout(sys.stderr):
            tr_h, buf, _ = case.build(1)
            case.fill(buf, np.random.RandomState(2), case.E)
            tr_d, _, _ = case.build(1)
            tr_d.use_device_noise(DeviceTorchGenerator(seed=3))
            arms = {"host": graph_arm(tr_h, buf, case.B), "device": graph_arm(tr_d, buf, case.B)}
            rates = {"host": [], "device": []}
            for _ in range(a.reps):
                for arm in ("host", "device"):
                    rates[arm].append(timed(arms[arm][0], a.steps, a.warmup))
            ms, words, n_fills = fill_ms(tr_d, case.B, a.fill_reps)
            losses = {k: float(t._eng["policy_0"].info[0]) for k, t in (("host", tr_h), ("device", tr_d))}
        assert all(np.isfinite(v) for v in losses.values()), losses
        rec = {"metric": "grad-steps/s", "shape": name, "unit": "steps/s", "batch": case.B, "buffer": case.E, "steps": a.steps,
               "warmup": a.warmup, "host_noise": rates["host"], "device_noise": rates["device"],
               "median_gain": float(np.median(rates["device"]) / np.median(rates["host"])),
               "fills_ms_per_update": ms, "fills_per_update": n_fills, "mt_words_per_update": words,
               "twists_per_update": -(-words // 624), "torch_threads": torch.get_num_threads(), "gpu": card, "last_critic_loss": losses}
        print(json.dumps(rec), flush=True)
        del arms
        torch.cuda.synchronize()


if __name__ == "__main__":
    main()
