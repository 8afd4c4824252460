"""Recurrent QMIX at SMAC's 27m_vs_30m shape, 36 actions (6 + 30 enemies): the Q-head kernels' two-actions-per-lane instantiation.

Workload: N 27, obs 285, 36 actions, state 1 170, episode 180, batch 32 (get_obs_size / get_state_size of the SMAC env with this
fork's defaults).  A replay of synthetic episodes is sampled on the device.  One JSON line with:
  * grad_steps_per_s: sample -> step -> soft update replayed from one captured CUDA graph (host clock around synchronised launches)
  * kernels_ms: per-kernel device time of one eager step (mx_profile_begin / end: CUDA events around each launch, serialised)
  * oracle_step_s: one step of the CPU oracle (oracle/qmix.py) at the same shape
The card's name, power limit and maximum SM clock are read in the same run.  Needs a CUDA device.

    python tools/bench_qmix_many_actions.py [--steps 30] [--episodes 64]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "off-policy_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

from bench_qmix_wide_state import card, fill  # noqa: E402

SHAPE = ("27m_vs_30m", 27, 285, 36, 1170, 180)


def run(B, steps, episodes):
    import qmix_checks as qc
    import replay_checks as rc
    from oracle.qmix import QmixConfig, QmixLearner, synth_batch
    from offpolicy._b200 import capi
    from offpolicy._b200.graph import StepGraph
    lib = capi.lib()
    name, N, O, A, S, T = SHAPE
    cfg = QmixConfig(n_agents=N, obs_dim=O, act_dim=A, state_dim=S, gain=1.0)
    torch.manual_seed(0)
    buf = rc.make_buffers(N, O, A, S, T, episodes, rng="device", max_batch=max(B, 64))
    fill(buf, cfg, T, episodes)
    buf.seed_device_rng(1)
    args, pol, tr = qc.build_trainer(cfg, B, T, debug=False)
    tr.use_step_graph = False
    tr.train_policy_on_batch(buf.sample(B))
    torch.cuda.synchronize()
    stream = capi.stream_ptr()
    lib.mx_profile_begin(stream)
    tr.train_policy_on_batch(buf.sample(B))
    tr.soft_target_updates()
    names = C.create_string_buffer(1 << 16)
    ms = (C.c_float * 512)()
    n = lib.mx_profile_end(stream, names, len(names), ms, 512)
    split = {}
    for k, v in zip(names.value.decode().split(";")[:n], list(ms)[:n]):
        split[k] = split.get(k, 0.0) + float(v)
    g = StepGraph(buf, tr, B)
    for _ in range(3):
        g.launch()
    g.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        g.launch()
    g.synchronize()
    dt = (time.perf_counter() - t0) / steps
    g.close()
    res = dict(workload=name, B=B, T=T, N=N, obs=O, actions=A, state=S, card=card(), grad_steps_per_s=round(1.0 / dt, 2),
               step_ms=round(dt * 1e3, 3), kernels_ms={k: round(v, 4) for k, v in sorted(split.items(), key=lambda kv: -kv[1])})
    torch.set_num_threads(8)
    L = QmixLearner(cfg, seed=3)
    batch = synth_batch(cfg, B, T, seed=5, avail_p=0.8, var_len=False) + (None, None)
    t0 = time.perf_counter()
    L.step(batch)
    res["oracle_step_s"] = round(time.perf_counter() - t0, 2)
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--episodes", type=int, default=64)
    ap.add_argument("--batch", type=int, default=32)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_qmix_many_actions: needs a CUDA device")
    run(a.batch, a.steps, a.episodes)


if __name__ == "__main__":
    main()
