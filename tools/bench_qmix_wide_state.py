"""Recurrent QMIX at SMAC global-all-local state shapes (the wide-state mixer path): one JSON line per workload.

Workloads: 3s5z_vs_3s6z with --use_global_all_local_state (train_smac_qmix.sh: N 8, obs 268, 15 actions, state 2 374, episode 170,
batch 32) and 8m with the same flag (N 8, obs 204, 14 actions, state 1 800, episode 120).  A replay of synthetic episodes (the full
3s5z_vs_3s6z episode is ~3.3 MB) is sampled on the device.  Reports:
  * grad_steps_per_s: sample -> step -> soft update replayed from one captured CUDA graph (host clock around synchronised launches)
  * kernels_ms: per-kernel device time of one eager step (mx_profile_begin / end: CUDA events around each launch, serialised)
  * state_layers: FLOPs of the state-layer GEMMs (3 TF32 products per multiply-add, counted as issued) and their rate against the
    data-sheet dense TF32 rate of the H100 SXM (495 TFLOP/s at 700 W)
  * oracle_step_s: one step of the CPU oracle (oracle/qmix.py) at the same shape
The card's name and power limit are read in the same run.  Needs a CUDA device.

    python tools/bench_qmix_wide_state.py [--steps 30] [--episodes 96]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "off-policy_b200"), os.path.join(ROOT, "tests")]

SHAPES = {"3s5z_vs_3s6z_global": (8, 268, 15, 2374, 170), "8m_global": (8, 204, 14, 1800, 120)}
TF32_DENSE = 495e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def fill(buf, cfg, T, E, seed=0):
    import replay_checks as rc
    rs = np.random.RandomState(seed)
    N, O, A, S = cfg.n_agents, cfg.obs_dim, cfg.act_dim, cfg.state_dim
    for c in range(0, E, 8):
        n = min(8, E - c)
        av = (rs.rand(T + 1, n, N, A) < 0.7) * 1.0
        av[..., 0] = 1.0
        ep = [rs.randn(T + 1, n, N, O), np.repeat(rs.randn(T + 1, n, 1, S), N, 2), np.eye(A)[rs.randint(0, A, (T, n, N))],
              np.repeat(rs.randn(T, n, 1, 1), N, 2), np.zeros((T, n, N, 1)), np.zeros((T, n, 1)), av]
        buf.insert(n, *[rc.d(x.astype(np.float32)) for x in ep])


def state_layer_flops(cfg, B, T):
    HY, ME, N, S = cfg.hyper_hidden, cfg.mixer_hidden, cfg.n_agents, cfg.state_dim
    C_ = 3 * HY + ME if cfg.hyper_layers == 2 else N * ME + 2 * ME + HY
    fwd = 2.0 * 2 * C_ * S * B * (T + 1)        # live + target over every state row
    wgrad = 2.0 * C_ * S * B * T
    return fwd, wgrad


def run(name, B, steps, episodes):
    import qmix_checks as qc
    import replay_checks as rc
    from oracle.qmix import QmixConfig, synth_batch
    from offpolicy._b200 import capi
    from offpolicy._b200.graph import StepGraph
    lib = capi.lib()
    N, O, A, S, T = SHAPES[name]
    cfg = QmixConfig(n_agents=N, obs_dim=O, act_dim=A, state_dim=S, gain=1.0)
    torch.manual_seed(0)
    buf = rc.make_buffers(N, O, A, S, T, episodes, rng="device", max_batch=max(B, 64))
    fill(buf, cfg, T, episodes)
    buf.seed_device_rng(1)
    args, pol, tr = qc.build_trainer(cfg, B, T, debug=False)
    # per-kernel split of one eager step (serialised by the profiler; the trainer's own step graph would hide the kernels)
    tr.use_step_graph = False
    smp = buf.sample(B)
    tr.train_policy_on_batch(smp)
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
    # the whole step as a graph
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
    fwd, wgrad = state_layer_flops(cfg, B, T)
    t_fwd, t_wg = split.get("k_mixw_fwd", 0.0) * 1e-3, split.get("k_mixw_wgrad", 0.0) * 1e-3
    res = dict(workload=name, B=B, T=T, N=N, obs=O, state=S, card=card(), grad_steps_per_s=round(1.0 / dt, 2), step_ms=round(dt * 1e3, 3),
               kernels_ms={k: round(v, 4) for k, v in sorted(split.items(), key=lambda kv: -kv[1])},
               state_layers=dict(fwd_gflop=round(fwd / 1e9, 3), wgrad_gflop=round(wgrad / 1e9, 3),
                                 fwd_tflops_3xtf32=round(3 * fwd / t_fwd / 1e12, 2) if t_fwd else None,
                                 wgrad_tflops_3xtf32=round(3 * wgrad / t_wg / 1e12, 2) if t_wg else None,
                                 fwd_share_of_tf32_peak=round(3 * fwd / t_fwd / TF32_DENSE, 4) if t_fwd else None,
                                 wgrad_share_of_tf32_peak=round(3 * wgrad / t_wg / TF32_DENSE, 4) if t_wg else None))
    # CPU oracle at the same shape: one step
    from oracle.qmix import QmixLearner
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
    ap.add_argument("--episodes", type=int, default=96)
    ap.add_argument("--batch", type=int, default=32)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_qmix_wide_state: needs a CUDA device")
    for name in SHAPES:
        run(name, a.batch, a.steps, a.episodes)


if __name__ == "__main__":
    main()
