"""Where the time of a tools/bench_mlp_maddpg.py update goes, for both shapes (simple_spread, simple_reference) and both algorithms,
alternating the shapes and repeating three times in one process: `graph_ms` is the captured whole-update graph replayed alone (noise
buffers left as they are), `host_ms` the host noise draws from torch's CPU generator and their copies through the graph's pinned ring
alone, `full_ms` both (MaddpgStepGraph.launch), as the benchmark runs them.  Then a per-kernel breakdown of eager MADDPG steps under
torch.profiler (a separate, traced run).  Needs a CUDA device; prints JSON lines.

    python tools/bench_mlp_maddpg_split.py
"""
import json
import os
import sys
import time

import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "off-policy_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]
import bench_mlp_maddpg as bm


def setup(shape, td3, B=1000, size=500_000):
    bm.set_shape(shape)
    from offpolicy._b200.factory import build_mlp_maddpg, act_space, Box
    from offpolicy._b200.graph import MaddpgStepGraph
    from offpolicy.utils.mlp_buffer import MlpReplayBuffer
    torch.manual_seed(1)
    act = bm.A if bm.SEGS is None else bm.SEGS
    args, pol, tr = build_mlp_maddpg(bm.N, bm.O, act, bm.S, B, discrete=True, td3=td3)
    info = {"policy_0": dict(obs_space=Box(bm.O), share_obs_space=Box(bm.S), act_space=act_space(act))}
    buf = MlpReplayBuffer(info, {"policy_0": list(range(bm.N))}, size, True, False, max_batch=B)
    bm.fill(buf, B, size, np.random.default_rng(2))
    buf.seed_device_rng(3)
    return tr, MaddpgStepGraph(buf, tr, B), buf


def timed(fn, n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n * 1e3


def main():
    if not torch.cuda.is_available():
        raise SystemExit("bench_mlp_maddpg_split: needs a CUDA device")
    from offpolicy._b200 import capi
    B = 1000
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        ctx = {}
        for shape in ("spread", "reference"):
            bm.N, bm.O, bm.A, bm.S, bm.SEGS = 3, 18, 5, 54, None
            for td3 in (False, True):
                bm.N, bm.O, bm.A, bm.S, bm.SEGS = 3, 18, 5, 54, None
                ctx[(shape, td3)] = (setup(shape, td3), (bm.N, bm.O, bm.A, bm.S, bm.SEGS))
        for rep in range(3):
            for shape in ("spread", "reference"):
                for td3 in (False, True):
                    (tr, g, buf), dims = ctx[(shape, td3)]
                    bm.N, bm.O, bm.A, bm.S, bm.SEGS = dims
                    launch = lambda: capi.check(g.lib.mx_graph_launch(g.graphs[1], g._sp))
                    host = lambda: g._stage_noise(1)
                    for _ in range(50):
                        g.launch()
                    r = dict(rep=rep, shape=shape, algo="matd3" if td3 else "maddpg", graph_ms=timed(launch, 500), host_ms=timed(host, 200),
                             full_ms=timed(g.launch, 500))
                    print(json.dumps(r), flush=True)
        # per-kernel breakdown of one replay batch each, eager step under the profiler
        from torch.profiler import profile, ProfilerActivity
        for shape in ("spread", "reference"):
            (tr, g, buf), dims = ctx[(shape, False)]
            bm.N, bm.O, bm.A, bm.S, bm.SEGS = dims
            for _ in range(5):
                tr.shared_train_policy_on_batch("policy_0", buf.sample(B))
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
                for _ in range(20):
                    tr.shared_train_policy_on_batch("policy_0", buf.sample(B))
                torch.cuda.synchronize()
            ev = {}
            for e in prof.key_averages():
                t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                if t and e.key.startswith("k_"):
                    ev[e.key] = round(t / 20, 2)
            print(json.dumps({"shape": shape, "kernels_us_per_step": dict(sorted(ev.items(), key=lambda kv: -kv[1])[:16]),
                              "sum_us": round(sum(ev.values()), 1)}), flush=True)


if __name__ == "__main__":
    main()
