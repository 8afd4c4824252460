"""The replays at training scale on the real kernels: SMAC-size episodes on both gather paths, transition PER over 100 000 to 500 000
slots at B = 1 000, uniform device draws at the fast path's edges, reward statistics over 20 000 inserts.  Everything is compared with
oracle/replay.py bit for bit (IS weights to rtol 1e-13, normalised rewards to 2e-6) and the statistics with a float64 rescan."""
import numpy as np
import pytest
import torch

import replay_checks as rc
from test_gpu_qmix_schedule import graph_structure

pytestmark = pytest.mark.gpu

# N, O, A, S, T: SMAC 27m_vs_30m, and 3s5z_vs_3s6z with the global state (--use_global_all_local_state)
SMAC = {"27m_vs_30m": (27, 285, 36, 1170, 180), "3s5z_vs_3s6z": (8, 268, 15, 2374, 170)}
E_SMAC = 40


def gather_kernels(pb, B):
    """Names of the gather kernels one device-drawn sample of B episodes launches: both paths launch under the name k_gather, so
    the sample is captured as a CUDA graph and its kernel nodes are read by function."""
    pb.sample_device_uniform(B)              # first launches (shared-memory attributes) outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph(keep_graph=True)
    with torch.cuda.graph(g):
        pb.sample_device_uniform(B)
    try:
        nodes, _ = graph_structure(g.raw_cuda_graph())
    finally:
        g.reset()
        torch.cuda.synchronize()
    return [n for n in nodes if n.startswith("k_gather")]


@pytest.fixture(scope="module", params=sorted(SMAC))
def smac_replay(request, gpu_engine):
    buf, ora = rc.fill_smac_replay(SMAC[request.param], E_SMAC, max_batch=32)
    buf.policy_buffers["policy_0"].seed_device_rng(1)     # for the captured device draws; buf.sample() keeps drawing on the host
    yield request.param, buf, ora
    del buf, ora
    torch.cuda.empty_cache()


def test_smac_episodes_both_gather_paths(gpu_engine, smac_replay):
    """Capacity 40, 51 episodes inserted (the ring wraps), avail masks and reward normalisation on.  Every sample is drawn on the host,
    gathered by the automatic path choice and again with gather_tma = 2 (TMA at any size), and compared with the oracle field by
    field; both paths return identical rewards.  The launcher's rule (TMA while bytes_per_episode x B <= 96 MB) is restated from the
    layout, and the kernel each choice launches is read from a captured sample.  At 3s5z_vs_3s6z B = 30 and 31 sit on either side of
    the switch; 27m_vs_30m's obs field ends in a 224-word partial line, 3s5z_vs_3s6z's acts field (85 lines) has none."""
    name, buf, ora = smac_replay
    lib = gpu_engine.lib()
    pb = buf.policy_buffers["policy_0"]
    per_ep = rc.episode_bytes(pb)
    L = pb.L
    if name == "3s5z_vs_3s6z":
        assert per_ep == 3283280 and int(L.ep_acts) % 256 == 0 and int(L.ep_obs) % 256 == 32
        Bs = (30, 31, 32)
        assert rc.TMA_GATHER_LIMIT // per_ep == 30
    else:
        assert per_ep == 7940960 and int(L.ep_obs) % 256 == 224
        Bs = (32,)
    seen = {}
    for B in Bs:
        rew = []
        for mode in (1, 2):
            lib.mx_set_option(b"gather_tma", mode)
            try:
                rew.append(rc.check_sample_vs_oracle(buf, ora, B, seed=100 + B))
                tma = mode == 2 or per_ep * B <= rc.TMA_GATHER_LIMIT
                ks = gather_kernels(pb, B)
                seen[(B, "auto" if mode == 1 else "gather_tma=2")] = ks
                assert ks == (["k_gather_tma"] if tma else ["k_gather"]), (B, mode, ks)
            finally:
                lib.mx_set_option(b"gather_tma", 1)
        assert np.array_equal(rew[0], rew[1])
    print("\n%s: %d bytes per episode; gather kernel per (B, choice): %s" % (name, per_ep, seen))


@pytest.mark.parametrize("E,spec,rng", [
    (500000, (1, 1, 1, 1), "device"), (500000, (1, 1, 1, 1), "numpy"),
    (131072, (1, 1, 1, 1), "device"), (131073, (1, 1, 1, 1), "numpy"),
    (100000, (3, 18, 54, 5), "device"),                 # simple_spread: 3 agents, obs 18, state 54, 5 actions
])
def test_per_transitions_at_scale(gpu_engine, E, spec, rng):
    worst, dup = rc.check_per_transitions_vs_oracle(E, spec, rounds=100, rng=rng)
    print("\nE %d %s %s: worst IS weight error %.2e (rtol), most repeats of one index in a draw %d" % (E, spec, rng, worst, dup))


def test_per_transition_policies_at_scale(gpu_engine):
    rc.check_per_transition_policies(131073, rounds=10)


@pytest.mark.parametrize("E", [2 ** k + j for k in (16, 19) for j in (-1, 0, 1)])
def test_device_rng_stream_fast_path_edges(gpu_engine, E):
    rc.check_device_rng_stream(seed=77, E=E, B=(255, 256, 257, 1000, 1024), rounds=3, starts=(None, 367, 368, 369),
                               dims=(1, 1, 1, 1, 1))


@pytest.mark.parametrize("loc,scale,vs_oracle", [(-1.5, 0.7, True), (1e3, 1e-2, False)])
def test_reward_stats_long_run(gpu_engine, loc, scale, vs_oracle):
    worst = rc.check_reward_stats_long_run(loc, scale, vs_oracle=vs_oracle)
    print("\nrewards N(%g, %g): worst reward-statistics error (mean, std) %.2f, %.2f fp32 ulps" % (loc, scale, worst[0], worst[1]))
