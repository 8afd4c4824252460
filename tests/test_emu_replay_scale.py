"""Training-scale replay checks (tests/test_gpu_replay_scale.py) on the CPU fiber emulator: the same kernels, the uniform draws at the
device sizes, the rest reduced -- PER trees of 2^12 to 2^13 leaves with draws of 1 000, 3 000 inserts into a ring of 300, an episode
shape whose fields span several 8 KB boxes (the emulator has no TMA: its gather is k_gather)."""
import pytest

import replay_checks as rc

TINY = (1, 1, 1, 1, 1)     # N, O, A, S, T: index draws only, the episodes' contents do not matter


@pytest.mark.parametrize("E", [2 ** k + j for k in (16, 19) for j in (-1, 0, 1)])
def test_device_rng_stream_fast_path_edges(emu_engine, E):
    rc.check_device_rng_stream(seed=77, E=E, B=(255, 256, 257, 1000, 1024), rounds=3, starts=(None, 367, 368, 369), dims=TINY)


@pytest.mark.parametrize("E,rng", [(4097, "device"), (4096, "numpy"), (2 ** 12 + 2 ** 11, "device")])
def test_per_transitions_vs_oracle(emu_engine, E, rng):
    rc.check_per_transitions_vs_oracle(E, rounds=30, rng=rng, gap=1000)


def test_per_transition_policies(emu_engine):
    rc.check_per_transition_policies(3000, rounds=3)


@pytest.mark.parametrize("loc,scale,vs_oracle", [(-1.5, 0.7, True), (1e3, 1e-2, False)])
def test_reward_stats_long_run(emu_engine, loc, scale, vs_oracle):
    worst = rc.check_reward_stats_long_run(loc, scale, E=300, inserts=3000, every=100, vs_oracle=vs_oracle)
    print("worst reward-statistics error (mean, std) in fp32 ulps:", worst)


def test_multi_box_episodes_vs_oracle(emu_engine):
    # obs 41 x 4 x 132 words = 84 lines of 1 KB (11 boxes of 8 KB, the last one clipped) + a 144-word tail; acts 40 x 4 x 16 = 10 lines
    # exactly, no partial line
    buf, ora = rc.fill_smac_replay((4, 130, 13, 300, 40), E=12, max_batch=8, chunk=5)
    for B in (1, 7, 8):
        rc.check_sample_vs_oracle(buf, ora, B, seed=B)
