"""The MADDPG-family update noise drawn on the device (torch's CPU generator continued in csrc/torch_rng.cu) on the H100: the stream
and the values against torch's, device-mode updates against host-mode updates fed the device draws, the stream position after k
updates, and the captured whole-update graph against eager updates -- at B = 1 000 transitions from 100 000 and at bench.py's
rmatd3_spread shapes.

Worst differences from torch's values measured on an H100 80GB HBM3 at 700 W, in units of the float32 spacing at max(|value|, 1)
(Gumbel) / max(|value|, std) (normal), over the sizes below: Gumbel 1.5, normal 4.0 (the emulated build: 1.0 and 4.0).  The tests hold
them to device_noise_checks.GUMBEL_ULPS / NORMAL_ULPS."""
import pytest

import device_noise_checks as dn
from checkpoint_maddpg_checks import Case

pytestmark = pytest.mark.gpu

SHAPES = [(1, 1, 1, 1), (3, 2, 7, 5), (1, 1, 1, 624), (1, 1, 1, 1249), (26, 3, 32, 5), (1, 3, 1000, 15), (1, 3, 1000, 5)]


@pytest.mark.parametrize("where", ["seeded", "mid_block", "pos_623", "pos_624", "odd_draws"])
def test_uniform_fills_are_torchs_stream(gpu_engine, where):
    dn.check_uniform_stream(where, SHAPES)


@pytest.mark.parametrize("n", [16, 17, 31, 32, 4992, 30000])
def test_gumbel_and_normal_values(gpu_engine, n):
    g = dn.check_transform(gpu_engine.TRNG_GUMBEL, n)
    z = dn.check_transform(gpu_engine.TRNG_NORMAL, n)
    print("n %d: worst Gumbel %.2f ulps, worst normal %.2f ulps" % (n, g, z))


def test_gumbel_at_u_zero(gpu_engine):
    print("u = 0: %.2f ulps" % dn.check_gumbel_at_zero())


def test_bad_fills_are_refused(gpu_engine):
    dn.check_refusals()


BIG = dict(S=54, B=1000, E=100_000, rng="device", insert=0)
UPDATES = {
    "maddpg_spread": Case("mlp", [(3, 18, 5)], **BIG),
    "matd3_spread_per": Case("mlp", [(3, 18, 5)], td3=True, per=True, **BIG),
    "matd3_reference": Case("mlp", [(2, 21, [5, 10])], td3=True, **dict(BIG, S=42)),
    "matd3_box": Case("mlp", [(3, 18, 2)], td3=True, discrete=False, **BIG),
    "rmatd3_spread": Case("rec", [(3, 18, 2)], S=54, B=32, E=5000, T=25, td3=True, discrete=False, rng="device", insert=0),
    "rmatd3_spread_disc": Case("rec", [(3, 18, 5)], S=54, B=32, E=5000, T=25, td3=True, rng="device", insert=0),
    # simple_spread with 5 agents and 5 landmarks: critic input 150 + 25 = 175, above 128 columns (FFMA k_front_fwd / k_front_bwd)
    "matd3_spread5_critic175": Case("mlp", [(5, 30, 5)], td3=True, **dict(BIG, S=150)),
    "rmatd3_spread5_critic175": Case("rec", [(5, 30, 5)], S=150, B=32, E=5000, T=25, td3=True, rng="device", insert=0),
}


@pytest.mark.parametrize("name", sorted(UPDATES))
def test_device_updates_equal_host_updates_fed_the_device_draws(gpu_engine, name):
    dn.check_updates(UPDATES[name], 3)


GRAPH = ["matd3_reference", "matd3_box", "rmatd3_spread", "rmatd3_spread_disc", "matd3_spread5_critic175", "rmatd3_spread5_critic175"]


@pytest.mark.parametrize("name", GRAPH)
def test_graph_launches_equal_eager_device_updates(gpu_engine, name):
    dn.check_graph(UPDATES[name], 5)
