"""The MADDPG-family update noise drawn on the device (torch's CPU generator continued in csrc/torch_rng.cu) on the CPU fiber
emulator: the stream and the values against torch's, the learner layout, the updates, the captured graph, the checkpoint and the
refusals."""
import pytest

import device_noise_checks as dn
from checkpoint_maddpg_checks import Case

SHAPES = [(1, 1, 1, 1), (1, 2, 3, 5), (3, 2, 7, 5), (1, 1, 1, 624), (1, 1, 1, 1249), (5, 3, 8, 5), (26, 3, 32, 5)]


@pytest.mark.parametrize("where", ["seeded", "mid_block", "pos_623", "pos_624", "odd_draws"])
def test_uniform_fills_are_torchs_stream(emu_engine, where):
    dn.check_uniform_stream(where, SHAPES)


@pytest.mark.parametrize("n", [16, 17, 31, 32, 4992, 30000])
def test_gumbel_and_normal_values(emu_engine, n):
    g = dn.check_transform(emu_engine.TRNG_GUMBEL, n)
    z = dn.check_transform(emu_engine.TRNG_NORMAL, n)
    print("n %d: worst Gumbel %.2f ulps, worst normal %.2f ulps" % (n, g, z))


def test_gumbel_at_u_zero(emu_engine):
    print("u = 0: %.2f ulps" % dn.check_gumbel_at_zero())


def test_bad_fills_are_refused(emu_engine):
    dn.check_refusals()


LAYOUT = {
    "rmaddpg_discrete": Case("rec", [(2, 6, 4)], S=8, B=4, E=8, T=4),
    "rmatd3_box": Case("rec", [(2, 6, 2)], S=8, B=4, E=8, T=4, td3=True, discrete=False),
    "rmatd3_discrete_avail": Case("rec", [(2, 6, 4)], S=8, B=4, E=8, T=4, td3=True, avail=True),
    "maddpg_discrete": Case("mlp", [(3, 6, 5)], S=10, B=8, E=40),
    "matd3_box": Case("mlp", [(2, 6, 2)], S=10, B=8, E=40, td3=True, discrete=False),
    "matd3_multidiscrete": Case("mlp", [(2, 8, [3, 4])], S=10, B=8, E=40, td3=True),
    "matd3_speaker_listener": Case("mlp", [(1, 3, 3), (1, 11, 5)], S=14, B=8, E=40, td3=True),
}


@pytest.mark.parametrize("name", sorted(LAYOUT))
def test_device_draws_land_where_host_draws_land(emu_engine, name):
    dn.check_layout(LAYOUT[name])


UPDATES = {
    "rmaddpg_discrete": Case("rec", [(2, 6, 4)], S=8, B=4, E=8, T=4, rng="device"),
    "rmatd3_box_per": Case("rec", [(2, 6, 2)], S=8, B=4, E=8, T=4, td3=True, discrete=False, per=True, rng="device"),
    "rmatd3_discrete_avail": Case("rec", [(2, 6, 4)], S=8, B=4, E=8, T=4, td3=True, avail=True, rng="device"),
    "maddpg_discrete_per": Case("mlp", [(3, 6, 5)], S=10, B=8, E=40, per=True, rng="device"),
    "matd3_box": Case("mlp", [(2, 6, 2)], S=10, B=8, E=40, td3=True, discrete=False, rng="device"),
    "matd3_multidiscrete": Case("mlp", [(2, 8, [3, 4])], S=10, B=8, E=40, td3=True, rng="device"),
    "matd3_speaker_listener": Case("mlp", [(1, 3, 3), (1, 11, 5)], S=14, B=8, E=40, td3=True, rng="device"),
}


@pytest.mark.parametrize("name", sorted(UPDATES))
def test_device_updates_equal_host_updates_fed_the_device_draws(emu_engine, name):
    dn.check_updates(UPDATES[name], 3)


@pytest.mark.parametrize("case", [Case("rec", [(2, 6, 3)], S=8, B=4, E=9, T=4, td3=True, rng="device"),
                                  Case("mlp", [(2, 8, [3, 4])], S=10, B=8, E=40, td3=True, rng="device")],
                         ids=["rmatd3_discrete", "matd3_multidiscrete"])
def test_graph_launches_equal_eager_device_updates(emu_engine, case):
    dn.check_graph(case, 4)


@pytest.mark.parametrize("case", [Case("rec", [(2, 6, 4)], S=8, B=4, E=9, T=4, td3=True, insert=1),
                                  Case("mlp", [(2, 6, 2)], S=10, B=8, E=40, td3=True, discrete=False, per=True, rng="device", insert=4)],
                         ids=["rmatd3_discrete", "matd3_box_per"])
def test_device_mode_checkpoint_resumes_bit_identically(emu_engine, case):
    dn.check_checkpoint(case, 2)
