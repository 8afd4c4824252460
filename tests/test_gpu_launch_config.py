"""Launch configurations on the device: every kernel node of a captured step with its grid, block and dynamic shared memory, and the
dependency edges with their types (programmatic dependent launch edges included).

tests/test_gpu_qmix_schedule.py pins which kernels a QMIX-family step runs and how they depend on each other; this module pins how
each of them is launched, for those steps and for the actor-critic updates: R-MADDPG and R-MATD3 at the bench.py rmaddpg_spread /
rmatd3_spread shapes and one MLP MADDPG update in device-noise mode.  The actor-critic updates are captured in device-noise mode where
they take noise (a host draw would be copied in from pageable memory, which a capture refuses); R-MATD3's graph holds two updates, the
actor update on and off.  Each configuration below was recorded on an H100 80GB HBM3 (132 SMs; the grids follow the SM count) from
the launchers as they stood before they were put on one launch function (mx_launch)."""
import ctypes as C

import numpy as np
import pytest
import torch

import test_gpu_qmix_schedule as qs

pytestmark = pytest.mark.gpu

# name: (Case, device noise, updates captured) -- the R-MADDPG / R-MATD3 shapes of bench.py's rmaddpg_spread / rmatd3_spread
MADDPG = {
    "rmaddpg_spread": (dict(kind="rec", specs=[(3, 18, 2)], S=54, B=32, E=64, T=25, discrete=False), False, 1),
    "rmatd3_spread": (dict(kind="rec", specs=[(3, 18, 2)], S=54, B=32, E=64, T=25, td3=True, discrete=False), True, 2),
    "mlp_maddpg_device_noise": (dict(kind="mlp", specs=[(3, 18, 5)], S=54, B=256, E=1024), True, 1),
}

EXPECTED = {
    "mlp_maddpg_device_noise": (
        [
            "k_act_transform grid=(6, 1, 1) block=(256, 1, 1) smem=0",
            "k_act_transform grid=(6, 1, 1) block=(256, 1, 1) smem=0",
            "k_actor_loss grid=(1, 1, 1) block=(256, 1, 1) smem=0",
            "k_adam grid=(4, 1, 1) block=(1024, 1, 1) smem=0",
            "k_adam grid=(9, 1, 1) block=(1024, 1, 1) smem=0",
            "k_critic_loss grid=(1, 1, 1) block=(256, 1, 1) smem=0",
            "k_front_bwd<2> grid=(24, 1, 1) block=(256, 1, 1) smem=140560",
            "k_front_bwd<2> grid=(48, 1, 1) block=(256, 1, 1) smem=115472",
            "k_front_bwd_tc grid=(2, 1, 1) block=(128, 1, 1) smem=204800",
            "k_front_fwd<2> grid=(24, 1, 1) block=(256, 1, 1) smem=29184",
            "k_front_fwd<2> grid=(8, 1, 1) block=(256, 1, 1) smem=29184",
            "k_front_fwd<2> grid=(8, 1, 1) block=(256, 1, 1) smem=29184",
            "k_front_fwd_tc2 grid=(12, 2, 1) block=(256, 1, 1) smem=208896",
            "k_grad_reduce grid=(140, 1, 1) block=(256, 1, 1) smem=0",
            "k_grad_reduce grid=(54, 1, 1) block=(256, 1, 1) smem=0",
            "k_mlp_dgi_cols grid=(192, 1, 1) block=(256, 1, 1) smem=0",
            "k_mlp_dgi_cols grid=(528, 1, 1) block=(256, 1, 1) smem=0",
            "k_mlp_head_cols grid=(1, 1, 1) block=(256, 1, 1) smem=0",
            "k_mlp_head_cols grid=(1, 1, 1) block=(256, 1, 1) smem=0",
            "k_mlp_head_cols grid=(3, 1, 1) block=(256, 1, 1) smem=0",
            "k_mlp_head_cols grid=(6, 1, 1) block=(256, 1, 1) smem=0",
            "k_mlp_head_cols grid=(6, 1, 1) block=(256, 1, 1) smem=0",
            "k_pack_critic_in grid=(216, 1, 1) block=(256, 1, 1) smem=0",
            "k_pack_critic_in grid=(72, 1, 1) block=(256, 1, 1) smem=0",
            "k_pack_critic_in grid=(72, 1, 1) block=(256, 1, 1) smem=0",
            "k_scatter_actor_grad grid=(6, 1, 1) block=(256, 1, 1) smem=0",
            "k_set_scalars grid=(1, 1, 1) block=(32, 1, 1) smem=0",
            "k_set_scalars grid=(1, 1, 1) block=(32, 1, 1) smem=0",
            "k_tc_prep_weights_T grid=(84, 1, 1) block=(256, 1, 1) smem=0",
            "k_trng_fill grid=(15, 1, 1) block=(256, 1, 1) smem=0",
            "k_trng_twist grid=(1, 1, 1) block=(256, 1, 1) smem=0",
            "k_wgrad_tc grid=(4, 1, 1) block=(512, 1, 1) smem=147456",
        ],
        [
            "k_act_transform -> k_pack_critic_in",
            "k_act_transform -> k_pack_critic_in",
            "k_actor_loss -> k_mlp_dgi_cols",
            "k_adam -> k_mlp_head_cols",
            "k_critic_loss -> k_mlp_dgi_cols",
            "k_front_bwd<2> -> k_grad_reduce [1,0,1]",
            "k_front_bwd<2> -> k_scatter_actor_grad",
            "k_front_bwd_tc -> k_wgrad_tc [1,0,1]",
            "k_front_fwd<2> -> k_front_fwd<2> [1,0,1]",
            "k_front_fwd<2> -> k_mlp_head_cols",
            "k_front_fwd<2> -> k_mlp_head_cols",
            "k_front_fwd_tc2 -> k_mlp_head_cols",
            "k_grad_reduce -> k_set_scalars",
            "k_grad_reduce -> k_set_scalars",
            "k_mlp_dgi_cols -> k_front_bwd<2> [1,0,1]",
            "k_mlp_dgi_cols -> k_tc_prep_weights_T [1,0,1]",
            "k_mlp_head_cols -> k_act_transform",
            "k_mlp_head_cols -> k_act_transform",
            "k_mlp_head_cols -> k_actor_loss",
            "k_mlp_head_cols -> k_critic_loss",
            "k_mlp_head_cols -> k_mlp_head_cols",
            "k_pack_critic_in -> k_front_fwd<2>",
            "k_pack_critic_in -> k_front_fwd<2> [1,0,1]",
            "k_pack_critic_in -> k_pack_critic_in",
            "k_scatter_actor_grad -> k_front_bwd<2> [1,0,1]",
            "k_set_scalars -> k_adam [1,0,1]",
            "k_set_scalars -> k_adam [1,0,1]",
            "k_tc_prep_weights_T -> k_front_bwd_tc [1,0,1]",
            "k_trng_fill -> k_front_fwd_tc2",
            "k_trng_twist -> k_trng_fill",
            "k_wgrad_tc -> k_grad_reduce [1,0,1]",
        ]),
    "mqmix_mpe_spread": (
        [
            "k_front_bwd<3> grid=(125, 1, 1) block=(256, 1, 1) smem=163216",
            "k_front_fwd_tc2 grid=(47, 2, 1) block=(256, 1, 1) smem=208896",
            "k_mix_core grid=(63, 1, 1) block=(512, 1, 1) smem=0",
            "k_mix_hyper_bwd<1,0> grid=(63, 1, 1) block=(256, 1, 1) smem=58896",
            "k_mix_hyper_fwd<1,0> grid=(63, 2, 1) block=(256, 1, 1) smem=58896",
            "k_mlp_dgi grid=(1056, 1, 1) block=(256, 1, 1) smem=0",
            "k_mlp_qselect grid=(12, 1, 1) block=(256, 1, 1) smem=0",
            "k_optim_fused grid=(221, 1, 1) block=(256, 1, 1) smem=0",
            "k_tc_prep_weights grid=(70, 2, 1) block=(256, 1, 1) smem=0",
        ],
        [
            "k_front_bwd<3> -> k_optim_fused [1,0,1]",
            "k_front_fwd_tc2 -> k_mlp_qselect [1,0,1]",
            "k_mix_core -> k_mix_hyper_bwd<1,0> [1,0,1]",
            "k_mix_core -> k_mlp_dgi [1,0,1]",
            "k_mix_hyper_bwd<1,0> -> k_optim_fused [1,0,1]",
            "k_mix_hyper_fwd<1,0> -> k_mix_core [1,0,1]",
            "k_mix_hyper_fwd<1,0> -> k_mix_hyper_bwd<1,0> [1,0,1]",
            "k_mlp_dgi -> k_front_bwd<3> [1,0,1]",
            "k_mlp_qselect -> k_mix_core [1,0,1]",
            "k_tc_prep_weights -> k_front_fwd_tc2 [1,0,1]",
            "k_tc_prep_weights -> k_mix_hyper_fwd<1,0> [1,0,1]",
        ]),
    "qmix_2s3z": (
        [
            "k_front_bwd_tc grid=(152, 1, 1) block=(128, 1, 1) smem=106496",
            "k_front_fwd_tc_wide2 grid=(132, 2, 1) block=(128, 1, 1) smem=98304",
            "k_gru_bwd2<1> grid=(160, 1, 1) block=(128, 1, 1) smem=0",
            "k_gru_fwd2<1> grid=(160, 2, 1) block=(128, 1, 1) smem=0",
            "k_mid<16,1> grid=(132, 1, 1) block=(512, 1, 1) smem=178064",
            "k_mix_hyper_bwd<2,0> grid=(120, 1, 1) block=(256, 1, 1) smem=133136",
            "k_mix_hyper_fwd<2,0> grid=(120, 2, 1) block=(256, 1, 1) smem=133136",
            "k_optim_fused grid=(312, 1, 1) block=(256, 1, 1) smem=0",
            "k_tc_prep_weights grid=(84, 2, 1) block=(256, 1, 1) smem=0",
            "k_tc_prep_weights_T grid=(84, 1, 1) block=(256, 1, 1) smem=0",
            "k_wgrad_tc grid=(132, 1, 1) block=(512, 1, 1) smem=147456",
        ],
        [
            "k_front_bwd_tc -> k_wgrad_tc",
            "k_front_fwd_tc_wide2 -> k_gru_fwd2<1>",
            "k_gru_bwd2<1> -> k_front_bwd_tc",
            "k_gru_fwd2<1> -> k_mid<16,1>",
            "k_mid<16,1> -> k_gru_bwd2<1>",
            "k_mid<16,1> -> k_mix_hyper_bwd<2,0>",
            "k_mix_hyper_bwd<2,0> -> k_optim_fused",
            "k_mix_hyper_fwd<2,0> -> k_mid<16,1>",
            "k_mix_hyper_fwd<2,0> -> k_mix_hyper_bwd<2,0>",
            "k_tc_prep_weights -> k_tc_prep_weights_T",
            "k_tc_prep_weights_T -> k_front_fwd_tc_wide2",
            "k_tc_prep_weights_T -> k_mix_hyper_fwd<2,0>",
            "k_wgrad_tc -> k_optim_fused",
        ]),
    "qmix_3m": (
        [
            "k_front_bwd<3> grid=(122, 1, 1) block=(256, 1, 1) smem=137104",
            "k_front_fwd_tc2 grid=(46, 2, 1) block=(256, 1, 1) smem=212992",
            "k_gru_bwd2<1> grid=(96, 1, 1) block=(128, 1, 1) smem=0",
            "k_gru_fwd2<1> grid=(96, 2, 1) block=(128, 1, 1) smem=0",
            "k_gru_wgrad<3> grid=(122, 1, 1) block=(256, 1, 1) smem=77712",
            "k_mid<16,1> grid=(120, 1, 1) block=(512, 1, 1) smem=133008",
            "k_mix_hyper_bwd<1,0> grid=(120, 1, 1) block=(256, 1, 1) smem=58896",
            "k_mix_hyper_fwd<1,0> grid=(120, 2, 1) block=(256, 1, 1) smem=58896",
            "k_optim_fused grid=(219, 1, 1) block=(256, 1, 1) smem=0",
            "k_tc_prep_weights grid=(72, 2, 1) block=(256, 1, 1) smem=0",
        ],
        [
            "k_front_bwd<3> -> k_optim_fused [1,0,1]",
            "k_front_fwd_tc2 -> k_gru_fwd2<1> [1,0,1]",
            "k_gru_bwd2<1> -> k_front_bwd<3> [1,0,1]",
            "k_gru_bwd2<1> -> k_gru_wgrad<3> [1,0,1]",
            "k_gru_fwd2<1> -> k_mid<16,1> [1,0,1]",
            "k_gru_wgrad<3> -> k_optim_fused [1,0,1]",
            "k_mid<16,1> -> k_gru_bwd2<1> [1,0,1]",
            "k_mid<16,1> -> k_mix_hyper_bwd<1,0> [1,0,1]",
            "k_mix_hyper_bwd<1,0> -> k_gru_wgrad<3> [1,0,1]",
            "k_mix_hyper_fwd<1,0> -> k_mid<16,1> [1,0,1]",
            "k_mix_hyper_fwd<1,0> -> k_mix_hyper_bwd<1,0> [1,0,1]",
            "k_tc_prep_weights -> k_front_fwd_tc2 [1,0,1]",
            "k_tc_prep_weights -> k_mix_hyper_fwd<1,0> [1,0,1]",
        ]),
    "qmix_8m_per": (
        [
            "k_front_bwd_tc grid=(264, 1, 1) block=(128, 1, 1) smem=106496",
            "k_front_fwd_tc_wide2 grid=(132, 2, 1) block=(128, 1, 1) smem=98304",
            "k_gru_bwd2<1> grid=(512, 1, 1) block=(128, 1, 1) smem=0",
            "k_gru_fwd2<1> grid=(512, 2, 1) block=(128, 1, 1) smem=0",
            "k_mid<8,1> grid=(132, 1, 1) block=(256, 1, 1) smem=131920",
            "k_mix_hyper_bwd<2,0> grid=(132, 1, 1) block=(256, 1, 1) smem=165904",
            "k_mix_hyper_fwd<2,0> grid=(132, 2, 1) block=(256, 1, 1) smem=165904",
            "k_optim_fused grid=(379, 1, 1) block=(256, 1, 1) smem=0",
            "k_tc_prep_weights grid=(84, 2, 1) block=(256, 1, 1) smem=0",
            "k_tc_prep_weights_T grid=(84, 1, 1) block=(256, 1, 1) smem=0",
            "k_wgrad_tc grid=(132, 1, 1) block=(512, 1, 1) smem=147456",
        ],
        [
            "k_front_bwd_tc -> k_wgrad_tc",
            "k_front_fwd_tc_wide2 -> k_gru_fwd2<1>",
            "k_gru_bwd2<1> -> k_front_bwd_tc",
            "k_gru_fwd2<1> -> k_mid<8,1>",
            "k_mid<8,1> -> k_gru_bwd2<1>",
            "k_mid<8,1> -> k_mix_hyper_bwd<2,0>",
            "k_mix_hyper_bwd<2,0> -> k_optim_fused",
            "k_mix_hyper_fwd<2,0> -> k_mid<8,1>",
            "k_mix_hyper_fwd<2,0> -> k_mix_hyper_bwd<2,0>",
            "k_tc_prep_weights -> k_tc_prep_weights_T",
            "k_tc_prep_weights_T -> k_front_fwd_tc_wide2",
            "k_tc_prep_weights_T -> k_mix_hyper_fwd<2,0>",
            "k_wgrad_tc -> k_optim_fused",
        ]),
    "qmix_mpe_spread": (
        [
            "k_front_bwd<2> grid=(78, 1, 1) block=(256, 1, 1) smem=98064",
            "k_front_fwd_tc2 grid=(20, 2, 1) block=(256, 1, 1) smem=208896",
            "k_gru_bwd2<1> grid=(96, 1, 1) block=(128, 1, 1) smem=0",
            "k_gru_fwd2<1> grid=(96, 2, 1) block=(128, 1, 1) smem=0",
            "k_gru_wgrad<2> grid=(78, 1, 1) block=(256, 1, 1) smem=51984",
            "k_mid<16,1> grid=(50, 1, 1) block=(512, 1, 1) smem=116624",
            "k_mix_hyper_bwd<1,0> grid=(50, 1, 1) block=(256, 1, 1) smem=58896",
            "k_mix_hyper_fwd<1,0> grid=(50, 2, 1) block=(256, 1, 1) smem=58896",
            "k_optim_fused grid=(221, 1, 1) block=(256, 1, 1) smem=0",
            "k_tc_prep_weights grid=(70, 2, 1) block=(256, 1, 1) smem=0",
        ],
        [
            "k_front_bwd<2> -> k_optim_fused [1,0,1]",
            "k_front_fwd_tc2 -> k_gru_fwd2<1> [1,0,1]",
            "k_gru_bwd2<1> -> k_front_bwd<2> [1,0,1]",
            "k_gru_bwd2<1> -> k_gru_wgrad<2> [1,0,1]",
            "k_gru_fwd2<1> -> k_mid<16,1> [1,0,1]",
            "k_gru_wgrad<2> -> k_optim_fused [1,0,1]",
            "k_mid<16,1> -> k_gru_bwd2<1> [1,0,1]",
            "k_mid<16,1> -> k_mix_hyper_bwd<1,0> [1,0,1]",
            "k_mix_hyper_bwd<1,0> -> k_gru_wgrad<2> [1,0,1]",
            "k_mix_hyper_fwd<1,0> -> k_mid<16,1> [1,0,1]",
            "k_mix_hyper_fwd<1,0> -> k_mix_hyper_bwd<1,0> [1,0,1]",
            "k_tc_prep_weights -> k_front_fwd_tc2 [1,0,1]",
            "k_tc_prep_weights -> k_mix_hyper_fwd<1,0> [1,0,1]",
        ]),
    "qmix_wide_state": (
        [
            "k_front_bwd<3> grid=(122, 1, 1) block=(256, 1, 1) smem=137104",
            "k_front_fwd_tc2 grid=(46, 2, 1) block=(256, 1, 1) smem=212992",
            "k_gru_bwd2<1> grid=(96, 1, 1) block=(128, 1, 1) smem=0",
            "k_gru_fwd2<1> grid=(96, 2, 1) block=(128, 1, 1) smem=0",
            "k_gru_wgrad<3> grid=(122, 1, 1) block=(256, 1, 1) smem=77712",
            "k_mid<16,1> grid=(120, 1, 1) block=(512, 1, 1) smem=133008",
            "k_mix_hyper_bwd<1,1> grid=(120, 1, 1) block=(256, 1, 1) smem=54544",
            "k_mix_hyper_fwd<1,1> grid=(120, 2, 1) block=(256, 1, 1) smem=54544",
            "k_mixw_fwd grid=(16, 4, 1) block=(128, 1, 1) smem=163840",
            "k_mixw_prep grid=(393, 2, 1) block=(256, 1, 1) smem=0",
            "k_mixw_wgrad grid=(7, 2, 1) block=(128, 1, 1) smem=94208",
            "k_optim_fused grid=(569, 1, 1) block=(256, 1, 1) smem=0",
            "k_tc_prep_weights grid=(72, 2, 1) block=(256, 1, 1) smem=0",
        ],
        [
            "k_front_bwd<3> -> k_optim_fused [1,0,1]",
            "k_front_fwd_tc2 -> k_gru_fwd2<1> [1,0,1]",
            "k_gru_bwd2<1> -> k_front_bwd<3> [1,0,1]",
            "k_gru_bwd2<1> -> k_gru_wgrad<3> [1,0,1]",
            "k_gru_fwd2<1> -> k_mid<16,1> [1,0,1]",
            "k_gru_wgrad<3> -> k_optim_fused [1,0,1]",
            "k_mid<16,1> -> k_gru_bwd2<1> [1,0,1]",
            "k_mid<16,1> -> k_mix_hyper_bwd<1,1> [1,0,1]",
            "k_mix_hyper_bwd<1,1> -> k_mixw_wgrad [1,0,1]",
            "k_mix_hyper_fwd<1,1> -> k_mid<16,1> [1,0,1]",
            "k_mix_hyper_fwd<1,1> -> k_mix_hyper_bwd<1,1> [1,0,1]",
            "k_mixw_fwd -> k_mix_hyper_fwd<1,1> [1,0,1]",
            "k_mixw_prep -> k_mixw_fwd [1,0,1]",
            "k_mixw_wgrad -> k_gru_wgrad<3> [1,0,1]",
            "k_tc_prep_weights -> k_front_fwd_tc2 [1,0,1]",
            "k_tc_prep_weights -> k_mixw_prep [1,0,1]",
        ]),
    "rmaddpg_spread": (
        [
            "k_actor_loss grid=(1, 1, 1) block=(256, 1, 1) smem=0",
            "k_adam grid=(10, 1, 1) block=(1024, 1, 1) smem=0",
            "k_adam grid=(9, 1, 1) block=(1024, 1, 1) smem=0",
            "k_critic_loss grid=(1, 1, 1) block=(256, 1, 1) smem=0",
            "k_front_bwd<2> grid=(25, 1, 1) block=(256, 1, 1) smem=115472",
            "k_front_bwd<2> grid=(75, 1, 1) block=(256, 1, 1) smem=115472",
            "k_front_bwd<2> grid=(78, 1, 1) block=(256, 1, 1) smem=115472",
            "k_front_fwd_tc grid=(19, 1, 1) block=(128, 1, 1) smem=229376",
            "k_front_fwd_tc grid=(7, 1, 1) block=(128, 1, 1) smem=229376",
            "k_front_fwd_tc grid=(7, 1, 1) block=(128, 1, 1) smem=229376",
            "k_front_fwd_tc grid=(7, 2, 1) block=(128, 1, 1) smem=229376",
            "k_front_fwd_tc2 grid=(20, 2, 1) block=(256, 1, 1) smem=208896",
            "k_grad_reduce grid=(139, 1, 1) block=(256, 1, 1) smem=0",
            "k_grad_reduce grid=(149, 1, 1) block=(256, 1, 1) smem=0",
            "k_gru_bwd2<1> grid=(32, 1, 1) block=(128, 1, 1) smem=0",
            "k_gru_bwd2<1> grid=(96, 1, 1) block=(128, 1, 1) smem=0",
            "k_gru_bwd<4> grid=(600, 1, 1) block=(256, 1, 1) smem=0",
            "k_gru_fwd2<1> grid=(32, 1, 1) block=(128, 1, 1) smem=0",
            "k_gru_fwd2<1> grid=(32, 2, 1) block=(128, 1, 1) smem=0",
            "k_gru_fwd2<1> grid=(96, 2, 1) block=(128, 1, 1) smem=0",
            "k_gru_fwd<4> grid=(200, 1, 1) block=(256, 1, 1) smem=0",
            "k_gru_fwd<4> grid=(600, 1, 1) block=(256, 1, 1) smem=0",
            "k_head_bwd grid=(25, 1, 1) block=(256, 1, 1) smem=0",
            "k_head_bwd grid=(75, 1, 1) block=(256, 1, 1) smem=0",
            "k_head_bwd grid=(78, 1, 1) block=(256, 1, 1) smem=0",
            "k_head_fwd grid=(100, 1, 1) block=(256, 1, 1) smem=0",
            "k_head_fwd grid=(100, 1, 1) block=(256, 1, 1) smem=0",
            "k_head_fwd grid=(300, 1, 1) block=(256, 1, 1) smem=0",
            "k_head_fwd grid=(312, 1, 1) block=(256, 1, 1) smem=0",
            "k_head_fwd grid=(312, 1, 1) block=(256, 1, 1) smem=0",
            "k_pack_critic_in grid=(188, 1, 1) block=(256, 1, 1) smem=0",
            "k_pack_critic_in grid=(188, 1, 1) block=(256, 1, 1) smem=0",
            "k_pack_critic_in grid=(528, 1, 1) block=(256, 1, 1) smem=0",
            "k_scatter_actor_grad grid=(10, 1, 1) block=(256, 1, 1) smem=0",
            "k_set_scalars grid=(1, 1, 1) block=(32, 1, 1) smem=0",
            "k_set_scalars grid=(1, 1, 1) block=(32, 1, 1) smem=0",
        ],
        [
            "k_actor_loss -> k_head_bwd",
            "k_adam -> k_front_fwd_tc",
            "k_critic_loss -> k_head_bwd",
            "k_front_bwd<2> -> k_grad_reduce [1,0,1]",
            "k_front_bwd<2> -> k_grad_reduce [1,0,1]",
            "k_front_bwd<2> -> k_scatter_actor_grad",
            "k_front_fwd_tc -> k_gru_fwd2<1> [1,0,1]",
            "k_front_fwd_tc -> k_gru_fwd2<1> [1,0,1]",
            "k_front_fwd_tc -> k_gru_fwd<4> [1,0,1]",
            "k_front_fwd_tc -> k_gru_fwd<4> [1,0,1]",
            "k_front_fwd_tc2 -> k_gru_fwd2<1> [1,0,1]",
            "k_grad_reduce -> k_set_scalars",
            "k_grad_reduce -> k_set_scalars",
            "k_gru_bwd2<1> -> k_front_bwd<2> [1,0,1]",
            "k_gru_bwd2<1> -> k_front_bwd<2> [1,0,1]",
            "k_gru_bwd<4> -> k_front_bwd<2> [1,0,1]",
            "k_gru_fwd2<1> -> k_head_fwd",
            "k_gru_fwd2<1> -> k_head_fwd",
            "k_gru_fwd2<1> -> k_pack_critic_in",
            "k_gru_fwd<4> -> k_head_fwd",
            "k_gru_fwd<4> -> k_head_fwd",
            "k_head_bwd -> k_gru_bwd2<1> [1,0,1]",
            "k_head_bwd -> k_gru_bwd2<1> [1,0,1]",
            "k_head_bwd -> k_gru_bwd<4> [1,0,1]",
            "k_head_fwd -> k_actor_loss",
            "k_head_fwd -> k_critic_loss",
            "k_head_fwd -> k_head_fwd",
            "k_head_fwd -> k_pack_critic_in",
            "k_head_fwd -> k_pack_critic_in",
            "k_pack_critic_in -> k_front_fwd_tc [1,0,1]",
            "k_pack_critic_in -> k_front_fwd_tc [1,0,1]",
            "k_pack_critic_in -> k_front_fwd_tc [1,0,1]",
            "k_scatter_actor_grad -> k_head_bwd",
            "k_set_scalars -> k_adam [1,0,1]",
            "k_set_scalars -> k_adam [1,0,1]",
        ]),
    "rmatd3_spread": (
        [
            "k_actor_loss grid=(1, 1, 1) block=(256, 1, 1) smem=0",
            "k_adam grid=(10, 1, 1) block=(1024, 1, 1) smem=0",
            "k_adam grid=(10, 1, 1) block=(1024, 1, 1) smem=0",
            "k_adam grid=(9, 1, 1) block=(1024, 1, 1) smem=0",
            "k_critic_loss grid=(1, 1, 1) block=(256, 1, 1) smem=0",
            "k_critic_loss grid=(1, 1, 1) block=(256, 1, 1) smem=0",
            "k_front_bwd<2> grid=(25, 1, 1) block=(256, 1, 1) smem=115472",
            "k_front_bwd<2> grid=(25, 1, 1) block=(256, 1, 1) smem=115472",
            "k_front_bwd<2> grid=(75, 1, 1) block=(256, 1, 1) smem=115472",
            "k_front_bwd<2> grid=(78, 1, 1) block=(256, 1, 1) smem=115472",
            "k_front_fwd_tc grid=(19, 1, 1) block=(128, 1, 1) smem=229376",
            "k_front_fwd_tc grid=(7, 1, 1) block=(128, 1, 1) smem=229376",
            "k_front_fwd_tc grid=(7, 1, 1) block=(128, 1, 1) smem=229376",
            "k_front_fwd_tc grid=(7, 1, 1) block=(128, 1, 1) smem=229376",
            "k_front_fwd_tc grid=(7, 2, 1) block=(128, 1, 1) smem=229376",
            "k_front_fwd_tc grid=(7, 2, 1) block=(128, 1, 1) smem=229376",
            "k_front_fwd_tc2 grid=(20, 2, 1) block=(256, 1, 1) smem=208896",
            "k_front_fwd_tc2 grid=(20, 2, 1) block=(256, 1, 1) smem=208896",
            "k_grad_reduce grid=(139, 1, 1) block=(256, 1, 1) smem=0",
            "k_grad_reduce grid=(150, 1, 1) block=(256, 1, 1) smem=0",
            "k_grad_reduce grid=(150, 1, 1) block=(256, 1, 1) smem=0",
            "k_gru_bwd2<1> grid=(32, 1, 1) block=(128, 1, 1) smem=0",
            "k_gru_bwd2<1> grid=(32, 1, 1) block=(128, 1, 1) smem=0",
            "k_gru_bwd2<1> grid=(96, 1, 1) block=(128, 1, 1) smem=0",
            "k_gru_bwd<4> grid=(600, 1, 1) block=(256, 1, 1) smem=0",
            "k_gru_fwd2<1> grid=(32, 1, 1) block=(128, 1, 1) smem=0",
            "k_gru_fwd2<1> grid=(32, 2, 1) block=(128, 1, 1) smem=0",
            "k_gru_fwd2<1> grid=(32, 2, 1) block=(128, 1, 1) smem=0",
            "k_gru_fwd2<1> grid=(96, 2, 1) block=(128, 1, 1) smem=0",
            "k_gru_fwd2<1> grid=(96, 2, 1) block=(128, 1, 1) smem=0",
            "k_gru_fwd<4> grid=(200, 1, 1) block=(256, 1, 1) smem=0",
            "k_gru_fwd<4> grid=(200, 1, 1) block=(256, 1, 1) smem=0",
            "k_gru_fwd<4> grid=(600, 1, 1) block=(256, 1, 1) smem=0",
            "k_head_bwd grid=(25, 1, 1) block=(256, 1, 1) smem=0",
            "k_head_bwd grid=(25, 1, 1) block=(256, 1, 1) smem=0",
            "k_head_bwd grid=(75, 1, 1) block=(256, 1, 1) smem=0",
            "k_head_bwd grid=(78, 1, 1) block=(256, 1, 1) smem=0",
            "k_head_fwd grid=(100, 1, 1) block=(256, 1, 1) smem=0",
            "k_head_fwd grid=(100, 1, 1) block=(256, 1, 1) smem=0",
            "k_head_fwd grid=(100, 1, 1) block=(256, 1, 1) smem=0",
            "k_head_fwd grid=(100, 1, 1) block=(256, 1, 1) smem=0",
            "k_head_fwd grid=(300, 1, 1) block=(256, 1, 1) smem=0",
            "k_head_fwd grid=(312, 1, 1) block=(256, 1, 1) smem=0",
            "k_head_fwd grid=(312, 1, 1) block=(256, 1, 1) smem=0",
            "k_head_fwd grid=(312, 1, 1) block=(256, 1, 1) smem=0",
            "k_head_fwd grid=(312, 1, 1) block=(256, 1, 1) smem=0",
            "k_pack_critic_in grid=(188, 1, 1) block=(256, 1, 1) smem=0",
            "k_pack_critic_in grid=(188, 1, 1) block=(256, 1, 1) smem=0",
            "k_pack_critic_in grid=(188, 1, 1) block=(256, 1, 1) smem=0",
            "k_pack_critic_in grid=(188, 1, 1) block=(256, 1, 1) smem=0",
            "k_pack_critic_in grid=(528, 1, 1) block=(256, 1, 1) smem=0",
            "k_scatter_actor_grad grid=(10, 1, 1) block=(256, 1, 1) smem=0",
            "k_set_scalars grid=(1, 1, 1) block=(32, 1, 1) smem=0",
            "k_set_scalars grid=(1, 1, 1) block=(32, 1, 1) smem=0",
            "k_set_scalars grid=(1, 1, 1) block=(32, 1, 1) smem=0",
            "k_trng_fill grid=(20, 1, 1) block=(256, 1, 1) smem=0",
            "k_trng_fill grid=(20, 1, 1) block=(256, 1, 1) smem=0",
            "k_trng_twist grid=(1, 1, 1) block=(256, 1, 1) smem=0",
            "k_trng_twist grid=(1, 1, 1) block=(256, 1, 1) smem=0",
        ],
        [
            "k_actor_loss -> k_head_bwd",
            "k_adam -> k_front_fwd_tc",
            "k_adam -> k_trng_twist",
            "k_critic_loss -> k_head_bwd",
            "k_critic_loss -> k_head_bwd",
            "k_front_bwd<2> -> k_grad_reduce [1,0,1]",
            "k_front_bwd<2> -> k_grad_reduce [1,0,1]",
            "k_front_bwd<2> -> k_grad_reduce [1,0,1]",
            "k_front_bwd<2> -> k_scatter_actor_grad",
            "k_front_fwd_tc -> k_gru_fwd2<1> [1,0,1]",
            "k_front_fwd_tc -> k_gru_fwd2<1> [1,0,1]",
            "k_front_fwd_tc -> k_gru_fwd2<1> [1,0,1]",
            "k_front_fwd_tc -> k_gru_fwd<4> [1,0,1]",
            "k_front_fwd_tc -> k_gru_fwd<4> [1,0,1]",
            "k_front_fwd_tc -> k_gru_fwd<4> [1,0,1]",
            "k_front_fwd_tc2 -> k_gru_fwd2<1> [1,0,1]",
            "k_front_fwd_tc2 -> k_gru_fwd2<1> [1,0,1]",
            "k_grad_reduce -> k_set_scalars",
            "k_grad_reduce -> k_set_scalars",
            "k_grad_reduce -> k_set_scalars",
            "k_gru_bwd2<1> -> k_front_bwd<2> [1,0,1]",
            "k_gru_bwd2<1> -> k_front_bwd<2> [1,0,1]",
            "k_gru_bwd2<1> -> k_front_bwd<2> [1,0,1]",
            "k_gru_bwd<4> -> k_front_bwd<2> [1,0,1]",
            "k_gru_fwd2<1> -> k_head_fwd",
            "k_gru_fwd2<1> -> k_head_fwd",
            "k_gru_fwd2<1> -> k_head_fwd",
            "k_gru_fwd2<1> -> k_head_fwd",
            "k_gru_fwd2<1> -> k_pack_critic_in",
            "k_gru_fwd<4> -> k_head_fwd",
            "k_gru_fwd<4> -> k_head_fwd",
            "k_gru_fwd<4> -> k_head_fwd",
            "k_head_bwd -> k_gru_bwd2<1> [1,0,1]",
            "k_head_bwd -> k_gru_bwd2<1> [1,0,1]",
            "k_head_bwd -> k_gru_bwd2<1> [1,0,1]",
            "k_head_bwd -> k_gru_bwd<4> [1,0,1]",
            "k_head_fwd -> k_actor_loss",
            "k_head_fwd -> k_critic_loss",
            "k_head_fwd -> k_critic_loss",
            "k_head_fwd -> k_head_fwd",
            "k_head_fwd -> k_head_fwd",
            "k_head_fwd -> k_pack_critic_in",
            "k_head_fwd -> k_pack_critic_in",
            "k_head_fwd -> k_pack_critic_in",
            "k_head_fwd -> k_pack_critic_in",
            "k_pack_critic_in -> k_front_fwd_tc [1,0,1]",
            "k_pack_critic_in -> k_front_fwd_tc [1,0,1]",
            "k_pack_critic_in -> k_front_fwd_tc [1,0,1]",
            "k_pack_critic_in -> k_front_fwd_tc [1,0,1]",
            "k_pack_critic_in -> k_front_fwd_tc [1,0,1]",
            "k_scatter_actor_grad -> k_head_bwd",
            "k_set_scalars -> k_adam [1,0,1]",
            "k_set_scalars -> k_adam [1,0,1]",
            "k_set_scalars -> k_adam [1,0,1]",
            "k_trng_fill -> k_front_fwd_tc2",
            "k_trng_fill -> k_front_fwd_tc2",
            "k_trng_twist -> k_trng_fill",
            "k_trng_twist -> k_trng_fill",
        ]),
    "vdn_3m": (
        [
            "k_front_bwd<3> grid=(122, 1, 1) block=(256, 1, 1) smem=137104",
            "k_front_fwd_tc2 grid=(46, 2, 1) block=(256, 1, 1) smem=212992",
            "k_gru_bwd2<1> grid=(96, 1, 1) block=(128, 1, 1) smem=0",
            "k_gru_fwd2<1> grid=(96, 2, 1) block=(128, 1, 1) smem=0",
            "k_gru_wgrad<3> grid=(122, 1, 1) block=(256, 1, 1) smem=77712",
            "k_optim_fused grid=(144, 1, 1) block=(256, 1, 1) smem=0",
            "k_qhead<1> grid=(528, 1, 1) block=(256, 1, 1) smem=0",
            "k_qhead_bwd<1> grid=(132, 1, 1) block=(256, 1, 1) smem=26368",
            "k_tc_prep_weights grid=(72, 2, 1) block=(256, 1, 1) smem=0",
            "k_vdn_mix grid=(8, 1, 1) block=(256, 1, 1) smem=0",
        ],
        [
            "k_front_bwd<3> -> k_optim_fused [1,0,1]",
            "k_front_fwd_tc2 -> k_gru_fwd2<1> [1,0,1]",
            "k_gru_bwd2<1> -> k_front_bwd<3> [1,0,1]",
            "k_gru_bwd2<1> -> k_gru_wgrad<3> [1,0,1]",
            "k_gru_fwd2<1> -> k_qhead<1> [1,0,1]",
            "k_gru_wgrad<3> -> k_optim_fused [1,0,1]",
            "k_qhead<1> -> k_vdn_mix [1,0,1]",
            "k_qhead_bwd<1> -> k_gru_bwd2<1> [1,0,1]",
            "k_tc_prep_weights -> k_front_fwd_tc2 [1,0,1]",
            "k_vdn_mix -> k_qhead_bwd<1> [1,0,1]",
        ]),
}

_structure = qs.graph_structure


def graph_configs(graph):
    """(sorted kernel nodes "name grid block smem", sorted edges as graph_structure gives them) of a cudaGraph_t."""
    cu = C.CDLL("libcuda.so.1")
    g = C.c_void_p(graph)
    n = C.c_size_t(0)
    qs._check(cu.cuGraphGetNodes(g, None, C.byref(n)), "cuGraphGetNodes")
    nodes = (C.c_void_p * max(n.value, 1))()
    qs._check(cu.cuGraphGetNodes(g, nodes, C.byref(n)), "cuGraphGetNodes")
    out = []
    for i in range(n.value):
        ty = C.c_int(-1)
        qs._check(cu.cuGraphNodeGetType(C.c_void_p(nodes[i]), C.byref(ty)), "cuGraphNodeGetType")
        if ty.value != 0:
            continue
        p = qs._KernelNodeParams()
        qs._check(cu.cuGraphKernelNodeGetParams_v2(C.c_void_p(nodes[i]), C.byref(p)), "cuGraphKernelNodeGetParams")
        s = C.c_char_p()
        if p.func:
            qs._check(cu.cuFuncGetName(C.byref(s), C.c_void_p(p.func)), "cuFuncGetName")
        else:
            qs._check(cu.cuKernelGetName(C.byref(s), C.c_void_p(p.kern)), "cuKernelGetName")
        out.append("%s grid=%s block=%s smem=%d" % (qs.kernel_name(s.value.decode()), tuple(p.grid), tuple(p.block), p.smem))
    return sorted(out), _structure(graph)[1]


def qmix_configs(name):
    """The QMIX-family step of shape `name` (test_gpu_qmix_schedule.SHAPES) as graph_configs()."""
    structure = qs.graph_structure
    qs.graph_structure = graph_configs
    try:
        return qs.capture_step(name)
    finally:
        qs.graph_structure = structure


def maddpg_configs(name):
    """`updates` actor-critic updates of configuration `name`, captured on one graph, as graph_configs()."""
    from checkpoint_maddpg_checks import Case
    from offpolicy._b200.torch_rng import DeviceTorchGenerator
    kw, device_noise, updates = MADDPG[name]
    case = Case(rng="device", **kw)
    tr, buf, pols = case.build(1)
    case.fill(buf, np.random.RandomState(5), case.E)
    torch.manual_seed(11)
    if device_noise:
        tr.use_device_noise(DeviceTorchGenerator(seed=3))
    smp = buf.sample(case.B)
    for _ in range(2):
        tr.train_policy_on_batch("policy_0", smp)      # first launches (module loading, smem attributes) outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph(keep_graph=True)
    with torch.cuda.graph(g):
        for _ in range(updates):
            tr.train_policy_on_batch("policy_0", smp)
    try:
        return graph_configs(g.raw_cuda_graph())
    finally:
        g.reset()
        torch.cuda.synchronize()


def configs(name):
    return maddpg_configs(name) if name in MADDPG else qmix_configs(name)


@pytest.mark.parametrize("name", sorted(qs.SHAPES) + sorted(MADDPG))
def test_captured_launch_configuration(gpu_engine, name):
    nodes, edges = configs(name)
    want_nodes, want_edges = EXPECTED[name]
    assert nodes == want_nodes, (name, nodes)
    assert edges == want_edges, (name, edges)
