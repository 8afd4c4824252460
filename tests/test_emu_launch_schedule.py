"""The launch schedule of the entry points outside the QMIX step on the CPU fiber emulator: for each call, the names of the kernels it
launched (mx_profile_begin / mx_profile_end, as tests/test_emu_qmix_schedule.py does for the step) and how far it moved
mx_launch_count().

Covered: the R-MADDPG / R-MATD3 and MLP MADDPG / MATD3 updates (Box, Discrete, MultiDiscrete, several policies with their centralised
action contributions, the actor update on and off, the device-noise fills), replay inserts with and without PER and reward
normalisation, uniform and PER draws, priority updates, the rollout policy step and the soft / hard target updates.  Each schedule
below was recorded from the launchers as they stood before they were put on one launch function (mx_launch); a change to a schedule
has to change it on purpose."""
import numpy as np
import pytest
import torch

from checkpoint_maddpg_checks import Case
import row_coverage_checks as rc

# name: (Case, device noise)
CASES = {
    "rmaddpg_box": (Case("rec", [(2, 6, 2)], S=8, B=4, E=9, T=4, discrete=False, rng="device"), False),
    "rmaddpg_discrete": (Case("rec", [(2, 6, 3)], S=8, B=4, E=9, T=4, rng="device"), False),
    "rmatd3_box_per_norm": (Case("rec", [(2, 6, 2)], S=8, B=4, E=9, T=4, td3=True, discrete=False, per=True, norm=True, rng="device"), False),
    "rmatd3_discrete": (Case("rec", [(2, 6, 3)], S=8, B=4, E=9, T=4, td3=True, rng="device"), False),
    "rmatd3_discrete_device_noise": (Case("rec", [(2, 6, 3)], S=8, B=4, E=9, T=4, td3=True, rng="device"), True),
    "maddpg_shared": (Case("mlp", [(3, 6, 5)], S=10, B=8, E=40, rng="device"), False),
    "maddpg_shared_per": (Case("mlp", [(3, 6, 5)], S=10, B=8, E=40, per=True, rng="device"), False),
    "maddpg_shared_device_noise": (Case("mlp", [(3, 6, 5)], S=10, B=8, E=40, rng="device"), True),
    "matd3_box_norm": (Case("mlp", [(2, 6, 2)], S=10, B=8, E=40, td3=True, discrete=False, norm=True, rng="device"), False),
    "matd3_multidiscrete": (Case("mlp", [(2, 8, [3, 4])], S=10, B=8, E=40, td3=True, rng="device"), False),
    "matd3_multidiscrete_device_noise": (Case("mlp", [(2, 8, [3, 4])], S=10, B=8, E=40, td3=True, rng="device"), True),
    "maddpg_two_policies": (Case("mlp", [(2, 6, 4), (1, 5, 3)], S=10, B=8, E=40, rng="device"), False),
    "matd3_two_policies_per": (Case("mlp", [(2, 6, 4), (1, 5, 3)], S=10, B=8, E=40, td3=True, per=True, rng="device"), False),
}

EXPECTED = {'maddpg_shared': [('insert', 'k_insert_scatter', 1),
                   ('sample', 'k_draw k_gather', 2),
                   ('train policy_0 #0',
                    'k_front_fwd_tc k_mlp_head_cols k_act_transform k_pack_critic_in k_pack_critic_in k_front_fwd_tc k_front_fwd_tc k_mlp_head_cols k_mlp_head_cols k_critic_loss k_mlp_dgi_cols '
                    'k_front_bwd k_grad_reduce k_set_scalars k_adam k_mlp_head_cols k_act_transform k_pack_critic_in k_front_fwd_tc k_mlp_head_cols k_actor_loss k_mlp_dgi_cols k_front_bwd '
                    'k_scatter_actor_grad k_front_bwd k_grad_reduce k_set_scalars k_adam',
                    28),
                   ('train policy_0 #1',
                    'k_front_fwd_tc k_mlp_head_cols k_act_transform k_pack_critic_in k_pack_critic_in k_front_fwd_tc k_front_fwd_tc k_mlp_head_cols k_mlp_head_cols k_critic_loss k_mlp_dgi_cols '
                    'k_front_bwd k_grad_reduce k_set_scalars k_adam k_mlp_head_cols k_act_transform k_pack_critic_in k_front_fwd_tc k_mlp_head_cols k_actor_loss k_mlp_dgi_cols k_front_bwd '
                    'k_scatter_actor_grad k_front_bwd k_grad_reduce k_set_scalars k_adam',
                    28),
                   ('soft_update', 'k_polyak k_polyak', 2),
                   ('hard_update', '', 0)],
 'maddpg_shared_device_noise': [('insert', 'k_insert_scatter', 1),
                                ('sample', 'k_draw k_gather', 2),
                                ('train policy_0 #0',
                                 'k_trng_twist k_trng_fill k_front_fwd_tc k_mlp_head_cols k_act_transform k_pack_critic_in k_pack_critic_in k_front_fwd_tc k_front_fwd_tc k_mlp_head_cols '
                                 'k_mlp_head_cols k_critic_loss k_mlp_dgi_cols k_front_bwd k_grad_reduce k_set_scalars k_adam k_mlp_head_cols k_act_transform k_pack_critic_in k_front_fwd_tc '
                                 'k_mlp_head_cols k_actor_loss k_mlp_dgi_cols k_front_bwd k_scatter_actor_grad k_front_bwd k_grad_reduce k_set_scalars k_adam',
                                 30),
                                ('train policy_0 #1',
                                 'k_trng_twist k_trng_fill k_front_fwd_tc k_mlp_head_cols k_act_transform k_pack_critic_in k_pack_critic_in k_front_fwd_tc k_front_fwd_tc k_mlp_head_cols '
                                 'k_mlp_head_cols k_critic_loss k_mlp_dgi_cols k_front_bwd k_grad_reduce k_set_scalars k_adam k_mlp_head_cols k_act_transform k_pack_critic_in k_front_fwd_tc '
                                 'k_mlp_head_cols k_actor_loss k_mlp_dgi_cols k_front_bwd k_scatter_actor_grad k_front_bwd k_grad_reduce k_set_scalars k_adam',
                                 30),
                                ('soft_update', 'k_polyak k_polyak', 2),
                                ('hard_update', '', 0)],
 'maddpg_shared_per': [('insert', 'k_insert_scatter k_tree_update', 2),
                       ('sample', 'k_draw k_gather', 2),
                       ('train policy_0 #0',
                        'k_front_fwd_tc k_mlp_head_cols k_act_transform k_pack_critic_in k_pack_critic_in k_front_fwd_tc k_front_fwd_tc k_mlp_head_cols k_mlp_head_cols k_critic_loss k_mlp_dgi_cols '
                        'k_front_bwd k_grad_reduce k_set_scalars k_adam k_mlp_head_cols k_act_transform k_pack_critic_in k_front_fwd_tc k_mlp_head_cols k_actor_loss k_mlp_dgi_cols k_front_bwd '
                        'k_scatter_actor_grad k_front_bwd k_grad_reduce k_set_scalars k_adam',
                        28),
                       ('update_priorities policy_0', 'k_tree_update', 1),
                       ('train policy_0 #1',
                        'k_front_fwd_tc k_mlp_head_cols k_act_transform k_pack_critic_in k_pack_critic_in k_front_fwd_tc k_front_fwd_tc k_mlp_head_cols k_mlp_head_cols k_critic_loss k_mlp_dgi_cols '
                        'k_front_bwd k_grad_reduce k_set_scalars k_adam k_mlp_head_cols k_act_transform k_pack_critic_in k_front_fwd_tc k_mlp_head_cols k_actor_loss k_mlp_dgi_cols k_front_bwd '
                        'k_scatter_actor_grad k_front_bwd k_grad_reduce k_set_scalars k_adam',
                        28),
                       ('soft_update', 'k_polyak k_polyak', 2),
                       ('hard_update', '', 0)],
 'maddpg_two_policies': [('insert', 'k_insert_scatter k_insert_scatter', 2),
                         ('sample', 'k_draw k_gather k_gather', 3),
                         ('train policy_0 #0',
                          'k_front_fwd_tc k_mlp_head_cols k_act_transform k_cent_scatter k_front_fwd_tc k_mlp_head_cols k_act_transform k_cent_scatter k_front_fwd_tc k_pack_critic_in '
                          'k_pack_critic_in k_front_fwd_tc k_front_fwd_tc k_mlp_head_cols k_mlp_head_cols k_critic_loss k_mlp_dgi_cols k_front_bwd k_grad_reduce k_set_scalars k_adam k_mlp_head_cols '
                          'k_act_transform k_pack_critic_in k_front_fwd_tc k_mlp_head_cols k_actor_loss k_mlp_dgi_cols k_front_bwd k_scatter_actor_grad k_front_bwd k_grad_reduce k_set_scalars k_adam',
                          34),
                         ('train policy_1 #0',
                          'k_front_fwd_tc k_mlp_head_cols k_act_transform k_cent_scatter k_front_fwd_tc k_mlp_head_cols k_act_transform k_cent_scatter k_front_fwd_tc k_pack_critic_in '
                          'k_pack_critic_in k_front_fwd_tc k_front_fwd_tc k_mlp_head_cols k_mlp_head_cols k_critic_loss k_mlp_dgi_cols k_front_bwd k_grad_reduce k_set_scalars k_adam k_mlp_head_cols '
                          'k_act_transform k_pack_critic_in k_front_fwd_tc k_mlp_head_cols k_actor_loss k_mlp_dgi_cols k_front_bwd k_scatter_actor_grad k_front_bwd k_grad_reduce k_set_scalars k_adam',
                          34),
                         ('train policy_0 #1',
                          'k_front_fwd_tc k_mlp_head_cols k_act_transform k_cent_scatter k_front_fwd_tc k_mlp_head_cols k_act_transform k_cent_scatter k_front_fwd_tc k_pack_critic_in '
                          'k_pack_critic_in k_front_fwd_tc k_front_fwd_tc k_mlp_head_cols k_mlp_head_cols k_critic_loss k_mlp_dgi_cols k_front_bwd k_grad_reduce k_set_scalars k_adam k_mlp_head_cols '
                          'k_act_transform k_pack_critic_in k_front_fwd_tc k_mlp_head_cols k_actor_loss k_mlp_dgi_cols k_front_bwd k_scatter_actor_grad k_front_bwd k_grad_reduce k_set_scalars k_adam',
                          34),
                         ('train policy_1 #1',
                          'k_front_fwd_tc k_mlp_head_cols k_act_transform k_cent_scatter k_front_fwd_tc k_mlp_head_cols k_act_transform k_cent_scatter k_front_fwd_tc k_pack_critic_in '
                          'k_pack_critic_in k_front_fwd_tc k_front_fwd_tc k_mlp_head_cols k_mlp_head_cols k_critic_loss k_mlp_dgi_cols k_front_bwd k_grad_reduce k_set_scalars k_adam k_mlp_head_cols '
                          'k_act_transform k_pack_critic_in k_front_fwd_tc k_mlp_head_cols k_actor_loss k_mlp_dgi_cols k_front_bwd k_scatter_actor_grad k_front_bwd k_grad_reduce k_set_scalars k_adam',
                          34),
                         ('soft_update', 'k_polyak k_polyak k_polyak k_polyak', 4),
                         ('hard_update', '', 0)],
 'matd3_box_norm': [('insert', 'k_reward_stats_update k_insert_scatter', 2),
                    ('sample', 'k_draw k_gather', 2),
                    ('train policy_0 #0',
                     'k_front_fwd_tc k_mlp_head_cols k_pack_critic_in k_pack_critic_in k_front_fwd_tc k_front_fwd_tc k_mlp_head_cols k_mlp_head_cols k_critic_loss k_mlp_dgi_cols k_front_bwd '
                     'k_grad_reduce k_set_scalars k_adam k_mlp_head_cols k_pack_critic_in k_front_fwd_tc k_mlp_head_cols k_actor_loss k_mlp_dgi_cols k_front_bwd k_scatter_actor_grad k_front_bwd '
                     'k_grad_reduce k_set_scalars k_adam',
                     26),
                    ('train policy_0 #1',
                     'k_front_fwd_tc k_mlp_head_cols k_pack_critic_in k_pack_critic_in k_front_fwd_tc k_front_fwd_tc k_mlp_head_cols k_mlp_head_cols k_critic_loss k_mlp_dgi_cols k_front_bwd '
                     'k_grad_reduce k_set_scalars k_adam k_mlp_head_cols k_pack_critic_in k_front_fwd_tc k_mlp_head_cols k_actor_loss k_mlp_dgi_cols k_front_bwd k_scatter_actor_grad k_front_bwd '
                     'k_grad_reduce k_set_scalars k_adam',
                     26),
                    ('soft_update', 'k_polyak k_polyak', 2),
                    ('hard_update', '', 0)],
 'matd3_multidiscrete': [('insert', 'k_insert_scatter', 1),
                         ('sample', 'k_draw k_gather', 2),
                         ('train policy_0 #0',
                          'k_front_fwd_tc k_mlp_head_cols k_act_transform k_pack_critic_in k_pack_critic_in k_front_fwd_tc k_front_fwd_tc k_mlp_head_cols k_mlp_head_cols k_critic_loss k_mlp_dgi_cols '
                          'k_front_bwd k_grad_reduce k_set_scalars k_adam k_mlp_head_cols k_act_transform k_pack_critic_in k_front_fwd_tc k_mlp_head_cols k_actor_loss k_mlp_dgi_cols k_front_bwd '
                          'k_scatter_actor_grad k_front_bwd k_grad_reduce k_set_scalars k_adam',
                          28),
                         ('train policy_0 #1',
                          'k_front_fwd_tc k_mlp_head_cols k_act_transform k_pack_critic_in k_pack_critic_in k_front_fwd_tc k_front_fwd_tc k_mlp_head_cols k_mlp_head_cols k_critic_loss k_mlp_dgi_cols '
                          'k_front_bwd k_grad_reduce k_set_scalars k_adam k_mlp_head_cols k_act_transform k_pack_critic_in k_front_fwd_tc k_mlp_head_cols k_actor_loss k_mlp_dgi_cols k_front_bwd '
                          'k_scatter_actor_grad k_front_bwd k_grad_reduce k_set_scalars k_adam',
                          28),
                         ('soft_update', 'k_polyak k_polyak', 2),
                         ('hard_update', '', 0)],
 'matd3_multidiscrete_device_noise': [('insert', 'k_insert_scatter', 1),
                                      ('sample', 'k_draw k_gather', 2),
                                      ('train policy_0 #0',
                                       'k_trng_twist k_trng_fill k_trng_twist k_trng_fill k_trng_twist k_trng_fill k_trng_twist k_trng_fill k_front_fwd_tc k_mlp_head_cols k_act_transform '
                                       'k_pack_critic_in k_pack_critic_in k_front_fwd_tc k_front_fwd_tc k_mlp_head_cols k_mlp_head_cols k_critic_loss k_mlp_dgi_cols k_front_bwd k_grad_reduce '
                                       'k_set_scalars k_adam k_mlp_head_cols k_act_transform k_pack_critic_in k_front_fwd_tc k_mlp_head_cols k_actor_loss k_mlp_dgi_cols k_front_bwd '
                                       'k_scatter_actor_grad k_front_bwd k_grad_reduce k_set_scalars k_adam',
                                       36),
                                      ('train policy_0 #1',
                                       'k_trng_twist k_trng_fill k_trng_twist k_trng_fill k_trng_twist k_trng_fill k_trng_twist k_trng_fill k_front_fwd_tc k_mlp_head_cols k_act_transform '
                                       'k_pack_critic_in k_pack_critic_in k_front_fwd_tc k_front_fwd_tc k_mlp_head_cols k_mlp_head_cols k_critic_loss k_mlp_dgi_cols k_front_bwd k_grad_reduce '
                                       'k_set_scalars k_adam k_mlp_head_cols k_act_transform k_pack_critic_in k_front_fwd_tc k_mlp_head_cols k_actor_loss k_mlp_dgi_cols k_front_bwd '
                                       'k_scatter_actor_grad k_front_bwd k_grad_reduce k_set_scalars k_adam',
                                       36),
                                      ('soft_update', 'k_polyak k_polyak', 2),
                                      ('hard_update', '', 0)],
 'matd3_two_policies_per': [('insert', 'k_insert_scatter k_tree_update k_insert_scatter k_tree_update', 4),
                            ('sample', 'k_draw k_gather k_gather', 3),
                            ('train policy_0 #0',
                             'k_front_fwd_tc k_mlp_head_cols k_act_transform k_cent_scatter k_front_fwd_tc k_mlp_head_cols k_act_transform k_cent_scatter k_front_fwd_tc k_pack_critic_in '
                             'k_pack_critic_in k_front_fwd_tc k_front_fwd_tc k_mlp_head_cols k_mlp_head_cols k_critic_loss k_mlp_dgi_cols k_front_bwd k_grad_reduce k_set_scalars k_adam '
                             'k_mlp_head_cols k_act_transform k_pack_critic_in k_front_fwd_tc k_mlp_head_cols k_actor_loss k_mlp_dgi_cols k_front_bwd k_scatter_actor_grad k_front_bwd k_grad_reduce '
                             'k_set_scalars k_adam',
                             34),
                            ('update_priorities policy_0', 'k_tree_update', 1),
                            ('train policy_1 #0',
                             'k_front_fwd_tc k_mlp_head_cols k_act_transform k_cent_scatter k_front_fwd_tc k_mlp_head_cols k_act_transform k_cent_scatter k_front_fwd_tc k_pack_critic_in '
                             'k_pack_critic_in k_front_fwd_tc k_front_fwd_tc k_mlp_head_cols k_mlp_head_cols k_critic_loss k_mlp_dgi_cols k_front_bwd k_grad_reduce k_set_scalars k_adam '
                             'k_mlp_head_cols k_act_transform k_pack_critic_in k_front_fwd_tc k_mlp_head_cols k_actor_loss k_mlp_dgi_cols k_front_bwd k_scatter_actor_grad k_front_bwd k_grad_reduce '
                             'k_set_scalars k_adam',
                             34),
                            ('update_priorities policy_1', 'k_tree_update', 1),
                            ('train policy_0 #1',
                             'k_front_fwd_tc k_mlp_head_cols k_act_transform k_cent_scatter k_front_fwd_tc k_mlp_head_cols k_act_transform k_cent_scatter k_front_fwd_tc k_pack_critic_in '
                             'k_pack_critic_in k_front_fwd_tc k_front_fwd_tc k_mlp_head_cols k_mlp_head_cols k_critic_loss k_mlp_dgi_cols k_front_bwd k_grad_reduce k_set_scalars k_adam '
                             'k_mlp_head_cols k_act_transform k_pack_critic_in k_front_fwd_tc k_mlp_head_cols k_actor_loss k_mlp_dgi_cols k_front_bwd k_scatter_actor_grad k_front_bwd k_grad_reduce '
                             'k_set_scalars k_adam',
                             34),
                            ('train policy_1 #1',
                             'k_front_fwd_tc k_mlp_head_cols k_act_transform k_cent_scatter k_front_fwd_tc k_mlp_head_cols k_act_transform k_cent_scatter k_front_fwd_tc k_pack_critic_in '
                             'k_pack_critic_in k_front_fwd_tc k_front_fwd_tc k_mlp_head_cols k_mlp_head_cols k_critic_loss k_mlp_dgi_cols k_front_bwd k_grad_reduce k_set_scalars k_adam '
                             'k_mlp_head_cols k_act_transform k_pack_critic_in k_front_fwd_tc k_mlp_head_cols k_actor_loss k_mlp_dgi_cols k_front_bwd k_scatter_actor_grad k_front_bwd k_grad_reduce '
                             'k_set_scalars k_adam',
                             34),
                            ('soft_update', 'k_polyak k_polyak k_polyak k_polyak', 4),
                            ('hard_update', '', 0)],
 'qmix_rollout_targets': [('policy_step greedy', 'k_policy_step', 1), ('policy_step explore', 'k_policy_step', 1), ('soft_update', 'k_polyak', 1), ('hard_update', 'hard_update_memcpy', 0)],
 'rmaddpg_box': [('insert', 'k_insert_scatter', 1),
                 ('sample', 'k_draw k_gather', 2),
                 ('train policy_0 #0',
                  'k_front_fwd_tc k_gru_fwd k_head_fwd k_head_fwd k_pack_critic_in k_front_fwd_tc k_gru_fwd k_head_fwd k_pack_critic_in k_front_fwd_tc k_gru_fwd k_head_fwd k_critic_loss k_head_bwd '
                  'k_gru_bwd k_front_bwd k_grad_reduce k_set_scalars k_adam k_front_fwd_tc k_gru_fwd k_pack_critic_in k_front_fwd_tc k_gru_fwd k_head_fwd k_actor_loss k_head_bwd k_gru_bwd '
                  'k_front_bwd k_scatter_actor_grad k_head_bwd k_gru_bwd k_front_bwd k_grad_reduce k_set_scalars k_adam',
                  36),
                 ('train policy_0 #1',
                  'k_front_fwd_tc k_gru_fwd k_head_fwd k_head_fwd k_pack_critic_in k_front_fwd_tc k_gru_fwd k_head_fwd k_pack_critic_in k_front_fwd_tc k_gru_fwd k_head_fwd k_critic_loss k_head_bwd '
                  'k_gru_bwd k_front_bwd k_grad_reduce k_set_scalars k_adam k_front_fwd_tc k_gru_fwd k_pack_critic_in k_front_fwd_tc k_gru_fwd k_head_fwd k_actor_loss k_head_bwd k_gru_bwd '
                  'k_front_bwd k_scatter_actor_grad k_head_bwd k_gru_bwd k_front_bwd k_grad_reduce k_set_scalars k_adam',
                  36),
                 ('soft_update', 'k_polyak k_polyak', 2),
                 ('hard_update', '', 0)],
 'rmaddpg_discrete': [('insert', 'k_insert_scatter', 1),
                      ('sample', 'k_draw k_gather', 2),
                      ('train policy_0 #0',
                       'k_front_fwd_tc k_gru_fwd k_head_fwd k_head_fwd k_act_transform k_pack_critic_in k_front_fwd_tc k_gru_fwd k_head_fwd k_pack_critic_in k_front_fwd_tc k_gru_fwd k_head_fwd '
                       'k_critic_loss k_head_bwd k_gru_bwd k_front_bwd k_grad_reduce k_set_scalars k_adam k_front_fwd_tc k_gru_fwd k_act_transform k_pack_critic_in k_front_fwd_tc k_gru_fwd '
                       'k_head_fwd k_actor_loss k_head_bwd k_gru_bwd k_front_bwd k_scatter_actor_grad k_head_bwd k_gru_bwd k_front_bwd k_grad_reduce k_set_scalars k_adam',
                       38),
                      ('train policy_0 #1',
                       'k_front_fwd_tc k_gru_fwd k_head_fwd k_head_fwd k_act_transform k_pack_critic_in k_front_fwd_tc k_gru_fwd k_head_fwd k_pack_critic_in k_front_fwd_tc k_gru_fwd k_head_fwd '
                       'k_critic_loss k_head_bwd k_gru_bwd k_front_bwd k_grad_reduce k_set_scalars k_adam k_front_fwd_tc k_gru_fwd k_act_transform k_pack_critic_in k_front_fwd_tc k_gru_fwd '
                       'k_head_fwd k_actor_loss k_head_bwd k_gru_bwd k_front_bwd k_scatter_actor_grad k_head_bwd k_gru_bwd k_front_bwd k_grad_reduce k_set_scalars k_adam',
                       38),
                      ('soft_update', 'k_polyak k_polyak', 2),
                      ('hard_update', '', 0)],
 'rmatd3_box_per_norm': [('insert', 'k_reward_stats_update k_insert_scatter k_tree_update', 3),
                         ('sample', 'k_draw k_gather', 2),
                         ('train policy_0 #0',
                          'k_front_fwd_tc k_gru_fwd k_head_fwd k_head_fwd k_pack_critic_in k_front_fwd_tc k_gru_fwd k_head_fwd k_pack_critic_in k_front_fwd_tc k_gru_fwd k_head_fwd k_critic_loss '
                          'k_head_bwd k_gru_bwd k_front_bwd k_grad_reduce k_set_scalars k_adam k_front_fwd_tc k_gru_fwd k_pack_critic_in k_front_fwd_tc k_gru_fwd k_head_fwd k_actor_loss k_head_bwd '
                          'k_gru_bwd k_front_bwd k_scatter_actor_grad k_head_bwd k_gru_bwd k_front_bwd k_grad_reduce k_set_scalars k_adam',
                          36),
                         ('update_priorities policy_0', 'k_tree_update', 1),
                         ('train policy_0 #1',
                          'k_front_fwd_tc k_gru_fwd k_head_fwd k_head_fwd k_pack_critic_in k_front_fwd_tc k_gru_fwd k_head_fwd k_pack_critic_in k_front_fwd_tc k_gru_fwd k_head_fwd k_critic_loss '
                          'k_head_bwd k_gru_bwd k_front_bwd k_grad_reduce k_set_scalars k_adam',
                          19),
                         ('soft_update', 'k_polyak k_polyak', 2),
                         ('hard_update', '', 0)],
 'rmatd3_discrete': [('insert', 'k_insert_scatter', 1),
                     ('sample', 'k_draw k_gather', 2),
                     ('train policy_0 #0',
                      'k_front_fwd_tc k_gru_fwd k_head_fwd k_head_fwd k_act_transform k_pack_critic_in k_front_fwd_tc k_gru_fwd k_head_fwd k_pack_critic_in k_front_fwd_tc k_gru_fwd k_head_fwd '
                      'k_critic_loss k_head_bwd k_gru_bwd k_front_bwd k_grad_reduce k_set_scalars k_adam k_front_fwd_tc k_gru_fwd k_act_transform k_pack_critic_in k_front_fwd_tc k_gru_fwd k_head_fwd '
                      'k_actor_loss k_head_bwd k_gru_bwd k_front_bwd k_scatter_actor_grad k_head_bwd k_gru_bwd k_front_bwd k_grad_reduce k_set_scalars k_adam',
                      38),
                     ('train policy_0 #1',
                      'k_front_fwd_tc k_gru_fwd k_head_fwd k_head_fwd k_act_transform k_pack_critic_in k_front_fwd_tc k_gru_fwd k_head_fwd k_pack_critic_in k_front_fwd_tc k_gru_fwd k_head_fwd '
                      'k_critic_loss k_head_bwd k_gru_bwd k_front_bwd k_grad_reduce k_set_scalars k_adam',
                      20),
                     ('soft_update', 'k_polyak k_polyak', 2),
                     ('hard_update', '', 0)],
 'rmatd3_discrete_device_noise': [('insert', 'k_insert_scatter', 1),
                                  ('sample', 'k_draw k_gather', 2),
                                  ('train policy_0 #0',
                                   'k_trng_twist k_trng_fill k_trng_twist k_trng_fill k_front_fwd_tc k_gru_fwd k_head_fwd k_head_fwd k_act_transform k_pack_critic_in k_front_fwd_tc k_gru_fwd '
                                   'k_head_fwd k_pack_critic_in k_front_fwd_tc k_gru_fwd k_head_fwd k_critic_loss k_head_bwd k_gru_bwd k_front_bwd k_grad_reduce k_set_scalars k_adam k_front_fwd_tc '
                                   'k_gru_fwd k_act_transform k_pack_critic_in k_front_fwd_tc k_gru_fwd k_head_fwd k_actor_loss k_head_bwd k_gru_bwd k_front_bwd k_scatter_actor_grad k_head_bwd '
                                   'k_gru_bwd k_front_bwd k_grad_reduce k_set_scalars k_adam',
                                   42),
                                  ('train policy_0 #1',
                                   'k_trng_twist k_trng_fill k_front_fwd_tc k_gru_fwd k_head_fwd k_head_fwd k_act_transform k_pack_critic_in k_front_fwd_tc k_gru_fwd k_head_fwd k_pack_critic_in '
                                   'k_front_fwd_tc k_gru_fwd k_head_fwd k_critic_loss k_head_bwd k_gru_bwd k_front_bwd k_grad_reduce k_set_scalars k_adam',
                                   22),
                                  ('soft_update', 'k_polyak k_polyak', 2),
                                  ('hard_update', '', 0)]}


def _run(lib, fn):
    n0 = lib.mx_launch_count()
    names = rc.kernels_run(lib, None, fn)
    return " ".join(names), int(lib.mx_launch_count() - n0)


def case_schedule(lib, name):
    """[(call, kernels, launches)] of: one insert, one draw, two updates of every policy (R-MATD3 / MATD3: the actor update on, then
    off), the PER priority write-back, and the soft and hard target updates."""
    from offpolicy._b200.torch_rng import DeviceTorchGenerator
    case, device_noise = CASES[name]
    tr, buf, pols = case.build(1)
    rs = np.random.RandomState(5)
    case.fill(buf, rs, case.E)
    torch.manual_seed(11)
    if device_noise:
        tr.use_device_noise(DeviceTorchGenerator(seed=3))
    out = [("insert",) + _run(lib, lambda: case.put(buf, rs, case.insert))]
    smp = []
    out.append(("sample",) + _run(lib, lambda: smp.append(buf.sample(case.B, 0.5, "policy_0") if case.per else buf.sample(case.B))))
    for k in range(2):
        for p in case.ids:
            res = []
            out.append(("train %s #%d" % (p, k),) + _run(lib, lambda: res.append(tr.train_policy_on_batch(p, smp[0]))))
            info, prio, idx = res[0]
            if case.per and k == 0:
                out.append(("update_priorities %s" % p,) + _run(lib, lambda: buf.update_priorities(idx, prio, p)))
    out.append(("soft_update",) + _run(lib, lambda: [pols[p].soft_target_updates() for p in case.ids]))
    out.append(("hard_update",) + _run(lib, lambda: [pols[p].hard_target_updates() for p in case.ids]))
    return out


def qmix_schedule(lib):
    """[(call, kernels, launches)] of the QMIX rollout policy step (greedy and exploring) and the QMIX target updates."""
    import qmix_checks as qc
    from oracle.qmix import QmixConfig
    cfg = QmixConfig(n_agents=3, obs_dim=11, act_dim=5, state_dim=13)
    args, pol, tr = qc.build_trainer(cfg, 4, 5)
    rs = np.random.RandomState(3)
    R = 6
    obs = rs.randn(R, cfg.obs_dim).astype(np.float32)
    avail = (rs.rand(R, cfg.act_dim) < 0.7).astype(np.float32)
    avail[:, 0] = 1
    h = np.zeros((R, cfg.hidden), np.float32)
    torch.manual_seed(5)
    np.random.seed(5)
    return [("policy_step greedy",) + _run(lib, lambda: pol.get_actions(obs, None, h, avail)),
            ("policy_step explore",) + _run(lib, lambda: pol.get_actions(obs, None, h, avail, t_env=20000, explore=True)),
            ("soft_update",) + _run(lib, tr.soft_target_updates),
            ("hard_update",) + _run(lib, tr.hard_target_updates)]


def schedules(lib):
    got = {name: case_schedule(lib, name) for name in sorted(CASES)}
    got["qmix_rollout_targets"] = qmix_schedule(lib)
    return got


@pytest.mark.parametrize("name", sorted(CASES))
def test_entry_point_schedule(emu_engine, name):
    assert case_schedule(emu_engine.lib(), name) == EXPECTED[name]


def test_rollout_and_qmix_target_update_schedule(emu_engine):
    assert qmix_schedule(emu_engine.lib()) == EXPECTED["qmix_rollout_targets"]
