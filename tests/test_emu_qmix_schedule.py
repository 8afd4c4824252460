"""The QMIX / VDN / M-QMIX / M-VDN step's launch schedule on the CPU fiber emulator: the exact kernel sequence of one learner step,
per configuration.

The emulator runs the step serially on one stream (no forked branch), with the split mixer it would fork on a device, so the order is
the device's caller-stream order with the side branch's kernels in line.  Each sequence below was recorded from the step as it stood
before its launches were rebuilt around one step builder (qmix.cu Step); a change to the schedule has to change them on purpose."""
import pytest

import qmix_checks as qc
import mqmix_checks as mc
import row_coverage_checks as rc

# name: (learner, QmixConfig overrides, debug, options) -> the kernels of one step.  Default shape: 3 agents, obs 11, 5 actions,
# state 13, B 4, T 5 (M-QMIX / M-VDN: B 4 transitions).
CASES = {
    # product (debug outputs off): k_mid between the recurrences; debug keeps k_qhead / k_mix_core / k_qhead_bwd
    "qmix_product": ("qmix", {}, False, {},
                     "k_tc_prep_weights k_front_fwd_tc k_gru_fwd k_mix_hyper_fwd k_mid k_mix_hyper_bwd k_gru_bwd k_gru_wgrad k_front_bwd "
                     "k_optim_fused"),
    "qmix_debug": ("qmix", {}, True, {},
                   "k_tc_prep_weights k_front_fwd_tc k_gru_fwd k_qhead k_mix_hyper_fwd k_mix_core k_mix_hyper_bwd k_qhead_bwd k_gru_bwd "
                   "k_gru_wgrad k_front_bwd k_optim_fused"),
    "qmix_hyper1_product": ("qmix", dict(hyper_layers=1), False, {},
                            "k_tc_prep_weights k_front_fwd_tc k_gru_fwd k_mix_hyper_fwd k_mid k_mix_hyper_bwd k_gru_bwd "
                            "k_gru_wgrad k_front_bwd k_optim_fused"),
    "qmix_hyper1_debug": ("qmix", dict(hyper_layers=1), True, {},
                          "k_tc_prep_weights k_front_fwd_tc k_gru_fwd k_qhead k_mix_hyper_fwd k_mix_core k_mix_hyper_bwd "
                          "k_qhead_bwd k_gru_bwd k_gru_wgrad k_front_bwd k_optim_fused"),
    "vdn_product": ("vdn", {}, False, {},
                    "k_tc_prep_weights k_front_fwd_tc k_gru_fwd k_qhead k_vdn_mix k_qhead_bwd k_gru_bwd k_gru_wgrad k_front_bwd k_optim_fused"),
    "vdn_debug": ("vdn", {}, True, {},
                  "k_tc_prep_weights k_front_fwd_tc k_gru_fwd k_qhead k_vdn_mix k_qhead_bwd k_gru_bwd k_gru_wgrad k_front_bwd "
                  "k_optim_fused"),
    "mqmix_product": ("mqmix", {}, False, {},
                      "k_tc_prep_weights k_front_fwd_tc k_mlp_qselect k_mix_hyper_fwd k_mix_core k_mix_hyper_bwd k_mlp_dgi "
                      "k_front_bwd k_optim_fused"),
    "mqmix_debug": ("mqmix", {}, True, {},
                    "k_tc_prep_weights k_front_fwd_tc k_mlp_qselect k_mix_hyper_fwd k_mix_core k_mix_hyper_bwd k_mlp_dgi "
                    "k_front_bwd k_optim_fused"),
    "mvdn_product": ("mvdn", {}, False, {},
                     "k_tc_prep_weights k_front_fwd_tc k_mlp_qselect k_vdn_mix k_mlp_dgi k_front_bwd k_optim_fused"),
    "prev_act_product": ("qmix", dict(prev_act_inp=True), False, {},
                         "k_pack_prev_act k_tc_prep_weights k_front_fwd_tc k_gru_fwd k_mix_hyper_fwd k_mid k_mix_hyper_bwd "
                         "k_gru_bwd k_gru_wgrad k_front_bwd k_optim_fused"),
    # observation widths: <= 56 above; 57..64 the one-thread-per-row front forward; 81..128 the wide forward and the tensor-core backward
    "obs60_product": ("qmix", dict(obs_dim=60), False, {},
                      "k_tc_prep_weights k_front_fwd_tc1 k_gru_fwd k_mix_hyper_fwd k_mid k_mix_hyper_bwd k_gru_bwd k_gru_wgrad "
                      "k_front_bwd k_optim_fused"),
    "obs120_product": ("qmix", dict(obs_dim=120), False, {},
                       "k_tc_prep_weights k_tc_prep_weights_T k_front_fwd_tc_wide k_gru_fwd k_mix_hyper_fwd k_mid k_mix_hyper_bwd k_gru_bwd "
                       "k_front_bwd_tc k_wgrad_tc k_optim_fused"),
    "obs120_debug": ("qmix", dict(obs_dim=120), True, {},
                     "k_tc_prep_weights k_tc_prep_weights_T k_front_fwd_tc_wide k_gru_fwd k_qhead k_mix_hyper_fwd k_mix_core "
                     "k_mix_hyper_bwd k_qhead_bwd k_gru_bwd k_front_bwd_tc k_wgrad_tc k_optim_fused"),
    # two actions per lane in the Q-head kernels; SMAC 8m widths take the 8-warp k_mid; at 8 agents x 64 actions k_mid does not fit
    "a36_product": ("qmix", dict(act_dim=36), False, {},
                    "k_tc_prep_weights k_front_fwd_tc k_gru_fwd k_mix_hyper_fwd k_mid k_mix_hyper_bwd k_gru_bwd k_gru_wgrad "
                    "k_front_bwd k_optim_fused"),
    "a64_product": ("qmix", dict(act_dim=64), False, {},
                    "k_tc_prep_weights k_front_fwd_tc k_gru_fwd k_mix_hyper_fwd k_mid k_mix_hyper_bwd k_gru_bwd k_gru_wgrad "
                    "k_front_bwd k_optim_fused"),
    "n8_a14_product": ("qmix", dict(n_agents=8, act_dim=14), False, {},
                       "k_tc_prep_weights k_front_fwd_tc k_gru_fwd k_mix_hyper_fwd k_mid k_mix_hyper_bwd k_gru_bwd k_gru_wgrad "
                       "k_front_bwd k_optim_fused"),
    "n8_a64_product": ("qmix", dict(n_agents=8, act_dim=64), False, {},
                       "k_tc_prep_weights k_front_fwd_tc k_gru_fwd k_qhead k_mix_hyper_fwd k_mix_core k_mix_hyper_bwd k_qhead_bwd "
                       "k_gru_bwd k_gru_wgrad k_front_bwd k_optim_fused"),
    # wide global state: the hypernetworks' state layers on the tensor cores, always the split pipeline
    "wide_state_product": ("qmix", dict(state_dim=448), False, {},
                           "k_tc_prep_weights k_front_fwd_tc k_gru_fwd k_mixw_prep k_mixw_fwd k_mix_hyper_fwd_wide k_mid k_mix_hyper_bwd_wide "
                           "k_mixw_wgrad k_gru_bwd k_gru_wgrad k_front_bwd k_optim_fused"),
    "wide_state_debug": ("qmix", dict(state_dim=448), True, {},
                         "k_tc_prep_weights k_front_fwd_tc k_gru_fwd k_qhead k_mixw_prep k_mixw_fwd k_mix_hyper_fwd_wide "
                         "k_mix_core k_mix_hyper_bwd_wide k_mixw_wgrad k_qhead_bwd k_gru_bwd k_gru_wgrad k_front_bwd "
                         "k_optim_fused"),
    # the options: fused k_mixer, the split pipeline forced, k_mid off
    "mixer_split0": ("qmix", {}, False, dict(mixer_split=0),
                     "k_tc_prep_weights k_front_fwd_tc k_gru_fwd k_qhead k_mixer k_qhead_bwd k_gru_bwd k_gru_wgrad k_front_bwd k_optim_fused"),
    "mixer_split2": ("qmix", {}, False, dict(mixer_split=2),
                     "k_tc_prep_weights k_front_fwd_tc k_gru_fwd k_mix_hyper_fwd k_mid k_mix_hyper_bwd k_gru_bwd k_gru_wgrad "
                     "k_front_bwd k_optim_fused"),
    "mid_fused0": ("qmix", {}, False, dict(mid_fused=0),
                   "k_tc_prep_weights k_front_fwd_tc k_gru_fwd k_qhead k_mix_hyper_fwd k_mix_core k_mix_hyper_bwd k_qhead_bwd "
                   "k_gru_bwd k_gru_wgrad k_front_bwd k_optim_fused"),
    "mqmix_mixer_split0": ("mqmix", {}, False, dict(mixer_split=0),
                           "k_tc_prep_weights k_front_fwd_tc k_mlp_qselect k_mixer k_mlp_dgi k_front_bwd k_optim_fused"),
    "wide_state_mixer_split0": ("qmix", dict(state_dim=448), False, dict(mixer_split=0),
                                "k_tc_prep_weights k_front_fwd_tc k_gru_fwd k_mixw_prep k_mixw_fwd k_mix_hyper_fwd_wide k_mid "
                                "k_mix_hyper_bwd_wide k_mixw_wgrad k_gru_bwd k_gru_wgrad k_front_bwd k_optim_fused"),
}
DEFAULT_OPTIONS = dict(mixer_split=1, mid_fused=1)


def _cfg(over):
    from oracle.qmix import QmixConfig
    base = dict(n_agents=3, obs_dim=11, act_dim=5, state_dim=13, gain=1.0)
    base.update(over)
    return QmixConfig(**base)


def _one_step(lib, learner, cfg, debug, B=4, T=5):
    """The names of the kernels one learner step launches."""
    if learner in ("qmix", "vdn"):
        from oracle.qmix import synth_batch
        args, pol, tr = qc.build_trainer(cfg, B, T, vdn=learner == "vdn", debug=debug)
        batch = qc.ref_tuple(synth_batch(cfg, B, T, seed=5, avail_p=0.8, var_len=True) + (None, None))
        return rc.kernels_run(lib, None, lambda: tr.train_policy_on_batch(batch))
    from oracle.mqmix import synth_transitions
    from offpolicy._b200 import capi
    if learner == "mqmix":
        args, pol, tr = mc.build(cfg, B, debug=debug)
    else:
        from offpolicy.algorithms.mvdn.algorithm.mVDNPolicy import M_VDNPolicy
        from offpolicy.algorithms.mvdn.mvdn import M_VDN
        from replay_checks import Discrete
        N, O, A, S = cfg.n_agents, cfg.obs_dim, cfg.act_dim, cfg.state_dim
        args = qc.make_args(cfg, B)
        info = dict(obs_space=[O], share_obs_space=[S], act_space=Discrete(A), cent_obs_dim=S, cent_act_dim=A * N)
        pol = M_VDNPolicy({"args": args, "device": capi.device()}, info)
        tr = M_VDN(args, N, {"policy_0": pol}, lambda a: "policy_0", device=capi.device())
        lib.mx_qmix_set_debug(tr.handle, 1 if debug else 0)
    batch = mc._to_dicts(synth_transitions(cfg, B, seed=5, avail=True))
    return rc.kernels_run(lib, None, lambda: tr.train_policy_on_batch(batch, True))


def step_kernels(lib, name):
    learner, over, debug, options, _ = CASES[name]
    if learner in ("vdn", "mvdn"):
        over = dict(over, vdn=True)
    try:
        for k, v in options.items():
            assert lib.mx_set_option(k.encode(), v) == 0, k
        return _one_step(lib, learner, _cfg(over), debug)
    finally:
        for k, v in DEFAULT_OPTIONS.items():
            lib.mx_set_option(k.encode(), v)


@pytest.mark.parametrize("name", sorted(CASES))
def test_step_kernel_sequence(emu_engine, name):
    names = step_kernels(emu_engine.lib(), name)
    assert " ".join(names) == CASES[name][4], (name, names)
