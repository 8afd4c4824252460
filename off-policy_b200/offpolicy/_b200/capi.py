"""ctypes binding of include/marl_b200.h (libmarl_b200.so).

The product path loads ONLY the nvcc-built sm_100a library that lives in-tree at
off-policy_b200/lib/libmarl_b200.so and refuses to run without a CUDA device: there is no CPU
fallback.  (`_install_for_tests` lets the CPU unit tests inject the fiber-emulated build of the same
kernels from tests/emu -- kernel-logic checks only; see tests/emu/emu_runtime.h.)
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_DIR = os.path.normpath(os.path.join(_HERE, "..", "..", "lib"))
LIB_PATH = os.path.join(LIB_DIR, "libmarl_b200.so")

MX_MAX_NAME = 64


class ReplayCfg(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("capacity", "episode_len", "n_agents", "obs_dim", "share_dim", "act_dim", "use_avail",
                                         "use_per", "reward_norm", "max_batch")] + [("per_alpha", C.c_double)]


class ReplayLayout(C.Structure):
    _fields_ = ([(n, C.c_int32) for n in ("obs_ld", "share_ld", "act_ld")] +
                [(n, C.c_int64) for n in ("ep_obs", "ep_share", "ep_acts", "ep_avail", "ep_rew", "ep_dones", "ep_dones_env", "ep_actidx",
                                          "off_obs", "off_share", "off_acts", "off_avail", "off_rew", "off_dones", "off_dones_env",
                                          "off_actidx", "off_sum_tree", "off_min_tree", "off_rng", "off_state", "off_stage",
                                          "stage_bytes", "off_b_obs", "off_b_share", "off_b_acts", "off_b_avail", "off_b_rew",
                                          "off_b_dones", "off_b_dones_env", "off_b_actidx", "off_b_idx", "off_b_weights", "off_b_wf32",
                                          "off_rstats")] +
                [("tree_cap", C.c_int32), ("total_bytes", C.c_int64)])


class Episodes(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("obs", "share_obs", "acts", "rewards", "dones", "dones_env", "avail")]


ABI_VERSION = 5        # MX_ABI_VERSION of include/marl_b200.h the struct mirrors below correspond to


class QmixCfg(C.Structure):
    _fields_ = ([(n, C.c_int32) for n in ("n_agents", "obs_dim", "act_dim", "state_dim", "hidden", "mixer_hidden", "hyper_hidden",
                                          "hyper_layers", "episode_len", "max_batch", "vdn", "double_q", "use_huber", "use_per",
                                          "use_avail", "world_size")] +
                [(n, C.c_float) for n in ("gamma", "huber_delta", "per_nu", "per_eps", "lr", "adam_beta1", "adam_beta2", "adam_eps",
                                          "max_grad_norm", "tau")] + [("prev_act_inp", C.c_int32), ("mlp", C.c_int32), ("no_feature_norm", C.c_int32), ("use_tanh", C.c_int32)])


MAX_ACT_SEG = 4        # MX_MAX_ACT_SEG: MultiDiscrete sub-spaces per agent (mx_maddpg_cfg.act_seg)


class MaddpgCfg(C.Structure):
    _fields_ = ([(n, C.c_int32) for n in ("n_agents", "obs_dim", "act_dim", "state_dim", "hidden", "episode_len", "max_batch", "num_q",
                                          "actor_update_interval", "use_huber", "use_per")] +
                [(n, C.c_float) for n in ("gamma", "huber_delta", "per_nu", "per_eps", "lr", "adam_beta1", "adam_beta2", "adam_eps",
                                          "max_grad_norm", "tau", "weight_decay", "target_noise")] +
                [("discrete", C.c_int32), ("no_feature_norm", C.c_int32), ("use_tanh", C.c_int32), ("cent_act_dim", C.c_int32), ("act_offset", C.c_int32),
                 ("mlp", C.c_int32), ("n_act_seg", C.c_int32), ("act_seg", C.c_int32 * MAX_ACT_SEG)])


class ParamEntry(C.Structure):
    _fields_ = [("name", C.c_char * MX_MAX_NAME), ("offset", C.c_int64), ("rows", C.c_int32), ("cols", C.c_int32)]


class Batch(C.Structure):
    _fields_ = ([(n, C.c_int32) for n in ("B", "obs_ld", "share_ld", "act_ld")] +
                [(n, C.c_void_p) for n in ("obs", "share", "acts", "act_idx", "avail", "rewards", "dones", "dones_env", "weights", "idx")] +
                [("ep_tn_ld", C.c_int32), ("ep_t_ld", C.c_int32)])


class PolicyStepArgs(C.Structure):
    _fields_ = ([("theta", C.c_void_p)] + [(n, C.c_int32) for n in ("in_dim", "out_dim", "rows", "x_ld", "avail_ld")] +
                [(n, C.c_void_p) for n in ("x", "h_in", "h_out", "out", "avail", "greedy", "greedy_q", "h_copy")] + [("mlp", C.c_int32), ("no_feature_norm", C.c_int32), ("use_tanh", C.c_int32)])


TRNG_WORDS = 640      # MX_TRNG_WORDS: the device copy of torch's CPU generator (key[624], left, next)
TRNG_UNIFORM, TRNG_GUMBEL, TRNG_NORMAL = 0, 1, 2
MADDPG_ACTOR, MADDPG_CRITIC = 0, 1    # MX_MADDPG_ACTOR / _CRITIC: the network of a data-parallel exchange
MADDPG_CRITIC_GRADS, MADDPG_CRITIC_APPLY, MADDPG_ACTOR_GRADS, MADDPG_ACTOR_APPLY = 0, 1, 2, 3     # mx_maddpg_step_phase


class TrngDraw(C.Structure):
    _fields_ = ([(n, C.c_int32) for n in ("kind", "T", "rows_n", "rows_b", "cols")] + [("std", C.c_float), ("dst", C.c_void_p)] +
                [(n, C.c_int64) for n in ("ld_t", "ld_n", "ld_b")])


class MxError(RuntimeError):
    pass


_lib = None
_device = None
_is_test_lib = False


def _declare(lib):
    vp, i32, i64, dbl, u32 = C.c_void_p, C.c_int32, C.c_int64, C.c_double, C.c_uint32
    sig = {
        "mx_last_error": (C.c_char_p, []),
        "mx_abi_version": (C.c_int, []),
        "mx_sizeof": (i64, [C.c_char_p]),
        "mx_host_fence_alloc": (C.c_int, []),
        "mx_host_fence_record": (C.c_int, [C.c_int, vp]),
        "mx_host_fence_wait": (C.c_int, [C.c_int]),
        "mx_host_fence_release": (C.c_int, [C.c_int]),
        "mx_is_cuda_build": (C.c_int, []),
        "mx_launch_count": (i64, []),
        "mx_replay_layout_query": (C.c_int, [C.POINTER(ReplayCfg), C.POINTER(ReplayLayout)]),
        "mx_replay_create": (C.c_int, [C.POINTER(ReplayCfg), vp, vp, C.POINTER(vp)]),
        "mx_replay_destroy": (None, [vp]),
        "mx_replay_insert_async": (C.c_int, [vp, C.POINTER(Episodes), i32, C.POINTER(i32), vp]),
        "mx_replay_insert_packed_layout": (i64, [vp, i32, C.POINTER(i64), C.POINTER(i64)]),
        "mx_replay_insert_packed_async": (C.c_int, [vp, vp, i64, i32, C.POINTER(i32), vp]),
        "mx_replay_restore": (C.c_int, [vp, vp]),
        "mx_replay_len": (i32, [vp]),
        "mx_replay_cursor": (i32, [vp]),
        "mx_replay_seed": (C.c_int, [vp, u32, vp]),
        "mx_replay_set_rng_state": (C.c_int, [vp, C.POINTER(u32), i32, vp]),
        "mx_replay_get_rng_state": (C.c_int, [vp, C.POINTER(u32), C.POINTER(i32), vp]),
        "mx_replay_sample_uniform": (C.c_int, [vp, i32, vp]),
        "mx_replay_gather": (C.c_int, [vp, vp, i32, vp]),
        "mx_replay_gather_host": (C.c_int, [vp, vp, i32, vp]),
        "mx_replay_sample_per": (C.c_int, [vp, i32, dbl, vp]),
        "mx_replay_set_beta": (C.c_int, [vp, dbl, vp]),
        "mx_replay_update_priorities": (C.c_int, [vp, vp, vp, vp, vp, i32, vp]),
        "mx_replay_batch": (C.c_int, [vp, i32, C.POINTER(Batch)]),
        "mx_qmix_param_layout": (C.c_int, [C.POINTER(QmixCfg), C.POINTER(ParamEntry), i32, C.POINTER(i64)]),
        "mx_qmix_workspace_bytes": (i64, [C.POINTER(QmixCfg)]),
        "mx_qmix_create": (C.c_int, [C.POINTER(QmixCfg), vp, vp, vp, vp, vp, i64, C.POINTER(vp)]),
        "mx_qmix_destroy": (None, [vp]),
        "mx_qmix_step": (C.c_int, [vp, C.POINTER(Batch), vp]),
        "mx_qmix_step_ex": (C.c_int, [vp, C.POINTER(Batch), u32, vp]),
        "mx_qmix_apply_ex": (C.c_int, [vp, u32, vp]),
        "mx_qmix_set_debug": (C.c_int, [vp, i32]),
        "mx_qmix_backward_only": (C.c_int, [vp, C.POINTER(Batch), vp]),
        "mx_qmix_apply": (C.c_int, [vp, vp]),
        "mx_qmix_grad_buffer": (vp, [vp, C.POINTER(i64)]),
        "mx_qmix_info": (vp, [vp]),
        "mx_qmix_priorities": (vp, [vp]),
        "mx_qmix_p2p_block_bytes": (i64, [vp]),
        "mx_qmix_set_peers": (C.c_int, [vp, i32, i32, C.POINTER(vp), vp]),
        "mx_qmix_p2p_publish": (C.c_int, [vp, vp]),
        "mx_qmix_p2p_reduce": (C.c_int, [vp, vp]),
        "mx_qmix_soft_update": (C.c_int, [vp, vp]),
        "mx_qmix_hard_update": (C.c_int, [vp, vp]),
        "mx_qmix_ws_lookup": (C.c_int, [vp, C.c_char_p, C.POINTER(i64), C.POINTER(i64)]),
        "mx_maddpg_param_layout": (C.c_int, [C.POINTER(MaddpgCfg), i32, C.POINTER(ParamEntry), i32, C.POINTER(i64)]),
        "mx_maddpg_workspace_bytes": (i64, [C.POINTER(MaddpgCfg)]),
        "mx_maddpg_create": (C.c_int, [C.POINTER(MaddpgCfg), C.POINTER(vp), C.POINTER(vp), vp, i64, C.POINTER(vp)]),
        "mx_maddpg_destroy": (None, [vp]),
        "mx_maddpg_step": (C.c_int, [vp, C.POINTER(Batch), vp, C.POINTER(i32), vp]),
        "mx_maddpg_step_ex": (C.c_int, [vp, C.POINTER(Batch), vp, vp, C.POINTER(i32), vp]),
        "mx_maddpg_cent_contribute": (C.c_int, [vp, C.POINTER(Batch), vp, vp, vp]),
        "mx_maddpg_step_phase": (C.c_int, [vp, i32, C.POINTER(Batch), vp, vp, C.POINTER(i32), vp]),
        "mx_maddpg_p2p_block_bytes": (i64, [vp, i32]),
        "mx_maddpg_set_peers": (C.c_int, [vp, i32, i32, i32, C.POINTER(vp), vp]),
        "mx_maddpg_p2p_publish": (C.c_int, [vp, i32, vp]),
        "mx_maddpg_p2p_reduce": (C.c_int, [vp, i32, vp]),
        "mx_maddpg_grad_buffer": (vp, [vp, i32, C.POINTER(i64)]),
        "mx_maddpg_info": (vp, [vp]),
        "mx_maddpg_priorities": (vp, [vp]),
        "mx_maddpg_grad_views": (C.c_int, [vp, C.POINTER(i64), C.POINTER(i64)]),
        "mx_maddpg_soft_update": (C.c_int, [vp, vp]),
        "mx_maddpg_hard_update": (C.c_int, [vp, vp]),
        "mx_policy_step": (C.c_int, [C.POINTER(PolicyStepArgs), vp]),
        "mx_set_option": (C.c_int, [C.c_char_p, i32]),
        "mx_tc_linear_probe": (C.c_int, [vp, vp, vp, i32, i32, i32, i32, i32, vp]),
        "mx_maddpg_graph_capture": (C.c_int, [vp, vp, i32, dbl, u32, vp, vp, i32, vp, C.POINTER(vp)]),
        "mx_maddpg_graph_capture_ex": (C.c_int, [vp, vp, i32, dbl, u32, vp, vp, i32, vp, C.POINTER(TrngDraw), i32, vp, i64, vp,
                                                 C.POINTER(vp)]),
        "mx_maddpg_batch_graph_capture": (C.c_int, [vp, vp, i32, i32, i32, dbl, u32, vp, vp, i32, vp, C.POINTER(TrngDraw), vp, vp, i64,
                                                    vp, C.POINTER(vp)]),
        "mx_trng_seed": (C.c_int, [vp, C.c_uint64, vp]),
        "mx_trng_set_state": (C.c_int, [vp, C.POINTER(u32), i32, i32, vp]),
        "mx_trng_get_state": (C.c_int, [vp, C.POINTER(u32), C.POINTER(i32), C.POINTER(i32), vp]),
        "mx_trng_words": (i64, [C.POINTER(TrngDraw)]),
        "mx_trng_fill": (C.c_int, [vp, C.POINTER(TrngDraw), vp, i64, vp]),
        "mx_maddpg_num_updates": (i64, [vp]),
        "mx_maddpg_set_num_updates": (C.c_int, [vp, i64]),
        "mx_maddpg_ws_lookup": (C.c_int, [vp, C.c_char_p, C.POINTER(i64), C.POINTER(i64)]),
        "mx_maddpg_set_valid": (C.c_int, [vp, vp]),
        "mx_graph_capture": (C.c_int, [vp, vp, i32, dbl, u32, vp, C.POINTER(vp)]),
        "mx_graph_launch": (C.c_int, [vp, vp]),
        "mx_graph_destroy": (None, [vp]),
        "mx_graph_num_kernels": (i32, [vp]),
        "mx_profile_begin": (C.c_int, [vp]),
        "mx_profile_end": (C.c_int, [vp, C.c_char_p, i32, C.POINTER(C.c_float), i32]),
    }
    missing = []
    for name, (res, args) in sig.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            missing.append(name)
            continue
        fn.restype = res
        fn.argtypes = args
    if missing:
        raise MxError("libmarl_b200 is missing symbols declared in include/marl_b200.h: %s" % ", ".join(missing))
    if int(lib.mx_abi_version()) != ABI_VERSION:      # the ctypes mirrors of the structs above were written for this version
        raise MxError("libmarl_b200 reports ABI version %d, these bindings expect %d: rebuild (python __graft_entry__.py build)"
                      % (int(lib.mx_abi_version()), ABI_VERSION))
    return lib


EXPORTED_SYMBOLS = None  # filled by tests from the header


def lib():
    """The CUDA library.  Raises (never falls back) when it is missing or there is no GPU."""
    global _lib, _device
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise MxError("libmarl_b200.so not built: run `python __graft_entry__.py build` (expected %s)" % LIB_PATH)
    if not torch.cuda.is_available():
        raise MxError("marl_b200: no CUDA device visible; this engine has no CPU path")
    handle = _declare(C.CDLL(LIB_PATH))
    if handle.mx_is_cuda_build() != 1:
        raise MxError("marl_b200: %s is not the nvcc sm_90a build" % LIB_PATH)
    _lib = handle
    _device = torch.device("cuda", torch.cuda.current_device())
    return _lib


def load_symbols_only(path=LIB_PATH):
    """dlopen + symbol check without touching a GPU (used by the CPU test that the C-ABI exports everything)."""
    return _declare(C.CDLL(path))


def _install_for_tests(path):
    """TEST HOOK: bind the CPU fiber-emulated build (tests/emu).  Never called by product code."""
    global _lib, _device, _is_test_lib
    _lib = _declare(C.CDLL(path))
    _device = torch.device("cpu")
    _is_test_lib = True
    return _lib


def _uninstall_for_tests():
    global _lib, _device, _is_test_lib
    _lib = None
    _device = None
    _is_test_lib = False


def device():
    lib()
    return _device


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None) or (lambda i: torch.cuda.current_stream(i).cuda_stream)


def stream_ptr():
    """cudaStream_t of torch's current stream (torch is plumbing: memory + streams)."""
    if _device is None or _device.type != "cuda":
        return None
    return C.c_void_p(_raw_stream(_device.index or 0))          # (torch.cuda.current_stream() builds a Stream object: ~3 us)


def check(rc):
    if rc != 0:
        raise MxError(lib().mx_last_error().decode())


def ptr(t, byte_offset=0):
    return C.c_void_p(t.data_ptr() + byte_offset) if t is not None else C.c_void_p(0)
