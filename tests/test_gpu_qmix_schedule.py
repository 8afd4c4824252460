"""The QMIX / VDN / M-QMIX step's fork / join structure on the device: one product-configuration step captured as a CUDA graph, its
kernel nodes by name and the dependency edges between them.

The emulator runs the step on one stream (tests/test_emu_qmix_schedule.py pins its kernel order).  On the device the state-only
kernels (mixer hypernetworks, GRU weight gradients) run on a forked branch, which only the captured graph shows.  The library launches
on torch's current stream, so torch.cuda.CUDAGraph captures the step exactly as the library enqueues it; the graph is read through the
CUDA driver API.  Each structure below was recorded from the step as it stood before its launches were rebuilt around one step
builder (qmix.cu Step)."""
import ctypes as C
import re

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# name: (learner, n_agents, obs, actions, state, T, B, PER, availability masks) -- the bench.py workloads of the same names, VDN at
# the qmix_3m shape, and the wide-state mixer (state 448) at the qmix_3m shape
SHAPES = {
    "qmix_3m": ("qmix", 3, 30, 9, 48, 60, 32, False, True),
    "qmix_8m_per": ("qmix", 8, 80, 14, 168, 120, 64, True, True),
    "qmix_2s3z": ("qmix", 5, 80, 11, 120, 120, 32, False, True),
    "qmix_mpe_spread": ("qmix", 3, 18, 5, 54, 25, 32, False, False),
    "mqmix_mpe_spread": ("mqmix", 3, 18, 5, 54, 1, 1000, False, False),
    "vdn_3m": ("vdn", 3, 30, 9, 48, 60, 32, False, True),
    "qmix_wide_state": ("qmix", 3, 30, 9, 448, 60, 32, False, True),
}

EXPECTED = {
    "mqmix_mpe_spread": (
        ["k_front_bwd<3>", "k_front_fwd_tc2", "k_mix_core", "k_mix_hyper_bwd<1,0>", "k_mix_hyper_fwd<1,0>", "k_mlp_dgi", "k_mlp_qselect", "k_optim_fused", "k_tc_prep_weights"],
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
        ["k_front_bwd_tc", "k_front_fwd_tc_wide2", "k_gru_bwd2<1>", "k_gru_fwd2<1>", "k_mid<16,1>", "k_mix_hyper_bwd<2,0>", "k_mix_hyper_fwd<2,0>", "k_optim_fused", "k_tc_prep_weights", "k_tc_prep_weights_T", "k_wgrad_tc"],
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
        ["k_front_bwd<3>", "k_front_fwd_tc2", "k_gru_bwd2<1>", "k_gru_fwd2<1>", "k_gru_wgrad<3>", "k_mid<16,1>", "k_mix_hyper_bwd<1,0>", "k_mix_hyper_fwd<1,0>", "k_optim_fused", "k_tc_prep_weights"],
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
        ["k_front_bwd_tc", "k_front_fwd_tc_wide2", "k_gru_bwd2<1>", "k_gru_fwd2<1>", "k_mid<8,1>", "k_mix_hyper_bwd<2,0>", "k_mix_hyper_fwd<2,0>", "k_optim_fused", "k_tc_prep_weights", "k_tc_prep_weights_T", "k_wgrad_tc"],
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
        ["k_front_bwd<2>", "k_front_fwd_tc2", "k_gru_bwd2<1>", "k_gru_fwd2<1>", "k_gru_wgrad<2>", "k_mid<16,1>", "k_mix_hyper_bwd<1,0>", "k_mix_hyper_fwd<1,0>", "k_optim_fused", "k_tc_prep_weights"],
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
        ["k_front_bwd<3>", "k_front_fwd_tc2", "k_gru_bwd2<1>", "k_gru_fwd2<1>", "k_gru_wgrad<3>", "k_mid<16,1>", "k_mix_hyper_bwd<1,1>", "k_mix_hyper_fwd<1,1>", "k_mixw_fwd", "k_mixw_prep", "k_mixw_wgrad", "k_optim_fused", "k_tc_prep_weights"],
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
    "vdn_3m": (
        ["k_front_bwd<3>", "k_front_fwd_tc2", "k_gru_bwd2<1>", "k_gru_fwd2<1>", "k_gru_wgrad<3>", "k_optim_fused", "k_qhead<1>", "k_qhead_bwd<1>", "k_tc_prep_weights", "k_vdn_mix"],
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


# ---- reading a captured graph (CUDA driver API) -------------------------------------------------------------------------------
class _KernelNodeParams(C.Structure):       # CUDA_KERNEL_NODE_PARAMS_v2
    _fields_ = [("func", C.c_void_p), ("grid", C.c_uint * 3), ("block", C.c_uint * 3), ("smem", C.c_uint),
                ("kernelParams", C.c_void_p), ("extra", C.c_void_p), ("kern", C.c_void_p), ("ctx", C.c_void_p)]


class _EdgeData(C.Structure):               # CUgraphEdgeData
    _fields_ = [("from_port", C.c_ubyte), ("to_port", C.c_ubyte), ("type", C.c_ubyte), ("reserved", C.c_ubyte * 5)]


_NODE_TYPES = {0: "kernel", 1: "memcpy", 2: "memset", 3: "host", 4: "graph", 5: "empty", 6: "wait_event", 7: "event_record",
               8: "ext_semas_signal", 9: "ext_semas_wait", 10: "mem_alloc", 11: "mem_free", 12: "batch_mem_op", 13: "conditional"}


def _check(rc, what):
    assert rc == 0, "%s failed: CUresult %d" % (what, rc)


def kernel_name(mangled):
    """`k_mid<16,1>` from `_Z5k_midILi16ELi1EEv7MidArgs7MidSmem`: the function name and its integer template arguments."""
    m = re.match(r"_Z(\d+)", mangled)
    if not m:
        return mangled
    n = int(m.group(1))
    name, rest = mangled[m.end():m.end() + n], mangled[m.end() + n:]
    t = re.match(r"I((?:L[a-z]n?\d+E)+)E", rest)
    if t:
        name += "<%s>" % ",".join(v.replace("n", "-") for v in re.findall(r"L[a-z](n?\d+)E", t.group(1)))
    return name


def graph_structure(graph):
    """(sorted node names, sorted edges "a -> b") of a cudaGraph_t.  Kernel nodes are named by their function, other nodes by their
    type; an edge that is not a plain full dependency (programmatic dependent launch) carries its ports and type."""
    cu = C.CDLL("libcuda.so.1")
    g = C.c_void_p(graph)
    n = C.c_size_t(0)
    _check(cu.cuGraphGetNodes(g, None, C.byref(n)), "cuGraphGetNodes")
    nodes = (C.c_void_p * max(n.value, 1))()
    _check(cu.cuGraphGetNodes(g, nodes, C.byref(n)), "cuGraphGetNodes")
    names = {}
    for i in range(n.value):
        ty = C.c_int(-1)
        _check(cu.cuGraphNodeGetType(C.c_void_p(nodes[i]), C.byref(ty)), "cuGraphNodeGetType")
        if ty.value != 0:
            names[nodes[i]] = _NODE_TYPES.get(ty.value, "type%d" % ty.value)
            continue
        p = _KernelNodeParams()
        _check(cu.cuGraphKernelNodeGetParams_v2(C.c_void_p(nodes[i]), C.byref(p)), "cuGraphKernelNodeGetParams")
        s = C.c_char_p()
        if p.func:
            _check(cu.cuFuncGetName(C.byref(s), C.c_void_p(p.func)), "cuFuncGetName")
        else:
            _check(cu.cuKernelGetName(C.byref(s), C.c_void_p(p.kern)), "cuKernelGetName")
        names[nodes[i]] = kernel_name(s.value.decode())
    m = C.c_size_t(0)
    _check(cu.cuGraphGetEdges_v2(g, None, None, None, C.byref(m)), "cuGraphGetEdges")
    k = max(m.value, 1)
    src, dst, data = (C.c_void_p * k)(), (C.c_void_p * k)(), (_EdgeData * k)()
    _check(cu.cuGraphGetEdges_v2(g, src, dst, data, C.byref(m)), "cuGraphGetEdges")
    edges = []
    for i in range(m.value):
        e = "%s -> %s" % (names[src[i]], names[dst[i]])
        d = data[i]
        if d.from_port or d.to_port or d.type:
            e += " [%d,%d,%d]" % (d.from_port, d.to_port, d.type)
        edges.append(e)
    return sorted(names.values()), sorted(edges)


# ---- one captured step ----------------------------------------------------------------------------------------------------------
def capture_step(name):
    """The graph of one learner step of shape `name` (product configuration), as graph_structure().  The batch is a device copy of a
    synthetic one (no replay buffer: the step is all the graph holds)."""
    import contextlib
    import io
    from oracle.qmix import QmixConfig, synth_batch
    from oracle.mqmix import synth_transitions
    from offpolicy._b200 import capi, factory
    import mqmix_checks as mc
    import qmix_checks as qc
    learner, N, O, A, S, T, B, per, avail = SHAPES[name]
    cfg = QmixConfig(n_agents=N, obs_dim=O, act_dim=A, state_dim=S, use_per=per, gain=1.0)
    lib = capi.lib()
    weights = (np.random.RandomState(1).rand(B) * 0.9 + 0.1, np.arange(B)) if per else (None, None)
    with contextlib.redirect_stdout(io.StringIO()):
        if learner == "mqmix":
            args, pol, tr = mc.build(cfg, B, debug=False)
            batch = mc._to_dicts(synth_transitions(cfg, B, seed=5, avail=avail), weights[0])
            tr.train_policy_on_batch(batch, True)      # first launches (module loading, smem attributes) outside the capture
            b = tr._host_batch.pack(batch, "policy_0", per)
        else:
            args, pol, tr = factory.build_qmix(cfg, B, T, vdn=learner == "vdn", debug=False)
            batch = list(qc.ref_tuple(synth_batch(cfg, B, T, seed=5, avail_p=0.8, var_len=True) + weights))
            if not avail:
                batch[6] = None
            tr.train_policy_on_batch(batch)
            b = tr._device_batch(batch)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph(keep_graph=True)
    with torch.cuda.graph(g):
        capi.check(lib.mx_qmix_step(tr.handle, C.byref(b), capi.stream_ptr()))
    try:
        return graph_structure(g.raw_cuda_graph())
    finally:
        g.reset()
        torch.cuda.synchronize()


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_captured_step_fork_join_structure(gpu_engine, name):
    nodes, edges = capture_step(name)
    want_nodes, want_edges = EXPECTED[name]
    assert nodes == want_nodes, (name, nodes)
    assert edges == want_edges, (name, edges)
