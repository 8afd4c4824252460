"""Tensor-core (wgmma) path: the 3xTF32 building block against fp64, then the whole QMIX step with the
time-batched front layers routed through k_front_fwd_tc, against the reference goldens and the oracle."""
import numpy as np
import pytest
import torch

import qmix_checks as qc

pytestmark = pytest.mark.gpu


def probe(capi, M, N, K, passes, swap):
    lib = capi.lib()
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N)
    X = torch.randn(M, K, device="cuda", generator=g)
    W = torch.randn(N, K, device="cuda", generator=g) * 0.3
    Y = torch.full((M, N), float("nan"), device="cuda")
    capi.check(lib.mx_tc_linear_probe(capi.ptr(X), capi.ptr(W), capi.ptr(Y), M, N, K, passes, swap, None))
    torch.cuda.synchronize()
    ref = X.double() @ W.double().t()
    return float((Y.double() - ref).abs().max() / ref.abs().max())


def detect_swap(capi):
    errs = [probe(capi, 256, 64, 64, 3, s) for s in (0, 1)]
    good = [s for s in (0, 1) if errs[s] < 1e-5]
    assert good, "neither descriptor convention reproduces the fp64 product: %r" % (errs,)
    return good[0]


def test_3xtf32_building_block_matches_fp64(gpu_engine):
    swap = detect_swap(gpu_engine)
    for (M, N, K) in [(128, 16, 8), (128, 64, 32), (300, 64, 64), (5856, 192, 64), (100, 256, 64)]:
        e3 = probe(gpu_engine, M, N, K, 3, swap)
        e1 = probe(gpu_engine, M, N, K, 1, swap)
        assert e3 < 2e-6, (M, N, K, e3)          # fp32-level
        assert 1e-5 < e1 < 5e-3, (M, N, K, e1)   # plain TF32 really is ~1e-3: the split is what buys the parity budget


@pytest.mark.parametrize("front_tc", [1, 0])
@pytest.mark.parametrize("name", ["qmix_small", "qmix_5ag"])
def test_qmix_step_front_paths_match_reference_golden(gpu_engine, name, front_tc):
    """The tensor-core front kernel is the default; the FFMA kernel stays selectable and both must hold parity."""
    lib = gpu_engine.lib()
    assert detect_swap(gpu_engine) == 0          # the convention compiled in as the default
    lib.mx_set_option(b"front_tc", front_tc)
    try:
        qc.check_step_against(None, name)
    finally:
        lib.mx_set_option(b"front_tc", 1)


def test_config2_full_size_with_tensor_core_front_vs_oracle(gpu_engine):
    from test_gpu_qmix import _oracle_and_trainer, _compare_step
    from oracle.qmix import QmixConfig, synth_batch
    lib = gpu_engine.lib()
    lib.mx_set_option(b"front_tc", 1)
    try:
        torch.set_num_threads(8)
        cfg = QmixConfig(gain=1.0)
        L, args, pol, tr = _oracle_and_trainer(cfg, 32, 60)
        batch = synth_batch(cfg, 32, 60, seed=5, avail_p=0.8, var_len=True) + (None, None)
        _compare_step(L, pol, tr, batch, cfg, steps=2)
    finally:
        lib.mx_set_option(b"front_tc", 1)
