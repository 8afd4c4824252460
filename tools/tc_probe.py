"""GPU probe of the wgmma 3xTF32 building block against an fp64 reference (descriptor-convention check)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "off-policy_b200")):
    sys.path.insert(0, p)
import torch
from offpolicy._b200 import capi

lib = capi.lib()
torch.manual_seed(0)
for (M, N, K) in [(128, 16, 8), (128, 64, 32), (300, 64, 64), (5856, 192, 64), (100, 256, 64)]:
    X = torch.randn(M, K, device="cuda")
    W = torch.randn(N, K, device="cuda") * 0.3
    ref = (X.double() @ W.double().t())
    for swap in (0, 1):
        for passes in (1, 3):
            Y = torch.full((M, N), float("nan"), device="cuda")
            rc = lib.mx_tc_linear_probe(capi.ptr(X), capi.ptr(W), capi.ptr(Y), M, N, K, passes, swap, None)
            torch.cuda.synchronize()
            err = float((Y.double() - ref).abs().max() / ref.abs().max())
            print("M=%d N=%d K=%d swap_ls=%d passes=%d rc=%d  max rel err %.3e  nan=%d" % (M, N, K, swap, passes, rc, err, int(torch.isnan(Y).sum())), flush=True)
