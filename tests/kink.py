"""ReLU-kink-aware gradient comparison (test infrastructure).

A ReLU network's gradient is discontinuous where a pre-activation crosses zero.  With ~10^5..10^6 hidden units per learner step a
few pre-activations land within round-off of zero; the engine (3xTF32 tensor-core or FFMA accumulation order) and the fp32 oracle
then legitimately pick different sides, and that single (row, unit) changes a gradient tensor by ~1/rows of its magnitude -- far
above the 1e-4 budget although both are exact gradients of the same function at a valid sub-gradient.  When a plain comparison
fails, `redo_with_engine_masks` re-runs the oracle step from the saved pre-step state with the backward masks of the live agent's two
ReLU layers forced to the ENGINE's (u > 0 of the activations the engine saved), and reports how many units were flipped and how far
from the kink they were.  The caller then demands (a) every flipped unit had |pre-activation| below `KINK_TOL` in the oracle and
(b) the 1e-4 comparison passes against the re-run.  A real kernel error cannot pass: it either flips no unit or flips units far
from zero, or still disagrees afterwards.

The QMIX mixer's |hyper_w1(s)| and |hyper_w2(s)| have the same kind of kink at zero: `resolve_abs_kinks` settles the hypernet outputs
within `ABS_KINK_TOL` of zero in the float64 reference of a whole-batch gradient comparison.
"""
import copy

import torch

KINK_TOL = 3e-5          # ~30x the 3xTF32 absolute error of a K<=128 dot product of O(1) operands


class _ForcedReLU(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, mask):
        ctx.save_for_backward(mask)
        return torch.relu(x)

    @staticmethod
    def backward(ctx, g):
        (mask,) = ctx.saved_tensors
        return g * mask, None


def _relu_modules(agent):
    base = agent.rnn if hasattr(agent, "rnn") else agent.mlp        # oracle.qmix._RNNBase / oracle.mqmix._MLPBase
    m = base.mlp
    return [m.fc1[1], m.fc2[0][1]]


def engine_masks(tr, B, T, N, mlp):
    """(u1 > 0, u2 > 0) of the engine's saved post-ReLU activations, in the oracle's row order."""
    out = []
    M = B * (T + 1) * N
    for name in ("u1", "u2"):
        u = tr.ws_view(name)[:M * 64].view(B, T + 1, N, 64).cpu()
        if mlp:
            u = u[:, 0].permute(1, 0, 2).reshape(N * B, 64)                      # oracle rows n*B + b of the step-0 call
        else:
            u = u.permute(1, 2, 0, 3).reshape(T + 1, N * B, 64)                  # oracle (T+1, n*B + b, .)
        out.append((u > 0).float())
    return out


def redo_with_engine_masks(L0, step_fn, masks):
    """Run `step_fn(L0)` (one oracle step) with the live agent's ReLU backward masks forced; returns (result, n_flipped, max |pre| of a flip)."""
    stats = {"flips": 0, "max_pre": 0.0, "used": 0}
    hooks = []
    for mod, mask in zip(_relu_modules(L0.agent), masks):
        def hook(_m, inp, _out, mask=mask):
            x = inp[0]
            if torch.is_grad_enabled() and x.requires_grad and x.shape == mask.shape:
                diff = (x.detach() > 0).float() != mask
                stats["used"] += 1
                stats["flips"] += int(diff.sum())
                if diff.any():
                    stats["max_pre"] = max(stats["max_pre"], float(x.detach().abs()[diff].max()))
                return _ForcedReLU.apply(x, mask)
            return None
        hooks.append(mod.register_forward_hook(hook))
    try:
        res = step_fn(L0)
    finally:
        for h in hooks:
            h.remove()
    assert stats["used"] == 2, "forced-mask hooks did not see the live agent's forward (shape mismatch?)"
    return res, stats["flips"], stats["max_pre"]


def snapshot(L):
    return copy.deepcopy(L)


def adopt(L, L2):
    """Continue the lock-step run from the re-run's state."""
    L.__dict__.update(L2.__dict__)


ABS_KINK_TOL = 1e-6


def resolve_abs_kinks(L64, batch, gv, g64):
    """The mixer takes |hyper_w1(s)| and |hyper_w2(s)|: an output element within round-off of zero may take the other sign in fp32, and
    then its whole loss gradient enters its hypernet with the opposite sign.  For every live element within ABS_KINK_TOL of its
    transition's largest output, the sign whose float64 gradient is closer to the engine's at that output's bias is adopted into g64
    (the element's share of the hypernet's weight and bias gradients, through the hidden ReLU of a 2-layer hypernet).  Returns
    [(module, t, b, column, |o| / max |o|)] of the flips adopted.

    This cannot hide a sign error in the kernels: such an error acts on every element of the hypernet output, not only on those within
    ABS_KINK_TOL of zero (a handful per step), so the columns and tensors it reaches keep their full float64 comparison; a flip is adopted
    only where it moves the bias gradient of its own column closer to the engine's, and everything the caller compares afterwards, that
    column included, must still meet its bound.  g64 holds the float64 gradients by parameter name ("mixer.hyper_w1.2.bias", ...) and
    is updated in place; gv the engine's."""
    share = torch.as_tensor(batch[1], dtype=torch.float64)[:-1]
    store = {}
    hooks = []
    for name in ("hyper_w1", "hyper_w2"):
        def hook(m, i, out, name=name):
            out.retain_grad()
            store[name] = out
        hooks.append(getattr(L64.mixer, name).register_forward_hook(hook))
    for p in L64.params:
        p.grad = None
    loss, _, aux = L64.loss_terms(batch)
    loss.backward()
    for h in hooks:
        h.remove()
    live = (1 - aux["bad"]).squeeze(-1) > 0
    flips = []
    for name in ("hyper_w1", "hyper_w2"):
        m = getattr(L64.mixer, name)
        two = isinstance(m, torch.nn.Sequential)
        out_lin = m[2] if two else m
        pre = "mixer.%s.%s" % (name, "2." if two else "")
        o, g_o = store[name].detach(), store[name].grad
        rel = o.abs() / o.abs().amax(-1, keepdim=True)
        for t, b, j in ((rel < ABS_KINK_TOL) & live.unsqueeze(-1)).nonzero().tolist():
            d = -2.0 * float(g_o[t, b, j])                      # the element's gradient with the other sign
            diff = float(gv[pre + "bias"][j] - g64[pre + "bias"][j])
            if abs(diff - d) >= abs(diff):
                continue
            x = share[t, b]
            g64[pre + "bias"][j] += d
            if two:
                hid_pre = m[0](x).detach()
                g64[pre + "weight"][j] += d * torch.relu(hid_pre)
                dh = d * out_lin.weight.detach()[j] * (hid_pre > 0).double()
                g64["mixer.%s.0.weight" % name] += torch.outer(dh, x)
                g64["mixer.%s.0.bias" % name] += dh
            else:
                g64[pre + "weight"][j] += d * x
            flips.append((name, t, b, j, float(rel[t, b, j])))
    return flips
