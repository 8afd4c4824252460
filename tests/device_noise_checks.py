"""The MADDPG-family update noise drawn on the device (offpolicy/_b200/torch_rng.py, csrc/torch_rng.cu) against torch's CPU generator:
the stream, the values, the layout, the updates, the captured graph and the checkpoint.  Shared by the emulated and the GPU test
modules."""
import contextlib
import os
import tempfile

import numpy as np
import torch

from offpolicy._b200 import capi
from offpolicy._b200.torch_rng import DeviceTorchGenerator, draw
from offpolicy.algorithms.r_maddpg.algorithm.rMADDPGPolicy import sample_gumbel
from checkpoint_maddpg_checks import Case, assert_same, snapshot

# worst differences from torch's transforms, in units of float32 spacing (see value_ulps): torch's vectorised log / sin / cos and the
# device's are each within about an ulp of the exact value
GUMBEL_ULPS, NORMAL_ULPS = 4, 8


def _sync():
    if capi.device().type == "cuda":
        torch.cuda.synchronize()


def torch_layout(kind, T, rows_n, rows_b, cols, std=0.0, gen=None):
    """One fill written in torch's own layout (T, rows_n * rows_b, cols), on the host."""
    x = torch.zeros(T, rows_n * rows_b, cols, dtype=torch.float32, device=capi.device())
    gen.fill(draw(kind, T, rows_n, rows_b, cols, x, 0, rows_n * rows_b * cols, rows_b * cols, cols, std))
    _sync()
    return x.cpu()


def _prepare(where):
    """torch's CPU generator at a given position, with a cached normal sample in its state (torch.randn(1) takes the scalar path)."""
    torch.manual_seed(1234)
    torch.randn(1)
    pre = {"seeded": 0, "mid_block": 300, "pos_623": 623 - 4, "pos_624": 624 - 4, "odd_draws": None}[where]
    if where == "seeded":
        torch.manual_seed(1234)
        return DeviceTorchGenerator(seed=1234)
    if pre is None:
        for n in (17, 1001, 3):
            torch.empty(n).uniform_()
    else:
        torch.empty(pre).uniform_()
    return DeviceTorchGenerator()


def check_uniform_stream(where, shapes):
    """Uniform fills bit-identical to torch's uniform_, and after every call the exported state byte-identical to torch's own."""
    gen = _prepare(where)
    for shape in shapes:
        want = torch.empty(shape[0], shape[1] * shape[2], shape[3]).uniform_()
        want_state = torch.get_rng_state().clone()
        got = torch_layout(capi.TRNG_UNIFORM, *shape, gen=gen)
        assert torch.equal(got, want), (where, shape)
        gen.export_rng_to_torch()
        assert torch.equal(torch.get_rng_state(), want_state), (where, shape)


def value_ulps(got, want, floor=None):
    """|got - want| in units of the float32 spacing at |want| (at max(|want|, floor) when a floor is given)."""
    w = np.abs(want.numpy().astype(np.float64))
    if floor is not None:
        w = np.maximum(w, floor)
    return float((np.abs(got.numpy().astype(np.float64) - want.numpy()) / np.spacing(w.astype(np.float32))).max())


def check_transform(kind, n, std=0.2):
    """Gumbel / normal fills of n values against sample_gumbel / normal_: the same positions, within the stated ulps; returns the worst
    ulps.  Values are compared in units of the spacing at max(|value|, 1) (Gumbel) or max(|value|, std) (normal): near a Gumbel value
    of 0 the last log's argument is near 1, and near a zero of cos / sin the normal value is small, so their own spacing says nothing
    about the accuracy of the draw."""
    torch.manual_seed(77)
    gen = DeviceTorchGenerator(seed=77)
    if kind == capi.TRNG_GUMBEL:
        want = sample_gumbel((1, n, 1))
        got = torch_layout(kind, 1, 1, n, 1, gen=gen)
        ulps, bound = value_ulps(got, want, floor=1.0), GUMBEL_ULPS
    else:
        want = torch.empty(1, n, 1).normal_(mean=0, std=std)
        got = torch_layout(kind, 1, 1, n, 1, std=std, gen=gen)
        ulps, bound = value_ulps(got, want, floor=std), NORMAL_ULPS
    want_state = torch.get_rng_state().clone()
    gen.export_rng_to_torch()
    assert torch.equal(torch.get_rng_state(), want_state), n
    assert ulps <= bound, (kind, n, ulps)
    return ulps


def check_gumbel_at_zero():
    """A word whose tempered value has 24 zero low bits gives u = 0: the transform's extreme (-log(-log(1e-20) + 1e-20))."""
    gen = DeviceTorchGenerator(seed=5)
    key, _, _ = gen.get_state()
    key = key.copy()
    key[10] = 0                                         # tempering maps 0 to 0
    gen.set_state(key, 625 - 10, 10)
    gen.export_rng_to_torch()
    want = sample_gumbel((1, 1, 1))
    gen.set_state(key, 625 - 10, 10)
    got = torch_layout(capi.TRNG_GUMBEL, 1, 1, 1, 1, gen=gen)
    ulps = value_ulps(got, want, floor=1.0)
    assert abs(float(want) - (-np.log(-np.log(1e-20)))) < 1e-5 and ulps <= GUMBEL_ULPS, (float(got), float(want))
    return ulps


def check_refusals():
    lib = capi.lib()
    gen = DeviceTorchGenerator(seed=1)
    x = torch.zeros(64, device=capi.device())
    for bad, msg in ((draw(capi.TRNG_NORMAL, 1, 3, 5, 1, x, 0, 0, 5, 1), b"< 16"), (draw(7, 1, 1, 4, 1, x, 0, 0, 4, 1), b"unknown kind"),
                     (draw(capi.TRNG_UNIFORM, 1, 0, 4, 1, x, 0, 0, 4, 1), b"empty")):
        try:
            gen.fill(bad)
        except capi.MxError as e:
            assert msg.decode() in str(e), str(e)
        else:
            raise AssertionError("a bad fill was accepted")
        assert msg in lib.mx_last_error()
    key, left, nxt = gen.get_state()
    assert lib.mx_trng_set_state(capi.ptr(gen.state), key.ctypes.data_as(capi.C.POINTER(capi.C.c_uint32)), 0, 0, None) != 0
    assert b"outside" in lib.mx_last_error()
    assert gen.get_state()[1:] == (left, nxt)


# ---- trainers ---------------------------------------------------------------------------------------------------------------
def _draw_plan(tr):
    """(p_id, which) of every noise draw one update of policy_0 makes, in the reference's order."""
    plan = []
    for q in (tr.policy_ids if tr.multi else ["policy_0"]):
        if tr._eng[q].pol.td3:
            plan.append((q, "target"))
    if tr._eng["policy_0"].pol.discrete:
        plan.append(("policy_0", "actor"))
    return plan


def check_layout(case, B=None):
    """Every device-mode draw lands where the host-mode draw lands after its permutation into the learner's layout."""
    B = B or case.B
    tr, _, _ = case.build(1)
    torch.manual_seed(31)
    host = {}
    for q, which in _draw_plan(tr):
        host[(q, which)] = tr._noise(B, q, which).cpu().clone()
    want_state = torch.get_rng_state().clone()
    torch.manual_seed(31)
    gen = DeviceTorchGenerator()
    tr.use_device_noise(gen)
    for q, which in _draw_plan(tr):
        got = tr._noise(B, q, which)
        _sync()
        got, want = got.cpu(), host[(q, which)]
        assert got.shape == want.shape, (q, which)
        assert torch.equal(got == 0, want == 0), (q, which)            # the same padding
        assert torch.allclose(got, want, rtol=1e-5, atol=1e-6), (q, which, float((got - want).abs().max()))
    gen.export_rng_to_torch()
    assert torch.equal(torch.get_rng_state(), want_state)


def _feed_device_values(tr, gen2):
    """Host-mode trainer whose draw_target_noise / draw_actor_noise return what gen2 (a twin of the device-mode generator) draws, in
    torch's layout: the host path then permutes and copies them in."""

    def values(B, p_id, which):
        ds = tr._noise_draws(B, p_id, which)
        parts = [torch_layout(d.kind, d.T, d.rows_n, d.rows_b, d.cols, d.std, gen=gen2) for d in ds]
        return torch.cat(parts, -1)

    orig_t, orig_a = tr.draw_target_noise, tr.draw_actor_noise

    def target(B, p_id=None):
        p = p_id or tr.policy_ids[0]
        return values(B, p, "target") if tr._eng[p].pol.td3 else orig_t(B, p_id)

    def actor(B, p_id=None):
        p = p_id or tr.policy_ids[0]
        return values(B, p, "actor") if tr._eng[p].pol.discrete else orig_a(B, p_id)

    tr.draw_target_noise, tr.draw_actor_noise = target, actor


def check_updates(case, k=3):
    """k device-mode rounds = k host-mode rounds fed the noise the device drew (train_info, sampled indices, priorities, every vector),
    bit for bit; the device rounds leave torch's host generator alone, and exporting afterwards gives torch the state k host-mode
    rounds leave."""
    assert case.rng == "device"
    rs_seed = 5
    runs = {}
    for mode in ("device", "fed", "host"):
        tr, buf, pols = case.build(1)
        rs = np.random.RandomState(rs_seed)
        case.fill(buf, rs, case.E)
        torch.manual_seed(11)
        start = torch.get_rng_state().clone()
        if mode == "device":
            gen = DeviceTorchGenerator()
            tr.use_device_noise(gen)
        elif mode == "fed":
            _feed_device_values(tr, DeviceTorchGenerator())
        rounds = [case.round(tr, buf, pols, rs, insert=False) for _ in range(k)]
        if mode == "device":
            assert torch.equal(torch.get_rng_state(), start), "device-mode updates touched torch's host generator"
            gen.export_rng_to_torch()
        runs[mode] = (rounds, snapshot(tr, buf), torch.get_rng_state().clone())
    assert_same(runs["device"][0], runs["fed"][0], "rounds")
    assert_same(runs["device"][1], runs["fed"][1], "state")
    assert torch.equal(runs["device"][2], runs["host"][2]), "stream position after k updates"


@contextlib.contextmanager
def _side_stream():
    if capi.device().type != "cuda":
        yield
        return
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        yield
    torch.cuda.current_stream().wait_stream(side)


def check_graph(case, n=4):
    """n launches of the device-mode MaddpgStepGraph = n eager device-mode updates, bit for bit, and torch's host generator does not
    move across the launches."""
    from offpolicy._b200.graph import MaddpgStepGraph
    assert case.rng == "device" and not case.per and len(case.specs) == 1
    out = {}
    for mode in ("eager", "graph"):
        tr, buf, pols = case.build(1)
        case.fill(buf, np.random.RandomState(5), case.E)
        torch.manual_seed(11)
        gen = DeviceTorchGenerator()
        tr.use_device_noise(gen)
        start = torch.get_rng_state().clone()
        rec = []
        with _side_stream():
            if mode == "eager":
                for _ in range(n):
                    r = case.round(tr, buf, pols, None, insert=False)
                    rec.append((r[0], dict(r[1])["critic_loss"], dict(r[1])["update_actor"]))
            else:
                g = MaddpgStepGraph(buf, tr, case.B)
                for _ in range(n):
                    upd = g.launch()
                    g.synchronize()
                    info = tr._eng["policy_0"].info
                    rec.append((np.asarray(case.first_store(buf).sampled_indices(case.B)).tolist(), float(info[0]), bool(upd)))
                g.close()
        _sync()
        assert torch.equal(torch.get_rng_state(), start), mode
        out[mode] = (rec, snapshot(tr, buf), gen.state_dict())
    assert_same(out["graph"][0], out["eager"][0], "rounds")
    assert_same(out["graph"][1], out["eager"][1], "state")
    assert_same({k: np.asarray(v).tolist() for k, v in out["graph"][2].items()}, {k: np.asarray(v).tolist() for k, v in out["eager"][2].items()})


def check_checkpoint(case, k=2):
    """Device mode: k rounds, save, k more; fresh objects under other seeds, load, the same k rounds: bit-identical, the generator
    included.  A host-mode checkpoint still loads into a host-mode trainer, and not into a device-mode one."""
    from offpolicy._b200.checkpoint import save_checkpoint, load_checkpoint

    def start(seed):
        tr, buf, pols = case.build(seed)
        gen = DeviceTorchGenerator(seed=seed + 100)
        tr.use_device_noise(gen)
        return tr, buf, pols, gen

    tr, buf, pols, gen = start(1)
    rs = np.random.RandomState(5)
    case.fill(buf, rs, case.E - k * case.insert)
    for _ in range(k):
        case.round(tr, buf, pols, rs)
    with tempfile.TemporaryDirectory() as d:
        path = save_checkpoint(os.path.join(d, "ck.pt"), tr, buf)
        rs_state = rs.get_state()
        want = [case.round(tr, buf, pols, rs) for _ in range(k)]
        want_snap, want_gen = snapshot(tr, buf), gen.state_dict()
        tr2, buf2, pols2, gen2 = start(2)
        load_checkpoint(path, tr2, buf2)
        rs.set_state(rs_state)
        got = [case.round(tr2, buf2, pols2, rs) for _ in range(k)]
        assert_same(got, want, "rounds")
        assert_same(snapshot(tr2, buf2), want_snap)
        g = gen2.state_dict()
        assert np.array_equal(g["key"], want_gen["key"]) and (g["left"], g["next"]) == (want_gen["left"], want_gen["next"])
        # host-mode checkpoints: the earlier format, loads into a host-mode trainer; a device-mode trainer refuses it
        tr3, buf3, _ = case.build(3)
        host_path = save_checkpoint(os.path.join(d, "host.pt"), tr3, buf3)
        assert "device_noise" not in torch.load(host_path, weights_only=False)["trainer"]
        tr4, buf4, _ = case.build(4)
        load_checkpoint(host_path, tr4, buf4)
        assert_same(snapshot(tr4, buf4), snapshot(tr3, buf3))
        try:
            load_checkpoint(host_path, tr2, None, restore_host_rng=False)
        except ValueError as e:
            assert "noise mode" in str(e)
        else:
            raise AssertionError("a host-mode checkpoint loaded into a device-mode trainer")
