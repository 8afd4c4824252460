"""MaddpgBatchTrainGraph against the eager runner: k batch_trains of a trainer with one policy per agent, replayed through the captured
graph, equal k eager batch_trains from the same seeds bit for bit.  Shared by the emulated and the GPU test modules.

The eager batch_train is the runner's (runner/{rnn,mlp}/base_runner.py): per policy in id order sample (PER: from that policy's tree),
`train_policy_on_batch`, write that policy's priorities back; then soft-update every policy when the actor was updated.  Between
batch_trains a few episodes / transitions are inserted (the same data in both runs), so the replay's ring wraps."""
import os
import tempfile

import numpy as np
import torch

from checkpoint_maddpg_checks import Case, assert_same, snapshot
from offpolicy._b200 import capi
from offpolicy._b200.checkpoint import load_checkpoint, save_checkpoint

BETA = 0.5


class BatchCase(Case):
    """A Case whose MLP trainer takes extra args fields (`over`, e.g. use_huber_loss)."""

    def __init__(self, *a, over=None, **kw):
        super().__init__(*a, **kw)
        self.over = dict(over or {})

    def _trainer(self):
        if self.kind != "mlp" or not self.over:
            return super()._trainer()
        from offpolicy._b200 import factory as fx
        _, pols, tr, _ = fx.build_mlp_maddpg_multi([(o, a, n) for n, o, a in self.specs], self.S, self.B, discrete=self.discrete,
                                                   td3=self.td3, use_per=self.per, **self.over)
        return tr, pols


def _sync():
    if capi.device().type == "cuda":
        torch.cuda.synchronize()


def _store(buf, p):
    pb = buf.policy_buffers[p]
    return getattr(pb, "rep", pb)


PER_BETA_AT = 40       # byte offset of MxReplayState.per_beta (csrc/mx_internal.h) in the replay's state block


def _blob(rep):
    """The store's persistent blob without the PER exponent scalar: only a captured draw reads it (mx_replay_set_beta), an eager draw
    takes beta by value and leaves it alone."""
    blob = rep.state_dict()["blob"].clone()
    at = int(rep.L.off_state) + PER_BETA_AT
    blob[at:at + 8] = 0
    return blob


def eager_batch_train(case, tr, buf, pols):
    upd = False
    for p in case.ids:
        smp = buf.sample(case.B, BETA, p) if case.per else buf.sample(case.B)
        info, prio, idx = tr.train_policy_on_batch(p, smp)
        if case.per:
            buf.update_priorities(idx, prio, p)
        upd = bool(info["update_actor"])
    if upd:
        for p in case.ids:
            pols[p].soft_target_updates()
    return upd


def record(case, tr, buf, upd):
    """What a caller can read after one batch_train: per policy its train_info scalars and priorities (the engine's views), the indices
    its store holds and, with PER, its trees."""
    _sync()
    out = {"update_actor": bool(upd)}
    for p in case.ids:
        info, rep = tr._eng[p].info, _store(buf, p)
        r = [float(info[0]), float(info[1])] + ([float(info[4]), float(info[5])] if upd else [])
        r.append(np.asarray(rep.sampled_indices(case.B)).tolist())
        if case.per:
            r.append(tr._eng[p].prio[:case.B].cpu().tolist())
            r.append([t.tolist() for t in rep.tree_values()])
        out[p] = r
    return out


def state(case, tr, buf):
    """The learner and replay state the next batch_trains depend on: every vector, Adam counters and update counts (snapshot), each
    store's persistent blob (episodes, PER trees, device MT19937), the device torch generator and torch's CPU generator."""
    s = snapshot(tr, buf)
    s["stores"] = [_blob(_store(buf, p)) for p in case.ids]
    s["device_gen"] = tr.noise_gen.state.cpu().clone() if tr.noise_gen is not None else None
    s["torch_rng"] = torch.get_rng_state().clone()
    return s


def _start(case, device_noise, seed=1):
    from offpolicy._b200.torch_rng import DeviceTorchGenerator
    tr, buf, pols = case.build(seed)
    case.fill(buf, np.random.RandomState(5), case.E)
    torch.manual_seed(11)
    if device_noise:
        tr.use_device_noise(DeviceTorchGenerator(seed=3))
    return tr, buf, pols


def _rounds(case, mode, tr, buf, pols, rs, k):
    """k batch_trains, eager or through a MaddpgBatchTrainGraph, each after an insert from `rs`."""
    from offpolicy._b200.graph import MaddpgBatchTrainGraph
    g = MaddpgBatchTrainGraph(buf, tr, case.B, beta=BETA) if mode == "graph" else None
    rec = []
    for _ in range(k):
        case.put(buf, rs, case.insert)
        _sync()                                # (the graph runs on a stream of its own)
        if g is None:
            upd = eager_batch_train(case, tr, buf, pols)
        else:
            upd = g.launch()
            g.synchronize()
        rec.append(record(case, tr, buf, upd))
    if g is not None:
        g.close()
    return rec


def run(case, mode, k, device_noise):
    tr, buf, pols = _start(case, device_noise)
    rec = _rounds(case, mode, tr, buf, pols, np.random.RandomState(7), k)
    return rec, state(case, tr, buf)


def check_graph_equals_eager(case, k=5, device_noise=False):
    """k graph launches = k eager batch_trains, bit for bit; the rounds must span what the case is meant to cover."""
    rec_e, st_e = run(case, "eager", k, device_noise)
    rec_g, st_g = run(case, "graph", k, device_noise)
    assert_same(rec_g, rec_e, "rounds")
    assert_same(st_g, st_e)
    return rec_e


def check_resume_through_graph(case, k=3, device_noise=True):
    """k eager batch_trains, checkpoint, k more eager (the uninterrupted run); fresh objects under other seeds, load, the same k
    batch_trains through the graph: equal bit for bit."""
    from offpolicy._b200.torch_rng import DeviceTorchGenerator
    tr, buf, pols = _start(case, device_noise)
    rs = np.random.RandomState(7)
    _rounds(case, "eager", tr, buf, pols, rs, k)
    with tempfile.TemporaryDirectory() as d:
        path = save_checkpoint(os.path.join(d, "ck.pt"), tr, buf)
        rs_state = rs.get_state()
        want = _rounds(case, "eager", tr, buf, pols, rs, k)
        want_st = state(case, tr, buf)
        del tr, buf, pols
        tr2, buf2, pols2 = case.build(2)
        if device_noise:
            tr2.use_device_noise(DeviceTorchGenerator(seed=99))
        np.random.seed(999)
        torch.manual_seed(999)
        load_checkpoint(path, tr2, buf2)
    rs.set_state(rs_state)
    got = _rounds(case, "graph", tr2, buf2, pols2, rs, k)
    assert_same(got, want, "rounds")
    assert_same(state(case, tr2, buf2), want_st)


def eager_launches(case, device_noise, upd_wanted=True):
    """(mx_launch_count delta of one eager batch_train that updates the actors iff upd_wanted, the graph's kernel count for it)."""
    from offpolicy._b200.graph import MaddpgBatchTrainGraph
    tr, buf, pols = _start(case, device_noise)
    lib = capi.lib()
    while (tr.num_updates[case.ids[0]] % tr.actor_update_interval == 0) != upd_wanted:
        eager_batch_train(case, tr, buf, pols)
    _sync()
    n0 = int(lib.mx_launch_count())
    eager_batch_train(case, tr, buf, pols)
    _sync()
    n_eager = int(lib.mx_launch_count()) - n0
    while (tr.num_updates[case.ids[0]] % tr.actor_update_interval == 0) != upd_wanted:
        eager_batch_train(case, tr, buf, pols)
    g = MaddpgBatchTrainGraph(buf, tr, case.B, beta=BETA)
    n_graph = g.num_kernels[1 if upd_wanted else 0]
    g.close()
    return n_eager, n_graph
