"""Data-parallel R-MADDPG / R-MATD3 and MADDPG / MATD3 on the CPU emulator: two ranks in one process whose symmetric blocks are host
tensors.  Each rank trains on half of a golden batch; both gradient exchanges of every update (the critic's, then the actor's) go
through the peer-memory kernels, and the result must be the reference's single-batch update on both ranks, bit-identical between them."""
import ctypes as C
import os
import subprocess
import sys

import pytest
import torch

import maddpg_dp_checks as dc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))

# R-MADDPG Box; R-MATD3 Discrete with masks (actor every 2nd update, three updates); R-MADDPG with PER; MLP MADDPG Discrete; MLP MATD3
# MultiDiscrete; MLP MADDPG with two policies
GOLDENS = ["maddpg_box", "matd3_disc_avail", "maddpg_box_per", "mlp_maddpg_disc", "mlp_matd3_md", "mlp_maddpg_multi_disc"]


@pytest.mark.parametrize("name", GOLDENS)
def test_two_rank_exchange_equals_single_batch_reference(emu_engine, name):
    dc.golden_dp(name)


@pytest.mark.parametrize("order", ["reverse", "random"])
def test_two_rank_exchange_thread_orders(order):
    """The same runs with the emulator's threads in reverse / pseudo-random order (a missing barrier or fence shows up as a wrong sum)."""
    env = dict(os.environ, EMU_ORDER=order)
    code = ("import sys; sys.path[:0] = [%r, %r, %r]\n"
            "import pytest\n"
            "sys.exit(pytest.main(['-q', '-x', '-p', 'no:cacheprovider', %r, '-k', "
            "'test_two_rank_exchange_equals_single_batch_reference and (matd3_disc_avail or mlp_maddpg_multi_disc)']))\n"
            % (ROOT, os.path.join(ROOT, "off-policy_b200"), HERE, os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]


def _rnn_ranks(world=2, B=4, T=6, td3=False):
    from maddpg_checks import build
    from oracle.maddpg import MaddpgConfig
    cfg = MaddpgConfig(act_dim=2, discrete=False, td3=td3, actor_update_interval=2 if td3 else 1, gain=1.0)
    out = []
    for r in range(world):
        torch.manual_seed(1)
        out.append(build(cfg, B, T, dp_world_size=world))
    return cfg, out


def test_set_peers_argument_errors(emu_engine):
    capi = emu_engine
    lib = capi.lib()
    _, [(args, pol, tr)] = _rnn_ranks(world=1)
    h = tr.handle
    n = tr.p2p_block_bytes("policy_0", capi.MADDPG_CRITIC)
    assert n > 0 and lib.mx_maddpg_p2p_block_bytes(h, 2) < 0
    blk = [torch.zeros(n // 4) for _ in range(4)]
    ptrs = lambda *bs: (C.c_void_p * len(bs))(*[b.data_ptr() for b in bs])
    c0, c1 = torch.zeros(4, dtype=torch.int32), torch.zeros(4, dtype=torch.int32)
    assert lib.mx_maddpg_p2p_publish(h, capi.MADDPG_CRITIC, None) != 0           # no peers yet
    assert lib.mx_maddpg_p2p_reduce(h, capi.MADDPG_ACTOR, None) != 0
    assert lib.mx_maddpg_set_peers(h, capi.MADDPG_CRITIC, 0, 1, ptrs(blk[0]), capi.ptr(c0)) != 0       # world 1
    assert lib.mx_maddpg_set_peers(h, capi.MADDPG_CRITIC, 2, 2, ptrs(blk[0], blk[1]), capi.ptr(c0)) != 0   # rank outside the world
    assert lib.mx_maddpg_set_peers(h, capi.MADDPG_CRITIC, 0, 17, ptrs(*(blk * 5)[:17]), capi.ptr(c0)) != 0  # more than 16 ranks
    assert lib.mx_maddpg_set_peers(h, 2, 0, 2, ptrs(blk[0], blk[1]), capi.ptr(c0)) != 0                 # no such network
    assert lib.mx_maddpg_set_peers(h, capi.MADDPG_CRITIC, 0, 2, (C.c_void_p * 2)(blk[0].data_ptr(), None), capi.ptr(c0)) != 0
    assert lib.mx_maddpg_set_peers(h, capi.MADDPG_CRITIC, 0, 2, ptrs(blk[0], blk[1]), None) != 0       # no counter
    assert lib.mx_maddpg_set_peers(h, capi.MADDPG_CRITIC, 0, 2, ptrs(blk[0], blk[0]), capi.ptr(c0)) != 0   # one block for two ranks
    assert lib.mx_maddpg_set_peers(h, capi.MADDPG_CRITIC, 0, 2, ptrs(blk[0], blk[1]), capi.ptr(c0)) == 0
    assert lib.mx_maddpg_set_peers(h, capi.MADDPG_ACTOR, 0, 2, ptrs(blk[0], blk[3]), capi.ptr(c1)) != 0    # the critic's block
    assert lib.mx_maddpg_set_peers(h, capi.MADDPG_ACTOR, 0, 2, ptrs(blk[2], blk[3]), capi.ptr(c0)) != 0    # the critic's counter
    assert lib.mx_maddpg_set_peers(h, capi.MADDPG_ACTOR, 1, 2, ptrs(blk[2], blk[3]), capi.ptr(c1)) != 0    # another rank than the critic's
    assert lib.mx_maddpg_set_peers(h, capi.MADDPG_ACTOR, 0, 2, ptrs(blk[2], blk[3]), capi.ptr(c1)) == 0
    # the phases of an update run in order
    upd = C.c_int32()
    assert lib.mx_maddpg_step_phase(h, capi.MADDPG_CRITIC_APPLY, None, None, None, C.byref(upd), None) != 0
    assert b"out of order" in lib.mx_last_error()
    assert lib.mx_maddpg_step_phase(h, 4, None, None, None, C.byref(upd), None) != 0


def test_graphs_refuse_a_data_parallel_trainer(emu_engine):
    from offpolicy._b200.graph import MaddpgStepGraph, MaddpgBatchTrainGraph
    _, [(args, pol, tr), _] = _rnn_ranks()
    with pytest.raises(ValueError, match="data-parallel"):
        MaddpgStepGraph(None, tr, 4)
    with pytest.raises(ValueError, match="data-parallel"):
        MaddpgBatchTrainGraph(None, tr, 4)


def test_preset_abort_word_applies_nothing_and_raises(emu_engine):
    """A rank whose abort word is already set (a peer timed out on an earlier exchange) applies no update at all, and the host raises."""
    from maddpg_checks import ref_tuple
    from oracle.maddpg import synth_batch_cont
    cfg, ranks = _rnn_ranks(td3=True)
    trs = [tr for _, _, tr in ranks]
    blocks = dc.host_blocks(trs)
    pol, tr = ranks[0][1], trs[0]
    for (p, net), bl in blocks.items():          # the peer's flags are up: only the abort word stands between the sums and Adam
        dc.flag_words(tr, p, net, bl[0], 2)[1] = 1 << 20
    tr._eng["policy_0"].abort.fill_(-1.0)
    before = [v.clone() for v in dc.vecs({"policy_0": pol})]
    batch = tuple(synth_batch_cont(cfg, 4, 6, seed=3)) + (None, None)
    torch.manual_seed(5)
    with pytest.raises(RuntimeError, match="did not deliver"):
        tr.train_policy_on_batch("policy_0", ref_tuple(batch))
    for a, b in zip(before, dc.vecs({"policy_0": pol})):
        assert torch.equal(a, b)
    assert float(tr._eng["policy_0"].abort[0]) == -1.0                   # sticky
