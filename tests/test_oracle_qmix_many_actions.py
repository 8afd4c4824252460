"""Pin the oracles (oracle/qmix.py, oracle/mqmix.py) against the unmodified reference at more than 32 actions
(tests/golden/make_goldens_qmix_many_actions.py; initial weights rebuilt by tests/qmix_many_actions_fixture.py): SMAC's 27m_vs_30m
has 36.  Same torch ops as the reference, so agreement is
expected at float32 round-off, as for the other fixtures."""
import pytest
import torch

from helpers import load_golden, oracle_from_golden, golden_batch, rel_err
import qmix_many_actions_fixture as mf
import test_oracle_mqmix as om

QMIX = ["qmix_a36_ties", "qmix_a64_hyper1", "qmix_a33_prev_act"]


@pytest.mark.parametrize("name", QMIX)
def test_oracle_reproduces_many_action_reference_step(name):
    torch.set_num_threads(1)
    g = mf.load(name)
    L, cfg, B, T, steps = oracle_from_golden(g)
    assert cfg.act_dim > 32
    for s in range(steps):
        info, prio, _ = L.step(golden_batch(g, s))
        assert rel_err(info["loss"], g["s%d.loss" % s]) < 1e-6
        assert rel_err(info["grad_norm"], g["s%d.grad_norm" % s]) < 1e-5
        assert rel_err(info["Q_tot"], g["s%d.Q_tot" % s]) < 1e-5
        for role, mod in (("agent", L.agent), ("mixer", L.mixer)):
            for k, p in mod.named_parameters():
                key = "s%d.grad.%s.%s" % (s, role, k)
                if key in g:
                    assert rel_err(p.grad, g[key]) < 2e-5, key
                else:
                    assert p.grad is None and "fc_h" in k
        L.soft_update()
        for tag, mod in (("agent", L.agent), ("mixer", L.mixer), ("tgt_agent", L.tgt_agent), ("tgt_mixer", L.tgt_mixer)):
            for k, v in mod.state_dict().items():
                assert rel_err(v, g["s%d.%s.%s" % (s, tag, k)]) < 2e-6, (tag, k)


def test_tied_fixture_has_ties():
    """The tied head rows of qmix_a36_ties are equal in the fixture's live net and distinct in its target net, so the lower-index
    rule decides the double-Q target."""
    g = mf.load("qmix_a36_ties")
    w, tw = g["init.agent.q.action_out.weight"], g["init.tgt_agent.q.action_out.weight"]
    for lo, hi in ((3, 35), (32, 33)):
        assert (w[lo] == w[hi]).all() and not (tw[lo] == tw[hi]).all()


def test_oracle_reproduces_many_action_mlp_reference_step():
    torch.set_num_threads(1)
    g = load_golden("mqmix_a36")
    L, cfg, B, steps = om.oracle_from_golden(g)
    assert cfg.act_dim == 36
    for s in range(steps):
        info, prio, _ = L.step(om.golden_transitions(g, s))
        assert rel_err(info["loss"], g["s%d.loss" % s]) < 1e-6
        assert rel_err(info["grad_norm"], g["s%d.grad_norm" % s]) < 1e-5
        assert rel_err(info["Q_tot"], g["s%d.Q_tot" % s]) < 1e-5
        for role, mod in (("agent", L.agent), ("mixer", L.mixer)):
            for k, p in mod.named_parameters():
                key = "s%d.grad.%s.%s" % (s, role, k)
                if key in g:
                    assert rel_err(p.grad, g[key]) < 2e-5, key
        L.soft_update()
        for tag, mod in (("agent", L.agent), ("mixer", L.mixer), ("tgt_agent", L.tgt_agent), ("tgt_mixer", L.tgt_mixer)):
            for k, v in mod.state_dict().items():
                assert rel_err(v, g["s%d.%s.%s" % (s, tag, k)]) < 2e-6, (tag, k)
