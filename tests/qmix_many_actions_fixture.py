"""Recurrent QMIX fixtures with more than 32 actions (tests/golden/qmix_a*.npz, written by
tests/golden/make_goldens_qmix_many_actions.py).

Like the wide-state fixtures (tests/qmix_wide_fixture.py) they store seeds instead of the initial weights, which would be most of a
fixture's size.  A fixture whose live head has tied rows also stores that head as `init_head.weight` / `init_head.bias`; `load`
puts it over the seeded one."""
import qmix_wide_fixture as wf


def load(name):
    """The fixture with its `init.<role>.<key>` entries rebuilt from the stored seeds and the stored live head, if any."""
    g = wf.load(name)
    for k in ("weight", "bias"):
        if "init_head." + k in g:
            g["init.agent.q.action_out." + k] = g["init_head." + k]
    return g
