"""Wide-state QMIX fixtures (tests/golden/qmix_wide_*.npz, written by tests/golden/make_goldens_qmix_wide.py).

The initial weights of a wide-state learner are most of a fixture's size (S x hypernet columns per net, four nets), so a fixture stores
seeds instead: `seeded_state_dict` fills a state_dict template deterministically from a seed, the generator loads the result into the
unmodified reference's networks before its step, and `load` rebuilds the same `init.*` entries the other QMIX fixtures carry."""
import numpy as np
import torch

from helpers import load_golden, golden_cfg

def seeded_state_dict(template, seed):
    """Same keys and shapes as `template`: 2-D weights U(-1, 1) / sqrt(fan_in), 1-D LayerNorm gains 1 + 0.2 N(0, 1),
    other 1-D tensors 0.2 N(0, 1); keys are filled in sorted order from one NumPy stream."""
    rs = np.random.RandomState(seed)
    out = {}
    for k in sorted(template):
        shape = tuple(template[k].shape)
        if len(shape) == 2:
            v = rs.uniform(-1.0, 1.0, shape) / np.sqrt(shape[1])
        elif k.endswith("weight"):
            v = 1.0 + 0.2 * rs.randn(*shape)
        else:
            v = 0.2 * rs.randn(*shape)
        out[k] = torch.from_numpy(v.astype(np.float32))
    return out


def init_state(templates, seeds):
    """templates: "agent" / "mixer" -> state_dict.  Live nets from seeds[0] / seeds[1]; the targets are the live nets plus
    0.05 N(0, 1) per element drawn from seeds[2] / seeds[3] (sorted key order), so that targets differ from the live nets."""
    out = {}
    for i, base in enumerate(("agent", "mixer")):
        live = seeded_state_dict(templates[base], int(seeds[i]))
        rs = np.random.RandomState(int(seeds[2 + i]))
        out[base] = live
        out["tgt_" + base] = {k: live[k] + torch.from_numpy((0.05 * rs.randn(*live[k].shape)).astype(np.float32)) for k in sorted(live)}
    return out


def load(name):
    """The fixture with its `init.<role>.<key>` entries rebuilt from the stored seeds (templates from the oracle's networks)."""
    from oracle.qmix import QmixLearner
    g = load_golden(name)
    cfg, B, T, steps = golden_cfg(g)
    L = QmixLearner(cfg)
    sds = init_state({"agent": L.agent.state_dict(), "mixer": L.mixer.state_dict()}, g["meta.init_seeds"])
    for role, sd in sds.items():
        for k, v in sd.items():
            g["init.%s.%s" % (role, k)] = v.numpy()
    return g
