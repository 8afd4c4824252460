"""Flat parameter vectors with named tensor views.

The CUDA learner owns ONE fp32 vector per role (live, target, Adam m, Adam v) laid out by
`mx_qmix_param_layout` (names = the reference's state_dict keys, SURVEY.md App. E).  The objects
below give the runner the module-like surface it touches: `state_dict()`, `load_state_dict()`,
`parameters()`, `train()/eval()` (offpolicy/runner/rnn/base_runner.py:286-337, qmix.py:218-232).
"""
from collections import OrderedDict

import torch


class FlatModule(object):
    def __init__(self, flat, entries, prefix):
        """flat: 1-D tensor; entries: [(name, offset, rows, cols)] with `prefix` ('agent.'/'mixer.') already in name."""
        self.prefix = prefix
        self.entries = [(n[len(prefix):], o, r, c) for (n, o, r, c) in entries if n.startswith(prefix)]
        self.bind(flat)

    def bind(self, flat):
        self.flat = flat
        self.views = OrderedDict()
        for name, off, rows, cols in self.entries:
            n = rows * (cols if cols else 1)
            v = flat[off:off + n]
            self.views[name] = v.view(rows, cols) if cols else v

    # -- nn.Module look-alike ----------------------------------------------------------------
    def state_dict(self):
        return OrderedDict((k, v.detach().clone()) for k, v in self.views.items())

    def load_state_dict(self, sd, strict=True):
        missing = [k for k in self.views if k not in sd]
        extra = [k for k in sd if k not in self.views]
        if strict and (missing or extra):
            raise KeyError("load_state_dict: missing %s unexpected %s" % (missing, extra))
        with torch.no_grad():
            for k, v in self.views.items():
                if k in sd:
                    v.copy_(torch.as_tensor(sd[k]).to(v.device, v.dtype).reshape(v.shape))

    def parameters(self):
        return list(self.views.values())

    def named_parameters(self):
        return list(self.views.items())

    def train(self, mode=True):
        return self

    def eval(self):
        return self

    def to(self, *a, **k):
        return self


def reference_style_init(entries, cfg, gain, use_orthogonal=True, hyper_layers=2, seed_modules=True, use_relu=True):
    """Initial weights in the construction ORDER of the reference so that, under the same torch.manual_seed, the
    CPU RNG is consumed the same way (mlp.py:14-23, rnn.py:8-17, act.py:10-20, q_mixer.py:33-66):
    nn.Linear/nn.GRU default init first, then orthogonal_/xavier_uniform_ x gain, biases 0, LayerNorm (1, 0).
    Returns {name: cpu tensor}."""
    import torch.nn as nn
    H, I, A = cfg["hidden"], cfg["obs_dim"], cfg["act_dim"]
    init_w = nn.init.orthogonal_ if use_orthogonal else nn.init.xavier_uniform_
    relu_gain = nn.init.calculate_gain("relu" if use_relu else "tanh")      # mlp.py:12: gain of the activation in use
    out = {}

    def linear(prefix, i, o, g):
        m = nn.Linear(i, o)
        init_w(m.weight.data, gain=g)
        m.bias.data.zero_()
        out[prefix + ".weight"], out[prefix + ".bias"] = m.weight.data, m.bias.data

    def lnorm(prefix, n):
        out[prefix + ".weight"], out[prefix + ".bias"] = torch.ones(n), torch.zeros(n)

    if any(n.startswith("agent.") for n, *_ in entries):
        if any(n == "agent.rnn.feature_norm.weight" for n, *_ in entries):      # absent with --use_feature_normalization off
            lnorm("agent.rnn.feature_norm", I)
        linear("agent.rnn.mlp.fc1.0", I, H, relu_gain)
        lnorm("agent.rnn.mlp.fc1.2", H)
        linear("agent.rnn.mlp.fc_h.0", H, H, relu_gain)
        lnorm("agent.rnn.mlp.fc_h.2", H)
        for k in ("0.weight", "0.bias", "2.weight", "2.bias"):          # fc2 = deepcopy(fc_h)  (mlp.py:23)
            out["agent.rnn.mlp.fc2.0." + k] = out["agent.rnn.mlp.fc_h." + k].clone()
        gru = nn.GRU(H, H, num_layers=1)
        for name, p in gru.named_parameters():
            if "bias" in name:
                p.data.zero_()
            else:
                init_w(p.data)
            out["agent.rnn.rnn.rnn." + name] = p.data
        lnorm("agent.rnn.rnn.norm", H)
        linear("agent.q.action_out", H, A, gain)
    if any(n.startswith("mixer.") for n, *_ in entries):
        S, N, ME, HY = cfg["state_dim"], cfg["n_agents"], cfg["mixer_hidden"], cfg["hyper_hidden"]
        if hyper_layers == 1:
            linear("mixer.hyper_w1", S, N * ME, 1.0)
            linear("mixer.hyper_w2", S, ME, 1.0)
        else:
            linear("mixer.hyper_w1.0", S, HY, 1.0)
            linear("mixer.hyper_w1.2", HY, N * ME, 1.0)
            linear("mixer.hyper_w2.0", S, HY, 1.0)
            linear("mixer.hyper_w2.2", HY, ME, 1.0)
        linear("mixer.hyper_b1", S, ME, 1.0)
        linear("mixer.hyper_b2.0", S, HY, 1.0)
        linear("mixer.hyper_b2.2", HY, 1, 1.0)
    return out


def mlp_init(in_dim, hidden, heads, use_orthogonal, use_relu=True, feature_norm=True):
    """MLPBase (mlp.py:52-89: feature LayerNorm, fc1, fc_h, fc2 = deepcopy of fc_h) then the heads [(prefix, out_dim, gain)], in the
    reference's construction order: nn.Linear's own init, then orthogonal_ / xavier_uniform_ x gain, biases 0.  Returns {name: tensor}."""
    import torch.nn as nn
    init_w = nn.init.orthogonal_ if use_orthogonal else nn.init.xavier_uniform_
    relu_gain = nn.init.calculate_gain("relu" if use_relu else "tanh")
    sd = {}

    def linear(prefix, i, o, g):
        m = nn.Linear(i, o)
        init_w(m.weight.data, gain=g)
        m.bias.data.zero_()
        sd[prefix + ".weight"], sd[prefix + ".bias"] = m.weight.data, m.bias.data

    def lnorm(prefix, n):
        sd[prefix + ".weight"], sd[prefix + ".bias"] = torch.ones(n), torch.zeros(n)

    if feature_norm:
        lnorm("mlp.feature_norm", in_dim)
    linear("mlp.mlp.fc1.0", in_dim, hidden, relu_gain)
    lnorm("mlp.mlp.fc1.2", hidden)
    linear("mlp.mlp.fc_h.0", hidden, hidden, relu_gain)
    lnorm("mlp.mlp.fc_h.2", hidden)
    for k in ("0.weight", "0.bias", "2.weight", "2.bias"):
        sd["mlp.mlp.fc2.0." + k] = sd["mlp.mlp.fc_h." + k].clone()
    for prefix, o, g in heads:
        linear(prefix, hidden, o, g)
    return sd
