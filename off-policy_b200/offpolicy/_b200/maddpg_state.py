"""Checkpoint / resume of the MADDPG-family trainers (SURVEY.md 8(f).3): R_MADDPG / R_MATD3 and MADDPG / MATD3 share it.

Per policy the learner is its eight flat vectors (actor and critic: live, target, Adam m, Adam v; the MLP critic's frozen live and
target heads sit in the critic vectors past the trunk), the two Adam step counters in its workspace (fp64 words) and the update count,
kept twice: the host `num_updates[p_id]` the trainer and the graph helpers read, and the handle's own count that picks the actor
phase of an eager step.  A trainer in device noise mode (`use_device_noise`) also saves its generator's key and position
("device_noise"); a host-mode checkpoint has no such entry and keeps the earlier format.  Loading writes every value in place, so the
mx_maddpg handles, the `mx_maddpg_set_valid` pointers, the generator's device state and any captured whole-update graph stay valid."""
import ctypes as C

import torch

from offpolicy._b200 import capi

KIND = "maddpg"
ADAM_COUNTERS = ("adam_ta", "adam_tc")


def _entries(es):
    return [(str(n), int(o), int(r), int(c)) for n, o, r, c in es]



class MaddpgLearnerState(object):
    """Mixin of the trainers: needs `_eng` ({p_id: engine with .handle, .workspace, .cfg, .pol}), `policy_ids`, `policy_agents`,
    `num_updates` and `actor_update_interval`."""

    def ws_view(self, name, p_id=None, dtype=torch.float32):
        """A named region of one policy's learner workspace (mx_maddpg_ws_lookup), e.g. ws_view("adam_ta", dtype=torch.float64)."""
        e = self._eng[p_id or self.policy_ids[0]]
        off, n = C.c_int64(), C.c_int64()
        capi.check(capi.lib().mx_maddpg_ws_lookup(e.handle, name.encode(), C.byref(off), C.byref(n)))
        return e.workspace[off.value:off.value + 4 * n.value].view(dtype)

    def _config_key(self):
        """Everything a checkpoint must agree with before any value is written."""
        pols = {}
        for p in self.policy_ids:
            e = self._eng[p]
            pol = e.pol
            critic = _entries(pol._c_entries) + _entries(getattr(pol, "_h_entries", []))
            pols[p] = {"agents": list(self.policy_agents[p]), "discrete": bool(pol.discrete), "td3": bool(pol.td3),
                       "actor_layout": _entries(pol._a_entries), "critic_layout": critic, "Pa": int(pol.Pa), "Pc": int(pol.Pc)}
        first = self._eng[self.policy_ids[0]]
        return {"kind": KIND, "recurrent": not bool(first.cfg.mlp), "td3": bool(first.pol.td3),
                "actor_update_interval": int(self.actor_update_interval), "policies": pols}

    def state_dict(self):
        """The whole learner of every policy (`policies[p].actor / critic / target_*.state_dict()` stay the reference's per-network
        checkpoints with its key names)."""
        if self.dev.type == "cuda":
            torch.cuda.synchronize(self.dev)      # a captured graph may have run on a stream of its own
        lib = capi.lib()
        state = {}
        for p in self.policy_ids:
            e = self._eng[p]
            state[p] = {"actor_vecs": [v.cpu().clone() for v in e.pol.actor_vecs], "critic_vecs": [v.cpu().clone() for v in e.pol.critic_vecs],
                        "num_updates": int(self.num_updates[p]), "engine_updates": int(lib.mx_maddpg_num_updates(e.handle))}
            for name in ADAM_COUNTERS:
                state[p][name] = self.ws_view(name, p, torch.float64).cpu().clone()
        sd = {"config": self._config_key(), "state": state}
        if getattr(self, "noise_gen", None) is not None:
            sd["device_noise"] = self.noise_gen.state_dict()
        return sd

    def load_state_dict(self, sd):
        want = self._config_key()
        got = sd.get("config") if isinstance(sd, dict) else None
        if not isinstance(got, dict) or got.get("kind") != KIND:
            raise ValueError("learner checkpoint was not written by an R-MADDPG / R-MATD3 / MADDPG / MATD3 trainer")
        for key in ("recurrent", "td3", "actor_update_interval"):
            if got.get(key) != want[key]:
                raise ValueError("learner checkpoint has %s = %r, this trainer %r" % (key, got.get(key), want[key]))
        if sorted(got["policies"]) != sorted(want["policies"]):
            raise ValueError("learner checkpoint holds policies %s, this trainer %s" % (sorted(got["policies"]), sorted(want["policies"])))
        for p, w in want["policies"].items():
            g = got["policies"][p]
            for key in w:
                if g.get(key) != w[key]:
                    raise ValueError("learner checkpoint of policy %s was written for a different %s" % (p, key))
        gen = getattr(self, "noise_gen", None)
        if (gen is not None) != ("device_noise" in sd):
            raise ValueError("learner checkpoint was written in %s noise mode, this trainer draws its noise on the %s"
                             % ("device" if "device_noise" in sd else "host", "device" if gen is not None else "host"))
        lib = capi.lib()
        for p in self.policy_ids:
            e, st = self._eng[p], sd["state"][p]
            for dst, src in zip(e.pol.actor_vecs + e.pol.critic_vecs, st["actor_vecs"] + st["critic_vecs"]):
                dst.copy_(torch.as_tensor(src).to(dst.device))
            for name in ADAM_COUNTERS:
                self.ws_view(name, p, torch.float64).copy_(torch.as_tensor(st[name]).to(self.dev))
            capi.check(lib.mx_maddpg_set_num_updates(e.handle, int(st["engine_updates"])))
            self.num_updates[p] = int(st["num_updates"])
        if gen is not None:
            gen.load_state_dict(sd["device_noise"])
        if self.dev.type == "cuda":
            torch.cuda.synchronize(self.dev)      # the next step may be a graph replay on another stream
