"""torch's CPU generator continued on the device (csrc/torch_rng.cu), for the actor-critic learners' update noise.

The reference draws the noise of every MADDPG / MATD3 / R-MADDPG / R-MATD3 update from torch's CPU generator: the Gumbel draws of
the actor update and of MATD3's target actions (`sample_gumbel`, utils/util.py:127-130) and MATD3's N(0, std) target-action noise
(util.py:217-218).  `DeviceTorchGenerator` holds a copy of that generator in device memory; a trainer switched to it with
`trainer.use_device_noise(gen)` (offpolicy/_b200/maddpg_trainer.py) makes each of those torch calls as one fill on the device, written
straight into the learner's noise layout, so an update (or a captured whole-update graph) needs no host draw and no copy.

The fills consume exactly the words torch's calls would, and their uniforms are bit-identical to torch's.  The Gumbel and normal
transforms agree with torch's to a few ulps, not bit for bit (torch's vectorised log / sin / cos differ from the device's in the last
bits), so a hard Gumbel arg-max can flip on a near-tie.  Rollout draws (`get_actions(explore=True)`, `get_random_actions`) stay on
torch's host generator: the two streams only meet through `adopt_torch_rng()` / `export_rng_to_torch()`, as the replay's
`rng="device"` stream meets NumPy's.
"""
import ctypes as C

import numpy as np
import torch

from offpolicy._b200 import capi

# byte offsets inside torch.get_rng_state() (the CPU generator's legacy state struct): int32 left, uint64 next, uint64 key[624]
_LEFT, _NEXT, _KEY = 8, 16, 24
MT_N = 624


class DeviceTorchGenerator(object):
    """A device copy of torch's CPU generator: seeded like `torch.manual_seed` (`seed`), or taking over the host generator's current
    state (`adopt_torch_rng`, the default)."""

    def __init__(self, seed=None):
        self.lib = capi.lib()
        self.dev = capi.device()
        self.state = torch.zeros(capi.TRNG_WORDS, dtype=torch.int32, device=self.dev)
        self._scratch = torch.zeros(0, dtype=torch.int32, device=self.dev)
        if seed is None:
            self.adopt_torch_rng()
        else:
            self.seed(seed)

    def seed(self, seed):
        """torch.manual_seed(seed) for this generator only (the low 32 bits key it, as in torch)."""
        capi.check(self.lib.mx_trng_seed(capi.ptr(self.state), int(seed) & 0xFFFFFFFFFFFFFFFF, capi.stream_ptr()))

    def set_state(self, key, left, next_):
        k = np.ascontiguousarray(np.asarray(key, dtype=np.uint32))
        if k.shape != (MT_N,):
            raise ValueError("generator key must hold 624 words, got shape %s" % (k.shape,))
        capi.check(self.lib.mx_trng_set_state(capi.ptr(self.state), k.ctypes.data_as(C.POINTER(C.c_uint32)), int(left), int(next_),
                                              capi.stream_ptr()))

    def get_state(self):
        """(key uint32[624], left, next) as torch's engine holds them."""
        key = np.zeros(MT_N, dtype=np.uint32)
        left, nxt = C.c_int32(), C.c_int32()
        capi.check(self.lib.mx_trng_get_state(capi.ptr(self.state), key.ctypes.data_as(C.POINTER(C.c_uint32)), C.byref(left), C.byref(nxt),
                                              capi.stream_ptr()))
        return key, int(left.value), int(nxt.value)

    def adopt_torch_rng(self):
        """Continue torch's CPU generator from where it stands now."""
        raw = torch.get_rng_state().numpy().tobytes()
        key = np.frombuffer(raw, dtype=np.uint64, count=MT_N, offset=_KEY).astype(np.uint32)
        left = int(np.frombuffer(raw, dtype=np.int32, count=1, offset=_LEFT)[0])
        nxt = int(np.frombuffer(raw, dtype=np.uint64, count=1, offset=_NEXT)[0])
        self.set_state(key, left, nxt)

    def export_rng_to_torch(self):
        """Hand the stream back to torch's CPU generator: its key and position become this generator's; every other byte of its state
        (the seed, the cached normal samples) stays as it is."""
        key, left, nxt = self.get_state()
        raw = bytearray(torch.get_rng_state().numpy().tobytes())
        raw[_KEY:_KEY + 8 * MT_N] = key.astype(np.uint64).tobytes()
        raw[_LEFT:_LEFT + 4] = np.array([left], dtype=np.int32).tobytes()
        raw[_NEXT:_NEXT + 8] = np.array([nxt], dtype=np.uint64).tobytes()
        torch.set_rng_state(torch.frombuffer(raw, dtype=torch.uint8).clone())

    def state_dict(self):
        key, left, nxt = self.get_state()
        return {"key": key, "left": left, "next": nxt}

    def load_state_dict(self, sd):
        self.set_state(sd["key"], sd["left"], sd["next"])

    def words(self, draw):
        n = int(self.lib.mx_trng_words(C.byref(draw)))
        if n < 0:
            raise capi.MxError(self.lib.mx_last_error().decode())
        return n

    def fill(self, draw):
        """Enqueue one torch call's draws (a capi.TrngDraw) on the current stream."""
        n = self.words(draw)
        if self._scratch.numel() < n:
            self._scratch = torch.zeros(n, dtype=torch.int32, device=self.dev)
        capi.check(self.lib.mx_trng_fill(capi.ptr(self.state), C.byref(draw), capi.ptr(self._scratch), self._scratch.numel(),
                                         capi.stream_ptr()))


def draw(kind, T, rows_n, rows_b, cols, dst, col, ld_t, ld_n, ld_b, std=0.0):
    """torch's draw of shape (T, rows_n * rows_b, cols) (rows agent-major) into dst: value (t, n * rows_b + b, c) lands at float
    col + t * ld_t + n * ld_n + b * ld_b + c."""
    return capi.TrngDraw(kind, int(T), int(rows_n), int(rows_b), int(cols), float(std), dst.data_ptr() + 4 * int(col), int(ld_t), int(ld_n),
                         int(ld_b))

