"""Whole-run checkpoint / resume (SURVEY.md section 8(f).3).

The reference runner saves network weights only (`torch.save(state_dict)` per net, runner/rnn/base_runner.py:286-337) and its
restore path is broken (`restore_q` runs before the trainer exists, App. D-3).  The drop-in classes keep those per-network
`state_dict()`s (same key names, so the reference's files load), and add what a bit-exact resume needs:

    save_checkpoint(path, trainer, buffer)     # live + target parameters, Adam moments / step count, the replay (episodes,
    load_checkpoint(path, trainer, buffer)     # PER trees, device MT19937), NumPy's and torch's host generators

After `load_checkpoint` into freshly constructed objects the next learner steps are bit-identical to the uninterrupted run
(tests/test_emu_checkpoint.py, tests/test_gpu_checkpoint.py, tests/test_{emu,gpu}_checkpoint_maddpg.py).

Trainers: `QMix`, `VDN`, `M_QMix`, `M_VDN` (QMix.state_dict), `R_MADDPG`, `R_MATD3`, `MADDPG`, `MATD3` (shared or one policy per agent;
offpolicy/_b200/maddpg_state.py).  Replays: `RecReplayBuffer`, `PrioritizedRecReplayBuffer`, `MlpReplayBuffer`,
`PrioritizedMlpReplayBuffer`.  A checkpoint of another configuration is refused with ValueError.
"""
import numpy as np
import torch

FORMAT = 1


def save_checkpoint(path, trainer=None, buffer=None, extra=None):
    ck = {"format": FORMAT, "numpy_rng": np.random.get_state(), "torch_rng": torch.get_rng_state(), "extra": extra}
    if trainer is not None:
        ck["trainer"] = trainer.state_dict()
    if buffer is not None:
        ck["buffer"] = buffer.state_dict()
    torch.save(ck, path)
    return path


def load_checkpoint(path, trainer=None, buffer=None, restore_host_rng=True):
    ck = torch.load(path, map_location="cpu", weights_only=False)
    if ck.get("format") != FORMAT:
        raise ValueError("unknown checkpoint format %r" % (ck.get("format"),))
    if trainer is not None:
        if "trainer" not in ck:
            raise KeyError("checkpoint holds no learner state")
        trainer.load_state_dict(ck["trainer"])
    if buffer is not None:
        if "buffer" not in ck:
            raise KeyError("checkpoint holds no replay state")
        buffer.load_state_dict(ck["buffer"])
    if restore_host_rng:
        np.random.set_state(ck["numpy_rng"])
        torch.set_rng_state(ck["torch_rng"])
    return ck.get("extra")
