"""The fallback exchange of the data-parallel actor-critic learners on CPU: 2 gloo ranks (no peer memory), each training on half of a
golden batch with the emulated kernels, must reproduce the reference's single-batch updates -- R-MADDPG (recurrent, Box) and MLP MATD3
-- and stay bit-identical to each other.  Each update all-reduces the critic's buffer, applies it, then the actor's."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from helpers import load_golden, rel_err

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("name", ["maddpg_box", "mlp_matd3_box"])
def test_two_gloo_ranks_equal_single_batch_reference(emu_engine, name):
    g = load_golden(name)
    with tempfile.TemporaryDirectory() as td:
        port = 29500 + (os.getpid() + (13 if name.startswith("mlp") else 3)) % 1000
        procs = []
        for r in range(2):
            env = dict(os.environ, RANK=str(r), WORLD_SIZE="2", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), OMP_NUM_THREADS="1")
            procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "dp_worker_maddpg.py"), td, name], env=env,
                                          stdout=subprocess.PIPE, stderr=subprocess.STDOUT))
        outs = [p.communicate(timeout=900)[0].decode() for p in procs]
        assert all(p.returncode == 0 for p in procs), "\n".join(outs)
        r0, r1 = dict(np.load(os.path.join(td, "rank0.npz"))), dict(np.load(os.path.join(td, "rank1.npz")))
    assert set(r0) == set(r1)
    steps = sorted({k.split(".")[0] for k in r0 if k.startswith("s")})
    assert len(steps) >= 2
    for s in steps:
        if "%s.update_actor" % s in g:
            assert int(r0["%s.update_actor" % s]) == int(g["%s.update_actor" % s])
        for k in ("critic_loss", "critic_grad_norm", "actor_loss", "actor_grad_norm"):
            key = "%s.%s" % (s, k)
            if key in r0:
                assert float(r0[key]) == float(r1[key])
                assert rel_err(float(r0[key]), float(g[key])) <= 1e-4, (key, float(r0[key]), float(g[key]))
    for k in r0:
        if k.startswith("vec"):
            assert np.array_equal(r0[k], r1[k]), k          # live, target and Adam vectors: bit-identical replicas
