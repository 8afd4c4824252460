"""The unmodified reference SMAC runner (runner/rnn/smac_runner.py) with QMIX on a synthetic SMAC-like env whose global state is wide
(4 agents, obs 150, state 702 as with --use_global_all_local_state; tests/integration/run_smac_like_wide.py): the drop-in engine,
which trains through its wide-state mixer path, against the pure reference with one seed.  Needs the reference checkout."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("OFFPOLICY_REFERENCE_ROOT", "/root/reference")
pytestmark = pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "offpolicy", "runner")), reason="reference checkout not present")


def test_reference_smac_runner_wide_state_on_the_drop_in_engine(emu_engine):
    script = os.path.join(ROOT, "tests", "integration", "run_smac_like_wide.py")
    procs = {e: subprocess.Popen([sys.executable, script, "--engine", e, "--steps", "200"], stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                                 env=dict(os.environ, OMP_NUM_THREADS="1")) for e in ("b200", "reference")}
    out = {}
    for e, p in procs.items():
        so, se = p.communicate(timeout=1500)
        assert p.returncode == 0, "%s failed:\n%s" % (e, se.decode()[-3000:])
        out[e] = json.loads(so.decode().strip().splitlines()[-1])
    ours, ref = out["b200"], out["reference"]
    assert "off-policy_b200" in ours["buffer"] and REF in ref["buffer"]
    assert ours["wide_state_path"] == 1
    assert ours["train_steps"] == ref["train_steps"] > 0
    assert ours["rewards"] == ref["rewards"]                     # identical episodes, bit for bit
    assert len(ours["train"]) == len(ref["train"]) > 0
    for a, b in zip(ours["train"], ref["train"]):
        assert set(a) == set(b)
        for k in a:
            assert abs(a[k] - b[k]) <= 2e-5 * max(1.0, abs(b[k])), (k, a[k], b[k])
