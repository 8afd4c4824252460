"""The unmodified reference SMAC runner (runner/rnn/smac_runner.py) with QMIX and VDN on a synthetic SMAC-like env with 36 actions
(5 agents, no-op always available; tests/integration/run_smac_like_many_actions.py): the drop-in engine against the pure reference
with one seed.  The reference's recurrent VDN mixer is shape-broken (SURVEY.md App. D-1), so VDN runs on the drop-in only, as in
test_emu_runner_integration.py: the env asserts that no unavailable action is ever chosen, and every train_info value is finite.
Needs the reference checkout."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("OFFPOLICY_REFERENCE_ROOT", "/root/reference")
pytestmark = pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "offpolicy", "runner")), reason="reference checkout not present")


@pytest.mark.parametrize("algo", ["qmix", "vdn"])
def test_reference_smac_runner_many_actions_on_the_drop_in_engine(emu_engine, algo):
    script = os.path.join(ROOT, "tests", "integration", "run_smac_like_many_actions.py")
    engines = ("b200", "reference") if algo == "qmix" else ("b200",)
    procs = {e: subprocess.Popen([sys.executable, script, "--engine", e, "--algo", algo, "--steps", "200"], stdout=subprocess.PIPE,
                                 stderr=subprocess.PIPE, env=dict(os.environ, OMP_NUM_THREADS="1")) for e in engines}
    out = {}
    for e, p in procs.items():
        so, se = p.communicate(timeout=1500)
        assert p.returncode == 0, "%s failed:\n%s" % (e, se.decode()[-3000:])
        out[e] = json.loads(so.decode().strip().splitlines()[-1])
    ours = out["b200"]
    assert "off-policy_b200" in ours["buffer"] and ours["act_dim"] == 36
    assert ours["train_steps"] > 0 and len(ours["rewards"]) >= 2
    for info in ours["train"]:
        assert all(v == v and abs(v) < 1e9 for v in info.values()), info            # finite
    if algo != "qmix":
        return
    ref = out["reference"]
    assert REF in ref["buffer"] and ref["act_dim"] == 36
    assert ours["train_steps"] == ref["train_steps"] > 0
    assert ours["rewards"] == ref["rewards"]                     # identical episodes, bit for bit
    assert len(ours["train"]) == len(ref["train"]) > 0
    for a, b in zip(ours["train"], ref["train"]):
        assert set(a) == set(b)
        for k in a:
            assert abs(a[k] - b[k]) <= 2e-5 * max(1.0, abs(b[k])), (k, a[k], b[k])
