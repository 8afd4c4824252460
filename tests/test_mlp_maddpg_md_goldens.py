"""The transition-level MADDPG / MATD3 with MultiDiscrete action spaces against outputs of the unmodified reference
(tests/golden/mlp_*md*.npz, made by make_goldens_mlp_maddpg_md.py): the oracle (oracle/maddpg_mlp_md.py) to fp32 round-off, with the
tolerances of test_mlp_maddpg_goldens.py, and its Gumbel draws (one call per sub-space) equal to the reference's."""
import pytest

import mlp_maddpg_md_checks as mdc


@pytest.mark.parametrize("name", mdc.GOLDENS_MD)
def test_oracle_reproduces_reference(name):
    mdc.oracle_against_golden(name)
