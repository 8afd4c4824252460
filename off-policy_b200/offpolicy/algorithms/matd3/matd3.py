"""Drop-in `MATD3` (reference: offpolicy/algorithms/matd3/matd3.py): MADDPG with twin Q heads and actor_update_interval = 2 -- which
the reference's transition-level trainer never applies (see algorithms/maddpg/maddpg.py)."""
from offpolicy.algorithms.maddpg.maddpg import MADDPG


class MATD3(MADDPG):
    def __init__(self, args, num_agents, policies, policy_mapping_fn, device=None):
        MADDPG.__init__(self, args, num_agents, policies, policy_mapping_fn, device=device, actor_update_interval=2)
