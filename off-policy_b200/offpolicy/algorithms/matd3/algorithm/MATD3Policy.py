"""Drop-in `MATD3Policy` (reference: offpolicy/algorithms/matd3/algorithm/MATD3Policy.py): twin Q heads + target smoothing noise."""
from offpolicy.algorithms.maddpg.algorithm.MADDPGPolicy import MADDPGPolicy


class MATD3Policy(MADDPGPolicy):
    def __init__(self, config, policy_config, train=True):
        MADDPGPolicy.__init__(self, config, policy_config, target_noise=config["args"].target_action_noise_std, td3=True, train=train)
