"""Run the UNMODIFIED reference SMAC runner (offpolicy/runner/rnn/smac_runner.py, what scripts/train_smac_qmix.sh starts) on a
synthetic SMAC-like environment with 36 actions, as on 27m_vs_30m (6 + 30 enemies): 5 agents, obs 40, state 60, availability masks
with the no-op always available, episode limit 20.  Past 32 actions the drop-in engine's Q-head kernels hold two actions per lane.
Same engines and output line as run_smac_like.py.  Test infrastructure only.
"""
import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from run_mpe import install_shims, ROOT  # noqa: E402
from run_smac_like import make_env_class  # noqa: E402


def make_many_actions_env_class():
    Base = make_env_class()

    class SyntheticSMACManyActions(Base):
        """Base's dynamics with 5 agents and 36 actions."""
        N, O, S, A, LIMIT = 5, 40, 60, 36, 20

    return SyntheticSMACManyActions

def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--engine", default="b200", choices=["b200", "b200-gpu", "reference"])
    ap.add_argument("--algo", default="qmix")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--seed", type=int, default=1)
    a, extra = ap.parse_known_args()
    rh = install_shims()
    import numpy as np
    import torch
    torch.set_num_threads(1)
    if a.engine == "reference":
        rh.import_reference()
        device = torch.device("cpu")
    else:
        sys.path.insert(0, os.path.join(ROOT, "off-policy_b200"))
        from offpolicy._b200 import capi
        if a.engine == "b200":
            sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
            from build_emu import build
            capi._install_for_tests(build())
        else:
            capi.lib()
        device = capi.device()
    from offpolicy.config import get_config
    from offpolicy.utils.util import get_cent_act_dim, get_dim_from_space
    from offpolicy.envs.env_wrappers import ShareDummyVecEnv
    from offpolicy.runner.rnn.smac_runner import SMACRunner
    import offpolicy.utils.rec_buffer as rb
    parser = get_config()
    parser.add_argument('--map_name', type=str, default='3m')                                    # train_smac.py:52-59
    parser.add_argument('--use_available_actions', action='store_false', default=True)
    parser.add_argument('--use_same_share_obs', action='store_false', default=True)
    parser.add_argument('--use_global_all_local_state', action='store_true', default=False)
    argv = ["--env_name", "StarCraft2", "--algorithm_name", a.algo, "--experiment_name", "b200", "--map_name", "many_actions", "--seed", str(a.seed),
            "--buffer_size", "32", "--lr", "5e-4", "--batch_size", "4", "--num_env_steps", str(a.steps),
            "--num_random_episodes", "2", "--log_interval", "100000", "--eval_interval", "10000000", "--save_interval", "10000000",
            "--gain", "1"] + list(extra)
    all_args = parser.parse_known_args(argv)[0]
    all_args.use_wandb = False
    torch.manual_seed(all_args.seed)
    np.random.seed(all_args.seed)
    Env = make_many_actions_env_class()
    env = ShareDummyVecEnv([lambda: Env(all_args.seed)])
    eval_env = ShareDummyVecEnv([lambda: Env(all_args.seed * 50000)])
    policy_info = {'policy_0': {"cent_obs_dim": get_dim_from_space(env.share_observation_space[0]), "cent_act_dim": get_cent_act_dim(env.action_space),
                                "obs_space": env.observation_space[0], "share_obs_space": env.share_observation_space[0],
                                "act_space": env.action_space[0]}}
    from pathlib import Path
    config = {"args": all_args, "policy_info": policy_info, "policy_mapping_fn": lambda i: 'policy_0', "env": env, "eval_env": eval_env,
              "num_agents": Env.N, "device": device, "run_dir": Path(tempfile.mkdtemp()), "buffer_length": Env.LIMIT,
              "use_same_share_obs": all_args.use_same_share_obs, "use_available_actions": all_args.use_available_actions}
    stdout = sys.stdout
    sys.stdout = sys.stderr
    runner = SMACRunner(config=config)
    rewards, infos = [], []
    collect = runner.collecter

    def recording_collect(*args, **kw):
        info = collect(*args, **kw)
        rewards.append(float(info["average_episode_rewards"]))
        return info
    runner.collecter = recording_collect
    train = runner.trainer.train_policy_on_batch

    def recording_train(*args, **kw):
        out = train(*args, **kw)
        infos.append({k: float(v) for k, v in out[0].items() if k != "update_actor"})
        return out
    runner.trainer.train_policy_on_batch = recording_train
    total = 0
    while total < all_args.num_env_steps:
        total = runner.run()
    sys.stdout = stdout
    print(json.dumps(dict(engine=a.engine, algo=a.algo, buffer=rb.__file__, trainer=type(runner.trainer).__module__, env_steps=int(total),
                          train_steps=int(runner.total_train_steps), rewards=rewards, train=infos, act_dim=Env.A)))


if __name__ == "__main__":
    main()
