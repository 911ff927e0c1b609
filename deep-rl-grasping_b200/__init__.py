"""b200grasp -- H100-native SAC / BDQ / DQN / PPO2 / TRPO learners behind the stable-baselines model API used by
BarisYazici/deep-rl-grasping (manipulation_main/training/sb_helper.py:104-128,175).

Import as ``b200grasp`` (``b200grasp.py`` at the repo root aliases this directory, whose name
``deep-rl-grasping_b200`` is not a Python identifier).
"""
from . import _lib, sb_io, synth  # noqa: F401
from . import callbacks, encoders, h5min, spaces, vec_env  # noqa: F401
from .learner import Learner  # noqa: F401
from .bdq import BDQ, BDQLearner  # noqa: F401
from .sac_model import SAC, CnnPolicy, MlpPolicy  # noqa: F401
from . import bench, common, deepq, evaluation, logger, ppo2, sac, trpo_mpi  # noqa: F401  (stable_baselines-shaped namespaces)
from .common import set_global_seeds  # noqa: F401
from .vec_env import DummyVecEnv, SubprocVecEnv, VecNormalize  # noqa: F401

_OUT_OF_SCOPE = ("DQN", "DDPG", "TD3", "TRPO", "PPO1", "PPO2", "A2C", "ACER", "ACKTR", "HER", "GAIL")


def __getattr__(name):           # sb.DQN / sb.TRPO / ... (sb_helper.py:139-199): the other branches of SBPolicy.learn
    if name == "DQN":
        raise NotImplementedError("b200grasp.DQN: the DQN learner is b200grasp.deepq.DQN (stable_baselines.deepq.DQN); "
                                  "write sb.deepq.DQN at the DQN call sites")
    if name == "PPO2":
        raise NotImplementedError("b200grasp.PPO2: the PPO2 learner is b200grasp.ppo2.PPO2 (stable_baselines.ppo2.PPO2); "
                                  "write sb.ppo2.PPO2 at the PPO call sites")
    if name == "TRPO":
        raise NotImplementedError("b200grasp.TRPO: the TRPO learner is b200grasp.trpo_mpi.TRPO (stable_baselines.trpo_mpi.TRPO); "
                                  "write sb.trpo_mpi.TRPO at the TRPO call sites")
    if name in _OUT_OF_SCOPE:
        raise NotImplementedError(f"b200grasp.{name}: only the SAC and BDQ learners are built (DESIGN.md section 7)")
    raise AttributeError(name)


__all__ = ["BDQ", "BDQLearner", "SAC", "CnnPolicy", "MlpPolicy", "Learner", "DummyVecEnv", "VecNormalize", "callbacks", "encoders", "h5min", "spaces", "sb_io", "synth", "vec_env"]
