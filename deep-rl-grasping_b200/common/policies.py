"""``stable_baselines.common.policies`` names imported by sb_helper.py:11,18 for the TRPO/PPO branches.  ``MlpPolicy`` is the
actor-critic MLP (tanh, net_arch=[dict(pi=[64, 64], vf=[64, 64])]) that ``ppo2.PPO2`` and ``trpo_mpi.TRPO`` build."""


class MlpPolicy:
    """A marker: the network itself lives in csrc/actor_critic.cu."""
    # ppo2.PPO2 and trpo_mpi.TRPO accept this class by identity; every other learner that reads ``unsupported`` (SAC) refuses it
    unsupported = ("common.policies.MlpPolicy is the actor-critic policy: use it with b200grasp.ppo2.PPO2 or "
                   "b200grasp.trpo_mpi.TRPO")


class CnnPolicy(MlpPolicy):
    pass
