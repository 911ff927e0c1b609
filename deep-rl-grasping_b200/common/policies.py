"""``stable_baselines.common.policies`` names imported by sb_helper.py:11,18 for the TRPO/PPO branches.  ``MlpPolicy`` is the
actor-critic MLP (tanh, net_arch=[dict(pi=[64, 64], vf=[64, 64])]) that ``ppo2.PPO2`` and ``trpo_mpi.TRPO`` build.
``nature_cnn`` is stable-baselines' default CNN extractor, for ``SAC(CnnPolicy, env, policy_kwargs={"cnn_extractor": nature_cnn})``."""


class MlpPolicy:
    """A marker: the network itself lives in csrc/actor_critic.cu."""
    # ppo2.PPO2 and trpo_mpi.TRPO accept this class by identity; every other learner that reads ``unsupported`` (SAC) refuses it
    unsupported = ("common.policies.MlpPolicy is the actor-critic policy: use it with b200grasp.ppo2.PPO2 or "
                   "b200grasp.trpo_mpi.TRPO")


class CnnPolicy(MlpPolicy):
    pass


def nature_cnn(scaled_images, **kwargs):
    """A sentinel at stable-baselines' import path: ``policy_kwargs["cnn_extractor"] = nature_cnn`` selects the plain
    extractor (c1 8x8/4 -> 32, c2 4x4/2 -> 64, c3 3x3/1 -> 64, fc1 1024 -> 512 over every plane).  The network itself is
    built by the device learner (b2g_sac_create3, B2G_CNN_NATURE); this function is never called."""
    raise NotImplementedError("nature_cnn is built by the SAC learner on the device: pass it as policy_kwargs['cnn_extractor']")
