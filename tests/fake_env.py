"""Synthetic stand-in for gripper-env-v0 (gym / pybullet are not installable here): same observation
layout as RobotEnv._observe (robot.py:183-205: depth plane + zero pad plane whose [0,0] holds the
gripper width), Box(0,255) observation space (robot.py:224-228), Box(-1,1)^5 actions
(actuator.py:72-73), sparse-ish reward, fixed horizon."""
import numpy as np

from b200grasp.spaces import Box


class FakeGraspEnv:
    def __init__(self, seed=0, horizon=20, obs_shape=(64, 64, 2)):
        self.observation_space = Box(0.0, 255.0, obs_shape)
        self.action_space = Box(-1.0, 1.0, (5,), seed=seed)
        self.rng = np.random.default_rng(seed)
        self.horizon, self.t = horizon, 0
        self.obs_shape = obs_shape

    def _obs(self):
        o = np.zeros(self.obs_shape, np.float32)
        o[..., :-1] = np.clip(self.rng.normal(0.3, 0.1, self.obs_shape[:2] + (self.obs_shape[2] - 1,)), 0.02, 2.0)
        o[0, 0, -1] = self.rng.uniform(0, 1)
        return o

    def reset(self):
        self.t = 0
        return self._obs()

    def step(self, action):
        self.t += 1
        r = float(-200.0 + 300.0 * (np.asarray(action)[2] > 0.5))
        return self._obs(), r, self.t >= self.horizon, {"is_success": r > 0}

    def close(self):
        pass


def make_env(config, evaluate=False, validate=False, test=False):
    """Factory with the signature train_cli expects (mirrors gym.make('gripper-env-v0', config=..., evaluate=..., ...))."""
    return FakeGraspEnv(seed=1 if evaluate else 0, horizon=20)


class FakeFlatEnv:
    """Flat observations of ``obs_dim`` floats in [0, 1) and a Box(-1, 1)^n_act action space, or Discrete(n_discrete) when
    that is given: the shape of the BDQ, DQN and PPO2 configurations."""

    def __init__(self, seed=0, horizon=5, obs_dim=6, n_act=3, n_discrete=None):
        from b200grasp.spaces import Discrete
        self.observation_space = Box(0.0, 1.0, (obs_dim,))
        self.action_space = Box(-1.0, 1.0, (n_act,), seed=seed) if n_discrete is None else Discrete(n_discrete, seed=seed)
        self.rng = np.random.default_rng(seed)
        self.horizon, self.t, self.obs_dim = horizon, 0, obs_dim

    def reset(self):
        self.t = 0
        return self.rng.uniform(0, 1, self.obs_dim).astype(np.float32)

    def step(self, action):
        self.t += 1
        return self.rng.uniform(0, 1, self.obs_dim).astype(np.float32), float(self.rng.normal()), self.t >= self.horizon, {}

    def close(self):
        pass
