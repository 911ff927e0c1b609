"""Synthetic stand-in for the encoded-depth env with a deferred sensor (encoders.DeferredEncodedDepthImgSensor): raw
observations [64*64 depth | T tail floats], the depth frames drawn from synth.make_depth_scenes, the tail in [0, 1)
(the actuator state, a time feature)."""
import numpy as np

from b200grasp import synth
from b200grasp.spaces import Box

PIXELS = 64 * 64


class FakeDeferredEnv:
    def __init__(self, seed=0, horizon=7, tail=1, n_act=5, pool=16):
        low = np.concatenate([np.zeros(PIXELS), np.zeros(tail)])
        high = np.concatenate([np.full(PIXELS, np.inf), np.ones(tail)])
        self.observation_space = Box(low, high, (PIXELS + tail,))
        self.action_space = Box(-1.0, 1.0, (n_act,), seed=seed)
        rng = np.random.default_rng(seed)
        self.pool = np.concatenate([synth.make_depth_scenes(pool, seed=seed).reshape(pool, PIXELS),
                                    rng.uniform(0, 1, (pool, tail))], axis=1).astype(np.float32)
        self.horizon, self.t, self.k = horizon, 0, seed % pool

    def _obs(self):
        self.k = (self.k + 1) % len(self.pool)
        return self.pool[self.k].copy()

    def reset(self):
        self.t = 0
        return self._obs()

    def step(self, action):
        self.t += 1
        return self._obs(), float(np.asarray(action).reshape(-1)[0]), self.t >= self.horizon, {}

    def close(self):
        pass


def make_env(config, evaluate=False, validate=False, test=False):
    """train_cli factory: actuator tail, like the reference env's encoded observation without `simplified`."""
    return FakeDeferredEnv(seed=1 if evaluate else 0, horizon=7, tail=1)
