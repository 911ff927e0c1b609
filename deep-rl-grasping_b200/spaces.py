"""Tiny stand-in for gym.spaces.Box (gym is not a dependency of the learner).  Any object with
.shape/.low/.high/.sample() works; RobotEnv's own gym spaces (robot.py:207-228) are used as-is."""
import numpy as np


class Box:
    def __init__(self, low, high, shape=None, dtype=np.float32, seed=None):
        if shape is None:
            shape = np.shape(low)
        self.shape = tuple(shape)
        self.dtype = np.dtype(dtype)
        self.low = np.broadcast_to(np.asarray(low, self.dtype), self.shape).copy()
        self.high = np.broadcast_to(np.asarray(high, self.dtype), self.shape).copy()
        self._rng = np.random.default_rng(seed)

    def sample(self):
        return self._rng.uniform(self.low, self.high).astype(self.dtype)

    def seed(self, seed=None):
        self._rng = np.random.default_rng(seed)

    def __repr__(self):
        return f"Box{self.shape}"


class Discrete:
    """Stand-in for gym.spaces.Discrete(n): actions 0 .. n-1 (the DQN learner's action space)."""

    def __init__(self, n, seed=None):
        self.n = int(n)
        self.shape = ()
        self.dtype = np.dtype(np.int64)
        self._rng = np.random.default_rng(seed)

    def sample(self):
        return int(self._rng.integers(0, self.n))

    def contains(self, x):
        return isinstance(x, (int, np.integer)) and 0 <= int(x) < self.n

    def seed(self, seed=None):
        self._rng = np.random.default_rng(seed)

    def __repr__(self):
        return f"Discrete({self.n})"
