"""Seeded synthetic replay data of the reference's shapes and statistics (SURVEY.md §8d).

Raw (un-normalised) transitions as ``replay_buffer.add`` would store them when VecNormalize wraps
the env: depth plane ~ clip(N(mean_ij, var_ij), 0.02, 2.0) from the shipped ``obs_rms`` (the last
image plane; with 2 or more image planes the ones before it are integer colour 0..255); the pad
plane is zero except pixel [0,0] = gripper width (robot.py:199-200); reward mixture from
config/gripper_grasp.yaml:42-46 / rewards.py:128-138; done ~ Bernoulli(1/15).
"""
from __future__ import annotations

import numpy as np

DATA_SEED = 20260924


def make_transitions(n: int, obs_mean: np.ndarray, obs_var: np.ndarray, seed: int = DATA_SEED, n_act: int = 5):
    rng = np.random.default_rng(seed)
    shape = obs_mean.shape
    sd = np.sqrt(obs_var)

    def draw_obs():
        o = rng.standard_normal((n,) + shape) * sd + obs_mean
        if len(shape) == 3:
            c = shape[2] - 1
            if c >= 2:                              # colour planes 0..255 before the depth plane (RGB-D when c = 4)
                o[..., :c - 1] = np.clip(np.round(o[..., :c - 1]), 0, 255)
            o[..., c - 1] = np.clip(o[..., c - 1], 0.02, 2.0)   # depth metres, the last image plane
            pad = np.zeros((n,) + shape[:2])
            pad[:, 0, 0] = rng.uniform(0, 1, n)
            o[..., c] = pad
        return o.astype(np.float32)

    obs, next_obs = draw_obs(), draw_obs()
    act = rng.uniform(-1, 1, (n, n_act)).astype(np.float32)
    kind = rng.random(n)
    rew = np.where(kind < 0.93, -200.0, np.where(kind < 0.99, 100.0 + 1000.0 * rng.uniform(0, 0.01, n), 10000.0))
    done = (rng.random(n) < 1.0 / 15.0).astype(np.float32)
    return dict(obs=obs, next_obs=next_obs, act=act, rew=rew.astype(np.float32), done=done)


def make_eps(n: int, n_act: int = 5, seed: int = DATA_SEED + 1) -> np.ndarray:
    return np.random.default_rng(seed).standard_normal((n, n_act)).astype(np.float32)


def make_indices(n_batch: int, n_slots: int, seed: int = DATA_SEED + 2) -> np.ndarray:
    return np.random.default_rng(seed).integers(0, n_slots, n_batch).astype(np.int64)


def make_depth_scenes(n: int, seed: int = 0, size: int = 64) -> np.ndarray:
    """Depth-like synthetic frames [n, size, size, 1] float32 for the perception encoder: background filtered to 0
    (as sensor.py:207-213 zeroes plane/robot/table/tray pixels), 1-4 box-shaped objects at 0.15-0.5 m."""
    rng = np.random.default_rng(seed)
    imgs = np.zeros((n, size, size, 1), np.float32)
    for i in range(n):
        for _ in range(int(rng.integers(1, 5))):
            y, x = rng.integers(5, size - 14, 2)
            h, w = rng.integers(5, 14, 2)
            imgs[i, y:y + h, x:x + w, 0] = rng.uniform(0.15, 0.5)
    return imgs
