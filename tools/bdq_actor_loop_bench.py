"""Times ``BDQ.learn`` with and without ``device_obs_norm`` on environments that cost nothing to step.

  python tools/bdq_actor_loop_bench.py [--n_envs 1 16 128] [--configs flat100 depth] [--seconds 2.0]

Both arms run ``BDQ.learn`` itself (prioritised replay, one gradient step per vectorised env step, batch 64, 33 bins, the
layers of the shipped zips) over a DummyVecEnv of ``n_envs`` environments that hand out pre-generated frames, wrapped in
VecNormalize(norm_obs, norm_reward).  flat100: 100-d observations (the shipped BDQ zips); depth: (64, 64, 2) frames that BDQ
flattens to 8192 floats (config/gripper_grasp.yaml, depth_observation).  The two arms alternate in one process; after a
warm-up each arm is timed over windows of at least --seconds.  Printed per case: env-steps/s of every window and overall, and
the bytes copied host->device per vectorised step (BDQLearner.upload_bytes).  The card's name and power limit are read in the
same run and printed first.  Needs a GPU: there is no fallback.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from b200grasp import BDQ  # noqa: E402
from b200grasp.spaces import Box  # noqa: E402
from b200grasp.vec_env import DummyVecEnv, VecNormalize  # noqa: E402

CONFIGS = {"flat100": (100,), "depth": (64, 64, 2)}


class PoolEnv:
    """Hands out frames from a small pre-generated pool: stepping costs an index increment."""

    def __init__(self, shape, seed, horizon=50, pool=8):
        self.observation_space = Box(-np.inf, np.inf, shape)
        self.action_space = Box(-1.0, 1.0, (5,))
        rng = np.random.default_rng(seed)
        self.pool = rng.uniform(0, 2, (pool,) + shape).astype(np.float32)
        self.horizon, self.t, self.k = horizon, 0, 0

    def _obs(self):
        self.k = (self.k + 1) % len(self.pool)
        return self.pool[self.k]

    def reset(self):
        self.t = 0
        return self._obs()

    def step(self, action):
        self.t += 1
        return self._obs(), 1.0, self.t >= self.horizon, {}


def card():
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bdq_actor_loop_bench needs a GPU")
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def make(shape, n_envs, device):
    venv = DummyVecEnv([(lambda i=i: PoolEnv(shape, seed=i)) for i in range(n_envs)])
    env = VecNormalize(venv, norm_obs=True, norm_reward=True, clip_obs=10.0)
    return BDQ("MlpActPolicy", env, buffer_size=20000, batch_size=64, learning_starts=64, num_actions_pad=33, prioritized_replay=True,
               policy_kwargs={"layers": [[64, 64], [32], [32]]}, seed=0, device_obs_norm=device)


def window(model, n_envs, seconds):
    """learn() in slices until `seconds` have passed (every gradient step returns its metrics: the stream is drained);
    returns (env steps, seconds)."""
    steps, t0 = 0, time.perf_counter()
    while time.perf_counter() - t0 < seconds:
        model.learn(n_envs * 20, reset_num_timesteps=False)
        steps += n_envs * 20
    return steps, time.perf_counter() - t0


def case(name, n_envs, seconds):
    shape = CONFIGS[name]
    arms = {"default": make(shape, n_envs, False), "device_obs_norm": make(shape, n_envs, True)}
    for m in arms.values():                      # warm-up: past learning_starts, graph captured, staging allocated
        window(m, n_envs, 0.5)
    base = {k: m.learner.upload_bytes() for k, m in arms.items()}
    tot = {k: [0, 0.0] for k in arms}
    rates = {k: [] for k in arms}
    for _ in range(3):
        for k, m in arms.items():
            s, t = window(m, n_envs, seconds)
            tot[k][0] += s
            tot[k][1] += t
            rates[k].append(round(s / t, 1))
    out = {"config": name, "n_envs": n_envs}
    for k, m in arms.items():
        up = m.learner.upload_bytes()
        vsteps = tot[k][0] / n_envs
        out[k] = {"env_steps_per_s": round(tot[k][0] / tot[k][1], 1), "windows": rates[k],
                  "ms_per_vec_step": round(1e3 * tot[k][1] / vsteps, 3),
                  "h2d_bytes_per_vec_step": round((up["observe"] + up["other"] - base[k]["observe"] - base[k]["other"]) / vsteps)}
    out["speedup"] = round(out["device_obs_norm"]["env_steps_per_s"] / out["default"]["env_steps_per_s"], 3)
    for m in arms.values():
        m.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n_envs", type=int, nargs="+", default=[1, 16, 128])
    ap.add_argument("--configs", nargs="+", default=["flat100", "depth"], choices=sorted(CONFIGS))
    ap.add_argument("--seconds", type=float, default=2.0)
    a = ap.parse_args()
    print(json.dumps(card()), flush=True)
    for name in a.configs:
        for n in a.n_envs:
            print(json.dumps(case(name, n, a.seconds)), flush=True)


if __name__ == "__main__":
    main()
