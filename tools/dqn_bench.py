"""Times the DQN learner's captured gradient step and ``DQN.learn`` on an environment that costs nothing to step.

  python tools/dqn_bench.py [--seconds 2.0] [--repeats 3]

Gradient steps/s of ``DQNLearner.step`` (one CUDA graph per step) at the shipped zip's shape (obs 100, 12 actions, layers
[64, 64], prioritised replay) with batch 32 and with batch 1024, and env-steps/s of ``DQN.learn`` (batch 32, PER, one gradient
step per env step past learning_starts) over a PoolEnv that hands out pre-generated frames.  Every case is warmed up and then
timed over --repeats windows of at least --seconds each, ending in a device synchronise.  The card's name and power limit are
read in the same run and printed first; one JSON line per case follows.  Needs a GPU: there is no fallback.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from b200grasp.deepq import DQN, DQNLearner  # noqa: E402
from b200grasp.spaces import Box, Discrete  # noqa: E402


class PoolEnv:
    """100-float frames from a small pre-generated pool, 12 actions; episodes of 50 steps."""
    observation_space = Box(-1.0, 1.0, (100,))
    action_space = Discrete(12)

    def __init__(self, seed=0, pool=8):
        self.pool = np.random.default_rng(seed).uniform(-1, 1, (pool, 100)).astype(np.float32)
        self.t = self.k = 0

    def _obs(self):
        self.k = (self.k + 1) % len(self.pool)
        return self.pool[self.k]

    def reset(self):
        self.t = 0
        return self._obs()

    def step(self, action):
        self.t += 1
        return self._obs(), float(int(np.asarray(action).reshape(-1)[0]) == self.k % 12), self.t >= 50, {}

    def close(self):
        pass


def card():
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("dqn_bench needs a GPU")
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def windows(fn, seconds, repeats):
    """fn(k) runs k units and returns once the device is idle; -> units/s of each window of >= seconds"""
    k, rates = 16, []
    while True:                       # size a window
        t0 = time.perf_counter()
        fn(k)
        dt = time.perf_counter() - t0
        if dt >= 0.25:
            break
        k *= 4
    k = int(k * seconds / dt) + 1
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn(k)
        rates.append(k / (time.perf_counter() - t0))
    return rates


def bench_step(B, seconds, repeats):
    rng = np.random.default_rng(0)
    L = DQNLearner(100, 12, (64, 64), B, 50000, 1.0, seed=1, prioritized_replay=True)
    n = 20000
    L.replay_add(rng.uniform(-1, 1, (n, 100)), rng.integers(0, 12, n).astype(np.float32), rng.random(n), rng.uniform(-1, 1, (n, 100)),
                 (rng.random(n) < 0.02).astype(np.float32))
    L.set_per_beta(0.5)
    L.step(50, 5e-4)                  # capture + warm-up (step returns after a synchronise)
    rates = windows(lambda k: L.step(k, 5e-4), seconds, repeats)
    L.close()
    return {"case": f"graph_step_b{B}_per", "unit": "gradient steps/s", "windows": [round(r, 1) for r in rates],
            "median": round(float(np.median(rates)), 1)}


def bench_learn(seconds, repeats):
    model = DQN("MlpPolicy", PoolEnv(), batch_size=32, prioritized_replay=True, learning_starts=1000, seed=1)
    model.learn(2000)                 # past learning_starts: every timed step trains
    rates = windows(lambda k: model.learn(k, reset_num_timesteps=False), seconds, repeats)
    model.close()
    return {"case": "learn_b32_per_zero_cost_env", "unit": "env steps/s", "windows": [round(r, 1) for r in rates],
            "median": round(float(np.median(rates)), 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=2.0)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    print(json.dumps({"card": card()}))
    for B in (32, 1024):
        print(json.dumps(bench_step(B, a.seconds, a.repeats)), flush=True)
    print(json.dumps(bench_learn(a.seconds, a.repeats)), flush=True)


if __name__ == "__main__":
    main()
