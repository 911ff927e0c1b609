"""PPO2 timings on the GPU: b2g_ppo_update per rollout (host clock around the call, which ends in a device synchronise) at
the harness's default shapes, and PPO2.learn env-steps/s with an environment that costs nothing.  Prints the card name and
power limit read in the same run, then one JSON line.

  python tools/ppo_bench.py [--reps 10]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import b200grasp  # noqa: E402,F401
from b200grasp.ppo2 import PPO2, PPO2Learner  # noqa: E402
from b200grasp.spaces import Box  # noqa: E402
from b200grasp.vec_env import DummyVecEnv  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def time_update(D, A, E, T=128, nmb=4, noe=4, reps=10):
    L = PPO2Learner(D, A, (64, 64), n_envs=E, n_steps=T, nminibatches=nmb, noptepochs=noe, seed=1)
    rng = np.random.default_rng(0)
    obs = rng.normal(0, 1, (E, D)).astype(np.float32)
    rew, done = np.zeros(E, np.float32), np.zeros(E, np.float32)
    times = []
    for r in range(reps + 2):                      # two warm-up updates (graph capture, first launches)
        for _ in range(T):
            L.rollout_act(obs)
            L.rollout_reward(rew, done)
        perms = np.stack([rng.permutation(T * E) for _ in range(noe)]).astype(np.int32)
        t0 = time.perf_counter()
        L.update(obs, perms, 2.5e-4, 0.2, 0.2)
        if r >= 2:
            times.append(time.perf_counter() - t0)
    L.close()
    return {"obs": D, "A": A, "n_envs": E, "n_steps": T, "minibatch": T * E // nmb, "update_ms_median": 1e3 * float(np.median(times)),
            "update_ms_min": 1e3 * float(np.min(times))}


class FreeEnv:
    def __init__(self, D=100, A=3):
        self.observation_space, self.action_space = Box(-1.0, 1.0, (D,)), Box(-1.0, 1.0, (A,))
        self.o = np.zeros(D, np.float32)

    def reset(self):
        return self.o

    def step(self, a):
        return self.o, 0.0, False, {}

    def close(self):
        pass


def learn_rate(D, A, n_envs, steps):
    env = DummyVecEnv([lambda: FreeEnv(D, A) for _ in range(n_envs)])
    m = PPO2("MlpPolicy", env, seed=0)
    m.learn(128 * n_envs)                         # warm-up: one update
    t0 = time.perf_counter()
    m.learn(steps)
    dt = time.perf_counter() - t0
    n = m.num_timesteps
    m.close()
    return {"obs": D, "A": A, "n_envs": n_envs, "env_steps": n, "env_steps_per_s": n / dt}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    c = card()
    print("card, power limit:", c)
    upd = [time_update(100, 3, 1, reps=args.reps)] + [time_update(8192, 5, E, reps=args.reps) for E in (1, 16, 128)]
    for u in upd:
        print(u)
    learn = [learn_rate(100, 3, 1, 128 * 20), learn_rate(8192, 5, 1, 128 * 10)]
    for x in learn:
        print(x)
    print(json.dumps({"card": c, "update": upd, "learn": learn}))


if __name__ == "__main__":
    main()
