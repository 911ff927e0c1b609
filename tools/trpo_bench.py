"""TRPO timings on the GPU: one b2g_trpo_update (host clock around the call, which ends in a device synchronise), median of 10
after 2 warm-ups, at the harness's shape on the simplified env and at flattened depth frames.  Prints one JSON line per case
with the card name and power limit read in the same run.

  python tools/trpo_bench.py [--reps 10]
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
from b200grasp.trpo_mpi import TRPOLearner, init_params  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def time_update(D, A, N, reps=10):
    L = TRPOLearner(D, A, (64, 64), N, seed=1)
    L.load_parameters(init_params(D, A, (64, 64), 1))
    rng = np.random.default_rng(0)
    obs = rng.uniform(0, 1, (N + 1, D)).astype(np.float32)
    rew = rng.normal(0, 1, N).astype(np.float32)
    times, accepted = [], []
    for r in range(reps + 2):                      # two warm-up updates (graph capture, first launches)
        for t in range(N):
            L.rollout_act(obs[t])
            L.rollout_reward(rew[t], float(t % 97 == 96))
        perms = np.stack([rng.permutation(N) for _ in range(L.vf_iters)]).astype(np.int32)
        t0 = time.perf_counter()
        m = L.update(obs[N], perms)
        if r >= 2:
            times.append(time.perf_counter() - t0)
            accepted.append(m["accepted"])
    L.close()
    return {"obs": D, "A": A, "timesteps_per_batch": N, "update_ms_median": 1e3 * float(np.median(times)),
            "update_ms_min": 1e3 * float(np.min(times)), "accepted": accepted}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    gpu = card()
    for D, A, N in ((100, 3, 400), (8192, 5, 1024), (8192, 5, 16384)):
        print(json.dumps(dict(time_update(D, A, N, a.reps), gpu=gpu)), flush=True)


if __name__ == "__main__":
    main()
