"""Step time of the replayed BDQ step (batch 64, 3 x 33 bins, prioritised replay) and the DQN step (batch 32, 12 actions) with the
replay in frames (replay_frames / frame_capacity) against the default two-rows-per-slot layout, on 100-d and 8192-d rows.  The
two layouts alternate in windows inside one process; each window times CUDA-graph steps with CUDA events.  The replay is
filled past L2 (50 MB): 16,384 slots of 8192-d rows are 1 GB per row array, 200,000 slots of 100-d rows 80 MB.  The fill
is the learn loop's stream of 256 vectorised envs with episodes of 10 steps: row i of a call continues row i of the
previous one, so the frame arm shares every observation but the first of an episode (about 1.1 frames per transition,
inside its 1.125 budget; its evicted_early is printed).

    python tools/bdq_replay_frames_bench.py [--windows 5] [--steps 2000] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from b200grasp.bdq import BDQLearner  # noqa: E402
from b200grasp.dqn import DQNLearner  # noqa: E402


def fill(L, n, E, act_cols, n_act, n_envs=256, episode=10):
    """n transitions of n_envs episodic streams, one call per env step: obs(t+1) = next_obs(t) within an episode, and a
    finished env continues from a reset frame; episodes are staggered across the envs"""
    rng = np.random.default_rng(0)
    cur = rng.normal(size=(n_envs, E)).astype(np.float32)
    t = np.arange(n_envs) % episode
    for c0 in range(0, n, n_envs):
        m = min(n_envs, n - c0)
        nxt = rng.normal(size=(n_envs, E)).astype(np.float32)
        t += 1
        done = (t % episode == 0).astype(np.float32)
        act = rng.integers(0, n_act, (n_envs, act_cols)).astype(np.float32)
        L.replay_add(cur[:m], act[:m], rng.normal(size=m).astype(np.float32), nxt[:m], done[:m])
        reset = rng.normal(size=(n_envs, E)).astype(np.float32)
        cur = np.where(done[:, None] != 0, reset, nxt)


def ms_per_step(L, steps):
    L.step(steps // 10)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    L.step(steps)          # one call: the graph replays back to back on the handle's stream; step() drains it before returning
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--out", default=None, help="also write the rows, card and power limit to this JSON file")
    args = ap.parse_args()
    name = torch.cuda.get_device_name(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True).stdout.strip()
    print(f"device: {name}, power limit {power}")
    rows = []
    for algo, E, cap in (("BDQ", 100, 200_000), ("BDQ", 8192, 16_384), ("DQN", 100, 200_000), ("DQN", 8192, 16_384)):
        fc = int(cap * 1.125) + 1
        make = {
            "BDQ": lambda f: BDQLearner(E, 3, 33, ((64, 64), (32,), (32,)), 64, cap, prioritized_replay=True, frame_capacity=f),
            "DQN": lambda f: DQNLearner(E, 12, (64, 64), 32, cap, frame_capacity=f),
        }[algo]
        learners = {"default": make(None), "frames": make(fc)}
        for L in learners.values():
            fill(L, cap, E, 3 if algo == "BDQ" else 1, 33 if algo == "BDQ" else 12)
        t = {k: [] for k in learners}
        for _ in range(args.windows):
            for k, L in learners.items():           # alternated: drift of clocks and neighbours hits both arms
                t[k].append(ms_per_step(L, args.steps) * 1e3)
        info = learners["frames"].replay_info()
        row = {"algo": algo, "obs_dim": E, "slots": cap, "frame_capacity": fc, "evicted_early": info["evicted_early"],
               "bytes_default": learners["default"].replay_info()["bytes"], "bytes_frames": info["bytes"]}
        for k in t:
            v = np.array(t[k])
            row[f"{k}_us_median"], row[f"{k}_us_min"], row[f"{k}_us_max"] = float(np.median(v)), float(v.min()), float(v.max())
        row["frames_over_default"] = row["frames_us_median"] / row["default_us_median"]
        rows.append(row)
        print(json.dumps(row))
        for L in learners.values():
            L.close()
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"device": name, "power_limit": power, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
