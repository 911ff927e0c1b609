"""Cost of TensorBoard logging (tensorboard_log) on the SAC hot path.

  python tools/tb_log_bench.py [--batches 64 256] [--n_envs 1 16] [--steps 2000] [--learn_steps 1600] [--reps 3]

1. Gradient steps/s of the replayed SAC step (depth CNN, bf16x3) with and without the metrics-ring node, at each batch size:
   two learners over the same replay, one with ``metrics_log(8192)``; each window enqueues --steps steps with
   ``step_async`` and ends in a synchronise (the log arm also drains its ring, as learn does at half full).
2. ``SAC.learn`` env-steps/s on environments that cost nothing to step (tools/actor_loop_bench.py's PoolEnv and model) with
   and without ``tensorboard_log``, at each env count; one learn call of --learn_steps vectorised steps per window, so the
   log arm pays its ring enable, drains, event writes and file close inside the window.

The arms alternate in one process, --reps windows each after a warm-up; printed per case: the median rate of each arm and
the relative cost.  The card's name and power limit are read in the same run and printed first.  Needs a GPU.
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import b200grasp  # noqa: E402,F401
from actor_loop_bench import card, make  # noqa: E402

def step_case(B, steps, reps):
    from tests.util import load_case, make_batch, make_learner
    cfg, params, vn = load_case("sac_depth")
    arms = {}
    for name in ("plain", "ring"):
        L = make_learner(cfg, vn, B, params, buffer_size=4096, precision=1)
        raw, _, _ = make_batch(vn, 1024)
        L.replay_add(raw["obs"], raw["act"], raw["rew"], raw["next_obs"], raw["done"])
        if name == "ring":
            L.metrics_log(8192)
        arms[name] = L

    def window(name):
        L = arms[name]
        t0 = time.perf_counter()
        for k in range(0, steps, 1000):
            L.step_async(min(1000, steps - k), 3e-4)
            if name == "ring":
                L.metrics_drain()          # synchronises, as learn's drain at half full does
        L.sync()
        return steps / (time.perf_counter() - t0)

    for name in arms:
        window(name)
    rates = {k: [] for k in arms}
    for _ in range(reps):
        for name in arms:
            rates[name].append(window(name))
    for L in arms.values():
        L.close()
    return {k: statistics.median(v) for k, v in rates.items()}

def learn_case(n_envs, learn_steps, reps, logdir):
    arms = {"plain": make((64, 64, 2), (), n_envs, False), "tensorboard": make((64, 64, 2), (), n_envs, False)}
    arms["tensorboard"].tensorboard_log = logdir

    def window(m):
        t0 = time.perf_counter()
        m.learn(n_envs * learn_steps, reset_num_timesteps=False)
        m.learner.sync()
        return n_envs * learn_steps / (time.perf_counter() - t0)

    for m in arms.values():                       # warm-up: past learning_starts, graphs captured
        window(m)
    rates = {k: [] for k in arms}
    for _ in range(reps):
        for k, m in arms.items():
            rates[k].append(window(m))
    for m in arms.values():
        m.close()
    return {k: statistics.median(v) for k, v in rates.items()}

def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--n_envs", type=int, nargs="+", default=[1, 16])
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--learn_steps", type=int, default=1600)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    print(json.dumps(card()))
    for B in a.batches:
        r = step_case(B, a.steps, a.reps)
        print(json.dumps({"case": "replayed_step", "batch": B, "steps_per_s": {k: round(v, 1) for k, v in r.items()},
                          "ring_cost_pct": round(100 * (r["plain"] / r["ring"] - 1), 2)}))
    with tempfile.TemporaryDirectory() as d:
        for n in a.n_envs:
            r = learn_case(n, max(a.learn_steps // n, 200), a.reps, d)
            print(json.dumps({"case": "sac_learn", "n_envs": n, "env_steps_per_s": {k: round(v, 1) for k, v in r.items()},
                              "tensorboard_cost_pct": round(100 * (r["plain"] / r["tensorboard"] - 1), 2)}))

if __name__ == "__main__":
    main()
