"""Gradient steps per second of SAC's CNN policy with stable-baselines' plain nature_cnn against the augmented extractor,
bf16x3 (engine v2), A = 3, head width 64, at batch 64 and 256:

  nature_cnn at (64, 64, 2)   the simplified environment's depth + pad observation
  augmented  at (64, 64, 2)   the same observation through create_augmented_nature_cnn(1) (conv1 over one plane)
  augmented  at (64, 64, 3)   the augmented net whose conv1 has nature_cnn's C = 2 shape

Each measurement is b2g_sac_step(n) (graph replays of the sampled step, timed by the host clock around a call that ends in a
device synchronise) over a replay of 2048 synthetic transitions, after a warm-up call.  The three learners of a batch size are
measured in turn, round after round, so that clock and neighbour drift fall on all of them alike; the median round is
reported.  One JSON line per (extractor, shape, batch), then the card's name and power limit read in the same run.

  python tools/sac_nature_cnn_bench.py [--steps 200] [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import b200grasp  # noqa: E402
from b200grasp import _lib, synth  # noqa: E402

VARIANTS = (("nature_cnn", (64, 64, 2)), ("augmented", (64, 64, 2)), ("augmented", (64, 64, 3)))
NS, A = 2048, 3


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def learner(extractor, shape, B):
    kw = {"extractor": extractor} if extractor != "augmented" else {}
    L = b200grasp.Learner(shape, n_act=A, batch_size=B, buffer_size=NS, target_entropy=-float(A), precision=_lib.B2G_PREC_BF16X3,
                          seed=3, **kw)
    rng = np.random.default_rng(7)
    params = {}
    for n, s in L.param_shapes.items():      # fresh parameters of the learner's own shapes (timing does not depend on values)
        params[n] = (rng.standard_normal(s) * (0.05 if n.endswith(("/w", "/kernel")) else 0.0)).astype(np.float32)
    L.load_parameters(params)
    mean = np.zeros(shape, np.float32)
    var = np.ones(shape, np.float32)
    mean[..., :-1], var[..., :-1] = 0.5, 0.04
    tr = synth.make_transitions(NS, mean, var, seed=11, n_act=A)
    L.set_norm_stats(mean, var, 1.0, 10.0, 10.0, 1e-8)
    L.replay_add(tr["obs"], tr["act"], tr["rew"], tr["next_obs"], tr["done"])
    return L


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    for B in (64, 256):
        Ls = [learner(e, s, B) for e, s in VARIANTS]
        for L in Ls:
            L.step(20, lr=3e-4)                  # graph capture, first launches
        rates = [[] for _ in Ls]
        for _ in range(a.rounds):
            for i, L in enumerate(Ls):
                t0 = time.perf_counter()
                L.step(a.steps, lr=3e-4)         # returns after the device synchronise that reads the metrics
                rates[i].append(a.steps / (time.perf_counter() - t0))
        for (e, s), L, r in zip(VARIANTS, Ls, rates):
            print(json.dumps({"extractor": e, "obs_shape": list(s), "A": A, "batch": B, "steps": a.steps, "rounds": a.rounds,
                              "grad_steps_per_s_median": round(float(np.median(r)), 1),
                              "grad_steps_per_s_min": round(float(np.min(r)), 1),
                              "grad_steps_per_s_max": round(float(np.max(r)), 1)}), flush=True)
            L.close()
    print(json.dumps({"gpu": card()}), flush=True)


if __name__ == "__main__":
    main()
