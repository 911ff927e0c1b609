"""Times the perception encoder in both precisions: fp32 on the CUDA cores and bf16x3 on the wgmma engine.

  python tools/encoder_tc_bench.py [--batches 1 16 128 256 512] [--n_envs 16 128] [--seconds 2.0] [--out FILE]
                                   [--profile DIR]

Part 1, ``encode()``: ``SimpleAutoEncoder(precision=p).encode(n)`` on the shipped weights (tests/golden) at every batch n, the
last one being max_batch.  Every shape is warmed up first; then the two precisions alternate, each timed over windows of at
least --seconds with a host clock.  ``encode`` ends in a synchronise of the encoder's stream, so a window times finished work
(upload, encode, download).
Part 2, the pass-raw ``SAC.learn`` loop of tools/encoded_actor_loop_bench.py (MLP policy, batch 64, free environments,
device_obs_norm=True, VecEncodeDepth in pass-raw mode) at each --n_envs, the encoder in either precision, alternated.
--profile DIR writes a torch.profiler kernel table of one encode(256) per precision (a separate run from the timed windows).
The card's name and power limit are read in the same run and printed first.  Needs a GPU.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

TOOLS = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(TOOLS))
sys.path.insert(0, TOOLS)
import b200grasp  # noqa: E402,F401
from b200grasp import synth  # noqa: E402
from b200grasp.encoders import SimpleAutoEncoder, keras_encoder_arrays  # noqa: E402
from b200grasp.sac_model import SAC, MlpPolicy  # noqa: E402
from b200grasp.vec_env import DummyVecEnv, VecEncodeDepth, VecNormalize, unwrap_encode_depth  # noqa: E402
from encoded_actor_loop_bench import GOLD, RawEnv  # noqa: E402

PRECISIONS = ("fp32", "bf16x3")


def make_encoder(max_batch, precision):
    w = {k.replace("__", "/"): v for k, v in np.load(os.path.join(GOLD, "encoder_weights.npz")).items()}
    cfg = json.load(open(os.path.join(GOLD, "encoder_config.json")))
    enc = SimpleAutoEncoder(cfg, max_batch=max_batch, precision=precision)
    enc.set_weights(keras_encoder_arrays(w, len(cfg["network"])))
    return enc, cfg


def macs_per_frame(cfg, hw=64, c=1):
    """Multiply-adds of one frame's forward (the convs' 'same' outputs, then the dense layer)."""
    total = 0
    for l in cfg["network"]:
        hw = -(-hw // l["strides"])
        total += hw * hw * l["filters"] * l["kernel_size"] ** 2 * c
        c = l["filters"]
    return total + hw * hw * c * cfg["encoding_dim"]


def window(fn, seconds):
    t0, calls = time.perf_counter(), 0
    while True:
        fn()
        calls += 1
        dt = time.perf_counter() - t0
        if dt >= seconds:
            return dt / calls


def bench_encode(a, card):
    N = max(a.batches)
    encs = {p: make_encoder(N, p)[0] for p in PRECISIONS}
    cfg = make_encoder(1, "fp32")[1]
    macs = macs_per_frame(cfg)
    imgs = synth.make_depth_scenes(N, seed=0).astype(np.float32)
    for p in PRECISIONS:                                   # warm-up of every shape
        for n in a.batches:
            for _ in range(3):
                encs[p].encode(imgs[:n])
    rows = []
    for n in a.batches:
        t = {p: [] for p in PRECISIONS}
        for _ in range(a.rounds):
            for p in PRECISIONS:
                t[p].append(window(lambda: encs[p].encode(imgs[:n]), a.seconds))
        row = {"part": "encode", "n": n, "card": card}
        for p in PRECISIONS:
            med = float(np.median(t[p]))
            row[f"{p}_us_per_call"] = round(med * 1e6, 1)
            row[f"{p}_spread_us"] = [round(min(t[p]) * 1e6, 1), round(max(t[p]) * 1e6, 1)]
            row[f"{p}_gmac_per_s"] = round(n * macs / med / 1e9, 1)       # whole call (upload + encode + download)
        row["bf16x3_speedup"] = round(row["fp32_us_per_call"] / row["bf16x3_us_per_call"], 3)
        print(json.dumps(row), flush=True)
        rows.append(row)
    if a.profile:
        import torch
        from torch.profiler import ProfilerActivity, profile
        os.makedirs(a.profile, exist_ok=True)
        for p in PRECISIONS:
            n = min(256, N)
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                for _ in range(20):
                    encs[p].encode(imgs[:n])
                torch.cuda.synchronize()
            table = prof.key_averages().table(sort_by="cuda_time_total", row_limit=25)
            with open(os.path.join(a.profile, f"encode_{p}_n{n}.txt"), "w") as f:
                f.write(f"{card}\n20 x encode({n}), precision {p}\n{table}\n")
            print(f"profile {p}:\n{table}", flush=True)
    for e in encs.values():
        e.close()
    return rows


def build_loop(n, precision):
    enc, _ = make_encoder(2 * n, precision)
    venv = VecEncodeDepth(DummyVecEnv([(lambda i=i: RawEnv(i)) for i in range(n)]), enc)
    env = VecNormalize(venv, norm_obs=True, norm_reward=True)
    model = SAC(MlpPolicy, env, batch_size=64, buffer_size=100000, learning_starts=64, seed=0, device_obs_norm=True)
    assert unwrap_encode_depth(env).pass_raw
    return model, enc


def bench_loop(a, card):
    rows = []
    for n in a.n_envs:
        built = {p: build_loop(n, p) for p in PRECISIONS}
        for p in PRECISIONS:
            built[p][0].learn(max(8 * n, 256))
        rates = {p: [] for p in PRECISIONS}
        for _ in range(a.rounds):
            for p in PRECISIONS:
                model = built[p][0]
                steps = max(64 * n, 512)
                t0, done = time.perf_counter(), 0
                while True:
                    model.learn(steps)
                    done += steps
                    if time.perf_counter() - t0 >= a.seconds:
                        break
                rates[p].append(done / (time.perf_counter() - t0))
        row = {"part": "sac_learn_pass_raw", "n_envs": n, "card": card,
               **{f"{p}_steps_per_s": round(float(np.median(rates[p]))) for p in PRECISIONS},
               "spread": {p: [round(min(rates[p])), round(max(rates[p]))] for p in PRECISIONS}}
        row["bf16x3_speedup"] = round(row["bf16x3_steps_per_s"] / row["fp32_steps_per_s"], 3)
        print(json.dumps(row), flush=True)
        rows.append(row)
        for model, enc in built.values():
            model.close()
            enc.close()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 16, 128, 256, 512])
    ap.add_argument("--n_envs", type=int, nargs="+", default=[16, 128])
    ap.add_argument("--seconds", type=float, default=2.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": card}), flush=True)
    results = bench_encode(a, card) + (bench_loop(a, card) if a.n_envs else [])
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
