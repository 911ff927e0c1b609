"""Auto-encoder training throughput (csrc/autoencoder.cu) at the shipped geometry: 16,200 seeded synthetic depth scenes,
batch 128, epochs over the device-resident dataset.  Prints one JSON line with images/s, ms per epoch and achieved fp32
FLOP/s from the algorithmic count (261.7 MFLOP per image forward + backward: 44.15 M MAC forward, 42.55 M input gradient,
44.15 M weight gradient), plus the card name and power limit of the run.

    python tools/ae_train_bench.py [--epochs 3] [--n 16200] [--batch 128] [--train_precision {fp32,bf16x3,both}]
                                   [--profile DIR]

--train_precision both builds one handle per precision from the same initial weights and dataset, warms both (the first
epoch captures the full-batch and the partial-batch graph), then alternates their timed epochs and adds the bf16x3 / fp32
speed-up.  --profile DIR then runs one more epoch of each under torch.profiler (CUDA activity) and writes the per-kernel
device times to DIR/ae_kernels.json.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import b200grasp  # noqa: E402,F401
from b200grasp import _lib, synth  # noqa: E402
from b200grasp.encoders import SimpleAutoEncoder, glorot_init, model_shapes  # noqa: E402

FLOP_PER_IMAGE = 2 * 130.86e6
SHIPPED = {"network": [{"filters": 32, "kernel_size": 7, "strides": 2}, {"filters": 32, "kernel_size": 5, "strides": 2},
                       {"filters": 32, "kernel_size": 3, "strides": 2}], "encoding_dim": 100, "alpha": 0.1,
           "learning_rate": 2e-4, "batch_size": 128}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [v.strip() for v in out.split(",")[:2]]
        return name, power
    except Exception:
        return "unknown", "unknown"


class Arm:
    """One training handle at one precision over the device-resident dataset x."""

    def __init__(self, precision, x, batch):
        self.precision, self.n, self.batch = precision, x.shape[0], batch
        self.ae = SimpleAutoEncoder(SHIPPED, max_batch=1, seed=0, train_precision=precision)
        self.ae.set_model_weights(glorot_init(model_shapes(SHIPPED["network"], 100), np.random.default_rng(0)))
        self.h = self.ae._autoencoder(batch)
        self.lib = _lib.load()
        _lib.check(self.lib.b2g_autoencoder_set_dataset(self.h, x.ctypes.data_as(C.POINTER(C.c_float)), None, self.n))
        self.rng = np.random.default_rng(0)
        self.loss = C.c_double()
        self.times = []

    def epoch(self):
        order = self.rng.permutation(self.n).astype(np.int32)
        t0 = time.perf_counter()
        _lib.check(self.lib.b2g_autoencoder_train_epoch(self.h, order.ctypes.data_as(C.POINTER(C.c_int32)), self.n, self.batch, 2e-4,
                                                        C.byref(self.loss)))
        return time.perf_counter() - t0          # train_epoch ends in a stream synchronise

    def result(self):
        best = min(self.times)
        return {"train_precision": self.precision, "images_per_s": self.n / best, "ms_per_epoch": 1e3 * best,
                "ms_per_epoch_median": 1e3 * float(np.median(self.times)),
                "ms_per_epoch_all": [round(1e3 * t, 2) for t in self.times], "tflops_fp32": self.n * FLOP_PER_IMAGE / best / 1e12,
                "last_loss": self.loss.value}


def profile(arms, out_dir):
    """One epoch per arm under torch.profiler: device time per kernel name (ms), per arm."""
    import torch
    from torch.profiler import ProfilerActivity, profile as tprof
    out = {}
    for arm in arms:
        torch.cuda.synchronize()
        with tprof(activities=[ProfilerActivity.CUDA]) as prof:
            arm.epoch()
            torch.cuda.synchronize()
        rows = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None)
            if t is None:
                t = e.cuda_time_total
            if t > 0:
                rows[e.key] = {"ms": round(t / 1e3, 3), "calls": e.count}
        out[arm.precision] = {"kernel_ms_total": round(sum(r["ms"] for r in rows.values()), 3),
                              "kernels": dict(sorted(rows.items(), key=lambda kv: -kv[1]["ms"]))}
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "ae_kernels.json"), "w") as f:
        json.dump(out, f, indent=1)
    return {p: v["kernel_ms_total"] for p, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--n", type=int, default=16200)
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--train_precision", choices=["fp32", "bf16x3", "both"], default="fp32")
    ap.add_argument("--profile", type=str, default=None, help="directory for a torch.profiler kernel-time table")
    a = ap.parse_args()
    x = synth.make_depth_scenes(a.n, seed=1234)
    arms = [Arm(p, x, a.batch) for p in (["fp32", "bf16x3"] if a.train_precision == "both" else [a.train_precision])]
    for arm in arms:
        arm.epoch()                               # graph capture of both batch shapes and first-touch
    for _ in range(a.epochs):                     # alternated: both arms see the same machine state
        for arm in arms:
            arm.times.append(arm.epoch())
    name, power = card()
    res = {"metric": "ae_train", "batch": a.batch, "n": a.n, "gpu": name, "power_limit": power}
    if len(arms) == 1:
        res.update(arms[0].result())
    else:
        res["arms"] = [arm.result() for arm in arms]
        res["speedup_bf16x3"] = res["arms"][0]["ms_per_epoch"] / res["arms"][1]["ms_per_epoch"]
    if a.profile:
        res["kernel_ms_per_epoch"] = profile(arms, a.profile)
    print(json.dumps(res))
    for arm in arms:
        arm.ae.close()


if __name__ == "__main__":
    main()
