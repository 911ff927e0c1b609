"""Auto-encoder training throughput (csrc/autoencoder.cu) at the shipped geometry: 16,200 seeded synthetic depth scenes,
batch 128, epochs over the device-resident dataset.  Prints one JSON line with images/s, ms per epoch and achieved fp32
FLOP/s from the algorithmic count (261.7 MFLOP per image forward + backward: 44.15 M MAC forward, 42.55 M input gradient,
44.15 M weight gradient), plus the card name and power limit of the run.

    python tools/ae_train_bench.py [--epochs 3] [--n 16200] [--batch 128]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--n", type=int, default=16200)
    ap.add_argument("--batch", type=int, default=128)
    a = ap.parse_args()
    x = synth.make_depth_scenes(a.n, seed=1234)
    ae = SimpleAutoEncoder(SHIPPED, max_batch=1, seed=0)
    ae.set_model_weights(glorot_init(model_shapes(SHIPPED["network"], 100), np.random.default_rng(0)))
    h = ae._autoencoder(a.batch)
    lib = _lib.load()
    fp = C.POINTER(C.c_float)
    _lib.check(lib.b2g_autoencoder_set_dataset(h, x.ctypes.data_as(fp), None, a.n))
    rng = np.random.default_rng(0)
    loss = C.c_double()

    def epoch():
        order = rng.permutation(a.n).astype(np.int32)
        t0 = time.perf_counter()
        _lib.check(lib.b2g_autoencoder_train_epoch(h, order.ctypes.data_as(C.POINTER(C.c_int32)), a.n, a.batch, 2e-4, C.byref(loss)))
        return time.perf_counter() - t0          # train_epoch ends in a stream synchronise

    epoch()                                       # graph capture and first-touch
    times = [epoch() for _ in range(a.epochs)]
    best = min(times)
    name, power = card()
    print(json.dumps({"metric": "ae_train", "images_per_s": a.n / best, "ms_per_epoch": 1e3 * best,
                      "ms_per_epoch_all": [round(1e3 * t, 2) for t in times], "tflops_fp32": a.n * FLOP_PER_IMAGE / best / 1e12,
                      "batch": a.batch, "n": a.n, "last_loss": loss.value, "gpu": name, "power_limit": power}))
    ae.close()


if __name__ == "__main__":
    main()
