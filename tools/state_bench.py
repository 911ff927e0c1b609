"""Times Learner.save_state / load_state (b2g_sac_state_save / _load) on full replays and reports GB/s.

  python tools/state_bench.py [--slots 1000000] [--dir /path/on/the/disk/to/measure] [--configs depth rgbd]

depth: (64, 64, 2), frame budget slots * 1.125 + 1 (train_cli --replay_spare 0.125); rgbd: (64, 64, 5) with 8-bit RGB planes and
the same budget.  The replay is filled with episodes of 9 steps, so the frame pool is full and the live window is what a long
run leaves.  The file goes to --dir (default: the system temporary directory) and is deleted afterwards; the disk, its free
space and the page-cache caveat (a load right after a save may read from RAM) are printed with the result.
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import b200grasp  # noqa: E402

CONFIGS = {"depth": ((64, 64, 2), ()), "rgbd": ((64, 64, 5), (0, 1, 2))}


def fill(L, shape, u8, slots, lanes=256, horizon=9, blocks=8):
    """slots rows from `lanes` parallel episodes of `horizon` steps: within an episode next_obs(t) == obs(t + 1), so the
    replay shares those frames as it does for the learn loop; the observations cycle through a few random blocks."""
    rng = np.random.default_rng(0)
    pool = rng.random((blocks, lanes) + shape, dtype=np.float32)
    if u8:
        pool[..., list(u8)] = np.floor(pool[..., list(u8)] * 255)
    act = rng.uniform(-1, 1, (lanes, 5)).astype(np.float32)
    rew = rng.standard_normal(lanes).astype(np.float32)
    cur = pool[0]
    for c in range((slots + lanes - 1) // lanes + 1):
        nx = pool[(c + 1) % blocks]
        end = c % horizon == horizon - 1
        L.replay_add(cur, act, rew, nx, np.full(lanes, float(end), np.float32))
        cur = pool[(c + blocks // 2) % blocks] if end else nx


def run(name, slots, directory):
    shape, u8 = CONFIGS[name]
    L = b200grasp.Learner(shape, n_act=5, hidden=64, batch_size=256, buffer_size=slots, precision=1,
                          frame_capacity=int(slots * 1.125) + 1, u8_planes=u8)
    t0 = time.perf_counter()
    fill(L, shape, u8, slots)
    t_fill = time.perf_counter() - t0
    L.step(1)
    path = os.path.join(directory, f"state_bench_{name}.state")
    try:
        t0 = time.perf_counter()
        L.save_state(path)
        t_save = time.perf_counter() - t0
        size = os.path.getsize(path)
        R = b200grasp.Learner(shape, n_act=5, hidden=64, batch_size=256, buffer_size=slots, precision=1,
                              frame_capacity=int(slots * 1.125) + 1, u8_planes=u8)
        t0 = time.perf_counter()
        R.load_state(path)
        t_load = time.perf_counter() - t0
        assert R.replay_info() == L.replay_info()
        R.close()
    finally:
        if os.path.exists(path):
            os.remove(path)
    info = L.replay_info()
    L.close()
    return {"config": name, "slots": slots, "replay_bytes": info["bytes"], "live_frames": info["live_frames"], "file_bytes": size,
            "fill_s": round(t_fill, 1), "save_s": round(t_save, 3), "load_s": round(t_load, 3),
            "save_GBps": round(size / t_save / 1e9, 2), "load_GBps": round(size / t_load / 1e9, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, default=1_000_000)
    ap.add_argument("--dir", default=tempfile.gettempdir())
    ap.add_argument("--configs", nargs="+", default=["depth", "rgbd"], choices=sorted(CONFIGS))
    a = ap.parse_args()
    du = shutil.disk_usage(a.dir)
    dev = os.stat(a.dir).st_dev
    print(json.dumps({"dir": os.path.abspath(a.dir), "free_GB": round(du.free / 1e9, 1), "st_dev": dev,
                      "note": "load follows save directly: the file may still be in the page cache"}))
    for name in a.configs:
        print(json.dumps(run(name, a.slots, a.dir)), flush=True)


if __name__ == "__main__":
    main()
