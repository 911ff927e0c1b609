"""Replay memory of the shipped SAC configurations, with two frames per replay slot and with a shared-frame budget.

    python tools/replay_budget.py            # the table (arithmetic, the same formula as b2g_replay_info)
    python tools/replay_budget.py --gpu      # plus, on the GPU: the RGB-D learner at 1M slots, 8-bit RGB, spare 1/8

The --gpu run creates the full_depth_obs.yaml learner (64x64x5 observations: RGB, depth, actuator plane) with
buffer_size = 1,000,000, fills it with an episodic stream through replay_add, runs gradient steps from the replay and prints
Learner.replay_info() with the steps per second, the card's name and its power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (run, config, zip data.buffer_size, observation shape, 8-bit planes when the observation holds RGB)
SHIPPED = [
    ("SAC_full_rgbd", "config/full_depth_obs.yaml", 1_000_000, (64, 64, 5), (0, 1, 2)),
    ("table_clearing/SAC_real_2m_buffer_128", "config/gripper_grasp.yaml", 2_000_000, (64, 64, 2), ()),
    ("SAC_depth_1mbuffer", "config/gripper_grasp.yaml", 1_000_000, (64, 64, 2), ()),
    ("SAC_10m_table", "config/gripper_grasp.yaml", 1_000_000, (64, 64, 2), ()),
]
N_ACT = 5
SPARE = 0.125


def frame_bytes(obs_shape, u8_planes=()):
    """Bytes of one replay frame (include/b200grasp.h: compact row, 8-bit planes first, 16-byte stride with 8-bit planes)."""
    if len(obs_shape) == 1:
        return 4 * obs_shape[0]
    h, w, c = obs_shape
    ci, n8 = c - 1, len(u8_planes)
    if n8 == 0:
        return 4 * (h * w * ci + 4)
    return (h * w * n8 + 4 * h * w * (ci - n8) + 16 + 15) // 16 * 16


def replay_bytes(cap, obs_shape, n_act=N_ACT, frame_capacity=None, u8_planes=()):
    """Device bytes of the replay: frames, two int32 frame indices, actions, reward and done per slot."""
    fc = 2 * cap if frame_capacity is None else frame_capacity
    return fc * frame_bytes(obs_shape, u8_planes) + cap * (2 * 4 + 4 * (n_act + 2))


def budget(cap, spare=SPARE, n_envs=1):
    """train_cli --replay_spare F: cap * (1 + F) + n_envs frames."""
    return int(cap * (1.0 + spare)) + n_envs


def table():
    rows = []
    for run, cfg, cap, obs, u8 in SHIPPED:
        rows.append({"run": run, "config": cfg, "buffer_size": cap, "obs": list(obs),
                     "two_frames_per_slot_GB": round(replay_bytes(cap, obs) / 1e9, 2),
                     "shared_frames_GB": round(replay_bytes(cap, obs, frame_capacity=budget(cap), u8_planes=u8) / 1e9, 2),
                     "u8_planes": list(u8)})
    return rows


def _card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return name, out


def episodic_fill(L, n_transitions, lanes, rng, p_done=0.05):
    """An episodic stream: next_obs(t) == obs(t+1) of the same lane except after done.  Frames come from a small pool of
    distinct observations (integer RGB, float depth, constant actuator plane), so the host does not generate gigabytes."""
    h, w, c = L.obs_shape
    pool = rng.integers(0, 256, size=(97, h, w, c)).astype(np.float32)
    pool[..., 3] = rng.random((97, h, w), dtype=np.float32)
    pool[..., -1] = rng.random((97, 1, 1), dtype=np.float32)
    k = 0
    cur = np.stack([pool[(k := k + 1) % 97] for _ in range(lanes)])
    added = 0
    while added < n_transitions:
        nxt = np.stack([pool[(k := k + 1) % 97] for _ in range(lanes)])
        done = (rng.random(lanes) < p_done).astype(np.float32)
        act = rng.uniform(-1, 1, (lanes, N_ACT)).astype(np.float32)
        L.replay_add(cur, act, rng.standard_normal(lanes).astype(np.float32), nxt, done)
        cur = nxt.copy()
        for i in np.nonzero(done)[0]:
            cur[i] = pool[(k := k + 1) % 97]
        added += lanes


def gpu_run(fill, steps, lanes):
    sys.path.insert(0, ROOT)
    import b200grasp
    name, power = _card()
    cap, obs, u8 = 1_000_000, (64, 64, 5), (0, 1, 2)
    out = []
    for B in (64, 1024):
        L = b200grasp.Learner(obs, n_act=N_ACT, batch_size=B, buffer_size=cap, seed=7, precision=b200grasp._lib.B2G_PREC_BF16X3,
                              frame_capacity=budget(cap, n_envs=lanes), u8_planes=u8)
        rng = np.random.default_rng(B)
        t0 = time.perf_counter()
        episodic_fill(L, fill, lanes, rng)
        t_fill = time.perf_counter() - t0
        L.step(10)
        L.sync()
        t0 = time.perf_counter()
        L.step(steps)
        L.sync()
        dt = time.perf_counter() - t0
        info = L.replay_info()
        out.append({"batch": B, "replay_info": info, "replay_GB": round(info["bytes"] / 1e9, 2),
                    "expected_GB": round(replay_bytes(cap, obs, frame_capacity=budget(cap, n_envs=lanes), u8_planes=u8) / 1e9, 2),
                    "fill_transitions": fill, "fill_s": round(t_fill, 2), "steps": steps, "steps_per_s": round(steps / dt, 1),
                    "gpu": name, "power_limit": power})
        L.close()
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--gpu", action="store_true", help="create, fill and step the 1M-slot RGB-D learner on cuda:0")
    ap.add_argument("--fill", type=int, default=200_000)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--lanes", type=int, default=64)
    a = ap.parse_args(argv)
    for r in table():
        print(json.dumps(r))
    if a.gpu:
        for r in gpu_run(a.fill, a.steps, a.lanes):
            print(json.dumps(r))


if __name__ == "__main__":
    main()
