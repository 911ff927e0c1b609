"""Times the actor side of ``SAC.learn`` with and without ``device_obs_norm`` on environments that cost nothing to step.

  python tools/actor_loop_bench.py [--n_envs 1 16 128] [--configs depth rgbd] [--seconds 2.0]

Both arms run ``SAC.learn`` itself (one gradient step per vectorised env step, batch 64, bf16x3) over a DummyVecEnv of
``n_envs`` environments that hand out pre-generated frames, wrapped in VecNormalize(norm_obs, norm_reward).  depth: (64, 64, 2);
rgbd: (64, 64, 5) with 8-bit RGB replay planes.  The two arms alternate in one process; after a warm-up each arm is timed
over windows of at least --seconds, every window ending in a synchronise of the learner's stream.  Printed per case:
env-steps/s of both arms, and for the default arm the host milliseconds per vectorised step that VecNormalize spends on
the float64 statistics and on normalising and that the loop spends in the calls that copy (Learner.set_norm_stats twice
and Learner.replay_add, which returns when its copies have landed), plus the bytes copied host->device per vectorised step
by each arm (Learner.upload_bytes).  The timers cost the default arm ten clock reads per step, well under a
microsecond against differences of 0.3 ms and more.  The card's name and power limit are read in the same run and printed
first.  Needs a GPU: there is no fallback.
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
from b200grasp.sac_model import SAC, CnnPolicy  # noqa: E402
from b200grasp.spaces import Box  # noqa: E402
from b200grasp.vec_env import DummyVecEnv, VecNormalize  # noqa: E402

CONFIGS = {"depth": ((64, 64, 2), ()), "rgbd": ((64, 64, 5), (0, 1, 2))}


class PoolEnv:
    """Hands out frames from a small pre-generated pool: stepping costs an index increment."""

    def __init__(self, shape, u8, seed, horizon=50, pool=8):
        self.observation_space = Box(0.0, 255.0, shape)
        self.action_space = Box(-1.0, 1.0, (5,), seed=seed)
        rng = np.random.default_rng(seed)
        self.pool = np.zeros((pool,) + shape, np.float32)
        self.pool[..., :-1] = rng.uniform(0, 255, (pool,) + shape[:2] + (shape[2] - 1,))
        for c in u8:
            self.pool[..., c] = np.rint(self.pool[..., c])
        self.pool[:, 0, 0, -1] = rng.uniform(0, 1, pool)
        self.horizon, self.t, self.k = horizon, 0, 0

    def _obs(self):
        self.k = (self.k + 1) % len(self.pool)
        return self.pool[self.k]

    def reset(self):
        self.t = 0
        return self._obs()

    def step(self, action):
        self.t += 1
        return self._obs(), 1.0, self.t >= self.horizon, {}


def card():
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("actor_loop_bench needs a GPU")
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


class Timed:
    """Accumulates the wall time of a bound method of the default arm."""

    def __init__(self, fn):
        self.fn, self.s = fn, 0.0

    def __call__(self, *a, **k):
        t0 = time.perf_counter()
        out = self.fn(*a, **k)
        self.s += time.perf_counter() - t0
        return out


def make(shape, u8, n_envs, device):
    venv = DummyVecEnv([(lambda i=i: PoolEnv(shape, u8, seed=i)) for i in range(n_envs)])
    env = VecNormalize(venv, norm_obs=True, norm_reward=True, clip_obs=10.0)
    cap = 20000
    return SAC(CnnPolicy, env, policy_kwargs={"cnn_extractor": "augmented_nature_cnn"}, buffer_size=cap, batch_size=64,
               learning_starts=64, seed=0, precision="bf16x3", replay_frames=cap + cap // 8 + n_envs, replay_u8_planes=u8,
               device_obs_norm=device)


def window(model, n_envs, seconds):
    """learn() in slices until `seconds` have passed, then drain the stream; returns (env steps, seconds)."""
    steps, t0 = 0, time.perf_counter()
    while time.perf_counter() - t0 < seconds:
        model.learn(n_envs * 20, reset_num_timesteps=False)
        steps += n_envs * 20
    model.learner.sync()
    return steps, time.perf_counter() - t0


def case(name, n_envs, seconds):
    shape, u8 = CONFIGS[name]
    arms = {"default": make(shape, u8, n_envs, False), "device_obs_norm": make(shape, u8, n_envs, True)}
    vn = arms["default"].get_vec_normalize_env()
    upd = Timed(vn.obs_rms.update)
    vn.obs_rms.update = upd
    nrm = vn.normalize_obs = Timed(vn.normalize_obs)
    L = arms["default"].learner
    cpy = [Timed(L.set_norm_stats), Timed(L.replay_add)]
    L.set_norm_stats, L.replay_add = cpy
    for m in arms.values():                      # warm-up: past learning_starts, graph captured, staging allocated
        window(m, n_envs, 0.5)
    upd.s = nrm.s = cpy[0].s = cpy[1].s = 0.0
    base = {k: m.learner.upload_bytes() for k, m in arms.items()}
    tot = {k: [0, 0.0] for k in arms}
    rates = {k: [] for k in arms}
    for _ in range(2):
        for k, m in arms.items():
            s, t = window(m, n_envs, seconds)
            tot[k][0] += s
            tot[k][1] += t
            rates[k].append(round(s / t, 1))
    out = {"config": name, "n_envs": n_envs}
    for k, m in arms.items():
        up = m.learner.upload_bytes()
        vsteps = tot[k][0] / n_envs
        out[k] = {"env_steps_per_s": round(tot[k][0] / tot[k][1], 1), "windows": rates[k],
                  "ms_per_vec_step": round(1e3 * tot[k][1] / vsteps, 3),
                  "h2d_bytes_per_vec_step": round((up["observe"] + up["other"] - base[k]["observe"] - base[k]["other"]) / vsteps)}
    vsteps = tot["default"][0] / n_envs
    out["default"]["host_ms_per_vec_step"] = {"statistics": round(1e3 * upd.s / vsteps, 3), "normalise": round(1e3 * nrm.s / vsteps, 3),
                                              "copies": round(1e3 * (cpy[0].s + cpy[1].s) / vsteps, 3)}
    out["speedup"] = round(out["device_obs_norm"]["env_steps_per_s"] / out["default"]["env_steps_per_s"], 3)
    for m in arms.values():
        m.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n_envs", type=int, nargs="+", default=[1, 16, 128])
    ap.add_argument("--configs", nargs="+", default=["depth", "rgbd"], choices=sorted(CONFIGS))
    ap.add_argument("--seconds", type=float, default=2.0)
    a = ap.parse_args()
    print(json.dumps(card()), flush=True)
    for name in a.configs:
        for n in a.n_envs:
            print(json.dumps(case(name, n, a.seconds)), flush=True)


if __name__ == "__main__":
    main()
