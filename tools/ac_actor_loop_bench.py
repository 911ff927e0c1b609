"""Times ``PPO2.learn`` and ``TRPO.learn`` with and without ``device_obs_norm`` on environments that cost nothing to step.

  python tools/ac_actor_loop_bench.py [--cases ...] [--seconds 2.0]

Both arms run ``learn`` itself (MlpPolicy [64, 64]; PPO2 with n_steps 128, 4 minibatches, 4 epochs; TRPO with
timesteps_per_batch 1024, 10 CG iterations, 3 value passes) over a DummyVecEnv of ``n_envs`` environments that hand out
pre-generated frames, wrapped in VecNormalize(norm_obs, norm_reward).  Cases (algo, observation, n_envs):
  ppo flat100 / depth8192 at 1, 16 and 128 envs: 100-float rows, and the 64x64x2 depth frame flattened to 8192 floats (the
      PPO branch's MlpPolicy on config/gripper_grasp.yaml);
  ppo encoded at 16 and 128 envs: raw [64*64 depth | actuator] rows under VecEncodeDepth (the shipped encoder, 100 + 1
      floats): the default arm encodes in the wrapper (host mode), the device arm passes the raw rows to the learner;
  trpo flat100 / depth8192 at 1 env.
The two arms alternate in one process; after a warm-up (one full rollout and update) each arm is timed over windows of
whole updates lasting at least --seconds, so every window ends in the update's metric read, a synchronise of the learner's
stream.  Printed per case: env-steps/s of every window and overall, and the host->device bytes per vectorised step of the
observation path: the device arm's counted observe uploads (b2g_*_upload_bytes), and for the default arm what
rollout_act uploads (n_envs x obs_dim x 4) plus, with the encoder, the raw rows the wrapper's encode call uploads.  The
card's name and power limit are read in the same run and printed first.  Needs a GPU: there is no fallback.
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
from b200grasp import synth  # noqa: E402
from b200grasp.encoders import SimpleAutoEncoder, keras_encoder_arrays  # noqa: E402
from b200grasp.ppo2 import PPO2  # noqa: E402
from b200grasp.spaces import Box  # noqa: E402
from b200grasp.trpo_mpi import TRPO  # noqa: E402
from b200grasp.vec_env import DummyVecEnv, VecEncodeDepth, VecNormalize  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
PIXELS = 64 * 64
DIMS = {"flat100": 100, "depth8192": 8192, "encoded": PIXELS + 1}
CASES = [("ppo", o, n) for o in ("flat100", "depth8192") for n in (1, 16, 128)] + [("ppo", "encoded", n) for n in (16, 128)] + \
        [("trpo", o, 1) for o in ("flat100", "depth8192")]


class PoolEnv:
    """Hands out rows from a small pre-generated pool: stepping costs an index increment."""

    def __init__(self, width, seed, horizon=50, pool=8):
        rng = np.random.default_rng(seed)
        if width == DIMS["encoded"]:
            self.pool = np.concatenate([synth.make_depth_scenes(pool, seed=seed).reshape(pool, PIXELS), rng.uniform(0, 1, (pool, 1))],
                                       axis=1).astype(np.float32)
            self.observation_space = Box(np.zeros(width), np.concatenate([np.full(PIXELS, np.inf), [1.0]]), (width,))
        else:
            self.pool = rng.uniform(0, 2, (pool, width)).astype(np.float32)
            self.observation_space = Box(-np.inf, np.inf, (width,))
        self.action_space = Box(-1.0, 1.0, (5,), seed=seed)
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
        raise SystemExit("ac_actor_loop_bench needs a GPU")
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def make_encoder(max_batch):
    w = dict(np.load(os.path.join(GOLD, "encoder_weights.npz")))
    w = {k.replace("__", "/"): v for k, v in w.items()}
    cfg = json.load(open(os.path.join(GOLD, "encoder_config.json")))
    enc = SimpleAutoEncoder(cfg, max_batch=max_batch)
    enc.set_weights(keras_encoder_arrays(w, len(cfg["network"])))
    return enc


def make(algo, obs, n_envs, device):
    venv = DummyVecEnv([(lambda i=i: PoolEnv(DIMS[obs], seed=i)) for i in range(n_envs)])
    if obs == "encoded":
        venv = VecEncodeDepth(venv, make_encoder(max(n_envs, 16)))
    env = VecNormalize(venv, norm_obs=True, norm_reward=True, clip_obs=10.0)
    if algo == "ppo":
        return PPO2("MlpPolicy", env, seed=0, device_obs_norm=device)
    return TRPO("MlpPolicy", env, seed=0, device_obs_norm=device)


def window(model, batch, seconds):
    """learn() one update at a time until `seconds` have passed; returns (env steps, seconds)."""
    steps, t0 = 0, time.perf_counter()
    while time.perf_counter() - t0 < seconds:
        model.learn(batch, reset_num_timesteps=False)
        steps += batch
    return steps, time.perf_counter() - t0


def case(algo, obs, n_envs, seconds):
    arms = {"default": make(algo, obs, n_envs, False), "device_obs_norm": make(algo, obs, n_envs, True)}
    batch = n_envs * 128 if algo == "ppo" else 1024
    for m in arms.values():                      # warm-up: one rollout and update (graph captured, staging allocated)
        m.learn(batch, reset_num_timesteps=False)
    base = {k: m.learner.upload_bytes()["observe"] if k != "default" else 0 for k, m in arms.items()}
    tot = {k: [0, 0.0] for k in arms}
    rates = {k: [] for k in arms}
    for _ in range(3):
        for k, m in arms.items():
            s, t = window(m, batch, seconds)
            tot[k][0] += s
            tot[k][1] += t
            rates[k].append(round(s / t, 1))
    out = {"algo": algo, "obs": obs, "n_envs": n_envs}
    D = 101 if obs == "encoded" else DIMS[obs]
    for k, m in arms.items():
        vsteps = tot[k][0] / n_envs
        if k == "default":       # rollout_act's row upload, and the raw rows the wrapper's encode call uploads
            h2d = n_envs * D * 4 + (n_envs * DIMS[obs] * 4 if obs == "encoded" else 0)
        else:
            h2d = round((m.learner.upload_bytes()["observe"] - base[k]) / vsteps)
        out[k] = {"env_steps_per_s": round(tot[k][0] / tot[k][1], 1), "windows": rates[k],
                  "ms_per_vec_step": round(1e3 * tot[k][1] / vsteps, 3), "obs_h2d_bytes_per_vec_step": h2d}
    out["speedup"] = round(out["device_obs_norm"]["env_steps_per_s"] / out["default"]["env_steps_per_s"], 3)
    for m in arms.values():
        m.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", nargs="+", default=[f"{a}:{o}:{n}" for a, o, n in CASES], help="algo:obs:n_envs")
    ap.add_argument("--seconds", type=float, default=2.0)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    a = ap.parse_args()
    lines = [json.dumps(card())]
    print(lines[-1], flush=True)
    for c in a.cases:
        algo, obs, n = c.split(":")
        lines.append(json.dumps(case(algo, obs, int(n), a.seconds)))
        print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
