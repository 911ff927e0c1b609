"""Times ``DQN.learn`` with and without ``device_obs_norm`` on environments that cost nothing to step.

  python tools/dqn_actor_loop_bench.py [--configs flat100 depth] [--seconds 2.0]

Both arms run ``DQN.learn`` itself (one environment, as stable-baselines' DQN requires; prioritised replay, one gradient step
per env step, batch 32, 12 actions, layers [64, 64]: the shipped DQN_simple_4pads.zip) over a DummyVecEnv whose env hands out
pre-generated frames, wrapped in VecNormalize(norm_obs, norm_reward).
  flat100: 100-d observations (what the shipped zip observes).
  depth:   raw 64x64 depth rows + 1 tail float under a VecEncodeDepth holding the encoder of tests/golden (encoding_dim 100).
           The default arm encodes in the wrapper (one encode call, download, upload per step); the device arm hands the
           encoder to the learner, which encodes the raw rows it uploads.
The two arms alternate in one process; after a warm-up each arm is timed over windows of at least --seconds.  Printed per
case: env-steps/s of every window and overall, and the bytes copied host->device per env step (DQNLearner.upload_bytes;
the wrapper's own encode uploads are not counted there).  The card's name and power limit are read in the same run and
printed first.  Needs a GPU: there is no fallback.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from b200grasp.deepq import DQN  # noqa: E402
from b200grasp.encoders import SimpleAutoEncoder, keras_encoder_arrays  # noqa: E402
from b200grasp.spaces import Box, Discrete  # noqa: E402
from b200grasp.vec_env import DummyVecEnv, VecEncodeDepth, VecNormalize  # noqa: E402

CONFIGS = {"flat100": 100, "depth": 64 * 64 + 1}


class PoolEnv:
    """Hands out frames from a small pre-generated pool: stepping costs an index increment."""

    def __init__(self, width, seed, horizon=50, pool=8):
        self.observation_space = Box(-np.inf, np.inf, (width,))
        self.action_space = Discrete(12)
        rng = np.random.default_rng(seed)
        self.pool = rng.uniform(0, 2, (pool, width)).astype(np.float32)
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
        raise SystemExit("dqn_actor_loop_bench needs a GPU")
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def encoder():
    gold = os.path.join(ROOT, "tests", "golden")
    w = {k.replace("__", "/"): v for k, v in np.load(os.path.join(gold, "encoder_weights.npz")).items()}
    cfg = json.load(open(os.path.join(gold, "encoder_config.json")))
    enc = SimpleAutoEncoder(cfg, max_batch=512)
    enc.set_weights(keras_encoder_arrays(w, len(cfg["network"])))
    return enc


def make(name, device):
    venv = DummyVecEnv([lambda: PoolEnv(CONFIGS[name], seed=0)])
    if name == "depth":
        venv = VecEncodeDepth(venv, encoder(), tail=1)
    env = VecNormalize(venv, norm_obs=True, norm_reward=True, clip_obs=10.0)
    return DQN("MlpPolicy", env, buffer_size=20000, batch_size=32, learning_starts=64, prioritized_replay=True,
               policy_kwargs={"layers": [64, 64]}, seed=0, device_obs_norm=device)


def window(model, seconds):
    """learn() in slices until `seconds` have passed (every gradient step returns its metrics: the stream is drained);
    returns (env steps, seconds)."""
    steps, t0 = 0, time.perf_counter()
    while time.perf_counter() - t0 < seconds:
        model.learn(50, reset_num_timesteps=False)
        steps += 50
    return steps, time.perf_counter() - t0


def case(name, seconds):
    arms = {"default": make(name, False), "device_obs_norm": make(name, True)}
    for m in arms.values():                      # warm-up: past learning_starts, graph captured, staging allocated
        window(m, 0.5)
    base = {k: m.learner.upload_bytes() for k, m in arms.items()}
    tot = {k: [0, 0.0] for k in arms}
    rates = {k: [] for k in arms}
    for _ in range(3):
        for k, m in arms.items():
            s, t = window(m, seconds)
            tot[k][0] += s
            tot[k][1] += t
            rates[k].append(round(s / t, 1))
    out = {"config": name}
    for k, m in arms.items():
        up = m.learner.upload_bytes()
        out[k] = {"env_steps_per_s": round(tot[k][0] / tot[k][1], 1), "windows": rates[k],
                  "ms_per_step": round(1e3 * tot[k][1] / tot[k][0], 3),
                  "h2d_bytes_per_step": round((up["observe"] + up["other"] - base[k]["observe"] - base[k]["other"]) / tot[k][0])}
    out["speedup"] = round(out["device_obs_norm"]["env_steps_per_s"] / out["default"]["env_steps_per_s"], 3)
    for m in arms.values():
        m.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="+", default=["flat100", "depth"], choices=sorted(CONFIGS))
    ap.add_argument("--seconds", type=float, default=2.0)
    a = ap.parse_args()
    print(json.dumps(card()), flush=True)
    for name in a.configs:
        print(json.dumps(case(name, a.seconds)), flush=True)


if __name__ == "__main__":
    main()
