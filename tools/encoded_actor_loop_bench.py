"""Times ``SAC.learn`` on the encoded-depth observation (config 5) with the encoder in three places.

  python tools/encoded_actor_loop_bench.py [--n_envs 1 16 128] [--seconds 2.0] [--out FILE]

Every arm runs ``SAC.learn`` itself (MLP policy, batch 64, one gradient step per vectorised env step, device_obs_norm=True)
over a DummyVecEnv of ``n_envs`` environments that cost nothing to step: they hand out pre-generated
``synth.make_depth_scenes`` frames plus one actuator float, wrapped in VecNormalize(norm_obs, norm_reward).
  per_env:  today's integration: every env encodes its own frame with its own encoder (``encode(1)`` per env step) and
            returns the 101-float encoding.  All encoders live in this one process, so this arm understates the cost of
            128 SubprocVecEnv workers, each with its own CUDA context.
  host:     VecEncodeDepth in host mode: one ``encode(n)`` per vectorised step (frames + terminal observations).
  pass_raw: VecEncodeDepth in pass-raw mode: raw frames go to the learner once and are encoded on its device.
The arms alternate in one process; after a warm-up each is timed over windows of at least --seconds, each window ending in
a synchronise of the learner's stream (``learn`` returns after its last observe call, which synchronises).  Printed per case:
env-steps/s of every arm and the bytes copied host->device per vectorised step (the learner's counters plus what the
encoder handles upload).  The card's name and power limit are read in the same run and printed first.  Needs a GPU.
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
from b200grasp.sac_model import SAC, MlpPolicy  # noqa: E402
from b200grasp.spaces import Box  # noqa: E402
from b200grasp.vec_env import DummyVecEnv, VecEncodeDepth, VecNormalize, unwrap_encode_depth  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
PIXELS = 64 * 64


class CountingEncoder:
    """An encoder that counts the bytes its encode calls upload."""

    def __init__(self, enc):
        self.enc, self.bytes = enc, 0
        self.input_shape, self.encoding_dim = enc.input_shape, enc.encoding_dim
        self._handle = enc._handle          # what Learner.set_obs_encoder copies from (pass_raw)

    def encode(self, imgs):
        imgs = np.ascontiguousarray(imgs, np.float32)
        self.bytes += imgs.nbytes
        return self.enc.encode(imgs)


class RawEnv:
    """Raw rows [64*64 depth | actuator] from a small pre-generated pool."""

    def __init__(self, seed, horizon=50, pool=8):
        low, high = np.zeros(PIXELS + 1), np.concatenate([np.full(PIXELS, np.inf), [1.0]])
        self.observation_space = Box(low, high, (PIXELS + 1,))
        self.action_space = Box(-1.0, 1.0, (5,), seed=seed)
        rng = np.random.default_rng(seed)
        self.pool = np.concatenate([synth.make_depth_scenes(pool, seed=seed).reshape(pool, PIXELS), rng.uniform(0, 1, (pool, 1))],
                                   axis=1).astype(np.float32)
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


class PerEnvEncoded(RawEnv):
    """The reference sensor: the env encodes its own frame (encode(1)) and returns [encoding | actuator]."""

    def __init__(self, seed, encoder):
        super().__init__(seed)
        self.encoder = encoder
        self.observation_space = Box(np.concatenate([-np.ones(100), [0.0]]), np.ones(101), (101,))

    def _obs(self):
        row = super()._obs()
        return np.concatenate([self.encoder.encode(row[:PIXELS].reshape(1, 64, 64, 1))[0], row[PIXELS:]])


def make_encoder(max_batch):
    w = dict(np.load(os.path.join(GOLD, "encoder_weights.npz")))
    w = {k.replace("__", "/"): v for k, v in w.items()}
    cfg = json.load(open(os.path.join(GOLD, "encoder_config.json")))
    enc = SimpleAutoEncoder(cfg, max_batch=max_batch)
    enc.set_weights(keras_encoder_arrays(w, len(cfg["network"])))
    return enc


def build(arm, n):
    if arm == "per_env":
        encs = [CountingEncoder(make_encoder(1)) for _ in range(n)]
        venv = DummyVecEnv([(lambda i=i: PerEnvEncoded(i, encs[i])) for i in range(n)])
    else:
        encs = [CountingEncoder(make_encoder(2 * n))]
        venv = VecEncodeDepth(DummyVecEnv([(lambda i=i: RawEnv(i)) for i in range(n)]), encs[0])
    env = VecNormalize(venv, norm_obs=True, norm_reward=True)
    model = SAC(MlpPolicy, env, batch_size=64, buffer_size=100000, learning_starts=64, seed=0, device_obs_norm=True)
    if arm == "host":                 # the learner gives the encoder back: the wrapper encodes
        model.learner.set_obs_encoder(None)
        unwrap_encode_depth(env).take_encoder_back()
    assert (arm == "pass_raw") == bool(getattr(unwrap_encode_depth(env), "pass_raw", False))
    return model, encs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n_envs", type=int, nargs="+", default=[1, 16, 128])
    ap.add_argument("--seconds", type=float, default=2.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(json.dumps({"card": card}), flush=True)
    results = []
    arms = ("per_env", "host", "pass_raw")
    for n in a.n_envs:
        built = {arm: build(arm, n) for arm in arms}
        for arm in arms:                                       # warm-up: every shape the windows use
            built[arm][0].learn(max(8 * n, 256))
        rates = {arm: [] for arm in arms}
        bytes_per_step = {}
        for _ in range(a.rounds):
            for arm in arms:
                model, encs = built[arm]
                steps = max(64 * n, 512)
                up0, enc0 = model.learner.upload_bytes(), sum(e.bytes for e in encs)
                t0, done = time.perf_counter(), 0
                while True:
                    model.learn(steps)
                    done += steps
                    if time.perf_counter() - t0 >= a.seconds:
                        break
                dt = time.perf_counter() - t0
                up1, enc1 = model.learner.upload_bytes(), sum(e.bytes for e in encs)
                rates[arm].append(done / dt)
                vsteps = done / n
                bytes_per_step[arm] = {"learner": (up1["observe"] + up1["other"] - up0["observe"] - up0["other"]) / vsteps,
                                       "encoders": (enc1 - enc0) / vsteps}
        row = {"n_envs": n, **{f"{arm}_steps_per_s": float(np.median(rates[arm])) for arm in arms},
               "spread": {arm: [round(min(rates[arm])), round(max(rates[arm]))] for arm in arms},
               "h2d_bytes_per_vec_step": bytes_per_step, "card": card}
        print(json.dumps(row), flush=True)
        results.append(row)
        for model, _ in built.values():
            model.close()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
