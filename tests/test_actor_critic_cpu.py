"""``PPO2.learn`` and ``TRPO.learn`` on a recording stand-in learner: every call each front end makes of its learner, with its
arguments as flattened float32 values, through two full updates, a callback stop in the middle of a rollout and ``predict``.
The record is kept in actor_critic_expected.json.  Needs no GPU."""
import json
import os

import numpy as np
import pytest

from b200grasp import ppo2, trpo_mpi
from b200grasp.vec_env import DummyVecEnv
from tests.fake_env import FakeFlatEnv

HERE = os.path.dirname(os.path.abspath(__file__))
LOG = []


def _flat(v):
    if isinstance(v, (bool, int, float, np.integer, np.floating, np.ndarray, list, tuple)):
        return [float(x) for x in np.asarray(v, np.float32).reshape(-1)]
    return v


class RecordingLearner:
    """Answers from its inputs alone, so that the record shows what the front end passed and what it did with the answers."""
    three_outputs = True          # PPO2Learner.act returns (actions, values, neglogp); TRPOLearner.act (actions, values)

    def __init__(self, obs_dim, n_actions, *a, **k):
        self.obs_dim, self.n_actions = int(obs_dim), int(n_actions)
        self.n_calls = 0
        self._log("__init__", obs_dim, n_actions, *a, *k.values())

    def _log(self, name, *args):
        LOG.append([name] + [_flat(x) for x in args])

    def _actions(self, obs):
        obs = np.asarray(obs, np.float32).reshape(-1, self.obs_dim)
        self.n_calls += 1
        return 3.0 * obs[:, :1] - 1.5 + 0.25 * np.arange(self.n_actions, dtype=np.float32) + 0.01 * self.n_calls

    def load_parameters(self, params, exact_match=True):
        self._log("load_parameters", *params.values())

    def rollout_reset(self):
        self._log("rollout_reset")

    def rollout_act(self, obs):
        self._log("rollout_act", obs)
        a = self._actions(obs)
        return a if self.three_outputs else a.reshape(-1)

    def rollout_reward(self, rew, done):
        self._log("rollout_reward", rew, done)

    def update(self, last_obs, perms, *hyper):
        self._log("update", last_obs, perms, *hyper)
        return {"policy_loss": 0.5 + 0.125 * self.n_calls, "value_loss": 0.25, "entropy": 1.0, "approxkl": 0.0, "clipfrac": 0.0,
                "optimgain": 0.5, "meankl": 0.01, "vf_loss": 0.125}

    def act(self, obs, deterministic=True):
        self._log("act", obs, deterministic)
        a = self._actions(obs)
        v = np.asarray(obs, np.float32).reshape(-1, self.obs_dim).sum(1)
        return (a, v, -v) if self.three_outputs else (a, v)

    def close(self):
        self._log("close")


class EpisodeEnv(FakeFlatEnv):
    """FakeFlatEnv that reports each finished episode in its info, as Monitor does."""

    def step(self, action):
        o, r, d, info = super().step(action)
        return o, r, d, ({"episode": {"r": round(r, 6), "l": self.t}} if d else info)


def _run(algo):
    LOG.clear()
    if algo == "ppo2":
        env = DummyVecEnv([lambda s=s: EpisodeEnv(seed=s, horizon=3, obs_dim=5, n_act=2) for s in (1, 2)])
        m = ppo2.PPO2("MlpPolicy", env, n_steps=4, nminibatches=2, noptepochs=3, seed=5, policy_kwargs={"layers": [8, 4]},
                      learning_rate=lambda f: 1e-3 * f, cliprange=0.3)
        n_batch = 8
    else:
        env = DummyVecEnv([lambda: EpisodeEnv(seed=3, horizon=3, obs_dim=5, n_act=2)])
        m = trpo_mpi.TRPO("MlpPolicy", env, timesteps_per_batch=4, vf_iters=2, seed=5, policy_kwargs={"layers": [8, 4]})
        n_batch = 4
    np.random.seed(31)
    m.learn(2 * n_batch)
    rec = {"first": {"num_timesteps": m.num_timesteps, "ep_info_buf": list(m.ep_info_buf), "last_metrics": m.last_metrics}}
    np.random.seed(37)
    m.learn(10 * n_batch, callback=lambda _l, _g: m.num_timesteps < n_batch + 3)
    rec["stopped"] = {"num_timesteps": m.num_timesteps, "n_ep": len(m.ep_info_buf)}
    for obs, det in ((np.linspace(0, 1, 5, dtype=np.float32), True), (np.linspace(0.2, 0.9, 15).reshape(3, 5), False)):
        a, state = m.predict(obs, deterministic=det)
        rec.setdefault("predict", []).append([list(np.shape(a)), _flat(a), state])
    m.close()
    rec["log"] = LOG[:]
    return json.loads(json.dumps(rec))


with open(os.path.join(HERE, "actor_critic_expected.json")) as _f:
    EXPECTED = json.load(_f)


@pytest.mark.parametrize("algo", ["ppo2", "trpo"])
def test_learn_and_predict_record(algo, monkeypatch):
    cls = type("RecordingLearner", (RecordingLearner,), {"three_outputs": algo == "ppo2"})
    monkeypatch.setattr(*((ppo2, "PPO2Learner") if algo == "ppo2" else (trpo_mpi, "TRPOLearner")), cls)
    assert _run(algo) == EXPECTED[algo]
