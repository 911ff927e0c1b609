"""The PPO2 learner (csrc/ppo.cu, b200grasp.ppo2.PPO2) against the float64 oracle (oracle/ppo_ref.py) and the restated
noise stream (oracle/philox_ref.py).

  * explicit minibatch steps at obs 1 / 100 / 8192 / 20480, A 1 / 3 / 5, widths 4 and 256, minibatch 1 / 32 / 16384: losses,
    metrics, the clipped gradient and the parameters after Adam (q unchanged, logstd updated), with ratios clipped on both sides
    and value clipping defaulted, on and off;
  * rollouts at n_envs 1, 3 and 16: actions = mean + std * noise(act_seed(seed), step), values, neglogp, GAE;
  * two whole updates in given permutations against the oracle's minibatch steps in sequence;
  * PPO2.learn's schedule, early stop, VecNormalize, predict, save / load, training state and the CLI.
Tolerances are those of tests/test_gpu_dqn.py: 1e-4 relative on forward values and losses, 1e-3 on gradients.  Parameters
after Adam are held to 5% of one Adam step (lr): a gradient component near Adam's epsilon (1e-5) moves the step by its own
relative error.
"""
import os

import numpy as np
import pytest
import yaml

import b200grasp
from b200grasp import train_cli
from b200grasp.common.policies import MlpPolicy
from b200grasp.ppo2 import PPO2, PPO2Learner
from b200grasp.spaces import Box
from b200grasp.vec_env import DummyVecEnv, VecNormalize
from oracle import philox_ref as PX
from oracle import ppo_ref as R
from tests.fake_env import FakeGraspEnv
from tests.util import rel_err

pytestmark = pytest.mark.gpu
TOL, GTOL, LR = 1e-4, 1e-3, 1e-3


def _params(obs, A, layers, seed, logstd=0.3):
    p = R.init_params(obs, A, layers, np.random.default_rng(seed))
    rng = np.random.default_rng(seed + 100)
    for k in p:                                   # non-zero biases / logstd so every path carries signal
        if p[k].ndim == 1 or k.endswith("logstd"):
            p[k] = rng.uniform(-logstd, logstd, p[k].shape).astype(np.float32)
    p["model/pi/w"] = (p["model/pi/w"] * 50).astype(np.float32)
    return p


def _minibatch(p, M, obs, A, seed, obs_scale=1.0):
    rng = np.random.default_rng(seed)
    x = (rng.normal(0, 1, (M, obs)) * obs_scale / np.sqrt(obs)).astype(np.float32)
    mean, v = R.forward(p, x)
    std = np.exp(p["model/pi/logstd"].astype(np.float64).reshape(-1))
    act = (mean + std * rng.normal(0, 1, (M, A))).astype(np.float32)
    nlp = R.neglogp(mean, p["model/pi/logstd"], act)
    old_nlp = (nlp + rng.uniform(-0.6, 0.6, M)).astype(np.float32)       # ratios on both sides of 1 +- 0.2
    old_v = (v + rng.uniform(-0.5, 0.5, M)).astype(np.float32)
    ret = (old_v + rng.normal(0, 1.0, M)).astype(np.float32)
    return x, ret, act, old_v, old_nlp


def _check_params(new, ref, old, lr):
    for k in new:
        if k.startswith("model/q/"):
            assert np.array_equal(new[k], old[k]), k
            continue
        err = np.max(np.abs(new[k].astype(np.float64) - ref[k]))
        assert err <= 0.05 * lr, (k, err)
    assert not np.array_equal(new["model/pi/logstd"], old["model/pi/logstd"])


EXPLICIT = [  # obs, A, H0, H1, M, cliprange_vf, obs_scale
    (100, 3, 64, 64, 32, None, 1.0),
    (1, 1, 4, 4, 1, None, 1.0),
    (8192, 5, 64, 64, 32, 0.1, 1.0),
    (20480, 5, 64, 64, 64, -1.0, 1.0),
    (7, 16, 256, 4, 33, 0.05, 1.0),
    (100, 3, 4, 256, 16384, None, 1.0),
    (100, 3, 64, 64, 32, -1.0, 0.01),        # small gradients: global norm below max_grad_norm
]


@pytest.mark.parametrize("obs,A,H0,H1,M,cvf,scale", EXPLICIT)
def test_explicit_step(obs, A, H0, H1, M, cvf, scale):
    seed = obs + 7 * A + M
    L = PPO2Learner(obs, A, (H0, H1), n_envs=1, n_steps=M, nminibatches=1, noptepochs=1, seed=seed)
    p = _params(obs, A, (H0, H1), seed)
    L.load_parameters(p)
    x, ret, act, ov, onlp = _minibatch(p, M, obs, A, seed, scale)
    cvf_dev = 0.2 if cvf is None else cvf
    out = L.train_step_explicit(x, ret, act, ov, onlp, LR, 0.2, cvf_dev, apply_update=True)
    ref_p, met, gc = R.train_step(R.as_float64(p), R.Adam(), x, ret, act, ov, onlp, LR, 0.2, cvf)
    for k in ("policy_loss", "value_loss", "entropy", "approxkl", "clipfrac", "grad_norm"):
        assert abs(out[k] - met[k]) <= TOL * max(1.0, abs(met[k])), (k, out[k], met[k])
    g = L.get_gradients()
    for k in gc:
        assert rel_err(g[k].reshape(-1), gc[k].reshape(-1)) <= GTOL, (k, rel_err(g[k].reshape(-1), gc[k].reshape(-1)))
    _check_params(L.get_parameters(), ref_p, p, LR)
    if scale == 1.0 and 1 < M <= 64:           # the large minibatch averages its gradient below max_grad_norm
        assert met["grad_norm"] > 0.5 and 0.0 < met["clipfrac"] < 1.0
    L.close()


def test_explicit_step_unapplied_leaves_parameters():
    L = PPO2Learner(100, 3, (64, 64), n_envs=1, n_steps=32, nminibatches=1, noptepochs=1, seed=3)
    p = _params(100, 3, (64, 64), 3)
    L.load_parameters(p)
    x, ret, act, ov, onlp = _minibatch(p, 32, 100, 3, 3)
    L.train_step_explicit(x, ret, act, ov, onlp, LR, 0.2, 0.2, apply_update=False)
    for k, a in L.get_parameters().items():
        assert np.array_equal(a, p[k]), k
    assert L.steps()[0] == 0
    L.close()


def _scripted(T, E, D, seed):
    rng = np.random.default_rng(seed)
    obs = rng.normal(0, 1, (T + 1, E, D)).astype(np.float32)
    rew = rng.normal(0, 1, (T, E)).astype(np.float32)
    done = (rng.random((T, E)) < 0.25).astype(np.float32)
    done[0, 0] = 1.0
    done[-1, -1] = 1.0
    if T > 3:
        done[1:3, 0] = 1.0                     # consecutive dones
    return obs, rew, done


def _rollout(L, p, obs, rew, done, seed):
    """Fills the rollout and checks every step's actions / values / neglogp against the oracle and the noise stream."""
    T, E, D = obs.shape[0] - 1, obs.shape[1], obs.shape[2]
    A = L.n_actions
    logstd = p["model/pi/logstd"].astype(np.float64).reshape(-1)
    step0 = L.steps()[1]
    for t in range(T):
        a = L.rollout_act(obs[t])
        mean, v = R.forward(p, obs[t])
        eps = PX.noise(PX.act_seed(seed), step0 + t, E * A).reshape(E, A)
        ref = mean + np.exp(logstd) * eps
        assert rel_err(a.reshape(-1), ref.reshape(-1)) <= TOL, t
        L.rollout_reward(rew[t], done[t])
    r = L.rollout_get()
    return r


@pytest.mark.parametrize("E", [1, 3, 16])
def test_rollout_and_gae(E):
    T, D, A, seed = 8, 100, 3, 20 + E
    L = PPO2Learner(D, A, (64, 64), n_envs=E, n_steps=T, nminibatches=1, noptepochs=1, seed=seed)
    p = _params(D, A, (64, 64), seed)
    L.load_parameters(p)
    obs, rew, done = _scripted(T, E, D, seed)
    r = _rollout(L, p, obs, rew, done, seed)
    mean, v = R.forward(p, obs[:T].reshape(T * E, D))
    assert rel_err(r["values"].reshape(-1), v) <= TOL
    nlp = R.neglogp(mean, p["model/pi/logstd"], r["actions"].reshape(T * E, A))
    assert rel_err(r["neglogp"].reshape(-1), nlp) <= TOL
    perm = np.stack([np.random.default_rng(seed).permutation(T * E)]).astype(np.int32)
    L.update(obs[T], perm, 0.0, 0.2, 0.2)                    # lr 0: the GAE of this rollout, parameters kept
    r = L.rollout_get()
    starts = np.concatenate([np.zeros((1, E), np.float32), done[:-1]])     # episode-start flags of each step
    _, lastv = R.forward(p, obs[T])
    adv, ret = R.gae(rew, r["values"], starts, lastv, done[-1], 0.99, 0.95)
    assert rel_err(r["advantages"].reshape(-1), adv.reshape(-1)) <= TOL
    assert rel_err(r["returns"].reshape(-1), ret.reshape(-1)) <= TOL
    L.close()


def test_two_updates_against_oracle():
    T, E, D, A, NMB, NOE, seed = 16, 4, 100, 3, 4, 4, 41
    L = PPO2Learner(D, A, (64, 64), n_envs=E, n_steps=T, nminibatches=NMB, noptepochs=NOE, seed=seed)
    p = _params(D, A, (64, 64), seed)
    L.load_parameters(p)
    opt = R.Adam()
    P = R.as_float64(p)
    rng = np.random.default_rng(seed)
    for u in range(2):
        cur = {k: v.astype(np.float32) for k, v in P.items()}
        obs, rew, done = _scripted(T, E, D, seed + u)
        if u == 0:
            r = _rollout(L, cur, obs, rew, done, seed)
        else:
            for t in range(T):
                L.rollout_act(obs[t])
                L.rollout_reward(rew[t], done[t])
        perms = np.stack([rng.permutation(T * E) for _ in range(NOE)]).astype(np.int32)
        m = L.update(obs[T], perms, LR, 0.2, -1.0 if u else 0.2)
        r = L.rollout_get()
        f = R.swap_and_flatten
        P, met = R.update(P, opt, f(obs[:T]), f(r["returns"]), f(r["actions"]), f(r["values"]), f(r["neglogp"]), perms, NMB, LR, 0.2,
                          -1.0 if u else None)
        for k in ("policy_loss", "value_loss", "entropy", "approxkl", "clipfrac"):
            assert abs(m[k] - met[k]) <= 1e-3 * max(1.0, abs(met[k])), (u, k, m[k], met[k])
        new = L.get_parameters()
        for k in new:
            if k.startswith("model/q/"):
                assert np.array_equal(new[k], p[k])
                continue
            d_dev, d_ref = new[k].astype(np.float64) - p[k], P[k] - p[k]
            assert rel_err(d_dev.reshape(-1), d_ref.reshape(-1)) <= 2e-2, (u, k, rel_err(d_dev.reshape(-1), d_ref.reshape(-1)))
        assert m["n_updates"] == (u + 1) * NMB * NOE
    L.close()


class FlatEnv:
    """A deterministic environment that costs nothing: obs the step counter's features, reward -|a - target|^2."""

    def __init__(self, D=6, A=3, horizon=7, seed=0):
        self.observation_space = Box(-10.0, 10.0, (D,))
        self.action_space = Box(-1.0, 1.0, (A,))
        self.D, self.A, self.horizon, self.t, self.k = D, A, horizon, 0, seed

    def _obs(self):
        return np.cos(np.arange(self.D) * 0.7 + self.t * 0.3 + self.k).astype(np.float32)

    def reset(self):
        self.t = 0
        return self._obs()

    def step(self, a):
        self.t += 1
        r = -float(np.sum((np.asarray(a) - 0.5) ** 2))
        return self._obs(), r, self.t >= self.horizon, {}

    def close(self):
        pass


class Counter(b200grasp.callbacks.BaseCallback):
    def __init__(self, stop_at=None):
        super().__init__()
        self.stop_at, self.calls = stop_at, 0

    def _on_step(self):
        self.calls += 1
        return self.stop_at is None or self.calls < self.stop_at


def test_learn_schedule_and_early_stop():
    env = DummyVecEnv([lambda: FlatEnv(seed=i) for i in range(2)])
    m = PPO2(MlpPolicy, env, n_steps=16, nminibatches=4, noptepochs=3, seed=5)
    cb = Counter()
    m.learn(100, callback=cb)                 # n_batch 32: 3 updates, 96 env steps
    assert m.num_timesteps == 96 and cb.calls == 48
    assert m.last_metrics["n_updates"] == 3 * 4 * 3
    cb = Counter(stop_at=20)
    m.learn(1000, callback=cb)                # stops during the second rollout: one more update
    assert cb.calls == 20 and m.num_timesteps == 40 and m.last_metrics["n_updates"] == 4 * 4 * 3
    with pytest.raises(NotImplementedError):
        b200grasp.PPO2
    m.close()


def test_learn_vecnormalize_stores_wrapper_obs():
    seen = []

    class Spy(VecNormalize):
        def reset(self):
            o = super().reset(); seen.append(np.array(o)); return o

        def step(self, a):
            o, r, d, i = super().step(a); seen.append(np.array(o)); return o, r, d, i

    env = Spy(DummyVecEnv([lambda: FlatEnv(D=9, seed=3)]), norm_obs=True, norm_reward=True, clip_obs=10.0)
    m = PPO2("MlpPolicy", env, n_steps=32, nminibatches=4, seed=2)
    p0 = m.learner.get_parameters()
    m.learn(32)
    r = m.learner.rollout_get()
    _, v = R.forward(p0, np.concatenate(seen[:32]).reshape(32, 9))
    assert rel_err(r["values"].reshape(-1), v) <= TOL
    m.close()


def test_predict_save_load_and_training_state(tmp_path):
    env = DummyVecEnv([lambda: FakeGraspEnv(seed=0, horizon=6, obs_shape=(8, 8, 2))])
    m = PPO2(MlpPolicy, env, n_steps=16, nminibatches=2, noptepochs=2, seed=9)
    m.learn(32)
    o = np.stack([FakeGraspEnv(seed=s, obs_shape=(8, 8, 2)).reset() for s in range(5)])
    a_det, _ = m.predict(o, deterministic=True)
    mean, _ = R.forward(m.learner.get_parameters(), o.reshape(5, -1))
    assert rel_err(a_det.reshape(-1), np.clip(mean, -1, 1).reshape(-1)) <= TOL
    a_sto, _ = m.predict(o, deterministic=False)
    assert a_sto.shape == (5, 5) and np.all(np.abs(a_sto) <= 1.0) and not np.allclose(a_sto, a_det)
    assert m.predict(o[0], deterministic=True)[0].shape == (5,)
    m.save(str(tmp_path / "ppo"))
    m2 = PPO2.load(str(tmp_path / "ppo"))
    assert np.array_equal(m2.predict(o, deterministic=True)[0], a_det)
    for k, v in m.get_parameters().items():
        assert np.array_equal(m2.get_parameters()[k], v)
    m2.close()
    m.close()
    # training state: save at an update boundary, continue; a model rebuilt from the state on a fresh copy of the (deterministic)
    # environment continues the same way
    def flat():
        return DummyVecEnv([lambda: FlatEnv(D=10, A=3, horizon=6)])
    np.random.seed(123)
    m = PPO2(MlpPolicy, flat(), n_steps=16, nminibatches=2, noptepochs=2, seed=9)
    m.learn(64)
    m.save_training_state(str(tmp_path / "state"))
    steps_at_save = m.learner.steps()[:2]
    m.learn(48, reset_num_timesteps=False)
    ref = m.get_parameters()
    r = PPO2.load_training_state(str(tmp_path / "state"), flat())
    assert r.num_timesteps == 64 and r.learner.steps()[:2] == steps_at_save
    r.learn(48, reset_num_timesteps=False)
    assert r.num_timesteps == m.num_timesteps == 112
    # split-R contractions accumulate with atomics, so the two runs agree to rounding; Adam can turn the rounding of a
    # gradient component near its epsilon into part of one step (lr = 2.5e-4) on a few elements
    for k, v in r.get_parameters().items():
        d = np.abs(v.astype(np.float64) - ref[k])
        assert np.quantile(d, 0.99) <= 1e-5 and d.max() <= 4 * 2.5e-4, (k, np.quantile(d, 0.99), d.max())
    m.close(); r.close()


def test_refusals():
    env = DummyVecEnv([lambda: FlatEnv()])
    from b200grasp.common.policies import CnnPolicy
    with pytest.raises(NotImplementedError):
        PPO2(CnnPolicy, env)
    with pytest.raises(ValueError):
        PPO2(MlpPolicy, env, n_steps=10, nminibatches=4)
    with pytest.raises(NotImplementedError):
        PPO2(MlpPolicy, env, policy_kwargs={"net_arch": [64, dict(pi=[64], vf=[64])]})
    with pytest.raises(NotImplementedError):
        PPO2(MlpPolicy, env, device_obs_norm=True)
    L = PPO2Learner(100, 3, (64, 64), n_envs=1, n_steps=4, nminibatches=1, noptepochs=1)
    with pytest.raises(RuntimeError, match="not full"):
        L.update(np.zeros((1, 100)), np.zeros((1, 4)), LR, 0.2, 0.2)
    for kw, what in ((dict(n_actions=17), "n_actions"), (dict(layers=(64, 260)), "hidden"), (dict(layers=(6, 64)), "hidden"),
                     (dict(n_envs=5000), "n_envs"), (dict(n_steps=3, nminibatches=2), "divisible"),
                     (dict(n_steps=40000, nminibatches=2), "16384")):
        args = dict(obs_dim=100, n_actions=3, layers=(64, 64), n_envs=1, n_steps=4, nminibatches=1, noptepochs=1)
        args.update(kw)
        with pytest.raises(RuntimeError, match=what):
            PPO2Learner(**args)
    L.close()


def make_env(config, evaluate=False, validate=False, test=False):
    return FlatEnv(D=12, A=3, horizon=5, seed=1 if evaluate else 0)


def test_cli_train_and_run_ppo(tmp_path):
    cfg = {"PPO": {"learning_rate": 3e-4, "total_timesteps": 300, "layers": [32, 32], "n_steps": 64}, "discount_factor": 0.99,
           "robot": {"discrete": False}, "reward": {}, "normalize": True}
    cpath = tmp_path / "c.yaml"
    cpath.write_text(yaml.safe_dump(cfg))
    out = tmp_path / "run"
    model = train_cli.main(["train", "--config", str(cpath), "--algo", "PPO", "--model_dir", str(out), "--env", "tests.test_gpu_ppo:make_env",
                            "--eval_freq", "100", "--checkpoint_freq", "150", "--state_freq", "128", "--n_envs", "2"])
    assert model.num_timesteps == 256 and model.n_steps == 128 and model.layers == [64, 64] and model.learning_rate == 3e-4
    assert os.path.exists(out / "final_model.zip") and os.path.exists(out / "training_state" / "host.json")
    model.close()
    res = train_cli.main(["run", "--model", str(out / "final_model.zip"), "--env", "tests.test_gpu_ppo:make_env", "--episodes", "2"])
    assert res["episodes"] == 2 and res["mean_steps"] == 5.0
