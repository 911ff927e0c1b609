"""TRPO without a device: the float64 restatement's pieces against each other, the front end on a recording stand-in learner,
the command line and the C ABI declarations."""
import inspect
import json
import os
import re
from collections import OrderedDict

import numpy as np
import pytest

import b200grasp
from b200grasp import _lib, train_cli, trpo_mpi
from b200grasp.common.policies import CnnPolicy, MlpPolicy
from b200grasp.spaces import Box, Discrete
from b200grasp.trpo_mpi import TRPO
from b200grasp.vec_env import DummyVecEnv, VecNormalize
from oracle import ppo_ref
from tests import trpo_ref as R
from tests.fake_env import FakeFlatEnv

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _params(D, A, layers=(8, 8), seed=0, logstd=None):
    p = OrderedDict((k[len("model/"):], np.asarray(v, np.float64)) for k, v in ppo_ref.init_params(D, A, layers, np.random.default_rng(seed)).items())
    rng = np.random.default_rng(seed + 1)
    for k in ("pi/w", "pi_fc0/b", "pi_fc1/b", "pi/b"):
        p[k] = p[k] + rng.normal(0, 0.3, p[k].shape)
    p["pi/logstd"] = rng.normal(0, 0.3, p["pi/logstd"].shape) if logstd is None else np.full(p["pi/logstd"].shape, logstd)
    return p


# ---------------------------------------------------------------- the algorithm's pieces
@pytest.mark.parametrize("D,A,N", [(5, 1, 11), (7, 3, 40), (3, 5, 23)])
def test_fvp_double_backprop_equals_gauss_newton(D, A, N):
    p = _params(D, A)
    rng = np.random.default_rng(3)
    obs = rng.normal(size=(N, D))[::5]
    n = len(R.flat(R.tensors(p)))
    for _ in range(3):
        v = rng.normal(size=n)
        a, b = R.fvp(p, obs, v, 1e-2), R.fvp_gauss_newton(p, obs, v, 1e-2)
        assert np.abs(a - b).max() <= 1e-12 * max(1.0, np.abs(a).max())


def test_cg_solves_spd_system():
    rng = np.random.default_rng(0)
    Q = rng.normal(size=(12, 12))
    F = Q @ Q.T + 12 * np.eye(12)
    b = rng.normal(size=12)
    x, it = R.cg(lambda p: F @ p, b.copy(), cg_iters=40)
    assert np.abs(F @ x - b).max() < 2e-5 and it <= 40


def test_cg_exits_after_one_iteration_on_logstd_only_gradient():
    p = _params(4, 3)
    obs = np.random.default_rng(1).normal(size=(20, 4))[::5]
    n = len(R.flat(R.tensors(p)))
    g = np.zeros(n)
    g[-3:] = [0.3, -0.2, 0.1]
    x, it = R.cg(lambda v: R.fvp(p, obs, v, 1e-2), g.copy(), 10)
    assert it == 1
    assert np.allclose(x[-3:], g[-3:] / 2.01, rtol=1e-12) and np.abs(x[:-3]).max() == 0.0


@pytest.mark.parametrize("seq,expect", [
    ([[0.1, 0.005, 0, 0.1, 1]], 0),                                                     # accepted at once
    ([[0.1, 0.02, 0, 0.1, 1], [0.05, 0.014, 0, 0.05, 1]], 1),                           # shrink for KL
    ([[-0.1, 0.001, 0, -0.1, 1], [-0.01, 0.001, 0, -0.01, 1], [0.02, 0.001, 0, 0.02, 1]], 2),   # shrink for no improvement
    ([[np.nan, 0.001, 0, 0.1, 1], [0.1, 0.001, 0, 0.1, 1]], 1),                         # shrink for a non-finite loss
    ([[-1.0, 1.0, 0, -1.0, 1]] * 10, -1),                                               # every candidate rejected
])
def test_line_search_outcomes(seq, expect):
    k, L = R.line_search(lambda i: seq[min(i, len(seq) - 1)], 0.0, 0.01)
    assert k == expect
    assert (L is None) == (expect < 0)


def test_value_minibatch_split():
    for split in (R.value_minibatches, trpo_mpi.value_minibatches):
        mb = split(400)
        assert mb == [(0, 128), (128, 256), (256, 384)] and 400 - mb[-1][1] == 16
        assert split(100) == []


def test_atarg_of_equal_advantages_is_zero():
    assert np.all(R.standardize(np.full(7, 3.5)) == 0.0)


def test_zero_gradient_leaves_policy_and_trains_value():
    p = _params(4, 2, layers=(4, 4))
    rng = np.random.default_rng(0)
    obs, act = rng.normal(size=(130, 4)), rng.normal(size=(130, 2))
    new, rec = R.iteration(p, R.MpiAdam(), obs, act, np.full(130, 2.0), rng.normal(size=130), [rng.permutation(130)])
    assert rec["accepted"] == -2
    for n in R.POLICY:
        assert np.array_equal(new[n], p[n])
    assert not np.array_equal(new["vf/w"], p["vf/w"]) and np.array_equal(new["q/w"], p["q/w"])


# ---------------------------------------------------------------- the front end on a recording stand-in learner
LOG = []


class FakeTRPOLearner:
    def __init__(self, obs_dim, n_actions, layers=(64, 64), timesteps_per_batch=1024, *args, **kw):
        LOG.append(("init", obs_dim, n_actions, tuple(layers), timesteps_per_batch) + tuple(args))
        specs = [(s + n, shp) for s in ("pi/model/", "oldpi/model/") for n, shp in
                 ((k[len("model/"):], v) for k, v in ppo_ref.param_specs(obs_dim, n_actions, tuple(layers)))]
        self.param_shapes = OrderedDict(specs)
        self.params = OrderedDict((n, np.zeros(s, np.float32)) for n, s in specs)
        self.obs_dim, self.n_actions, self.N = obs_dim, n_actions, timesteps_per_batch

    def load_parameters(self, params, exact_match=True):
        for n, a in params.items():
            n = n[:-2] if n.endswith(":0") else n
            self.params[n] = np.asarray(a, np.float32).reshape(self.param_shapes[n]).copy()

    def get_parameters(self):
        return OrderedDict((n, a.copy()) for n, a in self.params.items())

    def rollout_reset(self):
        LOG.append(("reset",))

    def rollout_act(self, obs):
        LOG.append(("act",))
        return np.full(self.n_actions, 2.0, np.float32)

    def rollout_reward(self, rew, done):
        LOG.append(("reward",))

    def update(self, last_obs, perms):
        LOG.append(("update", np.asarray(perms).shape))
        return {"accepted": 0}

    def act(self, obs, deterministic=True):
        return np.full((len(obs), self.n_actions), 5.0, np.float32), np.zeros(len(obs), np.float32)

    def save_state(self, path):
        LOG.append(("save_state",))
        with open(path, "wb") as f:
            f.write(b"fake")

    def load_state(self, path):
        LOG.append(("load_state",))

    def close(self):
        pass


@pytest.fixture
def fake(monkeypatch):
    monkeypatch.setattr(trpo_mpi, "TRPOLearner", FakeTRPOLearner)
    LOG.clear()
    yield
    LOG.clear()


def test_constructor_defaults():
    sig = inspect.signature(TRPO.__init__)
    want = dict(gamma=0.99, timesteps_per_batch=1024, max_kl=0.01, cg_iters=10, lam=0.98, entcoeff=0.0, cg_damping=1e-2,
                vf_stepsize=3e-4, vf_iters=3, verbose=0, tensorboard_log=None, _init_setup_model=True, policy_kwargs=None,
                full_tensorboard_log=False, seed=None, n_cpu_tf_sess=1, device=0)
    for k, v in want.items():
        assert sig.parameters[k].default == v, k


def test_refusals():
    with pytest.raises(NotImplementedError, match="trpo_mpi.TRPO"):
        b200grasp.TRPO
    with pytest.raises(NotImplementedError, match="trpo_mpi.TRPO"):
        b200grasp.SAC(MlpPolicy, None)
    for bad in (CnnPolicy, "CnnPolicy", "MlpLstmPolicy", "MlpLnLstmPolicy"):
        with pytest.raises(NotImplementedError):
            TRPO(bad, None)
    with pytest.raises(NotImplementedError):
        TRPO(MlpPolicy, None, policy_kwargs={"layer_norm": True})
    for kw in ("expert_dataset", "hidden_size_adversary", "g_step"):
        with pytest.raises(NotImplementedError, match="GAIL"):
            TRPO(MlpPolicy, None, **{kw: 1})
    with pytest.raises(NotImplementedError, match="device_obs_norm"):
        TRPO(MlpPolicy, None, device_obs_norm=True)
    with pytest.raises(ValueError, match="non vectorized environment or a single vectorized environment"):
        TRPO(MlpPolicy, DummyVecEnv([FakeFlatEnv, FakeFlatEnv]), _init_setup_model=False)
    with pytest.raises(NotImplementedError, match="Box"):
        TRPO(MlpPolicy, FakeFlatEnv(n_discrete=4), _init_setup_model=False)


def test_learn_iterations_and_early_stop(fake):
    m = TRPO(MlpPolicy, FakeFlatEnv(horizon=3), timesteps_per_batch=4, seed=2)
    assert LOG[0][:5] == ("init", 6, 3, (64, 64), 4)
    LOG.clear()
    m.learn(9)                                # ceil(9 / 4) = 3 iterations
    assert [e for e in LOG if e[0] == "update"] == [("update", (3, 4))] * 3 and m.num_timesteps == 12
    LOG.clear()
    m.learn(100, callback=lambda _l, _g: m.num_timesteps < 6)
    assert [e[0] for e in LOG].count("update") == 1 and m.num_timesteps == 6 and LOG[-1] == ("reset",)
    a, _ = m.predict(np.zeros(6, np.float32))
    assert a.shape == (3,) and np.all(a == 1.0)          # clipped to the Box


def test_zip_names_save_load_and_training_state(fake, tmp_path):
    m = TRPO(MlpPolicy, VecNormalize(DummyVecEnv([lambda: FakeFlatEnv(obs_dim=5, n_act=2)])), timesteps_per_batch=8, seed=4,
             policy_kwargs={"layers": [8, 12]})
    names = list(m.get_parameters())
    assert names[:15] == [f"pi/model/{k[len('model/'):]}:0" for k, _ in ppo_ref.param_specs(5, 2, (8, 12))]
    assert names[15:] == [f"oldpi/model/{k[len('model/'):]}:0" for k, _ in ppo_ref.param_specs(5, 2, (8, 12))]
    init = trpo_mpi.init_params(5, 2, (8, 12), 4)
    rng = np.random.default_rng(4)
    want = ppo_ref.init_params(5, 2, (8, 12), rng)
    want2 = ppo_ref.init_params(5, 2, (8, 12), rng)
    for k, v in want.items():
        assert np.array_equal(init["pi/" + k], v) and np.array_equal(init["oldpi/" + k], want2[k])
    m.save(str(tmp_path / "m.zip"))
    m2 = TRPO.load(str(tmp_path / "m"))
    assert m2.layers == [8, 12] and m2.timesteps_per_batch == 8 and m2.action_space.shape == (2,)
    for (k, a), (k2, b) in zip(m.get_parameters().items(), m2.get_parameters().items()):
        assert k == k2 and np.array_equal(a, b)
    m.learn(8)
    m.save_training_state(str(tmp_path / "state"))
    host = json.load(open(tmp_path / "state" / "host.json"))
    assert host["algo"] == "TRPO" and host["num_timesteps"] == 8 and host["init"]["timesteps_per_batch"] == 8
    st = np.random.get_state()
    np.random.seed(123)
    m3 = TRPO.load_training_state(str(tmp_path / "state"), VecNormalize(DummyVecEnv([lambda: FakeFlatEnv(obs_dim=5, n_act=2)])))
    assert m3.num_timesteps == 8 and ("load_state",) in LOG
    assert np.array_equal(np.random.get_state()[1], st[1])


# ---------------------------------------------------------------- the command line
def _cfg(tmp_path):
    cfg = {"discount_factor": 0.9, "normalize": False, "robot": {}, "reward": {},
           "TRPO": {"max_iters": 400, "step_size": 0.001, "total_timesteps": 10}}
    p = tmp_path / "c.yaml"
    import yaml
    yaml.safe_dump(cfg, open(p, "w"))
    return cfg, str(p)


def test_trpo_kwargs_and_cli_refusals(tmp_path):
    cfg, path = _cfg(tmp_path)
    assert train_cli.trpo_kwargs(cfg) == dict(verbose=2, gamma=0.9, timesteps_per_batch=400, vf_stepsize=0.001)
    for extra, exc in ((["--load_dir", "x/y.zip"], NotImplementedError), (["--device_norm"], NotImplementedError),
                       (["--n_envs", "2"], ValueError)):
        d = tmp_path / f"run{len(extra)}{extra[0]}"
        with pytest.raises(exc):
            train_cli.main(["train", "--config", path, "--algo", "TRPO", "--model_dir", str(d), "--env", "tests.fake_env:make_env"] + extra)
        assert not d.exists()


# ---------------------------------------------------------------- the C ABI
def test_abi_symbols_in_header_and_lib():
    hdr = open(os.path.join(ROOT, "include", "b200grasp.h")).read()
    names = ("create", "destroy", "param_count", "param_info", "get_param", "set_param", "get_grad", "rollout_act", "rollout_reward",
             "rollout_reset", "rollout_get", "update", "fvp", "step_explicit", "act", "get_step", "state_save", "state_load")
    for n in names:
        assert re.search(rf"\bint b2g_trpo_{n}\(", hdr), n
        assert f"b2g_trpo_{n}" in _lib.SYMBOLS, n
    assert [f for f, _ in _lib.TrpoCfg._fields_][:5] == ["obs_dim", "n_actions", "hidden0", "hidden1", "timesteps_per_batch"]
