"""The SAC, BDQ, DQN, PPO2 and TRPO front ends on a recording stand-in learner: what each one asks of its learner and what it writes,
through construction, save / load, training-state directories and close.  Needs no GPU."""
import hashlib
import io
import json
import os
import zipfile
from collections import OrderedDict

import numpy as np
import pytest

from b200grasp import bdq, dqn, learner, ppo2, sac_model, sb_io, training_state, trpo_mpi
from b200grasp.vec_env import DummyVecEnv, RunningMeanStd, VecNormalize
from oracle import bdq_ref, dqn_ref, ppo_ref, sac_ref
from tests.fake_env import FakeFlatEnv, FakeGraspEnv

HERE = os.path.dirname(os.path.abspath(__file__))
LOG = []


def _summary(v):
    """Arrays by shape and dtype and parameter sets by their size and a digest of their names (their values are checked on
    their own), paths by their file name."""
    if isinstance(v, (np.ndarray, np.generic)):
        return [list(np.shape(v)), np.asarray(v).dtype.str]
    if isinstance(v, dict) and v and all(isinstance(x, (np.ndarray, np.generic)) for x in v.values()):
        return ["params", len(v), hashlib.sha1(" ".join(v).encode()).hexdigest()[:16]]
    if isinstance(v, dict):
        return tuple((k, _summary(x)) for k, x in v.items())
    if isinstance(v, (list, tuple)):
        return tuple(_summary(x) for x in v)
    if isinstance(v, str) and os.sep in v:
        return os.path.basename(v)
    return v


class FakeLearner:
    """Keeps its parameters and device statistics in memory, logs every call with its arguments and writes a small file for
    ``save_state``.  ``specs(*args, **kwargs)`` gives the parameter table a learner of that configuration would have."""
    specs = None

    def __init__(self, *a, **k):
        self._log("__init__", *a, **k)
        self.param_shapes = OrderedDict(type(self).specs(*a, **k))
        self.params = OrderedDict((n, np.zeros(s, np.float32)) for n, s in self.param_shapes.items())
        self.obs_rms_version, self.stats = 0, None

    @staticmethod
    def _log(name, *a, **k):
        LOG.append((name, _summary(a), _summary(k)))

    def get_parameters(self):
        self._log("get_parameters")
        return OrderedDict((n, a.copy()) for n, a in self.params.items())

    def load_parameters(self, params, exact_match=True):
        self._log("load_parameters", params, exact_match=exact_match)
        for n, a in params.items():
            n = n[:-2] if n.endswith(":0") else n
            self.params[n] = np.asarray(a, np.float32).reshape(self.param_shapes[n]).copy()

    def save_state(self, path):
        self._log("save_state", path)
        with open(path, "wb") as f:
            f.write(b"fake learner state")

    def load_state(self, path):
        self._log("load_state", path)

    def set_norm_stats(self, *a, **k):
        self._log("set_norm_stats", *a, **k)

    def obs_rms_set(self, mean, var, count):
        self._log("obs_rms_set", mean, var, count)
        self.stats = (np.array(mean, np.float64), np.array(var, np.float64), float(count))
        self.obs_rms_version += 1

    def obs_rms_get(self):
        self._log("obs_rms_get")
        return self.stats[0].copy(), self.stats[1].copy(), self.stats[2]

    def close(self):
        self._log("close")


def _sac_specs(obs_shape, n_act, hidden, **_):
    return sac_ref.param_specs(sac_ref.SACConfig(obs_shape=tuple(obs_shape), n_act=n_act, layers=(hidden, hidden)))


def _bdq_cfg(obs_dim, n_br, n_bins, layers):
    return bdq_ref.BDQConfig(obs_dim, n_br, n_bins, tuple(layers[0]), layers[1][0], layers[2][0])


def _bdq_specs(obs_dim, n_br, n_bins, layers, *_, **__):
    return bdq_ref.all_specs(_bdq_cfg(obs_dim, n_br, n_bins, layers))


def _dqn_specs(obs_dim, n_actions, layers, *_, **__):
    return dqn_ref.all_specs(dqn_ref.DQNConfig(obs_dim, n_actions, tuple(layers)))


def _ppo_specs(obs_dim, n_actions, layers, *_, **__):
    return ppo_ref.param_specs(obs_dim, n_actions, tuple(layers))


def _trpo_specs(obs_dim, n_actions, layers, *_, **__):
    specs = ppo_ref.param_specs(obs_dim, n_actions, tuple(layers))
    return [(scope + n[len("model/"):], s) for scope in ("pi/model/", "oldpi/model/") for n, s in specs]


@pytest.fixture(autouse=True)
def fakes(monkeypatch):
    for mod, name, specs in ((sac_model, "Learner", _sac_specs), (bdq, "BDQLearner", _bdq_specs), (dqn, "DQNLearner", _dqn_specs),
                             (ppo2, "PPO2Learner", _ppo_specs), (trpo_mpi, "TRPOLearner", _trpo_specs)):
        monkeypatch.setattr(mod, name, type(name, (FakeLearner,), {"specs": staticmethod(specs)}))
    LOG.clear()
    yield
    LOG.clear()


def _vec(fn, norm):
    env = DummyVecEnv([fn])
    return VecNormalize(env, norm_obs=True, norm_reward=True) if norm else env


# ---- the cases: (make the model on an env, the expected initial parameters, the environment factory)
CNN_KW = {"cnn_extractor": "augmented_nature_cnn"}


def _sac(cnn, dev):
    obs_shape = (64, 64, 2) if cnn else (6,)
    env_fn = (lambda: FakeGraspEnv(seed=3, horizon=4)) if cnn else (lambda: FakeFlatEnv(seed=3, obs_dim=6, n_act=5))
    policy = sac_model.CnnPolicy if cnn else sac_model.MlpPolicy
    make = lambda env, **kw: sac_model.SAC(policy, env, buffer_size=500, batch_size=16, seed=7, learning_rate=1e-3, device_obs_norm=dev,
                                           policy_kwargs=dict(CNN_KW) if cnn else None, **kw)
    init = sac_ref.init_params(sac_ref.SACConfig(obs_shape=obs_shape, n_act=5), seed=7)
    return make, init, env_fn


def _bdq(dev):
    layers = [[16, 8], [4], [4]]
    make = lambda env, **kw: bdq.BDQ("MlpActPolicy", env, buffer_size=300, batch_size=8, seed=11, num_actions_pad=5,
                                     policy_kwargs={"layers": layers}, prioritized_replay=True, device_obs_norm=dev, **kw)
    init = bdq_ref.init_params(_bdq_cfg(6, 3, 5, layers), seed=11)
    return make, init, lambda: FakeFlatEnv(seed=4, obs_dim=6, n_act=3)


def _dqn():
    make = lambda env, **kw: dqn.DQN("MlpPolicy", env, buffer_size=200, batch_size=8, seed=13, policy_kwargs={"layers": [16, 8]}, **kw)
    init = dqn_ref.init_params(dqn_ref.DQNConfig(6, 4, (16, 8)), seed=13)
    return make, init, lambda: FakeFlatEnv(seed=5, obs_dim=6, n_discrete=4)


def _ppo():
    make = lambda env, **kw: ppo2.PPO2("MlpPolicy", env, n_steps=8, nminibatches=2, seed=17, policy_kwargs={"layers": [16, 8]}, **kw)
    init = ppo_ref.init_params(6, 3, (16, 8), rng=np.random.default_rng(17))
    return make, init, lambda: FakeFlatEnv(seed=6, obs_dim=6, n_act=3)


def _trpo():
    make = lambda env, **kw: trpo_mpi.TRPO("MlpPolicy", env, timesteps_per_batch=8, seed=19, policy_kwargs={"layers": [16, 8]}, **kw)
    rng = np.random.default_rng(19)
    init = OrderedDict((scope + n[len("model/"):], a) for scope in ("pi/model/", "oldpi/model/")
                       for n, a in ppo_ref.init_params(6, 3, (16, 8), rng=rng).items())
    return make, init, lambda: FakeFlatEnv(seed=8, obs_dim=6, n_act=3)


CASES = {"sac_mlp": lambda: _sac(False, False), "sac_mlp_dev": lambda: _sac(False, True), "sac_cnn": lambda: _sac(True, False),
         "sac_cnn_dev": lambda: _sac(True, True), "bdq": lambda: _bdq(False), "bdq_dev": lambda: _bdq(True), "dqn": _dqn, "ppo2": _ppo,
         "trpo": _trpo}


def _take_log():
    out = json.loads(json.dumps(LOG))
    LOG.clear()
    return out


def _spaces(m):
    return [[type(s).__name__, list(s.shape)] for s in (m.observation_space, m.action_space)]


def _assert_params(got, want):
    assert list(got) == list(want)
    for n in want:
        np.testing.assert_array_equal(np.asarray(got[n], np.float32).reshape(np.shape(want[n])), want[n], err_msg=n)


def _zip_entries(path):
    with zipfile.ZipFile(path) as z:
        data, names = json.loads(z.read("data")), json.loads(z.read("parameter_list"))
        arrs = np.load(io.BytesIO(z.read("parameters")))
        return data, names, OrderedDict((n[:-2], arrs[n]) for n in names)


def _advance_host_state(m):
    """Moves every counter and generator the algorithm keeps on the host away from its initial value."""
    m.num_timesteps = 40
    if isinstance(m, sac_model.SAC):
        m.n_updates, m.episode_rewards = 3, [0.0, 1.5]
        m.ep_info_buf.append({"r": 1.5})
    if isinstance(m, dqn.DQN):
        m.n_target_updates = 2
        m.predict_rng.random(4)
    if isinstance(m, (ppo2.PPO2, trpo_mpi.TRPO)):
        np.random.seed(23)
        m._boundary = (40, np.random.get_state())
        np.random.random(5)
    if hasattr(m, "_rng"):
        m._rng.random(3)


def _host_counters(m):
    out = {"num_timesteps": m.num_timesteps}
    if isinstance(m, sac_model.SAC):
        out.update(n_updates=m.n_updates, episode_rewards=m.episode_rewards, ep_info_buf=list(m.ep_info_buf))
    if isinstance(m, dqn.DQN):
        out.update(n_target_updates=m.n_target_updates, predict_rng=m.predict_rng.bit_generator.state)
    if isinstance(m, (ppo2.PPO2, trpo_mpi.TRPO)):
        out.update(boundary=[m._boundary[0], np.asarray(m._boundary[1][1]).tolist()])
    if hasattr(m, "_rng"):
        out["rng"] = m._rng.bit_generator.state
    return json.loads(json.dumps(out))


_REPLAY = ("gamma", "learning_rate", "batch_size", "buffer_size", "policy_kwargs", "seed")
HYPER = {"SAC": _REPLAY + ("tau", "n_envs", "device_obs_norm"), "BDQ": _REPLAY + ("num_actions_pad", "device_obs_norm"),
         "DQN": _REPLAY + ("target_network_update_freq",),
         "PPO2": ("gamma", "learning_rate", "n_steps", "nminibatches", "cliprange_vf", "policy_kwargs", "seed", "n_envs"),
         "TRPO": ("gamma", "timesteps_per_batch", "max_kl", "vf_stepsize", "vf_iters", "policy_kwargs", "seed", "n_envs")}


def run_case(case, norm, tmp):
    """Drives one front end through construction, save, training state, load and close; checks the values that must be
    bit-exact and returns a JSON-able record of everything else."""
    make, init, env_fn = CASES[case]()
    rec = {}
    m = make(_vec(env_fn, norm))
    rec["construct"] = _take_log()
    _assert_params(m.learner.params, init)
    _assert_params(OrderedDict((n[:-2], a) for n, a in m.get_parameters().items()), init)
    rec["get_parameters"] = _take_log()

    m.save(os.path.join(tmp, "sub", "m.zip"))
    rec["save"] = _take_log()
    rec["data"], names, arrs = _zip_entries(os.path.join(tmp, "sub", "m.zip"))
    assert names == [n + ":0" for n in init]
    _assert_params(arrs, init)

    _advance_host_state(m)
    counters = _host_counters(m)
    d = m.save_training_state(os.path.join(tmp, "ts"))
    rec["save_training_state"] = _take_log()
    assert sorted(os.listdir(d)) == sorted(["host.json", "learner.state", "model.zip"] + (["vecnormalize.pkl"] if norm else []))
    host = training_state.read_host(d)
    rec["host"] = {k: v for k, v in host.items() if k not in ("rng", "predict_rng", "np_random")}
    if isinstance(m, (ppo2.PPO2, trpo_mpi.TRPO)):
        np.random.seed(99)                         # the load must put numpy's generator back
    env2 = _vec(env_fn, norm)
    m2 = type(m).load_training_state(d, env2)
    rec["load_training_state"] = _take_log()
    assert _host_counters(m2) == counters
    if isinstance(m, (ppo2.PPO2, trpo_mpi.TRPO)):
        np.testing.assert_array_equal(np.random.get_state()[1], m._boundary[1][1])
    assert m2.get_env() is env2 and m2.get_vec_normalize_env() is (env2 if norm else None)
    if norm:
        vn, vn2 = m.get_vec_normalize_env(), env2
        np.testing.assert_array_equal(vn2.obs_rms.mean, vn.obs_rms.mean)
        assert vn2.ret_rms.count == vn.ret_rms.count
    other = sac_model.SAC if not isinstance(m, sac_model.SAC) else dqn.DQN
    with pytest.raises(ValueError, match=f"holds a {host['algo']} training state"):
        other.load_training_state(d, _vec(env_fn, norm))
    LOG.clear()

    for with_env in (False, True):
        env3 = _vec(env_fn, norm) if with_env else None
        m3 = type(m).load(os.path.join(tmp, "sub", "m"), env=env3)          # the ".zip" is added
        rec[f"load_env{int(with_env)}"] = {"log": _take_log(), "spaces": _spaces(m3), "env": m3.get_env() is env3,
                                           "vn": m3.get_vec_normalize_env() is (env3 if norm else None),
                                           "hyper": json.loads(json.dumps({k: getattr(m3, k) for k in HYPER[host["algo"]]}))}
        _assert_params(m3.learner.params, init)

    owned = m._owns_obs_rms() if hasattr(m, "_owns_obs_rms") else False
    m.close()
    rec["close"] = _take_log()
    assert m.learner is None
    if owned:                                      # the statistics went back to the wrapper
        vn = m.get_vec_normalize_env()
        assert not vn.learner_owns_obs_rms and type(vn.obs_rms) is RunningMeanStd
    rec["owned"] = owned
    return json.loads(json.dumps(rec))


RUNS = [(c, n) for c in CASES for n in ((True,) if c.endswith("_dev") else (False, True))]
with open(os.path.join(HERE, "model_base_expected.json")) as _f:
    EXPECTED = json.load(_f)


@pytest.mark.parametrize("case,norm", RUNS, ids=[f"{c}-{'vecnorm' if n else 'bare'}" for c, n in RUNS])
def test_front_end_record(case, norm, tmp_path):
    assert run_case(case, norm, str(tmp_path)) == EXPECTED[f"{case}-{norm}"]


def test_dqn_and_ppo2_env_refusals():
    flat = lambda **kw: (lambda: FakeFlatEnv(obs_dim=6, **kw))
    with pytest.raises(ValueError, match="DQN cannot be used with more than one environment"):
        dqn.DQN("MlpPolicy", DummyVecEnv([flat(n_discrete=4)] * 2))
    with pytest.raises(NotImplementedError, match="PPO2 here needs a Box action space"):
        ppo2.PPO2("MlpPolicy", DummyVecEnv([flat(n_discrete=4)]))
    with pytest.raises(ValueError, match="nminibatches=3 is not a factor of n_batch = n_envs \\* n_steps = 16"):
        ppo2.PPO2("MlpPolicy", DummyVecEnv([flat()] * 2), n_steps=8, nminibatches=3)
    assert LOG == []


def test_golden_dqn_zip_goes_through_load_and_save_unchanged(tmp_path):
    golden = os.path.join(HERE, "golden", "DQN_simple_4pads.zip")
    _, params = sb_io.load_sb_zip(golden)
    m = dqn.DQN.load(golden[:-4])
    _assert_params(m.learner.params, params)
    m.save(str(tmp_path / "again.zip"))
    data, names, arrs = _zip_entries(str(tmp_path / "again.zip"))
    with zipfile.ZipFile(golden) as z:
        assert names == json.loads(z.read("parameter_list"))
    _assert_params(arrs, params)
    assert data == EXPECTED["golden_dqn_data"]


# ---- the handle wrappers on a stub library: what they check before and after calling it
class StubLib:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*a):
            self.calls.append(name)
            return 0
        return fn


def _stub(cls, shapes, **attrs):
    L = cls.__new__(cls)
    L.lib, L.h, L._info = StubLib(), None, OrderedDict(shapes)
    for k, v in attrs.items():
        setattr(L, k, v)
    return L


STUBS = {"sac": (learner.Learner,), "bdq": (bdq.BDQLearner,), "dqn": (dqn.DQNLearner,), "ppo": (ppo2.PPO2Learner,),
         "trpo": (trpo_mpi.TRPOLearner,)}   # before any patching


@pytest.mark.parametrize("abi", list(STUBS))
def test_load_parameters_refusals(abi):
    L = _stub(STUBS[abi][0], [("a/w", (2, 3)), ("a/b", (3,)), ("b/w", (3, 1)), ("b/b", (1,)), ("c", ())])
    full = {n: np.zeros(s, np.float32) for n, s in L._info.items()}
    L.load_parameters(dict(full, **{"a/w:0": full.pop("a/w")}))
    set_param = L.lib.calls[-1]
    assert set_param == ("b2g_set_param" if abi == "sac" else f"b2g_{abi}_set_param") and len(L.lib.calls) == 5
    with pytest.raises(ValueError, match="unknown variable zz"):
        L.load_parameters(dict(full, zz=np.zeros(1)))
    L.load_parameters(dict(full, zz=np.zeros(1)), exact_match=False)
    with pytest.raises(ValueError, match=r"shape mismatch for a/b: \(4,\) vs \(3,\)"):
        L.load_parameters(dict(full, **{"a/b": np.zeros(4)}))
    with pytest.raises(ValueError, match=r"missing variables: \['a/w', 'b/b', 'b/w', 'c'\]$"):
        L.load_parameters({"a/b": full["a/b"]})


@pytest.mark.parametrize("abi", ["sac", "bdq"])
def test_set_norm_stats_moves_obs_rms_version_when_it_passes_statistics(abi):
    L = _stub(STUBS[abi][0], [], obs_elems=4, obs_dim=4, obs_shape=(4,))
    v0 = L.obs_rms_version
    L.set_norm_stats(None, None, 2.0)                          # the scalars only: the device statistics stay
    assert L.obs_rms_version == v0
    L.set_norm_stats(np.zeros(4), np.ones(4), 2.0)
    assert L.obs_rms_version == v0 + 1
    L.set_norm_stats(np.zeros(4), np.ones(4), norm_obs=False)
    assert L.obs_rms_version == v0 + 1
    with pytest.raises(AssertionError):
        L.set_norm_stats(np.zeros(5), np.ones(5))
    assert L.lib.calls == ["b2g_set_norm_stats" if abi == "sac" else "b2g_bdq_set_norm_stats"] * 3
