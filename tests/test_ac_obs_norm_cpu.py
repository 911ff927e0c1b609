"""CPU side of PPO2 / TRPO ``device_obs_norm=True``: the C ABI, the zip / host.json records, the CLI mapping, what ``learn`` asks
of its learner on the device path (a stand-in learner), and the sm_90a compile of the observe kernel without spills."""
import inspect
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from b200grasp import _lib, ppo2, train_cli, trpo_mpi
from b200grasp.vec_env import DummyVecEnv, RunningMeanStd, VecNormalize
from tests.fake_env import FakeFlatEnv

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = [f"b2g_{p}_{n}" for p in ("ppo", "trpo")
       for n in ("obs_rms_set", "obs_rms_get", "upload_bytes", "set_norm_stats", "set_obs_encoder", "observe_act", "act_raw")]


def test_abi_is_declared_and_exported():
    header = open(os.path.join(ROOT, "include", "b200grasp.h")).read()
    for s in NEW:
        assert s in _lib.SYMBOLS and f"int {s}(" in header, s
    if os.path.exists(_lib.LIB_PATH):
        lib = _lib.load()
        assert all(hasattr(lib, s) for s in NEW)


class StubLearner:
    """Records the learner calls of the device path; observe_act answers from the staged frames alone."""

    def __init__(self, obs_dim, n_actions, *a, **k):
        self.obs_dim, self.n_actions = int(obs_dim), int(n_actions)
        self.n_envs = int(a[1]) if len(a) > 1 and isinstance(self, StubPPO) else 1
        self.log, self.obs_rms_version, self.staged = [], 0, None
        self.rms = None

    def load_parameters(self, params, exact_match=True):
        self.log.append(("load_parameters",))

    def obs_rms_set(self, mean, var, count):
        self.rms = RunningMeanStd(shape=np.shape(mean))
        self.rms.mean, self.rms.var, self.rms.count = np.array(mean, np.float64), np.array(var, np.float64), float(count)
        self.obs_rms_version += 1
        self.log.append(("obs_rms_set",))

    def obs_rms_get(self):
        return self.rms.mean.copy(), self.rms.var.copy(), self.rms.count

    def set_norm_stats(self, clip_obs=10.0, epsilon=1e-8, norm_obs=True):
        self.log.append(("set_norm_stats", clip_obs, epsilon, norm_obs))

    def rollout_reset(self):
        self.log.append(("rollout_reset",))

    def observe_act(self, obs, update_stats=True, act=True):
        self.log.append(("observe_act", obs is not None, bool(update_stats), bool(act)))
        if obs is not None:
            obs = np.asarray(obs, np.float64).reshape(self.n_envs, -1)
            if update_stats:
                self.rms.update(obs)
                self.obs_rms_version += 1
            self.staged = obs
        return np.tile(self.staged[:, :1], (1, self.n_actions)).astype(np.float32) if act else None

    def rollout_act(self, obs):
        raise AssertionError("the device path observes; it does not upload observations through rollout_act")

    def rollout_reward(self, rew, done):
        self.log.append(("rollout_reward",))

    def update(self, last_obs, perms, *hyper):
        self.log.append(("update", last_obs is None))
        return {"policy_loss": 0.0, "value_loss": 0.0, "entropy": 0.0, "approxkl": 0.0, "clipfrac": 0.0, "optimgain": 0.0,
                "meankl": 0.0, "vf_loss": 0.0}

    def act(self, obs, deterministic=True, raw=False):
        self.log.append(("act", bool(raw)))
        a = np.zeros((np.asarray(obs).reshape(-1, self.obs_dim).shape[0], self.n_actions), np.float32)
        return (a, a[:, 0], a[:, 0]) if isinstance(self, StubPPO) else (a, a[:, 0])

    def close(self):
        pass


class StubPPO(StubLearner):
    pass


def _model(algo, monkeypatch, training=True, **kw):
    n_env = 2 if algo == "ppo2" else 1
    venv = DummyVecEnv([lambda s=s: FakeFlatEnv(seed=s, horizon=3, obs_dim=5, n_act=2) for s in range(n_env)])
    vn = VecNormalize(venv, training=training)
    if algo == "ppo2":
        monkeypatch.setattr(ppo2, "PPO2Learner", StubPPO)
        return ppo2.PPO2("MlpPolicy", vn, n_steps=3, nminibatches=1, noptepochs=1, seed=3, device_obs_norm=True, **kw), vn
    monkeypatch.setattr(trpo_mpi, "TRPOLearner", StubLearner)
    return trpo_mpi.TRPO("MlpPolicy", vn, timesteps_per_batch=3, vf_iters=0, seed=3, device_obs_norm=True, **kw), vn


@pytest.mark.parametrize("algo", ["ppo2", "trpo"])
@pytest.mark.parametrize("training", [True, False])
def test_learn_observes_each_frame_once(algo, training, monkeypatch):
    m, vn = _model(algo, monkeypatch, training=training)
    L = m.learner
    assert vn.learner_owns_obs_rms and vn.obs_rms_owner is L and m.predict_takes_raw_obs
    assert L.log[:3] == [("load_parameters",), ("obs_rms_set",), ("set_norm_stats", 10.0, 1e-8, True)]
    L.log.clear()
    m.learn(6 * m.n_envs)                  # two rollouts of 3 steps
    t = training
    step = [("observe_act", False, True, True), ("observe_act", True, t, False), ("rollout_reward",)]
    rollout = step * 3 + [("update", True)]
    assert L.log == [("rollout_reset",), ("set_norm_stats", 10.0, 1e-8, True), ("observe_act", True, t, False)] + rollout * 2
    n_env = m.n_envs
    assert vn.obs_rms.count == pytest.approx(1e-4 + (7 * n_env if training else 0))


@pytest.mark.parametrize("algo", ["ppo2", "trpo"])
def test_callback_sees_the_merged_statistics(algo, monkeypatch):
    m, vn = _model(algo, monkeypatch)
    seen = []
    m.learn(3 * m.n_envs, callback=lambda _l, _g: seen.append(vn.obs_rms.count) or True)
    n = m.n_envs
    assert seen == [pytest.approx(1e-4 + n * k) for k in (2, 3, 4)]          # reset frames, then one merge per step


@pytest.mark.parametrize("algo", ["ppo2", "trpo"])
def test_predict_normalises_raw_observations(algo, monkeypatch):
    m, vn = _model(algo, monkeypatch)
    m.learner.log.clear()
    m.predict(np.zeros(5, np.float32))
    assert m.learner.log == [("set_norm_stats", 10.0, 1e-8, True), ("act", True)]
    # a second model on the owned wrapper: normalised by the wrapper from the owner's statistics, then today's predict
    cls = ppo2.PPO2 if algo == "ppo2" else trpo_mpi.TRPO
    kw = dict(n_steps=3, nminibatches=1) if algo == "ppo2" else dict(timesteps_per_batch=3)
    other = cls("MlpPolicy", vn, device_obs_norm=True, **kw)
    assert vn.obs_rms_owner is m.learner and other.predict_takes_raw_obs
    other.learner.log.clear()
    other.predict(np.zeros(5, np.float32))
    assert other.learner.log == [("act", False)]
    with pytest.raises(RuntimeError, match="owned by another model"):
        other.learn(3)
    m.close()
    assert not vn.learner_owns_obs_rms


@pytest.mark.parametrize("algo", ["ppo2", "trpo"])
def test_records_and_refusals(algo, monkeypatch):
    m, vn = _model(algo, monkeypatch)
    assert m._data()["device_obs_norm"] is True and m._host_state()["init"]["device_obs_norm"] is True
    m.device_obs_norm = False
    assert "device_obs_norm" not in m._data() and "device_obs_norm" not in m._host_state()["init"]
    cls = ppo2.PPO2 if algo == "ppo2" else trpo_mpi.TRPO
    # the keyword takes over a VecNormalize's observation statistics: without one that normalises observations (or without
    # an env) it is refused before a learner exists
    venv = DummyVecEnv([lambda: FakeFlatEnv(seed=0, horizon=3, obs_dim=5, n_act=2)])
    kw = dict(n_steps=3, nminibatches=1) if algo == "ppo2" else dict(timesteps_per_batch=3)
    for env in (None, venv, VecNormalize(venv, norm_obs=False)):
        with pytest.raises(NotImplementedError, match="device_obs_norm"):
            cls("MlpPolicy", env, device_obs_norm=True, **kw)
    assert cls("MlpPolicy", VecNormalize(venv), device_obs_norm=True, _init_setup_model=False, **kw).device_obs_norm


@pytest.mark.parametrize("algo", ["ppo2", "trpo"])
def test_load_restores_the_keyword_where_a_wrapper_normalises(algo, monkeypatch):
    from b200grasp import actor_critic
    m, _ = _model(algo, monkeypatch)
    cls = type(m)
    data = dict(m._data(), device_obs_norm=True)
    params = actor_critic.init_params(5, 2, [64, 64], 0, scope=cls._scope)
    if algo == "trpo":
        params.update(actor_critic.init_params(5, 2, [64, 64], 0, scope="oldpi/model/"))
    monkeypatch.setattr(cls, "_read_zip", staticmethod(lambda path: (data, params)))

    def env(**k):
        return DummyVecEnv([lambda s=s: FakeFlatEnv(seed=s, horizon=3, obs_dim=5, n_act=2) for s in range(m.n_envs)])
    on = cls.load("zip", VecNormalize(env()))
    assert on.device_obs_norm and on.get_vec_normalize_env().obs_rms_owner is on.learner
    assert not cls.load("zip").device_obs_norm                      # no env: a plain model for predict / get_parameters
    assert not cls.load("zip", env()).device_obs_norm               # an env without VecNormalize: the zip's parameters only
    assert not cls.load("zip", VecNormalize(env()), device_obs_norm=False).device_obs_norm
    with pytest.raises(NotImplementedError, match="device_obs_norm"):
        cls.load("zip", env(), device_obs_norm=True)


def test_cli_passes_device_norm_to_ppo_and_trpo():
    src = inspect.getsource(train_cli.train)
    for cls in ("PPO2(", "TRPO("):
        line = next(l for l in src.splitlines() if f"model = {cls}" in l)
        assert "device_obs_norm=bool(args.device_norm)" in line, line
    assert "--device_norm is built for SAC, BDQ, PPO and TRPO only" in src          # DQN still refuses the flag
    p = train_cli.build_parser()
    for algo in ("PPO", "TRPO"):
        assert p.parse_args(["train", "--config", "c.yaml", "--algo", algo, "--model_dir", "m", "--device_norm"]).device_norm


@pytest.mark.parametrize("algo", ["PPO", "TRPO"])
def test_cli_device_norm_needs_normalize(algo, tmp_path):
    import yaml
    cfg = {"discount_factor": 0.9, "normalize": False, "robot": {}, "reward": {},
           algo: {"learning_rate": 3e-4, "max_iters": 400, "step_size": 0.001, "total_timesteps": 10}}
    (tmp_path / "c.yaml").write_text(yaml.safe_dump(cfg))
    d = tmp_path / "run"
    with pytest.raises(NotImplementedError, match="normalize"):
        train_cli.main(["train", "--config", str(tmp_path / "c.yaml"), "--algo", algo, "--model_dir", str(d), "--device_norm",
                        "--env", "tests.fake_env:make_env"])
    assert not d.exists()


def test_observe_kernel_compiles_for_sm90a_without_spills(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not shutil.which(nvcc):
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "deep-rl-grasping_b200", "csrc", "actor_critic.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-Xptxas", "-v",
                        "-c", src, "-o", str(tmp_path / "actor_critic.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert "ac_obs_norm_kernel" in r.stderr
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert spills and all(a == "0" and b == "0" for a, b in spills), r.stderr
