"""CPU side of ``DQN(device_obs_norm=True)``: the Philox stream-3 restatement of the epsilon-greedy actor at one branch, the C
ABI, what the device branch of ``learn`` asks of its learner (a stand-in learner), the records, and the sm_90a compile of
csrc/dqn.cu without spills."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from b200grasp import _lib, dqn
from b200grasp.vec_env import DummyVecEnv, RunningMeanStd, VecNormalize
from oracle import philox_ref as PX
from tests.fake_env import FakeFlatEnv
from tests.test_bdq_obs_norm_cpu import explore

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["b2g_dqn_" + n for n in ("observe_act", "observe_add", "act_raw", "obs_rms_set", "obs_rms_get", "upload_bytes", "set_obs_encoder")]
OBS, NA = 5, 4


def explore_dqn(key, step, n_env, n_actions, eps):
    """Stream 3 of one acting b2g_dqn_observe_act call (csrc/dqn.cu dqn_explore_kernel): BDQ's rule with one branch, block = env
    row -> (explore [n_env] bool, random action [n_env] int64)."""
    go, act = explore(key, step, n_env, 1, n_actions, eps)
    return go[:, 0], act[:, 0]


def test_stream3_at_one_branch():
    key, step = PX.train_seed(2), (1 << 32) + 5
    go, act = explore_dqn(key, step, 6, NA, 0.4)
    for e in range(6):
        r = PX.philox4x32_10(step & 0xFFFFFFFF, step >> 32, e, 3, key & 0xFFFFFFFF, key >> 32)
        assert go[e] == ((int(r[0]) + 0.5) / 2 ** 32 < float(np.float32(0.4)))
        assert act[e] == (int(r[1]) * NA) >> 32
    assert not explore_dqn(key, step, 64, NA, 0.0)[0].any() and explore_dqn(key, step, 64, NA, 1.0)[0].all()


def test_stream3_is_uniform_and_independent_at_one_branch():
    """2^18 env draws over 16 acting calls: the exploration rate is eps within 5 sigma, the actions pass a chi-square test at
    n_actions = 12 (the shipped zip), and the decision correlates neither with the action nor with the next env's decision."""
    from scipy import stats
    key, eps = PX.train_seed(6), 0.3
    go, act = zip(*[explore_dqn(key, s, 1 << 14, 12, eps) for s in range(16)])
    go, act = np.concatenate(go), np.concatenate(act)
    n = go.size
    assert n == 1 << 18
    assert abs(go.mean() - eps) <= 5 * np.sqrt(eps * (1 - eps) / n), go.mean()
    assert act.min() == 0 and act.max() == 11
    chi = stats.chisquare(np.bincount(act, minlength=12))
    assert chi.pvalue > 1e-4, chi
    for a, b in ((go.astype(float), act.astype(float)), (go[:-1].astype(float), go[1:].astype(float))):
        rho = np.corrcoef(a, b)[0, 1]
        assert abs(rho) <= 5 / np.sqrt(n), rho


def test_abi_is_declared_and_exported():
    header = open(os.path.join(ROOT, "include", "b200grasp.h")).read()
    for s in NEW:
        assert s in _lib.SYMBOLS and f"int {s}(" in header, s
    if os.path.exists(_lib.LIB_PATH):
        lib = _lib.load()
        assert all(hasattr(lib, s) for s in NEW)


class StubDQNLearner:
    """Records the learner calls of both branches of DQN.learn; the greedy action is always 0."""

    def __init__(self, obs_dim, n_actions, *a, **k):
        self.obs_dim, self.n_actions, self.batch_size = int(obs_dim), int(n_actions), int(a[1])
        self.param_shapes = {}
        self.log, self.obs_rms_version, self.rms, self.size = [], 0, None, 0
        self.raw_obs_elems = None

    def load_parameters(self, params, exact_match=True):
        pass

    def obs_rms_set(self, mean, var, count):
        self.rms = RunningMeanStd(shape=np.shape(mean))
        self.rms.mean, self.rms.var, self.rms.count = np.array(mean, np.float64), np.array(var, np.float64), float(count)
        self.obs_rms_version += 1
        self.log.append(("obs_rms_set",))

    def obs_rms_get(self):
        return self.rms.mean.copy(), self.rms.var.copy(), self.rms.count

    def set_norm_stats(self, obs_mean=None, obs_var=None, *a, **k):
        self.log.append(("set_norm_stats", obs_mean is None))

    def observe_act(self, obs, n=None, update_stats=True, eps=0.0, act=True):
        self.log.append(("observe_act", None if obs is None else np.array(obs, np.float32), bool(update_stats), bool(act)))
        if obs is not None and update_stats:
            self.rms.update(np.asarray(obs, np.float64).reshape(1, -1))
            self.obs_rms_version += 1
        return np.zeros(1, np.int32) if act else None

    def observe_add(self, act, rew, next_obs, done, reset_obs=None, update_stats=True):
        self.log.append(("observe_add", np.array(next_obs, np.float32).reshape(-1), float(np.reshape(done, -1)[0]),
                         None if reset_obs is None else np.array(reset_obs, np.float32).reshape(-1), bool(update_stats)))
        if update_stats:
            self.rms.update(np.asarray(reset_obs if reset_obs is not None else next_obs, np.float64).reshape(1, -1))
            self.obs_rms_version += 1
        self.size += 1

    def act(self, obs, with_q=False):
        raise AssertionError("the device branch acts through observe_act")

    def replay_add(self, *a):
        raise AssertionError("the device branch stores through observe_add")

    def replay_size(self):
        return self.size

    def set_per_beta(self, beta):
        self.log.append(("set_per_beta",))

    def step(self, n=1, lr=5e-4):
        self.log.append(("step",))
        return {}

    def update_target(self):
        self.log.append(("update_target",))

    def set_eps(self, eps):
        pass

    def close(self):
        pass


class Recorder(DummyVecEnv):
    """A DummyVecEnv that keeps what reset / step_wait return (raw frames and infos)."""

    def __init__(self, fns):
        super().__init__(fns)
        self.resets, self.steps = [], []

    def reset(self):
        o = super().reset()
        self.resets.append(np.array(o, copy=True))
        return o

    def step_wait(self):
        o, r, d, infos = super().step_wait()
        self.steps.append((np.array(o, copy=True), np.array(d, copy=True), [dict(i) for i in infos]))
        return o, r, d, infos


def _model(monkeypatch, wrap=True, training=True, **kw):
    monkeypatch.setattr(dqn, "DQNLearner", StubDQNLearner)
    rec = Recorder([lambda: FakeFlatEnv(seed=1, horizon=3, obs_dim=OBS, n_discrete=NA)])
    env = VecNormalize(rec, training=training) if wrap else rec
    args = dict(buffer_size=64, batch_size=4, learning_starts=4, seed=7, device_obs_norm=True, prioritized_replay=True)
    args.update(kw)
    return dqn.DQN("MlpPolicy", env, **args), env, rec


@pytest.mark.parametrize("training", [True, False])
def test_device_branch_with_vecnormalize_stores_the_original_obs(training, monkeypatch):
    """next_obs is get_original_obs(): a finished env's reset frame, as stable-baselines' DQN stores it; reset_obs goes with
    a finished env only; update_stats follows vn.training; the reward scalars are synced before every step."""
    m, vn, rec = _model(monkeypatch, training=training)
    L = m.learner
    assert vn.obs_rms_owner is L and m.predict_takes_raw_obs
    assert L.log == [("obs_rms_set",), ("set_norm_stats", True)]
    L.log.clear()
    m.learn(10)
    obs_calls = [c for c in L.log if c[0] == "observe_act"]
    adds = [c for c in L.log if c[0] == "observe_add"]
    assert len(obs_calls) == 11 and len(adds) == 10 == len(rec.steps)
    first = obs_calls[0]
    assert np.array_equal(first[1], rec.resets[0].reshape(1, -1)) and first[2] == training and not first[3]
    assert all(c[1] is None and c[3] for c in obs_calls[1:])
    n_done = 0
    for (o, d, infos), (_, nxt, done, reset, upd) in zip(rec.steps, adds):
        assert np.array_equal(nxt, o[0]) and done == float(d[0]) and upd == training
        if d[0]:
            n_done += 1
            assert np.array_equal(reset, o[0]) and not np.array_equal(nxt, infos[0]["terminal_observation"])
        else:
            assert reset is None
    assert n_done == 3
    steps = [i for i, c in enumerate(L.log) if c[0] == "step"]
    assert steps and all(L.log[i - 1] == ("set_norm_stats", True) for i in steps)
    assert vn.obs_rms.count == pytest.approx(1e-4 + (11 if training else 0))


def test_device_branch_without_vecnormalize_stores_the_terminal_frame(monkeypatch):
    m, env, rec = _model(monkeypatch, wrap=False)
    L = m.learner
    m.learn(7)
    adds = [c for c in L.log if c[0] == "observe_add"]
    assert [c for c in L.log if c[0] == "observe_act"][0][2] is False
    n_done = 0
    for (o, d, infos), (_, nxt, done, reset, upd) in zip(rec.steps, adds):
        assert not upd and done == float(d[0])
        if d[0]:
            n_done += 1
            assert np.array_equal(nxt, infos[0]["terminal_observation"]) and np.array_equal(reset, o[0])
        else:
            assert np.array_equal(nxt, o[0]) and reset is None
    assert n_done == 2
    assert not any(c[0] == "set_norm_stats" for c in L.log)


def test_records_and_refusals(monkeypatch):
    m, vn, _ = _model(monkeypatch)
    assert m._host_state()["init"]["device_obs_norm"] is True
    m.device_obs_norm = False
    assert "device_obs_norm" not in m._host_state()["init"]
    # a second model on the owned wrapper reads the owner's statistics and refuses to learn
    other = dqn.DQN("MlpPolicy", vn, buffer_size=64, batch_size=4, device_obs_norm=True)
    assert vn.obs_rms_owner is m.learner
    with pytest.raises(RuntimeError, match="owned by another"):
        other.learn(3)
    m.close()
    assert not vn.learner_owns_obs_rms
    m2, _, _ = _model(monkeypatch, wrap=False)
    m2.env = VecNormalize(m2.env, norm_obs=False)
    m2._vec_normalize_env = m2.env
    with pytest.raises(RuntimeError, match="norm_obs"):
        m2.learn(3)


def test_default_learn_keeps_its_calls(monkeypatch):
    """Without the keyword the host branch runs: act + replay_add per step, never the observe path."""
    m, vn, _ = _model(monkeypatch, device_obs_norm=False)
    assert not vn.learner_owns_obs_rms and not m.predict_takes_raw_obs
    calls = []
    m.learner.act = lambda obs, with_q=False: calls.append("act") or np.zeros(1, np.int32)
    m.learner.replay_add = lambda *a: calls.append("replay_add") or setattr(m.learner, "size", m.learner.size + 1)
    m.learn(5)
    assert calls == ["act", "replay_add"] * 5
    assert not any(c[0].startswith("observe") for c in m.learner.log)


def test_dqn_kernels_compile_for_sm90a_without_spills(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not shutil.which(nvcc):
        pytest.skip("nvcc not found")
    src = os.path.join(ROOT, "deep-rl-grasping_b200", "csrc", "dqn.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-Xptxas", "-v",
                        "-c", src, "-o", str(tmp_path / "dqn.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert "dqn_explore_kernel" in r.stderr
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert spills and all(a == "0" and b == "0" for a, b in spills), r.stderr
