"""The DQN surface without a GPU: the float64 oracle (oracle/dqn_ref.py) against the shipped zip and stable-baselines' formulas,
the imports and refusals of b200grasp.deepq.DQN, the CLI's DQN branch and its training-state host file."""
import json
import os

import numpy as np
import pytest
import torch
import yaml

import b200grasp as sb
from b200grasp import _lib, sb_io, train_cli, training_state
from b200grasp.vec_env import DummyVecEnv
from oracle import dqn_ref as DR

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ZIP = os.path.join(GOLD, "DQN_simple_4pads.zip")


def test_oracle_specs_match_the_shipped_zip():
    data, params = sb_io.load_sb_zip(ZIP)
    cfg = DR.DQNConfig(100, 12, (64, 64), 1.0)
    specs = DR.all_specs(cfg)
    assert [n for n, _ in specs] == list(params)                  # names and order (parameter_list)
    for n, shp in specs:
        assert params[n].shape == tuple(shp) and params[n].dtype == np.float32, n
    for k, v in DR.ZIP_DATA.items():
        assert data[k] == v, (k, data[k], v)
    assert "buffer_size" not in data
    assert "Discrete" in data["action_space"][":type:"] and "Box" in data["observation_space"][":type:"]


def test_oracle_huber_gradient_is_the_clipped_td():
    rng = np.random.default_rng(0)
    td = torch.tensor(np.concatenate([rng.uniform(-3, 3, 40), [1.0, -1.0, 0.0, 0.999, -1.001]]), requires_grad=True)
    w = torch.tensor(rng.uniform(0.2, 1.5, td.numel()))
    loss = (w * DR.huber(td)).mean()
    g, = torch.autograd.grad(loss, td)
    want = w.numpy() * np.clip(td.detach().numpy(), -1.0, 1.0) / td.numel()
    assert np.allclose(g.numpy(), want, rtol=1e-12, atol=1e-15)
    x = td.detach().numpy()
    assert np.allclose(DR.huber(td).detach().numpy(), np.where(np.abs(x) < 1, 0.5 * x * x, np.abs(x) - 0.5))


def test_oracle_clips_each_tensor_on_its_own():
    cfg = DR.DQNConfig(7, 5, (8, 12), 0.99)
    p = DR.init_params(cfg, seed=3)
    rng = np.random.default_rng(4)
    B = 9
    batch = dict(obs=rng.normal(size=(B, 7)) * 60, next_obs=rng.normal(size=(B, 7)), act=rng.integers(0, 5, B),
                 rew=rng.choice([0.0, 400.0], B), done=(rng.random(B) < 0.3).astype(float), weights=rng.uniform(0.5, 1.5, B))
    out, g, _, _ = DR.dqn_step(p, {"t": 0, "m": {}, "v": {}}, batch, 1e-3, cfg)
    assert 0 < out["n_clipped"] < len(g)                           # some tensors scaled, others not
    for n, pre in out["grads_pre"].items():
        norm = np.sqrt((pre ** 2).sum())
        assert np.isclose(out["norms"][n], norm)
        assert np.allclose(g[n], pre * DR.GRAD_CLIP / max(norm, DR.GRAD_CLIP), rtol=1e-13, atol=0)
        assert np.sqrt((g[n] ** 2).sum()) <= DR.GRAD_CLIP * (1 + 1e-12)
    assert np.isclose(out["grad_norm"], np.sqrt(sum(v ** 2 for v in out["norms"].values())))
    assert np.allclose(out["priorities"], np.abs(out["td"]) + 1e-6)


def test_deepq_imports_and_top_level_name_still_refuses():
    from b200grasp.deepq import DQN, DQNLearner  # noqa: F401
    from b200grasp.deepq.policies import MlpPolicy  # noqa: F401
    assert sb.deepq.DQN is DQN
    with pytest.raises(NotImplementedError, match="deepq.DQN"):
        sb.DQN
    for name in ("b2g_dqn_create", "b2g_dqn_step", "b2g_dqn_update_target", "b2g_dqn_act", "b2g_dqn_state_save"):
        assert name in _lib.SYMBOLS


class _Env:
    def __init__(self):
        self.observation_space = sb.spaces.Box(-1.0, 1.0, (6,))
        self.action_space = sb.spaces.Discrete(3)

    def reset(self):
        return np.zeros(6, np.float32)

    def step(self, a):
        return np.zeros(6, np.float32), 0.0, False, {}

    def close(self):
        pass


@pytest.mark.parametrize("kw,exc,msg", [
    (dict(double_q=False), NotImplementedError, "double_q"),
    (dict(param_noise=True), NotImplementedError, "param_noise"),
    (dict(policy_kwargs={"dueling": False}), NotImplementedError, "dueling"),
    (dict(policy_kwargs={"layer_norm": True}), NotImplementedError, "layer_norm"),
    (dict(policy_kwargs={"layers": [64]}), NotImplementedError, "two hidden layers"),
    (dict(policy_kwargs={"layers": [64, 64, 64]}), NotImplementedError, "two hidden layers"),
])
def test_keywords_that_select_unbuilt_code_fail_loudly(kw, exc, msg):
    with pytest.raises(exc, match=msg):
        sb.deepq.DQN("MlpPolicy", None, **kw)


def test_more_than_one_environment_is_refused():
    env = DummyVecEnv([_Env, _Env])
    with pytest.raises(ValueError, match="more than one"):
        sb.deepq.DQN(sb.deepq.policies.MlpPolicy, env)
    with pytest.raises(NotImplementedError, match="policy"):
        sb.deepq.DQN("CnnPolicy", None)


def test_discrete_space():
    d = sb.spaces.Discrete(12, seed=0)
    assert d.n == 12 and d.shape == () and all(d.contains(d.sample()) for _ in range(50))
    assert not d.contains(12) and not d.contains(-1)


def _config(tmp_path):
    cfg = {"DQN": {"batch_size": 32, "learning_rate": 0.001, "prioritized_replay": True, "total_timesteps": 100},
           "discount_factor": 1.0, "robot": {"discrete": False}, "reward": {}, "normalize": False}
    path = tmp_path / "c.yaml"
    path.write_text(yaml.safe_dump(cfg))
    return cfg, str(path)


def test_cli_dqn_keyword_mapping(tmp_path):
    cfg, _ = _config(tmp_path)
    kw = train_cli.dqn_kwargs(cfg)
    assert kw == dict(verbose=2, gamma=1.0, batch_size=32, prioritized_replay=True)      # learning_rate stays at 5e-4
    m = sb.deepq.DQN("MlpPolicy", None, **kw)
    assert m.learning_rate == 5e-4 and m.target_network_update_freq == 500 and m.learning_starts == 1000 and m.buffer_size == 50000


@pytest.mark.parametrize("extra,exc", [(["--n_envs", "2"], ValueError), (["--device_norm"], NotImplementedError)])
def test_cli_refuses_what_dqn_does_not_build(tmp_path, extra, exc):
    _, path = _config(tmp_path)
    out = tmp_path / "run"
    with pytest.raises(exc):
        train_cli.main(["train", "--config", path, "--algo", "DQN", "--model_dir", str(out), "--env", "tests.fake_env:make_env"] + extra)
    assert not out.exists()                                        # refused before the run directory is made


class _HostOnly(sb.deepq.DQN):
    """A DQN without a device learner: what save_training_state writes on the host side."""

    class _L:
        def save_state(self, path):
            open(path, "wb").close()

    def save(self, path, cloudpickle=False):
        open(path, "w").close()


def test_host_json_round_trip_for_dqn(tmp_path):
    m = _HostOnly("MlpPolicy", None, gamma=1.0, batch_size=7, prioritized_replay=True, seed=5, policy_kwargs={"layers": [16, 8]})
    m.learner = _HostOnly._L()
    m.num_timesteps, m.n_target_updates = 1234, 2
    m._rng.random(5)
    d = training_state.save_training_state(m, str(tmp_path / "ts"))
    host = training_state.read_host(d)
    assert host["algo"] == "DQN" and host["num_timesteps"] == 1234 and host["n_target_updates"] == 2
    json.dumps(host)
    m2 = sb.deepq.DQN("MlpPolicy", None, **host["init"])
    for k in ("gamma", "batch_size", "prioritized_replay", "seed", "layers", "learning_rate", "target_network_update_freq"):
        assert getattr(m2, k) == getattr(m, k), k
    r = np.random.default_rng(0)
    training_state.set_rng_state(r, host["rng"])
    assert np.array_equal(r.random(20), m._rng.random(20))


def test_sac_still_refuses_the_dqn_policy_marker():
    with pytest.raises(NotImplementedError, match="deepq.DQN"):
        sb.SAC(sb.deepq.policies.MlpPolicy, None, _init_setup_model=False)


def test_create_refuses_a_batch_beyond_the_gather_grid():
    with pytest.raises(_lib.B2GError, match="65535"):
        sb.deepq.DQNLearner(6, 4, (16, 16), batch_size=65536, buffer_size=10)


def test_load_applies_the_one_environment_refusal():
    with pytest.raises(ValueError, match="more than one"):
        sb.deepq.DQN.load(ZIP, env=DummyVecEnv([_Env, _Env]))
