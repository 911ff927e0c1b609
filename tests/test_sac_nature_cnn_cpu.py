"""SAC with stable-baselines' plain nature_cnn (the simplified environment's CnnPolicy): the parts that need no GPU.

  * the float64 restatement (tests/sac_nature_ref.py): stable-baselines' names and shapes in parameter_list order, and its
    forward against an independent torch nn.Conv2d / nn.Linear restatement;
  * train_cli's policy choice (sb_helper.py:85-96) for simplified / full and image / vector observations;
  * the SAC front end: policy_kwargs selection, host.json's extractor, load's layout detection, the refusals;
  * the C ABI's refusals (before any device is looked for) and the compile of the touched kernels without spills.
"""
import ctypes as C
import os
import re
import subprocess
import types

import numpy as np
import pytest
import torch

import b200grasp
from b200grasp import _lib, sac_model, train_cli
from b200grasp.common.policies import nature_cnn
from oracle import sac_ref as R
from tests import sac_nature_ref as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------ the restatement
def expected_specs(C_, A, H=64):
    out = []
    for net in ("model/pi", "model/values_fn", "target/values_fn"):
        part = [(f"{net}/c1/w", (8, 8, C_, 32)), (f"{net}/c1/b", (1, 32, 1, 1)), (f"{net}/c2/w", (4, 4, 32, 64)),
                (f"{net}/c2/b", (1, 64, 1, 1)), (f"{net}/c3/w", (3, 3, 64, 64)), (f"{net}/c3/b", (1, 64, 1, 1)),
                (f"{net}/fc1/w", (1024, 512)), (f"{net}/fc1/b", (512,))]
        if net == "model/pi":
            part += [("model/pi/fc0/kernel", (512, H)), ("model/pi/fc0/bias", (H,)), ("model/pi/fc1_1/kernel", (H, H)),
                     ("model/pi/fc1_1/bias", (H,)), ("model/pi/dense/kernel", (H, A)), ("model/pi/dense/bias", (A,)),
                     ("model/pi/dense_1/kernel", (H, A)), ("model/pi/dense_1/bias", (A,))]
        else:
            part += [(f"{net}/vf/fc0/kernel", (512, H)), (f"{net}/vf/fc0/bias", (H,)), (f"{net}/vf/fc1/kernel", (H, H)),
                     (f"{net}/vf/fc1/bias", (H,)), (f"{net}/vf/vf/kernel", (H, 1)), (f"{net}/vf/vf/bias", (1,))]
            if net == "model/values_fn":
                for q in ("qf1", "qf2"):
                    part += [(f"{net}/{q}/fc0/kernel", (512 + A, H)), (f"{net}/{q}/fc0/bias", (H,)),
                             (f"{net}/{q}/fc1/kernel", (H, H)), (f"{net}/{q}/fc1/bias", (H,)),
                             (f"{net}/{q}/{q}/kernel", (H, 1)), (f"{net}/{q}/{q}/bias", (1,))]
                part += [("model/log_ent_coef", ())]
        out += part
    return out


@pytest.mark.parametrize("C_,A", [(2, 3), (1, 5), (8, 3)])
def test_param_specs_are_stable_baselines_names_in_creation_order(C_, A):
    cfg = N.NatureConfig(obs_shape=(64, 64, C_), n_act=A, target_entropy=-float(A))
    assert N.param_specs(cfg) == expected_specs(C_, A)
    assert cfg.feat_dim == 512 and cfg.c_img == C_


def _torch_features(x, p, net):
    """nature_cnn with torch modules: NHWC /255 input, HWIO weights, NHWC flatten (conv_to_fc)."""
    h = x.permute(0, 3, 1, 2)
    for name, k, s in (("c1", 8, 4), ("c2", 4, 2), ("c3", 3, 1)):
        w = torch.as_tensor(p[f"{net}/{name}/w"], dtype=torch.float64)
        conv = torch.nn.Conv2d(w.shape[2], w.shape[3], k, stride=s).double()
        with torch.no_grad():
            conv.weight.copy_(w.permute(3, 2, 0, 1))
            conv.bias.copy_(torch.as_tensor(p[f"{net}/{name}/b"], dtype=torch.float64).reshape(-1))
        h = torch.relu(conv(h))
    flat = h.permute(0, 2, 3, 1).reshape(h.shape[0], -1)
    lin = torch.nn.Linear(1024, 512).double()
    with torch.no_grad():
        lin.weight.copy_(torch.as_tensor(p[f"{net}/fc1/w"], dtype=torch.float64).T)
        lin.bias.copy_(torch.as_tensor(p[f"{net}/fc1/b"], dtype=torch.float64))
    return torch.relu(lin(flat))


def _torch_mlp(z, p, pre, names):
    for n in names:
        lin = torch.nn.Linear(*p[f"{pre}/{n}/kernel"].shape).double()
        with torch.no_grad():
            lin.weight.copy_(torch.as_tensor(p[f"{pre}/{n}/kernel"], dtype=torch.float64).T)
            lin.bias.copy_(torch.as_tensor(p[f"{pre}/{n}/bias"], dtype=torch.float64))
        z = torch.relu(lin(z))
    return z


def test_forward_equals_an_independent_torch_restatement():
    cfg = N.NatureConfig(obs_shape=(64, 64, 2), n_act=3)
    p = N.init_params(cfg, seed=5)
    rng = np.random.default_rng(6)
    B = 4
    obs = np.zeros((B, 64, 64, 2), np.float32)
    obs[..., 0] = rng.uniform(0, 255, (B, 64, 64))
    nxt = obs.copy()
    nxt[..., 0] = rng.uniform(0, 255, (B, 64, 64))
    batch = dict(obs=obs, next_obs=nxt, act=rng.uniform(-1, 1, (B, 3)).astype(np.float32),
                 rew=rng.standard_normal(B).astype(np.float32), done=np.zeros(B, np.float32))
    eps = rng.standard_normal((B, 3)).astype(np.float32)
    out, grads, _, _ = N.sac_step(p, R.OptState.zeros(N.to_oracle(p)), batch, eps, 3e-4, cfg, torch.float64)
    x = torch.as_tensor(obs, dtype=torch.float64) / 255.0
    xn = torch.as_tensor(nxt, dtype=torch.float64) / 255.0
    act = torch.as_tensor(batch["act"], dtype=torch.float64)
    with torch.no_grad():
        f_pi = _torch_features(x, p, "model/pi")
        g = _torch_mlp(f_pi, p, "model/pi", ("fc0", "fc1_1"))
        mu = g @ torch.as_tensor(p["model/pi/dense/kernel"], dtype=torch.float64) + torch.as_tensor(p["model/pi/dense/bias"], dtype=torch.float64)
        f_v = _torch_features(x, p, "model/values_fn")
        z = _torch_mlp(torch.cat([f_v, act], 1), p, "model/values_fn/qf1", ("fc0", "fc1"))
        q1 = z @ torch.as_tensor(p["model/values_fn/qf1/qf1/kernel"], dtype=torch.float64) + float(p["model/values_fn/qf1/qf1/bias"][0])
        zt = _torch_mlp(_torch_features(xn, p, "target/values_fn"), p, "target/values_fn/vf", ("fc0", "fc1"))
        vt = zt @ torch.as_tensor(p["target/values_fn/vf/vf/kernel"], dtype=torch.float64) + float(p["target/values_fn/vf/vf/bias"][0])
    assert f_pi.shape == (B, 512)
    np.testing.assert_allclose(out["h_pi"], f_pi.numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(out["mu"], mu.numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(out["q1"], q1.numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(out["v_targ"], vt.numpy(), rtol=1e-12, atol=1e-12)
    # the zero pad plane takes no conv1 gradient
    assert not grads["model/pi/c1/w"][:, :, 1, :].any() and grads["model/pi/c1/w"][:, :, 0, :].any()
    assert set(grads) == {n for n, _ in N.param_specs(cfg) if not n.startswith("target/")}


# ------------------------------------------------------------------------------------------------ train_cli (sb_helper.py:85-96)
class _Stop(Exception):
    pass


def _policy_choice(monkeypatch, tmp_path, simplified, image, full_obs=False):
    """train_cli.train's SAC construction for a fake env of the given kind, captured before the learner is built."""
    seen = {}

    def fake_sac(policy, env, **kw):
        seen.update(policy=policy, **kw)
        raise _Stop

    shape = (64, 64, 2) if image else (12,)
    env = types.SimpleNamespace(observation_space=types.SimpleNamespace(shape=shape), close=lambda: None)
    monkeypatch.setattr(train_cli, "SAC", fake_sac)
    monkeypatch.setattr(train_cli, "DummyVecEnv", lambda fns: env)
    monkeypatch.setattr(train_cli, "Monitor", lambda e, path: e)
    monkeypatch.setattr(train_cli, "EvalCallback", lambda *a, **k: None)
    cfg = {"robot": {}, "reward": {}, "discount_factor": 0.99, "full_observation": full_obs,
           "SAC": {"layers": [128, 128], "buffer_size": 100, "batch_size": 16, "step_size": 3e-4, "total_timesteps": 10}}
    path = tmp_path / f"cfg_{simplified}_{image}_{full_obs}.yaml"
    import yaml
    path.write_text(yaml.safe_dump(cfg))
    argv = ["train", "--config", str(path), "--algo", "SAC", "--model_dir", str(tmp_path / f"m_{simplified}_{image}_{full_obs}"),
            "--env", "tests.fake_env:FakeGraspEnv"]
    if simplified:
        argv.append("-s")
    with pytest.raises(_Stop):
        train_cli.main(argv)
    return seen


@pytest.mark.parametrize("full_obs", [False, True])
def test_train_cli_policy_choice(monkeypatch, tmp_path, full_obs):
    s_img = _policy_choice(monkeypatch, tmp_path, True, True, full_obs)
    assert s_img["policy"] is sac_model.CnnPolicy
    assert s_img["policy_kwargs"] == {"cnn_extractor": "nature_cnn"}          # default [64, 64], not the config's layers
    assert "replay_u8_planes" not in s_img                                   # depth + pad: no 8-bit planes
    s_vec = _policy_choice(monkeypatch, tmp_path, True, False, full_obs)
    assert s_vec["policy"] is sac_model.MlpPolicy and s_vec["policy_kwargs"] == {"layers": [128, 128], "layer_norm": False}
    f_img = _policy_choice(monkeypatch, tmp_path, False, True, full_obs)
    assert f_img["policy"] is sac_model.CnnPolicy
    assert f_img["policy_kwargs"] == {"layers": [128, 128], "cnn_extractor": "augmented_nature_cnn"}
    assert f_img.get("replay_u8_planes") == ((0, 1, 2) if full_obs else None)
    f_vec = _policy_choice(monkeypatch, tmp_path, False, False, full_obs)
    assert f_vec["policy"] is sac_model.MlpPolicy and f_vec["policy_kwargs"] == {"layers": [128, 128], "layer_norm": False}
    for s in (s_vec, f_vec):
        assert "replay_u8_planes" not in s


# ------------------------------------------------------------------------------------------------ SAC front end
class RecordingLearner:
    """Stands in for the device learner: records the constructor and holds the parameter table the extractor implies."""

    def __init__(self, obs_shape, n_act=5, hidden=64, extractor="augmented", **kw):
        self.obs_shape, self.extractor = tuple(obs_shape), extractor
        if extractor == "nature_cnn":
            specs = N.param_specs(N.NatureConfig(obs_shape=self.obs_shape, n_act=n_act, layers=(hidden, hidden)))
        else:
            specs = R.param_specs(R.SACConfig(obs_shape=self.obs_shape, n_act=n_act, layers=(hidden, hidden)))
        self.param_shapes = dict(specs)
        self.params = {}
        self.loaded = []

    def load_parameters(self, p, exact_match=True):
        for n, a in p.items():
            if n not in self.param_shapes:
                if exact_match:
                    raise ValueError(n)
                continue
            self.loaded.append(n)
            self.params[n] = np.asarray(a, np.float32)

    def get_parameters(self):
        return dict(self.params)

    def set_norm_stats(self, *a, **k):
        pass

    def close(self):
        pass


@pytest.fixture
def fake_learner(monkeypatch):
    monkeypatch.setattr(sac_model, "Learner", RecordingLearner)


def test_policy_kwargs_select_the_extractor(fake_learner):
    from b200grasp.vec_env import DummyVecEnv
    for kw, want in (({"cnn_extractor": nature_cnn}, "nature_cnn"), ({"cnn_extractor": "nature_cnn"}, "nature_cnn"),
                     ({"cnn_extractor": None}, "augmented"), ({"cnn_extractor": "augmented_nature_cnn"}, "augmented"),
                     ({"cnn_extractor": object()}, "augmented")):
        m = sac_model.SAC(sac_model.CnnPolicy, DummyVecEnv([lambda: _SimpleEnv()]), policy_kwargs=kw, seed=1)
        assert m.learner.extractor == want and m.extractor == want
        names = list(m.learner.param_shapes)
        assert ("model/pi/c1/w" in names) == (want == "nature_cnn")
        assert ("model/pi/fc1_1/kernel" in names) == (want == "nature_cnn")


def test_empty_policy_kwargs_still_refused_and_names_both_extractors(fake_learner):
    from b200grasp.vec_env import DummyVecEnv
    with pytest.raises(NotImplementedError, match="cnn_extractor=nature_cnn.*create_augmented_nature_cnn"):
        sac_model.SAC(sac_model.CnnPolicy, DummyVecEnv([lambda: _SimpleEnv()]), policy_kwargs={})


def test_host_json_round_trips_nature_cnn(fake_learner):
    from b200grasp.vec_env import DummyVecEnv
    m = sac_model.SAC(sac_model.CnnPolicy, DummyVecEnv([lambda: _SimpleEnv()]), policy_kwargs={"cnn_extractor": nature_cnn}, seed=2)
    host = m._host_state()
    assert host["init"]["policy_kwargs"]["cnn_extractor"] == "nature_cnn"
    import json
    host = json.loads(json.dumps(host))
    m2 = sac_model.SAC(sac_model.SAC._policy_from_host(host), DummyVecEnv([lambda: _SimpleEnv()]), **host["init"])
    assert m2.extractor == "nature_cnn" and m2.learner.extractor == "nature_cnn"
    a = sac_model.SAC(sac_model.CnnPolicy, DummyVecEnv([lambda: _SimpleEnv()]), policy_kwargs={"cnn_extractor": object()})
    assert a._host_state()["init"]["policy_kwargs"]["cnn_extractor"] == "augmented_nature_cnn"


def test_load_detects_the_extractor_and_refuses_a_donor_of_the_other(fake_learner, tmp_path):
    from b200grasp.vec_env import DummyVecEnv
    m = sac_model.SAC(sac_model.CnnPolicy, DummyVecEnv([lambda: _SimpleEnv()]), policy_kwargs={"cnn_extractor": nature_cnn}, seed=3)
    m.save(str(tmp_path / "nat.zip"))
    back = sac_model.SAC.load(str(tmp_path / "nat.zip"))
    assert back.extractor == "nature_cnn" and tuple(back.observation_space.shape) == (64, 64, 2)
    assert back.hidden == 64 and back.learner.obs_shape == (64, 64, 2)
    aug = sac_model.SAC(sac_model.CnnPolicy, DummyVecEnv([lambda: _SimpleEnv()]), policy_kwargs={"cnn_extractor": None}, seed=4)
    for dst, src in ((aug, m), (m, aug)):
        before = list(dst.learner.loaded)
        for exact in (True, False):
            with pytest.raises(ValueError, match="extractor"):
                dst.load_parameters(src.get_parameters(), exact_match=exact)
        assert dst.learner.loaded == before             # nothing half loaded


class _SimpleEnv:
    """A simplified depth env: (64, 64, 2) observations whose second plane is a zero pad, Box(-1, 1)^3 actions."""

    def __init__(self):
        from b200grasp.spaces import Box
        self.observation_space = Box(0.0, 255.0, (64, 64, 2))
        self.action_space = Box(-1.0, 1.0, (3,))

    def reset(self):
        return np.zeros((64, 64, 2), np.float32)

    def step(self, a):
        return np.zeros((64, 64, 2), np.float32), 0.0, False, {}

    def close(self):
        pass


# ------------------------------------------------------------------------------------------------ C ABI
def _sac_cfg(obs_c=2, obs_h=64):
    cfg = _lib.SacCfg()
    cfg.obs_h, cfg.obs_w, cfg.obs_c, cfg.obs_dim = obs_h, obs_h, obs_c, 0 if obs_h else 12
    cfg.n_act, cfg.hidden, cfg.batch, cfg.buffer_capacity = 3, 64, 8, 64
    cfg.gamma, cfg.tau, cfg.target_entropy, cfg.precision, cfg.nranks = 0.99, 0.005, -3.0, 1, 1
    return cfg


@pytest.mark.parametrize("obs_h,obs_c,extractor,mask,msg", [
    (0, 0, 1, 0, "MLP policy"),
    (64, 2, 7, 0, "unknown extractor"),
    (64, 2, 1, 1 << 2, "below obs_c"),
])
def test_create3_refuses_before_any_device(obs_h, obs_c, extractor, mask, msg):
    lib = _lib.load()
    cfg = _sac_cfg(obs_c, obs_h)
    rcfg = _lib.ReplayCfg(128, mask) if mask else None
    net = _lib.SacNetCfg(extractor)
    h = C.c_void_p()
    assert lib.b2g_sac_create3(C.byref(cfg), None if rcfg is None else C.byref(rcfg), C.byref(net), C.byref(h)) == -1
    assert not h.value
    assert msg in lib.b2g_last_error().decode()


def test_learner_refuses_an_unknown_extractor_name():
    with pytest.raises(ValueError, match="extractor"):
        b200grasp.Learner((64, 64, 2), n_act=3, extractor="plain")


# spill stores some kernels of these files already had before nature_cnn existed; no kernel may add any
KNOWN_SPILLS = {"gather_kernelENS": 16, "gather2_kernelILi3E": 40, "tailw_kernelILi256E": 4, "tailw_kernelILi128E": 4}


def test_touched_kernels_compile_without_new_spills(tmp_path):
    """nvcc for sm_90a with -Xptxas -v: no kernel of the files this feature touches spills more than it did before."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not installed")
    src = os.path.join(ROOT, "deep-rl-grasping_b200", "csrc")
    for f in ("replay.cu", "engine_v2.cu", "obsnorm.cu", "tail.cu"):
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c",
                            os.path.join(src, f), "-o", str(tmp_path / (f + ".o"))], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-2000:]
        found = re.findall(r"Function properties for (\S+)\s+\d+ bytes stack frame, (\d+) bytes spill stores", r.stderr)
        assert found, f
        for fn, spill in found:
            allowed = max([v for k, v in KNOWN_SPILLS.items() if k in fn] + [0])
            assert int(spill) <= allowed, (f, fn, spill)
