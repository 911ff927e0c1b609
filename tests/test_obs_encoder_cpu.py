"""The encoded-depth observation with the encoding deferred to the learner's process (no GPU): the deferred sensor, the
VecEncodeDepth wrapper's spaces, host mode and the hand-over to a device learner, predict's raw-row refusal, train_cli
--device_encode, the ABI declarations and an sm_90a compile of the encoder stage."""
import os
import re
import shutil
import subprocess
import types

import numpy as np
import pytest
import yaml

import b200grasp
from b200grasp import _lib, encoders, train_cli
from b200grasp.base_model import BaseModel
from b200grasp.encoders import DeferredEncodedDepthImgSensor
from b200grasp.spaces import Box
from b200grasp.vec_env import DummyVecEnv, VecEncodeDepth, VecNormalize
from tests.deferred_env import PIXELS, FakeDeferredEnv

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class RecordingEncoder:
    """Stands in for SimpleAutoEncoder: the encoding of a frame is its first encoding_dim pixels + 1; every call is recorded."""
    input_shape = (64, 64, 1)

    def __init__(self, encoding_dim=10):
        self.encoding_dim = encoding_dim
        self.calls = []

    def encode(self, imgs):
        imgs = np.asarray(imgs, np.float32)
        assert imgs.ndim == 4 and imgs.shape[1:] == self.input_shape
        self.calls.append(imgs.shape[0])
        return imgs.reshape(imgs.shape[0], -1)[:, :self.encoding_dim] + 1.0

    def weights_digest(self):
        return "d" * 64


def _venv(n=3, tail=1, horizon=7):
    return DummyVecEnv([(lambda i=i: FakeDeferredEnv(seed=i, horizon=horizon, tail=tail)) for i in range(n)])


# ------------------------------------------------------------------------------------------------ the deferred sensor
class _Camera:
    def __init__(self, img, mask):
        self.state_space = Box(0.0, 1.0, img.shape + (1,))
        self._img, self._mask = img, mask

    def get_state(self):
        return None, self._img.copy(), self._mask


def _sensor_config(tmp_path, scene_type="OnTable", visualize=False):
    d = tmp_path / "enc"
    d.mkdir(exist_ok=True)
    (d / "config.yaml").write_text(yaml.safe_dump({"encoding_dim": 100, "network": []}))
    return {"scene": {"scene_type": scene_type}, "sensor": {"encoder_dir": str(d), "visualize": visualize}}


@pytest.fixture
def no_cuda_library(monkeypatch):
    """Any use of the CUDA library fails: the sensor must not load it (env workers hold no CUDA context)."""
    def refuse(*a, **k):
        raise AssertionError("the deferred sensor touched the CUDA library")

    class Blocked(types.ModuleType):
        def __getattr__(self, name):
            refuse()
    monkeypatch.setattr(_lib, "load", refuse)
    monkeypatch.setattr(encoders, "_lib", Blocked("b200grasp._lib"))


@pytest.mark.parametrize("scene_type", ["OnTable", "OnFloor"])
def test_deferred_sensor_filters_like_the_reference(tmp_path, no_cuda_library, scene_type):
    rng = np.random.default_rng(3)
    img = rng.uniform(0.1, 2.0, (64, 64)).astype(np.float32)
    mask = rng.integers(0, 8, (64, 64))
    robot = types.SimpleNamespace(robot_id=5)
    s = DeferredEncodedDepthImgSensor(_sensor_config(tmp_path, scene_type), _Camera(img, mask), robot)
    out = s.get_state()
    # the reference zeroes the plane (0) and the robot, and under OnTable the table (1) and the tray (2)
    zeroed = np.isin(mask, [0, 5, 1, 2] if scene_type == "OnTable" else [0, 5])
    assert out.dtype == np.float32 and out.shape == (64 * 64,)
    assert np.array_equal(out, np.where(zeroed, 0.0, img).reshape(-1))
    assert s.state_space.shape == (64 * 64,) and s.encoding_dim == 100


def test_deferred_sensor_refuses_visualize(tmp_path):
    img = np.ones((64, 64), np.float32)
    with pytest.raises(NotImplementedError, match="decoder"):
        DeferredEncodedDepthImgSensor(_sensor_config(tmp_path, visualize=True), _Camera(img, img), types.SimpleNamespace(robot_id=3))


# ------------------------------------------------------------------------------------------------ VecEncodeDepth
@pytest.mark.parametrize("tail", [0, 1, 2])
def test_wrapper_spaces(tail):
    w = VecEncodeDepth(_venv(2, tail), RecordingEncoder(10))
    assert w.tail == tail and w.raw_width == PIXELS + tail
    assert w.observation_space.shape == (10 + tail,)
    assert np.all(w.observation_space.low[:10] == -1) and np.all(w.observation_space.high[:10] == 1)
    assert np.all(w.observation_space.low[10:] == 0) and np.all(w.observation_space.high[10:] == 1)
    vn = VecNormalize(w)
    assert vn.obs_rms.mean.shape == (10 + tail,)
    with pytest.raises(ValueError, match="tail"):
        VecEncodeDepth(_venv(1, tail), RecordingEncoder(10), tail=tail + 1)


def test_host_mode_encodes_terminal_observations_in_the_same_call():
    enc = RecordingEncoder(10)
    raw = _venv(3, tail=1, horizon=2)
    w = VecEncodeDepth(raw, enc)
    obs = w.reset()
    assert obs.shape == (3, 11) and enc.calls == [3]
    a = np.zeros((3, 5), np.float32)
    _, _, done, _ = w.step(a)
    assert not done.any() and enc.calls == [3, 3]
    # the second step ends every episode: 3 frames + 3 terminal frames in one call
    term_raw = [e.pool[(e.k + 1) % len(e.pool)] for e in raw.envs]
    obs, _, done, infos = w.step(a)
    assert done.all() and enc.calls == [3, 3, 6]
    for i in range(3):
        t = infos[i]["terminal_observation"]
        assert t.shape == (11,)
        assert np.array_equal(t[:10], term_raw[i][:10] + 1.0) and t[10] == term_raw[i][-1]
        assert obs[i][10] == raw.envs[i].pool[raw.envs[i].k][-1]


class _FakeLearner:
    def __init__(self):
        self.attached = []

    def set_obs_encoder(self, encoder, tail=0):
        self.attached.append((encoder, tail))

    def close(self):
        pass


def _stub_model(env, device_obs_norm=True):
    m = BaseModel()
    m.device_obs_norm = device_obs_norm
    m._set_env(env)
    m.learner = _FakeLearner()
    return m


def test_mode_hand_over_and_back():
    enc = RecordingEncoder(10)
    w = VecEncodeDepth(_venv(2, tail=1), enc)
    m = _stub_model(w)
    m._attach_obs_encoder()
    assert m.learner.attached == [(enc, 1)] and w.pass_raw and w.encoder_owner is m.learner
    obs = w.reset()
    assert obs.shape == (2, PIXELS + 1) and enc.calls == []            # raw rows straight through
    w.step_async(np.zeros((2, 5)))
    for _ in range(7):
        obs, _, done, infos = w.step(np.zeros((2, 5)))
    assert done.all() and infos[0]["terminal_observation"].shape == (PIXELS + 1,) and enc.calls == []
    other = _stub_model(w)
    other._attach_obs_encoder()                                          # the encoder has an owner already
    assert other.learner.attached == [] and w.encoder_owner is m.learner
    with pytest.raises(RuntimeError, match="another learner"):
        w.give_encoder_to(other.learner)
    m.close()
    assert not w.pass_raw and w.reset().shape == (2, 11) and enc.calls == [2]


def test_host_mode_kept_without_device_obs_norm_or_under_a_host_vecnormalize():
    w = VecEncodeDepth(_venv(2), RecordingEncoder(10))
    m = _stub_model(w, device_obs_norm=False)
    m._attach_obs_encoder()
    assert not w.pass_raw and m.learner.attached == []
    vn = VecNormalize(w)                                                 # statistics not owned by the learner: encoded rows needed
    m = _stub_model(vn)
    m._attach_obs_encoder()
    assert not w.pass_raw and m.learner.attached == []


def test_predict_refuses_raw_rows():
    w = VecEncodeDepth(_venv(1), RecordingEncoder(10))
    m = _stub_model(w)
    with pytest.raises(ValueError, match="host-mode VecEncodeDepth"):
        m._check_encoded(np.zeros((4, PIXELS + 1), np.float32))
    with pytest.raises(ValueError, match="host-mode VecEncodeDepth"):
        m._check_encoded(np.zeros(PIXELS + 1, np.float32))
    m._check_encoded(np.zeros((4, 11), np.float32))


# ------------------------------------------------------------------------------------------------ train_cli --device_encode
def _cli_config(tmp_path, **kw):
    cfg = {"sensor": {"encoder_dir": str(tmp_path / "enc")}, "robot": {}, "reward": {}, "SAC": {}, "normalize": True,
           "discount_factor": 0.99}
    cfg.update(kw)
    p = tmp_path / "config.yaml"
    p.write_text(yaml.safe_dump(cfg))
    return str(p)


@pytest.mark.parametrize("key", ["depth_observation", "full_observation"])
def test_cli_refuses_image_configs_before_model_dir(tmp_path, key):
    model_dir = tmp_path / "run"
    with pytest.raises(ValueError, match="--device_encode"):
        train_cli.main(["train", "--config", _cli_config(tmp_path, **{key: True}), "--algo", "SAC", "--model_dir", str(model_dir),
                        "--device_encode", "--env", "tests.deferred_env:make_env"])
    assert not model_dir.exists()


def test_cli_stack(monkeypatch, tmp_path):
    enc = RecordingEncoder(10)
    seen = []
    monkeypatch.setattr(train_cli, "device_encoder", lambda config, n: seen.append((config["sensor"]["encoder_dir"], n)) or enc)
    env, test_env = train_cli.encode_depth(_venv(4), _venv(1), {"sensor": {"encoder_dir": "/x"}}, 4)
    assert seen == [("/x", 4)]
    assert isinstance(env, VecEncodeDepth) and isinstance(test_env, VecEncodeDepth)
    assert env.encoder is enc and test_env.encoder is enc and not env.pass_raw and not test_env.pass_raw
    assert env.observation_space.shape == (11,) and VecNormalize(env).obs_rms.mean.shape == (11,)
    args = train_cli.build_parser().parse_args(["train", "--device_encode", "--config", "c", "--algo", "SAC", "--model_dir", "m"])
    assert args.device_encode


# ------------------------------------------------------------------------------------------------ ABI and build
def test_abi_declarations():
    h = open(os.path.join(ROOT, "include", "b200grasp.h")).read()
    for abi in ("sac", "bdq"):
        sym = f"b2g_{abi}_set_obs_encoder"
        assert re.search(rf"int {sym}\(b2g_{abi}\* h, const b2g_encoder\* enc, int tail\);", h)
        assert sym in _lib.SYMBOLS
        assert sym in open(os.path.join(ROOT, "INTEGRATION.md")).read()
        assert hasattr(_lib.load(), sym)


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="needs nvcc")
def test_encoder_stage_compiles_for_sm90a_without_spills(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    src = os.path.join(ROOT, "deep-rl-grasping_b200", "csrc", "encoder.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-Xptxas", "-v",
                        "-c", src, "-o", str(tmp_path / "encoder.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    entries = re.findall(r"Compiling entry function '(\w+)'", r.stderr)
    assert any("enc_stage_in" in e for e in entries) and any("enc_stage_out" in e for e in entries)
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(spills) == len(entries) and all(a == "0" and b == "0" for a, b in spills), r.stderr
