"""The bf16x3 perception encoder's host side (no GPU): the precision keyword, train_cli --encoder_precision and its
config.yaml record, host.json's record of the encoder's precision and load_training_state's check of it, and the ABI."""
import os
import re
import types

import numpy as np
import pytest
import yaml

import b200grasp  # noqa: F401
from b200grasp import _lib, encoders, train_cli
from b200grasp.base_model import BaseModel
from b200grasp.encoders import SimpleAutoEncoder
from b200grasp.vec_env import DummyVecEnv, VecEncodeDepth
from tests.deferred_env import FakeDeferredEnv

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENC_CFG = {"network": [{"filters": 32, "kernel_size": 7, "strides": 2}], "encoding_dim": 10}


class FakeEncoder:
    input_shape = (64, 64, 1)

    def __init__(self, precision):
        self.encoding_dim, self.precision = 10, precision

    def encode(self, imgs):
        return np.zeros((len(imgs), self.encoding_dim), np.float32)

    def weights_digest(self):
        return "d" * 64


def _ve(precision):
    return VecEncodeDepth(DummyVecEnv([lambda: FakeDeferredEnv(seed=0, horizon=7, tail=1)]), FakeEncoder(precision))


def test_unknown_precision_raises_before_the_library():
    for bad in ("x", "bf16", "fp16", None):
        with pytest.raises(ValueError, match="precision"):
            SimpleAutoEncoder(ENC_CFG, precision=bad)
    assert encoders.ENCODER_PRECISIONS == {"fp32": _lib.B2G_PREC_FP32_SIMT, "bf16x3": _lib.B2G_PREC_BF16X3}


def test_flag_parsing_and_defaults(capsys):
    p = train_cli.build_parser()
    base = ["train", "--config", "c", "--algo", "SAC", "--model_dir", "m"]
    assert p.parse_args(base + ["--device_encode"]).encoder_precision is None
    assert p.parse_args(base + ["--device_encode", "--encoder_precision", "bf16x3"]).encoder_precision == "bf16x3"
    assert p.parse_args(base + ["--device_encode", "--encoder_precision", "fp32"]).encoder_precision == "fp32"
    with pytest.raises(SystemExit):
        p.parse_args(base + ["--device_encode", "--encoder_precision", "bf16"])
    with pytest.raises(SystemExit):          # the flag alone is an argparse error, before the config is read
        train_cli.main(base + ["--encoder_precision", "bf16x3"])
    assert "--encoder_precision needs --device_encode" in capsys.readouterr().err


class _Stop(Exception):
    pass


@pytest.mark.parametrize("flag, want", [(None, "fp32"), ("fp32", "fp32"), ("bf16x3", "bf16x3")])
def test_config_yaml_records_the_precision(tmp_path, monkeypatch, flag, want):
    cfg = {"sensor": {"encoder_dir": str(tmp_path / "enc")}, "robot": {}, "reward": {}, "SAC": {}, "normalize": True,
           "discount_factor": 0.99}
    cp = tmp_path / "config.yaml"
    cp.write_text(yaml.safe_dump(cfg))
    seen = []

    def encode_depth(env, test_env, config, n_envs):
        seen.append(config["device_encode_precision"])
        raise _Stop

    monkeypatch.setattr(train_cli, "encode_depth", encode_depth)
    md = tmp_path / "run"
    argv = ["train", "--config", str(cp), "--algo", "SAC", "--model_dir", str(md), "--device_encode", "--env",
            "tests.deferred_env:make_env"] + (["--encoder_precision", flag] if flag else [])
    with pytest.raises(_Stop):
        train_cli.main(argv)
    assert seen == [want]
    for sub in ("", "best_model"):
        assert yaml.safe_load(open(md / sub / "config.yaml"))["device_encode_precision"] == want


@pytest.mark.parametrize("recorded, want", [({}, "fp32"), ({"device_encode_precision": "bf16x3"}, "bf16x3"),
                                            ({"device_encode_precision": "fp32"}, "fp32")])
def test_device_encoder_builds_the_recorded_precision(tmp_path, monkeypatch, recorded, want):
    d = tmp_path / "enc"
    d.mkdir()
    (d / "config.yaml").write_text(yaml.safe_dump(ENC_CFG))
    built = []

    class Recording:
        def __init__(self, config, max_batch=1, device=0, seed=None, precision="fp32"):
            built.append((max_batch, precision))

        def load_weights(self, model_dir):
            assert model_dir == str(d)

    monkeypatch.setattr(encoders, "SimpleAutoEncoder", Recording)
    train_cli.device_encoder(dict({"sensor": {"encoder_dir": str(d)}}, **recorded), 3)
    assert built == [(6, want)]


def test_host_json_records_the_precision():
    for prec in ("fp32", "bf16x3"):
        ve = _ve(prec)
        learner = object()
        ve.give_encoder_to(learner)
        rec = BaseModel._encoder_host(types.SimpleNamespace(env=ve, learner=learner))
        assert rec == {"dir": None, "digest": "d" * 64, "precision": prec}


def test_load_refuses_a_precision_mismatch_and_reads_old_files_as_fp32():
    def host(**prec):
        return {"obs_encoder": dict({"dir": "/enc", "digest": "d" * 64}, **prec)}

    BaseModel._check_encoder_digest("p", host(precision="bf16x3"), _ve("bf16x3"))
    BaseModel._check_encoder_digest("p", host(precision="fp32"), _ve("fp32"))
    BaseModel._check_encoder_digest("p", host(), _ve("fp32"))                     # written before the field existed
    with pytest.raises(ValueError, match="bf16x3 encoder.*encodes in fp32"):
        BaseModel._check_encoder_digest("p", host(precision="bf16x3"), _ve("fp32"))
    with pytest.raises(ValueError, match="fp32 encoder.*encodes in bf16x3"):
        BaseModel._check_encoder_digest("p", host(), _ve("bf16x3"))


def test_abi_symbols():
    h = open(os.path.join(ROOT, "include", "b200grasp.h")).read()
    assert re.search(r"int b2g_encoder_create2\(const b2g_encoder_cfg\* cfg, int32_t precision, b2g_encoder\*\* out\);", h)
    assert re.search(r"int b2g_debug_encoder_layers\(b2g_encoder\* h, const float\* imgs, int n, float\* out, int64_t out_numel\);", h)
    lib = _lib.load()
    for sym in ("b2g_encoder_create2", "b2g_debug_encoder_layers"):
        assert sym in _lib.SYMBOLS and hasattr(lib, sym)
    assert "b2g_encoder_create2" in open(os.path.join(ROOT, "INTEGRATION.md")).read()


def test_create2_refusals_need_no_device():
    """Refused before check_device: on a machine without a Hopper GPU these still say B2G_EINVAL, with the reason."""
    import ctypes as C
    lib = _lib.load()
    cfg = _lib.EncoderCfg()
    cfg.height, cfg.width, cfg.channels, cfg.n_layers = 64, 64, 1, 3
    for i, (f, k, s) in enumerate(((4, 7, 2), (32, 5, 2), (32, 3, 2))):
        cfg.filters[i], cfg.kernel[i], cfg.strides[i] = f, k, s
    cfg.encoding_dim, cfg.alpha, cfg.max_batch, cfg.device = 100, 0.1, 4, 1 << 20
    h = C.c_void_p()
    for prec, what in ((_lib.B2G_PREC_BF16, "single-pass BF16"), (5, "precision 5")):
        assert lib.b2g_encoder_create2(C.byref(cfg), prec, C.byref(h)) == _lib.B2G_EINVAL
        assert what in lib.b2g_last_error().decode()
    assert lib.b2g_encoder_create2(C.byref(cfg), _lib.B2G_PREC_BF16X3, C.byref(h)) == _lib.B2G_EINVAL
    assert "conv layer 0 has 4 filters" in lib.b2g_last_error().decode()
    assert not h
