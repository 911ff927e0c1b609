"""The bf16x3 training handle's surface without a GPU: b2g_autoencoder_create2's refusals come before any CUDA call, the
keyword and the command-line flag, and the geometry matrix of tests/test_gpu_autoencoder_tc.py."""
import ctypes as C
import pickle

import numpy as np
import pytest
import yaml

import b200grasp  # noqa: F401
from b200grasp import _lib, encoders, train_encoder
from tests.test_gpu_autoencoder_configs import CASES, DENOISE, TWO, _cfg, geometry

SHIPPED = ((32, 7, 2), (32, 5, 2), (32, 3, 2))


def _create2(cfg, precision):
    lib = _lib.load()
    h = C.c_void_p()
    rc = lib.b2g_autoencoder_create2(C.byref(cfg), precision, C.byref(h))
    if rc == 0:
        lib.b2g_autoencoder_destroy(h)
    return rc, lib.b2g_last_error().decode()


@pytest.mark.parametrize("precision, match", [
    (_lib.B2G_PREC_BF16, "single-pass BF16"),
    (3, "expected B2G_PREC_FP32_SIMT (0) or B2G_PREC_BF16X3 (1)"),
    (-1, "expected B2G_PREC_FP32_SIMT (0) or B2G_PREC_BF16X3 (1)"),
], ids=["bf16", "three", "negative"])
def test_create2_refuses_precisions(precision, match):
    rc, msg = _create2(_cfg(SHIPPED, enc=100), precision)
    assert rc == _lib.B2G_EINVAL and match in msg, (rc, msg)


@pytest.mark.parametrize("precision", [_lib.B2G_PREC_FP32_SIMT, _lib.B2G_PREC_BF16X3])
@pytest.mark.parametrize("cfg, match", [
    (_cfg(TWO, alpha=-0.1), "alpha"),
    (_cfg(((380, 1, 2),)), "shared memory"),
    (_cfg(((132, 4, 2),)), "must be <= 2048"),
    (_cfg(((6, 3, 2), (8, 3, 2))), "multiples of 4"),
    (_cfg(TWO, channels=2), "channels must be 1"),
    (_cfg(((8, 3, 3),)), "decoder returns 66x66"),
    (_cfg(TWO, n_layers=0), "n_layers out of range"),
], ids=["alpha_neg", "k1_f380", "k4_f132", "filters6", "channels2", "stride3_64", "layers0"])
def test_create2_refuses_what_create_refuses(cfg, match, precision):
    """Both precisions refuse the geometries b2g_autoencoder_create refuses, naming the bound, before any device call."""
    rc, msg = _create2(cfg, precision)
    assert rc == _lib.B2G_EINVAL and match in msg, (rc, msg)


def test_create2_passes_every_check_before_the_device_at_the_shipped_geometry():
    """The shipped geometry (64x64x1, convs 32/32/32, k 7/5/3, stride 2, encoding 100) is accepted: without a GPU the call
    gets as far as the device check, with one it builds the handle."""
    rc, msg = _create2(_cfg(SHIPPED, enc=100, max_batch=128), _lib.B2G_PREC_BF16X3)
    assert rc != _lib.B2G_EINVAL, msg


def test_keyword_is_checked_before_any_handle():
    cfg = {"network": [{"filters": 8, "kernel_size": 3, "strides": 2}], "encoding_dim": 4}
    with pytest.raises(ValueError, match="train_precision"):
        encoders.SimpleAutoEncoder(cfg, train_precision="bf16")
    assert set(encoders.ENCODER_PRECISIONS) == {"fp32", "bf16x3"}


@pytest.mark.parametrize("argv, want", [([], "fp32"), (["--train_precision", "bf16x3"], "bf16x3"),
                                        (["--train_precision", "fp32"], "fp32")])
@pytest.mark.parametrize("cmd", ["train", "test"])
def test_cli_flag_parses_and_reaches_the_model(tmp_path, monkeypatch, cmd, argv, want):
    seen = {}

    class Fake:
        def __init__(self, config, **kw):
            seen.update(kw)

        def train(self, *a):
            return {"loss": [0.0]}

        def load_weights(self, d):
            pass

        def test(self, *a):
            return 0.0
    monkeypatch.setattr(encoders, "SimpleAutoEncoder", Fake)
    x = np.zeros((2, 64, 64, 1), np.float32)
    with open(tmp_path / "d.pkl", "wb") as f:
        pickle.dump({"train": {"depth": x.copy(), "masks": x.astype(np.int32)}, "test": {"depth": x.copy(), "masks": x.astype(np.int32)}}, f)
    cfg = {"data_path": str(tmp_path / "d.pkl"), "batch_size": 2, "epochs": 1}
    with open(tmp_path / "c.yaml", "w") as f:
        yaml.safe_dump(cfg, f)
    (tmp_path / "m").mkdir()
    with open(tmp_path / "m" / "config.yaml", "w") as f:
        yaml.safe_dump(cfg, f)
    extra = ["--config", str(tmp_path / "c.yaml")] if cmd == "train" else []
    train_encoder.main([str(tmp_path / "m"), cmd] + extra + argv)
    assert seen["train_precision"] == want
    with pytest.raises(SystemExit):
        train_encoder.main([str(tmp_path / "m"), cmd] + extra + ["--train_precision", "bf16"])


def test_matrix_covers_every_bf16x3_engine_path():
    """The GPU matrix runs every geometry the fp32 matrix runs (bf16x3 accepts all of them), and among them the paths the
    wgmma instantiations have of their own: a decoder conv's input gradient with u = 1..8 folded in (r-contiguous A and B),
    weight gradients whose R splits (conv layers) and does not (dense, R = batch), output tiles narrower than 64 columns and
    past one 64-column tile, encoding_dim in every residue mod 4 (the dense contractions' ragged column group and r tail)."""
    from tests import test_gpu_autoencoder_tc as T
    ids = {c.name for c in CASES + DENOISE}
    assert ids == set(c.name for c in T.CASES + T.DENOISE)
    geo = [geometry(c) for c in CASES + DENOISE]
    decs = [g for _, d, _ in geo for g in d]
    encs = [g for e, _, _ in geo for g in e]
    assert {g["up"] for g in decs[:-1] if g["f"] > 1} >= {1, 2, 3, 4, 8} or {g["up"] for g in decs} >= {1, 2, 3, 4, 8}
    assert any(g["f"] < 64 for g in encs) and any(g["f"] > 64 for g in encs)
    assert {c.enc % 4 for c in CASES} == {0, 1, 2, 3}
    assert any(c.enc > 64 for c in CASES)
    # the shipped geometry's conv weight gradients split R over the SMs (R = B * oh * ow >= 512)
    assert 128 * 16 * 16 // 512 > 1
