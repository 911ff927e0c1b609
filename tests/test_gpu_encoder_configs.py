"""The encoder forward (csrc/encoder.cu) at the geometries b2g_encoder_create accepts, against oracle/encoder_ref.py.

Where the code has a path of its own for these values:
  * layer 0 gathers its input with 128-bit loads when channels % 4 == 0 and element by element otherwise (channels 2, 3, 5);
  * the last conv may have any filter count (only hidden convs need multiples of 4); its output is the Dense layer's input;
  * encoding_dim 1 and 7 leave pad columns in z's rows (zs = round4), 130 spans three 64-column engine tiles;
  * n_layers 1 and 8 (B2G_ENC_MAX_LAYERS); strides 3, 4 and 8; kernels 1 and 2; stride > kernel clamps the 'same' padding;
  * alpha < 0, 0 and 1 in the LeakyReLU epilogue;
  * set_batch retiles every layer for each call's batch size; rows must not depend on it.
"""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

import b200grasp  # noqa: F401
from b200grasp import _lib
from b200grasp.encoders import SimpleAutoEncoder
from oracle import encoder_ref as E

TOL = 1e-4      # relative to the largest encoding magnitude (fp32 FFMA vs float64 oracle)


@dataclasses.dataclass(frozen=True)
class Case:
    name: str
    hwc: tuple
    network: tuple            # (filters, kernel, stride) per conv
    enc: int
    alpha: float


CASES = [
    Case("c2", (37, 23, 2), ((8, 3, 2), (6, 4, 3)), 7, 0.1),
    Case("c3", (37, 23, 3), ((4, 2, 1), (12, 1, 4), (3, 3, 3)), 1, -0.2),
    Case("c4", (37, 23, 4), ((8, 5, 3), (1, 3, 4)), 130, 0.0),
    Case("c5", (37, 23, 5), ((12, 4, 2), (8, 2, 2)), 7, 1.0),
    Case("c8_l1", (37, 23, 8), ((4, 3, 8),), 20, 0.1),
    Case("l8", (64, 64, 1), ((4, 3, 2), (4, 2, 2), (8, 3, 2), (8, 1, 2), (12, 3, 2), (16, 2, 2), (16, 3, 1), (20, 1, 1)), 7, -0.2),
]


def layers(case):
    """enc_geometry (csrc/enc_tables.cuh): [(in h, in w, in c, k, s, f, out h, out w)] per conv, and the flattened size."""
    (h, w, c), out = case.hwc, []
    for f, k, s in case.network:
        oh, ow = -(-h // s), -(-w // s)
        out.append((h, w, c, k, s, f, oh, ow))
        h, w, c = oh, ow, f
    return out, h * w * c


def test_matrix_covers_every_forward_path():
    for c in CASES:
        ls, flat = layers(c)
        assert all(f % 4 == 0 for f, _, _ in c.network[:-1]) and flat % 4 == 0, c.name      # what create accepts
    assert {c.hwc[2] for c in CASES} >= {2, 3, 4, 5, 8}
    assert any(c.hwc[0] != c.hwc[1] and c.hwc[0] % 2 and c.hwc[1] % 2 for c in CASES)
    assert {c.network[-1][0] for c in CASES} >= {1, 3, 6}
    assert {c.enc for c in CASES} >= {1, 7, 130}
    assert {len(c.network) for c in CASES} >= {1, 8}
    convs = [l for c in CASES for l in layers(c)[0]]
    assert {s for _, _, _, _, s, _, _, _ in convs} >= {3, 4, 8}
    assert {k for _, _, _, k, _, _, _, _ in convs} >= {1, 2}
    assert any(s > k for _, _, _, k, s, _, _, _ in convs)
    assert {c.alpha for c in CASES} >= {-0.2, 0.0, 1.0}


def model_class(hwc):
    return type(f"Encoder{hwc[0]}x{hwc[1]}x{hwc[2]}", (SimpleAutoEncoder,), {"input_shape": tuple(hwc)})


def weights(case, seed):
    """Kernels scaled by 1/sqrt(fan_in) and non-zero biases: every LeakyReLU sees both signs."""
    rng = np.random.default_rng(seed)
    ls, flat = layers(case)
    arr = [(rng.normal(0, 1 / np.sqrt(k * k * c), (k, k, c, f)).astype(np.float32), rng.normal(0, 0.1, f).astype(np.float32))
           for _, _, c, k, _, f, _, _ in ls]
    arr.append((rng.normal(0, 1 / np.sqrt(flat), (flat, case.enc)).astype(np.float32), rng.normal(0, 0.1, case.enc).astype(np.float32)))
    return arr


def make(case, max_batch, seed=1):
    cfg = {"network": [{"filters": f, "kernel_size": k, "strides": s} for f, k, s in case.network], "encoding_dim": case.enc,
           "alpha": case.alpha}
    enc = model_class(case.hwc)(cfg, max_batch=max_batch)
    arr = weights(case, seed)
    enc.set_weights(arr)
    return enc, arr


def oracle(case, imgs, arr):
    return E.encode(imgs, arr, [s for _, _, s in case.network], case.alpha, torch.float64)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_encoder_case_matches_oracle(case):
    enc, arr = make(case, 6)
    lib = _lib.load()
    assert lib.b2g_encoder_n_layers(enc._handle) == len(case.network) + 1
    for i, (k, b) in enumerate(arr):
        kn, bn = C.c_int64(), C.c_int64()
        _lib.check(lib.b2g_encoder_layer_shape(enc._handle, i, C.byref(kn), C.byref(bn)))
        assert (kn.value, bn.value) == (k.size, b.size)
    imgs = np.random.default_rng(2).normal(0, 1, (6,) + case.hwc).astype(np.float32)
    ref = oracle(case, imgs, arr)
    z = enc.encode(imgs)
    assert z.shape == (6, case.enc) and np.abs(z - ref).max() <= TOL * np.abs(ref).max()
    enc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["c3", "c4"])
def test_rows_do_not_depend_on_the_batch_size(name):
    """max_batch 70 called with n = 70, 1, 65, 70: every row bitwise equal across the calls, and held to the oracle."""
    case = next(c for c in CASES if c.name == name)
    enc, arr = make(case, 70)
    imgs = np.random.default_rng(3).normal(0, 1, (70,) + case.hwc).astype(np.float32)
    z = enc.encode(imgs)
    ref = oracle(case, imgs, arr)
    assert np.abs(z - ref).max() <= TOL * np.abs(ref).max()
    assert np.array_equal(enc.encode(imgs[:1]), z[:1])
    assert np.array_equal(enc.encode(imgs[:65]), z[:65])
    assert np.array_equal(enc.encode(imgs), z)
    # other rows in a smaller call: nothing of the earlier, larger call leaks into them
    assert np.array_equal(enc.encode(imgs[5:6]), z[5:6])
    enc.close()
