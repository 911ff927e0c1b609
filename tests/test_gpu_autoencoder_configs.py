"""The auto-encoder training handle (csrc/autoencoder.cu) at the geometries b2g_autoencoder_create accepts.

Where the code has a path of its own for these values:
  * n_layers = 1 leaves no decoder conv: the output conv upsamples the decoder Dense's output directly and the backward goes
    from the output conv straight to the decoder Dense; n_layers = 8 is B2G_ENC_MAX_LAYERS;
  * a decoder conv's input gradient folds its u x u upsampling block into the gather (R = u^2 k^2 f), u = 1, 2, 3, 4, 8;
  * kernels 1 and 2, and stride > kernel, where 'same' padding clamps at 0 and some input pixels are read by no output
    (their gradient must be exactly 0); odd padding totals put the extra row and column behind;
  * encoding_dim = 1 and any residue mod 4 leave pad columns in z's rows (zs = round4(encoding_dim)) that the dense dgrad
    and wgrad read past; encoding_dim > 64 spans more than one 64-column tile of the gather-GEMM engine (gg_simt);
  * filter counts of 4 and over 64 (a second engine tile, 4 columns wide at 68);
  * the output conv (ae_out_fwd / ae_out_wgrad, 8 x 8 pixel tiles staged in shared memory) at both of its bounds,
    kernel_0^2 * filters_0 <= 2048 and 96 KB of shared memory, and past the 48 KB default that needs an opt-in;
  * images whose height and width are not multiples of 8 (partial tiles) and H != W;
  * LeakyReLU alpha 0 (a negative pre-activation stores -0.0), 1 and > 1;
  * targets other than the inputs, through the explicit step, the captured epoch graph and evaluate.

The CPU tests keep the matrix honest from a restatement of the handle's geometry, and check the create refusals.  The GPU
tests hold every case to the float64 oracle of tests/ae_ref.py with the bars of tests/test_gpu_autoencoder.py.
"""
import ctypes as C
import dataclasses
import math

import numpy as np
import pytest
import torch

import b200grasp  # noqa: F401
from b200grasp import _lib
from b200grasp.encoders import SimpleAutoEncoder, model_shapes
from oracle import encoder_ref as E
from tests import ae_ref as R
from tests.test_gpu_autoencoder import check_step, check_updates, glorot, scenes, shipped

AE_TILE = 8
MAX_SMEM = 96 * 1024
WG_MAX = 256 * 8          # ae_out_wgrad: 256 threads x 8 weights each


# ------------------------------------------------------------------------------------------------ the cases
@dataclasses.dataclass(frozen=True)
class Case:
    name: str
    hw: tuple
    network: tuple            # (filters, kernel, stride) per encoder conv
    enc: int
    alpha: float
    Bs: tuple
    targets: bool = False

    def cfg(self):
        return {"network": [{"filters": f, "kernel_size": k, "strides": s} for f, k, s in self.network], "encoding_dim": self.enc,
                "alpha": self.alpha, "learning_rate": 1e-3, "batch_size": max(self.Bs)}


SHIPPED_NET = ((32, 7, 2), (32, 5, 2), (32, 3, 2))
ODD_S3 = dict(hw=(27, 45), network=((8, 4, 3), (12, 3, 3)), enc=5, alpha=0.1)
CASES = [
    Case("l1", (64, 64), ((8, 5, 2),), 7, 0.1, (1, 9)),
    Case("l8", (64, 64), ((4, 3, 2), (4, 2, 2), (8, 3, 2), (8, 1, 2), (12, 3, 2), (16, 2, 2), (16, 3, 1), (20, 1, 1)), 1, 0.1, (1, 65)),
    Case("s4_s8", (64, 64), ((16, 3, 4), (32, 4, 8)), 130, 0.1, (3, 16)),
    Case("outconv_2048", (64, 64), ((128, 4, 2), (68, 3, 2)), 12, 0.1, (2, 5)),
    Case("outconv_smem", (64, 64), ((376, 1, 4), (8, 3, 4)), 6, 0.1, (2,)),
    Case("odd_s3", Bs=(1, 7), **ODD_S3),
    Case("nonsq_relu", (36, 20), ((4, 6, 2), (8, 5, 2)), 16, 0.0, (4,)),
    Case("linear", (64, 64), ((8, 3, 2), (8, 3, 2)), 10, 1.0, (6,)),
    Case("steep", (64, 64), ((8, 3, 2), (8, 3, 2)), 10, 2.5, (6,)),
]
# targets != inputs (a denoising auto-encoder): the shipped geometry and a non-square one
DENOISE = [
    Case("denoise_shipped", (64, 64), SHIPPED_NET, 100, 0.1, (32,), targets=True),
    Case("denoise_odd_s3", Bs=(7,), targets=True, **ODD_S3),
]
BY_NAME = {c.name: c for c in CASES + DENOISE}


# ------------------------------------------------------------------------------------------------ the handle's geometry
def conv_layer(h, w, c, k, s, f):
    """enc_conv_layer (csrc/enc_tables.cuh): TF 'same' padding, the extra row / column behind."""
    oh, ow = -(-h // s), -(-w // s)
    ph, pw = max((oh - 1) * s + k - h, 0), max((ow - 1) * s + k - w, 0)
    return dict(h=h, w=w, c=c, k=k, s=s, f=f, oh=oh, ow=ow, pt=ph // 2, pb=ph - ph // 2, pl=pw // 2, pr=pw - pw // 2, up=1)


def geometry(case):
    """The encoder convs and the decoder convs (output conv last) of b2g_autoencoder_create, and the output conv's limits."""
    H, W = case.hw
    enc, (h, w, c) = [], (H, W, 1)
    for f, k, s in case.network:
        enc.append(conv_layer(h, w, c, k, s, f))
        h, w, c = enc[-1]["oh"], enc[-1]["ow"], f
    dec = []
    for i in reversed(range(len(case.network))):
        u = case.network[i][2]
        dec.append(dict(conv_layer(h * u, w * u, c, case.network[i][1], 1, case.network[i - 1][0] if i else 1), up=u))
        h, w, c = dec[-1]["oh"], dec[-1]["ow"], dec[-1]["f"]
    o = dec[-1]
    pw = AE_TILE + o["k"] - 1
    out = dict(weights=o["k"] ** 2 * o["c"], smem_fwd=(o["k"] ** 2 * o["c"] + pw * pw * (o["c"] + 1)) * 4,
               smem_wg=pw * pw * (o["c"] + 1) * 4, returns=(h, w) == (H, W))
    return enc, dec, out


def out_conv_limits(k, f):
    pw = AE_TILE + k - 1
    return k * k * f, (k * k * f + pw * pw * (f + 1)) * 4


# ------------------------------------------------------------------------------------------------ CPU: the matrix is complete
def test_matrix_covers_every_geometry_path():
    geo = {c.name: geometry(c) for c in CASES + DENOISE}
    for c in CASES + DENOISE:
        enc, dec, out = geo[c.name]
        assert out["returns"], c.name
        # the restatement agrees with model_shapes (what the GPU tests compare the handle's layer shapes with)
        shapes = model_shapes(c.cfg()["network"], c.enc, c.hw + (1,))
        convs = [s for s, _ in shapes[:len(enc)]] + [s for s, _ in shapes[len(enc) + 2:]]
        assert convs == [(g["k"], g["k"], g["c"], g["f"]) for g in enc + dec], c.name
        assert shapes[len(enc)][0] == (enc[-1]["oh"] * enc[-1]["ow"] * enc[-1]["f"], c.enc), c.name
        assert out["weights"] <= WG_MAX and out["smem_fwd"] <= MAX_SMEM, c.name
        assert all(f % 4 == 0 for f, _, _ in c.network), c.name
    all_enc = [g for n in geo for g in geo[n][0]]
    all_dec = [g for n in geo for g in geo[n][1]]
    assert {len(c.network) for c in CASES} >= {1, 8}
    assert {g["up"] for g in all_dec} >= {1, 2, 3, 4, 8}
    assert any(g["s"] > g["k"] for g in all_enc)
    assert any(g["pt"] != g["pb"] or g["pl"] != g["pr"] for g in all_enc)
    assert any(g["pt"] != g["pb"] or g["pl"] != g["pr"] for g in all_dec)
    assert {g["k"] for g in all_enc + all_dec} >= {1, 2}
    assert any(c.hw[0] != c.hw[1] and c.hw[0] % 8 and c.hw[1] % 8 for c in CASES)
    assert {c.enc % 4 for c in CASES} == {0, 1, 2, 3} and 1 in {c.enc for c in CASES}
    assert any(c.enc > 64 for c in CASES)
    filters = {f for c in CASES for f, _, _ in c.network}
    assert 4 in filters and any(f > 64 for f in filters) and any(f > 64 and f % 64 == 4 for f in filters)
    # both output-conv bounds are reached: a case at the 2048-weight limit, and one where 4 more filters break the
    # shared-memory bound while still inside the weight limit
    outs = {n: (geo[n][1][-1]["k"], geo[n][1][-1]["c"], geo[n][2]) for n in geo}
    assert any(o["weights"] == WG_MAX for _, _, o in outs.values())
    assert any(out_conv_limits(k, f + 4)[1] > MAX_SMEM and out_conv_limits(k, f + 4)[0] <= WG_MAX for k, f, _ in outs.values())
    assert any(o["smem_fwd"] > 48 * 1024 and o["smem_wg"] > 48 * 1024 for _, _, o in outs.values())
    assert {0.0, 1.0} <= {c.alpha for c in CASES} and any(c.alpha > 1 for c in CASES)
    assert any(c.targets for c in DENOISE) and any(c.hw != (64, 64) for c in DENOISE)


def test_refusal_limits_are_the_bounds_they_name():
    """The refusal cases below sit just past one bound and inside the other."""
    assert out_conv_limits(1, 380) == (380, 99056) and out_conv_limits(1, 376)[1] == 98016
    assert out_conv_limits(2, 292)[0] <= WG_MAX and out_conv_limits(2, 292)[1] > MAX_SMEM
    assert out_conv_limits(4, 132)[0] > WG_MAX and out_conv_limits(4, 132)[1] <= MAX_SMEM
    assert out_conv_limits(4, 128) == (2048, 70628)


# ------------------------------------------------------------------------------------------------ CPU: create refusals
def _cfg(network, enc=10, hw=(64, 64), channels=1, alpha=0.1, max_batch=4, n_layers=None):
    cfg = _lib.EncoderCfg()
    cfg.height, cfg.width, cfg.channels = hw[0], hw[1], channels
    cfg.n_layers = len(network) if n_layers is None else n_layers
    for i, (f, k, s) in enumerate(network[:_lib.ENC_MAX_LAYERS]):
        cfg.filters[i], cfg.kernel[i], cfg.strides[i] = f, k, s
    cfg.encoding_dim, cfg.alpha, cfg.max_batch, cfg.device = enc, alpha, max_batch, 0
    return cfg


def _refused(create, destroy, cfg, match):
    lib = _lib.load()
    h = C.c_void_p()
    rc = getattr(lib, create)(C.byref(cfg), C.byref(h))
    if rc == 0:
        getattr(lib, destroy)(h)
    msg = lib.b2g_last_error().decode()
    assert rc == _lib.B2G_EINVAL, (rc, msg)
    assert match in msg, msg


TWO = ((8, 3, 2), (8, 3, 2))


@pytest.mark.parametrize("cfg, match", [
    (_cfg(TWO, alpha=-0.1), "alpha"),
    (_cfg(TWO, alpha=float("nan")), "alpha"),
    (_cfg(TWO, alpha=float("inf")), "alpha"),
    (_cfg(((380, 1, 2),)), "shared memory"),
    (_cfg(((292, 2, 2),)), "shared memory"),
    (_cfg(((132, 4, 2),)), "must be <= 2048"),
    (_cfg(((6, 3, 2), (8, 3, 2))), "multiples of 4"),
    (_cfg(TWO, channels=2), "channels must be 1"),
    (_cfg(((8, 3, 3),)), "decoder returns 66x66"),
    (_cfg(TWO, n_layers=0), "n_layers out of range"),
    (_cfg(TWO * 5, n_layers=9), "n_layers out of range"),
], ids=["alpha_neg", "alpha_nan", "alpha_inf", "k1_f380", "k2_f292", "k4_f132", "filters6", "channels2", "stride3_64",
        "layers0", "layers9"])
def test_autoencoder_create_refusals(cfg, match):
    """Each is B2G_EINVAL naming its reason, before any device is touched (so also on a machine without one)."""
    _refused("b2g_autoencoder_create", "b2g_autoencoder_destroy", cfg, match)


def test_encoder_create_checks_every_layer_for_32bit_offsets():
    """Layer 0's input (9000 x 66 x 66) and output (9000 x 64 x 64 x 4) fit in 32-bit offsets, but the Dense layer's input
    holds 9000 x 64 x 64 x 64 = 2.36e9 floats."""
    cfg = _cfg(((4, 3, 1), (64, 3, 1)), max_batch=9000)
    assert 9000 * 66 * 66 < 2 ** 31 and 9000 * 64 * 64 * 4 < 2 ** 31 and 9000 * 64 * 64 * 64 >= 2 ** 31
    _refused("b2g_encoder_create", "b2g_encoder_destroy", cfg, "32-bit offset")


# ------------------------------------------------------------------------------------------------ GPU helpers
def model_class(hw):
    """SimpleAutoEncoder reads its image geometry from the class attribute input_shape."""
    if tuple(hw) == (64, 64):
        return SimpleAutoEncoder
    return type(f"AutoEncoder{hw[0]}x{hw[1]}", (SimpleAutoEncoder,), {"input_shape": (hw[0], hw[1], 1)})


def images(n, hw, seed):
    """Depth scenes cut to hw: exact zeros on the floor and the gripper band, objects with a little noise."""
    return np.ascontiguousarray(scenes(n, seed)[:, :hw[0], :hw[1]])


def noisy(x, seed):
    """A corrupted copy of x for denoising: sensor noise everywhere and dropped-out pixels."""
    rng = np.random.default_rng(seed)
    y = x + rng.normal(0, 0.02, x.shape).astype(np.float32)
    return np.where(rng.random(x.shape) < 0.05, 0, y).astype(np.float32)


def init(case, seed=3):
    """Glorot kernels; zero biases on even layers (exact-zero LeakyReLU inputs on the zeroed floor), random ones on odd."""
    arrays = glorot(case.cfg(), seed, case.hw + (1,))
    rng = np.random.default_rng(seed + 100)
    return [(k, rng.normal(0, 0.05, b.shape).astype(np.float32) if i % 2 else b) for i, (k, b) in enumerate(arrays)]


def batch(case, n, seed):
    x = images(n, case.hw, seed)
    return (noisy(x, seed + 1), x) if case.targets else x


def check_layer_shapes(ae, case):
    lib, h = _lib.load(), ae._autoencoder(1)
    shapes = model_shapes(case.cfg()["network"], case.enc, case.hw + (1,))
    assert lib.b2g_autoencoder_n_layers(h) == len(shapes) == 2 * len(case.network) + 2
    for i, (ks, nb) in enumerate(shapes):
        kn, bn = C.c_int64(), C.c_int64()
        _lib.check(lib.b2g_autoencoder_layer_shape(h, i, C.byref(kn), C.byref(bn)))
        assert (kn.value, bn.value) == (math.prod(ks), nb), (i, kn.value, bn.value, ks, nb)


def check_predict_and_test(cfg, arrays, cls, x, t=None):
    """predict within 1e-4 of the largest reconstruction, and test (evaluate from the device dataset) within 1e-5."""
    ae = cls(cfg, max_batch=1)
    ae.set_model_weights(arrays)
    ref = R.predict(arrays, x, cfg["network"], cfg["alpha"])
    y = ae.predict(x)
    assert y.shape == x.shape and np.abs(y - ref).max() <= 1e-4 * np.abs(ref).max()
    mse = float(((ref - (x if t is None else t)) ** 2).mean())
    got = ae.test(x, x if t is None else t)
    assert abs(got - mse) <= 1e-5 * mse, (got, mse)
    return ae


def set_dataset(h, x, t):
    fp = C.POINTER(C.c_float)
    _lib.check(_lib.load().b2g_autoencoder_set_dataset(h, x.ctypes.data_as(fp), None if t is None else t.ctypes.data_as(fp), x.shape[0]))


def train_epoch(h, order, bs, lr):
    loss = C.c_double()
    order = np.ascontiguousarray(order, np.int32)
    _lib.check(_lib.load().b2g_autoencoder_train_epoch(h, order.ctypes.data_as(C.POINTER(C.c_int32)), order.size, bs, lr, C.byref(loss)))
    return loss.value


def evaluate(h, start, count):
    loss = C.c_double()
    _lib.check(_lib.load().b2g_autoencoder_evaluate(h, start, count, C.byref(loss)))
    return loss.value


# ------------------------------------------------------------------------------------------------ GPU: the matrix
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES + DENOISE, ids=lambda c: c.name)
def test_case_matches_oracle(case):
    cfg, cls, arrays = case.cfg(), model_class(case.hw), init(case)
    for B in case.Bs:
        b = batch(case, B, seed=10 * B + 1)
        check_step(cfg, arrays, *(b if case.targets else (b,)), cls=cls)
    check_updates(cfg, arrays, [batch(case, max(case.Bs), seed=200 + s) for s in range(3)], cls=cls)
    b = batch(case, 2 * max(case.Bs) + 3, seed=300)          # predict and evaluate in max_batch chunks and a partial one
    ae = check_predict_and_test(cfg, arrays, cls, *(b if case.targets else (b,)))
    check_layer_shapes(ae, case)
    ae.close()


@pytest.mark.gpu
def test_denoising_shipped_weights_step_epoch_and_evaluate():
    """The reference's weights, trained towards clean targets from corrupted inputs: explicit steps alternate with
    one-batch epochs over a device dataset that holds the targets."""
    cfg, arrays = shipped()
    B = 32
    pool_x = images(96, (64, 64), seed=400)
    pool_in = noisy(pool_x, 401)
    orders = [np.random.default_rng(402 + s).permutation(96)[:B] for s in range(4)]
    batches = [(pool_in[o], pool_x[o]) for o in orders]

    def step(ae, s, x, t):
        if s % 2 == 0:
            return ae.step(x, t)
        h = ae._autoencoder(B)
        set_dataset(h, pool_in, pool_x)
        loss = train_epoch(h, orders[s], B, cfg["learning_rate"])
        return loss, ae._pull(_lib.load().b2g_autoencoder_get_grad)
    check_updates(cfg, arrays, batches, step=step)


@pytest.mark.gpu
def test_epoch_graph_and_dataset_changes_match_oracle():
    """Each epoch is one Adam step (n_order == batch: the full-batch graph; n_order < batch: the partial one), held with
    check_updates at the GPU's parameters, through a sequence of datasets: 300 rows -> 100 different rows (no regrow: the
    captured graphs stay and must read the new rows) -> 500 rows (regrow: graphs recaptured) -> the same size with targets
    (regrow for the target buffer) -> other rows without targets (the targets are the inputs again).  After each epoch,
    evaluate at start > 0 over a count that is not a multiple of max_batch, against the oracle at the new parameters."""
    case = BY_NAME["odd_s3"]
    cfg, cls, arrays = dict(case.cfg(), batch_size=16), model_class(case.hw), init(case, seed=9)
    bs, rng = 16, np.random.default_rng(500)
    a, b, c, e = (images(n, case.hw, seed) for n, seed in ((300, 501), (100, 502), (500, 503), (500, 505)))
    d_in = noisy(c, 504)
    plan = []        # (dataset to load or None, targets, the rows the device holds, their targets, order)
    for data, tg, n_order in ((a, None, 16), (None, None, 11), (b, None, 16), (c, None, 16), (d_in, c, 16), (e, None, 11)):
        rows = data if data is not None else plan[-1][2]
        tgts = (tg if tg is not None else rows) if data is not None else plan[-1][3]
        order = rng.choice(rows.shape[0], n_order, replace=False)
        order[0] = rows.shape[0] - 1                 # the last row: past the old capacity after a regrow
        plan.append((data, tg, rows, tgts, order.astype(np.int32)))
    batches = [(rows[o], tgts[o]) for _, _, rows, tgts, o in plan]

    def step(ae, s, x, t):
        data, tg, rows, tgts, order = plan[s]
        h = ae._autoencoder(bs)
        if data is not None:
            set_dataset(h, data, tg)
        loss = train_epoch(h, order, bs, cfg["learning_rate"])
        grads = ae._pull(_lib.load().b2g_autoencoder_get_grad)
        start, count = 5 + s, 37                       # max_batch 16: chunks of 16, 16 and 5
        ref = R.predict(ae.get_weights(), rows[start:start + count], cfg["network"], cfg["alpha"])
        mse = float(((ref - tgts[start:start + count]) ** 2).mean())
        got = evaluate(h, start, count)
        assert abs(got - mse) <= 1e-5 * mse, (s, got, mse)
        return loss, grads
    check_updates(cfg, arrays, batches, cls=cls, step=step)


# ------------------------------------------------------------------------------------------------ GPU: the Python surface
@pytest.mark.gpu
def test_negative_alpha_encodes_but_does_not_train(tmp_path):
    """The encoder forward is right for any alpha; training reads the LeakyReLU derivative from the sign of the stored
    output, which alpha < 0 makes ambiguous, so the training handle refuses it."""
    cfg = dict(BY_NAME["linear"].cfg(), alpha=-0.2)
    ae = SimpleAutoEncoder(cfg, max_batch=4)
    arrays = glorot(cfg)
    ae.set_model_weights(arrays)
    x = images(4, (64, 64), seed=600) - 0.1                  # negative pixels: both LeakyReLU sides
    ref = E.encode(x, arrays[:3], [2, 2], -0.2, torch.float64)
    z = ae.encode(x)
    assert np.abs(z - ref).max() <= 1e-4 * np.abs(ref).max()
    with pytest.raises(_lib.B2GError, match="alpha"):
        ae.predict(x)
    with pytest.raises(_lib.B2GError, match="alpha"):
        SimpleAutoEncoder(cfg, max_batch=4, seed=0).train(images(20, (64, 64), seed=601), None, 4, 1, str(tmp_path))
    ae.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["l1", "l8"])
def test_weights_round_trip_is_bit_exact(name, tmp_path):
    """save_weights -> load_weights through the device arena (filter strides padded to 4) and model.h5."""
    case = BY_NAME[name]
    cfg = case.cfg()
    arrays = init(case, seed=11)
    ae = SimpleAutoEncoder(cfg, max_batch=2)
    ae.set_model_weights(arrays)
    x = images(2, (64, 64), seed=700)
    y = ae.predict(x)                         # the handle holds the weights; save_weights reads them back from it
    ae.save_weights(str(tmp_path / "model.h5"))
    fresh = SimpleAutoEncoder(cfg, max_batch=2)
    fresh.load_weights(str(tmp_path))
    assert np.array_equal(fresh.predict(x), y)
    for (k0, b0), (k1, b1) in zip(arrays, fresh.get_weights()):
        assert k0.shape == k1.shape and np.array_equal(k0, k1) and np.array_equal(b0, b1)
    ae.close()
    fresh.close()
