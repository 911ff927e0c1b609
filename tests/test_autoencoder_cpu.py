"""Auto-encoder training, CPU side: the model.h5 writer against the shipped Keras file, Keras fit's bookkeeping driven by
fakes, and the float64 oracle's gradient against finite differences."""
import csv
import gzip
import os

import numpy as np
import pytest
import torch

import b200grasp  # noqa: F401
from b200grasp import h5min
from b200grasp.encoders import fit, glorot_init, keras_layer_names, model_shapes
from tests import ae_ref as R
from tests.test_encoder_cpu import SAMPLED_H5, load_fixture
from tests.util import GOLD


def _layers(w, n_conv=3):
    names = keras_layer_names(n_conv)
    ws = [(f"{n}/{t}:0", w[f"{n}/{t}"]) for n in names for t in ("kernel", "bias")]
    return [("input_1", []), ("encoder", ws[:2 * (n_conv + 1)]), ("decoder", ws[2 * (n_conv + 1):])]


def test_writer_round_trip_and_keras_structure(tmp_path):
    w, _ = load_fixture()
    out = tmp_path / "model.h5"
    h5min.write_keras_weights(str(out), _layers(w))
    got = h5min.load_keras_weights(str(out))
    assert sorted(got) == sorted(w)
    for k in w:
        assert got[k].dtype == w[k].dtype and np.array_equal(got[k], w[k]), k
    shipped = tmp_path / "shipped.h5"
    shipped.write_bytes(gzip.decompress(open(os.path.join(GOLD, SAMPLED_H5), "rb").read()))
    a, b = h5min.read_structure(str(out)), h5min.read_structure(str(shipped))
    assert sorted(a) == sorted(b)
    for k in b:
        if isinstance(b[k], dict):       # groups: the attributes Keras' load_weights reads
            assert sorted(a[k]) == sorted(b[k]), k
            for name in b[k]:
                x, y = a[k][name], b[k][name]
                if isinstance(y, np.ndarray):
                    assert isinstance(x, np.ndarray) and x.dtype == y.dtype and x.shape == y.shape, (k, name)
                else:
                    assert x == y, (k, name)
        else:                            # datasets: shape and dtype
            assert a[k] == b[k], k
    assert b["/"]["layer_names"] == [b"input_1", b"encoder", b"decoder"]
    assert b["/"]["keras_version"] == b"2.2.4" and b["/"]["backend"] == b"tensorflow"


def test_writer_handles_many_layers(tmp_path):
    """More children than one symbol node holds (8) spill into further nodes of the group's B-tree."""
    arrs = [(f"conv2d_{i}/kernel:0", np.full((2, 3), i, np.float32)) for i in range(1, 21)]
    out = tmp_path / "m.h5"
    h5min.write_keras_weights(str(out), [("encoder", arrs)])
    got = h5min.load_keras_weights(str(out))
    assert sorted(got) == sorted(f"conv2d_{i}/kernel" for i in range(1, 21))
    assert all(np.array_equal(got[f"conv2d_{i}/kernel"], np.full((2, 3), i, np.float32)) for i in range(1, 21))


class _Fake:
    def __init__(self, val_losses):
        self.val, self.epochs, self.saved, self.batches, self.n_order = list(val_losses), 0, [], [], []

    def train_epoch(self, order, bs):
        self.n_order.append(np.array(order))
        sizes = [min(bs, order.size - s) for s in range(0, order.size, bs)]
        self.batches.append(sizes)
        losses = [0.1 * (i + 1) for i in range(len(sizes))]          # batch losses; the epoch loss is their weighted mean
        return float(np.dot(losses, sizes) / order.size)

    def evaluate(self, start, count):
        self.eval_slice = (start, count)
        v = self.val[self.epochs]
        self.epochs += 1
        return v


def test_fit_split_batches_and_epoch_mean(tmp_path):
    f = _Fake([1.0, 0.5])
    hist = fit(18000, 128, 2, f.train_epoch, f.evaluate, f.saved.append, str(tmp_path / "h.csv"), np.random.default_rng(0))
    assert f.eval_slice == (16200, 1800)
    assert f.batches[0] == [128] * 126 + [72]
    for o in f.n_order:
        assert sorted(o.tolist()) == list(range(16200))          # only training rows, reshuffled every epoch
    assert not np.array_equal(f.n_order[0], f.n_order[1])
    sizes = np.array(f.batches[0])
    expect = np.dot(0.1 * np.arange(1, 128), sizes) / 16200
    assert hist["loss"][0] == pytest.approx(expect, rel=1e-12) and hist["val_loss"] == [1.0, 0.5]


def test_fit_checkpoint_on_strict_improvement_and_early_stop(tmp_path):
    val = [1.0, 0.9, 0.9, 0.95] + [0.9] * 30
    f = _Fake(val)
    hist = fit(100, 10, 200, f.train_epoch, f.evaluate, f.saved.append, None, np.random.default_rng(1))
    assert f.saved == [0, 1]                  # 0.9 again is not an improvement
    assert len(hist["val_loss"]) == 1 + 1 + 25   # stops on the 25th epoch after the last improvement (epoch 1)
    f = _Fake([1.0 - 0.01 * i for i in range(40)])
    hist = fit(100, 10, 40, f.train_epoch, f.evaluate, f.saved.append, None, np.random.default_rng(1))
    assert len(hist["loss"]) == 40 and f.saved == list(range(40))


def test_history_csv_matches_the_shipped_format(tmp_path):
    shipped = open(os.path.join(GOLD, "encoder_history_head.csv"), newline="").read()
    rows = list(csv.reader(shipped.splitlines()))
    vals = [(float(r[1]), float(r[2])) for r in rows[1:]]
    it = iter(vals)
    cur = {}

    def train_epoch(order, bs):
        cur["v"] = next(it)
        return cur["v"][0]
    path = tmp_path / "history.csv"
    fit(100, 10, len(vals), train_epoch, lambda s, c: cur["v"][1], lambda e: None, str(path), np.random.default_rng(0))
    assert open(path, newline="").read() == shipped


def test_glorot_limits_and_zero_biases():
    _, cfg = load_fixture()
    shapes = model_shapes(cfg["network"], cfg["encoding_dim"])
    w, _ = load_fixture()
    assert [s for s, _ in shapes] == [w[f"{n}/kernel"].shape for n in keras_layer_names(3)]
    arrs = glorot_init(shapes, np.random.default_rng(0))
    for (k, b), (shape, nb) in zip(arrs, shapes):
        rf = int(np.prod(shape[:-2])) if len(shape) > 2 else 1
        lim = np.sqrt(6.0 / (rf * (shape[-2] + shape[-1])))
        assert k.shape == shape and k.dtype == np.float32 and np.abs(k).max() <= lim and np.abs(k).max() > 0.9 * lim
        assert b.shape == (nb,) and not b.any()


TINY = [{"filters": 4, "kernel_size": 3, "strides": 2}, {"filters": 4, "kernel_size": 2, "strides": 2}]


def test_oracle_gradient_matches_finite_differences():
    rng = np.random.default_rng(0)
    shapes = model_shapes(TINY, 5, (8, 8, 1))
    arrays = [(rng.normal(0, 0.4, s), rng.normal(0, 0.1, nb)) for s, nb in shapes]
    x = rng.uniform(0, 1, (3, 8, 8, 1))
    t = rng.uniform(0, 1, (3, 8, 8, 1))
    loss, grads = R.loss_and_grads(arrays, x, t, TINY, 0.2)

    def f(arrs):
        return R.loss_and_grads(arrs, x, t, TINY, 0.2)[0]
    h = 1e-6
    for li in range(len(arrays)):
        for which in (0, 1):
            a = arrays[li][which]
            for idx in list(np.ndindex(a.shape))[:: max(1, a.size // 6)]:
                plus = [(k.copy(), b.copy()) for k, b in arrays]
                minus = [(k.copy(), b.copy()) for k, b in arrays]
                plus[li][which][idx] += h
                minus[li][which][idx] -= h
                fd = (f(plus) - f(minus)) / (2 * h)
                assert abs(fd - grads[li][which][idx]) <= 1e-6 + 1e-5 * abs(fd), (li, which, idx)


def test_leaky_relu_gradient_at_zero_is_zero():
    x = torch.tensor([-1.0, 0.0, 2.0], dtype=torch.float64, requires_grad=True)
    R.lrelu(x, 0.1).sum().backward()
    assert x.grad.tolist() == [0.1, 0.0, 1.0]
    # torch's own leaky_relu would give alpha at 0: the oracle must not use it
    y = torch.tensor([0.0], dtype=torch.float64, requires_grad=True)
    torch.nn.functional.leaky_relu(y, 0.1).sum().backward()
    assert y.grad.item() != 0.0


def test_oracle_adam_is_keras_adam():
    opt = R.Adam([(np.array([1.0]), np.array([0.0]))], lr=0.1)
    opt.step([(np.array([0.5]), np.array([0.0]))])
    # t = 1: lr_t = lr * sqrt(1 - b2) / (1 - b1); m = 0.05, v = 0.00025 -> step = lr_t * m / (sqrt(v) + 1e-7)
    lr_t = 0.1 * np.sqrt(1 - 0.999) / (1 - 0.9)
    assert opt.p[0][0] == pytest.approx(1.0 - lr_t * 0.05 / (np.sqrt(0.00025) + 1e-7), rel=1e-14)
    assert opt.p[1][0] == 0.0


def test_oracle_adam_update_bound_covers_moment_errors():
    """update_bound holds for a second Adam whose gradients are off by up to d at every step (the bound the GPU test uses)."""
    rng = np.random.default_rng(3)
    shape = (4000,)
    a = R.Adam([(np.zeros(shape), np.zeros(1))], lr=2e-4)
    b = R.Adam([(np.zeros(shape), np.zeros(1))], lr=2e-4)
    em, ev = [np.zeros(shape), np.zeros(1)], [np.zeros(shape), np.zeros(1)]
    for _ in range(10):
        g = rng.normal(0, 1, shape) * rng.choice([1e-9, 1e-6, 1e-3, 1.0], shape)
        d = 1e-4 * np.abs(g).max()
        gb = g + rng.uniform(-d, d, shape)
        em[0] = a.b1 * em[0] + (1 - a.b1) * d
        ev[0] = a.b2 * ev[0] + (1 - a.b2) * d * (2 * np.abs(g) + d)
        grads, grads_b = [(g, np.zeros(1))], [(gb, np.zeros(1))]
        bound = a.update_bound(grads, em, ev)[0]
        diff = np.abs(a.update(grads)[0] - b.update(grads_b)[0])
        assert (diff <= bound * (1 + 1e-9) + 1e-18).all()
        a.step(grads)
        b.step(grads_b)
