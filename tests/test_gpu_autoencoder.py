"""Auto-encoder training (encoders.py:40-61 train / test / predict) on the GPU, through the C ABI, against the float64
oracle of tests/ae_ref.py: explicit steps from the shipped weights and from Glorot init, a non-shipped geometry, predict and
test, an epoch from a device-resident dataset, and the train_encoder command line end to end."""
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch
import yaml

import b200grasp  # noqa: F401
from b200grasp import _lib, h5min, synth
from b200grasp.encoders import SimpleAutoEncoder, glorot_init, keras_layer_names, model_shapes
from tests import ae_ref as R
from tests.test_encoder_cpu import load_fixture

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OTHER = {"network": [{"filters": 8, "kernel_size": 3, "strides": 1}, {"filters": 16, "kernel_size": 4, "strides": 2},
                     {"filters": 16, "kernel_size": 5, "strides": 2}], "encoding_dim": 20, "alpha": 0.2, "learning_rate": 1e-3,
         "batch_size": 16}


def rel_err(a, b):
    return float(np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-30))


def scenes(n, seed):
    """Preprocessed depth scenes: objects on a zeroed floor, a zeroed gripper band, a little sensor noise on the objects."""
    x = synth.make_depth_scenes(n, seed=seed)
    rng = np.random.default_rng(seed + 1)
    x = np.where(x > 0, x + rng.normal(0, 0.01, x.shape).astype(np.float32), 0).astype(np.float32)
    x[:, 56:, 20:44] = 0
    return x


def shipped():
    w, cfg = load_fixture()
    arrays = [(w[f"{n}/kernel"], w[f"{n}/bias"]) for n in keras_layer_names(3)]
    return dict(cfg, learning_rate=2e-4, batch_size=128), arrays


def glorot(cfg, seed=3, input_shape=(64, 64, 1)):
    return glorot_init(model_shapes(cfg["network"], cfg["encoding_dim"], input_shape), np.random.default_rng(seed))


def grad_bars(arrays, x, cfg, ref, t=None):
    """Gradient bar of each tensor: 1e-4 of its largest element, or 3x the distance of the fp32 oracle from the float64 one
    when fp32 itself cannot resolve the tensor that well: a LeakyReLU input within fp32 rounding of zero takes slope 1 on one
    side and alpha on the other, and which side an fp32 forward lands on is decided by rounding.  t: the targets (None: x)."""
    _, r32 = R.loss_and_grads(arrays, x, x if t is None else t, cfg["network"], cfg["alpha"], torch.float32)
    return [max(1e-4, 3 * rel_err(a32, a64)) for kb32, kb64 in zip(r32, ref) for a32, a64 in zip(kb32, kb64)]


def check_step(cfg, arrays, x, t=None, cls=SimpleAutoEncoder):
    """Loss and every gradient of one explicit step against the float64 oracle.  t: the targets (None: the inputs);
    cls: the model class, whose input_shape sets the image geometry."""
    ae = cls(cfg, max_batch=1)
    ae.set_model_weights(arrays)
    loss, grads = ae.step(x, t, apply_update=False)
    ref_loss, ref = R.loss_and_grads(arrays, x, x if t is None else t, cfg["network"], cfg["alpha"])
    assert abs(loss - ref_loss) <= 1e-5 * ref_loss, (loss, ref_loss)
    bars = grad_bars(arrays, x, cfg, ref, t)
    for i, (a, b) in enumerate(zip((a for kb in grads for a in kb), (b for kb in ref for b in kb))):
        assert rel_err(a, b) <= bars[i], (i, rel_err(a, b), bars[i])
    ae.close()
    return ref


def explicit_step(ae, s, x, t):
    """The default step of check_updates: one explicit Adam step on the host batch; returns (loss, gradients)."""
    return ae.step(x, t)


def check_updates(cfg, arrays, batches, cls=SimpleAutoEncoder, step=explicit_step):
    """Parameter change of every Adam step and of the whole run, against Keras Adam in float64 applied along the GPU's own
    trajectory: at each step the oracle takes the float64 gradient at the GPU's current parameters (the GPU's gradient must
    be within the gradient bar of it, see grad_bars) and its own moments.  The two updates may then
    differ by 1e-3 of the largest update plus what a gradient error at that bar, carried in Adam's moments, can move:
    Keras Adam moves every weight by about lr whatever the size of its gradient (eps = 1e-7), so a gradient that fp32
    cannot resolve still moves its weight by up to 2 lr.  Anchoring each step at the GPU's parameters keeps the comparison
    from following two trajectories that drift apart through exactly those weights.  One ulp of each fp32 parameter is
    added to its allowance at every step: the GPU cannot store a change more finely than that.

    batches: host batches x, or (inputs, targets) pairs.  step(ae, s, x, t) makes the GPU's Adam step s on that batch (t is
    None when the targets are the inputs) and returns (its loss, taken before the update, and its gradients); an epoch
    whose order covers exactly that batch can stand in for the explicit step."""
    ae = cls(cfg, max_batch=1)
    ae.set_model_weights(arrays)
    opt = R.Adam(arrays, cfg["learning_rate"])
    p0 = [np.array(a, np.float64) for kb in ae.get_weights() for a in kb]
    em = [np.zeros(a.shape) for a in p0]             # bounds on |m_gpu - m_ref| and |v_gpu - v_ref|
    ev = [np.zeros(a.shape) for a in p0]
    total_ref = [np.zeros(a.shape) for a in p0]
    total_allow = [np.zeros(a.shape) for a in p0]
    cur = p0
    for s, b in enumerate(batches):
        x, t = b if isinstance(b, tuple) else (b, None)
        opt.p = [a.copy() for a in cur]
        ref_loss, g = R.loss_and_grads(opt.arrays(), x, x if t is None else t, cfg["network"], cfg["alpha"])
        loss, gg = step(ae, s, x, t)
        assert abs(loss - ref_loss) <= 1e-5 * ref_loss, (s + 1, loss, ref_loss)
        gflat = [a for kb in g for a in kb]
        bars = grad_bars(opt.arrays(), x, cfg, g, t)
        for i, (a, b) in enumerate(zip(gflat, (b for kb in gg for b in kb))):
            assert rel_err(b, a) <= bars[i], (s + 1, i, rel_err(b, a), bars[i])
            d = bars[i] * np.abs(a).max()
            em[i] = opt.b1 * em[i] + (1 - opt.b1) * d
            ev[i] = opt.b2 * ev[i] + (1 - opt.b2) * d * (2 * np.abs(a) + d)
        u_ref = opt.update(g)
        allow = opt.update_bound(g, em, ev)
        opt.step(g)
        nxt = [np.array(a, np.float64) for kb in ae.get_weights() for a in kb]
        errs = []
        for i in range(len(p0)):
            # each parameter is stored in fp32, so its change is resolved only to an ulp of the parameter; that matters
            # where the gradient is so small that Adam's eps shrinks the whole update to a few ulps (deep, narrow nets)
            allow[i] = allow[i] + np.spacing(np.maximum(np.abs(cur[i]), np.abs(nxt[i])).astype(np.float32)).astype(np.float64)
            total_ref[i] += u_ref[i]
            total_allow[i] += allow[i]
            for got, ref, al in ((nxt[i] - cur[i], u_ref[i], allow[i]), (nxt[i] - p0[i], total_ref[i], total_allow[i])):
                over = np.abs(got - ref) - 1e-3 * np.abs(ref).max() - al
                errs.append((i, float(over.max()), float(np.abs(got - ref).max() / np.abs(ref).max()), float(np.abs(ref).max())))
        assert all(e[1] <= 0 for e in errs), (s + 1, [e for e in errs if e[1] > 0])
        cur = nxt
    ae.close()


@pytest.mark.parametrize("init", ["shipped", "glorot"])
@pytest.mark.parametrize("B", [128, 72, 1])
def test_explicit_step_matches_oracle(init, B):
    cfg, arrays = shipped()
    if init == "glorot":
        arrays = glorot(cfg)
    x = scenes(B, seed=B)
    check_step(cfg, arrays, x)
    check_updates(cfg, arrays, [scenes(B, seed=100 * B + s) for s in range(10)])


@pytest.mark.parametrize("B", [16, 3])
def test_other_geometry_matches_oracle(B):
    cfg = OTHER
    arrays = glorot(cfg, seed=B)
    arrays = [(k, np.random.default_rng(i).normal(0, 0.05, b.shape).astype(np.float32)) for i, (k, b) in enumerate(arrays)]
    x = scenes(B, seed=7 + B)
    check_step(cfg, arrays, x)
    check_updates(cfg, arrays, [scenes(B, seed=70 + s) for s in range(3)])


def test_glorot_first_step_has_exact_zeros():
    """Zero biases and zeroed image regions give pre-activations of exactly 0; the gradient through them must be 0."""
    cfg, _ = shipped()
    arrays = glorot(cfg)
    x = scenes(8, seed=5)
    ref = check_step(cfg, arrays, x)
    assert all(np.isfinite(k).all() for k, _ in ref)


def test_predict_and_test_match_oracle():
    cfg, arrays = shipped()
    ae = SimpleAutoEncoder(cfg, max_batch=1)
    ae.set_model_weights(arrays)
    x = scenes(300, seed=21)
    ref = R.predict(arrays, x, cfg["network"], cfg["alpha"])
    y = ae.predict(x)
    assert y.shape == x.shape and y.dtype == np.float32
    assert np.abs(y - ref).max() <= 1e-4 * np.abs(ref).max()
    mse = float(((ref - x) ** 2).mean())
    assert abs(ae.test(x, x) - mse) <= 1e-5 * mse
    ae.close()


def test_epoch_matches_explicit_steps():
    cfg, arrays = shipped()
    x = scenes(300, seed=31)
    order = np.random.default_rng(4).permutation(300).astype(np.int32)
    a = SimpleAutoEncoder(cfg, max_batch=1)
    a.set_model_weights(arrays)
    ae = a._autoencoder(128)
    import ctypes as C
    fp = C.POINTER(C.c_float)
    lib = _lib.load()
    _lib.check(lib.b2g_autoencoder_set_dataset(ae, x.ctypes.data_as(fp), None, 300))
    loss = C.c_double()
    _lib.check(lib.b2g_autoencoder_train_epoch(ae, order.ctypes.data_as(C.POINTER(C.c_int32)), 300, 128, cfg["learning_rate"],
                                               C.byref(loss)))
    b = SimpleAutoEncoder(cfg, max_batch=1)
    b.set_model_weights(arrays)
    losses, sizes = [], []
    for s in range(0, 300, 128):
        rows = order[s:s + 128]
        losses.append(b.step(x[rows])[0])
        sizes.append(rows.size)
    mean = float(np.dot(losses, sizes) / 300)
    assert abs(loss.value - mean) <= 1e-4 * mean, (loss.value, mean)
    p0 = np.concatenate([q.reshape(-1) for kb in arrays for q in kb]).astype(np.float64)
    pa = np.concatenate([q.reshape(-1) for kb in a.get_weights() for q in kb]).astype(np.float64)
    pb = np.concatenate([q.reshape(-1) for kb in b.get_weights() for q in kb]).astype(np.float64)
    # Adam's first steps move every weight by about lr whatever its gradient's size, so a near-zero gradient whose fp32 sign
    # differs between the two runs (atomics sum in run-dependent order) moves one weight by 2 lr: compare in norm
    assert np.linalg.norm(pa - pb) <= 1e-2 * np.linalg.norm(pb - p0)
    # a second epoch replays the captured graphs
    _lib.check(lib.b2g_autoencoder_train_epoch(ae, order.ctypes.data_as(C.POINTER(C.c_int32)), 300, 128, cfg["learning_rate"],
                                               C.byref(loss)))
    assert np.isfinite(loss.value)
    a.close(); b.close()


def test_train_checkpoints_the_best_epoch(tmp_path):
    cfg = dict(shipped()[0], learning_rate=1e-3)
    x = scenes(400, seed=41)
    ae = SimpleAutoEncoder(cfg, max_batch=1, seed=0)
    best = {}
    orig = ae.save_weights

    def save(path):
        best["w"] = [(k.copy(), b.copy()) for k, b in ae.get_weights()]
        orig(path)
    ae.save_weights = save
    hist = ae.train(x, x, 64, 4, str(tmp_path))
    assert len(hist["loss"]) == len(hist["val_loss"]) == 4
    rows = open(tmp_path / "history.csv").read().splitlines()
    assert rows[0] == "epoch,loss,val_loss" and len(rows) == 5
    assert hist["val_loss"][-1] < hist["val_loss"][0]
    # the model keeps the last epoch; model.h5 holds the best one, bit for bit
    fresh = SimpleAutoEncoder(cfg, max_batch=8)
    fresh.load_weights(str(tmp_path))
    ref = SimpleAutoEncoder(cfg, max_batch=8)
    ref.set_model_weights(best["w"])
    probe = x[:8]
    assert np.array_equal(fresh.encode(probe), ref.encode(probe))
    assert np.array_equal(fresh.predict(probe), ref.predict(probe))
    last = SimpleAutoEncoder(cfg, max_batch=8)
    last.set_model_weights(ae.get_weights())
    assert np.array_equal(ae.encode(probe), last.encode(probe))
    for o in (ae, fresh, ref, last):
        o.close()


def _pickle(path, n_train, n_test, seed):
    rng = np.random.default_rng(seed)

    def part(n, s):
        depth = synth.make_depth_scenes(n, seed=s)
        floor = rng.uniform(0.55, 0.6, depth.shape).astype(np.float32)
        masks = np.where(depth > 0, 2, 0).astype(np.int32)
        masks[:, 56:, 20:44] = 5                                   # the gripper: mask == max
        return {"rgb": np.zeros(depth.shape[:3] + (3,), np.uint8), "depth": np.where(depth > 0, depth, floor), "masks": masks}
    with open(path, "wb") as f:
        pickle.dump({"train": part(n_train, seed), "test": part(n_test, seed + 1)}, f)


def test_train_encoder_cli_end_to_end(tmp_path):
    data = tmp_path / "imgs.pkl"
    _pickle(data, 640, 96, 50)
    cfg = {"batch_size": 64, "data_path": str(data), "encoding_dim": 100, "epochs": 5, "learning_rate": 1e-3,
           "network": [{"filters": 32, "kernel_size": 7, "strides": 2}, {"filters": 32, "kernel_size": 5, "strides": 2},
                       {"filters": 32, "kernel_size": 3, "strides": 2}]}
    cpath = tmp_path / "cfg.yaml"
    cpath.write_text(yaml.safe_dump(cfg))
    model_dir = tmp_path / "model"
    env = dict(os.environ, PYTHONPATH=ROOT)
    run = lambda *a: subprocess.run([sys.executable, "-m", "b200grasp.train_encoder", str(model_dir), *a], cwd=ROOT, env=env,
                                    capture_output=True, text=True, timeout=900)
    r = run("train", "--config", str(cpath), "--seed", "1")
    assert r.returncode == 0, r.stderr[-3000:]
    rows = (model_dir / "history.csv").read_text().splitlines()
    assert len(rows) == 1 + cfg["epochs"]
    hist = np.array([[float(v) for v in row.split(",")] for row in rows[1:]])
    from b200grasp.train_encoder import _load_data_set, _preprocess_depth
    train = _preprocess_depth(_load_data_set(str(data), False))
    val = train[int(640 * 0.9):]
    assert hist[-1, 2] < hist[0, 2] and hist[-1, 2] < float((val.astype(np.float64) ** 2).mean())
    assert yaml.safe_load((model_dir / "config.yaml").read_text()) == cfg
    r = run("test")
    assert r.returncode == 0, r.stderr[-3000:]
    got = float(r.stdout.strip().split("Test loss: ")[-1])
    w = h5min.load_keras_weights(str(model_dir / "model.h5"))
    arrays = [(w[f"{n}/kernel"], w[f"{n}/bias"]) for n in keras_layer_names(3)]
    test = _preprocess_depth(_load_data_set(str(data), True))
    ref = float(((R.predict(arrays, test, cfg["network"], 0.1) - test) ** 2).mean())
    assert abs(got - ref) <= 1e-5 * ref, (got, ref)


def test_non_returning_geometry_is_refused():
    cfg = {"network": [{"filters": 8, "kernel_size": 3, "strides": 1}, {"filters": 8, "kernel_size": 3, "strides": 2},
                       {"filters": 8, "kernel_size": 3, "strides": 3}], "encoding_dim": 10}
    ae = SimpleAutoEncoder(cfg, max_batch=1)
    ae.set_model_weights(glorot(cfg))
    with pytest.raises(_lib.B2GError, match="decoder returns"):
        ae.predict(np.zeros((1, 64, 64, 1), np.float32))
    ae.close()
