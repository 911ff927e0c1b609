"""The auto-encoder's bf16x3 training handle (b2g_autoencoder_create2(cfg, B2G_PREC_BF16X3), SimpleAutoEncoder(...,
train_precision="bf16x3")) on the GPU.

Every contraction of one explicit step is held, element by element, to a float64 contraction of the operands the GPU read
(b2g_debug_autoencoder_tensor), within the wgmma engine's error model (tests/gg_tc_ref.py: SPLIT2 plus U_TC per k-step,
gg_gammas(K, split_k, x3=1), whose U32 per split covers the double-atomic accumulation of the weight gradients) times the
sum of |products|.  The contractions that stay on the CUDA cores (conv1's forward and weight gradient, the output conv) are
held to the same bar, which their double sums meet with room to spare.  Then Adam on the GPU's own gradients, predict and
evaluate, the epoch graph against explicit steps, training quality against fp32, and the defaults.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import b200grasp  # noqa: F401
from b200grasp import _lib, synth
from b200grasp.encoders import SimpleAutoEncoder
from tests import ae_ref as R
from tests.gg_tc_ref import gg_gammas
from tests.test_gpu_autoencoder import glorot, scenes, shipped
from tests.test_gpu_autoencoder_configs import BY_NAME, CASES, DENOISE, batch, geometry, init, model_class, set_dataset, train_epoch

pytestmark = pytest.mark.gpu
F64 = np.float64
U32 = 2.0 ** -24
SHIPPED_CFG, SHIPPED_ARRAYS = shipped()


def cdiv(a, b):
    return -(-a // b)


def read(ae, layer, which):
    lib, h = _lib.load(), ae._ae
    n = lib.b2g_debug_autoencoder_tensor_numel(h, layer, which)
    out = np.empty(n, np.float32)
    _lib.check(lib.b2g_debug_autoencoder_tensor(h, layer, which, out.ctypes.data_as(C.POINTER(C.c_float)), n, None))
    return out.astype(F64)


def engines(ae, layer):
    on = (C.c_int32 * 3)()
    _lib.check(_lib.load().b2g_debug_autoencoder_tensor(ae._ae, layer, 0, None, 0, on))
    return tuple(on)


def lrelu(x, a):
    return np.where(x > 0, x, a * x)


def lgrad(m, a):
    """gg_simt / gg_tc GG_EPI_LRELU_GRAD: 1 / alpha / 0 for a stored output > 0 / < 0 / == 0."""
    return np.where(m > 0, 1.0, np.where(m < 0, a, 0.0))


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x, F64))


def conv(x, w, s):
    """x [n, H, W, c] (already bordered), w HWIO -> [n, oh, ow, f] (valid, stride s), float64."""
    return torch.nn.functional.conv2d(t(x).permute(0, 3, 1, 2), t(w).permute(3, 2, 0, 1), stride=s).permute(0, 2, 3, 1).numpy()


def conv_dx(shape, w, dz, s):
    """Gradient w.r.t. a bordered input [n, H, W, c] of conv(x, w, s) given dz [n, oh, ow, f]."""
    n, H, W, c = shape
    g = torch.nn.grad.conv2d_input((n, c, H, W), t(w).permute(3, 2, 0, 1), t(dz).permute(0, 3, 1, 2), stride=s)
    return g.permute(0, 2, 3, 1).numpy()


def conv_dw(x, wshape, dz, s):
    k, _, c, f = wshape
    g = torch.nn.grad.conv2d_weight(t(x).permute(0, 3, 1, 2), (f, c, k, k), t(dz).permute(0, 3, 1, 2), stride=s)
    return g.permute(2, 3, 1, 0).numpy()


class Layers:
    """The handle's layer list (autoencoder.cu): geometry, buffer views and the GPU's tensors after one step on n samples."""

    def __init__(self, ae, case_hw, network, enc, n, max_batch):
        class _C:
            pass
        c = _C()
        c.hw, c.network = case_hw, network
        encg, decg, _ = geometry(c)
        self.L = len(network)
        self.encg, self.decg, self.enc, self.n, self.N = encg, decg, enc, n, max_batch
        self.zs = cdiv(enc, 4) * 4
        self.ae = ae

    def conv_geo(self, j):
        return self.encg[j] if j < self.L else self.decg[j - self.L - 2]

    def conv_in(self, j):
        """Bordered input [n, hp, wp, c] of conv j."""
        g = self.conv_geo(j)
        hp, wp = g["h"] + g["pt"] + g["pb"], g["w"] + g["pl"] + g["pr"]
        return read(self.ae, j, 0).reshape(self.N, hp, wp, g["c"])[:self.n]

    def interior(self, j):
        g = self.conv_geo(j)
        x = self.conv_in(j)
        return x[:, g["pt"]:g["pt"] + g["h"], g["pl"]:g["pl"] + g["w"], :]

    def dz(self, j):
        """Pre-activation gradient of layer j: convs [n, oh, ow, f], dense [n, f]."""
        if j in (self.L, self.L + 1):
            f = self.enc if j == self.L else self.dense_f()
            fs = cdiv(f, 4) * 4
            return read(self.ae, j, 2).reshape(self.N, fs)[:self.n, :f]
        g = self.conv_geo(j)
        dh, dw = g["h"] + g["pt"] + g["k"] - 1, g["w"] + g["pl"] + g["k"] - 1
        D = read(self.ae, j, 2).reshape(self.N, dh, dw, g["f"])[:self.n]
        k, s = g["k"], g["s"]
        return D[:, k - 1:k - 1 + (g["oh"] - 1) * s + 1:s, k - 1:k - 1 + (g["ow"] - 1) * s + 1:s, :]

    def dense_f(self):
        g = self.encg[-1]
        return g["oh"] * g["ow"] * g["f"]

    def out_map(self, j):
        """The stored LeakyReLU output of conv j as [n, oh, ow, f] (where the next layer reads it)."""
        if j < self.L - 1:
            return self.interior(j + 1)
        if j == self.L - 1:
            return read(self.ae, self.L, 0).reshape(self.N, -1)[:self.n].reshape(self.n, self.encg[j]["oh"], self.encg[j]["ow"], -1)
        g = self.conv_geo(j)
        return read(self.ae, j, 1).reshape(self.N, g["oh"], g["ow"], g["f"])[:self.n]


def hold(fails, worst, name, got, ref, bar):
    err = np.abs(np.asarray(got, F64) - ref)
    ratio = np.where(bar > 0, err / np.where(bar > 0, bar, 1), np.where(err > 0, np.inf, 0))
    w = float(ratio.max()) if ratio.size else 0.0
    worst[name] = w
    if w > 1:
        i = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
        fails.append(f"{name}: err/bar {w:.3g} at {i}: got {np.asarray(got)[i]!r} ref {ref[i]!r} bar {bar[i]:.3g}")


def check_contractions(ae, cfg, arrays, x, tg, hw):
    """One explicit step (no update) on x; every contraction against float64 of the GPU's own operands."""
    n = x.shape[0]
    loss, grads = ae.step(x, tg, apply_update=False)
    assert np.isfinite(loss)
    net = [(l["filters"], l["kernel_size"], l["strides"]) for l in cfg["network"]]
    Ly = Layers(ae, hw, net, cfg["encoding_dim"], n, ae._ae_batch)
    L, a = Ly.L, cfg["alpha"]
    A = max(1.0, a)
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    fails, worst = [], {}
    nlay = 2 * L + 2
    for j in range(nlay):
        kind = "enc" if j < L else "encd" if j == L else "decd" if j == L + 1 else "dec"
        W, b = (np.asarray(v, F64) for v in arrays[j])
        gW, gb = (np.asarray(v, F64) for v in grads[j])
        if kind in ("enc", "dec"):
            g = Ly.conv_geo(j)
            X = Ly.conv_in(j)
            dz = Ly.dz(j)
            K = g["k"] ** 2 * g["c"]
            _, gam = gg_gammas(K, 1, 1)
            # ---- forward (the output conv's is the direct kernel fused with the loss seed: held through predict)
            if j < nlay - 1:
                ref = lrelu(conv(X, W, g["s"]) + b, a)
                mag = conv(np.abs(X), np.abs(W), g["s"]) + np.abs(b)
                hold(fails, worst, f"L{j} fwd", Ly.out_map(j), ref, (gam + 4 * U32) * mag * A)
            # ---- weight and bias gradients
            R_ = n * g["oh"] * g["ow"]
            M_, N_ = K, g["f"]
            split = max(1, min(nsm // (cdiv(M_, 128) * cdiv(N_, 64)), R_ // 512))
            _, gamw = gg_gammas(R_, split, 1)
            ref = conv_dw(X, W.shape, dz, g["s"])
            mag = conv_dw(np.abs(X), W.shape, np.abs(dz), g["s"])
            hold(fails, worst, f"L{j} wgrad", gW, ref, gamw * mag + U32 * np.abs(ref))
            chunk = cdiv(cdiv(R_, split), 64) * 64
            refb, magb = dz.sum((0, 1, 2)), np.abs(dz).sum((0, 1, 2))
            hold(fails, worst, f"L{j} bgrad", gb, refb, 1.01 * (chunk / 8 + 2) * U32 * magb + U32 * np.abs(refb))
            # ---- input gradient into the previous layer's D (not for conv 0)
            if j == 0:
                continue
            u = g["up"]
            dX = conv_dx(X.shape, W, dz, g["s"])[:, g["pt"]:g["pt"] + g["h"], g["pl"]:g["pl"] + g["w"], :]
            mX = conv_dx(X.shape, np.abs(W), np.abs(dz), g["s"])[:, g["pt"]:g["pt"] + g["h"], g["pl"]:g["pl"] + g["w"], :]
            hq, wq = g["h"] // u, g["w"] // u
            dX = dX.reshape(n, hq, u, wq, u, -1).sum((2, 4))
            mX = mX.reshape(n, hq, u, wq, u, -1).sum((2, 4))
            mask = Ly.interior(j)[:, ::u, ::u, :]
            gm = lgrad(mask, a)
            _, gamd = gg_gammas(u * u * K // g["c"] * g["f"], 1, 1)
            if j == L + 2:                                   # previous: the decoder dense, rows [n, h*w*c]
                got = Ly.dz(L + 1).reshape(n, hq, wq, -1)
            else:
                got = Ly.dz(j - 1)
            hold(fails, worst, f"L{j} dgrad", got, dX * gm, (gamd + U32) * mX * np.abs(gm))
        else:
            Xd = read(ae, j, 0).reshape(ae._ae_batch, -1)[:n]
            Xd = Xd[:, :W.shape[0]]
            dz = Ly.dz(j)
            _, gam = gg_gammas(W.shape[0], 1, 1)
            ref = lrelu(Xd @ W + b, a)
            mag = np.abs(Xd) @ np.abs(W) + np.abs(b)
            out = read(ae, j, 1).reshape(ae._ae_batch, -1)[:n, :W.shape[1]]
            hold(fails, worst, f"L{j} fwd", out, ref, (gam + 4 * U32) * mag * A)
            M_, N_ = W.shape
            split = max(1, min(nsm // (cdiv(M_, 128) * cdiv(N_, 64)), n // 512))
            _, gamw = gg_gammas(n, split, 1)
            ref, mag = Xd.T @ dz, np.abs(Xd).T @ np.abs(dz)
            hold(fails, worst, f"L{j} wgrad", gW, ref, gamw * mag + U32 * np.abs(ref))
            refb, magb = dz.sum(0), np.abs(dz).sum(0)
            hold(fails, worst, f"L{j} bgrad", gb, refb, 1.01 * (cdiv(n, 8) + 2) * U32 * magb + U32 * np.abs(refb))
            gm = lgrad(Xd, a)
            _, gamd = gg_gammas(N_, 1, 1)
            ref, mag = (dz @ W.T) * gm, (np.abs(dz) @ np.abs(W.T)) * np.abs(gm)
            if j == L:
                got = Ly.dz(L - 1).reshape(n, -1)
            else:
                got = Ly.dz(L)
            hold(fails, worst, f"L{j} dgrad", got, ref, (gamd + U32) * mag)
    print("\nworst err/bar:", {k: round(v, 3) for k, v in worst.items()})
    assert not fails, "\n".join(fails)
    return grads


def make(cfg, arrays, tp="bf16x3", cls=SimpleAutoEncoder, batch_=None):
    ae = cls(cfg, max_batch=1, train_precision=tp)
    ae.set_model_weights(arrays)
    if batch_:
        ae._autoencoder(batch_)
    return ae


# ------------------------------------------------------------------------------------------------ 1. every contraction
@pytest.mark.parametrize("B", [128, 72, 1])
@pytest.mark.parametrize("start", ["shipped", "glorot"])
def test_every_contraction_within_the_engine_bound(start, B):
    cfg = SHIPPED_CFG
    arrays = SHIPPED_ARRAYS if start == "shipped" else glorot(cfg, seed=5)
    ae = make(cfg, arrays, batch_=128)
    L = 3
    # which engine runs what: every forward but conv1's and the output conv's, every input gradient but the output conv's and
    # every weight gradient but conv1's on the wgmma engine
    on = [engines(ae, j) for j in range(2 * L + 2)]
    assert on[0] == (0, -1, 0) and on[-1] == (-1, 0, -1), on
    assert all(o == (1, 1, 1) for o in on[1:-1]), on
    check_contractions(ae, cfg, arrays, scenes(B, seed=20 + B), None, (64, 64))
    ae.close()


# ------------------------------------------------------------------------------------------------ 2. the geometry matrix
@pytest.mark.parametrize("case", CASES + DENOISE, ids=lambda c: c.name)
def test_geometry_matrix_within_the_engine_bound(case):
    cfg, cls, arrays = case.cfg(), model_class(case.hw), init(case)
    B = max(case.Bs)
    ae = make(cfg, arrays, cls=cls, batch_=B)
    b = batch(case, B, seed=10 * B + 7)
    x, tg = b if case.targets else (b, None)
    check_contractions(ae, cfg, arrays, x, tg, case.hw)
    ae.close()


# ------------------------------------------------------------------------------------------------ 3. Adam, predict, evaluate
def test_adam_on_the_gpu_gradients_and_forward_calls():
    cfg, arrays = SHIPPED_CFG, glorot(SHIPPED_CFG, seed=7)
    lr = 1e-3
    ae = make(cfg, arrays, batch_=32)
    opt = R.Adam(ae.get_weights(), lr)
    for s in range(3):
        x = scenes(32, seed=300 + s)
        before = [a for kb in ae.get_weights() for a in kb]
        _, grads = ae.step(x, lr=lr)
        after = [a for kb in ae.get_weights() for a in kb]
        g64 = [(np.asarray(k, F64), np.asarray(b, F64)) for k, b in grads]
        upd = opt.update(g64)
        t_ = opt.t + 1
        lr_t = lr * np.sqrt(1 - 0.999 ** t_) / (1 - 0.9 ** t_)
        for i, (p0, p1, du) in enumerate(zip(before, after, upd)):
            ref = np.asarray(p0, F64) + du
            bar = 4 * U32 * np.abs(ref) + 1e-4 * lr_t * (np.abs(du) / lr_t + 1e-3)
            err = np.abs(np.asarray(p1, F64) - ref)
            assert (err <= bar).all(), (s, i, float((err / bar).max()))
        opt.step(g64)
    # predict and evaluate: the forward at bf16x3 against float64 at the GPU's weights
    w = ae.get_weights()
    x = scenes(77, seed=400)
    ref = R.predict(w, x, cfg["network"], cfg["alpha"])
    y = ae.predict(x)
    e = float(np.abs(y - ref).max() / np.abs(ref).max())
    mse = float(((ref - x) ** 2).mean())
    got = ae.test(x, x)
    print(f"\npredict rel err {e:.3g}, evaluate rel err {abs(got - mse) / mse:.3g}")
    assert e <= 1e-3, e
    assert abs(got - mse) <= 1e-3 * mse, (got, mse)
    ae.close()


# ------------------------------------------------------------------------------------------------ 4. the epoch graph
def test_epoch_graph_equals_explicit_steps_across_dataset_changes():
    """Epochs (full batches and a partial last one) against explicit steps on the same batches, from the same weights,
    through a dataset that shrinks (captured graphs kept) and grows (graphs recaptured)."""
    case = BY_NAME["odd_s3"]
    cfg, cls, arrays = dict(case.cfg(), batch_size=16), model_class(case.hw), init(case, seed=9)
    lr, bs = 1e-3, 16
    ep = make(cfg, arrays, cls=cls, batch_=bs)
    ex = make(cfg, arrays, cls=cls, batch_=bs)
    rng = np.random.default_rng(800)
    from tests.test_gpu_autoencoder_configs import images
    for n_rows, n_order, seed in ((300, 37, 801), (100, 16, 802), (500, 43, 803)):
        rows = images(n_rows, case.hw, seed)
        set_dataset(ep._ae, rows, None)
        order = rng.permutation(n_rows)[:n_order].astype(np.int32)
        order[0] = n_rows - 1
        loss = train_epoch(ep._ae, order, bs, lr)
        losses = []
        for s in range(0, n_order, bs):
            o = order[s:s + bs]
            lo, _ = ex.step(rows[o], lr=lr)
            losses.append(lo * len(o))
        assert abs(loss - sum(losses) / n_order) <= 1e-5 * abs(loss), (loss, sum(losses) / n_order)
        for (k0, b0), (k1, b1) in zip(ep.get_weights(), ex.get_weights()):
            for p, q in ((k0, k1), (b0, b1)):
                assert np.abs(p.astype(F64) - q).max() <= 2 * U32 * np.abs(q).max() + 1e-3 * lr, (n_rows, np.abs(p - q).max())
    ep.close()
    ex.close()


# ------------------------------------------------------------------------------------------------ 5. training quality
# Measured on an H100 80GB HBM3 (700 W): final val_loss 9.0999e-4 (fp32) vs 9.0648e-4 (bf16x3), 0.39 % apart; over the 12
# epochs the two curves are at most 2.1 % apart at any one epoch (epoch 9).  3 % holds the final value to that per-epoch gap
# with some margin; a bf16x3 path that lost a gradient term or trained noticeably worse lands far outside it.
QUALITY_TOL = 0.03


def test_training_quality_matches_fp32(tmp_path):
    """Same init and shuffling (seed) for both precisions, 12 epochs on seeded synthetic depth scenes at the shipped geometry:
    both losses fall, and bf16x3's final validation MSE is within QUALITY_TOL of fp32's."""
    cfg = dict(SHIPPED_CFG, learning_rate=1e-3)
    x = synth.make_depth_scenes(2400, seed=77)
    hist = {}
    for tp in ("fp32", "bf16x3"):
        ae = SimpleAutoEncoder(cfg, max_batch=1, seed=123, train_precision=tp)
        hist[tp] = ae.train(x, None, 64, 12, str(tmp_path / tp))
        ae.close()
    for tp, h in hist.items():
        assert h["loss"][-1] < 0.5 * h["loss"][0] and h["val_loss"][-1] < h["val_loss"][0], (tp, h)
    f, b = hist["fp32"]["val_loss"][-1], hist["bf16x3"]["val_loss"][-1]
    print(f"\nfinal val_loss fp32 {f:.6g} bf16x3 {b:.6g} rel {abs(b - f) / f:.3g}")
    print("fp32  ", [round(v, 7) for v in hist["fp32"]["val_loss"]])
    print("bf16x3", [round(v, 7) for v in hist["bf16x3"]["val_loss"]])
    assert abs(b - f) <= QUALITY_TOL * f, (f, b)


# ------------------------------------------------------------------------------------------------ 6. defaults
def _one_step(create, cfg, arrays, x):
    lib = _lib.load()
    ecfg = _lib.EncoderCfg.from_buffer_copy(SimpleAutoEncoder(cfg, max_batch=1)._cfg)
    ecfg.max_batch = x.shape[0]
    h = C.c_void_p()
    _lib.check(create(ecfg, h))
    fp = C.POINTER(C.c_float)
    for i, (k, b) in enumerate(arrays):
        k, b = np.ascontiguousarray(k, np.float32), np.ascontiguousarray(b, np.float32)
        _lib.check(lib.b2g_autoencoder_set_weights(h, i, k.ctypes.data_as(fp), k.size, b.ctypes.data_as(fp), b.size))
    loss = C.c_double()
    _lib.check(lib.b2g_autoencoder_step(h, x.ctypes.data_as(fp), None, x.shape[0], 1e-3, 1, C.byref(loss)))
    out = []
    for i, (k, b) in enumerate(arrays):
        kk, bb = np.empty(np.shape(k), np.float32), np.empty(np.shape(b), np.float32)
        _lib.check(lib.b2g_autoencoder_get_weights(h, i, kk.ctypes.data_as(fp), kk.size, bb.ctypes.data_as(fp), bb.size))
        out += [kk, bb]
    lib.b2g_autoencoder_destroy(h)
    return out


def test_create_is_create2_fp32_and_precision_alone_trains_in_fp32():
    lib = _lib.load()
    cfg, arrays = SHIPPED_CFG, SHIPPED_ARRAYS
    x = scenes(16, seed=900)
    c1 = lambda cf, h: lib.b2g_autoencoder_create(C.byref(cf), C.byref(h))
    c2 = lambda cf, h: lib.b2g_autoencoder_create2(C.byref(cf), _lib.B2G_PREC_FP32_SIMT, C.byref(h))
    a, b, c = _one_step(c1, cfg, arrays, x), _one_step(c1, cfg, arrays, x), _one_step(c2, cfg, arrays, x)
    for pa, pb, pc in zip(a, b, c):
        d_ref = np.abs(pa.astype(F64) - pb).max()
        assert np.abs(pa.astype(F64) - pc).max() <= max(d_ref, 2 * U32 * np.abs(pa).max()), (d_ref,)
    # precision="bf16x3" is encode()'s; the training handle stays fp32 unless train_precision says otherwise
    ae = SimpleAutoEncoder(cfg, max_batch=4, precision="bf16x3")
    ae.set_model_weights(arrays)
    ae._autoencoder(4)
    assert ae.train_precision == "fp32" and all(engines(ae, j) in ((0, -1, 0), (0, 0, 0), (-1, 0, -1)) for j in range(8))
    ae.close()
    ae = SimpleAutoEncoder(cfg, max_batch=4, train_precision="bf16x3")
    ae.set_model_weights(arrays)
    ae._autoencoder(4)
    assert engines(ae, 1) == (1, 1, 1)
    ae.close()


def test_cli_flag_reaches_the_handle(tmp_path, monkeypatch):
    """train_encoder test --train_precision bf16x3 evaluates through a bf16x3 handle."""
    from b200grasp import encoders, train_encoder
    seen = []
    real = encoders.SimpleAutoEncoder.test

    def spy(self, inputs, targets):
        out = real(self, inputs, targets)
        seen.append(engines(self, 1))
        return out
    monkeypatch.setattr(encoders.SimpleAutoEncoder, "test", spy)
    import pickle
    import yaml
    x = synth.make_depth_scenes(12, seed=5)
    masks = np.where(x > 0, 3, 0).astype(np.int32)
    with open(tmp_path / "data.pkl", "wb") as f:
        pickle.dump({"train": {"depth": x.copy(), "masks": masks}, "test": {"depth": x.copy(), "masks": masks}}, f)
    cfg = dict(SHIPPED_CFG, data_path=str(tmp_path / "data.pkl"), batch_size=4, epochs=1)
    model_dir = tmp_path / "m"
    model_dir.mkdir()
    with open(model_dir / "config.yaml", "w") as f:
        yaml.safe_dump(cfg, f)
    ae = SimpleAutoEncoder(cfg, max_batch=1)
    ae.set_model_weights(SHIPPED_ARRAYS)
    ae.save_weights(str(model_dir / "model.h5"))
    ae.close()
    loss = train_encoder.main([str(model_dir), "test", "--train_precision", "bf16x3"])
    assert np.isfinite(loss) and seen == [(1, 1, 1)]
