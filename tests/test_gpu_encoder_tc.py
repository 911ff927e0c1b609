"""The perception encoder on the wgmma engine (SimpleAutoEncoder(precision="bf16x3"), b2g_encoder_create2): every layer held
element by element to a float64 contraction of its own GPU inputs, the encodings to the float64 oracle, a frame's encoding
independent of its batch and row, the learners' observe-path stage equal to the encoder bit for bit, the refusals, and the
fp32 default unchanged."""
import ctypes as C

import numpy as np
import pytest
import torch

import b200grasp  # noqa: F401
from b200grasp import _lib, synth
from b200grasp.bdq import BDQLearner
from b200grasp.encoders import SimpleAutoEncoder, keras_encoder_arrays
from b200grasp.learner import Learner
from oracle import encoder_ref as ER
from tests.deferred_env import PIXELS
from tests.gg_tc_ref import U32, Report, gg_gammas
from tests.test_encoder_cpu import load_fixture
from tests.test_gpu_encoder_configs import CASES, TOL, Case, layers, model_class, weights
from tests.test_gpu_obs_encoder import _done, _raw

pytestmark = pytest.mark.gpu
fp = C.POINTER(C.c_float)


def tc_accepts(case):
    """b2g_encoder_create2(B2G_PREC_BF16X3): every conv but the last feeds BF16 plane rows of 8-channel groups."""
    return all(f % 8 == 0 for f, _, _ in case.network[:-1])


# geometries of the bf16x3 path beyond the fp32 matrix's: layer 0's unfolded rows padded (k * C = 7, 9, 10 -> 8, 16, 16), a
# dense input whose rows are padded to 8 (flat 60), strides 1 to 3, encoding_dim 100 and 130
TC_CASES = [c for c in CASES if tc_accepts(c)] + [
    Case("t1", (64, 64, 1), ((8, 7, 2), (16, 5, 2), (8, 3, 2)), 100, 0.1),
    Case("t3", (29, 31, 3), ((16, 3, 1), (8, 4, 2), (2, 5, 3)), 130, -0.2),
    Case("t5", (64, 64, 5), ((24, 2, 2),), 7, 1.0),
]


def shipped(max_batch, precision="bf16x3"):
    w, cfg = load_fixture()
    arr = keras_encoder_arrays(w, len(cfg["network"]))
    enc = SimpleAutoEncoder(cfg, max_batch=max_batch, precision=precision)
    enc.set_weights(arr)
    return enc, arr, cfg


def shipped_case():
    _, cfg = load_fixture()
    return Case("shipped", (64, 64, 1), tuple((l["filters"], l["kernel_size"], l["strides"]) for l in cfg["network"]),
                cfg["encoding_dim"], float(cfg.get("alpha", 0.1)))


def layer_outputs(enc, imgs, case):
    """b2g_debug_encoder_layers: [conv l output [n, oh, ow, f]] + [encodings [n, enc]]."""
    n = imgs.shape[0]
    ls, _ = layers(case)
    shapes = [(n, oh, ow, f) for _, _, _, _, _, f, oh, ow in ls] + [(n, case.enc)]
    out = np.empty(sum(int(np.prod(s)) for s in shapes), np.float32)
    imgs = np.ascontiguousarray(imgs, np.float32)
    _lib.check(_lib.load().b2g_debug_encoder_layers(enc._handle, imgs.ctypes.data_as(fp), n, out.ctypes.data_as(fp), out.size))
    res, o = [], 0
    for s in shapes:
        res.append(out[o:o + int(np.prod(s))].reshape(s))
        o += int(np.prod(s))
    return res


def hold_layers(case, enc, arr, imgs, rep):
    """Each layer against leaky(x @ w + b) in float64 of the x the GPU read: the raw frames for conv 0, the previous layer's
    planes (hi + lo) after that.  Bar: the engine's split and k-step allowance over its reduction length (layer 0: k kernel rows
    of round8(k * C) taps) times sum |x||w| + |b|, plus the bias add and the LeakyReLU's product, times max(1, |alpha|); hidden
    outputs also carry the hi/lo split of the stored value (2^-17 of it)."""
    outs = layer_outputs(enc, imgs, case)
    ls, _ = layers(case)
    x = imgs.astype(np.float64)
    a = case.alpha
    for l, (w, b) in enumerate(arr):
        dense = l == len(ls)
        w64, b64 = torch.tensor(w, dtype=torch.float64), torch.tensor(b, dtype=torch.float64)
        if dense:
            xf = torch.tensor(x.reshape(x.shape[0], -1))
            pre, mag = xf @ w64 + b64, xf.abs() @ w64.abs() + b64.abs()
            K = xf.shape[1]
        else:
            _, _, c, k, s, _, _, _ = ls[l]
            xt = torch.tensor(x).permute(0, 3, 1, 2)
            pre = ER.conv_same(xt, w64, b64, s).permute(0, 2, 3, 1)
            mag = ER.conv_same(xt.abs(), w64.abs(), b64.abs(), s).permute(0, 2, 3, 1)
            K = k * (-(-k * c // 8) * 8) if l == 0 else k * k * c
        ref = torch.where(pre > 0, pre, a * pre).numpy()
        _, tot = gg_gammas(K, 1, 1)
        gamma = (tot + 2 * U32) * max(1.0, abs(a))
        r = U32 + (0.0 if dense else 2.0 ** -17)
        rep.hold(f"layer{l}", outs[l], ref, mag.numpy(), gamma, r)
        x = outs[l].astype(np.float64)
    return outs


@pytest.mark.parametrize("case", TC_CASES + [shipped_case()], ids=lambda c: c.name)
def test_every_layer_holds_to_float64_of_its_own_inputs(case):
    n = 5
    if case.name == "shipped":
        enc, arr, _ = shipped(n)
        imgs = synth.make_depth_scenes(n, seed=11).astype(np.float32)
    else:
        cfg = {"network": [{"filters": f, "kernel_size": k, "strides": s} for f, k, s in case.network], "encoding_dim": case.enc,
               "alpha": case.alpha}
        enc = model_class(case.hwc)(cfg, max_batch=n, precision="bf16x3")
        arr = weights(case, 1)
        enc.set_weights(arr)
        imgs = np.random.default_rng(2).normal(0, 1, (n,) + case.hwc).astype(np.float32)
    rep = Report(case.name)
    outs = hold_layers(case, enc, arr, imgs, rep)
    assert not rep.fail, rep.fail
    assert np.array_equal(outs[-1], enc.encode(imgs))          # the debug entry's last layer is encode()
    # and end to end against the oracle at today's fp32 bar
    ref = ER.encode(imgs, arr, [s for _, _, s in case.network], case.alpha, torch.float64)
    assert np.abs(outs[-1] - ref).max() <= TOL * np.abs(ref).max()
    enc.close()


def test_shipped_weights_end_to_end():
    enc, arr, cfg = shipped(256)
    imgs = synth.make_depth_scenes(256, seed=3).astype(np.float32)
    z = enc.encode(imgs)
    ref = ER.encode(imgs, arr, [l["strides"] for l in cfg["network"]], cfg.get("alpha", 0.1), torch.float64)
    assert np.abs(z - ref).max() <= TOL * np.abs(ref).max()
    f32, _, _ = shipped(256, "fp32")
    assert not np.array_equal(f32.encode(imgs), z)              # another arithmetic, not the fp32 path under a new name
    f32.close(), enc.close()


def test_a_frame_encodes_the_same_in_any_batch_and_row():
    N = 70
    enc, _, _ = shipped(N)
    imgs = synth.make_depth_scenes(N, seed=4).astype(np.float32)
    z = enc.encode(imgs)
    for i in range(N):
        assert np.array_equal(enc.encode(imgs[i:i + 1]), z[i:i + 1]), i
    perm = np.random.default_rng(0).permutation(N)
    assert np.array_equal(enc.encode(imgs[perm]), z[perm])
    assert np.array_equal(enc.encode(np.repeat(imgs[7:8], N, axis=0)), np.repeat(z[7:8], N, axis=0))
    assert np.array_equal(enc.encode(imgs[:33]), z[:33])
    enc.close()


@pytest.mark.parametrize("n,tail,kind", [(1, 1, "all"), (3, 0, "some"), (128, 1, "some"), (256, 2, "all"), (256, 1, "none")])
def test_sac_stage_equals_the_bf16x3_encoder(n, tail, kind):
    enc, _, cfg = shipped(512)
    D = cfg["encoding_dim"]
    L = Learner((D + tail,), n_act=2, batch_size=64, buffer_size=2 * n, precision=_lib.B2G_PREC_FP32_SIMT)
    L.set_obs_encoder(enc, tail)
    r0, r1, r3 = _raw(n, tail, 1), _raw(n, tail, 2), _raw(n, tail, 3)
    done = _done(kind, n)
    reset = np.full_like(r1, np.nan)
    reset[done != 0] = _raw(n, tail, 4)[done != 0]
    act, rew = np.zeros((n, 2), np.float32), np.zeros(n, np.float32)
    L.observe_act(r0, update_stats=False, act=False)
    L.observe_add(act, rew, r1, done, reset_obs=reset if done.any() else None, update_stats=False)
    L.observe_add(act, rew, r3, np.zeros(n, np.float32), update_stats=False)
    staged = np.where(done[:, None] != 0, reset, r1)

    def host(rows):
        return np.concatenate([enc.encode(rows[:, :PIXELS].reshape(-1, 64, 64, 1)), rows[:, PIXELS:]], axis=1)
    want = [(host(r0), host(r1)), (host(staged), host(r3))]
    for i in range(n):
        for j, (wo, wn) in enumerate(want):
            t = L.replay_get(j * n + i)
            assert np.array_equal(t["obs"], wo[i]) and np.array_equal(t["next_obs"], wn[i]), (j, i)
    L.close(), enc.close()


def test_bdq_stage_equals_the_bf16x3_encoder():
    enc, _, cfg = shipped(512)
    n, tail = 128, 1
    E = cfg["encoding_dim"] + tail
    mk = lambda: BDQLearner(E, 2, 4, ((64, 64), (32,), (32,)), 16, 1024, seed=3)
    A, B = mk(), mk()
    for L in (A, B):
        L.obs_rms_set(np.zeros(E), np.ones(E), 1e-4)
    B.load_parameters(A.get_parameters())
    A.set_obs_encoder(enc, tail)

    def host(rows):
        return np.concatenate([enc.encode(rows[:, :PIXELS].reshape(-1, 64, 64, 1)), rows[:, PIXELS:]], axis=1)
    r0, r1 = _raw(n, tail, 5), _raw(n, tail, 6)
    done = _done("some", n)
    reset = np.full_like(r1, np.nan)
    reset[done != 0] = _raw(n, tail, 7)[done != 0]
    reset_enc = np.full((n, E), np.nan, np.float32)
    reset_enc[done != 0] = host(reset[done != 0])
    a0 = A.observe_act(r0, eps=0.0)
    assert np.array_equal(a0, B.observe_act(host(r0), eps=0.0))
    A.observe_add(a0.astype(np.float32), np.ones(n), r1, done, reset_obs=reset)
    B.observe_add(a0.astype(np.float32), np.ones(n), host(r1), done, reset_obs=reset_enc)
    for x, y in zip(A.obs_rms_get(), B.obs_rms_get()):
        assert np.array_equal(x, y)
    assert np.array_equal(A.observe_act(None, n=n, eps=0.0), B.observe_act(None, n=n, eps=0.0))     # staged rows
    for i in range(n):
        assert np.array_equal(A.replay_get(i)["next_obs"], B.replay_get(i)["next_obs"]), i
    A.close(), B.close(), enc.close()


def _cfg(case, device=0, max_batch=4):
    c = _lib.EncoderCfg()
    c.height, c.width, c.channels = case.hwc
    c.n_layers = len(case.network)
    for i, (f, k, s) in enumerate(case.network):
        c.filters[i], c.kernel[i], c.strides[i] = f, k, s
    c.encoding_dim, c.alpha, c.max_batch, c.device = case.enc, case.alpha, max_batch, device
    return c


def test_refusals_come_before_any_cuda_call():
    lib = _lib.load()
    h = C.c_void_p()
    far = 1 << 20                 # no such device: a refusal that reached check_device would say B2G_ECUDA
    ship = shipped_case()
    for prec, what in ((_lib.B2G_PREC_BF16, "single-pass BF16"), (7, "precision 7"), (-1, "precision -1")):
        assert lib.b2g_encoder_create2(C.byref(_cfg(ship, far)), prec, C.byref(h)) == _lib.B2G_EINVAL
        assert what in lib.b2g_last_error().decode()
    l8 = next(c for c in CASES if c.name == "l8")
    assert lib.b2g_encoder_create2(C.byref(_cfg(l8, far)), _lib.B2G_PREC_BF16X3, C.byref(h)) == _lib.B2G_EINVAL
    assert "filters % 8" in lib.b2g_last_error().decode()
    assert lib.b2g_encoder_create2(C.byref(_cfg(l8, far)), _lib.B2G_PREC_FP32_SIMT, C.byref(h)) == _lib.B2G_ECUDA
    assert lib.b2g_encoder_create2(C.byref(_cfg(l8, 0)), _lib.B2G_PREC_BF16X3, C.byref(h)) == _lib.B2G_EINVAL
    assert not h
    with pytest.raises(ValueError, match="precision"):
        SimpleAutoEncoder(load_fixture()[1], precision="x")


def test_create_and_create2_fp32_encode_bit_identically():
    enc, arr, cfg = shipped(64, "fp32")
    lib = _lib.load()
    h = C.c_void_p()
    _lib.check(lib.b2g_encoder_create(C.byref(enc._cfg), C.byref(h)))
    for i, (k, b) in enumerate(arr):
        k, b = np.ascontiguousarray(k, np.float32), np.ascontiguousarray(b, np.float32)
        _lib.check(lib.b2g_encoder_set_weights(h, i, k.ctypes.data_as(fp), k.size, b.ctypes.data_as(fp), b.size))
    imgs = synth.make_depth_scenes(64, seed=9).astype(np.float32)
    z = np.empty((64, cfg["encoding_dim"]), np.float32)
    _lib.check(lib.b2g_encoder_encode(h, imgs.ctypes.data_as(fp), 64, z.ctypes.data_as(fp)))
    assert np.array_equal(enc.encode(imgs), z)
    lib.b2g_encoder_destroy(h)
    enc.close()
