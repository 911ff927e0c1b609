"""Host mirror of the reference's perception encoder (SURVEY.md section 8 row a12).

Same names and call shapes as /root/reference/manipulation_main/gripperEnv/encoders.py:
``SimpleAutoEncoder(config)`` (:67-136), ``load_weights(model_dir)`` (:27-31), ``encode(imgs)`` (:59-61),
``encoding_shape`` (:63-65), ``train`` / ``test`` / ``predict`` (:40-57).  ``DeferredEncodedDepthImgSensor`` stands in for the
reference's ``EncodedDepthImgSensor`` (sensor.py:169-230) in env workers that hold no CUDA context: it hands out the filtered
depth frame, and ``vec_env.VecEncodeDepth`` encodes the frames of every env in the learner's process.  ``encode`` runs on the GPU through libb200grasp
(csrc/encoder.cu); ``train``, ``test`` and ``predict`` run the whole auto-encoder there (csrc/autoencoder.cu), with the
bookkeeping of Keras' ``fit`` restated in :func:`fit`.  ``plot`` (pydot) raises ``NotImplementedError``.  ``model.h5`` is read
and written by ``h5min`` (no h5py/keras needed).
"""
from __future__ import annotations

import csv
import ctypes as C
import hashlib
import math
import os
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import _lib, h5min


def keras_encoder_arrays(weights: Dict[str, np.ndarray], n_conv: int):
    """Orders Keras auto-named layers the way the reference builds them: encoder convs are the first ``n_conv``
    ``conv2d_*`` layers, the encoder's Dense is the first ``dense_*`` layer (encoders.py:92-104 precede :110-128).
    Returns [(kernel, bias)] for conv_0..conv_{n-1}, dense."""
    def ordered(prefix):
        idx = sorted({int(k.split("/")[0].split("_")[-1]) for k in weights if k.startswith(prefix)})
        return [f"{prefix}{i}" for i in idx]
    convs, denses = ordered("conv2d_"), ordered("dense_")
    if len(convs) < n_conv or not denses:
        raise ValueError(f"model.h5 holds {len(convs)} conv / {len(denses)} dense layers; config needs {n_conv} / 1")
    return [(weights[f"{n}/kernel"], weights[f"{n}/bias"]) for n in convs[:n_conv] + denses[:1]]


def keras_layer_names(n_conv: int) -> List[str]:
    """Keras auto-names of the auto-encoder's weighted layers in model.h5 order: encoder convs, encoder Dense, decoder Dense,
    decoder convs (encoders.py:92-124 create them in that order)."""
    return ([f"conv2d_{i}" for i in range(1, n_conv + 1)] + ["dense_1", "dense_2"] +
            [f"conv2d_{i}" for i in range(n_conv + 1, 2 * n_conv + 1)])


def model_shapes(network: Sequence[dict], encoding_dim: int, input_shape=(64, 64, 1)) -> List[Tuple[tuple, int]]:
    """[(kernel shape, bias length)] of the 2L+2 weighted layers in model.h5 order (encoders.py:84-124)."""
    h, w, c = input_shape
    out = []
    for l in network:
        k, s, f = int(l["kernel_size"]), int(l["strides"]), int(l["filters"])
        out.append(((k, k, c, f), f))
        h, w, c = -(-h // s), -(-w // s), f
    flat = h * w * c
    out += [((flat, encoding_dim), encoding_dim), ((encoding_dim, flat), flat)]
    for i in reversed(range(1, len(network))):
        k = int(network[i]["kernel_size"])
        f = int(network[i - 1]["filters"])
        out.append(((k, k, c, f), f))
        c = f
    k = int(network[0]["kernel_size"])
    out.append(((k, k, c, 1), 1))
    return out


def glorot_init(shapes, rng: np.random.Generator):
    """Keras defaults: glorot_uniform kernels (limit sqrt(6 / (fan_in + fan_out)), a conv's fans are kh*kw*in and kh*kw*out),
    zero biases."""
    out = []
    for shape, nb in shapes:
        rf = int(np.prod(shape[:-2])) if len(shape) > 2 else 1
        fan_in, fan_out = shape[-2] * rf, shape[-1] * rf
        lim = math.sqrt(6.0 / (fan_in + fan_out))
        out.append((rng.uniform(-lim, lim, shape).astype(np.float32), np.zeros(nb, np.float32)))
    return out


def fit(n: int, batch_size: int, epochs: int, train_epoch: Callable[[np.ndarray, int], float],
        evaluate: Callable[[int, int], float], on_best: Callable[[int], None], history_path: Optional[str],
        rng: np.random.Generator, validation_split: float = 0.1, patience: int = 25) -> Dict[str, List[float]]:
    """Keras 2.2.4 ``fit(x, x, batch_size, epochs, validation_split, shuffle=True)`` with the reference's callbacks
    (encoders.py:40-51): CSVLogger, ModelCheckpoint(save_best_only, save_weights_only), EarlyStopping(patience).

    The validation rows are the last ``n - int(n * (1 - validation_split))``, cut before any shuffling.  Each epoch,
    ``train_epoch(order, batch_size)`` runs one pass over the training rows in a fresh random order and returns the
    sample-weighted mean of its batch losses; ``evaluate(start, count)`` returns the mean squared error of a row slice with
    the end-of-epoch weights.  ``on_best(epoch)`` runs when val_loss is strictly below every earlier one (the checkpoint);
    training stops after the epoch on which ``patience`` epochs have passed without such an improvement."""
    n_train = int(n * (1.0 - validation_split))
    if n_train < 1 or n_train >= n:
        raise ValueError(f"validation_split {validation_split} leaves no training or no validation rows of {n}")
    history: Dict[str, List[float]] = {"loss": [], "val_loss": []}
    fh = open(history_path, "w", newline="") if history_path else None
    writer = csv.writer(fh) if fh else None
    if writer:
        writer.writerow(["epoch", "loss", "val_loss"])
        fh.flush()
    best, wait = math.inf, 0
    try:
        for epoch in range(epochs):
            loss = float(train_epoch(rng.permutation(n_train).astype(np.int32), batch_size))
            val_loss = float(evaluate(n_train, n - n_train))
            history["loss"].append(loss)
            history["val_loss"].append(val_loss)
            if writer:
                writer.writerow([epoch, repr(loss), repr(val_loss)])
                fh.flush()
            if val_loss < best:
                best, wait = val_loss, 0
                on_best(epoch)
            else:
                wait += 1
                if wait >= patience:
                    break
    finally:
        if fh:
            fh.close()
    return history


ENCODER_PRECISIONS = {"fp32": _lib.B2G_PREC_FP32_SIMT, "bf16x3": _lib.B2G_PREC_BF16X3}


class Encoder(object):
    """Base class for learning abstract representations of image observations.

    ``precision`` is the arithmetic of ``encode`` and of the observe-path stage a learner copies from this encoder: "fp32"
    (fp32 FFMA on the CUDA cores, the default) or "bf16x3" (the tensor-core engine, BF16 hi/lo operand splits summed in fp32:
    about 2^-16 relative per layer).

    ``train_precision`` is the arithmetic of the training handle behind ``train``, ``test``, ``predict`` and ``step``:
    "fp32" (every product exact in fp32, summed in double on the CUDA cores, the default) or "bf16x3" (every conv and dense
    contraction but conv1's forward and weight gradient and the one-filter output conv on the tensor-core engine: each
    element within about 2^-15 of the sum of |products| of its contraction).  The two keywords are independent: a
    ``precision="bf16x3"`` encoder still trains in fp32 unless ``train_precision`` says otherwise."""

    def __init__(self, config, max_batch: int = 1, device: int = 0, seed: Optional[int] = None, precision: str = "fp32",
                 train_precision: str = "fp32"):
        if precision not in ENCODER_PRECISIONS:
            raise ValueError(f"precision must be one of {sorted(ENCODER_PRECISIONS)}, got {precision!r}")
        if train_precision not in ENCODER_PRECISIONS:
            raise ValueError(f"train_precision must be one of {sorted(ENCODER_PRECISIONS)}, got {train_precision!r}")
        self.precision = precision
        self.train_precision = train_precision
        self._handle = C.c_void_p()
        self._ae = C.c_void_p()
        self._ae_batch = 0
        self._max_batch, self._device = int(max_batch), int(device)
        self._rng = np.random.default_rng(seed)
        self._lib = _lib.load()
        self._build(config)

    def _build(self, config):
        raise NotImplementedError

    def plot(self, *a, **k):
        raise NotImplementedError("plot needs pydot / graphviz, which this package does not use")


class SimpleAutoEncoder(Encoder):
    """Vanilla autoencoder.  ``encode`` runs the encoder half; ``train``, ``test`` and ``predict`` the whole model."""

    input_shape = (64, 64, 1)          # encoders.py:87

    def _build(self, config):
        self.network: List[dict] = list(config["network"])
        self.encoding_dim = int(config["encoding_dim"])
        self.alpha = float(config.get("alpha", 0.1))
        cfg = _lib.EncoderCfg()
        cfg.height, cfg.width, cfg.channels = self.input_shape
        cfg.n_layers = len(self.network)
        if cfg.n_layers > _lib.ENC_MAX_LAYERS:
            raise ValueError("too many conv layers")
        for i, layer in enumerate(self.network):
            cfg.filters[i], cfg.kernel[i], cfg.strides[i] = int(layer["filters"]), int(layer["kernel_size"]), int(layer["strides"])
        cfg.encoding_dim, cfg.alpha = self.encoding_dim, self.alpha
        cfg.max_batch, cfg.device = self._max_batch, self._device
        self._cfg = cfg
        self._learning_rate = float(config.get("learning_rate", 2e-4))
        self._train_batch = int(config.get("batch_size", 128))
        self._weights = None            # [(kernel, bias)] of all 2L+2 layers once the decoder half is known
        _lib.check(self._lib.b2g_encoder_create2(C.byref(cfg), ENCODER_PRECISIONS[self.precision], C.byref(self._handle)))

    # ---- whole auto-encoder (csrc/autoencoder.cu)
    def _shapes(self):
        return model_shapes(self.network, self.encoding_dim, self.input_shape)

    def _autoencoder(self, batch: int):
        """The training handle, holding self._weights, for batches up to ``batch``."""
        if self._weights is None:
            raise NotImplementedError("the decoder half has no weights: load a model.h5 that holds it, or train first")
        if not self._ae or batch > self._ae_batch:
            self._close_ae()
            cfg = _lib.EncoderCfg.from_buffer_copy(self._cfg)
            cfg.max_batch = max(batch, self._train_batch)
            _lib.check(self._lib.b2g_autoencoder_create2(C.byref(cfg), ENCODER_PRECISIONS[self.train_precision], C.byref(self._ae)))
            self._ae_batch = cfg.max_batch
            self._push_weights()
        return self._ae

    def _push_weights(self):
        fp = C.POINTER(C.c_float)
        for i, (k, b) in enumerate(self._weights):
            k = np.ascontiguousarray(k, np.float32)
            b = np.ascontiguousarray(b, np.float32)
            _lib.check(self._lib.b2g_autoencoder_set_weights(self._ae, i, k.ctypes.data_as(fp), k.size, b.ctypes.data_as(fp), b.size))

    def _pull(self, fn) -> List[Tuple[np.ndarray, np.ndarray]]:
        fp = C.POINTER(C.c_float)
        out = []
        for i, (shape, nb) in enumerate(self._shapes()):
            k, b = np.empty(shape, np.float32), np.empty(nb, np.float32)
            _lib.check(fn(self._ae, i, k.ctypes.data_as(fp), k.size, b.ctypes.data_as(fp), b.size))
            out.append((k, b))
        return out

    def get_weights(self) -> List[Tuple[np.ndarray, np.ndarray]]:
        """All 2L+2 (kernel, bias) pairs in model.h5 order (None before the decoder half has weights)."""
        if self._ae and self._weights is not None:
            self._weights = self._pull(self._lib.b2g_autoencoder_get_weights)
        return self._weights

    def set_model_weights(self, arrays):
        """arrays: [(kernel, bias)] of all 2L+2 layers in model.h5 order (Keras layouts)."""
        shapes = self._shapes()
        if len(arrays) != len(shapes):
            raise ValueError(f"expected {len(shapes)} (kernel, bias) pairs, got {len(arrays)}")
        for (k, b), (ks, nb) in zip(arrays, shapes):
            if tuple(np.shape(k)) != ks or np.size(b) != nb:
                raise ValueError(f"expected kernel {ks} and bias ({nb},), got {np.shape(k)} and {np.shape(b)}")
        self._weights = [(np.array(k, np.float32), np.array(b, np.float32).reshape(-1)) for k, b in arrays]
        self.set_weights(self._weights[:len(self.network) + 1])
        if self._ae:
            self._push_weights()

    def save_weights(self, path: str):
        """Writes the Keras ``save_weights`` layout of the reference's model (input_1, encoder, decoder) to ``path``."""
        arrays = self.get_weights()
        names = keras_layer_names(len(self.network))
        ws = [(f"{n}/{t}:0", a) for n, (k, b) in zip(names, arrays) for t, a in (("kernel", k), ("bias", b))]
        n_enc = 2 * (len(self.network) + 1)
        h5min.write_keras_weights(path, [("input_1", []), ("encoder", ws[:n_enc]), ("decoder", ws[n_enc:])])

    def _check_imgs(self, imgs, what="imgs"):
        imgs = np.ascontiguousarray(imgs, np.float32)
        if imgs.ndim != 4 or imgs.shape[1:] != self.input_shape:
            raise ValueError(f"expected {what} of shape (n, {self.input_shape}), got {imgs.shape}")
        return imgs

    def train(self, inputs, targets, batch_size, epochs, model_dir):
        """Keras ``fit(inputs, targets, batch_size, epochs, validation_split=0.1, shuffle=True)`` with the reference's
        callbacks: writes ``history.csv`` and, at every strict val_loss improvement, ``model.h5`` into ``model_dir``.
        Returns ``{"loss": [...], "val_loss": [...]}``; the model keeps the last epoch's weights."""
        inputs = self._check_imgs(inputs, "inputs")
        same = targets is None or targets is inputs
        targets = inputs if same else self._check_imgs(targets, "targets")
        if targets.shape != inputs.shape:
            raise ValueError("inputs and targets differ in shape")
        if self._weights is None:
            self.set_model_weights(glorot_init(self._shapes(), self._rng))
        model_dir = os.path.expanduser(model_dir)
        os.makedirs(model_dir, exist_ok=True)
        ae = self._autoencoder(int(batch_size))
        fp = C.POINTER(C.c_float)
        _lib.check(self._lib.b2g_autoencoder_set_dataset(ae, inputs.ctypes.data_as(fp),
                                                          None if same else targets.ctypes.data_as(fp), inputs.shape[0]))
        lr = self._learning_rate

        def train_epoch(order, bs):
            loss = C.c_double()
            _lib.check(self._lib.b2g_autoencoder_train_epoch(ae, order.ctypes.data_as(C.POINTER(C.c_int32)), order.size, bs, lr,
                                                             C.byref(loss)))
            return loss.value

        def evaluate(start, count):
            loss = C.c_double()
            _lib.check(self._lib.b2g_autoencoder_evaluate(ae, start, count, C.byref(loss)))
            return loss.value

        model_path = os.path.join(model_dir, "model.h5")
        history = fit(inputs.shape[0], int(batch_size), int(epochs), train_epoch, evaluate,
                      lambda epoch: self.save_weights(model_path), os.path.join(model_dir, "history.csv"), self._rng)
        self.set_model_weights(self.get_weights())     # encode() follows the last epoch
        return history

    def test(self, inputs, targets):
        """Keras ``evaluate``: the mean squared error over the set."""
        inputs = self._check_imgs(inputs, "inputs")
        same = targets is None or targets is inputs
        targets = inputs if same else self._check_imgs(targets, "targets")
        ae = self._autoencoder(self._train_batch)
        fp = C.POINTER(C.c_float)
        _lib.check(self._lib.b2g_autoencoder_set_dataset(ae, inputs.ctypes.data_as(fp),
                                                          None if same else targets.ctypes.data_as(fp), inputs.shape[0]))
        loss = C.c_double()
        _lib.check(self._lib.b2g_autoencoder_evaluate(ae, 0, inputs.shape[0], C.byref(loss)))
        return float(loss.value)

    def predict(self, imgs):
        """Reconstructions [n, 64, 64, 1]."""
        imgs = self._check_imgs(imgs)
        ae = self._autoencoder(self._train_batch)
        out = np.empty(imgs.shape, np.float32)
        fp = C.POINTER(C.c_float)
        _lib.check(self._lib.b2g_autoencoder_predict(ae, imgs.ctypes.data_as(fp), imgs.shape[0], out.ctypes.data_as(fp)))
        return out

    def step(self, inputs, targets=None, lr=None, apply_update=True):
        """One explicit training step on a host batch; returns (loss, gradients [(kernel, bias)] in model.h5 order)."""
        inputs = self._check_imgs(inputs, "inputs")
        ae = self._autoencoder(inputs.shape[0])
        fp = C.POINTER(C.c_float)
        tg = None if targets is None else self._check_imgs(targets, "targets")
        loss = C.c_double()
        _lib.check(self._lib.b2g_autoencoder_step(ae, inputs.ctypes.data_as(fp), None if tg is None else tg.ctypes.data_as(fp),
                                                  inputs.shape[0], self._learning_rate if lr is None else float(lr),
                                                  1 if apply_update else 0, C.byref(loss)))
        return loss.value, self._pull(self._lib.b2g_autoencoder_get_grad)

    def reset_optimizer(self):
        if self._ae:
            _lib.check(self._lib.b2g_autoencoder_reset_optimizer(self._ae))

    def set_weights(self, arrays):
        """arrays: [(kernel, bias)] for each conv then the dense layer (Keras layouts)."""
        n = self._lib.b2g_encoder_n_layers(self._handle)
        if len(arrays) != n:
            raise ValueError(f"expected {n} (kernel, bias) pairs, got {len(arrays)}")
        fp = C.POINTER(C.c_float)
        loaded = []
        for i, (k, b) in enumerate(arrays):
            k = np.ascontiguousarray(k, np.float32)
            b = np.ascontiguousarray(b, np.float32)
            _lib.check(self._lib.b2g_encoder_set_weights(self._handle, i, k.ctypes.data_as(fp), k.size, b.ctypes.data_as(fp), b.size))
            loaded.append((k.copy(), b.copy()))
        self._encoder_arrays = loaded

    def weights_digest(self) -> str:
        """sha256 over the encoder half's shapes and float32 weights (what a training state records of the encoder it was
        trained through)."""
        arrays = getattr(self, "_encoder_arrays", None)
        if arrays is None:
            raise ValueError("the encoder has no weights (load_weights first)")
        h = hashlib.sha256()
        for k, b in arrays:
            for a in (k, b):
                h.update(repr(a.shape).encode())
                h.update(a.tobytes())
        return h.hexdigest()

    def load_weights(self, model_dir):
        """Loads model.h5; when it also holds the decoder half (the shipped files do), predict / test / train use it."""
        model_dir = os.path.expanduser(model_dir)
        weights = h5min.load_keras_weights(os.path.join(model_dir, "model.h5"))
        self.model_dir = model_dir
        names = keras_layer_names(len(self.network))
        if all(f"{n}/kernel" in weights and f"{n}/bias" in weights for n in names):
            self.set_model_weights([(weights[f"{n}/kernel"], weights[f"{n}/bias"]) for n in names])
        else:
            self.set_weights(keras_encoder_arrays(weights, len(self.network)))

    def encode(self, imgs):
        imgs = np.ascontiguousarray(imgs, np.float32)
        if imgs.ndim != 4 or imgs.shape[1:] != self.input_shape:
            raise ValueError(f"expected imgs of shape (n, {self.input_shape}), got {imgs.shape}")
        n = imgs.shape[0]
        out = np.empty((n, self.encoding_dim), np.float32)
        fp = C.POINTER(C.c_float)
        for s in range(0, n, self._max_batch):          # keras predict() batches internally too (batch_size=32)
            e = min(n, s + self._max_batch)
            _lib.check(self._lib.b2g_encoder_encode(self._handle, imgs[s:e].ctypes.data_as(fp), e - s, out[s:e].ctypes.data_as(fp)))
        return out

    @property
    def encoding_shape(self):
        return (self.encoding_dim,)

    def _close_ae(self):
        if self._ae:
            self._lib.b2g_autoencoder_destroy(self._ae)
            self._ae = C.c_void_p()
            self._ae_batch = 0

    def close(self):
        self._close_ae()
        if self._handle:
            self._lib.b2g_encoder_destroy(self._handle)
            self._handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DeferredEncodedDepthImgSensor:
    """Drop-in for the reference's ``EncodedDepthImgSensor(config, sensor, robot)`` (sensor.py:169-230) that defers the
    encoding: ``get_state()`` renders and filters the depth frame exactly as the reference does and returns it flattened in
    HWC order, NOT encoded.  The env's observation is then ``[H*W depth | tail]``; ``vec_env.VecEncodeDepth`` encodes the
    frames of all envs at once in the learner's process (or hands them to the learner, which encodes them on its device).
    It never touches the CUDA library, so ``SubprocVecEnv`` workers hold no CUDA context and no copy of the encoder.
    ``visualize: true`` is refused: the reconstruction window needs the decoder in the worker."""

    def __init__(self, config, sensor, robot):
        import yaml
        from .spaces import Box
        self.scope = 'encoded_img_sensor'
        self._sensor = sensor
        self._robot = robot
        self.scene_type = config['scene'].get('scene_type', "OnTable")
        config = config['sensor']
        if config.get('visualize', False):
            raise NotImplementedError("DeferredEncodedDepthImgSensor: sensor.visualize needs the decoder in the env worker; use "
                                      "the reference's EncodedDepthImgSensor to watch reconstructions")
        self.encoder_dir = os.path.expanduser(config['encoder_dir'])
        with open(os.path.join(self.encoder_dir, 'config.yaml')) as f:
            self.encoding_dim = int(yaml.safe_load(f)['encoding_dim'])
        self.height, self.width = (int(d) for d in sensor.state_space.shape[:2])
        self.state_space = Box(0.0, np.inf, (self.height * self.width,), np.float32)

    def get_state(self):
        """The filtered depth frame [H*W] (HWC order, one channel), the input of ``encoder.encode``."""
        # Render
        _, img, mask = self._sensor.get_state()

        # Filter (sensor.py:212-219)
        img[mask == 0] = 0.
        img[mask == self._robot.robot_id] = 0.
        if self.scene_type == "OnTable":
            img[mask == 1] = 0.
            img[mask == 2] = 0.
        return np.asarray(img, np.float32).reshape(-1)
