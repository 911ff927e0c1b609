"""Float64 PyTorch-CPU restatement of one training step of the reference's auto-encoder (encoders.py:84-136, Keras 2.2.4 on
TF 1.14), the yardstick of csrc/autoencoder.cu.  The forward follows oracle/encoder_ref.py; the choices Keras makes and
this file restates:

1. LeakyReLU is ``K.relu(x, alpha) = relu(x) - alpha * relu(-x)``; TF's ReLU gradient at exactly 0 is 0, so the LeakyReLU
   gradient at 0 is 0 (``torch.nn.functional.leaky_relu`` would give alpha there).  Zeroed image regions and zero biases
   make exact zeros common on the first step.
2. Initialisation: glorot_uniform kernels (``b200grasp.encoders.glorot_init``), zero biases.
3. Keras Adam: b1 = 0.9, b2 = 0.999, eps = K.epsilon() = 1e-7; lr_t = lr * sqrt(1 - b2^t) / (1 - b1^t) with t = 1 on the
   first step; m = b1 m + (1 - b1) g; v = b2 v + (1 - b2) g^2; p -= lr_t * m / (sqrt(v) + eps).
4. Loss: mean_squared_error over every pixel of the batch.
"""
from __future__ import annotations

import math
from typing import Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from oracle.encoder_ref import same_pad


def conv_same(x: torch.Tensor, w_hwio: torch.Tensor, b: torch.Tensor, s: int) -> torch.Tensor:
    """oracle/encoder_ref.py's 'same' conv, with the kernel made contiguous so that autograd's CPU conv can take its gradient."""
    kh, kw = w_hwio.shape[:2]
    pt, pb = same_pad(x.shape[2], kh, s)
    pl, pr = same_pad(x.shape[3], kw, s)
    return F.conv2d(F.pad(x, (pl, pr, pt, pb)), w_hwio.permute(3, 2, 0, 1).contiguous(), b, stride=s)


def lrelu(x: torch.Tensor, alpha: float) -> torch.Tensor:
    return F.relu(x) - alpha * F.relu(-x)


def forward(params: Sequence[Tuple[torch.Tensor, torch.Tensor]], x: torch.Tensor, network, alpha: float) -> torch.Tensor:
    """params: 2L+2 (kernel, bias) in model.h5 order; x [N,H,W,1].  Returns the reconstruction [N,H,W,1]."""
    L = len(network)
    strides = [int(l["strides"]) for l in network]
    h = x.permute(0, 3, 1, 2)
    for (k, b), s in zip(params[:L], strides):
        h = lrelu(conv_same(h, k, b, s), alpha)
    shape = h.shape[1:]
    z = lrelu(h.permute(0, 2, 3, 1).reshape(h.shape[0], -1) @ params[L][0] + params[L][1], alpha)
    h = lrelu(z @ params[L + 1][0] + params[L + 1][1], alpha)
    h = h.reshape(-1, shape[1], shape[2], shape[0]).permute(0, 3, 1, 2)
    for j, i in enumerate(reversed(range(1, L))):
        h = F.interpolate(h, scale_factor=strides[i], mode="nearest")
        k, b = params[L + 2 + j]
        h = lrelu(conv_same(h, k, b, 1), alpha)
    h = F.interpolate(h, scale_factor=strides[0], mode="nearest")
    k, b = params[-1]
    return conv_same(h, k, b, 1).permute(0, 2, 3, 1)


def loss_and_grads(arrays, x: np.ndarray, t: np.ndarray, network, alpha: float, dtype=torch.float64):
    """Mean squared error and its gradients [(dkernel, dbias)] (numpy, float64)."""
    params = [(torch.tensor(np.asarray(k), dtype=dtype, requires_grad=True), torch.tensor(np.asarray(b), dtype=dtype, requires_grad=True))
              for k, b in arrays]
    y = forward(params, torch.tensor(x, dtype=dtype), network, alpha)
    loss = ((y - torch.tensor(t, dtype=dtype)) ** 2).mean()
    loss.backward()
    return loss.item(), [(k.grad.numpy(), b.grad.numpy()) for k, b in params]


def predict(arrays, x: np.ndarray, network, alpha: float, dtype=torch.float64) -> np.ndarray:
    with torch.no_grad():
        params = [(torch.tensor(np.asarray(k), dtype=dtype), torch.tensor(np.asarray(b), dtype=dtype)) for k, b in arrays]
        return forward(params, torch.tensor(x, dtype=dtype), network, alpha).numpy()


class Adam:
    """Keras Adam over a list of (kernel, bias) pairs (float64)."""

    def __init__(self, arrays, lr: float, b1=0.9, b2=0.999, eps=1e-7):
        self.p = [np.array(a, np.float64) for kb in arrays for a in kb]
        self.m = [np.zeros_like(a) for a in self.p]
        self.v = [np.zeros_like(a) for a in self.p]
        self.t, self.lr, self.b1, self.b2, self.eps = 0, lr, b1, b2, eps

    def arrays(self):
        return [(self.p[2 * i], self.p[2 * i + 1]) for i in range(len(self.p) // 2)]

    def update(self, grads):
        """The change this step makes to every parameter (without advancing the optimiser)."""
        t = self.t + 1
        lr_t = self.lr * math.sqrt(1 - self.b2 ** t) / (1 - self.b1 ** t)
        out = []
        for i, g in enumerate(a for kb in grads for a in kb):
            m = self.b1 * self.m[i] + (1 - self.b1) * g
            v = self.b2 * self.v[i] + (1 - self.b2) * g * g
            out.append(-lr_t * m / (np.sqrt(v) + self.eps))
        return out

    def update_bound(self, grads, em, ev):
        """How far this step's update can move when the first moments m (after this step's gradient) are off by up to em
        and the second moments v by up to ev, element by element.  The update is monotone in m and in v, so the extremes
        sit at the corners of that box."""
        t = self.t + 1
        lr_t = self.lr * math.sqrt(1 - self.b2 ** t) / (1 - self.b1 ** t)
        out = []
        for i, g in enumerate(a for kb in grads for a in kb):
            m = self.b1 * self.m[i] + (1 - self.b1) * g
            v = self.b2 * self.v[i] + (1 - self.b2) * g * g
            u = lambda mm, vv: lr_t * mm / (np.sqrt(np.maximum(vv, 0.0)) + self.eps)
            u0 = u(m, v)
            out.append(np.max([np.abs(u(m + sm * em[i], v + sv * ev[i]) - u0) for sm in (-1, 1) for sv in (-1, 1)], axis=0))
        return out

    def step(self, grads):
        self.t += 1
        lr_t = self.lr * math.sqrt(1 - self.b2 ** self.t) / (1 - self.b1 ** self.t)
        for i, g in enumerate(a for kb in grads for a in kb):
            self.m[i] = self.b1 * self.m[i] + (1 - self.b1) * g
            self.v[i] = self.b2 * self.v[i] + (1 - self.b2) * g * g
            self.p[i] = self.p[i] - lr_t * self.m[i] / (np.sqrt(self.v[i]) + self.eps)
