"""Every contraction of engine v2's fused forward and backward launches, held element by element to a float64 contraction of
the inputs it actually read.

The step-level tests compare whole outputs and per-tensor gradient norms with the float64 oracle.  A kernel bug confined to
one tile, one split, one N block or one precision class of a contraction (a dropped correction product, a wrong row limit)
moves those norms by less than their bars.  Here, after one explicit step, `b2g_debug_tensor` reads back every plane tensor of
the engine (include/b200grasp.h lists the layouts) and each problem of csrc/engine_v2.cu is recomputed in float64 from the
planes its operands came from:
  * bit for bit where the answer is known: the weight planes (planes2_kernel), the normalised image S and the feature-row
    columns the gather writes (gather2_kernel), the zero pads, the fp32 copy of the features, and the zeros of every gradient
    map where the stored ReLU mask is zero;
  * within |got - ref| <= gamma * sum|a||b| + r * |ref| elsewhere, every sum over the element's own reduction (bias included
    as one more term), with gamma written out per problem from the engine's arithmetic (`_gamma`): the operand split, one
    allowance per tensor-core k-step of the accumulator chain, and the fp32 additions outside the tensor core; r is the
    rounding of the stored planes.  relu is 1-Lipschitz, so the same bar holds across the ReLU kink.
`heads_wgrad_kernel` (fp32 FMAs on the CUDA cores) is held the same way, and the wgmma gather-GEMM engine (gg_tc, the MLP
policy's engine) through `b2g_debug_gemm` at the tile edges of M, N and K.

`pytest -s` prints the worst err/bar of every problem of every case.
"""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from b200grasp import _lib, synth
from oracle import sac_ref as R
from oracle import sac_ref_np as N
from tests.test_conv1_s2d_cpu import conv1_krow, s2d, w1t
from tests.gg_tc_ref import SPLIT2, U32, U_TC, Report, bf, bf16_split, gg_gammas
from tests.test_gpu_configs import vecnorm_for
from tests.util import load_case, make_batch, make_learner

KF = 576
NETS = ("pi", "values", "target")
SCOPES = ("model/pi", "model/values_fn", "target/values_fn")
HEADS = (("pi", "model/pi"), ("vf", "model/values_fn/vf"), ("qf1", "model/values_fn/qf1"), ("qf2", "model/values_fn/qf2"))

# ------------------------------------------------------------------------------------------------ error model
# 3 planes, 6 products (p + q <= 2): the missing A_1 B_2 + A_2 B_1 + A_2 B_2, with |A_1| <= 2^-8 (1 + 2^-8) |a|, |A_2| <= 2^-16 |a|
SPLIT3 = 2 * 2.0 ** -8 * (1 + 2.0 ** -8) * 2.0 ** -16 + 2.0 ** -32
R2 = 2.0 ** -16           # a value stored as 2 BF16 planes (3 planes hold an fp32 value exactly)


def _gamma(split, ksteps, adds):
    """split: the operand split's missing products; ksteps: k-steps of 16 in one accumulator chain, each allowed two units
    (products, accumulator) of 2^-23 of the chain's sum|a||b|, which bounds every partial sum, times 1 + 2^-6 for the
    correction groups' own chains; adds: fp32 additions after the chain (group sum, bias, split-K workspace, red.add).  The
    1 % covers the second-order terms of these bounds."""
    return 1.01 * (split + 2 * U_TC * ksteps * (1 + 2.0 ** -6) + U32 * adds)


def _cdiv(a, b):
    return -(-a // b)


def problem_gammas(B, ci, split_fc1=3, split_dgrad=1):
    """gamma of every problem, from the tile shapes of csrc/engine_v2.cu v2_create (chunks of 64 K rows = 4 k-steps unless
    noted; splits = K-splits of one output tile)."""
    cp = 1 if ci == 1 else 4
    c3 = _cdiv(B, 4)                                                      # conv3 / conv2 wgrad chunks: 4 samples
    s3 = max(1, min(c3, max(14, _cdiv(c3, 16))))
    s2 = max(1, min(c3, max(8, _cdiv(c3, 8))))
    c1 = 4 * B                                                            # conv1 wgrad chunks: a quarter sample
    s1 = max(1, min(c1, max(84 // (1 if cp == 1 else 2), _cdiv(c1, 16))))
    return {
        # forward: 3 planes, 6 products, 3 accumulator groups summed (2 adds) + bias
        "conv1": _gamma(SPLIT3, 4 * cp, 3),
        "conv2": _gamma(SPLIT3, 32, 3),
        "conv3": _gamma(SPLIT3, 36, 3),
        "cnn_fc1": _gamma(SPLIT3, 4 * _cdiv(16, split_fc1), 3 + split_fc1),
        "fc0": _gamma(SPLIT3, 4, 2 + 9),                                  # one K-chunk per CTA, 9 red.adds
        # backward: 2 planes, 3 products, 2 groups (1 add); heads_dgrad (K = H | 3H) in check_step
        "fc1_dgrad": _gamma(SPLIT2, 4 * _cdiv(8, split_dgrad), 1 + split_dgrad),
        "fc1_wgrad": _gamma(SPLIT2, 4 * _cdiv(B, 64), 1),
        "conv3_dgrad": _gamma(SPLIT2, 36, 1),
        "conv3_wgrad": _gamma(SPLIT2, 4 * _cdiv(c3, s3), 1 + s3),
        "conv2_dgrad": _gamma(SPLIT2, 16, 1),
        "conv2_wgrad": _gamma(SPLIT2, 9 * _cdiv(c3, s2), 1 + s2),          # 144-row chunks: 9 k-steps
        "conv1_wgrad": _gamma(SPLIT2, 4 * _cdiv(c1, s1), 1 + s1),
    }


# ------------------------------------------------------------------------------------------------ layouts in float64
def img_from_s(S, ci):
    """S [B, 16, 16, 4, 4, Cp] -> image [B, 64, 64, ci] (inverse of test_conv1_s2d_cpu.s2d)."""
    B = S.shape[0]
    return S.transpose(0, 1, 3, 2, 4, 5).reshape(B, 64, 64, -1)[..., :ci]


def hwio_from_w1t(W, ci):
    """W1T rows [32][64 Cp] -> HWIO [8, 8, ci, 32]."""
    return W[:, [conv1_krow(r, ci) for r in range(64 * ci)]].T.reshape(8, 8, ci, 32)


def hwio_from_t(WT, shape):
    """A transposed K-major weight [N][K] (W2T, W3T) -> HWIO shape."""
    return WT.reshape(shape[-1], -1).T.reshape(shape)


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x, np.float64))


def conv(x, w, s):
    """NHWC x, HWIO w -> NHWC sum, and the same over |x|, |w|."""
    f = lambda a, b: Fn.conv2d(_t(a).permute(0, 3, 1, 2), _t(b).permute(3, 2, 0, 1), stride=s).permute(0, 2, 3, 1).numpy()
    return f(x, w), f(np.abs(x), np.abs(w))


def conv_t(dz, w, s, out_hw):
    """The input gradient of conv(., w, s) for the output gradient dz (NHWC), and over |dz|, |w|."""
    op = out_hw - ((dz.shape[1] - 1) * s + w.shape[0])

    def f(a, b):
        return Fn.conv_transpose2d(_t(a).permute(0, 3, 1, 2), _t(b).permute(3, 2, 0, 1), stride=s,
                                   output_padding=op).permute(0, 2, 3, 1).numpy()
    return f(dz, w), f(np.abs(dz), np.abs(w))


def conv_w(x, dz, k, s):
    """The weight gradient (HWIO [k, k, Ci, Co]) of conv(x, ., s) for the output gradient dz, and over |x|, |dz|."""
    def f(a, b):
        g = torch.nn.grad.conv2d_weight(_t(a).permute(0, 3, 1, 2), (b.shape[3], a.shape[3], k, k), _t(b).permute(0, 3, 1, 2),
                                        stride=s)
        return g.permute(2, 3, 1, 0).numpy()
    return f(x, dz), f(np.abs(x), np.abs(dz))


def mm(a, b):
    return a @ b, np.abs(a) @ np.abs(b)


# ------------------------------------------------------------------------------------------------ checks
def read(L, name):
    """All planes of one debug tensor: uint16 [planes][numel] for BF16 planes, float32 [1][numel] for fp32 buffers."""
    n, p, eb = C.c_int64(), C.c_int32(), C.c_int32()
    _lib.check(L.lib.b2g_debug_tensor_info(L.h, name.encode(), C.byref(n), C.byref(p), C.byref(eb)))
    out = np.empty((p.value, n.value), np.uint16 if eb.value == 2 else np.float32)
    for k in range(p.value):
        _lib.check(L.lib.b2g_debug_tensor(L.h, name.encode(), k, out[k].ctypes.data_as(C.c_void_p), out[k].nbytes))
    return out


def check_weight_planes(rep, T, params, ci, A, H):
    """planes2_kernel: every weight layout of the engine, bit for bit, pads included."""
    cp = 1 if ci == 1 else 4

    def t3(w):                               # [K][N] -> planes of the transposed [N][K]
        return [p.T for p in bf16_split(w, 3)]

    for k in range(3):
        want = np.zeros((64, 64 * cp), np.uint16)
        want_t = np.zeros((32, 64 * cp), np.uint16)
        rows = [conv1_krow(r, ci) for r in range(64 * ci)]
        for half, scope in enumerate(SCOPES[:2]):
            want[32 * half:32 * half + 32, rows] = t3(params[f"{scope}/cnn1/w"].reshape(64 * ci, 32))[k]
        want_t[:, rows] = t3(params["target/values_fn/cnn1/w"].reshape(64 * ci, 32))[k]
        rep.exact(f"planes2/W1T/online[{k}]", T["W1T/online"][k].reshape(64, -1), want)
        rep.exact(f"planes2/W1T/target[{k}]", T["W1T/target"][k].reshape(32, -1), want_t)
    for n, scope in enumerate(SCOPES):
        for tn, wn, K, Nn in (("W2T", "cnn2", 512, 64), ("W3T", "cnn3", 576, 64), ("WfT", "cnn_fc1", 1024, 512)):
            w = params[f"{scope}/{wn}/w"].reshape(K, Nn)
            for k, p in enumerate(t3(w)):
                rep.exact(f"planes2/{tn}/{NETS[n]}[{k}]", T[f"{tn}/{NETS[n]}"][k].reshape(Nn, K), p)
            if n < 2:
                nt = tn[:-1] + "n"
                for k, p in enumerate(bf16_split(w, 2)):
                    rep.exact(f"planes2/{nt}/{NETS[n]}[{k}]", T[f"{nt}/{NETS[n]}"][k].reshape(K, Nn), p)
        heads = [("pi", "model/pi")] if n == 0 else HEADS[1:] if n == 1 else [("vf", "target/values_fn/vf")]
        kt = np.zeros((3, len(heads) * H, KF), np.uint16)
        kn = np.zeros((2, KF, len(heads) * H), np.uint16)
        for j, (_, hp) in enumerate(heads):
            w = params[f"{hp}/fc0/kernel"]                    # [513 (+ A)][H]
            for k, p in enumerate(bf16_split(w, 3)):
                kt[k, j * H:(j + 1) * H, :w.shape[0]] = p.T
                if k < 2:
                    kn[k, :w.shape[0], j * H:(j + 1) * H] = p
        for k in range(3):
            rep.exact(f"planes2/K0T/{NETS[n]}[{k}]", T[f"K0T/{NETS[n]}"][k].reshape(kt[k].shape), kt[k])
        if n < 2:
            for k in range(2):
                rep.exact(f"planes2/K0n/{NETS[n]}[{k}]", T[f"K0n/{NETS[n]}"][k].reshape(kn[k].shape), kn[k])


def normalised(x, mean, var, vn, norm_obs):
    """gather2's value of raw fp32 observations x: float64 (x - mean) * istd, clipped, rounded to fp32, then / 255 in fp32."""
    x = np.asarray(x, np.float32).astype(np.float64)
    if norm_obs:
        istd = 1.0 / np.sqrt(np.asarray(var, np.float64) + float(vn["epsilon"]))
        clip = float(vn["clip_obs"])
        x = np.clip((x - np.asarray(mean, np.float64)) * istd, -clip, clip)
    return (x.astype(np.float32) / np.float32(255.0)).astype(np.float32)


def check_gather(rep, T, obs_raw, next_raw, act, vn, ci, B, norm_obs=True):
    """gather2_kernel: S and the feature-row columns it writes, bit for bit; pad channels zero."""
    for key, raw in (("S/obs", obs_raw), ("S/next_obs", next_raw)):
        y = normalised(raw[..., :ci], vn["obs_mean"][..., :ci], vn["obs_var"][..., :ci], vn, norm_obs)
        planes = bf16_split(y, 3)
        for k in range(3):
            want = s2d(planes[k].astype(np.float64)).astype(np.uint16)     # pad channels: zero
            rep.exact(f"gather2/{key}[{k}]", T[key][k].reshape(want.shape), want)
    m, v = vn["obs_mean"][0, 0, ci], vn["obs_var"][0, 0, ci]                # the actuator value: pixel [0, 0] of the last plane
    a, an = (normalised(raw[:, 0, 0, ci], m, v, vn, norm_obs) for raw in (obs_raw, next_raw))
    for n in range(3):
        Fp = T[f"F/{NETS[n]}"].reshape(3, B, KF)
        cols = [(a if n < 2 else an)[:, None]] + ([np.asarray(act, np.float32)] if n == 1 else [])
        v = np.concatenate(cols, 1).astype(np.float32)
        for k, p in enumerate(bf16_split(v, 3)):
            rep.exact(f"gather2/F/{NETS[n]}[{k}] cols 512..", Fp[k][:, 512:512 + v.shape[1]], p)


def check_step(rep, T, G, params, B, ci, A, H, gam):
    """Every ACT / RAW / DGRAD / WGRAD problem and the bias column sums, against float64 of the planes the engine read."""
    cp = 1 if ci == 1 else 4
    FS = _cdiv(513 + A, 8) * 8
    s3 = lambda name: bf(T[name][0]) + bf(T[name][1]) + bf(T[name][2])      # 3-plane value (forward operands)
    s2 = lambda name: bf(T[name][0]) + bf(T[name][1])                       # the 2 planes the backward reads
    # ---------------------------------------------------------------- forward
    H1 = {n: s3(f"H1/{n}").reshape(B, 15, 15, 32) for n in NETS}
    H2 = {n: s3(f"H2/{n}").reshape(B, 6, 6, 64) for n in NETS}
    H3 = {n: s3(f"H3/{n}").reshape(B, 1024) for n in NETS}
    F = {n: s3(f"F/{n}").reshape(B, KF) for n in NETS}
    W1 = {"online": s3("W1T/online").reshape(64, 64 * cp), "target": s3("W1T/target").reshape(32, 64 * cp)}
    w1 = {"pi": W1["online"][:32], "values": W1["online"][32:], "target": W1["target"]}
    img = {"obs": img_from_s(s3("S/obs").reshape(B, 16, 16, 4, 4, cp), ci),
           "next_obs": img_from_s(s3("S/next_obs").reshape(B, 16, 16, 4, 4, cp), ci)}
    for n, scope in zip(NETS, SCOPES):
        b1, b2, b3, bf1 = (params[f"{scope}/{k}/b"].reshape(-1).astype(np.float64) for k in ("cnn1", "cnn2", "cnn3", "cnn_fc1"))
        z, m = conv(img["next_obs" if n == "target" else "obs"], hwio_from_w1t(w1[n], ci), 4)
        rep.hold(f"conv1/{n}", H1[n], np.maximum(z + b1, 0), m + np.abs(b1), gam["conv1"])
        z, m = conv(H1[n], hwio_from_t(s3(f"W2T/{n}"), (4, 4, 32, 64)), 2)
        rep.hold(f"conv2/{n}", H2[n], np.maximum(z + b2, 0), m + np.abs(b2), gam["conv2"])
        z, m = conv(H2[n], hwio_from_t(s3(f"W3T/{n}"), (3, 3, 64, 64)), 1)
        rep.hold(f"conv3/{n}", H3[n].reshape(B, 4, 4, 64), np.maximum(z + b3, 0), m + np.abs(b3), gam["conv3"])
        z, m = mm(H3[n], s3(f"WfT/{n}").reshape(512, 1024).T)
        rep.hold(f"cnn_fc1/{n}", F[n][:, :512], np.maximum(z + bf1, 0), m + np.abs(bf1), gam["cnn_fc1"])
        # ACT bit-exact facts: the pads stay zero, the fp32 copy is the 3-plane value, the mask is value > 0
        ncol = 513 + (A if n == "values" else 0)
        for k in range(3):
            rep.exact(f"F/{n}[{k}] pad columns", T[f"F/{n}"][k].reshape(B, KF)[:, ncol:], np.zeros((B, KF - ncol), np.uint16))
        f32 = T[f"F32/{n}"][0].reshape(B, FS).astype(np.float64)
        rep.exact(f"F32/{n} = 3-plane F", f32[:, :ncol], F[n][:, :ncol])
        rep.exact(f"F/{n} mask = F32 > 0", T[f"F/{n}"][0].reshape(B, KF)[:, :512] != 0, f32[:, :512] > 0)
        Nn = 3 * H if n == "values" else H
        z, m = mm(F[n], s3(f"K0T/{n}").reshape(Nn, KF).T)
        got = T["z0v"][0] if n == "values" else T[f"z0/{n}"][0]
        rep.hold(f"fc0/{n}", got.reshape(B, Nn), z, m, gam["fc0"])
    # ---------------------------------------------------------------- backward (pi, values)
    dZ1 = s2("dZ1").reshape(B, 15, 15, 2, 32)
    dZ1_raw = [T["dZ1"][k].reshape(B, 15, 15, 2, 32) for k in range(2)]
    for j, (n, scope) in enumerate(zip(NETS[:2], SCOPES[:2])):
        dz0 = s2("dz0pi" if n == "pi" else "dz0v").reshape(B, -1)
        Kd = dz0.shape[1]
        dZ4, dZ3 = s2(f"dZ4/{n}").reshape(B, 512), s2(f"dZ3/{n}").reshape(B, 1024)
        dZ2 = s2(f"dZ2/{n}").reshape(B, 6, 6, 64)
        masks = {"dZ4": T[f"F/{n}"][0].reshape(B, KF)[:, :512] != 0, "dZ3": T[f"H3/{n}"][0].reshape(B, 1024) != 0,
                 "dZ2": T[f"H2/{n}"][0].reshape(B, 6, 6, 64) != 0, "dZ1": T[f"H1/{n}"][0].reshape(B, 15, 15, 32) != 0}
        cs = {}

        def dgrad(name, got, z, m, mask, g, key, n_red):
            """n_red: red.adds into one bias element (epilogue warps x column groups x tiles of the problem)"""
            ref = np.where(mask, z, 0.0)
            rep.hold(name, got, ref, np.where(mask, m, 0.0), g, R2)
            cs[key] = (ref, np.where(mask, m, 0.0), g, n_red)

        z, m = mm(dz0, s2(f"K0n/{n}").reshape(KF, Kd)[:512].T)
        dgrad(f"heads_dgrad/{n}", dZ4, z, m, masks["dZ4"], _gamma(SPLIT2, Kd // 16, 1), "cnn_fc1", 4 * _cdiv(B, 128))
        z, m = mm(dZ4, s2(f"Wfn/{n}").reshape(1024, 512).T)
        dgrad(f"fc1_dgrad/{n}", dZ3, z, m, masks["dZ3"], gam["fc1_dgrad"], "cnn3", 4 * 16 * _cdiv(B, 128))
        z, m = mm(s2(f"H3/{n}").reshape(B, 1024).T, dZ4)
        rep.hold(f"fc1_wgrad/{n}", G[f"{scope}/cnn_fc1/w"], z, m, gam["fc1_wgrad"])
        z, m = conv_t(dZ3.reshape(B, 4, 4, 64), s2(f"W3n/{n}").reshape(3, 3, 64, 64), 1, 6)
        dgrad(f"conv3_dgrad/{n}", dZ2, z, m, masks["dZ2"], gam["conv3_dgrad"], "cnn2", 4 * _cdiv(B, 3))
        H2b = s2(f"H2/{n}").reshape(B, 6, 6, 64)
        z, m = conv_w(H2b, dZ3.reshape(B, 4, 4, 64), 3, 1)
        rep.hold(f"conv3_wgrad/{n}", G[f"{scope}/cnn3/w"], z, m, gam["conv3_wgrad"])
        z, m = conv_t(dZ2, s2(f"W2n/{n}").reshape(4, 4, 32, 64), 2, 15)
        dgrad(f"conv2_dgrad/{n}", dZ1[:, :, :, j], z, m, masks["dZ1"], gam["conv2_dgrad"], "cnn1", 4 * 4 * _cdiv(B, 2))
        z, m = conv_w(s2(f"H1/{n}").reshape(B, 15, 15, 32), dZ2, 4, 2)
        rep.hold(f"conv2_wgrad/{n}", G[f"{scope}/cnn2/w"], z, m, gam["conv2_wgrad"])
        Sb = img_from_s(s2("S/obs").reshape(B, 16, 16, 4, 4, cp), ci)
        z, m = conv_w(Sb, dZ1[:, :, :, j], 8, 4)
        rep.hold(f"conv1_wgrad/{n}", G[f"{scope}/cnn1/w"], z, m, gam["conv1_wgrad"])
        # DGRAD zeros wherever the stored mask is zero
        for key, got in (("dZ4", [T[f"dZ4/{n}"][k].reshape(B, 512) for k in range(2)]),
                         ("dZ3", [T[f"dZ3/{n}"][k].reshape(B, 1024) for k in range(2)]),
                         ("dZ2", [T[f"dZ2/{n}"][k].reshape(B, 6, 6, 64) for k in range(2)]),
                         ("dZ1", [p[:, :, :, j] for p in dZ1_raw])):
            for k in range(2):
                rep.exact(f"{key}/{n}[{k}] = 0 off the mask", np.where(masks[key], 0, got[k]), np.zeros_like(got[k]))
        # bias gradients: the DGRAD epilogues' column sums (butterfly over 32 rows, one red.add per warp and column)
        # (the fp32 values are summed: each element's own bar, then 5 butterfly levels and n_red red.adds of at most the
        # column's sum|x| each)
        for bname, (ref, mag, g, n_red) in cs.items():
            ch = 64 if bname in ("cnn3", "cnn2") else 32 if bname == "cnn1" else 512
            r2, m2 = ref.reshape(-1, ch), mag.reshape(-1, ch)
            own = g * m2.sum(0)
            rep.hold(f"colsum {bname}/b/{n}", G[f"{scope}/{bname}/b"].reshape(-1), r2.sum(0),
                     own + 1.01 * U32 * (5 + n_red) * (np.abs(r2).sum(0) + own), 1.0)


def check_heads_wgrad(rep, T, G, B, A, H):
    """heads_wgrad_kernel: fc0 / fc1 kernel and bias gradients of the four head MLPs, fp32 FMAs over a quarter of the batch per
    CTA, then 4 red.adds."""
    FS = _cdiv(513 + A, 8) * 8
    g = 1.01 * U32 * (_cdiv(B, 4) + 4)
    F0, F1 = (T[f"F32/{n}"][0].reshape(B, FS).astype(np.float64) for n in ("pi", "values"))
    dz0 = {"pi": T["dz0_pi"][0].reshape(B, H).astype(np.float64)}
    v3 = T["dz0_v3"][0].reshape(B, 3 * H).astype(np.float64)
    for j, q in enumerate(("vf", "qf1", "qf2")):
        dz0[q] = v3[:, j * H:(j + 1) * H]
    for q, hp in HEADS:
        M0 = 513 + (A if q.startswith("qf") else 0)
        X = (F0 if q == "pi" else F1)[:, :M0]
        z, m = mm(X.T, dz0[q])
        rep.hold(f"heads_wgrad/{q}/fc0/kernel", G[f"{hp}/fc0/kernel"], z, m, g)
        rep.hold(f"heads_wgrad/{q}/fc0/bias", G[f"{hp}/fc0/bias"], dz0[q].sum(0), np.abs(dz0[q]).sum(0), g)
        a0, d1 = (T[f"{k}/{q}"][0].reshape(B, H).astype(np.float64) for k in ("a0", "dz1"))
        z, m = mm(a0.T, d1)
        rep.hold(f"heads_wgrad/{q}/fc1/kernel", G[f"{hp}/fc1/kernel"], z, m, g)
        rep.hold(f"heads_wgrad/{q}/fc1/bias", G[f"{hp}/fc1/bias"], d1.sum(0), np.abs(d1).sum(0), g)


# ------------------------------------------------------------------------------------------------ the cases
@dataclasses.dataclass(frozen=True)
class Case:
    name: str
    B: int
    ci: int = 1
    A: int = 5
    H: int = 64
    params: str = "fresh"            # "fresh" (R.init_params) | "trained" (the depth run's weights) | "coherent" (trained,
                                     # cnn_fc1/w from coherent_fc1_weights)
    env: tuple = ()                  # (variable, value) pairs set before create
    seed: int = 0
    sampled: bool = False            # a graph-path step sampled from a replay with 8-bit RGB planes (else an explicit step)

    @property
    def cfg(self):
        return R.SACConfig(obs_shape=(64, 64, self.ci + 1), n_act=self.A, layers=(self.H, self.H), target_entropy=-float(self.A))

    @property
    def splits(self):
        e = dict(self.env)
        return int(e.get("B2G_SPLIT_FC1", 3)), int(e.get("B2G_SPLIT_FC1_DGRAD", 1))


CASES = [Case(f"depth_b{B}", B, params="trained") for B in (1, 3, 9, 129, 383)] + [
    Case("ci2_b77", 77, ci=2, seed=11),
    Case("ci3_a3_b77", 77, ci=3, A=3, seed=12),
    Case("rgbd_b77", 77, ci=4, seed=13),
    Case("h128_b63", 63, H=128, seed=14),
    Case("h256_b129", 129, H=256, seed=15),
    Case("a1_b40", 40, A=1, seed=16),
    Case("a8_b40", 40, A=8, seed=17),
] + [Case(f"split_fc1_{s}_b129", 129, params="trained", env=(("B2G_SPLIT_FC1", str(s)),)) for s in (1, 2, 6)] + [
    Case(f"split_dgrad_{s}_b129", 129, params="trained", env=(("B2G_SPLIT_FC1_DGRAD", str(s)),)) for s in (3, 8)] + [
    Case("coherent_fc1_split16_b129", 129, params="coherent", env=(("B2G_SPLIT_FC1", "16"),)),
    Case("rgbd_u8_sampled_b77", 77, ci=4, seed=18, sampled=True),
]
U8_PLANES = (0, 1, 2)                # the sampled RGB-D case stores its colour planes as one byte per pixel


# A dropped forward correction group (order 2: A0 B2 + A1 B1 + A2 B0, each ~2^-16 |a||b|) has random signs with ordinary
# weights, so over a K-long reduction it shrinks to ~2^-16 / sqrt(K) of sum|a||b|: below the tensor core's accumulation
# allowance of every forward problem.  The coherent case makes it add up: every cnn_fc1 weight is positive, with the
# significand 1.00000000 11111111 0 111111, so that its BF16 planes are p0 = 2^e, p1 = 2^e (2^-8 - 2^-16) and
# p2 = 2^e (2^-17 - 2^-23), all positive; its input H3 is a ReLU output, so A0 >= 0, and sum_k A0 B2 ~ 2^-17 sum|a||b|
# with one sign.  B2G_SPLIT_FC1 = 16 leaves one K-chunk (4 k-steps) per accumulator chain, which puts cnn_fc1's bar near
# 19 * 2^-23 sum|a||b|: a dropped g2 (or B2 plane) misses it by more than 3x (test_coherent_case_sees_a_dropped_g2).
COHERENT_MANTISSA = 0b00000000_11111111_0_111111


def coherent_fc1_weights(shape, seed):
    """Positive fp32 weights of the significand above and exponents 2^-9 .. 2^-6."""
    e = np.random.default_rng(seed).integers(127 - 9, 127 - 5, size=shape).astype(np.uint32)
    return ((e << 23) | np.uint32(COHERENT_MANTISSA)).view(np.float32)


# ================================================================================================ CPU
def test_coherent_case_sees_a_dropped_g2():
    w = coherent_fc1_weights((1024, 512), 0)
    p = [bf(x) for x in bf16_split(w, 3)]
    w64 = w.astype(np.float64)
    assert np.array_equal(p[0] + p[1] + p[2], w64) and (p[1] > 0).all() and (p[2] > 0).all()
    frac = p[2] / w64                                         # B2 / B: the same for every weight
    g = problem_gammas(129, 1, split_fc1=16)["cnn_fc1"]
    assert frac.min() > 3 * g, (frac.min(), g)                # sum_k A0 B2 >= frac sum A0 B, with A0 >= 0 (ReLU input)


def test_case_matrix_reaches_every_edge():
    depth = {c.B for c in CASES if c.ci == 1 and c.A == 5 and c.H == 64 and not c.env}
    assert {1, 3, 9, 129, 383} <= depth                       # one partial tile of each small period; a second partial tile
    assert {2, 3, 4} <= {c.ci for c in CASES if c.B == 77}    # Cp = 4 with 2, 1 and 0 pad channels
    assert ("h128", 63) in {(f"h{c.H}", c.B) for c in CASES} and ("h256", 129) in {(f"h{c.H}", c.B) for c in CASES}
    assert {514, 521} <= {513 + c.A for c in CASES}           # the q-nets' fc0 K of 576 rows
    assert {1, 2, 6} <= {c.splits[0] for c in CASES if c.B == 129} and {3, 8} <= {c.splits[1] for c in CASES if c.B == 129}
    for c in CASES:                                           # every split leaves each K-split a chunk (create refuses others)
        assert (c.splits[0] - 1) * _cdiv(16, c.splits[0]) < 16 and (c.splits[1] - 1) * _cdiv(8, c.splits[1]) < 8
    assert any(c.params == "coherent" and c.splits[0] == 16 for c in CASES)              # a dropped g2 adds up
    assert any(c.sampled and c.ci == 4 for c in CASES)        # the u8 frame_load4 gather from replay frames


def test_layout_restatements_reproduce_the_oracle():
    """The float64 side without a GPU: the oracle's own activations (oracle/sac_ref_np.py) through this file's layout
    restatements give the oracle's next layers, and random gradient maps give its input and weight gradients (im2col /
    col2im), to 1e-12."""
    rng = np.random.default_rng(5)
    for ci in (1, 3):
        B = 3
        cfg = R.SACConfig(obs_shape=(64, 64, ci + 1))
        p = {k: v.astype(np.float64) for k, v in R.init_params(cfg, seed=ci).items()}
        for k in [k for k in p if k.endswith("/b")]:
            p[k] = rng.standard_normal(p[k].shape) * 0.1
        x = rng.uniform(0, 1, (B, 64, 64, ci + 1))
        _, cache = N.cnn_fwd(x, p, "model/pi", ci)
        y1, y2, y3 = (cache[k][2].reshape(B, o, o, -1) for k, o in (("cnn1", 15), ("cnn2", 6), ("cnn3", 4)))
        W1 = w1t(p["model/pi/cnn1/w"])                        # the transposed K rows planes2 writes
        z, _ = conv(img_from_s(s2d(x[..., :ci]), ci), hwio_from_w1t(W1, ci), 4)
        np.testing.assert_allclose(np.maximum(z + p["model/pi/cnn1/b"].reshape(-1), 0), y1, rtol=1e-12, atol=1e-12)
        z, _ = conv(y1, hwio_from_t(p["model/pi/cnn2/w"].reshape(512, 64).T, (4, 4, 32, 64)), 2)     # W2T = [64][512]
        np.testing.assert_allclose(np.maximum(z + p["model/pi/cnn2/b"].reshape(-1), 0), y2, rtol=1e-12, atol=1e-12)
        z, _ = conv(y2, hwio_from_t(p["model/pi/cnn3/w"].reshape(576, 64).T, (3, 3, 64, 64)), 1)
        np.testing.assert_allclose(np.maximum(z + p["model/pi/cnn3/b"].reshape(-1), 0), y3, rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(np.maximum(y3.reshape(B, -1) @ p["model/pi/cnn_fc1/w"] + p["model/pi/cnn_fc1/b"], 0),
                                   cache["fc"][1], rtol=1e-12, atol=1e-12)
        # backward: the oracle's im2col / col2im forms
        for name, k, s, (xin, o) in (("cnn3", 3, 1, (y2, 4)), ("cnn2", 4, 2, (y1, 6)), ("cnn1", 8, 4, (x[..., :ci], 15))):
            w = p[f"model/pi/{name}/w"]
            dz = rng.standard_normal((B, o, o, w.shape[3]))
            cols, _ = N.im2col(np.ascontiguousarray(xin), k, s)
            np.testing.assert_allclose(conv_w(xin, dz, k, s)[0], (cols.T @ dz.reshape(-1, w.shape[3])).reshape(w.shape),
                                       rtol=1e-12, atol=1e-10)
            if name != "cnn1":
                ref = N.col2im(dz.reshape(-1, w.shape[3]) @ w.reshape(-1, w.shape[3]).T, xin.shape, k, s)
                np.testing.assert_allclose(conv_t(dz, w, s, xin.shape[1])[0], ref, rtol=1e-12, atol=1e-12)
        # conv1's weight gradient through S
        dz = rng.standard_normal((B, 15, 15, 32))
        cols, _ = N.im2col(np.ascontiguousarray(x[..., :ci]), 8, 4)
        np.testing.assert_allclose(conv_w(img_from_s(s2d(x[..., :ci]), ci), dz, 8, 4)[0],
                                   (cols.T @ dz.reshape(-1, 32)).reshape(8, 8, ci, 32), rtol=1e-12, atol=1e-10)


def test_bf16_split_matches_the_planes_arithmetic():
    """bf16_split is split3: each plane the round-to-nearest BF16 of the residual, the 3-plane sum exact for fp32."""
    x = np.random.default_rng(0).standard_normal(100000).astype(np.float32) * np.float32(3.7)
    p = bf16_split(x, 3)
    assert np.array_equal(bf(p[0]) + bf(p[1]) + bf(p[2]), x.astype(np.float64))
    r1 = x.astype(np.float64) - bf(p[0])
    assert np.all(np.abs(r1) <= 2.0 ** -8 * np.abs(x))
    assert np.all(np.abs(r1 - bf(p[1])) <= 2.0 ** -16 * np.abs(x))


# ================================================================================================ GPU
def _build(case):
    if case.params == "trained":
        cfg, params, vn = load_case("sac_depth")
    else:
        cfg, vn = case.cfg, vecnorm_for(case.ci)
        params = R.init_params(cfg, seed=case.seed)
        rng = np.random.default_rng(case.seed)
        for k in [k for k in params if k.endswith("/b") or k.endswith("/bias")]:     # non-zero biases (fresh init has zeros)
            params[k] = (rng.standard_normal(params[k].shape) * 0.05).astype(np.float32)
    if case.params == "coherent":
        for n, scope in enumerate(SCOPES):
            params[f"{scope}/cnn_fc1/w"] = coherent_fc1_weights(params[f"{scope}/cnn_fc1/w"].shape, n)
    return cfg, params, vn


NS = 256          # replay transitions behind the sampled case


def _sampled_step(L, vn, case):
    """Fills the replay (colour planes integers 0 .. 255, stored as bytes), runs one graph-path step and returns the stored
    transitions at the slots it drew, as the gather read them."""
    tr = synth.make_transitions(NS, vn["obs_mean"], vn["obs_var"], seed=case.seed, n_act=case.A)
    rng = np.random.default_rng(case.seed)
    for k in ("obs", "next_obs"):
        tr[k] = np.array(tr[k], np.float32)
        tr[k][..., list(U8_PLANES)] = rng.integers(0, 256, tr[k].shape[:3] + (len(U8_PLANES),)).astype(np.float32)
    L.replay_add(tr["obs"], tr["act"], tr["rew"], tr["next_obs"], tr["done"])
    L.step(1, lr=3e-4)
    rows = [L.replay_get(int(s)) for s in L.last_batch()["indices"]]
    return {k: np.stack([np.asarray(r[k], np.float32).reshape(np.shape(tr[k][0])) for r in rows]) for k in ("obs", "next_obs", "act")}


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_contractions_match_float64_of_their_inputs(case, monkeypatch):
    for k, v in case.env:
        monkeypatch.setenv(k, v)
    cfg, params, vn = _build(case)
    B, ci, A, H = case.B, case.ci, case.A, case.H
    kw = dict(buffer_size=NS, u8_planes=U8_PLANES) if case.sampled else dict(buffer_size=max(64, B))
    L = make_learner(cfg, vn, B, params, precision=1, hidden=H, **kw)
    try:
        if case.sampled:
            raw = _sampled_step(L, vn, case)
        else:
            raw, _, eps = make_batch(vn, B, n_act=A)
            L.step_explicit(raw["obs"], raw["act"], raw["rew"], raw["next_obs"], raw["done"], eps, lr=3e-4, apply_update=False)
        names =["S/obs", "S/next_obs", "dz0pi", "dz0v", "dZ1", "W1T/online", "W1T/target", "z0/pi", "z0/target", "z0v",
                 "dz0_pi", "dz0_v3"]
        names += [f"{t}/{n}" for t in ("H1", "H2", "H3", "F", "W2T", "W3T", "WfT", "K0T", "F32") for n in NETS]
        names += [f"{t}/{n}" for t in ("dZ4", "dZ3", "dZ2", "W2n", "W3n", "Wfn", "K0n") for n in NETS[:2]]
        names += [f"{t}/{q}" for t in ("a0", "dz1") for q, _ in HEADS]
        T = {n: read(L, n) for n in names}
        G = L.get_gradients()
        G = {k: np.asarray(v, np.float64) for k, v in G.items()}
    finally:
        L.close()
    rep = Report(case.name)
    check_weight_planes(rep, T, params, ci, A, H)
    check_gather(rep, T, raw["obs"], raw["next_obs"], raw["act"], vn, ci, B, norm_obs=bool(vn.get("norm_obs", True)))
    gam = problem_gammas(B, ci, *case.splits)
    check_step(rep, T, G, {k: np.asarray(v) for k, v in params.items()}, B, ci, A, H, gam)
    check_heads_wgrad(rep, T, G, B, A, H)
    rep.finish()


@pytest.mark.gpu
def test_debug_tensor_refuses_bad_requests():
    cfg, params, vn = load_case("sac_depth")
    L = make_learner(cfg, vn, 4, params, buffer_size=64, precision=1)
    try:
        buf = np.empty(4 * 512 * 2, np.uint16)
        vp = buf.ctypes.data_as(C.c_void_p)
        assert L.lib.b2g_debug_tensor(L.h, b"dZ4/pi", 0, vp, 4 * 512 * 2) == 0
        assert L.lib.b2g_debug_tensor(L.h, b"no/such", 0, vp, 4 * 512 * 2) == _lib.B2G_EINVAL
        assert L.lib.b2g_debug_tensor(L.h, b"dZ4/pi", 2, vp, 4 * 512 * 2) == _lib.B2G_EINVAL        # 2 planes
        assert L.lib.b2g_debug_tensor(L.h, b"dZ4/pi", 0, vp, 4 * 512 * 2 - 2) == _lib.B2G_EINVAL
        assert L.lib.b2g_debug_tensor(L.h, b"dZ4/target", 0, vp, 4 * 512 * 2) == _lib.B2G_EINVAL    # no target backward
        for q in (b"z0/vf", b"z0/qf1", b"z0/qf2"):                       # engine v2 writes them into z0v
            assert L.lib.b2g_debug_tensor(L.h, q, 0, vp, 4 * 64 * 4) == _lib.B2G_ESTATE
        assert L.lib.b2g_debug_tensor(L.h, b"rew_n", 0, vp, 4 * 4 - 4) == _lib.B2G_EINVAL          # [B] fp32
        assert L.lib.b2g_debug_tensor(L.h, b"done_n", 1, vp, 4 * 4) == _lib.B2G_EINVAL             # one plane
    finally:
        L.close()
    L0 = make_learner(cfg, vn, 4, params, buffer_size=64, precision=0)
    try:
        assert L0.lib.b2g_debug_tensor(L0.h, b"dZ4/pi", 0, vp, 4 * 512 * 2) == _lib.B2G_ESTATE
        n = C.c_int64()
        assert L0.lib.b2g_debug_tensor_info(L0.h, b"F32/pi", C.byref(n), None, None) == 0
        for q in (b"z0/vf", b"z0/qf1", b"z0/qf2"):                       # separate buffers without engine v2
            assert L0.lib.b2g_debug_tensor_info(L0.h, q, C.byref(n), None, None) == 0 and n.value == 4 * 64
    finally:
        L0.close()


# ------------------------------------------------------------------------------------------------ gg_tc (b2g_debug_gemm)
GG_M, GG_N = (1, 127, 128, 129, 300), (1, 16, 17, 33, 64, 65, 130)


@pytest.mark.gpu
@pytest.mark.parametrize("x3", [1, 0])
@pytest.mark.parametrize("split_k", [1, 3, 8])
@pytest.mark.parametrize("K", [8, 72, 1000, 4096])
def test_gg_tc_gemm_elementwise(K, split_k, x3):
    lib = _lib.load()
    fp = C.POINTER(C.c_float)
    rng = np.random.default_rng(K * 10 + split_k + 100 * x3)
    rep = Report(f"gg_tc K={K} split_k={split_k} x3={x3}")
    g_same, g_exact = gg_gammas(K, split_k, x3)
    for M in GG_M:
        for Nn in GG_N:
            A = rng.standard_normal((M, K)).astype(np.float32)
            Bm = rng.standard_normal((Nn, K)).astype(np.float32)
            out = np.zeros((M, Nn), np.float32)
            _lib.check(lib.b2g_debug_gemm(M, Nn, K, A.ctypes.data_as(fp), Bm.ctypes.data_as(fp), out.ctypes.data_as(fp), x3,
                                          split_k))
            ah, al = (bf(p) for p in bf16_split(A, 2))
            bh, bl = (bf(p) for p in bf16_split(Bm, 2))
            same = ah @ bh.T + ((ah @ bl.T + al @ bh.T) if x3 else 0.0)
            mag = np.abs(A).astype(np.float64) @ np.abs(Bm).astype(np.float64).T
            rep.hold(f"same split M={M} N={Nn}", out, same, mag, g_same)
            rep.hold(f"exact M={M} N={Nn}", out, A.astype(np.float64) @ Bm.astype(np.float64).T, mag, g_exact)
    rep.finish()
