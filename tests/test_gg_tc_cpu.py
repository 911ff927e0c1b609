"""b2g_debug_gg_tc without a device: every refusal of its contract checks (they run before any CUDA call), and the SAC table
formulas tests/gg_tc_ref.py restates, contracted on the CPU, against torch's float64 convolutions, their weight and input
gradients, and linear layers.  The second part shows that tests/test_gpu_gg_tc.py asks the engine the questions SAC asks."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from b200grasp import _lib
from tests import gg_tc_ref as T
from tests.gg_tc_ref import GG, iota

F32, F64 = np.float32, np.float64


# ------------------------------------------------------------------ refusals of b2g_debug_gg_tc
def _fp32(flags=GG["A_RVEC"] | GG["EPI_BIAS_RELU"], M=70, N=12, R=21, **kw):
    """A valid fp32 problem: A rows of 24 (r-contiguous) or columns of 72 per r (m-contiguous), B rows of 12 per r
    (n-contiguous) or 24 per n (r-contiguous)."""
    L = T.Launch(1)
    rng = np.random.default_rng(0)
    ar = flags & GG["A_RVEC"]
    br = flags & GG["B_RVEC"]
    A = rng.standard_normal(M * 24 if ar else R * 72).astype(F32)
    B = rng.standard_normal(N * 24 if br else R * 12).astype(F32)
    aM, aR = (iota(M, 24), iota(R)) if ar else (iota(M), iota(R, 72))
    bR, bN = (iota(R), iota(N, 24)) if br else (iota(R, 12), iota(N))
    bias = rng.standard_normal(N).astype(F32) if flags & GG["EPI_BIAS_RELU"] else None
    L.add(M, N, R, flags, A, aM, aR, B, bR, bN, iota(M, 12), iota(N), bias=bias, **kw)
    return L


def _conv1(ci=3, wgrad=False):
    """conv1 of a 1 x 16 x 16 x ci image on the plane kernel: the forward (K-major, ROWLANES, ALIGN4 at odd ci) or the weight
    gradient (MN-major)."""
    L = T.Launch(1)
    rng = np.random.default_rng(1)
    c = T.conv_geometry(16, 16, ci)[0]
    rowoff, koff, crow = T.conv_fwd_tables(1, c)
    x = rng.random(16 * 16 * ci).astype(F32)
    R = 64 * ci
    odd = GG["A_ALIGN4"] if ci & 1 else 0
    if wgrad:
        dz = rng.standard_normal(len(rowoff) * 32).astype(F32)
        L.add(R, 32, len(rowoff), GG["PLANES"] | GG["MN_MAJOR"] | GG["A_ROWLANES"] | GG["EPI_ATOMIC"] | odd, x, koff, rowoff, dz,
              iota(len(rowoff), 32), iota(32), iota(R, 32), iota(32), splitR=2)
    else:
        WT = rng.standard_normal(32 * R).astype(F32)
        L.add(len(rowoff), 32, R, GG["PLANES"] | GG["A_RVEC"] | GG["B_RVEC"] | GG["EPI_BIAS_RELU"] | GG["A_ROWLANES"] | odd, x,
              rowoff, koff, WT, iota(R, 32), iota(32), crow, iota(32), bR_p=iota(R), bN_p=iota(32, R),
              bias=rng.standard_normal(32).astype(F32), c_planes=True)
    return L


def _rc(L, edit=None, x3=None, n=None):
    st = L.structs()
    f32, u16, tabs = L.arenas()
    if edit:
        edit(st[0], tabs)
    if n is not None:
        st = (_lib.GgTcProblem * n)(*([st[0]] * n))
    rc, _ = L.run((f32, u16, tabs), st, x3=x3)
    return rc, _lib.load().b2g_last_error().decode()


def _refused(L, edit, words, **kw):
    rc, msg = _rc(L, edit, **kw)
    assert rc == _lib.B2G_EINVAL, (rc, msg)
    assert words in msg, msg


def _passes(L, edit=None):
    rc, msg = _rc(L, edit)
    assert rc in (0, _lib.B2G_ECUDA), msg                     # ECUDA: refused only for want of a GPU


@pytest.mark.parametrize("make", [lambda: _fp32(), lambda: _fp32(GG["COLSUM"], colsum=True),
                                  lambda: _fp32(GG["A_RVEC"] | GG["B_RVEC"] | GG["EPI_MASK"], mask=np.ones(70 * 12, F32)),
                                  lambda: _fp32(GG["B_RVEC"]), lambda: _conv1(3), lambda: _conv1(4), lambda: _conv1(1, True)])
def test_valid_problems_pass_the_checks(make):
    _passes(make())


def test_refuses_launch_arguments():
    L = _fp32()
    _refused(L, None, "x3 must be 0", x3=2)
    _refused(L, None, "1 to 16 problems", n=17)
    _refused(L, None, "1 to 16 problems", n=0)


def test_refuses_problems_of_different_kernels():
    for second in (_fp32(GG["A_RVEC"] | GG["B_RVEC"]), _conv1(3)):
        L = _fp32()
        L.problems.append(second.problems[0])           # its offsets point into the other launch's arenas: refused before use
        rc, msg = _rc(L)
        assert rc == _lib.B2G_EINVAL and "another gg_tc kernel" in msg, msg
    # the plane kernel runs K-major and MN-major problems whatever their GG_A_RVEC / GG_B_RVEC
    fwd = _conv1(3)
    st = (_lib.GgTcProblem * 2)(fwd.structs()[0], fwd.structs()[0])
    st[1].flags &= ~(GG["A_RVEC"] | GG["B_RVEC"])
    rc, _ = fwd.run(None, st)
    assert rc in (0, _lib.B2G_ECUDA), _lib.load().b2g_last_error()


@pytest.mark.parametrize("flag", ["EPI_BIAS", "EPI_SCALE", "A_SCALAR", "EPI_BIAS_LRELU", "EPI_LRELU_GRAD", "EPI_BIAS_TANH",
                                  "EPI_TANH_GRAD", 1 << 8])
def test_refuses_flags_gg_tc_does_not_implement(flag):
    f = GG[flag] if isinstance(flag, str) else flag
    _refused(_fp32(), lambda s, t: setattr(s, "flags", s.flags | f), "not implemented by gg_tc")


@pytest.mark.parametrize("flag", ["MN_MAJOR", "A_ROWLANES", "A_ALIGN4"])
def test_refuses_plane_producer_modes_without_planes(flag):
    _refused(_fp32(), lambda s, t: setattr(s, "flags", s.flags | GG[flag]), "need GG_PLANES")


def test_refuses_splits_outputs_and_column_sums():
    L = _fp32()
    _refused(L, lambda s, t: setattr(s, "splitR", 2), "splitR > 1 needs GG_EPI_ATOMIC")
    _refused(L, lambda s, t: setattr(s, "splitR", 22), "splitR must be in 1..R")
    _refused(L, lambda s, t: setattr(s, "R", 0), "M, N and R must be >= 1")
    _refused(L, lambda s, t: setattr(s, "C_hi", 0), "C_hi and C_lo go together")
    La = _fp32(GG["A_RVEC"] | GG["EPI_ATOMIC"])
    _refused(La, lambda s, t: (setattr(s, "C_hi", 0), setattr(s, "C_lo", 0)), "under GG_EPI_ATOMIC")
    Lc = _fp32(GG["A_RVEC"] | GG["B_RVEC"] | GG["COLSUM"], colsum=True)
    _refused(Lc, None, "cannot take GG_B_RVEC or GG_PLANES")
    _refused(_conv1(1, True), lambda s, t: (setattr(s, "flags", s.flags | GG["COLSUM"]), setattr(s, "colsum", 0)),
             "cannot take GG_B_RVEC or GG_PLANES")
    _refused(L, lambda s, t: setattr(s, "bias", -1), "needs bias")
    _refused(L, lambda s, t: setattr(s, "flags", s.flags | GG["EPI_MASK"]), "needs mask")
    _refused(L, lambda s, t: setattr(s, "colsum", 0), "colsum goes with GG_COLSUM")


def test_refuses_operands_of_the_wrong_kind():
    _refused(_fp32(), lambda s, t: setattr(s, "A_hi", 0), "fp32 problems read A and B, not planes")
    _refused(_fp32(), lambda s, t: setattr(s, "B", -1), "fp32 problems read A and B")
    _refused(_conv1(3), lambda s, t: setattr(s, "A", 0), "GG_PLANES reads A_hi, A_lo, B_hi and B_lo")
    _refused(_conv1(3), lambda s, t: setattr(s, "B_lo", -1), "GG_PLANES reads A_hi, A_lo, B_hi and B_lo")
    _refused(_fp32(), lambda s, t: setattr(s, "bR_p", s.bR), "K-major plane problems only")
    _refused(_conv1(1, True), lambda s, t: setattr(s, "bN_p", s.bN), "K-major plane problems only")
    _refused(_fp32(), lambda s, t: setattr(s, "cN", -1), "cN is required")


@pytest.mark.parametrize("what", ["aM", "aR", "bR", "bN", "cM", "cN"])
def test_refuses_a_table_entry_out_of_range(what):
    def edit(s, tabs):
        tabs[getattr(s, what) + 1] = 10 ** 7
    _refused(_fp32(), edit, "outside its arena")


def test_refuses_plane_reads_outside_the_arena():
    # K-major: the plane B through bR_p / bN_p; a plane base past the end
    _refused(_conv1(3), lambda s, t: t.__setitem__(s.bN_p + 31, 10 ** 6), "B_hi / B_lo[bR + bN] reaches outside")
    L = _conv1(3)
    n16 = len(L.arenas()[1])
    _refused(L, lambda s, t: setattr(s, "A_lo", n16 - 8), "A_hi / A_lo[aM + aR] reaches outside")
    # MN-major: 8 elements from the start of every 8-group of aM, even past M
    Lw = _conv1(1, True)
    st, (f32, u16, tabs) = Lw.structs(), Lw.arenas()
    p = Lw.problems[0]
    top = int(p.aM.v.max() + p.aR.v.max())
    st[0].A_lo = len(u16) - top - 2                        # room for aM[m] + aR[r], not for the 8-group's tail
    if st[0].A_lo % 4 == 0:
        st[0].A_lo -= 1
    rc, _ = Lw.run((f32, u16, tabs), st)
    assert rc == _lib.B2G_EINVAL, _lib.load().b2g_last_error()


def test_refuses_r_tables_the_k_major_producers_read_past_tabs():
    L = _conv1(3)
    st, (f32, u16, tabs) = L.structs(), L.arenas()
    R = 129                                               # a third chunk with one valid row: aR is read up to index 184
    tabs2 = np.concatenate([tabs, tabs[st[0].aR:st[0].aR + R]]).astype(np.int32)
    st[0].aR, st[0].R = len(tabs), R
    rc, _ = L.run((f32, u16, tabs2), st)
    msg = _lib.load().b2g_last_error().decode()
    assert rc == _lib.B2G_EINVAL and "aR runs past the end of tabs" in msg, msg


def test_refuses_broken_groups_and_misaligned_addresses():
    # fp32: r-direction 4-groups, m- / n-direction 4-groups, their 16-byte alignment, int4 table loads
    _refused(_fp32(), lambda s, t: t.__setitem__(s.aR + 5, 6), "GG_A_RVEC: aR is not contiguous")
    _refused(_fp32(), lambda s, t: setattr(s, "A", s.A + 2), "not 16-byte aligned")
    _refused(_fp32(GG["COLSUM"], colsum=True), lambda s, t: t.__setitem__(s.aM + 1, 100), "m-direction A: aM is not contiguous")
    _refused(_fp32(GG["COLSUM"], colsum=True), lambda s, t: t.__setitem__(s.bN + 2, 7), "n-direction B: bN is not contiguous")
    _refused(_fp32(GG["COLSUM"], colsum=True), lambda s, t: setattr(s, "aR", s.aR + 1), "aR must start 16-byte aligned")
    _refused(_fp32(GG["A_RVEC"]), lambda s, t: setattr(s, "bR", s.bR + 1), "bR must start 16-byte aligned")
    # r-vector tables are read one entry at a time: any start will do (a copy of aR in its zero padding, at 1 mod 4)
    _passes(_fp32(GG["A_RVEC"] | GG["B_RVEC"]), lambda s, t: (t.__setitem__(slice(s.aR + 25, s.aR + 46), iota(21)),
                                                            setattr(s, "aR", s.aR + 25)))
    # planes: 8-groups of 16 bytes (8-byte halves of A under GG_A_ALIGN4)
    _refused(_conv1(4), lambda s, t: t.__setitem__(s.aR + 9, 0), "K-major A: aR is not contiguous in the 8-group at 8")
    _refused(_conv1(4), lambda s, t: setattr(s, "A_hi", s.A_hi + 4), "K-major A: the 8-groups of aR are not 16-byte aligned")
    _passes(_conv1(3), lambda s, t: setattr(s, "A_hi", s.A_hi + 4))
    _refused(_conv1(3), lambda s, t: setattr(s, "A_hi", s.A_hi + 2), "not 8-byte aligned")
    _refused(_conv1(3), lambda s, t: setattr(s, "B_lo", s.B_lo + 4), "K-major B: the 8-groups of bR_p are not 16-byte aligned")
    _refused(_conv1(1, True), lambda s, t: t.__setitem__(s.aM + 3, 0), "MN-major A: aM is not contiguous")
    _refused(_conv1(1, True), lambda s, t: setattr(s, "B_hi", s.B_hi + 4), "MN-major B: the 8-groups of bN are not 16-byte aligned")
    # vector epilogue stores
    _refused(_fp32(), lambda s, t: setattr(s, "C", s.C + 1), "C, mask, C_hi and C_lo must start")
    _refused(_conv1(3), lambda s, t: setattr(s, "C_lo", s.C_lo + 2), "C, mask, C_hi and C_lo must start")
    Lm = _fp32(GG["A_RVEC"] | GG["B_RVEC"] | GG["EPI_MASK"], mask=np.ones(70 * 12 + 4, F32))
    _refused(Lm, lambda s, t: setattr(s, "mask", s.mask + 1), "C, mask, C_hi and C_lo must start")


# ------------------------------------------------------------------ the tables against torch
def contract(A, aM, aR, B, bR, bN):
    return np.asarray(A, F64)[aM[:, None] + aR[None, :]] @ np.asarray(B, F64)[bR[:, None] + bN[None, :]]


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x, F64))


def nchw(x):
    return _t(x).permute(0, 3, 1, 2)


def oihw(w):
    return _t(w).permute(3, 2, 0, 1)


@pytest.mark.parametrize("hw,ci", [((64, 64), 1), ((64, 64), 3), ((72, 96), 5)])
def test_conv_tables_against_torch(hw, ci):
    """Forward (rowoff / koff, and the transposed weight planes through bR_p / bN_p), weight gradients (koff as m, rowoff
    as r, dZ rows of the zero-bordered maps) and input gradients (conv3's dgrad over dZ3p, conv2's four parity classes over
    dZ2p, cnn_fc1's dgrad into dZ3p) of every layer, for B = 2."""
    rng = np.random.default_rng(ci)
    B = 2
    g = T.conv_geometry(*hw, ci)
    xs = [rng.standard_normal((B, c[0], c[1], c[2])) for c in g]
    ws = [rng.standard_normal((c[3], c[3], c[2], c[7])) for c in g]
    for c, x, w in zip(g, xs, ws):
        Hi, Wi, Ci, k, s, Ho, Wo, Co = c
        rowoff, koff, crow = T.conv_fwd_tables(B, c)
        R = k * k * Ci
        WT = w.reshape(R, Co).T.ravel()
        y = contract(x.ravel(), rowoff, koff, WT, iota(R), iota(Co, R))
        ref = Fn.conv2d(nchw(x), oihw(w), stride=s).permute(0, 2, 3, 1).numpy()
        assert np.allclose(y.reshape(ref.shape), ref, rtol=1e-12, atol=1e-10)
        # the output rows crow / cN are the NHWC layout
        assert np.array_equal(crow[:, None] + iota(Co)[None, :], np.arange(B * Ho * Wo * Co).reshape(-1, Co))
    (_, _, _, _, _, H1, W1, _), (_, _, _, _, _, H2, W2, _), (_, _, _, _, _, H3, W3, _) = g
    P2h, P2w, P3h, P3w = H2 + 3, W2 + 3, H3 + 4, W3 + 4
    dz = [rng.standard_normal((B, c[5], c[6], c[7])) for c in g]
    dz2p = np.zeros((B, P2h, P2w, 64)); dz2p[:, 1:1 + H2, 1:1 + W2] = dz[1]
    dz3p = np.zeros((B, P3h, P3w, 64)); dz3p[:, 2:2 + H3, 2:2 + W3] = dz[2]
    rows = [iota(B * H1 * W1, 32), T.bordered_rows(B, H2, W2, P2h, P2w, 1), T.bordered_rows(B, H3, W3, P3h, P3w, 2)]
    maps = [dz[0], dz2p, dz3p]
    for l, c in enumerate(g):
        Hi, Wi, Ci, k, s, Ho, Wo, Co = c
        rowoff, koff, _ = T.conv_fwd_tables(B, c)
        dw = contract(xs[l].ravel(), koff, rowoff, maps[l].ravel(), rows[l], iota(Co))
        ref = torch.nn.grad.conv2d_weight(nchw(xs[l]), (Co, Ci, k, k), nchw(dz[l]), stride=s).permute(2, 3, 1, 0).numpy()
        assert np.allclose(dw.reshape(ref.shape), ref, rtol=1e-12, atol=1e-10), l

    def dgrad(l):
        x = nchw(xs[l]).requires_grad_(True)
        Fn.conv2d(x, oihw(ws[l]), stride=g[l][4]).backward(nchw(dz[l]))
        return x.grad.permute(0, 2, 3, 1).numpy()
    # conv3: dZ2p rows (bordered), the interior is the input gradient, the border is never addressed
    am, ar, br, bn, cm = T.conv3_dgrad_tables(B, H2, W2, H3, W3)
    out = np.zeros(B * P2h * P2w * 64)
    out[cm[:, None] + iota(64)[None, :]] = contract(dz3p.ravel(), am, ar, ws[2].ravel(), br, bn)
    out = out.reshape(B, P2h, P2w, 64)
    assert np.allclose(out[:, 1:1 + H2, 1:1 + W2], dgrad(2), rtol=1e-12, atol=1e-10)
    assert not out[:, 0].any() and not out[:, 1 + H2:].any() and not out[:, :, 0].any() and not out[:, :, 1 + W2:].any()
    # conv2: the four parity classes tile dZ1 exactly once
    out, hit = np.zeros(B * H1 * W1 * 32), np.zeros(B * H1 * W1 * 32, int)
    for py in range(2):
        for px in range(2):
            am, ar, br, bn, cm = T.conv2_dgrad_tables(B, H1, W1, H2, W2, py, px)
            idx = cm[:, None] + iota(32)[None, :]
            out[idx] = contract(dz2p.ravel(), am, ar, ws[1].ravel(), br, bn)
            hit[idx.ravel()] += 1
    assert np.all(hit == 1)
    assert np.allclose(out.reshape(B, H1, W1, 32), dgrad(1), rtol=1e-12, atol=1e-10)
    # cnn_fc1 (conv3 output rows of 64 H3 W3) dgrad into dZ3p, and its forward / weight gradient
    K = 64 * H3 * W3
    h3 = rng.standard_normal((B, K))
    Wf, dZ4 = rng.standard_normal((K, 512)), rng.standard_normal((B, 512))
    rowP3, cN3p = T.fc1_dgrad_tables(B, H3, W3)
    out = np.zeros(B * P3h * P3w * 64)
    out[rowP3[:, None] + cN3p[None, :]] = contract(dZ4.ravel(), iota(B, 512), iota(512), Wf.ravel(), iota(512), iota(K, 512))
    out = out.reshape(B, P3h, P3w, 64)
    assert np.allclose(out[:, 2:2 + H3, 2:2 + W3].reshape(B, K), dZ4 @ Wf.T, rtol=1e-12, atol=1e-10)
    assert np.abs(out).sum() == pytest.approx(np.abs(dZ4 @ Wf.T).sum())
    x = _t(h3).requires_grad_(True)
    w = _t(Wf).requires_grad_(True)
    y = Fn.linear(x, w.T)
    assert np.allclose(contract(h3.ravel(), iota(B, K), iota(K), Wf.T.ravel(), iota(K), iota(512, K)), y.detach().numpy())
    y.backward(_t(dZ4))
    assert np.allclose(contract(h3.ravel(), iota(K), iota(B, K), dZ4.ravel(), iota(B, 512), iota(512)), w.grad.numpy())


def test_head_tables_against_torch():
    """heads_fc0 (F rows of FS through rowFS / iFS, kernels through kH / iH), heads_wgrad (m-direction F, dz0 columns of the
    [B][3H] block) and heads_dgrad (the values net's three fc0 kernels through brv)."""
    rng = np.random.default_rng(9)
    B, fd, A, H = 5, 516, 3, 64
    FS = T.r4(fd + A + 3)
    F = rng.standard_normal((B, FS))
    K0 = [rng.standard_normal((fd + (A if q >= 2 else 0), H)) for q in range(4)]
    dz0v = rng.standard_normal((B, 3 * H))
    for q in range(4):
        R = K0[q].shape[0]
        y = contract(F.ravel(), iota(B, FS), iota(R), K0[q].ravel(), iota(R, H), iota(H))
        assert np.allclose(y, Fn.linear(_t(F[:, :R]), _t(K0[q]).T).numpy())
    for q in range(3):
        R = K0[q + 1].shape[0]
        x = _t(F[:, :R]).requires_grad_(True)
        w = _t(K0[q + 1]).requires_grad_(True)
        Fn.linear(x, w.T).backward(_t(dz0v[:, q * H:(q + 1) * H]))
        dw = contract(F.ravel(), iota(R), iota(B, FS), dz0v.ravel(), iota(B, 3 * H), iota(H, 1, q * H))
        assert np.allclose(dw, w.grad.numpy())
    P = np.zeros(3 * (fd * H + 40) + 8)
    offs = [4 + q * (fd * H + 40) for q in range(3)]
    for q in range(3):
        P[offs[q]:offs[q] + fd * H] = K0[q + 1][:fd].ravel()
    br = np.concatenate([o + iota(H) for o in offs])
    dF = contract(dz0v.ravel(), iota(B, 3 * H), iota(3 * H), P, br, iota(512, H))
    want = sum(dz0v[:, q * H:(q + 1) * H] @ K0[q + 1][:512].T for q in range(3))
    assert np.allclose(dF, want)
