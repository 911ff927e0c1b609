"""The wgmma gather-GEMM engine (csrc/gg_tc.cu) held element by element, through b2g_debug_gg_tc, in all five of its kernels.

Each case is one grouped launch built with the SAC handle's own table formulas (sac.cu build_groups, restated in
tests/gg_tc_ref.py) and run at x3 = 1 and x3 = 0.  For every output:
  1. against the exact split: a float64 contraction of the BF16 operands the engine multiplies (hi*hi + hi*lo + lo*hi, or hi*hi),
     within the accumulation-only bar gg_gammas(R, splitR, x3)[0] * sum|a||b| (+ one fp32 rounding for the bias) over the
     element's own reduction; ReLU is 1-Lipschitz, so the bar holds across the kink;
  2. against the exact float64 contraction of the fp32 sources, with the split's own error added to the bar;
  3. bit for bit: zeros wherever the mask is <= 0; C_hi = RN_bf16(o), C_lo = RN_bf16(o - hi) of the engine's own fp32 result o;
     every arena element no problem writes (inputs, slack, NaN-payload sentinels around every C, C_hi, C_lo and colsum) is
     unchanged; a second launch gives bit-identical outputs for every problem without GG_EPI_ATOMIC;
  4. column sums (GG_COLSUM) within gamma_(R + splitR) sum|B| of their float64 sums, added once whatever tiles_m is.
Run with -s to see the worst err/bar of each problem.
"""
import numpy as np
import pytest
import torch

from tests import gg_tc_ref as T
from tests.gg_simt_ref import bf16_rn, bf16_to_f32, gamma
from tests.gg_tc_ref import BK, BM, BN, GG, U32, Report, cdiv, gg_gammas, iota, r4

pytestmark = pytest.mark.gpu
F32, F64 = np.float32, np.float64
X3 = pytest.mark.parametrize("x3", [1, 0])


def normal(rng, n, scale=1.0):
    return (rng.standard_normal(n) * scale).astype(F32)


def relu_like(rng, n, zeros=0.4):
    """ReLU outputs (and masks): non-negative with exact zeros."""
    v = np.abs(normal(rng, n))
    v[rng.random(n) < zeros] = 0
    return v


# ------------------------------------------------------------------ the checker
def check(L, case):
    arenas = L.arenas()
    rc, (f32, u16) = L.run(arenas)
    assert rc == 0, T._lib.load().b2g_last_error()
    rc2, (f32b, u16b) = L.run(arenas)
    assert rc2 == 0, T._lib.load().b2g_last_error()
    rep = Report(f"{case} x3={L.x3}")
    written = {"f32": np.zeros(len(f32), bool), "u16": np.zeros(len(u16), bool)}
    for i, p in enumerate(L.problems):
        tag = f"p{i} M{p.M} N{p.N} R{p.R} s{p.splitR}"
        Am, Bm = T.gathered(p)
        ah, al = (bf16_to_f32(x).astype(F64) for x in T.split2(Am))
        bh, bl = (bf16_to_f32(x).astype(F64) for x in T.split2(Bm))
        same = ah @ bh + ((ah @ bl + al @ bh) if L.x3 else 0.0)
        A64, B64 = Am.astype(F64), Bm.astype(F64)
        exact = A64 @ B64
        mag = np.abs(A64) @ np.abs(B64)
        g_same, g_exact = gg_gammas(p.R, p.splitR, L.x3)
        if p.bias is not None:
            b = p.bias.v[:p.N].astype(F64)[None, :]
            same, exact, mag = np.maximum(same + b, 0), np.maximum(exact + b, 0), mag + np.abs(b)
            g_same, g_exact = g_same + U32, g_exact + U32
        if p.mask is not None:
            keep = T.mask_of(p) > 0
            same, exact = np.where(keep, same, 0), np.where(keep, exact, 0)
            mag = np.where(keep, mag, 0)                       # masked outputs are held to exact zeros
        idx = p.oC + T.out_index(p)
        got = f32[idx]
        written["f32"][idx.ravel()] = True
        rep.hold(f"{tag} same split", got, same, mag, g_same)
        rep.hold(f"{tag} float64", got, exact, mag, g_exact)
        if p.oC_hi >= 0:
            hi = bf16_rn(got)
            lo = bf16_rn(got - bf16_to_f32(hi))
            hidx, lidx = p.oC_hi + T.out_index(p), p.oC_lo + T.out_index(p)
            written["u16"][hidx.ravel()] = True
            written["u16"][lidx.ravel()] = True
            rep.exact(f"{tag} C_hi", u16[hidx], hi)
            rep.exact(f"{tag} C_lo", u16[lidx], lo)
        if p.colsum is not None:
            cs = f32[p.colsum.off:p.colsum.off + p.N]
            written["f32"][p.colsum.off:p.colsum.off + p.N] = True
            rep.hold(f"{tag} colsum", cs, B64.sum(0), np.abs(B64).sum(0), gamma(p.R + p.splitR, U32))
        if not p.flags & GG["EPI_ATOMIC"]:
            rep.exact(f"{tag} rerun", got.view(np.uint32), f32b[idx].view(np.uint32))
            if p.oC_hi >= 0:
                rep.exact(f"{tag} rerun C_hi / C_lo", np.stack([u16[hidx], u16[lidx]]), np.stack([u16b[hidx], u16b[lidx]]))
    for name, before, after in (("f32", arenas[0].view(np.uint32), f32.view(np.uint32)), ("u16", arenas[1], u16)):
        keep = ~written[name]
        rep.exact(f"untouched {name}", after[keep], before[keep])
    rep.finish()


def tc_split(M, N, R, num_sms=132):
    """finalize_group's split-R for a GG_EPI_ATOMIC problem on the wgmma engine."""
    tiles = cdiv(M, BM) * cdiv(N, BN)
    return min(max(1, num_sms // tiles), max(1, R // (2 * BK)))


# ------------------------------------------------------------------ MLP heads (fp32 operands)
def heads(L, rng, B, fd, A, H, flags, shared=True, atomic_split=False):
    """heads_fc0: F rows [B][FS] x fc0 kernels [R][H] -> z0 [B][H], R = fd (pi, vf) or fd + A (qf1, qf2).  shared: heads 0 and 1
    share one column table and one bias (one col_id), heads 2 and 3 have their own."""
    FS = r4(fd + A + 3)
    F = normal(rng, B * FS)
    cn = L.tab(iota(H))
    bias = L.f32(normal(rng, H, 0.5)) if flags & GG["EPI_BIAS_RELU"] else None
    for q in range(4):
        R = fd + A if q >= 2 else fd
        K0 = normal(rng, R * H, 1 / np.sqrt(R))
        own = not shared or q >= 2
        b = (normal(rng, H, 0.5) if own else bias) if bias is not None else None
        s = tc_split(B, H, R) if atomic_split else 1
        L.add(B, H, R, flags, F, iota(B, FS), iota(R), K0, iota(R, H), iota(H), iota(B, H), iota(H) if own else cn, bias=b, splitR=s)


@X3
@pytest.mark.parametrize("M", [1, 127, 128, 129, 1025])
def test_heads_fc0_forward(M, x3):
    """heads_fc0 at batch M: <true,false,false> with BIAS_RELU, two heads on one col_id; and the policy-inference form
    (act_heads_fc0: no epilogue)."""
    L = T.Launch(x3, seed=M)
    rng = np.random.default_rng(100 + M)
    heads(L, rng, M, 516, 3, 256, GG["A_RVEC"] | GG["EPI_BIAS_RELU"])
    FS, R, H = 524, 513, 64
    L.add(M, H, R, GG["A_RVEC"], normal(rng, M * FS), iota(M, FS), iota(R), normal(rng, R * H, 0.05), iota(R, H), iota(H),
          iota(M, H), iota(H))
    check(L, f"heads_fc0 M={M}")


@X3
def test_heads_fc0_training_split(x3):
    """The training step's heads_fc0: GG_EPI_ATOMIC with finalize_group's split-R, B = 256, H = 256."""
    L = T.Launch(x3, seed=7)
    heads(L, np.random.default_rng(107), 256, 516, 3, 256, GG["A_RVEC"] | GG["EPI_ATOMIC"], atomic_split=True)
    assert [p.splitR for p in L.problems] == [4, 4, 4, 4]
    check(L, "heads_fc0 split")


@X3
def test_heads_backward(x3):
    """heads_wgrad (<false,false,false>): COLSUM with split-R ATOMIC over 3 M tiles (the last split empty) and plain COLSUM;
    heads_dgrad (<true,true,false>): MASK by the feature rows, C_hi / C_lo."""
    rng = np.random.default_rng(200)
    B, fd, A, H = 300, 300, 3, 128
    FS = r4(fd + A + 3)
    F = relu_like(rng, B * FS)
    dz0v = normal(rng, B * 3 * H)
    L = T.Launch(x3, seed=20)
    for q, (M, splitR) in enumerate([(fd + A, 4), (fd, 1)]):
        # wgrad: dK0[j, h] = sum_b F[b, j] dz0[b, h]; A m-direction (iFS), r = b (rowFS); B = dz0 columns q H .. of [B][3H]
        assert splitR == 1 or T.cdiv(T.cdiv(B, splitR), BK) * BK * (splitR - 1) >= B      # one empty split
        L.add(M, H, B, GG["COLSUM"] | (GG["EPI_ATOMIC"] if splitR > 1 else 0), F, iota(M), iota(B, FS), dz0v, iota(B, 3 * H),
              iota(H, 1, q * H), iota(M, H), iota(H), splitR=splitR, colsum=True)
    check(L, "heads wgrad")
    L = T.Launch(x3, seed=21)
    fd = 516                                                           # CNN features: 512 cnn_fc1 columns, the actuator value
    FS = r4(fd + A + 3)
    F = relu_like(rng, B * FS)
    P = normal(rng, 3 * (fd * H + 40) + 8, 0.05)
    offs = [4 + q * (fd * H + 40) for q in range(3)]                   # the three value heads' fc0 kernels in the arena
    br = np.concatenate([o + iota(H) for o in offs])
    # dgrad: dZ4[b, j] = sum_r dz0v[b, r] K0[j, r]  (values net: r over vf | qf1 | qf2), masked by F > 0
    L.add(B, 512, 3 * H, GG["A_RVEC"] | GG["B_RVEC"] | GG["EPI_MASK"], dz0v, iota(B, 3 * H), iota(3 * H), P, br, iota(512, H),
          iota(B, 512), iota(512), kM=iota(B, FS), kN=iota(512), mask=F, c_planes=True)
    check(L, "heads dgrad")


@X3
def test_m_direction_a_with_r_direction_b(x3):
    """<false,true,false>: no SAC group selects it (an m-direction A with an r-direction B); a wgrad with B stored transposed,
    BIAS_RELU and a masked variant, and a split-R ATOMIC one."""
    rng = np.random.default_rng(300)
    L = T.Launch(x3, seed=30)
    for M, N, R, fl, s in [(130, 70, 200, GG["EPI_BIAS_RELU"], 1), (64, 33, 77, GG["EPI_MASK"], 1), (260, 64, 520, GG["EPI_ATOMIC"], 3)]:
        HS, RS = r4(M + 1), r4(R + 2)
        h = relu_like(rng, R * HS)
        dzT = normal(rng, N * RS)
        kw = {}
        if fl & GG["EPI_BIAS_RELU"]:
            kw["bias"] = normal(rng, N, 0.5)
        if fl & GG["EPI_MASK"]:
            kw["mask"] = relu_like(rng, M * r4(N))
        L.add(M, N, R, fl | GG["B_RVEC"], h, iota(M), iota(R, HS), dzT, iota(R), iota(N, RS), iota(M, r4(N)), iota(N), splitR=s, **kw)
    check(L, "m-direction A, r-direction B")


# ------------------------------------------------------------------ CNN (BF16 plane operands)
BATCH = 3


def conv_w(rng, R, Co):
    return normal(rng, R * Co, 1 / np.sqrt(R))


def add_conv_fwd(L, rng, c, x, bias_planes=True, rowlanes=False):
    """conv forward on the plane kernel: A = NHWC input planes (rowoff / koff), B = the transposed weight planes [Co][R]
    through bR_p / bN_p, C = NHWC output with C_hi / C_lo, BIAS_RELU."""
    Hi, Wi, Ci, k, s, Ho, Wo, Co = c
    rowoff, koff, crow = T.conv_fwd_tables(BATCH, c)
    R = k * k * Ci
    W = conv_w(rng, R, Co)
    WT = W.reshape(R, Co).T.ravel()
    fl = GG["PLANES"] | GG["A_RVEC"] | GG["B_RVEC"] | GG["EPI_BIAS_RELU"]
    if rowlanes:
        fl |= GG["A_ROWLANES"] | (GG["A_ALIGN4"] if Ci & 1 else 0)
    return L.add(len(rowoff), Co, R, fl, x, rowoff, koff, WT, iota(R, Co), iota(Co), crow, iota(Co), bR_p=iota(R), bN_p=iota(Co, R),
                 bias=normal(rng, Co, 0.3), c_planes=bias_planes)


@X3
@pytest.mark.parametrize("ci", [1, 3, 4, 5])
def test_conv1_forward(ci, x3):
    """conv1 forward: ROWLANES (and ALIGN4 for odd Ci), N = 32 (the mma_chunk<32> and 16-column epilogue path)."""
    rng = np.random.default_rng(400 + ci)
    L = T.Launch(x3, seed=40 + ci)
    c = T.conv_geometry(64, 64, ci)[0]
    add_conv_fwd(L, rng, c, rng.random(BATCH * 64 * 64 * ci).astype(F32), rowlanes=True)
    check(L, f"conv1 fwd ci={ci}")


@X3
def test_conv2_conv3_fc1_forward(x3):
    """conv2 and conv3 forward writing C_hi / C_lo, cnn_fc1 forward into the fp32 feature rows (N = 512: 8 column blocks)."""
    rng = np.random.default_rng(500)
    L = T.Launch(x3, seed=50)
    g = T.conv_geometry(64, 64, 1)
    for c in g[1:]:
        add_conv_fwd(L, rng, c, relu_like(rng, BATCH * c[0] * c[1] * c[2]))
    # cnn_fc1: h3 rows [B][1024] x Wf^T planes [512][1024] -> F rows [B][FS]
    FS = 576
    Wf = conv_w(rng, 1024, 512)
    L.add(BATCH, 512, 1024, GG["PLANES"] | GG["A_RVEC"] | GG["B_RVEC"] | GG["EPI_BIAS_RELU"], relu_like(rng, BATCH * 1024),
          iota(BATCH, 1024), iota(1024), Wf.reshape(1024, 512).T.ravel(), iota(1024, 512), iota(512), iota(BATCH, FS), iota(512),
          bR_p=iota(1024), bN_p=iota(512, 1024), bias=normal(rng, 512, 0.3))
    check(L, "conv2 conv3 fc1 fwd")


def _bordered(rng, B, h, w, pad_lo, pad_hi, C=64):
    m = np.zeros((B, h + pad_lo + pad_hi, w + pad_lo + pad_hi, C), F32)
    m[:, pad_lo:pad_lo + h, pad_lo:pad_lo + w] = rng.standard_normal((B, h, w, C))
    return m.ravel()


def conv_wgrad(L, rng, c, x, dz_rows, dz, ci_odd=False, conv1=False):
    """conv wgrad on the plane kernel, MN-major: A = input planes (koff as m, rowoff as r), B = output-gradient planes
    (dz_rows as r, n), C = dW [R][Co], split-R ATOMIC as finalize_group sizes it."""
    Hi, Wi, Ci, k, s, Ho, Wo, Co = c
    rowoff, koff, _ = T.conv_fwd_tables(BATCH, c)
    M = k * k * Ci
    fl = GG["PLANES"] | GG["MN_MAJOR"] | GG["EPI_ATOMIC"]
    if conv1:
        fl |= GG["A_ROWLANES"] | (GG["A_ALIGN4"] if ci_odd else 0)
    return L.add(M, Co, len(rowoff), fl, x, koff, rowoff, dz, dz_rows, iota(Co), iota(M, Co), iota(Co),
                 splitR=tc_split(M, Co, len(rowoff)))


@X3
@pytest.mark.parametrize("ci", [1, 3])
def test_cnn_backward(ci, x3):
    """conv1_wgrad (ROWLANES, ALIGN4 at odd Ci); conv2_bwd: both nets' wgrads and the 4 parity-class dgrads each (10 problems,
    K- and MN-major in one launch); conv3_bwd and fc1_bwd: wgrad + MASK dgrad writing C_hi / C_lo, both nets."""
    rng = np.random.default_rng(600 + ci)
    g = T.conv_geometry(64, 64, ci)
    (_, _, _, _, _, H1, W1, _), (_, _, _, _, _, H2, W2, _), (_, _, _, _, _, H3, W3, _) = g
    L = T.Launch(x3, seed=60 + ci)
    x = rng.random(BATCH * 64 * 64 * ci).astype(F32)
    for net in range(2):
        dZ1 = normal(rng, BATCH * H1 * W1 * 32)
        conv_wgrad(L, rng, g[0], x, iota(BATCH * H1 * W1, 32), dZ1, ci_odd=bool(ci & 1), conv1=True)
    check(L, f"conv1 wgrad ci={ci}")

    L = T.Launch(x3, seed=70 + ci)
    P2h, P2w = H2 + 3, W2 + 3
    for net in range(2):
        h1 = relu_like(rng, BATCH * H1 * W1 * 32)
        dZ2p = _bordered(rng, BATCH, H2, W2, 1, 2)
        dz2row = T.bordered_rows(BATCH, H2, W2, P2h, P2w, 1)
        conv_wgrad(L, rng, g[1], h1, dz2row, dZ2p)
        W2m = conv_w(rng, 512, 64)
        dZ1 = L.put("f32", n=BATCH * H1 * W1 * 32)
        dZ1p = (L.put("u16", n=BATCH * H1 * W1 * 32), L.put("u16", n=BATCH * H1 * W1 * 32))
        for py in range(2):
            for px in range(2):
                am, ar, br, bn, cm = T.conv2_dgrad_tables(BATCH, H1, W1, H2, W2, py, px)
                p = L.add(len(am), 32, 256, GG["PLANES"] | GG["A_RVEC"] | GG["B_RVEC"] | GG["EPI_MASK"], dZ2p, am, ar, W2m, br, bn, cm,
                          iota(64)[:32], mask=h1, c_at=dZ1)
                p.oC_hi, p.oC_lo = dZ1p
    assert len(L.problems) == 10
    check(L, f"conv2 bwd ci={ci}")

    L = T.Launch(x3, seed=80 + ci)
    P3h, P3w = H3 + 4, W3 + 4
    for net in range(2):
        h2 = relu_like(rng, BATCH * H2 * W2 * 64)
        dZ3p = _bordered(rng, BATCH, H3, W3, 2, 2)
        conv_wgrad(L, rng, g[2], h2, T.bordered_rows(BATCH, H3, W3, P3h, P3w, 2), dZ3p)
        am, ar, br, bn, cm = T.conv3_dgrad_tables(BATCH, H2, W2, H3, W3)
        L.add(len(am), 64, 576, GG["PLANES"] | GG["A_RVEC"] | GG["B_RVEC"] | GG["EPI_MASK"], dZ3p, am, ar, conv_w(rng, 576, 64), br,
              bn, cm, iota(64), mask=h2, kM=iota(BATCH * H2 * W2, 64), kN=iota(64), c_planes=True, c_len=BATCH * P2h * P2w * 64)
    check(L, f"conv3 bwd ci={ci}")

    L = T.Launch(x3, seed=90 + ci)
    rowP3, cN3p = T.fc1_dgrad_tables(BATCH, H3, W3)
    for net in range(2):
        h3 = relu_like(rng, BATCH * 1024)
        dZ4 = normal(rng, BATCH * 512)
        # fc1 wgrad: dWf[j, h] = sum_b h3[b, j] dZ4[b, h]  (MN-major, no split)
        L.add(1024, 512, BATCH, GG["PLANES"] | GG["MN_MAJOR"], h3, iota(1024), iota(BATCH, 1024), dZ4, iota(BATCH, 512), iota(512),
              iota(1024, 512), iota(512))
        # fc1 dgrad: dZ3p[b, j] = sum_h dZ4[b, h] Wf[j, h], masked by h3 > 0
        L.add(BATCH, 1024, 512, GG["PLANES"] | GG["A_RVEC"] | GG["B_RVEC"] | GG["EPI_MASK"], dZ4, iota(BATCH, 512), iota(512),
              conv_w(rng, 1024, 512), iota(512), iota(1024, 512), rowP3, cN3p, mask=h3, kM=iota(BATCH, 1024), kN=iota(1024),
              c_planes=True, c_len=BATCH * P3h * P3w * 64)
    check(L, f"fc1 bwd ci={ci}")


# ------------------------------------------------------------------ epilogue paths and column tables
@X3
@pytest.mark.parametrize("planes", [False, True])
def test_epilogue_paths(planes, x3):
    """The same problems with column tables that do and do not satisfy GG_CN_AFFINE4 (fast and generic epilogue), N tails
    17, 33, 36, 63 and 100 (AFFINE4 tables with a partial last 16-column group), MASK with its own kM / kN layout, BIAS_RELU,
    C_hi / C_lo."""
    rng = np.random.default_rng(700 + planes)
    L = T.Launch(x3, seed=70 + planes)
    base = GG["A_RVEC"] | GG["B_RVEC"] | (GG["PLANES"] if planes else 0)
    for j, N in enumerate([17, 33, 36, 63, 64, 100, 128]):
        for affine in (True, False):
            M, R = [129, 200, 64, 300, 7, 257, 130][j], [72, 64, 200, 136, 520, 64, 8][j]
            AS, BS = r4(R) + 8, r4(R) + 8
            Am, Bt = normal(rng, M * AS), normal(rng, N * BS)
            cs = r4(N) + (4 if affine else 2)            # row stride: a multiple of 4, or not
            mask = (j % 2 == 0)
            fl = base | (GG["EPI_MASK"] if mask else GG["EPI_BIAS_RELU"])
            ms = r4(N) + (8 if affine else 3)            # mask row stride: a multiple of 4, or not
            kw = dict(mask=relu_like(rng, M * ms), kM=iota(M, ms), kN=iota(N)) if mask else dict(bias=normal(rng, N, 0.5))
            L.add(M, N, R, fl, Am, iota(M, AS), iota(R), Bt, iota(R), iota(N, BS), iota(M, cs), iota(N), c_planes=True,
                  c_shift=0, **kw)
    check(L, f"epilogue paths planes={planes}")


def schedule(L, num_sms):
    """(problem, n0, col_id) of the consecutive tiles of every CTA, as gg_tc_kernel walks the flattened tile list."""
    col, ids, tiles = {}, [], []
    for i, p in enumerate(L.problems):
        key = (p.cN.off, -1 if p.kN is None else p.kN.off, p.bias.off if p.flags & GG["EPI_BIAS_RELU"] else -1, p.N)
        ids.append(col.setdefault(key, len(col)))
        tn = cdiv(p.N, BN)
        for t in range(cdiv(p.M, BM) * tn * p.splitR):
            tiles.append((i, (t % tn) * BN, ids[-1]))
    return [tiles[b::num_sms] for b in range(min(num_sms, len(tiles)))]


@X3
def test_sixteen_problem_group(x3):
    """16 problems of one launch whose consecutive tiles on one CTA change col_id at the same n0 and n0 at the same col_id."""
    rng = np.random.default_rng(800)
    L = T.Launch(x3, seed=80)
    num_sms = torch.cuda.get_device_properties(0).multi_processor_count
    tabs = [L.tab(iota(128)), L.tab(iota(128))]
    biases = [L.f32(normal(rng, 128, 0.5)), L.f32(normal(rng, 128, 0.5))]
    for i in range(16):
        N = (128, 64, 128, 100)[i % 4]
        M = 128 * (6 + i % 7) - 3 * (i % 3)
        R = 64 + 24 * (i % 3)
        k = (i // 2) % 2
        X, W = normal(rng, M * r4(R)), normal(rng, N * r4(R))
        L.add(M, N, R, GG["A_RVEC"] | GG["B_RVEC"] | GG["EPI_BIAS_RELU"], X, iota(M, r4(R)), iota(R), W, iota(R), iota(N, r4(R)),
              iota(M, 128), tabs[k] if N == 128 else iota(N), bias=biases[k] if N == 128 else normal(rng, N, 0.5))
    steps = [(a, b) for cta in schedule(L, num_sms) for a, b in zip(cta, cta[1:])]
    assert any(a[2] != b[2] and a[1] == b[1] for a, b in steps), "no CTA changes col_id at the same n0"
    assert any(a[2] == b[2] and a[1] != b[1] for a, b in steps), "no CTA changes n0 at the same col_id"
    assert any(a[2] == b[2] and a[0] != b[0] for a, b in steps), "no CTA hops between problems of one col_id"
    check(L, "16 problems")
