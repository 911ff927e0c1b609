"""The fp32 gather-GEMM engine (csrc/gg_simt.cu) held element by element, through b2g_debug_gg_simt, in all three builds.

Each case is one grouped launch modelled on a real call site, its tables built with the handles' formulas (dqn.cu / bdq.cu /
ppo.cu gemm_desc arguments, enc_fwd_tables, autoencoder.cu's add_conv_dgrad / add_conv_wgrad / add_dense_dgrad).  Checks:
  1. builds 0 and 2 without GG_EPI_ATOMIC: bit for bit against the fmaf chain of tests/gg_simt_ref.py and the fp32 epilogue
     (BIAS, BIAS_RELU, BIAS_LRELU, MASK, SCALE; C_hi = bf16_rn(v), C_lo = bf16_rn(v - hi)); BIAS_TANH within 2 ulp of float64
     tanh of the bit-exact argument; TANH_GRAD within 2.01 * 2^-24 |v| of v (1 - y^2), which allows 1 - y*y to be contracted;
  2. build 1 without GG_EPI_ATOMIC: bit for bit against the float64 chain rounded once to fp32, then the epilogue;
  3. GG_EPI_ATOMIC: within (splitR - 1) 2^-24 sum|partials| (2^-53 for build 1's double accumulators) of the sum of the
     per-split chains restated as in 1 / 2 (R <= 4096; longer sums are held to 4 only);
  4. every output against float64: |got - ref| <= gamma_L (sum|a||b| + |bias|) + the epilogue's own roundings;
  5. column sums within gamma_R sum|B| of float64, added once whatever tiles_m is;
  6. every arena element that no problem writes (inputs, slack, NaN-payload sentinels in f32, f64 and u16) is unchanged;
  7. a second launch gives bit-identical non-ATOMIC outputs.
Run with -s to see the worst err/bar of each case.
"""
import numpy as np
import pytest

from b200grasp import _lib
from tests import gg_simt_ref as G
from tests.gg_simt_ref import GG

pytestmark = pytest.mark.gpu
F32, F64 = np.float32, np.float64
U24, U53 = 2.0 ** -24, 2.0 ** -53
EXACT_R = 4096
EPI = ("EPI_BIAS_RELU", "EPI_BIAS", "EPI_BIAS_LRELU", "EPI_MASK", "EPI_LRELU_GRAD", "EPI_BIAS_TANH", "EPI_TANH_GRAD", "EPI_SCALE")


def r4(x):
    return -(-x // 4) * 4


def iota(n, stride=1, base=0):
    return base + np.arange(n, dtype=np.int64) * stride


def normal(rng, n, scale=1.0):
    return (rng.standard_normal(n) * scale).astype(F32)


def relu_like(rng, n, zeros=0.4):
    """ReLU outputs: non-negative with exact zeros."""
    v = np.abs(normal(rng, n))
    v[rng.random(n) < zeros] = 0
    return v


# ------------------------------------------------------------------ the checker
def _flag(p, name):
    return bool(p.flags & GG[name])


def check(L, case):
    arenas = L.arenas()
    rc, out = L.run(arenas)
    assert rc == 0, _lib.load().b2g_last_error()
    rc2, out2 = L.run(arenas)
    assert rc2 == 0, _lib.load().b2g_last_error()
    f32, f64, u16 = out
    worst = {}

    def note(key, err, bar):
        r = float(np.max(np.where(bar > 0, err / np.where(bar > 0, bar, 1), np.where(err > 0, np.inf, 0)))) if err.size else 0.0
        worst[key] = max(worst.get(key, 0.0), r)
        return r

    written = {"f32": np.zeros(len(f32), bool), "f64": np.zeros(len(f64), bool), "u16": np.zeros(len(u16), bool)}
    for i, p in enumerate(L.problems):
        tag = f"p{i} M{p.M} N{p.N} R{p.R} s{p.splitR}"
        Am, Bm = G.gathered(p)
        idx = p.oC + G.out_index(p)
        atomic = _flag(p, "EPI_ATOMIC")
        got = (f64 if p.c64 else f32)[idx]
        got_again = (out2[1] if p.c64 else out2[0])[idx]
        written["f64" if p.c64 else "f32"][idx.ravel()] = True
        bias = None if p.bias_arr is None else np.asarray(p.bias_arr, F32)[:p.N]
        mask = G.mask_of(p)
        A64, B64 = Am.astype(F64), Bm.astype(F64)
        ref = A64 @ B64
        absab = np.abs(A64) @ np.abs(B64)
        u = U53 if L.build == 1 else U24

        # ---- 1 / 2 / 3: the restated chains
        if p.R <= EXACT_R:
            parts = []
            for r0, r1 in G.split_ranges(p.R, p.splitR):
                if L.build == 1:
                    parts.append(G.chain_f64(Am[:, r0:r1], Bm[r0:r1]))
                else:
                    parts.append(G.chain_f32(Am[:, r0:r1], Bm[r0:r1]))
            if not atomic:
                v = parts[0].astype(F32)
                want = G.epilogue(v, p.flags, bias, mask, p.alpha, L.build)
                if _flag(p, "EPI_BIAS_TANH"):
                    arg = (v + bias[None, :]).astype(F32)
                    t = np.tanh(arg.astype(F64))
                    err = np.abs(got.astype(F64) - t)
                    note("1 tanh ulp/2", err, 2 * np.spacing(np.abs(t).astype(F32)).astype(F64))
                elif _flag(p, "EPI_TANH_GRAD"):
                    y = mask.astype(F64)
                    t = v.astype(F64) * (1 - y * y)
                    note("1 tanh_grad", np.abs(got.astype(F64) - t), 2.01 * U24 * np.abs(v.astype(F64)))
                else:
                    bad = got.view(np.uint32 if got.dtype == F32 else np.uint64) != want.view(np.uint32)
                    note(f"{'2' if L.build == 1 else '1'} bit-exact (mismatches)", bad.astype(F64), np.zeros(bad.shape))
                    assert not bad.any(), (case, tag, int(bad.sum()), np.argwhere(bad)[:5], got[bad][:5], want[bad][:5])
                if p.oC_hi >= 0:
                    hi = G.bf16_rn(want)
                    lo = G.bf16_rn(want - G.bf16_to_f32(hi))
                    hidx, lidx = p.oC_hi + G.out_index(p), p.oC_lo + G.out_index(p)
                    written["u16"][hidx.ravel()] = True
                    written["u16"][lidx.ravel()] = True
                    assert np.array_equal(u16[hidx], hi) and np.array_equal(u16[lidx], lo), (case, tag, "C_hi / C_lo")
            else:
                assert not any(_flag(p, e) for e in EPI), "the split checks assume no epilogue"
                tot = np.sum([q.astype(F64) for q in parts], axis=0)
                bar = (p.splitR - 1) * u * np.sum([np.abs(q.astype(F64)) for q in parts], axis=0)
                err = np.abs(got.astype(F64) - tot)
                r = note("3 split sum", err, bar)
                assert r <= 1, (case, tag, "split sum", r)

        # ---- 4: against float64
        pre = ref + (bias[None, :].astype(F64) if bias is not None else 0)
        if L.build == 1:        # double chain, one rounding of the sum to fp32, one fp32 bias add
            bar = G.gamma(p.R + p.splitR, U53) * absab + U24 * np.abs(ref) + (U24 * np.abs(pre) if bias is not None else 0)
        else:                   # fp32 chain of R terms, the split adds and the bias add
            bar = G.gamma(p.R + p.splitR + 2, U24) * (absab + (np.abs(bias[None, :]).astype(F64) if bias is not None else 0))
        post, lip = pre, 1.0
        a = float(np.float32(p.alpha))
        if _flag(p, "EPI_BIAS_RELU"):
            post = np.maximum(post, 0)
        if _flag(p, "EPI_BIAS_LRELU"):
            post, lip = np.where(post > 0, post, a * post), max(1.0, abs(a))
        if _flag(p, "EPI_MASK"):
            post = np.where(mask > 0, post, 0)
        if _flag(p, "EPI_LRELU_GRAD"):
            g = np.where(mask > 0, 1.0, np.where(mask < 0, a, 0.0))
            post, lip = post * g, lip * max(1.0, abs(a))
        if _flag(p, "EPI_BIAS_TANH"):
            post = np.tanh(post)
        if _flag(p, "EPI_TANH_GRAD"):
            post = post * (1 - mask.astype(F64) ** 2)
        if _flag(p, "EPI_SCALE"):
            post, lip = post * a, lip * abs(a)
        bar = lip * bar + 4 * U24 * np.abs(post)
        r = note("4 float64", np.abs(got.astype(F64) - post), bar)
        assert r <= 1, (case, tag, "float64", r)

        # ---- 5: column sums
        if p.ocolsum >= 0:
            cs = (f64 if p.s64 else f32)[p.ocolsum:p.ocolsum + p.N].astype(F64)
            written["f64" if p.s64 else "f32"][p.ocolsum:p.ocolsum + p.N] = True
            r = note("5 colsum", np.abs(cs - B64.sum(0)), G.gamma(p.R, U53 if p.s64 else U24) * np.abs(B64).sum(0))
            assert r <= 1, (case, tag, "colsum", r)

        # ---- 7: determinism
        if not atomic:
            assert np.array_equal(got.view(np.uint8), got_again.view(np.uint8)), (case, tag, "second launch differs")

    # ---- 6: nothing else moved
    for name, before, after in (("f32", arenas[0], f32), ("f64", arenas[1], f64), ("u16", arenas[2], u16)):
        keep = ~written[name]
        b8 = before.view(np.uint16 if name == "u16" else (np.uint32 if name == "f32" else np.uint64))
        a8 = after.view(b8.dtype)
        moved = np.flatnonzero(keep & (b8 != a8))
        assert moved.size == 0, (case, name, "untouched elements changed at", moved[:8])
    print(f"\n[{case}] worst err/bar: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(worst.items())))
    return worst


# ------------------------------------------------------------------ call-site models
def dense_fwd(L, rng, M, N, R, flags, XS=None, perm=None, c_stride=None, c_base=0, cN=None, c_len=None, planes=False, alpha=1.0):
    """DQN / BDQ tower layer: A = X rows of stride XS (rows gathered through perm), B = W [R][fs], C rows of c_stride."""
    XS = XS or r4(R)
    rows = perm if perm is not None else np.arange(M)
    X = normal(rng, (int(rows.max()) + 1) * XS)
    fs = r4(N)
    W = normal(rng, R * fs, 1 / np.sqrt(R))
    cs = c_stride or r4(N)
    bias = normal(rng, N, 0.5) if flags & (GG["EPI_BIAS"] | GG["EPI_BIAS_RELU"] | GG["EPI_BIAS_LRELU"] | GG["EPI_BIAS_TANH"]) else None
    return L.add(X, rows * XS, iota(R), W, iota(R, fs), iota(N), iota(M, cs, c_base), iota(N) if cN is None else cN, M, N, R, flags,
                 bias=bias, c_len=c_len, planes=planes, alpha=alpha)


def wgrad(L, rng, M, N, R, flags, splitR=1, colsum=True):
    """DQN / PPO weight gradient: A = h [R batch rows][HS] read m-direction, B = dz [R][NS] n-direction, C = dW [M][fs]."""
    HS, NS = r4(M), r4(N)
    h = relu_like(rng, R * HS)
    dz = normal(rng, R * NS)
    return L.add(h, iota(M), iota(R, HS), dz, iota(R, NS), iota(N), iota(M, r4(N)), iota(N), M, N, R, flags, splitR=splitR,
                 colsum=colsum)


@pytest.mark.parametrize("flags", ["BIAS_RELU", "BIAS"])
def test_forward_towers_plain(flags):
    L = G.Launch(0, seed=1)
    rng = np.random.default_rng(11)
    f = GG["A_RVEC"] | GG["EPI_" + flags]
    shapes = [(1, 2, 1), (33, 4, 7), (64, 12, 15), (65, 63, 16), (130, 64, 17), (1024, 65, 100), (33, 512, 512), (130, 12, 512),
              (1, 512, 17), (65, 65, 100), (1024, 2, 7), (64, 63, 1)]
    if flags == "BIAS":
        shapes = [(m, n, r) for (m, _, r), (_, n, _) in zip(shapes, shapes[3:] + shapes[:3])]
    for M, N, R in shapes:
        dense_fwd(L, rng, M, N, R, f)
    check(L, "fwd " + flags)


def test_weight_gradients_colsum_and_split_atomic():
    L = G.Launch(0, seed=2)
    rng = np.random.default_rng(12)
    for M, N, R in [(1, 64, 32), (3, 12, 100), (65, 65, 64), (130, 4, 33)]:
        wgrad(L, rng, M, N, R, GG["COLSUM"])
    for (M, N, R), s in [((65, 64, 300), 1), ((130, 65, 300), 2), ((3, 12, 1000), 7), ((1, 64, 40), 4)]:
        wgrad(L, rng, M, N, R, GG["COLSUM"] | GG["EPI_ATOMIC"], splitR=s)
    check(L, "wgrad")


def test_input_gradients_mask_and_scale():
    """BDQ's branch dgrad into the concatenated map (kM / kN differ from cM / cN) and the trunk's MASK|SCALE rescale."""
    L = G.Launch(0, seed=3)
    rng = np.random.default_rng(13)
    B, HB, NBS, D = 65, 64, 6, 3
    hin = relu_like(rng, B * HB)
    cat = L.put("f32", n=B * (D + 1) * HB)
    for q, (N_out, M) in enumerate([(NBS, B), (4, B)]):
        dz = normal(rng, M * r4(N_out))
        W = normal(rng, HB * r4(N_out))
        # dz [M][N_out] . W^T: A = dz (r = output column), B(r, n) = W[n * fs + r]
        L.add(dz, iota(M, r4(N_out)), iota(N_out), W, iota(N_out), iota(HB, r4(N_out)), iota(M, (D + 1) * HB), iota(HB, 1, q * HB),
              M, HB, N_out, GG["A_RVEC"] | GG["B_RVEC"] | GG["EPI_MASK"], mask=hin, kM=iota(M, HB), kN=iota(HB), c_at=cat)
    T1, NCAT = 130, (D + 1) * HB
    dcat = normal(rng, 33 * NCAT)
    Wt = normal(rng, T1 * NCAT)
    h2 = relu_like(rng, 33 * T1)
    L.add(dcat, iota(33, NCAT), iota(NCAT), Wt, iota(NCAT), iota(T1, NCAT), iota(33, r4(T1)), iota(T1), 33, T1, NCAT,
          GG["A_RVEC"] | GG["B_RVEC"] | GG["EPI_MASK"] | GG["EPI_SCALE"], mask=h2, kM=iota(33, T1), kN=iota(T1), alpha=1 / (D + 1))
    check(L, "dgrad mask")


def test_ppo_tanh_build():
    L = G.Launch(2, seed=4)
    rng = np.random.default_rng(14)
    M, H0, H1 = 70, 64, 33
    H1s = r4(H1)
    Y0 = np.tanh(normal(rng, M * 2 * H0, 2)).astype(F32)
    Y0[::7] = 0
    Y0[1::11] = 1
    Y0[2::13] = -1
    Y1 = L.put("f32", n=M * 2 * H1s)
    for tw in range(2):       # two BIAS_TANH problems writing the column halves of one [M, 2 H1] output
        W1 = normal(rng, H0 * H1s, 0.3)
        L.add(Y0[tw * H0:], iota(M, 2 * H0), iota(H0), W1, iota(H0, H1s), iota(H1), iota(M, 2 * H1s), iota(H1), M, H1, H0,
              GG["A_RVEC"] | GG["EPI_BIAS_TANH"], bias=normal(rng, H1, 0.5), c_at=Y1 + tw * H1s)
    for tw in range(2):       # dgrad through the stored tanh outputs (y in {-1, 0, 1} among ordinary values)
        dZ1 = normal(rng, M * 2 * H1s)
        W1 = normal(rng, H0 * H1s, 0.3)
        L.add(dZ1[tw * H1s:], iota(M, 2 * H1s), iota(H1), W1, iota(H1), iota(H0, H1s), iota(M, 2 * H0), iota(H0), M, H0, H1,
              GG["A_RVEC"] | GG["B_RVEC"] | GG["EPI_TANH_GRAD"], mask=Y0[tw * H0:], c_len=M * 2 * H0)
    check(L, "ppo tanh")


def splits_for(tiles, R):
    return max(1, min(-(-264 // tiles), -(-R // 64)))


@pytest.mark.parametrize("D", [20480, 65536])
def test_ppo_layer0_long_split_sums(D):
    """The plain layer-0 forward over a permuted rollout (rowoff = perm * XS), split-R over D as ppo.cu splits it."""
    L = G.Launch(0, seed=5)
    rng = np.random.default_rng(15)
    n_rows, XS, H0 = 9, r4(D), 64
    for M in (64, 5):
        perm = rng.permutation(n_rows)[:M] if M <= n_rows else rng.integers(0, n_rows, M)
        tiles = -(-M // 64) * -(-(2 * H0) // 64)
        s = splits_for(tiles, D)
        obs = normal(rng, n_rows * XS)
        W0 = normal(rng, D * 2 * H0, 1 / np.sqrt(D))
        L.add(obs, perm * XS, iota(D), W0, iota(D, 2 * H0), iota(2 * H0), iota(M, 2 * H0), iota(2 * H0), M, 2 * H0, D,
              GG["A_RVEC"] | GG["EPI_ATOMIC"], splitR=s)
    check(L, f"ppo l0 D={D}")


def enc_fwd(L, rng, n_img, ih, iw, ic, k, s, f, alpha=0.3):
    """enc_fwd_tables: 'same' conv over a zero-bordered NHWC input, output into the next layer's bordered map."""
    oh, ow = -(-ih // s), -(-iw // s)
    ph, pw = max((oh - 1) * s + k - ih, 0), max((ow - 1) * s + k - iw, 0)
    hp, wp = ih + ph, iw + pw
    fs = r4(f)
    o_pt, o_pl, o_hp, o_wp = 1, 1, oh + 2, ow + 2
    x = np.zeros((n_img, hp, wp, ic), F32)
    x[:, ph // 2:ph // 2 + ih, pw // 2:pw // 2 + iw] = rng.standard_normal((n_img, ih, iw, ic))
    aM, cM = [], []
    for b in range(n_img):
        for oy in range(oh):
            for ox in range(ow):
                aM.append(((b * hp + oy * s) * wp + ox * s) * ic)
                cM.append(((b * o_hp + oy + o_pt) * o_wp + ox + o_pl) * f)
    R = k * k * ic
    r = np.arange(R)
    c, kx, ky = r % ic, (r // ic) % k, r // (ic * k)
    aR = (ky * wp + kx) * ic + c
    W = normal(rng, R * fs, 1 / np.sqrt(R))
    flags = GG["A_RVEC"] | GG["EPI_BIAS_LRELU"] | (GG["A_SCALAR"] if ic & 3 else 0)
    return L.add(x.ravel(), np.array(aM), aR, W, iota(R, fs), iota(f), np.array(cM), iota(f), len(aM), f, R, flags,
                 bias=normal(rng, f, 0.5), alpha=alpha, c_len=n_img * o_hp * o_wp * f)


def test_encoder_forward_im2col():
    L = G.Launch(0, seed=6)
    rng = np.random.default_rng(16)
    enc_fwd(L, rng, 3, 21, 19, 1, 5, 2, 16)     # in_c 1: element-wise A gathers
    enc_fwd(L, rng, 2, 13, 13, 3, 3, 2, 6)      # in_c 3, f 6: outputs rows of 6 floats (scalar stores)
    enc_fwd(L, rng, 2, 9, 9, 8, 3, 1, 12)       # in_c 8: r-vector loads
    check(L, "encoder fwd")


def _lrelu_out(rng, n):
    """Stored LeakyReLU outputs: > 0, < 0 and exactly 0."""
    v = normal(rng, n)
    v[rng.random(n) < 0.2] = 0
    return v


def test_autoencoder_ext_dgrads():
    L = G.Launch(1, seed=7)
    rng = np.random.default_rng(17)
    alpha = 0.3
    # dense dgrad (add_dense_dgrad): A = D [N][dw], B(r, n) = W[n * fs + r], mask = the dense input [N][in_ld]
    N, F, Rin = 33, 24, 132
    dw, fs, in_ld = r4(F), r4(F), r4(Rin)
    Dm, W, act = normal(rng, N * dw), normal(rng, Rin * fs), _lrelu_out(rng, N * in_ld)
    L.add(Dm, iota(N, dw), iota(F), W, iota(F), iota(Rin, fs), iota(N, Rin), iota(Rin), N, Rin, F,
          GG["A_RVEC"] | GG["B_RVEC"] | GG["EPI_LRELU_GRAD"], mask=act, kM=iota(N, in_ld), kN=iota(Rin), alpha=alpha)
    # output-conv dgrad (add_conv_dgrad, f = 1 so fs = 1): A_SCALAR r gathers, n-direction B over the c input channels
    n_img, h, w, c, k, f = 2, 12, 10, 8, 3, 1
    pad = k // 2
    dh, dwid = h + 2 * pad, w + 2 * pad
    Dc = np.zeros((n_img, dh, dwid, f), F32)
    Dc[:, pad:pad + h, pad:pad + w] = rng.standard_normal((n_img, h, w, f))
    Wc = normal(rng, k * k * c * 1)
    aM, kM, cM = [], [], []
    for b in range(n_img):
        for yy in range(h):
            for xx in range(w):
                aM.append(((b * dh + yy) * dwid + xx) * f)
                kM.append(((b * h + yy) * w + xx) * c)
                cM.append(((b * (h + 2) + yy + 1) * (w + 2) + xx + 1) * c)
    R = k * k * f
    r = np.arange(R)
    fi, kx, ky = r % f, (r // f) % k, r // (f * k)
    aR = (ky * dwid + kx) * f + fi
    bR = ((k - 1 - ky) * k + (k - 1 - kx)) * c * 1 + fi
    L.add(Dc.ravel(), np.array(aM), aR, Wc, bR, iota(c, 1), np.array(cM), iota(c), len(aM), c, R,
          GG["A_RVEC"] | GG["A_SCALAR"] | GG["EPI_LRELU_GRAD"], mask=_lrelu_out(rng, n_img * h * w * c), kM=np.array(kM), kN=iota(c),
          alpha=alpha, c_len=n_img * (h + 2) * (w + 2) * c)
    # forward of a decoder dense layer in the same build (no atomics: bit for bit)
    dense_fwd(L, rng, 33, 20, 36, GG["A_RVEC"] | GG["EPI_BIAS_LRELU"], alpha=alpha)
    check(L, "ae ext dgrad")


def conv_wgrad(L, rng, n_img, ih, iw, ic, k, s, f):
    """add_conv_wgrad: M = (ky, kx, c), N = filters, R = (b, oy, ox); m-direction A (A_SCALAR when ic & 3), double sums."""
    oh, ow = -(-ih // s), -(-iw // s)
    ph, pw = max((oh - 1) * s + k - ih, 0), max((ow - 1) * s + k - iw, 0)
    hp, wp = ih + ph, iw + pw
    fs = r4(f)
    x = np.zeros((n_img, hp, wp, ic), F32)
    x[:, ph // 2:ph // 2 + ih, pw // 2:pw // 2 + iw] = rng.standard_normal((n_img, ih, iw, ic))
    M = k * k * ic
    m = np.arange(M)
    aM = ((m // (ic * k)) * wp + (m // ic) % k) * ic + m % ic
    P = oh * ow
    R = n_img * P
    b, rem = np.arange(R) // P, np.arange(R) % P
    oy, ox = rem // ow, rem % ow
    aR = ((b * hp + oy * s) * wp + ox * s) * ic
    Dm = normal(rng, R * fs)
    bR = np.arange(R) * fs
    tiles = -(-M // 64) * -(-f // 64)
    splitR = max(1, min(-(-2 * 132 // tiles), R // 256))
    flags = GG["EPI_ATOMIC"] | GG["COLSUM"] | (GG["A_SCALAR"] if ic & 3 else 0)
    return L.add(x.ravel(), aM, aR, Dm, bR, iota(f), iota(M, fs), iota(f), M, f, R, flags, splitR=splitR, colsum=True)


def test_autoencoder_ext_wgrads_into_double():
    L = G.Launch(1, seed=8)
    rng = np.random.default_rng(18)
    p1 = conv_wgrad(L, rng, 8, 32, 32, 1, 3, 2, 16)     # in_c 1, R = 2048: splitR 8
    p3 = conv_wgrad(L, rng, 4, 24, 24, 3, 5, 2, 8)      # in_c 3
    p8 = conv_wgrad(L, rng, 2, 16, 16, 8, 3, 1, 12)     # in_c 8: m-direction ld4 on the A side, M = 72 (two tile rows)
    assert p1.splitR == 8 and p3.splitR == 2 and p8.splitR == 2
    # dense wgrad (add_dense_wgrad): A = the input rows [N][in_ld] m-direction, B = D [N][dw]
    N, Min, F = 64, 130, 20
    L.add(normal(rng, N * r4(Min)), iota(Min), iota(N, r4(Min)), normal(rng, N * r4(F)), iota(N, r4(F)), iota(F), iota(Min, r4(F)),
          iota(F), Min, F, N, GG["EPI_ATOMIC"] | GG["COLSUM"], colsum=True)
    check(L, "ae ext wgrad")


def test_output_forms():
    """C_hi / C_lo planes, the scalar store path (cN stride 2; C rows at 2 mod 4), and one group of 12 problems of 1 to 9
    tiles, mixing epilogues."""
    L = G.Launch(0, seed=9)
    rng = np.random.default_rng(19)
    dense_fwd(L, rng, 70, 65, 33, GG["A_RVEC"] | GG["EPI_BIAS_RELU"], planes=True)
    dense_fwd(L, rng, 65, 12, 20, GG["A_RVEC"] | GG["EPI_BIAS"], cN=iota(12, 2), c_stride=24)
    dense_fwd(L, rng, 66, 16, 20, GG["A_RVEC"] | GG["EPI_BIAS"], c_stride=20, c_base=2)
    for M, N, R in [(1, 1, 1), (3, 4, 5), (64, 64, 16), (65, 1, 9), (129, 130, 31), (7, 200, 18), (2, 3, 64), (190, 8, 4),
                    (64, 65, 3)]:
        fl = [GG["EPI_BIAS_RELU"], GG["EPI_BIAS"], GG["EPI_BIAS_LRELU"]][len(L.problems) % 3]
        dense_fwd(L, rng, M, N, R, GG["A_RVEC"] | fl, alpha=0.2)
    assert len(L.problems) == 12
    check(L, "output forms")
