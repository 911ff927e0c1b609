"""conv1 of engine v2 reads the normalised image space-to-depth and runs as a 2x2 stride-1 convolution over it.

Restated here in numpy, index for index as `csrc/engine_v2.cu` and `csrc/sac_internal.cuh` build them:
  - the S layout the gather writes: S[sample][Y 16][X 16][b 4][c 4][ci < Cp] = pixel (4Y + b, 4X + c), Cp = 1 for one channel,
    else 4 with zero pad channels;
  - the K order of the transposed weight planes W1T (`conv1_krow`): window (a, a') = (ky // 4, kx // 4), then (b, c, ci);
  - the forward row tiles: tile tm = 2 s + t reads block rows 8 tm + a of S with the sample folded into the block row, and
    its row r = 16 yl + ox goes to H1 row 225 s + 15 (8 t + yl) + ox unless ox = 15 or 8 t + yl = 15 (junk rows);
  - the weight-gradient rows (M = conv1's K rows) and their scatter to the HWIO gradient, junk pixels zeroed by dZ1's
    out-of-bounds fill;
and checked, in float64, against the 8x8 stride-4 convolution and its weight gradient for 1, 3 and 4 channels."""
import numpy as np
import pytest

HW, OUT, COUT = 64, 15, 32


def s2d_channels(ci):
    return 1 if ci == 1 else 4


def conv1_krow(r, ci_n):
    ci, kx, ky = r % ci_n, (r // ci_n) % 8, r // (8 * ci_n)
    return ((((ky >> 2) * 2 + (kx >> 2)) * 4 + (ky & 3)) * 4 + (kx & 3)) * s2d_channels(ci_n) + ci


def s2d(img):
    """[B, 64, 64, Ci] -> S [B, 16, 16, 4, 4, Cp] (the gather's store index)."""
    B, _, _, ci_n = img.shape
    cp = s2d_channels(ci_n)
    S = np.zeros((B, 16, 16, 4, 4, cp))
    for y in range(HW):
        for x in range(HW):
            S[:, y // 4, x // 4, y % 4, x % 4, :ci_n] = img[:, y, x, :]
    return S


def w1t(w):
    """HWIO [8, 8, Ci, 32] -> W1T [32][64 Cp] in conv1_krow order (pad rows zero)."""
    ci_n = w.shape[2]
    out = np.zeros((COUT, 64 * s2d_channels(ci_n)))
    rows = w.reshape(64 * ci_n, COUT)
    for r in range(64 * ci_n):
        out[:, conv1_krow(r, ci_n)] = rows[r]
    return out


def s_box(S, a, a2):
    """Window (a, a') of every output position of the 16 x 16 grid: S shifted by (a, a') blocks, zero beyond the image -- the
    view folds the sample into the block row, so block row 16 of sample s is sample s + 1's row 0 (out of bounds after the
    last sample).  [B, 16 oy, 16 ox, 16 Cp]."""
    B = S.shape[0]
    flat = S.reshape(B * 16, 16, -1)                       # {16 Cp, 16 X, 16 B Y}
    pad = np.zeros((B * 16 + 1, 17, flat.shape[2]))
    pad[:B * 16, :16] = flat
    out = np.zeros((B, 16, 16, flat.shape[2]))
    for s in range(B):
        out[s] = pad[16 * s + a:16 * s + a + 16, a2:a2 + 16]
    return out


def direct_conv(img, w):
    B = img.shape[0]
    z = np.zeros((B, OUT, OUT, COUT))
    for oy in range(OUT):
        for ox in range(OUT):
            patch = img[:, 4 * oy:4 * oy + 8, 4 * ox:4 * ox + 8, :].reshape(B, -1)
            z[:, oy, ox] = patch @ w.reshape(-1, COUT)
    return z


def direct_wgrad(img, dz):
    ci_n = img.shape[3]
    g = np.zeros((8, 8, ci_n, COUT))
    for oy in range(OUT):
        for ox in range(OUT):
            g += np.einsum("bhwc,bn->hwcn", img[:, 4 * oy:4 * oy + 8, 4 * ox:4 * ox + 8, :], dz[:, oy, ox])
    return g


def forward_rows(B):
    """(tile, row) -> H1 row or -1: the epilogue's band mapping (d0 = 16, d1 = 8, tm_sub = 2, lim_i0 = lim_i1 = 15)."""
    dst = np.full((2 * B, 128), -1)
    for tm in range(2 * B):
        tq, tr = divmod(tm, 2)
        for r in range(128):
            i0, i1 = r % 16, (r // 16) % 8
            if i0 < 15 and tr * 8 + i1 < 15:
                dst[tm, r] = (tq * 225 * 32 + tr * 8 * 15 * 32 + i1 * 15 * 32 + i0 * 32) // 32
    return dst


def wgrad_rows(ci_n):
    """(tile, row) -> HWIO weight row or -1: the in-place WGRAD epilogue's row offsets (d0, d1, o0, o1, o_tm, rgrp_off, lim_i0,
    lim_rows) of the conv1 wgrad problem, and the window / M-row order of its A atoms."""
    cp = s2d_channels(ci_n)
    if cp == 1:
        tiles, d0, d1, o0, o1, o_tm, lim_i0 = 1, 4, 4, 32, 8 * 32, 0, 0
        rgrp = [(32 * (l >> 1) + 4 * (l & 1)) * 32 for l in range(4)] + [0] * 4
        window = lambda tm, r: r // 16                      # four 16-row atoms
    else:
        tiles, d0, d1, o0, o1, o_tm, lim_i0 = 2, 4, 4, 32, ci_n * 32, 32 * ci_n * 32, ci_n
        rgrp = [(8 * ci_n * (j & 3) + 4 * ci_n * (j >> 2)) * 32 for j in range(8)]
        window = lambda tm, r: 2 * tm + r // 64             # two 64-row atoms: windows (tm, 0), (tm, 1)
    dst = np.full((tiles, 128), -1)
    mrow = np.full((tiles, 128), -1)                        # the K row of W1T this M row holds
    for tm in range(tiles):
        for r in range(128):
            i0, i1 = r % d0, (r // d0) % d1
            if tm * 128 + r >= 64 * cp or (lim_i0 > 0 and i0 >= lim_i0):
                continue
            off = i0 * o0 + i1 * o1 + rgrp[min(r // 16, 7)] + tm * o_tm
            dst[tm, r] = off // 32
            mrow[tm, r] = window(tm, r) * 16 * cp + r % (16 * cp)
    return dst, mrow


@pytest.mark.parametrize("ci_n", [1, 3, 4])
def test_krow_is_a_permutation_into_the_padded_k_range(ci_n):
    cp = s2d_channels(ci_n)
    rows = [conv1_krow(r, ci_n) for r in range(64 * ci_n)]
    assert len(set(rows)) == len(rows) and min(rows) >= 0 and max(rows) < 64 * cp
    assert all(k % cp < ci_n for k in rows)                  # pad channels get no weight


@pytest.mark.parametrize("ci_n", [1, 3, 4])
def test_conv1_forward_over_s_equals_the_8x8_stride4_convolution(ci_n):
    rng = np.random.default_rng(ci_n)
    B = 3
    img = rng.standard_normal((B, HW, HW, ci_n))
    w = rng.standard_normal((8, 8, ci_n, COUT))
    S, W = s2d(img), w1t(w)
    cp = s2d_channels(ci_n)
    # the MMA: K = 4 windows x 16 Cp, window (a, a') = K rows [16 Cp (2a + a'), + 16 Cp)
    acc = np.zeros((B, 16, 16, COUT))
    for a in range(2):
        for a2 in range(2):
            k0 = 16 * cp * (2 * a + a2)
            acc += s_box(S, a, a2) @ W[:, k0:k0 + 16 * cp].T
    h1 = np.full((B * 225, COUT), np.nan)
    dst = forward_rows(B)
    for tm in range(2 * B):
        s, t = divmod(tm, 2)
        tile = acc[s, 8 * t:8 * t + 8].reshape(128, COUT)     # box rows: (yl, ox)
        for r in range(128):
            if dst[tm, r] >= 0:
                assert np.isnan(h1[dst[tm, r]]).all(), "an H1 row is written twice"
                h1[dst[tm, r]] = tile[r]
    ref = direct_conv(img, w).reshape(B * 225, COUT)
    assert not np.isnan(h1).any(), "an H1 row is never written"
    np.testing.assert_allclose(h1, ref, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("ci_n", [1, 3, 4])
def test_conv1_wgrad_over_s_equals_the_weight_gradient(ci_n):
    rng = np.random.default_rng(10 + ci_n)
    B = 3
    img = rng.standard_normal((B, HW, HW, ci_n))
    dz = rng.standard_normal((B, OUT, OUT, COUT))
    S = s2d(img)
    cp = s2d_channels(ci_n)
    # B operand: dZ1 viewed as {64, 15 ox, 15 oy, B} with 16 x 16 boxes -> zeros at ox = 15 and oy = 15
    dzp = np.zeros((B, 16, 16, COUT))
    dzp[:, :15, :15] = dz
    # M x N sums of every window: [4 windows x 16 Cp, 32]
    m = np.concatenate([np.einsum("syxk,syxn->kn", s_box(S, a, a2), dzp) for a in range(2) for a2 in range(2)])
    g = np.zeros(64 * ci_n * COUT)
    dst, mrow = wgrad_rows(ci_n)
    hits = np.zeros(64 * ci_n, int)
    for tm in range(dst.shape[0]):
        for r in range(128):
            if dst[tm, r] >= 0:
                g[dst[tm, r] * COUT:(dst[tm, r] + 1) * COUT] += m[mrow[tm, r]]
                hits[dst[tm, r]] += 1
    assert (hits == 1).all(), "every HWIO row is written exactly once"
    # the scatter is the inverse of the forward K permutation
    inv = {conv1_krow(r, ci_n): r for r in range(64 * ci_n)}
    for tm in range(dst.shape[0]):
        for r in range(128):
            if dst[tm, r] >= 0:
                assert inv[mrow[tm, r]] == dst[tm, r]
    ref = direct_wgrad(img, dz).reshape(-1)
    np.testing.assert_allclose(g, ref, rtol=1e-12, atol=1e-9)
