"""Restatement of the wgmma gather-GEMM engine (csrc/gg_tc.cu) and of the SAC handle's tables for it, shared by
tests/test_gpu_gg_tc.py, tests/test_gg_tc_cpu.py and tests/test_gpu_contractions.py.

The engine multiplies BF16 splits of its operands on the tensor cores: x = hi + lo with hi = RN_bf16(x), lo = RN_bf16(x - hi),
and one output is hi*hi + hi*lo + lo*hi (x3 = 1) or hi*hi (x3 = 0) summed over 64-row r-chunks into an fp32 accumulator,
split-R partials added into the zeroed output with fp32 atomics.  ``gg_gammas`` is the error allowance of that sum per element,
``Report`` holds outputs to a float64 reference under such a bar.

``Launch`` lays problems out in the three arenas of ``b2g_debug_gg_tc`` (f32, u16, int32 tables) with NaN-payload sentinels in
the slack, and ``run`` calls the entry.  The ``*_tables`` functions restate sac.cu's build_groups formulas for the CNN and head
contractions that run on this engine.
"""
import ctypes as C

import numpy as np
import torch

from b200grasp import _lib
from tests.gg_simt_ref import SENT16, SENT32, bf16_rn, bf16_to_f32

GG = dict(_lib.GG, **_lib.GG_TC)
F32, F64 = np.float32, np.float64
BM, BN, BK = 128, 64, 64       # GG_TC_BM / BN / BK: output tile 128 x 64, 64-row r-chunks

U_TC = 2.0 ** -23         # one tensor-core k-step: the products' alignment and the accumulator are truncated, not rounded
U32 = 2.0 ** -24          # one round-to-nearest fp32 addition or FMA
# 2 planes, 3 products: the missing A_1 B_1
SPLIT2 = (2.0 ** -8 * (1 + 2.0 ** -8)) ** 2


def cdiv(a, b):
    return -(-a // b)


def bf16_split(x, n):
    """The first n BF16 planes of fp32 x as uint16: plane k = round-to-nearest of the k-th residual (split3 / planes2)."""
    x = torch.from_numpy(np.ascontiguousarray(x, np.float32))
    out = []
    for _ in range(n):
        h = x.to(torch.bfloat16)
        out.append(h.view(torch.int16).numpy().view(np.uint16).copy())
        x = x - h.float()
    return out


def bf(u16):
    return (np.asarray(u16).astype(np.uint32) << 16).view(np.float32).astype(np.float64)


def gg_gammas(K, split_k, x3):
    """gg_tc: chunks of 64 K rows, all products of a k-step into ONE accumulator (hi*hi, then hi*lo, lo*hi), split-K partials
    summed with red.add into the zeroed output."""
    per = cdiv(cdiv(K, split_k), 64) * 64 if split_k > 1 else cdiv(K, 64) * 64
    acc = 1.01 * (2 * U_TC * (per // 16) * (3 if x3 else 1) + U32 * split_k)
    # the split against the exact product: x3 misses lo*lo and each operand's residual below its lo plane; x3 = 0 misses all
    # but hi*hi
    split = (SPLIT2 + 2 * 2.0 ** -16 + 2.0 ** -32) if x3 else (2 * 2.0 ** -8 + 2.0 ** -16)
    return acc, 1.01 * split + acc


class Report:
    def __init__(self, case):
        self.case, self.worst, self.fail = case, {}, []

    def hold(self, name, got, ref, mag, gamma, r=0.0):
        got, ref, mag = (np.asarray(a, np.float64) for a in (got, ref, mag))
        bar = gamma * mag + r * np.abs(ref)
        err = np.abs(got - ref)
        ratio = np.where(bar > 0, err / np.where(bar > 0, bar, 1.0), np.where(err > 0, np.inf, 0.0))
        worst = float(ratio.max()) if ratio.size else 0.0
        self.worst[name] = max(worst, self.worst.get(name, 0.0))
        if worst > 1.0:
            i = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
            self.fail.append(f"{name}: err/bar {worst:.3g} at {tuple(int(k) for k in i)} (got {got[i]:.9g}, ref {ref[i]:.9g}, "
                             f"bar {bar[i]:.3g}); {int((ratio > 1).sum())} of {ratio.size} elements over")

    def exact(self, name, got, want):
        got, want = np.asarray(got), np.asarray(want)
        bad = int((got != want).sum())
        self.worst[name] = max(self.worst.get(name, 0.0), 0.0 if bad == 0 else np.inf)
        if bad:
            i = np.unravel_index(int(np.argmax(got != want)), got.shape)
            self.fail.append(f"{name}: {bad} of {got.size} elements differ (first at {tuple(int(k) for k in i)}: "
                             f"{got[i]} != {want[i]})")

    def finish(self):
        print(f"\n[{self.case}] worst err/bar per problem (bit-exact checks: 0 = equal):")
        for k, v in self.worst.items():
            print(f"  {k:28s} {v:.3g}")
        assert not self.fail, "\n".join(self.fail)


def split2(x):
    """The engine's operand split of fp32 x: (hi, lo) as BF16 bits."""
    x = np.asarray(x, F32)
    hi = bf16_rn(x)
    return hi, bf16_rn(x - bf16_to_f32(hi))


def iota(n, stride=1, base=0):
    return base + np.arange(n, dtype=np.int64) * stride


def r4(x):
    return -(-x // 4) * 4


# ------------------------------------------------------------------------------------------------ SAC's tables (sac.cu)
def conv_geometry(Hi, Wi, Ci):
    """Nature-CNN layer shapes of the SAC handle: (Hi, Wi, Ci, k, s, Ho, Wo, Co) of conv1..3."""
    H1, W1 = (Hi - 8) // 4 + 1, (Wi - 8) // 4 + 1
    H2, W2 = (H1 - 4) // 2 + 1, (W1 - 4) // 2 + 1
    H3, W3 = H2 - 2, W2 - 2
    return [(Hi, Wi, Ci, 8, 4, H1, W1, 32), (H1, W1, 32, 4, 2, H2, W2, 64), (H2, W2, 64, 3, 1, H3, W3, 64)]


def conv_fwd_tables(B, c):
    """rowoff (output pixel -> NHWC input patch corner), koff (HWIO row -> patch offset), crow (output pixel rows of Co)."""
    Hi, Wi, Ci, k, s, Ho, Wo, Co = c
    b, oy, ox = np.meshgrid(np.arange(B), np.arange(Ho), np.arange(Wo), indexing="ij")
    rowoff = (((b * Hi + oy * s) * Wi + ox * s) * Ci).ravel()
    ky, kx, ci = np.meshgrid(np.arange(k), np.arange(k), np.arange(Ci), indexing="ij")
    koff = ((ky * Wi + kx) * Ci + ci).ravel()
    return rowoff, koff, iota(B * Ho * Wo, Co)


def bordered_rows(B, Ho, Wo, Ph, Pw, pad, C=64):
    """Rows of a [B][Ph][Pw][C] zero-bordered map holding an Ho x Wo map at (pad, pad) (dz2row / dz3row)."""
    b, y, x = np.meshgrid(np.arange(B), np.arange(Ho), np.arange(Wo), indexing="ij")
    return (((b * Ph + y + pad) * Pw + x + pad) * C).ravel()


def conv3_dgrad_tables(B, H2, W2, H3, W3):
    """dZ2 = dZ3 * W3^T over the zero-bordered dZ3p [B][H3+4][W3+4][64]: output into dZ2p [B][H2+3][W2+3][64]."""
    P2h, P2w, P3h, P3w = H2 + 3, W2 + 3, H3 + 4, W3 + 4
    am = bordered_rows(B, H2, W2, P3h, P3w, 2)
    cm = bordered_rows(B, H2, W2, P2h, P2w, 1)
    ky, kx, n = np.meshgrid(np.arange(3), np.arange(3), np.arange(64), indexing="ij")
    ar = (-(ky * P3w + kx) * 64 + n).ravel()
    br = ((ky * 3 + kx) * 64 * 64 + n).ravel()
    return am, ar, br, iota(64, 64), cm


def conv2_dgrad_tables(B, H1, W1, H2, W2, py, px):
    """Parity class (py, px) of dZ1 = dZ2 * W2^T over the zero-bordered dZ2p [B][H2+3][W2+3][64]: output rows of dZ1 [B][H1][W1][32]."""
    P2h, P2w = H2 + 3, W2 + 3
    ny, nx = (H1 - py + 1) // 2, (W1 - px + 1) // 2
    b, yy, xx = np.meshgrid(np.arange(B), np.arange(ny), np.arange(nx), indexing="ij")
    am = (((b * P2h + yy + 1) * P2w + xx + 1) * 64).ravel()
    cm = (((b * H1 + 2 * yy + py) * W1 + 2 * xx + px) * 32).ravel()
    jy, jx, q = np.meshgrid(np.arange(2), np.arange(2), np.arange(64), indexing="ij")
    ar = (-(jy * P2w + jx) * 64 + q).ravel()
    br = ((((py + 2 * jy) * 4 + (px + 2 * jx)) * 32) * 64 + q).ravel()
    return am, ar, br, iota(32, 64), cm


def fc1_dgrad_tables(B, H3, W3):
    """dZ3 = dZ4 * Wf^T into the zero-bordered dZ3p [B][H3+4][W3+4][64] (rowP3, cN3p)."""
    P3h, P3w = H3 + 4, W3 + 4
    y, x, c = np.meshgrid(np.arange(H3), np.arange(W3), np.arange(64), indexing="ij")
    cn = (((y + 2) * P3w + (x + 2)) * 64 + c).ravel()
    return iota(B, P3h * P3w * 64), cn


# ------------------------------------------------------------------------------------------------ the launch
class Ref:
    """Something placed in an arena: its offset and its values (tables: int64, operands: float32)."""

    def __init__(self, off, v):
        self.off, self.v = off, v


class Problem:
    def __init__(self, **kw):
        self.__dict__.update(kw)


class Launch:
    """Problems of one grouped launch laid out in the arenas of b2g_debug_gg_tc."""

    def __init__(self, x3, seed=0):
        self.x3 = x3
        self.rng = np.random.default_rng(seed)
        self.parts = {"f32": [], "u16": [], "tabs": []}
        self.size = {"f32": 0, "u16": 0, "tabs": 0}
        self.problems = []

    def put(self, arena, arr=None, n=None, align=4, shift=0, slack=None):
        """Places arr (or reserves n sentinel elements) at an offset = shift mod align, after some slack; returns the offset."""
        if slack is None:
            slack = int(self.rng.integers(4, 13))
        off = -(-(self.size[arena] + slack) // align) * align + shift
        n = len(arr) if arr is not None else n
        if arr is not None:
            self.parts[arena].append((off, arr))
        self.size[arena] = off + n
        return off

    def tab(self, v):
        """A table, 16-byte aligned, followed by 64 zero entries (the K-major plane producers read r tables a chunk ahead)."""
        v = np.asarray(v, np.int64)
        off = self.put("tabs", v.astype(np.int32), slack=0)
        self.size["tabs"] += BK
        return Ref(off, v)

    def f32(self, v, shift=0):
        v = np.asarray(v, F32)
        return Ref(self.put("f32", v, shift=shift), v)

    def planes(self, v):
        """The hi / lo BF16 planes of fp32 v, each 16-byte aligned in u16."""
        hi, lo = split2(v)
        return Ref(self.put("u16", hi, align=8), v), Ref(self.put("u16", lo, align=8), v)

    def add(self, M, N, R, flags, A, aM, aR, B, bR, bN, cM, cN, kM=None, kN=None, bR_p=None, bN_p=None, bias=None, mask=None,
            splitR=1, colsum=False, c_planes=False, c_len=None, c_at=None, c_shift=0):
        """A, B: fp32 sources (Ref or array), placed in f32, or split into u16 planes under GG_PLANES; tables: Ref (shared) or
        arrays; bias / mask: Ref or array.  C gets its own region of c_len elements (default: the largest address + 1) unless
        c_at gives its offset; it is zeroed where the problem accumulates (GG_EPI_ATOMIC), sentinel elsewhere."""
        t = lambda v: None if v is None else (v if isinstance(v, Ref) else self.tab(v))
        f = lambda v, shift=0: None if v is None else (v if isinstance(v, Ref) else self.f32(v, shift))
        planes = bool(flags & GG["PLANES"])
        p = Problem(M=M, N=N, R=R, flags=flags, splitR=splitR)
        p.aM, p.aR, p.bR, p.bN, p.cM, p.cN, p.kM, p.kN, p.bR_p, p.bN_p = (t(v) for v in (aM, aR, bR, bN, cM, cN, kM, kN, bR_p, bN_p))
        if planes:
            p.A, p.B = None, None
            p.A_hi, p.A_lo = A if isinstance(A, tuple) else self.planes(A)
            p.B_hi, p.B_lo = B if isinstance(B, tuple) else self.planes(B)
            p.A_src, p.B_src = p.A_hi.v, p.B_hi.v
        else:
            p.A, p.B = f(A), f(B)
            p.A_hi = p.A_lo = p.B_hi = p.B_lo = None
            p.A_src, p.B_src = p.A.v, p.B.v
        p.bias, p.mask = f(bias), f(mask)
        if c_len is None:
            c_len = int(p.cM.v.max()) + int(p.cN.v.max()) + 1
        p.oC = self.put("f32", n=c_len, shift=c_shift) if c_at is None else c_at
        p.colsum = self.f32(np.zeros(N, F32)) if colsum else None
        p.oC_hi = p.oC_lo = -1
        if c_planes:
            p.oC_hi = self.put("u16", n=c_len, shift=c_shift)
            p.oC_lo = self.put("u16", n=c_len, shift=c_shift)
        self.problems.append(p)
        return p

    def arenas(self):
        f32 = np.full(self.size["f32"] + 8, SENT32, np.uint32).view(F32)
        u16 = np.full(self.size["u16"] + 8, SENT16, np.uint16)
        tabs = np.zeros(self.size["tabs"], np.int32)
        for name, arr in (("f32", f32), ("u16", u16), ("tabs", tabs)):
            for off, v in self.parts[name]:
                arr[off:off + len(v)] = v
        for p in self.problems:                       # accumulated outputs start from zero
            if p.flags & GG["EPI_ATOMIC"]:
                f32[p.oC + out_index(p)] = 0
        return f32, u16, tabs

    def structs(self):
        arr = (_lib.GgTcProblem * len(self.problems))()
        o = lambda r: -1 if r is None else r.off
        for i, p in enumerate(self.problems):
            s = arr[i]
            s.A, s.B, s.C, s.bias, s.mask, s.colsum = o(p.A), o(p.B), p.oC, o(p.bias), o(p.mask), o(p.colsum)
            for k in ("aM", "aR", "bR", "bN", "cM", "cN", "kM", "kN", "bR_p", "bN_p", "A_hi", "A_lo", "B_hi", "B_lo"):
                setattr(s, k, o(getattr(p, k)))
            s.C_hi, s.C_lo = p.oC_hi, p.oC_lo
            s.M, s.N, s.R, s.flags, s.splitR = p.M, p.N, p.R, p.flags, p.splitR
        return arr

    def run(self, arenas=None, structs=None, x3=None):
        """Calls b2g_debug_gg_tc on copies of the arenas; returns (rc, (f32, u16))."""
        f32, u16, tabs = (a.copy() for a in (arenas or self.arenas()))
        st = structs if structs is not None else self.structs()
        rc = _lib.load().b2g_debug_gg_tc(self.x3 if x3 is None else x3, st, len(st), f32.ctypes.data_as(C.POINTER(C.c_float)),
                                         len(f32), u16.ctypes.data_as(C.POINTER(C.c_uint16)), len(u16),
                                         tabs.ctypes.data_as(C.POINTER(C.c_int32)), len(tabs))
        return rc, (f32, u16)


def b_tables(p):
    """The (bR, bN) tables the engine reads B through: the plane B's own tables of a K-major plane problem when given."""
    kmajor = p.flags & GG["PLANES"] and not p.flags & GG["MN_MAJOR"]
    bR = p.bR_p if kmajor and p.bR_p is not None else p.bR
    bN = p.bN_p if kmajor and p.bN_p is not None else p.bN
    return bR.v, bN.v


def gathered(p):
    """A [M, R] and B [R, N] as the problem's tables read them, float32."""
    bR, bN = b_tables(p)
    Am = np.asarray(p.A_src, F32)[p.aM.v[:, None] + p.aR.v[None, :]]
    Bm = np.asarray(p.B_src, F32)[bR[:, None] + bN[None, :]]
    return Am, Bm


def mask_of(p):
    kM = (p.kM or p.cM).v
    kN = (p.kN or p.cN).v
    return p.mask.v[kM[:, None] + kN[None, :]]


def out_index(p):
    return p.cM.v[:, None] + p.cN.v[None, :]
