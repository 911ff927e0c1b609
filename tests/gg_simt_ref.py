"""Restatement of the fp32 gather-GEMM engine (csrc/gg_simt.cu) for tests/test_gpu_gg_simt.py and tests/test_gg_simt_cpu.py.

The engine's sum for one output is a chain in r order starting from +0: builds 0 and 2 step ``acc = fmaf(a_r, b_r, acc)`` in
fp32, build 1 steps ``acc = fma((double)a_r, (double)b_r, acc)`` in double and rounds once to fp32.  ``fmaf`` below restates
one fp32 step exactly: the float64 product of two fp32 values is exact, TwoSum gives the float64 sum and its error, and when
that sum sits exactly on an fp32 midpoint (the only place where rounding to float64 first can change the fp32 result) the
sign of the error picks the side.  A split-R problem is one chain per split; its chunk is the engine's
``ceil(ceil(R / splitR) / 16) * 16`` rows.

``Launch`` lays problems out in the four arenas of ``b2g_debug_gg_simt`` (f32, f64, u16, int32 tables), with slack filled
with a NaN-payload sentinel between regions, and ``run`` calls the entry.
"""
import ctypes as C

import numpy as np

from b200grasp import _lib

GG = _lib.GG
F32, F64 = np.float32, np.float64
SENT32 = np.uint32(0x7FC1A5A5)            # quiet NaNs with a payload no arithmetic produces
SENT64 = np.uint64(0x7FF8DEADBEEF0001)
SENT16 = np.uint16(0xDEAD)
BK = 16


def fmaf(a, b, c):
    """IEEE fmaf(a, b, c), round to nearest even, for float32 arrays (finite, no overflow / underflow)."""
    a64, b64, c64 = (np.asarray(x, F32).astype(F64) for x in (a, b, c))
    p = a64 * b64                                  # exact: 24 + 24 significant bits
    s = p + c64
    z = s - p
    e = (p - (s - z)) + (c64 - z)                  # TwoSum: s + e == p + c exactly
    r = s.astype(F32)
    d = s - r.astype(F64)
    nb = np.nextafter(r, np.where(d > 0, F32(np.inf), F32(-np.inf)).astype(F32))
    mid = (d != 0) & (2 * s == r.astype(F64) + nb.astype(F64))
    return np.where(mid & (e != 0) & (np.sign(e) == np.sign(d)), nb, r).astype(F32)


def fmaf_naive(a, b, c):
    """float64 product and sum, then one rounding to fp32: double rounding, wrong near fp32 midpoints."""
    return (np.asarray(a, F32).astype(F64) * np.asarray(b, F32).astype(F64) + np.asarray(c, F32).astype(F64)).astype(F32)


def chain_f32(Am, Bm):
    """acc[m, n] = fmaf(Am[m, r], Bm[r, n], acc) for r = 0, 1, ... from +0 (builds 0 and 2)."""
    acc = np.zeros((Am.shape[0], Bm.shape[1]), F32)
    for r in range(Am.shape[1]):
        acc = fmaf(Am[:, r:r + 1], Bm[r:r + 1, :], acc)
    return acc


def chain_f64(Am, Bm):
    """acc[m, n] = RN64(Am[m, r] * Bm[r, n] + acc) for r = 0, 1, ... from +0 (build 1; the products are exact)."""
    acc = np.zeros((Am.shape[0], Bm.shape[1]), F64)
    A64, B64 = Am.astype(F64), Bm.astype(F64)
    for r in range(Am.shape[1]):
        acc = acc + A64[:, r:r + 1] * B64[r:r + 1, :]
    return acc


def split_ranges(R, splitR):
    chunk = -(-(-(-R // splitR)) // BK) * BK
    return [(min(R, s * chunk), min(R, (s + 1) * chunk)) for s in range(splitR)]


def gamma(L, u=2.0 ** -24):
    return L * u / (1 - L * u)


def bf16_rn(v):
    """fp32 -> bf16 bits, round to nearest even (finite values)."""
    u = np.asarray(v, F32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def bf16_to_f32(h):
    return (np.asarray(h, np.uint16).astype(np.uint32) << 16).view(F32)


def epilogue(v, flags, bias, mask, alpha, build):
    """The engine's fp32 epilogue on v [M, N] (bias [N], mask [M, N] already gathered), in its order."""
    v = v.astype(F32)
    a = F32(alpha)
    if flags & GG["EPI_BIAS_RELU"]:
        v = np.maximum(v + bias[None, :], F32(0))
    if flags & GG["EPI_BIAS"]:
        v = v + bias[None, :]
    if flags & GG["EPI_BIAS_LRELU"]:
        v = v + bias[None, :]
        v = np.where(v > 0, v, a * v).astype(F32)
    if flags & GG["EPI_MASK"]:
        v = np.where(mask > 0, v, F32(0)).astype(F32)
    if build == 1 and flags & GG["EPI_LRELU_GRAD"]:
        v = v * np.where(mask > 0, F32(1), np.where(mask < 0, a, F32(0))).astype(F32)
    if flags & GG["EPI_SCALE"]:
        v = v * a
    return v.astype(F32)


class Problem:
    """One problem: gathered tables (int32 arrays), operand arrays, and where everything landed in the arenas."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


class Launch:
    """Problems of one grouped launch laid out in the arenas of b2g_debug_gg_simt."""

    def __init__(self, build, seed=0):
        self.build = build
        self.rng = np.random.default_rng(seed)
        self.parts = {"f32": [], "f64": [], "u16": [], "tabs": []}
        self.size = {"f32": 0, "f64": 0, "u16": 0, "tabs": 0}
        self.problems = []

    def put(self, arena, arr=None, n=None, shift=0, slack=None):
        """Places arr (or reserves n sentinel elements) at a 16-byte-aligned offset + shift; returns the offset."""
        if slack is None:
            slack = int(self.rng.integers(4, 13))
        off = -(-(self.size[arena] + slack) // 4) * 4 + shift
        n = len(arr) if arr is not None else n
        if arr is not None:
            self.parts[arena].append((off, arr))
        self.size[arena] = off + n
        return off

    def tab(self, v):
        return self.put("tabs", np.asarray(v, np.int32), slack=0)

    def add(self, A, aM, aR, B, bR, bN, cM, cN, M, N, R, flags, splitR=1, alpha=1.0, bias=None, mask=None, kM=None, kN=None,
            c_len=None, c_at=None, colsum=False, planes=False, c_zero=None):
        """A, B, bias, mask: float32 arrays placed in f32; C gets its own region of c_len elements (default: the max address
        + 1), or starts at c_at of a region reserved with put(); zeroed where this problem accumulates (GG_EPI_ATOMIC),
        sentinel elsewhere."""
        b = self.build
        c64 = b == 1 and bool(flags & GG["EPI_ATOMIC"])
        s64 = b == 1 and colsum
        p = Problem(M=M, N=N, R=R, flags=flags, splitR=splitR, alpha=float(alpha))
        p.aM, p.aR, p.bR, p.bN, p.cM, p.cN = (np.asarray(t, np.int32) for t in (aM, aR, bR, bN, cM, cN))
        p.kM = None if kM is None else np.asarray(kM, np.int32)
        p.kN = None if kN is None else np.asarray(kN, np.int32)
        p.A_arr, p.B_arr, p.bias_arr, p.mask_arr = A, B, bias, mask
        p.oA = self.put("f32", np.asarray(A, F32))
        p.oB = self.put("f32", np.asarray(B, F32))
        p.obias = -1 if bias is None else self.put("f32", np.asarray(bias, F32))
        p.omask = -1 if mask is None else self.put("f32", np.asarray(mask, F32))
        if c_len is None:
            c_len = int(p.cM.max()) + int(p.cN.max()) + 1
        p.c64 = c64
        p.oC = self.put("f64" if c64 else "f32", n=c_len) if c_at is None else c_at
        p.ocolsum = -1
        if colsum:
            p.ocolsum = self.put("f64" if s64 else "f32", np.zeros(N, F64 if s64 else F32))
        p.s64 = s64
        p.oC_hi = p.oC_lo = -1
        if planes:
            p.oC_hi = self.put("u16", n=c_len)
            p.oC_lo = self.put("u16", n=c_len)
        p.toff = {k: (self.tab(getattr(p, k)) if getattr(p, k) is not None else -1) for k in ("aM", "aR", "bR", "bN", "cM", "cN", "kM", "kN")}
        p.c_zero = bool(flags & GG["EPI_ATOMIC"]) if c_zero is None else c_zero
        self.problems.append(p)
        return p

    def arenas(self):
        f32 = np.full(self.size["f32"] + 8, SENT32, np.uint32).view(F32)
        f64 = np.full(self.size["f64"] + 8, SENT64, np.uint64).view(F64)
        u16 = np.full(self.size["u16"] + 8, SENT16, np.uint16)
        tabs = np.zeros(self.size["tabs"], np.int32)
        for name, arr in (("f32", f32), ("f64", f64), ("u16", u16), ("tabs", tabs)):
            for off, v in self.parts[name]:
                arr[off:off + len(v)] = v
        for p in self.problems:                       # accumulated outputs start from zero
            if p.c_zero:
                idx = p.oC + p.cM[:, None].astype(np.int64) + p.cN[None, :]
                (f64 if p.c64 else f32)[idx] = 0
        return f32, f64, u16, tabs

    def structs(self):
        arr = (_lib.GgProblem * len(self.problems))()
        for i, p in enumerate(self.problems):
            s = arr[i]
            s.A, s.B, s.C, s.bias, s.mask, s.colsum = p.oA, p.oB, p.oC, p.obias, p.omask, p.ocolsum
            for k, v in p.toff.items():
                setattr(s, k, v)
            s.C_hi, s.C_lo = p.oC_hi, p.oC_lo
            s.M, s.N, s.R, s.flags, s.splitR, s.alpha = p.M, p.N, p.R, p.flags, p.splitR, p.alpha
        return arr

    def run(self, arenas=None, structs=None):
        """Calls b2g_debug_gg_simt on copies of the arenas; returns (rc, (f32, f64, u16))."""
        f32, f64, u16, tabs = (a.copy() for a in (arenas or self.arenas()))
        st = structs if structs is not None else self.structs()
        lib = _lib.load()
        rc = lib.b2g_debug_gg_simt(self.build, st, len(st), f32.ctypes.data_as(C.POINTER(C.c_float)), len(f32),
                                   f64.ctypes.data_as(C.POINTER(C.c_double)), len(f64), u16.ctypes.data_as(C.POINTER(C.c_uint16)),
                                   len(u16), tabs.ctypes.data_as(C.POINTER(C.c_int32)), len(tabs))
        return rc, (f32, f64, u16)


def gathered(p):
    """A [M, R] and B [R, N] as the problem's tables read them (offsets relative to the operand arrays)."""
    Am = np.asarray(p.A_arr, F32)[p.aM[:, None].astype(np.int64) + p.aR[None, :]]
    Bm = np.asarray(p.B_arr, F32)[p.bR[:, None].astype(np.int64) + p.bN[None, :]]
    return Am, Bm


def mask_of(p):
    if p.mask_arr is None:
        return None
    kM = p.kM if p.kM is not None else p.cM
    kN = p.kN if p.kN is not None else p.cN
    return np.asarray(p.mask_arr, F32)[kM[:, None].astype(np.int64) + kN[None, :]]


def out_index(p):
    return p.cM[:, None].astype(np.int64) + p.cN[None, :]
