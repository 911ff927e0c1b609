"""CPU tests of tests/gg_simt_ref.py (the restatement tests/test_gpu_gg_simt.py holds the fp32 gather-GEMM engine to) and of the
refusals of b2g_debug_gg_simt, which it makes before any CUDA call."""
import ctypes as C
from fractions import Fraction

import numpy as np
import pytest

from b200grasp import _lib
from tests import gg_simt_ref as G

F32 = np.float32


def _round_f32(x):
    """Fraction -> nearest fp32, ties to even (finite, normal range)."""
    r = np.float32(float(x))
    cands = [np.nextafter(r, F32(-np.inf)), r, np.nextafter(r, F32(np.inf))]
    best = min(cands, key=lambda c: (abs(Fraction(float(c)) - x), int(np.asarray(c, F32).view(np.uint32)) & 1))
    return F32(best)


def _fmaf_exact(a, b, c):
    return np.array([_round_f32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))) for x, y, z in zip(a, b, c)], F32)


def _random_triples(rng, n):
    a = (rng.standard_normal(n) * 2.0 ** rng.integers(-8, 9, n)).astype(F32)
    b = (rng.standard_normal(n) * 2.0 ** rng.integers(-8, 9, n)).astype(F32)
    c = (rng.standard_normal(n) * 2.0 ** rng.integers(-20, 21, n)).astype(F32)
    c[: n // 4] = -(a[: n // 4].astype(np.float64) * b[: n // 4]).astype(F32)     # cancellation: c ~ -a*b
    return a, b, c


def _traps(rng, n):
    """c with an odd last mantissa bit and a*b = +-(half an ulp of c)(1 - u^2 2^-46): the exact sum lies 2^-70 ulp(c) short of
    the midpoint next to c, the float64 sum lands on it, and ties-to-even picks the wrong neighbour."""
    m = (rng.integers(1 << 22, 1 << 23, n) * 2 + 1).astype(np.float64) * 2.0 ** -23        # [1, 2), odd last bit
    k = rng.integers(-10, 11, n).astype(np.float64)
    sgn = np.where(rng.random(n) < 0.5, -1.0, 1.0)
    c = (sgn * m * 2.0 ** k).astype(F32)
    u = rng.integers(1, 300, n).astype(np.float64)
    side = np.where(rng.random(n) < 0.5, -1.0, 1.0)
    a = (side * sgn * (1 - u * 2.0 ** -23) * 2.0 ** (k - 24)).astype(F32)
    b = (1 + u * 2.0 ** -23).astype(F32)
    return a, b, c


def test_fmaf_restatement_matches_exact_rounding_on_random_triples():
    rng = np.random.default_rng(1)
    a, b, c = _random_triples(rng, 20000)
    want = _fmaf_exact(a, b, c)
    assert np.array_equal(G.fmaf(a, b, c).view(np.uint32), want.view(np.uint32))


def test_fmaf_restatement_survives_double_rounding_traps():
    rng = np.random.default_rng(2)
    a, b, c = _traps(rng, 4000)
    want = _fmaf_exact(a, b, c)
    assert np.array_equal(G.fmaf(a, b, c).view(np.uint32), want.view(np.uint32))
    naive = G.fmaf_naive(a, b, c)
    wrong = int((naive.view(np.uint32) != want.view(np.uint32)).sum())
    assert wrong >= len(a) // 2, wrong          # the traps do catch the float64-then-fp32 shortcut


def test_chain_restatements_match_exact_arithmetic():
    rng = np.random.default_rng(3)
    Am = (rng.standard_normal((3, 40)) * 2.0 ** rng.integers(-6, 7, (3, 40))).astype(F32)
    Bm = (rng.standard_normal((40, 5)) * 2.0 ** rng.integers(-6, 7, (40, 5))).astype(F32)
    got32, got64 = G.chain_f32(Am, Bm), G.chain_f64(Am, Bm)
    for m in range(3):
        for n in range(5):
            acc32, acc64 = F32(0), 0.0
            for r in range(40):
                exact = Fraction(float(Am[m, r])) * Fraction(float(Bm[r, n]))
                acc32 = _round_f32(exact + Fraction(float(acc32)))
                acc64 = float(exact + Fraction(acc64))        # Fraction -> float rounds correctly
            assert got32[m, n].view(np.uint32) == np.asarray(acc32, F32).view(np.uint32)
            assert got64[m, n] == acc64


def test_split_ranges_and_bf16_split():
    assert G.split_ranges(40, 4) == [(0, 16), (16, 32), (32, 40), (40, 40)]
    assert G.split_ranges(100, 1) == [(0, 100)]
    assert G.split_ranges(65536, 132)[127] == (65024, 65536) and G.split_ranges(65536, 132)[128] == (65536, 65536)
    v = np.array([1.0, 1 + 2.0 ** -8, 1 + 3 * 2.0 ** -8, 1 + 5 * 2.0 ** -10, -3.14159, 1e-3], F32)
    hi = G.bf16_rn(v)
    assert list(hi[:4]) == [0x3F80, 0x3F80, 0x3F82, 0x3F81]           # ties to even both ways; past the midpoint rounds up
    assert np.all(np.abs(G.bf16_to_f32(hi) - v) <= np.abs(v) * 2.0 ** -8)


# ------------------------------------------------------------------ refusals of b2g_debug_gg_simt (before any CUDA call)
def _base(build=0, flags=None, M=70, N=9, R=21, **kw):
    """A valid dense problem: A r-contiguous (rows of stride 24) under GG_A_RVEC, else m-contiguous (rows of 72 per r); B
    n-contiguous (rows of 12 per r), or r-contiguous (rows of 24 per n) under GG_B_RVEC."""
    L = G.Launch(build)
    rng = np.random.default_rng(0)
    f = G.GG["A_RVEC"] | G.GG["EPI_BIAS_RELU"] if flags is None else flags
    A = rng.standard_normal(M * 24 if f & G.GG["A_RVEC"] else R * 72).astype(F32)
    B = rng.standard_normal(R * 12 if not f & G.GG["B_RVEC"] else N * 24).astype(F32)
    aM, aR = (np.arange(M) * 24, np.arange(R)) if f & G.GG["A_RVEC"] else (np.arange(M), np.arange(R) * 72)
    bR, bN = (np.arange(R), np.arange(N) * 24) if f & G.GG["B_RVEC"] else (np.arange(R) * 12, np.arange(N))
    bias = rng.standard_normal(N).astype(F32) if f & (G.GG["EPI_BIAS_RELU"] | G.GG["EPI_BIAS"]) else None
    L.add(A, aM, aR, B, bR, bN, np.arange(M) * N, np.arange(N), M, N, R, f, bias=bias, **kw)
    return L


def _refused(L, edit, words):
    st = L.structs()
    f32, f64, u16, tabs = L.arenas()
    edit(st[0], tabs)
    rc, _ = L.run((f32, f64, u16, tabs), st)
    msg = _lib.load().b2g_last_error().decode()
    assert rc == _lib.B2G_EINVAL, (rc, msg)
    assert words in msg, msg


def test_valid_problem_passes_the_checks():
    rc, _ = _base().run()
    assert rc in (0, _lib.B2G_ECUDA), _lib.load().b2g_last_error()      # ECUDA: refused only for want of a GPU


@pytest.mark.parametrize("what", ["aM", "aR", "bR", "bN", "cM", "cN"])
def test_refuses_a_table_entry_out_of_range(what):
    L = _base()
    big = {"aM": 10 ** 6, "aR": 10 ** 6, "bR": 10 ** 6, "bN": 10 ** 6, "cM": 10 ** 6, "cN": 10 ** 6}[what]

    def edit(s, tabs):
        tabs[getattr(s, what) + 1] = big                              # entry 1 keeps the 4-groups of entry 0 aside
    _refused(L, edit, "outside its arena")


def test_refuses_negative_address_and_table_past_its_arena():
    L = _base()
    _refused(L, lambda s, t: t.__setitem__(s.aR + 2, -10 ** 6), "outside its arena")
    _refused(L, lambda s, t: setattr(s, "cN", len(t) - 3), "past the end of tabs")


def test_refuses_a_broken_r_group():
    L = _base()
    _refused(L, lambda s, t: t.__setitem__(s.aR + 5, 6), "GG_A_RVEC: aR is not contiguous")
    Lb = _base(flags=G.GG["A_RVEC"] | G.GG["B_RVEC"])
    _refused(Lb, lambda s, t: t.__setitem__(s.bR + 2, 0), "GG_B_RVEC: bR is not contiguous")


def test_a_scalar_lifts_the_r_group_contract_on_a_only():
    L = _base(flags=G.GG["A_RVEC"] | G.GG["A_SCALAR"])
    st = L.structs()
    f32, f64, u16, tabs = L.arenas()
    tabs[st[0].aR + 5] = 6
    rc, _ = L.run((f32, f64, u16, tabs), st)
    assert rc in (0, _lib.B2G_ECUDA), _lib.load().b2g_last_error()


def test_refuses_misaligned_r_groups_and_m_n_groups():
    L = _base()
    _refused(L, lambda s, t: setattr(s, "A", s.A + 2), "not 16-byte aligned")
    _refused(L, lambda s, t: t.__setitem__(s.aM + 3, t[s.aM + 3] + 1), "not 16-byte aligned")
    # n-direction B: columns 0..3 must be one contiguous, aligned 4-group
    _refused(L, lambda s, t: t.__setitem__(s.bN + 2, 7), "n-direction B: bN is not contiguous")
    # m-direction A (no GG_A_RVEC)
    Lm = _base(flags=G.GG["COLSUM"], colsum=True)
    _refused(Lm, lambda s, t: t.__setitem__(s.aM + 1, 100), "m-direction A: aM is not contiguous")


def test_refuses_misaligned_c():
    L = _base()
    _refused(L, lambda s, t: setattr(s, "C", s.C + 1), "C must be 16-byte aligned")


@pytest.mark.parametrize("build,flag", [(0, "EPI_BIAS_TANH"), (1, "EPI_TANH_GRAD"), (0, "EPI_LRELU_GRAD"), (2, "EPI_LRELU_GRAD"),
                                        (0, 1 << 6)])
def test_refuses_a_flag_of_another_build(build, flag):
    L = _base(build)
    f = G.GG[flag] if isinstance(flag, str) else flag
    _refused(L, lambda s, t: setattr(s, "flags", s.flags | f), "are not flags of build")


def test_refuses_m_direction_a_scalar_outside_build_1():
    L = _base(0, flags=G.GG["COLSUM"], colsum=True)
    _refused(L, lambda s, t: setattr(s, "flags", s.flags | G.GG["A_SCALAR"]), "m-direction GG_A_SCALAR exists in build 1 only")


def test_refuses_bad_extents_splits_and_operands():
    L = _base()
    _refused(L, lambda s, t: setattr(s, "R", 0), "M, N and R must be >= 1")
    _refused(L, lambda s, t: setattr(s, "splitR", 2), "splitR > 1 needs GG_EPI_ATOMIC")
    _refused(L, lambda s, t: setattr(s, "splitR", 0), "splitR must be in 1..R")
    _refused(L, lambda s, t: setattr(s, "bias", -1), "needs bias")
    _refused(L, lambda s, t: setattr(s, "flags", s.flags | G.GG["EPI_MASK"]), "needs mask")
    _refused(L, lambda s, t: setattr(s, "C_hi", 0), "C_hi and C_lo go together")
    Lc = _base(flags=G.GG["COLSUM"] | G.GG["B_RVEC"] | G.GG["A_RVEC"], colsum=True)
    _refused(Lc, lambda s, t: None, "cannot take GG_B_RVEC")


def test_refuses_group_size_and_build():
    L = _base()
    st = L.structs()
    f32, f64, u16, tabs = L.arenas()
    lib = _lib.load()
    args = (f32.ctypes.data_as(C.POINTER(C.c_float)), len(f32), f64.ctypes.data_as(C.POINTER(C.c_double)), len(f64),
            u16.ctypes.data_as(C.POINTER(C.c_uint16)), len(u16), tabs.ctypes.data_as(C.POINTER(C.c_int32)), len(tabs))
    assert lib.b2g_debug_gg_simt(0, st, 0, *args) == _lib.B2G_EINVAL
    assert lib.b2g_debug_gg_simt(0, st, 17, *args) == _lib.B2G_EINVAL
    assert lib.b2g_debug_gg_simt(3, st, 1, *args) == _lib.B2G_EINVAL
    assert b"build must be" in lib.b2g_last_error()
