"""How exact is the tensor core's fp32 accumulation on cancelling reductions?

C = A B^T through the wgmma engine (b2g_debug_gemm) against float64 evaluated on the SAME bf16-split operands
(hi*hi + hi*lo + lo*hi in float64), so the operand split drops out and what is left is the accumulation itself.
Rows of A / B are built so that the products cancel to a chosen fraction of their absolute sum."""
import ctypes as C
import os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from b200grasp import _lib

lib = _lib.load()
fp = C.POINTER(C.c_float)


def gemm(A, B, x3, split=1):
    M, K = A.shape; N = B.shape[0]
    out = np.zeros((M, N), np.float32)
    rc = lib.b2g_debug_gemm(M, N, K, A.ctypes.data_as(fp), B.ctypes.data_as(fp), out.ctypes.data_as(fp), x3, split)
    assert rc == 0, rc
    return out


def bf(x):
    return torch.from_numpy(x.astype(np.float32)).bfloat16().float().numpy().astype(np.float64)


rng = np.random.default_rng(0)
for K in (64, 256, 4096, 57600 // 8 * 8):
    for cancel in (1.0, 0.02):
        M, N = 128, 64
        A = rng.standard_normal((M, K)).astype(np.float32)
        B = rng.standard_normal((N, K)).astype(np.float32)
        if cancel == 1.0:
            A, B = np.abs(A), np.abs(B)          # no cancellation: all products positive
        A64, B64 = A.astype(np.float64), B.astype(np.float64)
        ah, bh = bf(A64), bf(B64)
        al, bl = bf(A64 - ah), bf(B64 - bh)
        exact = A64 @ B64.T
        split3 = ah @ bh.T + ah @ bl.T + al @ bh.T                  # what the three MMAs compute with exact accumulation
        split1 = ah @ bh.T
        absum = np.abs(A64) @ np.abs(B64).T
        for x3, ref, name in ((1, split3, "bf16x3"), (0, split1, "bf16  ")):
            for split in (1, 8):
                if split > 1 and K < 1024:
                    continue
                c = gemm(A, B, x3, split).astype(np.float64)
                err = c - ref
                print(f"K={K:6d} {'positive ' if cancel == 1.0 else 'cancelling'} {name} split_k={split}: "
                      f"accum err / |sum| rms {np.sqrt((err**2).mean()) / np.sqrt((ref**2).mean()):.2e}   "
                      f"err / sum|products| rms {np.sqrt(((err/absum)**2).mean()):.2e}  mean(signed) {(err/absum).mean():+.2e}   "
                      f"[split-vs-exact {np.sqrt(((ref-exact)**2).mean()) / np.sqrt((exact**2).mean()):.1e}]", flush=True)
