"""The contraction engine keeps one K-chunk of wgmmas in flight: in the compiled `cg_kernel`, every chunk of every instantiated
shape is one run of HGMMAs with no WARPGROUP.DEPBAR (wgmma.wait_group) inside it.  ptxas inserts such a wait after every
wgmma when it cannot prove the sequence safe to chain (a run-time k-step count, partly overlapping accumulator ranges, a
divergent branch between the wgmmas); the kernel then still computes the right result, only with the tensor pipe drained after
every instruction, so only the machine code shows it."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "deep-rl-grasping_b200", "libb200grasp.so")
CG_CU = os.path.join(ROOT, "deep-rl-grasping_b200", "csrc", "cg.cu")


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None and os.path.exists("/usr/local/cuda/bin/cuobjdump"):
        exe = "/usr/local/cuda/bin/cuobjdump"
    return exe


def _cg_kernel_sass():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found")
    if not os.path.exists(LIB):
        pytest.skip("libb200grasp.so not built")
    sass = subprocess.run([exe, "-sass", LIB], capture_output=True, text=True, check=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    body = [f for f in funcs if f.split("\n", 1)[0].find("cg_kernel") >= 0]
    assert len(body) == 1, "expected exactly one cg_kernel in the library"
    return [m.group(1) for m in re.finditer(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", body[0])]


def _chunk_sizes():
    """HGMMAs per K-chunk of every shape the kernel dispatches to: k-steps x products (one MMA per product)."""
    shapes = re.findall(r"CG_CONSUME\((\d+), (\d+), (\d), (\d+)\)", open(CG_CU).read())
    assert shapes, "no consume_tile instantiations found in cg.cu"
    return [int(ks) * int(nprod) for _, nprod, _, ks in shapes]


def test_cg_kernel_wgmma_chunks_are_not_serialised():
    ins = _cg_kernel_sass()
    chunks = _chunk_sizes()
    hgmma = [i for i, t in enumerate(ins) if "HGMMA" in t]
    waits = [i for i, t in enumerate(ins) if "WARPGROUP.DEPBAR" in t]
    assert len(hgmma) == sum(chunks), (len(hgmma), chunks)
    # one wait_group 1 inside each chunk loop and one wait_group 0 after it
    assert len(waits) <= 2 * len(chunks), (len(waits), len(chunks))
    runs, n = [], 0
    for t in ins:
        if "HGMMA" in t:
            n += 1
        elif "WARPGROUP.DEPBAR" in t and n:
            runs.append(n)
            n = 0
    if n:
        runs.append(n)
    assert sorted(runs) == sorted(chunks), f"HGMMA runs between waits {sorted(runs)}, chunks {sorted(chunks)}"
