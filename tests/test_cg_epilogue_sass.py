"""The contraction engine runs the ACT / DGRAD epilogue in a warpgroup of its own, so that the MMA warps can start the next
tile's mainloop while it runs.  Two properties of the compiled `cg_kernel` say that the split happened:
  - setmaxnreg gives the three roles (MMA, epilogue, producer warpgroups) the register counts cg.cu chooses, and they fit the
    register file;
  - the BF16 plane split of the epilogue (F2FP.BF16 pack instructions) is reached only from the epilogue warpgroup's setmaxnreg,
    and no HGMMA is reached from there: the MMA warps never run that code, and the epilogue warps never issue a wgmma.
Both only show in the machine code: a kernel where the MMA warps still run the epilogue computes the same results."""
import os
import re
import subprocess

import pytest

from tests.test_cg_sass import CG_CU, LIB, _cuobjdump

BRA = re.compile(r"^(@!?U?P\w+\s+)?BRA(?:\.\w+)*\s+(?:(!?U?P\w+),\s*)?(0x[0-9a-f]+)")


def _regs(name):
    m = re.search(r"\b%s = (\d+)" % name, open(CG_CU).read())
    assert m, f"{name} not found in cg.cu"
    return int(m.group(1))


def _setmaxnreg(ins):
    """(kind, count) of every setmaxnreg in the kernel: kind 'inc' or 'dec'."""
    out = []
    for t in ins:
        m = re.search(r"USETMAXREG\.(TRY_ALLOC|DEALLOC)\S*\s+(?:U?P\w+,\s*)?(0x[0-9a-f]+|\d+)", t)
        if m:
            out.append(("inc" if m.group(1) == "TRY_ALLOC" else "dec", int(m.group(2), 0)))
    return out


def _reachable(ins, addrs, start):
    """Instruction indices reachable from index `start` by fall-through and direct branches."""
    index = {a: i for i, a in enumerate(addrs)}
    seen, todo = set(), [start]
    while todo:
        i = todo.pop()
        while i < len(ins) and i not in seen:
            seen.add(i)
            t = ins[i].strip()
            assert not re.match(r"^(@!?U?P\w+\s+)?(BRX|JMX|CALL|RET)\b", t), f"indirect control flow reached: {t}"
            m = BRA.match(t)
            if m:
                todo.append(index[int(m.group(3), 16)])
                if not (m.group(1) or m.group(2)):
                    break
            elif re.match(r"^EXIT\b", t):
                break
            i += 1
    return seen


def test_setmaxnreg_per_role_counts():
    mma, epi, prod = _regs("MMA_REGS"), _regs("EPI_REGS"), _regs("PROD_REGS")
    assert 2 * mma + epi + prod <= 512, (mma, epi, prod)
    assert all(v % 8 == 0 for v in (mma, epi, prod)) and prod >= 24
    got = sorted(_setmaxnreg([t for _, t in _raw_cg_sass()]))
    assert got == sorted([("inc", mma), ("inc", epi), ("dec", prod)]), got


def test_bf16_plane_split_only_in_epilogue_warpgroup():
    sass = _raw_cg_sass()
    addrs = [int(a, 16) for a, _ in sass]
    ins = [t for _, t in sass]
    epi = _regs("EPI_REGS")
    starts = [i for i, t in enumerate(ins) if re.search(r"USETMAXREG\.TRY_ALLOC\S*\s+(?:U?P\w+,\s*)?%s\b" % hex(epi), t)]
    assert len(starts) == 1, f"expected one setmaxnreg to {epi} (the epilogue warpgroup), found {len(starts)}"
    reach = _reachable(ins, addrs, starts[0])
    pack = [i for i, t in enumerate(ins) if "F2FP.BF16" in t]
    assert pack, "no BF16 pack instructions in cg_kernel"
    assert not [i for i in reach if "HGMMA" in ins[i]], "the epilogue warpgroup reaches wgmma code"
    outside = [hex(addrs[i]) for i in pack if i not in reach]
    assert not outside, f"BF16 plane split outside the epilogue warpgroup at {outside}"


def _raw_cg_sass():
    """(address, instruction) of every instruction of cg_kernel."""
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found")
    if not os.path.exists(LIB):
        pytest.skip("libb200grasp.so not built")
    sass = subprocess.run([exe, "-sass", LIB], capture_output=True, text=True, check=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    body = [f for f in funcs if f.split("\n", 1)[0].find("cg_kernel") >= 0]
    assert len(body) == 1, "expected exactly one cg_kernel in the library"
    return [(m.group(1), m.group(2)) for m in re.finditer(r"/\*([0-9a-f]{4,})\*/\s+([^;]*);", body[0])]
