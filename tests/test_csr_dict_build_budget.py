"""CPU: build budgets of the kernels on the constant-coefficient encoding (cg_persist_dict, spmv_dict_kernel), read
from the build artefacts like tests/test_build_budget.py: register budget of 3 CTAs of 288 threads per SM without
spills, no Float64 vector read through the non-coherent path while the vectors change inside the launch, and the
gathers of a row issued together."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "krylov.jl_b200", "build")


def _ptxas(name):
    path = os.path.join(BUILD, name + ".ptxas.log")
    if not os.path.exists(path):
        pytest.skip("build logs absent: run __graft_entry__.build()")
    txt = open(path).read()
    out = []
    for m in re.finditer(r"Compiling entry function '(\S+)' for 'sm_90a'.*?Used (\d+) registers[^\n]*", txt, re.S):
        spill = [int(v) for v in re.findall(r"(\d+) bytes spill", m.group(0))]
        out.append((m.group(1), int(m.group(2)), max(spill or [0])))
    return out


def _sass(obj, mangled_substr):
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not available")
    path = os.path.join(BUILD, obj + ".o")
    if not os.path.exists(path):
        pytest.skip("objects absent: run __graft_entry__.build()")
    sass = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True).stdout
    out, keep = [], False
    for line in sass.splitlines():
        if "Function :" in line:
            keep = mangled_substr in line
        elif keep:
            out.append(line)
    assert out, mangled_substr
    return out


def test_dict_kernels_register_budget():
    ents = [e for e in _ptxas("cg_fused") if "cg_persist_dict" in e[0]]
    assert len(ents) == 8                        # {double, float} x {plain, Jacobi} x {3, 2 CTAs per SM}
    for name, regs, spill in ents:
        assert regs <= 72 and spill == 0, (name, regs, spill)
    ents = [e for e in _ptxas("spmv") if "spmv_dict_kernel" in e[0]]
    assert len(ents) == 2
    for name, regs, spill in ents:
        assert spill == 0, (name, spill)


def test_dict_cg_reads_changing_vectors_coherently():
    """r, p and x change between the phases of one launch: no 64-bit read-only load in the plain kernel.  The Jacobi
    kernel may read the diagonal of M (constant during the solve) that way -- at most one per slot and row."""
    for prec in ("d", "f"):
        body = _sass("cg_fused", f"cg_persist_dictI{prec}Li0ELi3E")
        assert not any(".CONSTANT" in l and "LDG.E.64" in l for l in body)
        assert not any("LDG.E.CONSTANT" in l for l in body)           # 32-bit: Float32 vectors
        assert any("LDG.E.U8.CONSTANT" in l for l in body)            # the masks
    body = _sass("cg_fused", "cg_persist_dictIdLi2ELi3E")
    assert sum("LDG.E.64.CONSTANT" in l for l in body) <= 2 * 9


def test_dict_gathers_in_flight():
    """At least 6 64-bit gathers of a row are issued with no FP64 arithmetic between them."""
    def longest_run(body):
        best = cur = 0
        for l in body:
            if "LDG.E.64" in l and "STRONG" not in l:
                cur += 1
                best = max(best, cur)
            elif "DMUL" in l or "DADD" in l or "DFMA" in l:
                cur = 0
        return best
    assert longest_run(_sass("cg_fused", "cg_persist_dictIdLi0ELi3E")) >= 6
    assert longest_run(_sass("cg_fused", "cg_persist_dictIdLi2ELi3E")) >= 6
    assert longest_run(_sass("spmv", "spmv_dict_kernelIdE")) >= 6
