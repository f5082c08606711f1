"""CPU: register and spill budgets of the fused passes of bilqr! / trilqr! (the Adjoint* functors of fused_phases.cu),
read from the build's ptxas log: the staged T1 / T2 SpMV instantiations keep the 3-CTA/SM budget of the other staged
families (at most 72 registers: 288 threads x 72 x 3 CTAs fill the 64K register file), and no update pass spills."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "krylov.jl_b200", "build", "fused_phases.ptxas.log")


def _kernels():
    if not os.path.exists(LOG):
        pytest.skip("build logs absent: run __graft_entry__.build()")
    if not shutil.which("c++filt"):
        pytest.skip("c++filt not available")
    txt = open(LOG).read()
    ents = []
    for m in re.finditer(r"Compiling entry function '(\S+)' for 'sm_90a'.*?Used (\d+) registers[^\n]*", txt, re.S):
        spill = [int(v) for v in re.findall(r"(\d+) bytes spill", m.group(0))]
        ents.append((m.group(1), int(m.group(2)), max(spill or [0])))
    names = subprocess.run(["c++filt"], input="\n".join(e[0] for e in ents), capture_output=True, text=True).stdout.splitlines()
    return [(d, r, s) for d, (_, r, s) in zip(names, ents) if "kb::Adjoint" in d]


def test_update_passes_do_not_spill():
    hit = [e for e in _kernels() if e[0].startswith("void kb::stream_epi<")]
    # BiLQR and TriLQR update passes: both halves, primal only, dual only, x Float32 / Float64
    assert len([e for e in hit if "AdjointBilqrBody" in e[0]]) == 6, hit
    assert len([e for e in hit if "AdjointTrilqrBody" in e[0]]) == 6, hit
    for name, regs, spill in hit:
        assert spill == 0, (name, regs, spill)


def test_ssy_passes_fit_three_ctas_per_sm():
    hit = [e for e in _kernels() if e[0].startswith(("void kb::spmv_epi_tma<", "void kb::spmv_epi_rows<"))]
    assert len([e for e in hit if e[0].startswith("void kb::spmv_epi_tma<")]) == 4, hit     # T1, T2 x 2 precisions
    assert len([e for e in hit if e[0].startswith("void kb::spmv_epi_rows<")]) == 4, hit
    f32 = sorted(e[0].replace("float", "double") for e in hit if "<float" in e[0])
    assert f32 == sorted(e[0] for e in hit if "<double" in e[0])                           # both precisions, in pairs
    for name, regs, spill in hit:
        assert spill == 0, (name, regs, spill)
        if name.startswith("void kb::spmv_epi_tma<"):
            assert regs <= 72, (name, regs)
