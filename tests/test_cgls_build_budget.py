"""CPU: the fused CGLS / CRLS phases and LSLQ's update pass (fused_phases.cu) keep the 3-CTA/SM budget of the staged SpMV family: every
staged-epilogue instantiation of spmv_epi_tma uses at most 72 registers (288 threads x 72 x 3 CTAs fill the 64K register
file), and none of the new kernels spills."""
import os
import re
import shutil
import subprocess

import pytest

BUILD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "krylov.jl_b200", "build")


def test_cgls_crls_phase_kernels_fit_three_ctas_per_sm():
    path = os.path.join(BUILD, "fused_phases.ptxas.log")
    if not os.path.exists(path):
        pytest.skip("build logs absent: run __graft_entry__.build()")
    if not shutil.which("c++filt"):
        pytest.skip("c++filt not available")
    txt = open(path).read()
    ents = [(m.group(1), int(m.group(2)), max([int(v) for v in re.findall(r"(\d+) bytes spill", m.group(0))] or [0]))
            for m in re.finditer(r"Compiling entry function '(\S+)' for 'sm_90a'.*?Used (\d+) registers[^\n]*", txt, re.S)]
    names = subprocess.run(["c++filt"], input="\n".join(e[0] for e in ents), capture_output=True, text=True).stdout.splitlines()
    new = [(d, r, s) for d, (_, r, s) in zip(names, ents) if "kb::Cgls" in d or "kb::Crls" in d]
    staged = [e for e in new if "spmv_epi_tma<" in e[0]]
    assert len(staged) == 8, staged                   # CGLS K1, K3 and CRLS L2, L4 x Float32 / Float64
    for name, regs, spill in staged:
        assert regs <= 72 and spill == 0, (name, regs, spill)
    assert len([e for e in new if "spmv_epi_rows<" in e[0]]) == 8
    assert len([e for e in new if "stream_epi<" in e[0]]) == 8      # CGLS K2, K4 and CRLS L1, L3 x 2
    for name, regs, spill in new:
        assert spill == 0, (name, regs, spill)
    lslq = [(d, r, s) for d, (_, r, s) in zip(names, ents) if "kb::LslqUpdateBody" in d]
    assert len(lslq) == 2 and all(s == 0 for _, _, s in lslq), lslq  # LSLQ's update pass (P1 / P2 are LSQR's)
