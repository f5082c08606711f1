"""CPU: the fused LSQR / LSMR phases (fused_phases.cu) keep the 3-CTA/SM budget of the staged SpMV family: the P1 and
P2 instantiations of spmv_epi_tma use at most 72 registers (288 threads x 72 x 3 CTAs fill the 64K register file) and
spill nothing; the P3 streaming passes spill nothing either."""
import os
import re
import shutil
import subprocess

import pytest

BUILD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "krylov.jl_b200", "build")


def test_ls_phase_kernels_fit_three_ctas_per_sm():
    path = os.path.join(BUILD, "fused_phases.ptxas.log")
    if not os.path.exists(path):
        pytest.skip("build logs absent: run __graft_entry__.build()")
    if not shutil.which("c++filt"):
        pytest.skip("c++filt not available")
    txt = open(path).read()
    ents = [(m.group(1), int(m.group(2)), max([int(v) for v in re.findall(r"(\d+) bytes spill", m.group(0))] or [0]))
            for m in re.finditer(r"Compiling entry function '(\S+)' for 'sm_90a'.*?Used (\d+) registers[^\n]*", txt, re.S)]
    names = subprocess.run(["c++filt"], input="\n".join(e[0] for e in ents), capture_output=True, text=True).stdout.splitlines()
    staged = [(d, r, s) for d, (_, r, s) in zip(names, ents) if "spmv_epi_tma<" in d and "kb::LsqP" in d]
    assert len(staged) == 6, staged                             # P1, P2 (LSQR), P2 (LSMR) x Float32 / Float64
    for name, regs, spill in staged:
        assert regs <= 72 and spill == 0, (name, regs, spill)
    streams = [(d, r, s) for d, (_, r, s) in zip(names, ents) if "stream_epi<" in d and ("LsqrP3" in d or "LsmrP3" in d)]
    assert len(streams) == 4
    for name, regs, spill in streams:
        assert spill == 0, (name, regs, spill)
