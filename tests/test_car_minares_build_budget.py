"""CPU: the fused CAR / MINARES passes (fused_phases.cu) keep the 3-CTA/SM budget of the staged SpMV family: the C2
and M1 instantiations of spmv_epi_tma use at most 72 registers (288 threads x 72 x 3 CTAs fill the 64K register file)
and spill nothing, in Float32 and Float64; the streaming passes spill nothing either."""
import os
import re
import shutil
import subprocess

import pytest

BUILD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "krylov.jl_b200", "build")


def test_car_minares_phase_kernels_fit_three_ctas_per_sm():
    path = os.path.join(BUILD, "fused_phases.ptxas.log")
    if not os.path.exists(path):
        pytest.skip("build logs absent: run __graft_entry__.build()")
    if not shutil.which("c++filt"):
        pytest.skip("c++filt not available")
    txt = open(path).read()
    ents = [(m.group(1), int(m.group(2)), max([int(v) for v in re.findall(r"(\d+) bytes spill", m.group(0))] or [0]))
            for m in re.finditer(r"Compiling entry function '(\S+)' for 'sm_90a'.*?Used (\d+) registers[^\n]*", txt, re.S)]
    names = subprocess.run(["c++filt"], input="\n".join(e[0] for e in ents), capture_output=True, text=True).stdout.splitlines()
    new = [(d, r, s) for d, (_, r, s) in zip(names, ents) if "kb::Car" in d or "kb::Minares" in d]
    for epi in ("CarC2Epi", "MinaresM1Epi"):
        staged = [e for e in new if "spmv_epi_tma<" in e[0] and epi in e[0]]
        for dt in ("float", "double"):
            assert any(f"spmv_epi_tma<{dt}," in e[0] for e in staged), (epi, dt)
        for name, regs, spill in staged:
            assert regs <= 72 and spill == 0, (name, regs, spill)
    streams = [e for e in new if "stream_epi<" in e[0]]
    assert len(streams) == 10, streams                 # C1, C3, M2, M3 and the w-only pass x Float32 / Float64
    for name, regs, spill in new:
        assert spill == 0, (name, regs, spill)
