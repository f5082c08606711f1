"""CPU: register and spill budgets of the fused passes of craig! / craigmr! (the Craig* / Craigmr* functors of
fused_phases.cu), read from the build's ptxas log: the staged SpMV instantiations keep the 3-CTA/SM budget of the other
staged families (at most 72 registers), both precisions come in pairs, and nothing spills."""
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
    return [(d, r, s) for d, (_, r, s) in zip(names, ents) if "kb::Craig" in d]


def test_counts_pairs_and_budgets():
    hit = _kernels()
    count = lambda kernel: len([e for e in hit if e[0].startswith(f"void kb::{kernel}<")])   # noqa: E731
    # CRAIG C1, C2 and CRAIGMR R1, R2, in both precisions, staged and untiled
    assert count("spmv_epi_tma") == 8 and count("spmv_epi_rows") == 8, hit
    # CRAIG's x flush and CRAIGMR's R3, in both precisions
    assert count("stream_epi") == 4, hit
    f32 = sorted(e[0].replace("float", "double") for e in hit if "<float" in e[0])
    assert f32 == sorted(e[0] for e in hit if "<double" in e[0])
    for name, regs, spill in hit:
        assert spill == 0, (name, regs, spill)
        if name.startswith("void kb::spmv_epi_tma<"):
            assert regs <= 72, (name, regs)
