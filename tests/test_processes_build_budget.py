"""CPU: the passes of the Krylov processes (fused_phases.cu launchers, `Proc*` functors of kb_internal.h) keep the
register budget of the staged SpMV family, read from the sm_90a build's `-Xptxas -v` log: the staged instantiations use
at most 72 registers (288 threads x 72 x 3 CTAs fill the 64K register file), no kernel spills, and the new kernels
carry no other family's functor."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "krylov.jl_b200", "build", "fused_phases.ptxas.log")
# kernel template -> instantiations, Float32 and Float64 together: one SpMV epilogue on a divided gather (staged and
# untiled), the streaming update / dot pass and the final normalisation pass
COUNTS = {"spmv_epi_tma": 2, "spmv_epi_rows": 2, "stream_epi": 4}


def _entries():
    if not os.path.exists(LOG):
        pytest.skip("build logs absent: run __graft_entry__.build()")
    if not shutil.which("c++filt"):
        pytest.skip("c++filt not available")
    txt = open(LOG).read()
    ents = []
    for m in re.finditer(r"Compiling entry function '(\S+)' for 'sm_90a'.*?Used (\d+) registers[^\n]*", txt, re.S):
        spill = [int(v) for v in re.findall(r"(\d+) bytes spill", m.group(0))]
        ents.append((m.group(1), int(m.group(2)), max(spill or [0])))
    names = subprocess.run(["c++filt"], input="\n".join(e[0] for e in ents), capture_output=True, text=True).stdout
    return [(d, r, s) for d, (_, r, s) in zip(names.splitlines(), ents)]


def test_process_passes_fit_three_ctas_per_sm():
    hit = [e for e in _entries() if "kb::Proc" in e[0]]
    for tmpl, count in COUNTS.items():
        assert len([e for e in hit if e[0].startswith(f"void kb::{tmpl}<")]) == count, (tmpl, hit)
    f32 = sorted(e[0].replace("float", "double") for e in hit if "<float" in e[0])
    assert f32 == sorted(e[0] for e in hit if "<double" in e[0]), hit
    for name, regs, spill in hit:
        assert spill == 0, (name, regs, spill)
        if "spmv_epi_tma<" in name:
            assert regs <= 72, (name, regs)


def test_no_other_family_functor_in_the_process_kernels():
    for name, _, _ in _entries():
        if "kb::Proc" in name:
            others = re.sub(r"kb::Proc\w+|kb::NoFin|kb::Csr\b|kb::DistComm", "", name)
            assert not re.search(r"kb::[A-Z]", others), name
