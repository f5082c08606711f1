"""CPU: the CGNE and CRMR fused passes (fused_phases.cu, `Cgne*` / `Crmr*` functors) keep the register budget of the
staged SpMV family, read from the sm_90a build's `-Xptxas -v` log: every spmv_epi_tma instantiation uses at most 72
registers (288 threads x 72 x 3 CTAs fill the 64K register file), and no kernel of either family spills."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "krylov.jl_b200", "build", "fused_phases.ptxas.log")
# family -> {kernel template: instantiations, Float32 and Float64 together}
COUNTS = {"Cgne": {"spmv_epi_tma": 4, "spmv_epi_rows": 4},                    # E1 on A, E2 on Aᵀ, staged and untiled
          "Crmr": {"spmv_epi_tma": 4, "spmv_epi_rows": 4, "stream_epi": 4}}   # R1, R3 and the streaming R2, R4


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


@pytest.mark.parametrize("family", sorted(COUNTS))
def test_passes_fit_three_ctas_per_sm(family):
    hit = [e for e in _entries() if f"kb::{family}" in e[0]]
    for tmpl in ("spmv_epi_tma", "spmv_epi_rows", "stream_epi"):
        got = len([e for e in hit if e[0].startswith(f"void kb::{tmpl}<")])
        assert got == COUNTS[family].get(tmpl, 0), (tmpl, hit)
    f32 = sorted(e[0].replace("float", "double") for e in hit if "<float" in e[0])
    assert f32 == sorted(e[0] for e in hit if "<double" in e[0]), hit          # both precisions, in pairs
    for name, regs, spill in hit:
        assert spill == 0, (name, regs, spill)
        if "spmv_epi_tma<" in name:
            assert regs <= 72, (name, regs)


def test_no_other_family_functor_in_their_kernels():
    """The new kernels carry only their own functors: no functor of the least-squares, least-norm or CAR / MINARES
    families, whose instantiation counts other budget tests pin by substring."""
    for name, _, _ in _entries():
        if "kb::Cgne" in name or "kb::Crmr" in name:
            assert not re.search(r"kb::(Craig|Cgls|Crls|Lnlq|Car|Minares|Lsq)", name), name
