"""CPU: register / spill / SASS budgets of the hot kernels, read from the build artefacts (`-Xptxas -v` logs and
cuobjdump).  Guards the occupancy assumptions the persistent grids rely on: a kernel that silently grows past its
register budget drops a resident CTA per SM (cg_k1 then runs its tiles in 1.5 waves)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "krylov.jl_b200", "build")


def _entries(name):
    path = os.path.join(BUILD, name + ".ptxas.log")
    if not os.path.exists(path):
        pytest.skip("build logs absent: run __graft_entry__.build()")
    txt = open(path).read()
    out = []
    for m in re.finditer(r"Compiling entry function '(\S+)' for 'sm_90a'.*?Used (\d+) registers[^\n]*", txt, re.S):
        spill = [int(v) for v in re.findall(r"(\d+) bytes spill", m.group(0))]
        out.append((m.group(1), int(m.group(2)), max(spill or [0])))
    assert out, path
    return out


def _demangle(names):
    if not shutil.which("c++filt"):
        return {n: n for n in names}
    res = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    return dict(zip(names, res))


def test_fused_cg_kernels_fit_three_ctas_per_sm():
    ents = _entries("cg_fused")
    dm = _demangle([e[0] for e in ents])
    k1 = [(dm[n], r, s) for n, r, s in ents if "cg_k1_tma<double" in dm[n] and ", 3, " in dm[n]]
    assert k1, "the 3-CTA/SM variants of cg_k1_tma are gone"
    for name, regs, spill in k1:
        assert regs <= 72, (name, regs)                                # 288 threads x 72 regs x 3 CTAs fit the 64K file
        # the single-GPU kernels (MODE 0 plain, 2 Jacobi) hold everything in registers; the row-partitioned variant
        # (MODE 1) may park the few words its in-kernel all-reduce needs
        assert spill == 0 if ("<double, 0, 3" in name or "<double, 2, 3" in name) else spill <= 16, (name, spill)
    for name, regs, spill in [(dm[n], r, s) for n, r, s in ents if "cg_k2<" in dm[n]]:
        assert spill == 0 and regs <= 64, (name, regs, spill)


def test_staged_spmv_family_register_budget():
    for obj, pat in (("spmv", "spmv_tma_kernel<double"), ("fused_phases", "spmv_epi_tma<double"), ("block", "spmm_tma_kernel<double")):
        ents = _entries(obj)
        dm = _demangle([e[0] for e in ents])
        hit = [(dm[n], r, s) for n, r, s in ents if pat in dm[n]]
        assert hit, pat
        for name, regs, spill in hit:
            assert spill <= 16, (name, spill)                          # at most the finaliser's scalars
            assert regs <= 96, (name, regs)                            # >= 2 CTAs of 288 threads per SM
            if "XPlain" in name or "spmm_tma_kernel<double, 8>" in name:
                assert regs <= 72, (name, regs)                        # the single-GPU variants keep 3 CTAs per SM


# The fused passes of each solver family (fused_phases.cu): family -> [(filter on the demangled kernel name,
# {kernel template: instantiations it matches, Float32 and Float64 together}[, foreign])].  The optional foreign field
# is a pair (names set aside or None, pattern): the pattern must not match what remains of any kernel name the filter
# matches, so those kernels carry no other family's functor.
_NOT_LSQ_FUNCTORS = (None, r"kb::(Craig|Cgls|Crls|Lnlq|Car|Minares|Lsq)")
PHASE_KERNELS = {
    "lsq": [(r"kb::(LsqP|LsqrP3|LsmrP3)", {"spmv_epi_tma": 6,        # P1, P2 (LSQR), P2 (LSMR) x Float32 / Float64
                                           "stream_epi": 4})],       # the LSQR and LSMR P3 passes x 2
    "cgls": [(r"kb::(Cgls|Crls)", {"spmv_epi_tma": 8,                # CGLS K1, K3 and CRLS L2, L4 x Float32 / Float64
                                   "spmv_epi_rows": 8,
                                   "stream_epi": 8}),                # CGLS K2, K4 and CRLS L1, L3 x 2
             (r"kb::LslqUpdateBody", {"stream_epi": 2})],            # LSLQ's update pass (P1 / P2 are LSQR's)
    "biorth": [(r"kb::Biorth", {"spmv_epi_tma": 4,                   # B1, B2 x Float32 / Float64
                                "spmv_epi_rows": 4,
                                "stream_epi": 6})],                  # QMR (first / later iterations), BiLQ x 2
    "car_minares": [(r"kb::Car", {"spmv_epi_tma": 4,                 # C2 on a plain or gathered x, x Float32 / Float64
                                  "stream_epi": 4}),                 # C1, C3 x 2
                    (r"kb::Minares", {"spmv_epi_tma": 4,             # M1 on a plain or gathered x, x Float32 / Float64
                                      "stream_epi": 6})],            # M2, M3 and the w-only pass x 2
    # the BiLQR and TriLQR update passes: both halves, primal only, dual only, x Float32 / Float64
    "adjoint_update": [(r"kb::AdjointBilqrBody", {"stream_epi": 6}),
                       (r"kb::AdjointTrilqrBody", {"stream_epi": 6})],
    "adjoint_ssy": [(r"kb::AdjointT[12]", {"spmv_epi_tma": 4,        # TriLQR's T1, T2 x Float32 / Float64
                                           "spmv_epi_rows": 4})],
    "leastnorm": [(r"kb::Craig", {"spmv_epi_tma": 8,                 # CRAIG C1, C2 and CRAIGMR R1, R2 x 2
                                  "spmv_epi_rows": 8,
                                  "stream_epi": 4})],                # CRAIG's x flush and CRAIGMR's R3 x 2
    # L1 on A and L2 on Aᵀ (staged and untiled), the y / w̄ flush and the terminal x pass, x Float32 / Float64
    "lnlq": [(r"kb::Lnlq", {"spmv_epi_tma": 4, "spmv_epi_rows": 4, "stream_epi": 4})],
    "cgne": [(r"kb::Cgne", {"spmv_epi_tma": 4,                       # E1 on A, E2 on Aᵀ, staged and untiled, x 2
                            "spmv_epi_rows": 4,
                            "stream_epi": 0}, _NOT_LSQ_FUNCTORS)],
    "crmr": [(r"kb::Crmr", {"spmv_epi_tma": 4,                       # R1, R3 and the streaming R2, R4, x 2
                            "spmv_epi_rows": 4,
                            "stream_epi": 4}, _NOT_LSQ_FUNCTORS)],
    # one SpMV epilogue on a divided gather (staged and untiled), the streaming update / dot pass and the final
    # normalisation pass, x Float32 / Float64; besides their own Proc* functors the kernels name only shared types
    "processes": [(r"kb::Proc", {"spmv_epi_tma": 2, "spmv_epi_rows": 2, "stream_epi": 4},
                   (r"kb::Proc\w+|kb::NoFin|kb::Csr\b|kb::DistComm", r"kb::[A-Z]"))],
}


def _phase_kernels(pat):
    """(demangled name, registers, spill bytes) of every fused_phases.cu kernel whose name matches pat."""
    ents = _entries("fused_phases")
    if not shutil.which("c++filt"):
        pytest.skip("c++filt not available")
    dm = _demangle([e[0] for e in ents])
    return [(dm[n], r, s) for n, r, s in ents if re.search(pat, dm[n])]


@pytest.mark.parametrize("family", sorted(PHASE_KERNELS))
def test_phase_kernels_fit_three_ctas_per_sm(family):
    """The fused passes keep the 3-CTA/SM budget of the staged SpMV family: every spmv_epi_tma instantiation uses at
    most 72 registers (288 threads x 72 x 3 CTAs fill the 64K register file), and no kernel of the family spills."""
    for pat, counts, *_ in PHASE_KERNELS[family]:
        hit = _phase_kernels(pat)
        for tmpl, count in counts.items():
            assert len([e for e in hit if e[0].startswith(f"void kb::{tmpl}<")]) == count, (pat, tmpl, hit)
        f32 = sorted(e[0].replace("float", "double") for e in hit if "<float" in e[0])
        assert f32 == sorted(e[0] for e in hit if "<double" in e[0]), (pat, hit)     # both precisions, in pairs
        for name, regs, spill in hit:
            assert spill == 0, (name, regs, spill)
            if "spmv_epi_tma<" in name:
                assert regs <= 72, (name, regs)


@pytest.mark.parametrize("family", sorted(f for f, rows in PHASE_KERNELS.items() if any(len(r) > 2 for r in rows)))
def test_phase_kernels_carry_no_foreign_functor(family):
    """The kernels of a row with a foreign field carry no other family's functor, so the instantiation counts that
    other rows pin by name stay theirs."""
    for pat, _, *foreign in PHASE_KERNELS[family]:
        for own, other in foreign:
            for name, _, _ in _phase_kernels(pat):
                assert not re.search(other, re.sub(own, "", name) if own else name), (pat, name)


def test_block_fast_kernels_do_not_spill():
    ents = _entries("block")
    dm = _demangle([e[0] for e in ents])
    fast = [(dm[n], r, s) for n, r, s in ents if "panel_fast_kernel<" in dm[n] and dm[n].rstrip(")").split(",")[5].strip().startswith("false")]
    assert fast
    for name, regs, spill in fast:
        assert spill == 0, (name, regs, spill)                         # the default (non-prefetch) variants


def test_tma_and_mbarrier_instructions_present_in_sass():
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not available")
    for obj in ("cg_fused", "spmv", "fused_phases", "block"):
        path = os.path.join(BUILD, obj + ".o")
        if not os.path.exists(path):
            pytest.skip("objects absent: run __graft_entry__.build()")
        sass = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True).stdout
        assert "UBLKCP" in sass, obj                                   # 1-D bulk TMA copies (cp.async.bulk)
        assert "SYNCS.PHASECHK" in sass or "SYNCS.ARRIVE" in sass, obj  # mbarrier wait / arrive


def _sass_of(obj, mangled_substr):
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


def test_persistent_cg_register_budget_and_coherent_loads():
    """cg_persist: 72 registers (3 CTAs of 288 threads per SM) without spills, and -- because the vectors change
    between the phases of ONE launch -- no vector is read through the non-coherent path (LDG...CONSTANT may only
    appear for the matrix structure / tile order, which are 32-bit loads)."""
    ents = _entries("cg_fused")
    dm = _demangle([e[0] for e in ents])
    hit = [(dm[n], r, s) for n, r, s in ents if re.search(r"cg_persist<double, \d, 3>", dm[n])]      # the 3-CTA/SM variants
    assert len(hit) >= 3
    for name, regs, spill in hit:
        assert regs <= 72 and spill == 0, (name, regs, spill)
    for mode in (0, 1):
        body = _sass_of("cg_fused", f"cg_persistIdLi{mode}ELi3E")
        # row-partitioned variant: the communicator's constants (mailbox pointer, spin budget; dist.cuh) are 64-bit
        # read-only loads, two per barrier -- nothing else may be
        allowed = 0 if mode == 0 else 4
        assert sum("LDG.E.64.CONSTANT" in l for l in body) <= allowed, "a Float64 vector is read through the read-only path"


def test_gather_batches_keep_loads_in_flight():
    """The x gathers of a row must be ISSUED together (clamped indices, spmv_tiles.cuh): in the SASS of the hot
    kernels the longest run of 64-bit global loads with no FP64 instruction in between is at least 6 (round 1's
    guarded gathers compiled to load -> use chains with 2 in flight)."""
    def longest_run(body):
        best = cur = 0
        for l in body:
            if "LDG.E.64" in l and "STRONG" not in l:
                cur += 1
                best = max(best, cur)
            elif "DMUL" in l or "DADD" in l or "DFMA" in l:
                cur = 0
        return best
    assert longest_run(_sass_of("cg_fused", "cg_persistIdLi0ELi3E")) >= 6
    assert longest_run(_sass_of("cg_fused", "cg_persistIdLi1ELi3E")) >= 6       # row-partitioned variant
    assert longest_run(_sass_of("cg_fused", "cg_k1_tmaIdLi0ELi3ELb1")) >= 6
    assert longest_run(_sass_of("spmv", "spmv_tma_kernelIdLb0ENS_6XPlain")) >= 6


def test_block_panel_kernels_use_fp64_tensor_cores():
    """SURVEY 8f-2 / north_star: the tall-skinny panel products of block_gmres! run on the tensor cores --
    mma.sync.m8n8k4.f64 = SASS DMMA in every panel_mma_kernel instantiation (p = 8, 16, 32)."""
    for p in (8, 16, 32):
        body = _sass_of("block", f"panel_mma_kernelILi{p}ELb1ELb1")
        n = sum("DMMA" in l for l in body)
        assert n >= (p // 8) * (p // 4) + 2 * (p // 8) ** 2, (p, n)
    ents = _entries("block")
    dm = _demangle([e[0] for e in ents])
    for name, regs, spill in [(dm[n], r, s) for n, r, s in ents if "panel_mma_kernel<" in dm[n]]:
        assert regs <= 128 and spill <= 96, (name, regs, spill)      # p = 32 fused sits at the 128-register cap of 2 CTAs per SM
