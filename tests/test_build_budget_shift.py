"""CPU: the shift solvers' fused passes (fused_phases.cu: kb::Shift*), counted by instantiation in both precisions, with
their register budgets, read from the build's `-Xptxas -v` log like tests/test_build_budget.py."""
import re

from test_build_budget import _demangle, _entries

# kernel template -> instantiations carrying a kb::Shift functor, Float32 and Float64 together
SHIFT_KERNELS = {
    "stream_epi": 4,        # the shift update (ShiftUpdBody) and CGLS-Lanczos-shift's u pass (ShiftGkUBody) x 2
    "spmv_epi_tma": 8,      # u_next = A v and v = A^T u_next, on a plain or gathered x, x 2
    "spmv_epi_rows": 8,     # the same on untiled operators
}


def _shift_kernels():
    ents = _entries("fused_phases")
    dm = _demangle([e[0] for e in ents])
    return [(dm[n], r, s) for n, r, s in ents if re.search(r"kb::Shift", dm[n])]


def test_shift_passes_by_instantiation():
    hits = _shift_kernels()
    for kernel, count in SHIFT_KERNELS.items():
        mine = [h for h in hits if h[0].startswith(f"void kb::{kernel}<")]
        assert len(mine) == count, (kernel, [h[0][:120] for h in mine])
        for dtype in ("float", "double"):
            assert any(f"kb::{kernel}<{dtype}," in h[0] for h in mine), (kernel, dtype)
    assert len(hits) == sum(SHIFT_KERNELS.values())


def test_shift_passes_fit_their_budget():
    for name, regs, spill in _shift_kernels():
        assert spill == 0, (name, spill)
        if name.startswith("void kb::spmv_epi_tma<"):
            assert regs <= 72, (name, regs)          # 3 CTAs of 288 threads per SM
        else:
            assert regs <= 64, (name, regs)


def test_shift_functors_carry_no_other_family():
    for name, _, _ in _shift_kernels():
        rest = re.sub(r"kb::Shift\w*", "", name)
        assert not re.search(r"kb::(Cgls|Crls|Lsq|Biorth|Car|Minares|Adjoint|Craig|Lnlq|Cgne|Crmr|Proc|Lan)", rest), name
