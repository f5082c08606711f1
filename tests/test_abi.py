"""CPU-side checks of the C ABI: the shared object loads, exports every symbol
include/krylov_b200.h declares, and the GPU-free entry points behave like the
reference's (interfaces/test/C/test_api.c:105-139,175-182)."""
import ctypes as C
import math
import os
import re

import pytest

from krylov_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "krylov_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    names = re.findall(r"\b((?:krylov|kb200)_[a-z0-9_A-Z]+)\s*\(", src)
    return sorted(set(names))


def test_header_symbols_are_exported_and_bound():
    L = _lib.lib()
    names = declared_symbols()
    assert len(names) >= 50
    for n in names:
        assert hasattr(L, n), f"{n} declared in the header but not exported"
        assert n in _lib.SIGNATURES, f"{n} has no ctypes signature"


def test_signature_argument_counts_match_header():
    """Each ctypes signature takes as many arguments as the header's prototype (the kernel test entry points
    kb200_spmm_csr, krylov_b200_block_panel_op, the block-Jacobi kernels and the fused vector primitives among
    them)."""
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "krylov_b200.h")).read(), flags=re.S)
    protos = dict(re.findall(r"\b((?:krylov|kb200)_[a-z0-9_A-Z]+)\s*\(([^()]*)\)\s*;", src))
    for name in ("kb200_spmm_csr", "krylov_b200_block_panel_op", "kb200_spmv_csr", "kb200_blockdiag_mul",
                 "kb200_blockdiag_invert", "kb200_dot2", "kb200_cg_prologue", "kb200_diagmul"):
        assert name in protos
    for name, params in protos.items():
        params = params.strip()
        n = 0 if params in ("", "void") else params.count(",") + 1
        assert len(_lib.SIGNATURES[name][1]) == n, name


def test_default_option_sentinels():               # test_api.c:105-118
    L = _lib.lib()
    o = L.krylov_default_options()
    assert math.isnan(o.atol) and math.isnan(o.rtol) and o.itmax == 0 and o.verbose == 0 and o.lambda_ == 0.0
    assert math.isnan(o.timemax) and o.radius == 0.0 and o.restart == 0 and o.linesearch == 0
    w = L.krylov_default_workspace_options()
    assert w.memory == 0 and w.window == 0
    e = L.krylov_b200_default_options()
    assert e.fused == 1 and e.history == 0 and math.isnan(e.etol)


def test_struct_layouts_match_reference():         # interfaces/src/c_enums.jl:30-62
    assert C.sizeof(_lib.KrylovWorkspaceOptions) == 8
    assert C.sizeof(_lib.KrylovOptions) == 80
    offs = {f: getattr(_lib.KrylovOptions, f).offset for f, _ in _lib.KrylovOptions._fields_}
    assert offs == dict(atol=0, rtol=8, itmax=16, verbose=20, lambda_=24, tau=32, nu=40, timemax=48, radius=56,
                        restart=64, reorthogonalization=68, linesearch=72)


def test_version():                                # test_api.c:120-129
    L = _lib.lib()
    a, b, c = C.c_int(-1), C.c_int(-1), C.c_int(-1)
    L.krylov_get_version(C.byref(a), C.byref(b), C.byref(c))
    assert (a.value, b.value, c.value) == (0, 10, 8)


def test_unknown_solver_and_bad_handles():         # test_api.c:131-139, 175-182
    L = _lib.lib()
    ws = C.c_void_p()
    assert L.krylov_workspace_create(999, 4, 4, 1, 0, None, C.byref(ws)) == -2 and not ws.value
    assert L.krylov_workspace_create(_lib.KRYLOV_CG, 4, 4, 2, 0, None, C.byref(ws)) == -2      # complex: outside the path
    assert L.krylov_workspace_create(2, 4, 4, 1, 0, None, C.byref(ws)) == -2                   # SYMMLQ: outside the path
    bogus = C.c_void_p(0x1234)
    assert L.krylov_workspace_free(bogus) == 1
    assert L.krylov_is_solved(bogus) == -1 and L.krylov_niter(bogus) == -1 and L.krylov_elapsed_time(bogus) == -1.0
    assert L.krylov_block_workspace_create(1, 4, 4, 2, 1, 0, None, C.byref(ws)) == -2          # block_minres: outside the path
    assert L.krylov_block_workspace_create(0, 4, 4, 2, 2, 0, None, C.byref(ws)) == -2          # complex block_gmres
    assert L.krylov_block_workspace_free(bogus) == 1 and L.krylov_block_is_solved(bogus) == -1


def test_no_cpu_fallback_without_gpu():
    L = _lib.lib()
    if L.krylov_b200_device_count() > 0:
        pytest.skip("a GPU is present")
    ws = C.c_void_p()
    assert L.krylov_workspace_create(_lib.KRYLOV_CG, 4, 4, 1, 0, None, C.byref(ws)) == -1
    assert not ws.value
    assert "no usable CUDA device" in _lib.last_error()


def test_fortran_interface_names_are_exported():
    """interfaces/include/krylov.f90 binds these C names (bind(c, name='...')): a Fortran caller of the reference links
    against libkrylov_b200.so with the reference's own module, unchanged (SURVEY.md 8f-4, Fortran header parity).
    No Fortran compiler exists in this image, so only the symbol contract is checked."""
    names = """krylov_block_elapsed_time krylov_block_get_X krylov_block_is_solved krylov_block_niter krylov_block_solve
               krylov_block_warm_start krylov_block_workspace_create krylov_block_workspace_free krylov_default_options
               krylov_default_workspace_options krylov_elapsed_time krylov_get_version krylov_get_x krylov_get_y
               krylov_is_solved krylov_niter krylov_solve krylov_warm_start krylov_warm_start2 krylov_workspace_create
               krylov_workspace_free""".split()
    L = C.CDLL(_lib.SO_PATH)
    for n in names:
        assert hasattr(L, n), n
