"""CPU, static (no Julia in the image): the lsqr! / lsmr! methods of the Julia face accept every keyword argument of
the reference (src/lsqr.jl:145-162, src/lsmr.jl:149-166) and reach the library through one krylov_solve per solve;
rectangular SparseMatrixCSC operators are uploaded through kb200_csr_create_rect.  The ccall signatures themselves are
checked against the header by tests/test_julia_binding.py."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JL = open(os.path.join(ROOT, "krylov.jl_b200", "julia", "KrylovB200.jl")).read()
REFERENCE_KWARGS = ("M", "N", "ldiv", "sqd", "λ", "radius", "etol", "axtol", "btol", "conlim", "atol", "rtol", "itmax",
                    "timemax", "verbose", "history", "callback", "iostream")


def test_ls_methods_accept_the_reference_kwargs():
    m = re.search(r"function ls_solve!\(method::Symbol, ws, A::B200CSR\{T\}, b::B200Vector\{T\};(.*?)\) where T", JL, flags=re.S)
    assert m
    kws = set(re.findall(r"(\w+|λ)(?:::[^=]+?)?\s*=(?!=)", m.group(1)))
    for kw in REFERENCE_KWARGS:
        assert kw in kws, kw
    # atol / rtol default to zero as in Julia (not the C ABI's sqrt(eps))
    assert re.search(r"atol::T = zero\(T\)", m.group(1)) and re.search(r"rtol::T = zero\(T\)", m.group(1))
    for fn, ws, sym in (("lsqr!", "LsqrWorkspace", "lsqr"), ("lsmr!", "LsmrWorkspace", "lsmr")):
        assert re.search(r"Krylov\." + re.escape(fn) + r"\(ws::Krylov\." + ws + r"\{T,T,B200Vector\{T\},B200Vector\{T\}\}, A::B200CSR\{T\}, "
                         r"b::B200Vector\{T\}; kw\.\.\.\) where T =\s*\n\s*ls_solve!\(:" + sym, JL), fn
    assert ":lsqr => 21" in JL and ":lsmr => 22" in JL


def test_rectangular_csr_upload():
    assert "(:kb200_csr_create_rect, lib)" in JL
    body = re.search(r"function rect_csr\(A::SparseMatrixCSC\{T,Int64\}\) where T<:BlasT(.*?)\nend", JL, flags=re.S).group(1)
    assert "A.colptr, A.rowval, A.nzval" in body and "adjoint(At)" in body     # CSC(A) = CSR(A^T): one transpose
