"""CPU, static (no Julia in the image): the Krylov-process methods of the Julia face take the reference's positional
arguments and keywords with their defaults (src/krylov_processes.jl:28, 133, 250, 323, 431), reach the library through
exactly one `kb200_<process>` call each, and return the reference's tuple with B200Matrix bases and the coefficient
patterns of krylov_processes.jl."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JL = open(os.path.join(ROOT, "krylov.jl_b200", "julia", "KrylovB200.jl")).read()

CASES = {  # name -> (positional arguments, keywords, returned tuple, coefficient pattern)
    "hermitian_lanczos": ("A::B200CSR{T}, b::B200Vector{T}, k::Int", {"allow_breakdown", "reorthogonalization"},
                          "V, T(β[]), SparseMatrixCSC(k+1, k, colptr, rowval, T.(nz))", "tridiagonal_pattern"),
    "arnoldi": ("A::B200CSR{T}, b::B200Vector{T}, k::Int", {"allow_breakdown", "reorthogonalization"}, "V, T(β[]), T.(H)", None),
    "golub_kahan": ("A::B200CSR{T}, b::B200Vector{T}, k::Int", {"allow_breakdown"},
                    "V, U, T(β[]), SparseMatrixCSC(k+1, k+1, colptr, rowval, T.(nz))", "bidiagonal_pattern"),
    "nonhermitian_lanczos": ("A::B200CSR{T}, b::B200Vector{T}, c::B200Vector{T}, k::Int", {"allow_breakdown"},
                             "V, T(β[]), SparseMatrixCSC(k+1, k, colptr, rowval, T.(nzT)), U, T(γ[])", "tridiagonal_pattern"),
    "saunders_simon_yip": ("A::B200CSR{T}, b::B200Vector{T}, c::B200Vector{T}, k::Int", {"allow_breakdown"},
                           "V, T(β[]), SparseMatrixCSC(k+1, k, colptr, rowval, T.(nzT)), U, T(γ[])", "tridiagonal_pattern"),
}


def _method(name):
    m = re.search(rf"function Krylov\.{name}\((.*?);(.*?)\) where T<:BlasT\n", JL, flags=re.S)
    assert m, name
    body = JL[m.end():JL.index("\nend\n", m.end())]
    return " ".join(m.group(1).split()), m.group(2), body


@pytest.mark.parametrize("name", sorted(CASES))
def test_reference_arguments_and_keywords(name):
    args, kws, body = _method(name)
    want_args, want_kws, _, _ = CASES[name]
    assert args == want_args
    got = dict(re.findall(r"(\w+)::Bool\s*=\s*(\w+)", kws))
    assert set(got) == want_kws and set(got.values()) == {"false"}, got


@pytest.mark.parametrize("name", sorted(CASES))
def test_one_library_call_and_the_reference_outputs(name):
    _, kws, body = _method(name)
    _, _, ret, pattern = CASES[name]
    assert body.count("ccall((:kb200_") == 1 and f"ccall((:kb200_{name}, lib)" in body
    assert f'"{name}")' in body                                # the error carries the reference's message
    assert "B200Matrix{T}(undef" in body
    flags = "proc_flags(allow_breakdown, reorthogonalization)" if "reorthogonalization" in kws else "proc_flags(allow_breakdown)"
    assert flags in body
    assert "return " + ret in " ".join(body.split())
    if pattern:
        assert f"{pattern}(k)" in body


def test_patterns_restate_the_reference():
    tri = JL[JL.index("function tridiagonal_pattern"):]
    tri = tri[:tri.index("\nend\n")]
    assert "colptr[i+1] = 3i" in tri and "rowval[pos] = i-1; rowval[pos+1] = i; rowval[pos+2] = i+1" in tri
    bi = JL[JL.index("function bidiagonal_pattern"):]
    bi = bi[:bi.index("\nend\n")]
    assert "colptr[i+1] = pos + 2; rowval[pos] = i; rowval[pos+1] = i+1" in bi and "colptr[i+1] = pos + 1; rowval[pos] = i" in bi
