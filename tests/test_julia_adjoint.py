"""CPU, static (no Julia in the image): the bilqr! / trilqr! methods of the Julia face accept the keyword arguments of
the reference (src/bilqr.jl:99-107, src/trilqr.jl) with its defaults, reach the library through one krylov_solve per
solve, read y back, and the mirrored KrylovB200Stats carries the adjoint fields in the header's order."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JL = open(os.path.join(ROOT, "krylov.jl_b200", "julia", "KrylovB200.jl")).read()
HDR = open(os.path.join(ROOT, "include", "krylov_b200.h")).read()
KWARGS = {"transfer_to_bicg", "transfer_to_usymcg", "atol", "rtol", "itmax", "timemax", "verbose", "history", "callback",
          "iostream"}


def test_adjoint_methods_accept_the_reference_kwargs():
    m = re.search(r"function adjoint_solve!\(method::Symbol, ws, A::B200CSR\{T\}, b::B200Vector\{T\}, c::B200Vector\{T\};"
                  r"(.*?)\) where T", JL, flags=re.S)
    assert m
    kws = set(re.findall(r"(\w+)(?:::[^=]+?)?\s*=(?!=)", m.group(1)))
    assert kws == KWARGS, kws ^ KWARGS
    for kw in ("atol", "rtol"):
        assert re.search(kw + r"::T = √eps\(T\)", m.group(1)), kw
    assert re.search(r"transfer_to_bicg::Bool = true", m.group(1)) and re.search(r"transfer_to_usymcg::Bool = true", m.group(1))
    assert re.search(r"Krylov\.bilqr!\(ws::Krylov\.BilqrWorkspace\{T,T,B200Vector\{T\}\}, A::B200CSR\{T\}, b::B200Vector\{T\}, "
                     r"c::B200Vector\{T\}; kw\.\.\.\) where T =\s*\n\s*adjoint_solve!\(:bilqr", JL)
    assert re.search(r"Krylov\.trilqr!\(ws::Krylov\.TrilqrWorkspace\{T,T,B200Vector\{T\},B200Vector\{T\}\}, A::B200CSR\{T\}, "
                     r"b::B200Vector\{T\}, c::B200Vector\{T\};\s*kw\.\.\.\) where T =\s*\n\s*adjoint_solve!\(:trilqr", JL)
    assert ":trilqr => 18" in JL and ":bilqr => 19" in JL
    body = JL[m.start():JL.index("\nend", m.start())]
    assert body.count("(:krylov_solve, lib)") == 1
    assert "(:krylov_get_y, lib)" in body and "(:krylov_warm_start2, lib)" in body


def test_stats_mirror_ends_with_the_adjoint_fields():
    body = re.search(r"typedef struct \{((?:(?!typedef).)*?)\} KrylovB200Stats;", HDR, flags=re.S).group(1)
    c_fields = re.findall(r"\b(\w+)(?:\[\d+\])?;", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert c_fields[-4:] == ["nerr_ubnds_cg", "solved_primal", "solved_dual", "nresiduals_dual"], c_fields
    jl = re.findall(r"(\w+)::", re.search(r"struct CStats(.*?)\nend", JL, flags=re.S).group(1))
    assert jl[-4:] == c_fields[-4:] and len(jl) == len(c_fields), (jl, c_fields)
