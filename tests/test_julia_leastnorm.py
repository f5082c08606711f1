"""CPU, static (no Julia in the image): the craig! / craigmr! methods of the Julia face accept the keyword arguments of
the reference (src/craig.jl:151-166, src/craigmr.jl:141-153) with its defaults, reach the library through one
krylov_solve per solve and read y back with krylov_get_y."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JL = open(os.path.join(ROOT, "krylov.jl_b200", "julia", "KrylovB200.jl")).read()
KWARGS = {"M", "N", "ldiv", "transfer_to_lsqr", "sqd", "λ", "btol", "conlim", "atol", "rtol", "itmax", "timemax",
          "verbose", "history", "callback", "iostream"}


def test_leastnorm_methods_accept_the_reference_kwargs():
    m = re.search(r"function leastnorm_solve!\(method::Symbol, ws, A::B200CSR\{T\}, b::B200Vector\{T\};(.*?)\) where T",
                  JL, flags=re.S)
    assert m
    kws = set(re.findall(r"(\w+)(?:::[^=]+?)?\s*=(?!=)", m.group(1)))
    assert kws == KWARGS, kws ^ KWARGS
    for kw in ("atol", "rtol", "btol"):
        assert re.search(kw + r"::T = √eps\(T\)", m.group(1)), kw
    assert re.search(r"conlim::T = 1/√eps\(T\)", m.group(1))
    assert re.search(r"transfer_to_lsqr::Bool = false", m.group(1)) and re.search(r"sqd::Bool = false", m.group(1))
    for solver, ws in (("craig", "CraigWorkspace"), ("craigmr", "CraigmrWorkspace")):
        assert re.search(rf"Krylov\.{solver}!\(ws::Krylov\.{ws}\{{T,T,B200Vector\{{T\}},B200Vector\{{T\}}\}}, A::B200CSR\{{T\}}, "
                         rf"b::B200Vector\{{T\}}; kw\.\.\.\) where T =\s*\n\s*leastnorm_solve!\(:{solver}", JL), solver
    assert ":craig => 28" in JL and ":craigmr => 29" in JL
    body = JL[m.start():JL.index("\nend", m.start())]
    assert body.count("(:krylov_solve, lib)") == 1
    assert "(:krylov_get_y, lib)" in body and "(:krylov_get_x, lib)" in body
    assert 'error("sqd cannot be set to true if λ ≠ 0 !")' in body
