"""CPU, static (no Julia in the image): the lnlq! method of the Julia face accepts the keyword arguments of the
reference (src/lnlq.jl:144-160) with its defaults, reaches the library through one krylov_solve per solve and reads y
back with krylov_get_y."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JL = open(os.path.join(ROOT, "krylov.jl_b200", "julia", "KrylovB200.jl")).read()
KWARGS = {"M", "N", "ldiv", "transfer_to_craig", "sqd", "λ", "σ", "utolx", "utoly", "atol", "rtol", "itmax", "timemax",
          "verbose", "history", "callback", "iostream"}


def test_lnlq_method_accepts_the_reference_kwargs():
    m = re.search(r"function lnlq_solve!\(ws, A::B200CSR\{T\}, b::B200Vector\{T\};(.*?)\) where T", JL, flags=re.S)
    assert m
    kws = set(re.findall(r"(\w+)(?:::[^=]+?)?\s*=(?!=)", m.group(1)))
    assert kws == KWARGS, kws ^ KWARGS
    for kw in ("utolx", "utoly", "atol", "rtol"):
        assert re.search(kw + r"::T = √eps\(T\)", m.group(1)), kw
    for kw in ("λ", "σ"):
        assert re.search(kw + r"::T = zero\(T\)", m.group(1)), kw
    assert re.search(r"transfer_to_craig::Bool = true", m.group(1)) and re.search(r"sqd::Bool = false", m.group(1))
    assert re.search(r"ldiv::Bool = false", m.group(1)) and re.search(r"itmax::Int = 0", m.group(1))
    assert re.search(r"timemax::Float64 = Inf", m.group(1))
    assert re.search(r"Krylov\.lnlq!\(ws::Krylov\.LnlqWorkspace\{T,T,B200Vector\{T\},B200Vector\{T\}\}, A::B200CSR\{T\}, "
                     r"b::B200Vector\{T\}; kw\.\.\.\) where T =\s*\n\s*lnlq_solve!\(ws, A, b; kw\.\.\.\)", JL)
    assert ":lnlq => 30" in JL
    body = JL[m.start():JL.index("\nend", m.start())]
    assert body.count("(:krylov_solve, lib)") == 1
    assert "(:krylov_get_y, lib)" in body and "(:krylov_get_x, lib)" in body
    assert 'error("sqd cannot be set to true if λ ≠ 0 !")' in body
    assert "handle_for(:lnlq" in body


def test_lnlq_stats_read_both_bound_histories():
    assert "(3, :error_bnd_x, s.nerr_lbnds)" in JL and "(4, :error_bnd_y, s.nerr_ubnds_lq)" in JL
