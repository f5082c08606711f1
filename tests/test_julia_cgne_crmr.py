"""CPU, static (no Julia in the image): the cgne! and crmr! methods of the Julia face accept the keyword arguments of
the reference (src/cgne.jl:116-126, src/crmr.jl:114-124) with their defaults, reach the library through one
krylov_solve per solve, and route through their own helper, so that the kwargs of normal_ls_solve! (cgls!, crls!) and
leastnorm_solve! (craig!, craigmr!) stay as they are."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JL = open(os.path.join(ROOT, "krylov.jl_b200", "julia", "KrylovB200.jl")).read()
KWARGS = {"N", "ldiv", "λ", "atol", "rtol", "itmax", "timemax", "verbose", "history", "callback", "iostream"}
SIG = r"function normal_ln_solve!\(method::Symbol, ws, A::B200CSR\{T\}, b::B200Vector\{T\};(.*?)\) where T"


def test_helper_accepts_the_reference_kwargs():
    m = re.search(SIG, JL, flags=re.S)
    assert m
    kws = set(re.findall(r"(\w+)(?:::[^=]+?)?\s*=(?!=)", m.group(1)))
    assert kws == KWARGS, kws ^ KWARGS
    for kw in ("atol", "rtol"):
        assert re.search(kw + r"::T = √eps\(T\)", m.group(1)), kw
    assert re.search(r"λ::T = zero\(T\)", m.group(1)) and re.search(r"N = I", m.group(1))
    assert re.search(r"ldiv::Bool = false", m.group(1)) and re.search(r"itmax::Int = 0", m.group(1))
    assert re.search(r"timemax::Float64 = Inf", m.group(1)) and re.search(r"history::Bool = false", m.group(1))
    body = JL[m.start():JL.index("\nend", m.start())]
    assert body.count("(:krylov_solve, lib)") == 1
    assert "(:krylov_get_x, lib)" in body and "(:krylov_get_y, lib)" not in body
    assert "set_precond!(h, 0, I)" in body and "set_precond!(h, 1, N)" in body


@pytest.mark.parametrize("name,sid", [("cgne", 26), ("crmr", 27)])
def test_methods_route_through_the_helper(name, sid):
    ws = name.capitalize() + "Workspace"
    assert re.search(rf"Krylov\.{name}!\(ws::Krylov\.{ws}\{{T,T,B200Vector\{{T\}},B200Vector\{{T\}}\}}, A::B200CSR\{{T\}}, "
                     rf"b::B200Vector\{{T\}}; kw\.\.\.\) where T =\s*\n\s*normal_ln_solve!\(:{name}, ws, A, b; kw\.\.\.\)", JL)
    assert f":{name} => {sid}" in JL
