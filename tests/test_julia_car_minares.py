"""CPU, static (no Julia in the image): the car! / minares! methods of the Julia face accept the keyword arguments of
the reference (src/car.jl:90-99, src/minares.jl:93-104) with their defaults, reach the library through fused_solve!
(one krylov_solve per solve), and MINARES's Artol reaches the axtol field of the extended options."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JL = open(os.path.join(ROOT, "krylov.jl_b200", "julia", "KrylovB200.jl")).read()
CAR_KWARGS = {"M", "ldiv", "atol", "rtol", "itmax", "timemax", "verbose", "history", "callback", "iostream"}
MINARES_KWARGS = CAR_KWARGS | {"λ", "Artol"}


def _fused_solve_kwargs():
    m = re.search(r"function fused_solve!\(method::Symbol, ws, A::B200CSR\{T\}, b::B200Vector\{T\};(.*?)\) where T", JL,
                  flags=re.S)
    assert m
    return m, set(re.findall(r"(\w+|λ)(?:::[^=]+?)?\s*=(?!=)", m.group(1)))


def test_car_and_minares_methods_accept_the_reference_kwargs():
    m, kws = _fused_solve_kwargs()
    assert MINARES_KWARGS <= kws, MINARES_KWARGS - kws
    for kw in ("atol", "rtol", "Artol"):
        assert re.search(kw + r"::T = √eps\(T\)", m.group(1)), kw
    assert re.search(r"λ::T = zero\(T\)", m.group(1)) and re.search(r"itmax::Int = 0", m.group(1))
    for fn, ws, sym in (("car!", "CarWorkspace", "car"), ("minares!", "MinaresWorkspace", "minares")):
        assert f"(:{fn}, :{ws}, :{sym}, :(0))" in JL, fn
    assert re.search(r"Krylov\.\$fn\(ws::Krylov\.\$WS\{T,T,B200Vector\{T\}\}, A::B200CSR\{T\}, b::B200Vector\{T\}; kw\.\.\.\) "
                     r"where T =\s*\n\s*fused_solve!\(", JL)
    assert ":car => 32" in JL and ":minares => 33" in JL
    body = JL[m.start():JL.index("\nend", m.start())]
    assert body.count("(:krylov_solve, lib)") == 1


def test_artol_fills_the_axtol_field():
    m, _ = _fused_solve_kwargs()
    body = JL[m.start():JL.index("\nend", m.start())]
    call = re.search(r"CExt\((.*?)\)\)", body, flags=re.S).group(1)
    args = [a.strip() for a in re.sub(r"\([^()]*\)", "", call).split(",")]   # arguments, nested calls collapsed
    fields = re.findall(r"(\w+)::", re.search(r"struct CExt(.*?)\nend", JL, flags=re.S).group(1))
    assert args[fields.index("axtol")] == "Artol"
