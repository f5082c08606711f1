"""CPU, static (no Julia in the image): the cgls! / crls! methods of the Julia face accept exactly the keyword arguments
of the reference (src/cgls.jl:110-121, src/crls.jl:101-112) with its defaults, and reach the library through one
krylov_solve per solve."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JL = open(os.path.join(ROOT, "krylov.jl_b200", "julia", "KrylovB200.jl")).read()
REFERENCE_KWARGS = {"M", "ldiv", "radius", "λ", "atol", "rtol", "itmax", "timemax", "verbose", "history", "callback",
                    "iostream"}


def test_normal_ls_methods_accept_the_reference_kwargs():
    m = re.search(r"function normal_ls_solve!\(method::Symbol, ws, A::B200CSR\{T\}, b::B200Vector\{T\};(.*?)\) where T",
                  JL, flags=re.S)
    assert m
    kws = set(re.findall(r"(\w+|λ)(?:::[^=]+?)?\s*=(?!=)", m.group(1)))
    assert kws == REFERENCE_KWARGS, kws ^ REFERENCE_KWARGS
    # atol / rtol default to √eps(T) as in cgls.jl / crls.jl (unlike lsqr!'s zero)
    assert re.search(r"atol::T = √eps\(T\)", m.group(1)) and re.search(r"rtol::T = √eps\(T\)", m.group(1))
    assert re.search(r"radius::T = zero\(T\)", m.group(1)) and re.search(r"λ::T = zero\(T\)", m.group(1))
    for fn, ws, sym in (("cgls!", "CglsWorkspace", "cgls"), ("crls!", "CrlsWorkspace", "crls")):
        assert re.search(r"Krylov\." + re.escape(fn) + r"\(ws::Krylov\." + ws + r"\{T,T,B200Vector\{T\},B200Vector\{T\}\}, A::B200CSR\{T\}, "
                         r"b::B200Vector\{T\}; kw\.\.\.\) where T =\s*\n\s*normal_ls_solve!\(:" + sym, JL), fn
    assert ":cgls => 24" in JL and ":crls => 25" in JL
    body = JL[m.start():JL.index("\nend", m.start())]
    assert body.count("(:krylov_solve, lib)") == 1


LSLQ_KWARGS = {"M", "N", "ldiv", "transfer_to_lsqr", "sqd", "λ", "σ", "etol", "utol", "btol", "conlim", "atol", "rtol",
               "itmax", "timemax", "verbose", "history", "callback", "iostream"}


def test_lslq_method_accepts_the_reference_kwargs():
    m = re.search(r"function lslq_solve!\(ws, A::B200CSR\{T\}, b::B200Vector\{T\};(.*?)\) where T", JL, flags=re.S)
    assert m
    kws = set(re.findall(r"(\w+|λ|σ)(?:::[^=]+?)?\s*=(?!=)", m.group(1)))
    assert kws == LSLQ_KWARGS, kws ^ LSLQ_KWARGS
    for kw in ("atol", "rtol", "etol", "utol", "btol"):                 # lslq.jl:186-191: all √eps(T)
        assert re.search(kw + r"::T = √eps\(T\)", m.group(1)), kw
    assert re.search(r"Krylov\.lslq!\(ws::Krylov\.LslqWorkspace\{T,T,B200Vector\{T\},B200Vector\{T\}\}, A::B200CSR\{T\}, "
                     r"b::B200Vector\{T\}; kw\.\.\.\) where T =\s*\n\s*lslq_solve!\(ws", JL)
    assert ":lslq => 20" in JL
    body = JL[m.start():JL.index("\nend", m.start())]
    assert body.count("(:krylov_solve, lib)") == 1
