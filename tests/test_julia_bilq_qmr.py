"""CPU, static (no Julia in the image): the bilq! / qmr! methods of the Julia face accept the keyword arguments of the
reference (src/bilq.jl:97-109, src/qmr.jl:104-115) with its defaults, and reach the library through one krylov_solve
per solve."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JL = open(os.path.join(ROOT, "krylov.jl_b200", "julia", "KrylovB200.jl")).read()
HDR = open(os.path.join(ROOT, "include", "krylov_b200.h")).read()
BILQ_KWARGS = {"c", "transfer_to_bicg", "M", "N", "ldiv", "atol", "rtol", "itmax", "timemax", "verbose", "history",
               "callback", "iostream"}


def test_biorth_methods_accept_the_reference_kwargs():
    m = re.search(r"function biorth_solve!\(method::Symbol, ws, A::B200CSR\{T\}, b::B200Vector\{T\};(.*?)\) where T",
                  JL, flags=re.S)
    assert m
    kws = set(re.findall(r"(\w+)(?:::[^=]+?)?\s*=(?!=)", m.group(1)))
    assert kws == BILQ_KWARGS, kws ^ BILQ_KWARGS                   # qmr!'s are the same minus transfer_to_bicg
    for kw in ("atol", "rtol"):
        assert re.search(kw + r"::T = √eps\(T\)", m.group(1)), kw
    assert re.search(r"c::B200Vector\{T\} = b", m.group(1)) and re.search(r"transfer_to_bicg::Bool = true", m.group(1))
    for fn, ws, sym in (("bilq!", "BilqWorkspace", "bilq"), ("qmr!", "QmrWorkspace", "qmr")):
        assert re.search(r"Krylov\." + re.escape(fn) + r"\(ws::Krylov\." + ws + r"\{T,T,B200Vector\{T\}\}, A::B200CSR\{T\}, "
                         r"b::B200Vector\{T\}; kw\.\.\.\) where T =\s*\n\s*biorth_solve!\(:" + sym, JL), fn
    assert ":bilq => 12" in JL and ":qmr => 13" in JL
    body = JL[m.start():JL.index("\nend", m.start())]
    assert body.count("(:krylov_solve, lib)") == 1


def test_transfer_to_bicg_is_the_last_option_field_in_c_and_julia():
    c_fields = re.search(r"typedef struct \{(.*?)\} KrylovB200Options;", HDR, flags=re.S).group(1)
    assert re.findall(r"\b(\w+);", c_fields)[-1] == "transfer_to_bicg"
    jl = re.search(r"struct CExt(.*?)\nend", JL, flags=re.S).group(1)
    assert re.findall(r"(\w+)::", jl)[-1] == "transfer_to_bicg"
