"""CPU checks of the shift solvers' binding (krylov_b200: CgLanczosShiftWorkspace, CglsLanczosShiftWorkspace and their
solver functions) with the library replaced by a recorder, as tests/test_binding_keywords.py does for the single-RHS
solvers: each keyword reaches its option field, unknown keywords are refused, host callables get the right lengths.
Then the Julia methods' keywords, statically, against the reference's def_kwargs."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest
import scipy.sparse as sp

import krylov_b200 as kb
from krylov_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JL = open(os.path.join(ROOT, "krylov.jl_b200", "julia", "KrylovB200.jl")).read()

# def_kwargs_cg_lanczos_shift (src/cg_lanczos_shift.jl:89-99) and def_kwargs_cgls_lanczos_shift
# (src/cgls_lanczos_shift.jl:91-100), written out
REFERENCE_KW = {
    "cg_lanczos_shift": ("M", "ldiv", "check_curvature", "atol", "rtol", "itmax", "timemax", "verbose", "history",
                         "callback", "iostream"),
    "cgls_lanczos_shift": ("M", "ldiv", "atol", "rtol", "itmax", "timemax", "verbose", "history", "callback", "iostream"),
}
O, E = "KrylovOptions", "KrylovB200Options"
FIELDS = {   # keyword: (struct, field, a value other than the default, what the field then holds)
    "atol": (O, "atol", 1e-3, 1e-3), "rtol": (O, "rtol", 1e-4, 1e-4), "itmax": (O, "itmax", 17, 17),
    "timemax": (O, "timemax", 2.5, 2.5), "verbose": (O, "verbose", 3, 3), "history": (E, "history", True, 1),
    "fused": (E, "fused", False, 0), "ldiv": (E, "ldiv", True, 1), "check_curvature": (E, "check_curvature", True, 1),
    "callback": (E, "callback", lambda ws: False, True),
}
SHAPES = {"cg_lanczos_shift": (5, 5), "cgls_lanczos_shift": (7, 4)}


def fields(struct):
    out = {}
    for name, _ in struct._fields_:
        v = getattr(struct, name)
        if name == "callback":
            v = bool(v)
        elif isinstance(v, float) and math.isnan(v):
            v = "nan"
        out[(type(struct).__name__, name)] = v
    return out


class Recorder:
    """Stands in for libkrylov_b200: forwards the default-option constructors, answers every other call with 0, and
    records what krylov_b200_shift_solve receives: the option structs, the shifts and the operator lengths."""

    FORWARD = ("krylov_default_options", "krylov_b200_default_options")

    def __init__(self, real):
        self.real, self.solves, self.ext, self.seen = real, [], None, []

    def __getattr__(self, name):
        if name in self.FORWARD:
            return getattr(self.real, name)

        def call(*args):
            if name == "krylov_b200_shift_workspace_create":
                args[-1]._obj.value = 0x1000
            elif name == "krylov_b200_set_options":
                self.ext = fields(args[1]._obj)
            elif name == "krylov_b200_shift_solve":
                lengths = []
                for f in args[1:4]:
                    if not f:
                        lengths.append(None)
                        continue
                    x, y = (C.c_double * 64)(), (C.c_ubyte * 512)(*([0xFF] * 512))
                    f(C.cast(x, C.c_void_p), C.cast(y, C.c_void_p), None)
                    lengths.append((self.seen.pop(), sum(v != 0xFF for v in bytes(y)) // 8))
                self.solves.append(dict(options={**fields(args[-1]._obj), **self.ext}, ops=lengths, shifts=list(args[5])))
            return 0
        return call

    def probe(self, x):
        self.seen.append(len(x))
        return 1.0


@pytest.fixture
def rec(monkeypatch):
    r = Recorder(_lib.lib())
    monkeypatch.setattr(kb, "lib", lambda: r)
    monkeypatch.setattr(_lib, "lib", lambda: r)
    return r


def problem(name):
    m, n = SHAPES[name]
    return sp.csr_matrix(np.eye(m, n) * 4.0 + np.eye(m, n, 1)), np.ones(m)


@pytest.mark.parametrize("name", list(SHAPES))
def test_each_keyword_reaches_its_field(rec, name):
    A, b = problem(name)
    kb.__dict__[name](A, b, [1.0, 2.0])
    base = rec.solves[-1]["options"]
    assert rec.solves[-1]["shifts"][:2] == [1.0, 2.0]
    taken = [k for k in FIELDS if k != "check_curvature" or name == "cg_lanczos_shift"]
    for kw in taken:
        struct, fld, val, held = FIELDS[kw]
        kb.__dict__[name](A, b, [1.0, 2.0], **{kw: val})
        got = rec.solves[-1]["options"]
        assert got[(struct, fld)] == held, (kw, got[(struct, fld)])
        assert {k: v for k, v in got.items() if k != (struct, fld)} == {k: v for k, v in base.items() if k != (struct, fld)}, kw


@pytest.mark.parametrize("name", list(SHAPES))
def test_unknown_keywords_are_refused(rec, name):
    A, b = problem(name)
    bad = ["radius", "lambda_", "memory", "N"] + (["check_curvature"] if name == "cgls_lanczos_shift" else [])
    for kw in bad:
        with pytest.raises(kb.B200Error, match=rf"{name}!: unsupported keyword argument\(s\) {kw}"):
            kb.__dict__[name](A, b, [1.0], **{kw: 1})
    ws = kb.__dict__["CgLanczosShiftWorkspace" if name == "cg_lanczos_shift" else "CglsLanczosShiftWorkspace"](*SHAPES[name], 1)
    with pytest.raises(kb.B200Error, match="unsupported keyword"):
        kb.__dict__[name + "_"](ws, A, b, [1.0], restart=True)
    with pytest.raises(kb.B200Error, match="inconsistent with length"):
        kb.__dict__[name + "_"](ws, A, b, [1.0, 2.0])


def test_host_callables_get_their_lengths(rec):
    m, n = SHAPES["cg_lanczos_shift"]
    kb.cg_lanczos_shift(rec.probe, np.ones(m), [1.0], M=rec.probe)
    assert rec.solves[-1]["ops"] == [(n, n), None, (n, n)]
    m, n = SHAPES["cgls_lanczos_shift"]
    kb.cgls_lanczos_shift((rec.probe, rec.probe), np.ones(m), [1.0], n=n)
    assert rec.solves[-1]["ops"] == [(n, m), (m, n), None]


def test_cgls_refuses_M_before_the_library(rec):
    A, b = problem("cgls_lanczos_shift")
    with pytest.raises(kb.B200Error, match="Preconditioner `M` is not supported."):
        kb.cgls_lanczos_shift(A, b, [1.0], M=np.ones(A.shape[0]))


def test_shift_solvers_stay_outside_the_single_solver_tables():
    assert "cg_lanczos_shift" not in _lib.SOLVER_IDS and "cgls_lanczos_shift" not in _lib.SOLVER_IDS
    assert "cg_lanczos_shift" not in kb._SOLVERS and "cgls_lanczos_shift" not in kb._SOLVERS
    for sym in ("krylov_b200_shift_workspace_create", "krylov_b200_shift_workspace_free", "krylov_b200_shift_solve",
                "krylov_b200_shift_get_x", "krylov_b200_shift_get_stats", "krylov_b200_shift_get_history"):
        assert sym in _lib.SIGNATURES, sym


@pytest.mark.parametrize("name", list(REFERENCE_KW))
def test_julia_methods_take_the_reference_keywords(name):
    m = re.search(r"function Krylov\." + name + r"!\(ws::.*?;(.*?)\) where T", JL, flags=re.S)
    assert m, name
    kws = set(re.findall(r"(\w+)(?:::[^=]+?)?\s*=(?!=)", m.group(1)))
    assert kws == set(REFERENCE_KW[name]), (name, kws ^ set(REFERENCE_KW[name]))
    assert JL.count("(:krylov_workspace_create, lib)") == 1           # the shift methods use their own create
    assert "(:krylov_b200_shift_workspace_create, lib)" in JL and "HANDLES[ws] = h" in JL
