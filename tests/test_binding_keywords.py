"""CPU checks of the Python binding's solve path (krylov_b200/__init__.py): which keywords every solver takes, which
option field each one reaches, how host callables are sized, and what the out-of-place forms return.

The library is replaced by a recorder, so this needs the built shared object (for the default option structs) but no
GPU.  The table below is written from the solvers' signatures (the reference's keywords and defaults); it does not
read the binding's own table."""
import ctypes as C
import math

import numpy as np
import pytest
import scipy.sparse as sp

import krylov_b200 as kb
from krylov_b200 import _lib

COMMON = ("atol", "rtol", "itmax", "timemax", "verbose", "history", "callback", "fused")
SQUARE = ("c", "M", "N", "ldiv", "radius", "linesearch", "lambda_", "etol", "conlim", "restart", "reorthogonalization",
          "batch", "time_kernels", "check_curvature", "gamma", "artol")
LSQ = ("M", "N", "ldiv", "sqd", "lambda_", "radius", "etol", "axtol", "btol", "conlim")
NORMAL = ("M", "ldiv", "radius", "lambda_")
BIORTH = ("c", "M", "N", "ldiv")
LEASTNORM = ("M", "N", "ldiv", "sqd", "lambda_")
SQ, TALL, WIDE = (5, 5), (7, 4), (4, 7)
ADJOINT = ("bilqr", "trilqr")        # c is their third positional argument

# solver: ((m, n), keywords besides COMMON, {host-callable M / N: its length}, applies A^T, what the out-of-place form
# returns, the statistics type)
SOLVERS = {
    **{s: (SQ, SQUARE, {"M": 5, "N": 5}, False, "x", kb.SimpleStats)
       for s in ("cg", "cr", "minres", "diom", "fom", "dqgmres", "gmres", "fgmres", "bicgstab", "cgs", "cg_lanczos")},
    "car": (SQ, ("M", "ldiv"), {"M": 5}, False, "x", kb.SimpleStats),
    "minares": (SQ, ("M", "ldiv", "lambda_", "artol"), {"M": 5}, False, "x", kb.SimpleStats),
    "lsqr": (TALL, LSQ, {"M": 7, "N": 4}, True, "x", kb.SimpleStats),
    "lsmr": (TALL, LSQ, {"M": 7, "N": 4}, True, "x", kb.SimpleStats),
    "lslq": (TALL, ("M", "N", "ldiv", "transfer_to_lsqr", "sqd", "lambda_", "sigma", "etol", "utol", "btol", "conlim"),
             {"M": 7, "N": 4}, True, "x", kb.SimpleStats),
    "cgls": (TALL, NORMAL, {"M": 7}, True, "x", kb.SimpleStats),
    "crls": (TALL, NORMAL, {"M": 7}, True, "x", kb.SimpleStats),
    "bilq": (SQ, BIORTH + ("transfer_to_bicg",), {"M": 5, "N": 5}, True, "x", kb.SimpleStats),
    "qmr": (SQ, BIORTH, {"M": 5, "N": 5}, True, "x", kb.SimpleStats),
    "bilqr": (SQ, ("transfer_to_bicg",), {}, True, "xy", kb.AdjointStats),
    "trilqr": (TALL, ("transfer_to_usymcg",), {}, True, "xy", kb.AdjointStats),
    "craig": (WIDE, LEASTNORM + ("transfer_to_lsqr", "btol", "conlim"), {"M": 4, "N": 7}, True, "xy", kb.SimpleStats),
    "craigmr": (WIDE, LEASTNORM, {"M": 4, "N": 7}, True, "xy", kb.SimpleStats),
    "lnlq": (WIDE, LEASTNORM + ("transfer_to_craig", "sigma", "utolx", "utoly"), {"M": 4, "N": 7}, True, "xy",
             kb.SimpleStats),
    "cgne": (WIDE, ("N", "ldiv", "lambda_"), {"N": 4}, True, "x", kb.SimpleStats),
    "crmr": (WIDE, ("N", "ldiv", "lambda_"), {"N": 4}, True, "x", kb.SimpleStats),
}

O, E = "KrylovOptions", "KrylovB200Options"
FIELDS = {   # keyword: (struct, field, a value other than the default, what the field then holds)
    "atol": (O, "atol", 1e-3, 1e-3), "rtol": (O, "rtol", 1e-4, 1e-4), "itmax": (O, "itmax", 17, 17),
    "timemax": (O, "timemax", 2.5, 2.5), "verbose": (O, "verbose", 3, 3), "history": (E, "history", True, 1),
    "fused": (E, "fused", False, 0), "ldiv": (E, "ldiv", True, 1), "radius": (O, "radius", 0.5, 0.5),
    "linesearch": (O, "linesearch", True, 1), "lambda_": (O, "lambda_", 0.25, 0.25), "restart": (O, "restart", True, 1),
    "reorthogonalization": (O, "reorthogonalization", True, 1), "etol": (E, "etol", 1e-5, 1e-5),
    "conlim": (E, "conlim", 1e6, 1e6), "batch": (E, "batch", 4, 4), "time_kernels": (E, "time_kernels", True, 1),
    "check_curvature": (E, "check_curvature", True, 1), "gamma": (E, "cr_gamma", 0.75, 0.75),
    "artol": (E, "axtol", 1e-6, 1e-6), "axtol": (E, "axtol", 1e-6, 1e-6), "btol": (E, "btol", 1e-7, 1e-7),
    "sqd": (O, "lambda_", True, 1.0), "sigma": (E, "sigma", 0.5, 0.5), "utol": (E, "utol", 1e-8, 1e-8),
    "utolx": (E, "utol", 1e-8, 1e-8), "utoly": (E, "etol", 1e-9, 1e-9),
    "transfer_to_lsqr": (E, "transfer_to_lsqr", True, 1), "transfer_to_bicg": (E, "transfer_to_bicg", False, 0),
    "transfer_to_craig": (E, "transfer_to_bicg", False, 0), "transfer_to_usymcg": (E, "transfer_to_bicg", False, 0),
    "callback": (E, "callback", lambda ws: False, True),
}


def fields(struct):
    """Field values of an option struct; NaN as a string so that dicts compare, the callback as set / not set."""
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
    """Stands in for libkrylov_b200: forwards the default-option constructors, answers every other call with 0 (a
    zeroed statistics struct), and records the option structs and operator lengths krylov_solve receives."""

    FORWARD = ("krylov_default_options", "krylov_b200_default_options", "krylov_default_workspace_options")

    def __init__(self, real):
        self.real, self.solves, self.ext, self.seen = real, [], None, []

    def probe(self, x):
        """A host operator: notes its input length; the recorder counts the entries it writes."""
        self.seen.append(len(x))
        return 1.0

    def __getattr__(self, name):
        if name in self.FORWARD:
            return getattr(self.real, name)

        def call(*args):
            if name == "krylov_workspace_create":
                args[-1]._obj.value = 0x1000
            elif name == "krylov_b200_set_options":
                self.ext = fields(args[1]._obj)
            elif name == "krylov_solve":
                lengths = []
                for f in args[1:5]:
                    if not f:
                        lengths.append(None)
                        continue
                    x, y = (C.c_double * 64)(), (C.c_ubyte * 512)(*([0xFF] * 512))
                    f(C.cast(x, C.c_void_p), C.cast(y, C.c_void_p), None)
                    lengths.append((self.seen.pop(), sum(v != 0xFF for v in bytes(y)) // 8))
                self.solves.append(dict(options={**fields(args[-1]._obj), **self.ext}, ops=lengths,
                                        c=args[6] is not None and bool(args[6].value)))
            return 0
        return call


@pytest.fixture
def rec(monkeypatch):
    r = Recorder(_lib.lib())
    monkeypatch.setattr(kb, "lib", lambda: r)
    monkeypatch.setattr(_lib, "lib", lambda: r)
    return r


def problem(solver):
    (m, n), _, _, _, _, _ = SOLVERS[solver]
    A = sp.csr_matrix(np.eye(m, n) * 4.0 + np.eye(m, n, 1))
    return A, np.ones(m), np.ones(n)


def solve_inplace(solver, A, b, c_adjoint, **kw):
    """solver!(ws, A, b; kw...) on a fresh workspace; c_adjoint is the third positional argument of BiLQR / TriLQR."""
    (m, n), _, _, _, _, _ = SOLVERS[solver]
    ws = kb.krylov_workspace(solver, m, n, np.float64)
    try:
        return getattr(kb, solver + "_")(ws, A, b, *((c_adjoint,) if solver in ADJOINT else ()), **kw)
    finally:
        ws.free()


def default_options(rec, solver):
    A, b, c = problem(solver)
    solve_inplace(solver, A, b, c)
    return rec.solves.pop()["options"]


@pytest.mark.parametrize("solver", sorted(SOLVERS))
def test_defaults_leave_the_library_defaults(rec, solver):
    """A solve without keywords sends the library's default options, but for LSQR / LSMR, whose atol and rtol
    default to 0 as in the reference."""
    L = _lib.lib()
    lib_defaults = {**fields(L.krylov_default_options()), **fields(L.krylov_b200_default_options())}
    got = default_options(rec, solver)
    diff = {k: v for k, v in got.items() if lib_defaults[k] != v}
    assert diff == ({(O, "atol"): 0.0, (O, "rtol"): 0.0} if solver in ("lsqr", "lsmr") else {})


@pytest.mark.parametrize("solver", sorted(SOLVERS))
def test_each_keyword_reaches_its_field(rec, solver):
    """Each keyword the solver takes, alone at a value other than its default, changes its documented field and
    nothing else."""
    _, taken, _, _, _, _ = SOLVERS[solver]
    base = default_options(rec, solver)
    A, b, c = problem(solver)
    for kw in COMMON + tuple(k for k in taken if k in FIELDS):
        struct, field, value, held = FIELDS[kw]
        solve_inplace(solver, A, b, c, **{kw: value})
        got = rec.solves.pop()["options"]
        assert {k: v for k, v in got.items() if base[k] != v} == {(struct, field): held}, kw


@pytest.mark.parametrize("solver", sorted(SOLVERS))
def test_c_reaches_the_library(rec, solver):
    _, taken, _, _, out, _ = SOLVERS[solver]
    A, b, c = problem(solver)
    if solver in ADJOINT:
        solve_inplace(solver, A, b, c)
        assert rec.solves.pop()["c"]
        with pytest.raises(kb.B200Error, match="c must be given"):
            solve_inplace(solver, A, b, None)
    elif "c" in taken:
        solve_inplace(solver, A, b, None, c=b)
        assert rec.solves.pop()["c"]
        solve_inplace(solver, A, b, c)
        assert not rec.solves.pop()["c"]
    else:
        with pytest.raises(kb.B200Error, match=rf"{solver}!: unsupported keyword argument\(s\) c$"):
            solve_inplace(solver, A, b, None, c=b)


@pytest.mark.parametrize("solver", sorted(SOLVERS))
def test_unknown_keyword_is_refused(rec, solver):
    A, b, c = problem(solver)
    msg = rf"{solver}!: unsupported keyword argument\(s\) bogus, x1$"
    with pytest.raises(kb.B200Error, match=msg):
        solve_inplace(solver, A, b, c, x1=0, bogus=1)
    args = (c,) if solver in ADJOINT else ()
    with pytest.raises(kb.B200Error, match=msg):
        getattr(kb, solver)(A, b, *args, x1=0, bogus=1)
    assert not rec.solves


@pytest.mark.parametrize("solver", sorted(SOLVERS))
def test_host_callables_get_the_solvers_lengths(rec, solver):
    """A host-callable A (and A^T where the solver applies it), M and N are called with vectors of the lengths of the
    spaces they act on, and write as many entries."""
    (m, n), _, lengths, adjoint, _, _ = SOLVERS[solver]
    _, b, c = problem(solver)
    A = (rec.probe, rec.probe) if adjoint else rec.probe
    solve_inplace(solver, A, b, c, **{side: rec.probe for side in lengths})
    fA, fAt, fM, fN = rec.solves.pop()["ops"]
    assert fA == (n, m) and fAt == ((m, n) if adjoint else None)
    assert fM == ((lengths["M"],) * 2 if "M" in lengths else None)
    assert fN == ((lengths["N"],) * 2 if "N" in lengths else None)


@pytest.mark.parametrize("solver", sorted(SOLVERS))
def test_out_of_place_forms_return(rec, solver):
    _, _, _, _, out, stats = SOLVERS[solver]
    A, b, c = problem(solver)
    got = getattr(kb, solver)(A, b, *((c,) if solver in ADJOINT else ()))
    assert len(got) == len(out) + 1 and isinstance(got[-1], stats)
    assert [len(v) for v in got[:-1]] == [A.shape[1], A.shape[0]][:len(out)]
    assert len(rec.solves) == 1
