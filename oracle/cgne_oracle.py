"""ctypes front-end of the CPU restatement of cgne! and crmr! -- TEST INFRASTRUCTURE ONLY.

Same status as oracle/oracle.py (only tests/ may import it; the product never does).  The solvers live in
krylov_oracle_cgne.h, built into the oracle library that oracle.py builds and loads, so oracle.dot_mode (re-exported
here) switches the dot products of these solvers as of every other family.  The generators of test/test_utils.jl
that the reference's test/test_cgne.jl and test/test_crmr.jl use are re-exported from leastnorm_oracle.py and
oracle.py.
Parity pinning: tests/test_oracle_cgne_crmr.py and tests/golden/oracle_cgne_crmr.json (frozen histories).
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import scipy.sparse as sp

from oracle.leastnorm_oracle import (over_consistent, over_inconsistent, small_sp, square_consistent,  # noqa: F401
                                     square_inconsistent, under_consistent, under_inconsistent, zero_rhs)
from oracle.oracle import _ITER_CB, Stats, _csr, _p, _suf, _vec, dot_mode, lib, square_preconditioned  # noqa: F401


class CgneOpts(C.Structure):
    _fields_ = [("atol", C.c_double), ("rtol", C.c_double), ("lambda_", C.c_double), ("itmax", C.c_int),
                ("history", C.c_int), ("ldiv", C.c_int), ("hist_cap", C.c_int)]


def _run(name, A, b, N, timemax, callback, dtype, kw):
    suf, _ = _suf(dtype)
    A = sp.csr_matrix(A)
    m, n = A.shape
    _, rp, ci, va = _csr(A, dtype)
    _, trp, tci, tva = _csr(A.T, dtype)
    b, N = _vec(b, dtype), _vec(N, dtype)
    o = CgneOpts()
    o.lambda_ = kw.pop("lambda_", 0.0)
    o.atol, o.rtol = kw.pop("atol", math.nan), kw.pop("rtol", math.nan)
    o.itmax, o.history = kw.pop("itmax", 0), int(kw.pop("history", True))
    o.ldiv = int(kw.pop("ldiv", False))
    itmax = o.itmax if o.itmax > 0 else m + n
    o.hist_cap = min(itmax + 2, 1 << 22)
    if kw:
        raise TypeError(f"unknown options {sorted(kw)}")
    x = np.zeros(n, dtype)
    res, ares = np.zeros(o.hist_cap, dtype), np.zeros(o.hist_cap, dtype)
    st = Stats()
    cb = _ITER_CB(lambda it, _u: int(bool(callback(it)))) if callback is not None else _ITER_CB()
    f = getattr(lib(), f"oracle_{name}_{suf}")
    head = [_p(rp), _p(ci), _p(va), _p(trp), _p(tci), _p(tva), _p(b), _p(N), C.cast(C.byref(o), C.c_void_p),
            -1.0 if math.isinf(timemax) else float(timemax), cb, None, _p(x), _p(res)]
    tail = ([_p(ares)] if name == "crmr" else []) + [C.cast(C.byref(st), C.c_void_p)]
    f.argtypes = [C.c_int] * 2 + [C.c_void_p] * 9 + [C.c_double, _ITER_CB] + [C.c_void_p] * (len(head) - 11 + len(tail))
    f(m, n, *head, *tail)
    stats = dict(niter=st.niter, solved=bool(st.solved), inconsistent=bool(st.inconsistent), status=st.status.decode("utf-8"),
                 residuals=res[:min(st.nres, o.hist_cap)].copy())
    if name == "crmr":
        stats["Aresiduals"] = ares[:min(st.nAres, o.hist_cap)].copy()
    return x, stats


def cgne(A, b, N=None, timemax=math.inf, callback=None, dtype=np.float64, **kw):
    """cgne! (src/cgne.jl:134-252) -> (x, stats).  N (m entries): None or the diagonal of a Diagonal operator on the
    residual space.  kwargs: lambda_, atol, rtol, itmax, ldiv, history.  callback(iter) -> bool."""
    return _run("cgne", A, b, N, timemax, callback, dtype, kw)


def crmr(A, b, N=None, timemax=math.inf, callback=None, dtype=np.float64, **kw):
    """crmr! (src/crmr.jl:132-244) -> (x, stats); stats also has Aresiduals.  Same arguments as cgne."""
    return _run("crmr", A, b, N, timemax, callback, dtype, kw)
