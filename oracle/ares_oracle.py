"""ctypes front-end of the CPU restatement of car! / minares! -- TEST INFRASTRUCTURE ONLY.

Same status as oracle/oracle.py (only tests/ may import it; the product never does).  The solvers live in
krylov_oracle_ares.h, built with the BLAS-1 wrappers of krylov_oracle_impl.h into libkrylov_oracle_ares.so by ares.mk.
The symmetric problem generators of test/test_utils.jl that test/test_car.jl and test/test_minares.jl use are
re-exported from oracle.py; symmetric_inconsistent (test/test_utils.jl:128-132) is restated here.  Parity pinning:
tests/test_oracle_car_minares.py and tests/golden/oracle_car_minares.json (frozen histories).
"""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess

import numpy as np
import scipy.sparse as sp

from oracle.oracle import (Stats, _csr, _opts, _p, _result, _suf, _vec, almost_singular, cartesian_poisson,  # noqa: F401
                           get_div_grad, sparse_laplacian, singular_consistent, square_inconsistent,
                           square_preconditioned, symmetric_definite, symmetric_indefinite, zero_rhs)

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
_ITER_CB = C.CFUNCTYPE(C.c_int, C.c_int, C.c_void_p)


def build(force: bool = False) -> str:
    """Compile oracle/libkrylov_oracle_ares.so with the committed ares.mk (when missing or older than its sources)."""
    so = os.path.join(_HERE, "libkrylov_oracle_ares.so")
    srcs = [os.path.join(_HERE, f) for f in ("krylov_oracle_ares.c", "krylov_oracle_ares.h", "krylov_oracle_impl.h", "ares.mk")]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["make", "-C", _HERE, "-f", "ares.mk", "-s"])
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
    return _LIB


class dot_mode:
    """with dot_mode(1): ...  -- this library's dot products accumulate in double and round once (test knob,
    krylov_oracle_impl.h: kdot); the default 0 is the restatement's sequential sum in the working precision."""

    def __init__(self, mode):
        self.mode = int(mode)

    def __enter__(self):
        lib().oracle_set_dot_mode(self.mode)

    def __exit__(self, *a):
        lib().oracle_set_dot_mode(0)


def symmetric_inconsistent():
    """test/test_utils.jl:128-132: a symmetric, singular 4 x 4 system whose b is outside the range of A."""
    A = np.array([[3.0, 2.0, -1.0, 5.0], [2.0, -2.0, 4.0, 0.0], [-1.0, 4.0, 1.0, 3.0], [5.0, 0.0, 3.0, 5.0]])
    return sp.csr_matrix(A), np.array([1.0, -8.0, 5.0, 2.0])


def _run(name, A, b, x0, extra, timemax, callback, dtype, kw):
    suf, _ = _suf(dtype)
    n, rp, ci, va = _csr(A, dtype)
    b, x0 = _vec(b, dtype), _vec(x0, dtype)
    o = _opts(n, kw, 1 << 22)
    x = np.zeros(n, dtype)
    res, ares = np.zeros(o.hist_cap, dtype), np.zeros(o.hist_cap, dtype)
    st = Stats()
    cb = _ITER_CB(lambda it, _u: int(bool(callback(it)))) if callback is not None else _ITER_CB()
    f = getattr(lib(), f"oracle_{name}_{suf}")
    f.argtypes = [C.c_int] + [C.c_void_p] * 5 + [extra[0], C.c_double, _ITER_CB] + [C.c_void_p] * 6
    f(n, _p(rp), _p(ci), _p(va), _p(b), _p(x0), extra[1], -1.0 if math.isinf(timemax) else float(timemax), cb, None,
      C.cast(C.byref(o), C.c_void_p), _p(x), _p(res), _p(ares), C.cast(C.byref(st), C.c_void_p))
    k = min(st.nAres, o.hist_cap)
    return _result(st, x, res, dict(Aresiduals=ares[:k].copy()))


def car(A, b, x0=None, M=None, timemax=math.inf, callback=None, dtype=np.float64, **kw):
    """car! (src/car.jl:108-256).  M: None or the diagonal of a Diagonal preconditioner (ldiv=True applies its
    inverse); callback(iter) -> bool stops the solve when true; timemax in seconds.  Extra stats key: Aresiduals."""
    M = _vec(M, dtype)
    return _run("car", A, b, x0, (C.c_void_p, _p(M)), timemax, callback, dtype, kw)


def minares(A, b, x0=None, lambda_=0.0, artol=None, timemax=math.inf, callback=None, dtype=np.float64, **kw):
    """minares! (src/minares.jl:113-595), M = I.  lambda_: the shift λ; artol: the kwarg Artol (None -> sqrt(eps)).
    Extra stats key: Aresiduals."""
    kw["lambda_"] = lambda_
    return _run("minares", A, b, x0, (C.c_double, math.nan if artol is None else float(artol)), timemax, callback,
                dtype, kw)
