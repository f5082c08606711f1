"""ctypes front-end of the CPU restatement of bilq! / qmr! -- TEST INFRASTRUCTURE ONLY.

Same status as oracle/oracle.py (only tests/ may import it; the product never does).  The solvers live in
krylov_oracle_biorth.h, built with the BLAS-1 wrappers of krylov_oracle_impl.h into libkrylov_oracle_biorth.so by
biorth.mk.  The square problem generators of test/test_utils.jl that test/test_bilq.jl and test/test_qmr.jl use are
re-exported from oracle.py; unsymmetric_breakdown (test/test_utils.jl:196-201) is restated here.  Parity pinning:
tests/test_oracle_bilq_qmr.py and tests/golden/oracle_bilq_qmr.json (frozen histories).
"""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess

import numpy as np
import scipy.sparse as sp

from oracle.oracle import (Stats, _csr, _opts, _p, _result, _suf, _vec, bc_breakdown, kron_unsymmetric,  # noqa: F401
                           nonsymmetric_definite, nonsymmetric_indefinite, polar_poisson, sparse_laplacian,
                           square_preconditioned, symmetric_definite, symmetric_indefinite, two_preconditioners,
                           zero_rhs)

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
_ITER_CB = C.CFUNCTYPE(C.c_int, C.c_int, C.c_void_p)


def build(force: bool = False) -> str:
    """Compile oracle/libkrylov_oracle_biorth.so with the committed biorth.mk (when missing or older than its sources)."""
    so = os.path.join(_HERE, "libkrylov_oracle_biorth.so")
    srcs = [os.path.join(_HERE, f) for f in ("krylov_oracle_biorth.c", "krylov_oracle_biorth.h", "krylov_oracle_impl.h", "biorth.mk")]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["make", "-C", _HERE, "-f", "biorth.mk", "-s"])
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


def unsymmetric_breakdown():
    """test/test_utils.jl:196-201: b and c start a Lanczos biorthogonalization that breaks down (pᴴq = 0)."""
    return sp.csr_matrix(np.array([[0.0, 1.0], [-1.0, 0.0]])), np.array([1.0, 0.0]), np.array([-1.0, 0.0])


def _biorth(qmr, A, b, c, x0, M, N, transfer_to_bicg, timemax, callback, dtype, kw):
    suf, _ = _suf(dtype)
    n, rp, ci, va = _csr(A, dtype)
    _, trp, tci, tva = _csr(sp.csr_matrix(A).T, dtype)
    b, c, x0, M, N = (_vec(v, dtype) for v in (b, c, x0, M, N))
    o = _opts(n, kw, 1 << 22)
    x = np.zeros(n, dtype)
    res = np.zeros(o.hist_cap, dtype)
    st = Stats()
    cb = _ITER_CB(lambda it, _u: int(bool(callback(it)))) if callback is not None else _ITER_CB()
    f = getattr(lib(), f"oracle_biorth_{suf}")
    f.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 11 + [C.c_int, C.c_double, _ITER_CB] + [C.c_void_p] * 5
    f(int(qmr), n, _p(rp), _p(ci), _p(va), _p(trp), _p(tci), _p(tva), _p(b), _p(c), _p(x0), _p(M), _p(N),
      int(transfer_to_bicg), -1.0 if math.isinf(timemax) else float(timemax), cb, None,
      C.cast(C.byref(o), C.c_void_p), _p(x), _p(res), C.cast(C.byref(st), C.c_void_p))
    return _result(st, x, res)


def bilq(A, b, c=None, x0=None, M=None, N=None, transfer_to_bicg=True, timemax=math.inf, callback=None,
         dtype=np.float64, **kw):
    """bilq! (src/bilq.jl:118-407).  c: None (= b) or the shadow vector; M, N: None or the diagonal of a Diagonal
    preconditioner; callback(iter) -> bool stops the solve when true; timemax in seconds."""
    return _biorth(False, A, b, c, x0, M, N, transfer_to_bicg, timemax, callback, dtype, kw)


def qmr(A, b, c=None, x0=None, M=None, N=None, timemax=math.inf, callback=None, dtype=np.float64, **kw):
    """qmr! (src/qmr.jl:124-405); arguments as for bilq."""
    return _biorth(True, A, b, c, x0, M, N, False, timemax, callback, dtype, kw)
