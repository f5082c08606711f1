"""ctypes front-end of the CPU restatement of craig! / craigmr! -- TEST INFRASTRUCTURE ONLY.

Same status as oracle/oracle.py (only tests/ may import it; the product never does).  The solvers live in
krylov_oracle_leastnorm.h, built with the shared BLAS-1 wrappers of krylov_oracle_impl.h by leastnorm.mk into a library
that links against the shared oracle library and uses its test knobs: oracle.dot_mode (re-exported here) switches the
dot products of these solvers as of every other family.  The generators of test/test_utils.jl that the reference's
test/test_craig.jl and test/test_craigmr.jl use are restated here, or re-exported from oracle.py and lsq_oracle.py.
Parity pinning: tests/test_oracle_leastnorm.py and tests/golden/oracle_leastnorm.json (frozen histories).
"""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess

import numpy as np
import scipy.sparse as sp

from oracle import oracle as _shared
from oracle.lsq_oracle import regularization, saddle_point, sqd  # noqa: F401
from oracle.oracle import (_ITER_CB, Stats, _csr, _p, _suf, _vec, dot_mode, square_inconsistent,  # noqa: F401
                           two_preconditioners, zero_rhs)

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
_SOURCES = ("krylov_oracle_leastnorm.c", "krylov_oracle_leastnorm.h", "krylov_oracle_impl.h", "leastnorm.mk",
            "libkrylov_oracle.so")


def build(force: bool = False) -> str:
    """Compile oracle/libkrylov_oracle_leastnorm.so with leastnorm.mk (when missing or older than its sources), after the
    shared oracle library it links against."""
    _shared.build()
    so = os.path.join(_HERE, "libkrylov_oracle_leastnorm.so")
    srcs = [os.path.join(_HERE, f) for f in _SOURCES]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "leastnorm.mk"])
    return so


def lib():
    global _LIB
    if _LIB is None:
        _shared.lib()                 # the shared library first: this one resolves the test knobs against it
        _LIB = C.CDLL(build())
    return _LIB


class LnOpts(C.Structure):
    _fields_ = [("atol", C.c_double), ("rtol", C.c_double), ("btol", C.c_double), ("conlim", C.c_double),
                ("lambda_", C.c_double), ("itmax", C.c_int), ("history", C.c_int), ("ldiv", C.c_int),
                ("transfer_to_lsqr", C.c_int), ("hist_cap", C.c_int)]


def _leastnorm(mr, A, b, M, N, timemax, callback, dtype, kw):
    suf, _ = _suf(dtype)
    A = sp.csr_matrix(A)
    m, n = A.shape
    _, rp, ci, va = _csr(A, dtype)
    _, trp, tci, tva = _csr(A.T, dtype)
    b, M, N = _vec(b, dtype), _vec(M, dtype), _vec(N, dtype)
    o = LnOpts()
    o.lambda_ = kw.pop("lambda_", 0.0)
    if kw.pop("sqd", False):
        if o.lambda_ != 0:
            raise ValueError("sqd cannot be set to true if λ ≠ 0 !")
        o.lambda_ = 1.0
    o.atol, o.rtol = kw.pop("atol", math.nan), kw.pop("rtol", math.nan)
    o.btol, o.conlim = kw.pop("btol", math.nan), kw.pop("conlim", math.nan)
    o.itmax, o.history = kw.pop("itmax", 0), int(kw.pop("history", True))
    o.ldiv, o.transfer_to_lsqr = int(kw.pop("ldiv", False)), int(kw.pop("transfer_to_lsqr", False))
    itmax = o.itmax if o.itmax > 0 else m + n
    o.hist_cap = min(itmax + 2, 1 << 22)
    if kw:
        raise TypeError(f"unknown options {sorted(kw)}")
    x, y = np.zeros(n, dtype), np.zeros(m, dtype)
    res, ares = np.zeros(o.hist_cap, dtype), np.zeros(o.hist_cap, dtype)
    st = Stats()
    cb = _ITER_CB(lambda it, _u: int(bool(callback(it)))) if callback is not None else _ITER_CB()
    f = getattr(lib(), f"oracle_leastnorm_{suf}")
    f.argtypes = [C.c_int] * 3 + [C.c_void_p] * 10 + [C.c_double, _ITER_CB] + [C.c_void_p] * 6
    f(int(mr), m, n, _p(rp), _p(ci), _p(va), _p(trp), _p(tci), _p(tva), _p(b), _p(M), _p(N), C.cast(C.byref(o), C.c_void_p),
      -1.0 if math.isinf(timemax) else float(timemax), cb, None, _p(x), _p(y), _p(res), _p(ares),
      C.cast(C.byref(st), C.c_void_p))
    stats = dict(niter=st.niter, solved=bool(st.solved), inconsistent=bool(st.inconsistent), status=st.status.decode("utf-8"),
                 residuals=res[:min(st.nres, o.hist_cap)].copy())
    if mr:
        stats["Aresiduals"] = ares[:min(st.nAres, o.hist_cap)].copy()
    return x, y, stats


def craig(A, b, M=None, N=None, timemax=math.inf, callback=None, dtype=np.float64, **kw):
    """craig! (src/craig.jl:174-405) -> (x, y, stats).  M (m) / N (n): None or the diagonal of a Diagonal operator.
    kwargs: lambda_, sqd, transfer_to_lsqr, btol, conlim, atol, rtol, itmax, ldiv, history.  callback(iter) -> bool."""
    return _leastnorm(0, A, b, M, N, timemax, callback, dtype, kw)


def craigmr(A, b, M=None, N=None, timemax=math.inf, callback=None, dtype=np.float64, **kw):
    """craigmr! (src/craigmr.jl:161-396) -> (x, y, stats); stats also has Aresiduals.  Same arguments as craig, without
    transfer_to_lsqr, btol and conlim."""
    return _leastnorm(1, A, b, M, N, timemax, callback, dtype, kw)


# ---- problem generators of test/test_utils.jl (real case) ----------------------------------------------------------
def _ij_minus_ji(n, m):
    """[i/j - j/i for i=1:n, j=1:m]"""
    i, j = np.indices((n, m)) + 1.0
    return i / j - j / i


def under_consistent(n=10, m=25):
    """test/test_utils.jl:94-100: A = [i/j - j/i] (n x m, n < m), b = A 1."""
    A = _ij_minus_ji(n, m)
    return sp.csr_matrix(A), A @ np.ones(m)


def under_inconsistent(n=10, m=25):
    """test/test_utils.jl:103-109: A = ones(n, m), b = [-1, 2, 3, ..., n]."""
    b = np.arange(1.0, n + 1)
    b[0] = -1.0
    return sp.csr_matrix(np.ones((n, m))), b


def square_consistent(n=10):
    """test/test_utils.jl:112-117"""
    A = _ij_minus_ji(n, n)
    return sp.csr_matrix(A), A @ np.ones(n)


def over_consistent(n=25, m=10):
    """test/test_utils.jl:135-141: A = [i/j - j/i] (n x m, n > m), b = A 1."""
    A = _ij_minus_ji(n, m)
    return sp.csr_matrix(A), A @ np.ones(m)


def over_inconsistent(n=25, m=10):
    """test/test_utils.jl:144-150"""
    b = np.arange(1.0, n + 1)
    b[0] = -1.0
    return sp.csr_matrix(np.ones((n, m))), b


def _small_A(transpose):
    A = np.array([[1.0, 0.0], [0.0, -1.0], [3.0, 0.0]])
    return A.T.copy() if transpose else A


def small_sp(transpose=False):
    """test/test_utils.jl:342-350 -> (A, b, c, diag(D)), D = diag(2i), i = 1..rows(A)."""
    A = _small_A(transpose)
    n, m = A.shape
    return sp.csr_matrix(A), np.ones(n), -np.ones(m), 2.0 * np.arange(1, n + 1)


def small_sqd(transpose=False):
    """test/test_utils.jl:376-385 -> (A, b, c, diag(M), diag(N))."""
    A = _small_A(transpose)
    n, m = A.shape
    return sp.csr_matrix(A), np.ones(n), -np.ones(m), 3.0 * np.arange(1, n + 1), 5.0 * np.arange(1, m + 1)


def small_ln():
    """test/test_utils.jl:422-426: A = [0 1], b = [1]."""
    return sp.csr_matrix(np.array([[0.0, 1.0]])), np.array([1.0])
