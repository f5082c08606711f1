"""ctypes front-end of the CPU restatement of lsqr! / lsmr! -- TEST INFRASTRUCTURE ONLY.

Same status as oracle/oracle.py (only tests/ may import it; the product never does).  The solvers live in
krylov_oracle_lsq.h, built with the BLAS-1 wrappers of krylov_oracle_impl.h into libkrylov_oracle_lsq.so by lsq.mk.
The problem generators restate test/gen_lsq.jl and the least-squares helpers of test/test_utils.jl; the square
generators the reference's LSQR / LSMR tests also use (zero_rhs, two_preconditioners, ddx) are re-exported from
oracle.py.  Parity pinning: tests/test_oracle_lsq.py (the reference's assertions of test/test_lsqr.jl and
test/test_lsmr.jl) and tests/golden/oracle_lsq.json (frozen histories).
"""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess

import numpy as np
import scipy.sparse as sp

from oracle.oracle import Stats, _p, _result, _suf, _vec, ddx, two_preconditioners, zero_rhs  # noqa: F401

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build(force: bool = False) -> str:
    """Compile oracle/libkrylov_oracle_lsq.so with the committed lsq.mk (when missing or older than its sources)."""
    so = os.path.join(_HERE, "libkrylov_oracle_lsq.so")
    srcs = [os.path.join(_HERE, f) for f in ("krylov_oracle_lsq.c", "krylov_oracle_lsq.h", "krylov_oracle_impl.h", "lsq.mk")]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["make", "-C", _HERE, "-f", "lsq.mk", "-s"])
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
    return _LIB


class LsqOpts(C.Structure):
    _fields_ = [("atol", C.c_double), ("rtol", C.c_double), ("etol", C.c_double), ("axtol", C.c_double),
                ("btol", C.c_double), ("conlim", C.c_double), ("lambda_", C.c_double), ("radius", C.c_double),
                ("itmax", C.c_int), ("history", C.c_int), ("window", C.c_int), ("ldiv", C.c_int), ("hist_cap", C.c_int)]


def _lsq(lsmr, A, b, M, N, dtype, kw):
    suf, ct = _suf(dtype)
    A = sp.csr_matrix(A)
    A.sort_indices()
    m, n = A.shape
    rp, ci = np.ascontiguousarray(A.indptr, dtype=np.int32), np.ascontiguousarray(A.indices, dtype=np.int32)
    va = np.ascontiguousarray(A.data, dtype=dtype)
    b, M, N = _vec(b, dtype), _vec(M, dtype), _vec(N, dtype)
    sqd = kw.pop("sqd", False)
    o = LsqOpts()
    o.lambda_ = kw.pop("lambda_", 0.0)
    if sqd:
        if o.lambda_ != 0:
            raise ValueError("sqd cannot be set to true if λ ≠ 0 !")
        o.lambda_ = 1.0
    o.atol, o.rtol = kw.pop("atol", 0.0), kw.pop("rtol", 0.0)           # Julia's kwarg defaults (lsqr.jl:155-156)
    o.etol, o.axtol, o.btol = kw.pop("etol", math.nan), kw.pop("axtol", math.nan), kw.pop("btol", math.nan)
    o.conlim, o.radius = kw.pop("conlim", math.nan), kw.pop("radius", 0.0)
    o.itmax, o.history = kw.pop("itmax", 0), int(kw.pop("history", True))
    o.window, o.ldiv = kw.pop("window", 0), int(kw.pop("ldiv", False))
    itmax = o.itmax if o.itmax > 0 else m + n
    o.hist_cap = kw.pop("hist_cap", min(itmax + 2, 1 << 22))
    if kw:
        raise TypeError(f"unknown options {sorted(kw)}")
    x = np.zeros(n, dtype)
    res, ares = np.zeros(o.hist_cap, dtype), np.zeros(o.hist_cap, dtype)
    anorm = ct(0)
    st = Stats()
    f = getattr(lib(), f"oracle_lsq_{suf}")
    f.argtypes = [C.c_int] * 3 + [C.c_void_p] * 12
    rc = f(int(lsmr), m, n, _p(rp), _p(ci), _p(va), _p(b), _p(M), _p(N), C.cast(C.byref(o), C.c_void_p), _p(x), _p(res),
           _p(ares), C.cast(C.byref(anorm), C.c_void_p), C.cast(C.byref(st), C.c_void_p))
    if rc:
        raise ArithmeticError({12: "zero direction", 13: "outside of the trust region"}.get(rc, "no real roots"))
    k = min(st.nAres, o.hist_cap)
    return _result(st, x, res, dict(Aresiduals=ares[:k].copy(), Anorm=float(anorm.value)))


def lsqr(A, b, M=None, N=None, dtype=np.float64, **kw):
    """lsqr! (src/lsqr.jl:174-440) on an m x n matrix.  M (m) / N (n): None or the diagonal of a Diagonal operator.
    kwargs: lambda_, sqd, radius, etol, axtol, btol, conlim, atol, rtol (default 0), itmax, window, ldiv, history.
    Extra stats key: Aresiduals."""
    return _lsq(0, A, b, M, N, dtype, kw)


def lsmr(A, b, M=None, N=None, dtype=np.float64, **kw):
    """lsmr! (src/lsmr.jl:178-455); same arguments as lsqr.  Extra stats keys: Aresiduals, Anorm (LsmrStats)."""
    return _lsq(1, A, b, M, N, dtype, kw)



# ---- least-squares problems of test/gen_lsq.jl and test/test_utils.jl (restated; dense ones returned as CSR) ------
def lstp(nrow, ncol, ndupl, npower, lam, x):
    """test/gen_lsq.jl:2-51: A = HY D HZ (nrow >= ncol) with a known solution x.  Returns (b, A, D, HY, HZ, Acond, rnorm)."""
    assert nrow >= ncol
    fourpi = 4 * 3.141592                               # the approximation of the original subroutine
    alpha, beta = fourpi / nrow, fourpi / ncol
    hy = np.sin(np.arange(1, nrow + 1) * alpha)
    hz = np.cos(np.arange(1, ncol + 1) * beta)
    hy = hy / np.linalg.norm(hy)
    hz = hz / np.linalg.norm(hz)
    HY = np.eye(nrow) - 2 * np.outer(hy, hy)
    HZ = np.eye(ncol) - 2 * np.outer(hz, hz)
    d = (((np.arange(ncol) + ndupl) // ndupl) * ndupl / ncol) ** npower
    D = np.zeros((nrow, ncol))
    D[np.arange(ncol), np.arange(ncol)] = d
    A = HY @ D @ HZ
    Acond = abs(d[ncol - 1] / d[0])
    x = np.asarray(x, dtype=float)
    r = np.zeros(nrow)
    r[:ncol] = HZ @ x / d
    t = 1.0
    for i in range(ncol + 1, nrow + 1):
        r[i - 1] = t * (i - ncol) / nrow
        t = -t
    r = HY @ r
    return r + A @ x, sp.csr_matrix(A), D, HY, HZ, Acond, np.linalg.norm(r)


def lsq_test(nrow, ncol, ndupl, npower, damp):
    """test(nrow, ncol, ndupl, npower, damp) of test/gen_lsq.jl:54-58: desired solution x = ncol - (1:ncol)."""
    return lstp(nrow, ncol, ndupl, npower, damp, ncol - np.arange(1, ncol + 1, dtype=float))


def _reg_matrix(n):
    return np.array([[2 ** (i / j) * j + (-1) ** (i - j) * n * (i - 1) for j in range(1, n + 1)] for i in range(1, n + 1)])


def regularization(n=5):
    """test/test_utils.jl:326-331 -> (A, b, lambda = 4)."""
    return sp.csr_matrix(_reg_matrix(n)), np.ones(n), 4.0


def saddle_point(n=5):
    """test/test_utils.jl:334-339 -> (A, b, diag(D))."""
    return sp.csr_matrix(_reg_matrix(n)), np.ones(n), 2.0 * np.arange(1, n + 1)


def sqd(n=5):
    """test/test_utils.jl:367-373 -> (A, b, diag(M), diag(N))."""
    return sp.csr_matrix(_reg_matrix(n)), np.ones(n), 3.0 * np.arange(1, n + 1), 5.0 * np.arange(1, n + 1)
