"""ctypes front-end of the CPU restatement of cgls! / crls! / lslq! -- TEST INFRASTRUCTURE ONLY.

Same status as oracle/oracle.py (only tests/ may import it; the product never does).  The solvers live in
krylov_oracle_cgls.h and krylov_oracle_lslq.h, on the rectangular products of krylov_oracle_lsq.h, built into the
oracle library that oracle.py builds and loads.  The least-squares problem generators are re-exported from
lsq_oracle.py.  Parity pinning: tests/test_oracle_cgls.py (the reference's assertions of test/test_cgls.jl and
test/test_crls.jl) and tests/golden/oracle_cgls.json (frozen histories).
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import scipy.sparse as sp

from oracle.lsq_oracle import lsq_test, lstp, regularization, saddle_point, sqd  # noqa: F401
from oracle.oracle import Stats, _p, _result, _suf, _vec, lib, zero_rhs  # noqa: F401


class CglsOpts(C.Structure):
    _fields_ = [("atol", C.c_double), ("rtol", C.c_double), ("lambda_", C.c_double), ("radius", C.c_double),
                ("itmax", C.c_int), ("history", C.c_int), ("ldiv", C.c_int), ("hist_cap", C.c_int)]


def _run(crls, A, b, M, dtype, kw):
    suf, _ = _suf(dtype)
    A = sp.csr_matrix(A)
    A.sort_indices()
    m, n = A.shape
    rp, ci = np.ascontiguousarray(A.indptr, dtype=np.int32), np.ascontiguousarray(A.indices, dtype=np.int32)
    va = np.ascontiguousarray(A.data, dtype=dtype)
    b, M = _vec(b, dtype), _vec(M, dtype)
    o = CglsOpts()
    o.atol, o.rtol = kw.pop("atol", math.nan), kw.pop("rtol", math.nan)    # Julia's kwarg defaults: sqrt(eps(T))
    o.lambda_, o.radius = kw.pop("lambda_", 0.0), kw.pop("radius", 0.0)
    o.itmax, o.history = kw.pop("itmax", 0), int(kw.pop("history", True))
    o.ldiv = int(kw.pop("ldiv", False))
    itmax = o.itmax if o.itmax > 0 else m + n
    o.hist_cap = kw.pop("hist_cap", min(itmax + 2, 1 << 22))
    if kw:
        raise TypeError(f"unknown options {sorted(kw)}")
    x = np.zeros(n, dtype)
    res, ares = np.zeros(o.hist_cap, dtype), np.zeros(o.hist_cap, dtype)
    st = Stats()
    f = getattr(lib(), f"oracle_cgls_{suf}")
    f.argtypes = [C.c_int] * 3 + [C.c_void_p] * 10
    rc = f(int(crls), m, n, _p(rp), _p(ci), _p(va), _p(b), _p(M), C.cast(C.byref(o), C.c_void_p), _p(x), _p(res),
           _p(ares), C.cast(C.byref(st), C.c_void_p))
    if rc:
        raise ArithmeticError({12: "zero direction", 13: "outside of the trust region"}.get(rc, "no real roots"))
    k = min(st.nAres, o.hist_cap)
    return _result(st, x, res, dict(Aresiduals=ares[:k].copy()))


def cgls(A, b, M=None, dtype=np.float64, **kw):
    """cgls! (src/cgls.jl:129-243) on an m x n matrix.  M (m entries): None or the diagonal of a Diagonal operator.
    kwargs: lambda_, radius, atol, rtol (default sqrt(eps)), itmax, ldiv, history.  Extra stats key: Aresiduals."""
    return _run(0, A, b, M, dtype, kw)


def crls(A, b, M=None, dtype=np.float64, **kw):
    """crls! (src/crls.jl:120-268); same arguments as cgls."""
    return _run(1, A, b, M, dtype, kw)


class LslqOpts(C.Structure):
    _fields_ = [("atol", C.c_double), ("rtol", C.c_double), ("etol", C.c_double), ("utol", C.c_double), ("btol", C.c_double),
                ("conlim", C.c_double), ("lambda_", C.c_double), ("sigma", C.c_double), ("itmax", C.c_int),
                ("history", C.c_int), ("window", C.c_int), ("ldiv", C.c_int), ("transfer_to_lsqr", C.c_int),
                ("hist_cap", C.c_int)]


def lslq(A, b, M=None, N=None, dtype=np.float64, **kw):
    """lslq! (src/lslq.jl:201-520) on an m x n matrix.  M (m) / N (n): None or the diagonal of a Diagonal operator.
    kwargs: lambda_, sqd, sigma, etol, utol, btol, conlim, atol, rtol (default sqrt(eps)), itmax, window, ldiv,
    transfer_to_lsqr, history.  Extra stats keys: Aresiduals, err_lbnds, err_ubnds_lq, err_ubnds_cg, error_with_bnd."""
    suf, _ = _suf(dtype)
    A = sp.csr_matrix(A)
    A.sort_indices()
    m, n = A.shape
    rp, ci = np.ascontiguousarray(A.indptr, dtype=np.int32), np.ascontiguousarray(A.indices, dtype=np.int32)
    va = np.ascontiguousarray(A.data, dtype=dtype)
    b, M, N = _vec(b, dtype), _vec(M, dtype), _vec(N, dtype)
    o = LslqOpts()
    o.lambda_ = kw.pop("lambda_", 0.0)
    if kw.pop("sqd", False):
        if o.lambda_ != 0:
            raise ValueError("sqd cannot be set to true if λ ≠ 0 !")
        o.lambda_ = 1.0
    o.sigma = kw.pop("sigma", 0.0)
    for f in ("atol", "rtol", "etol", "utol", "btol", "conlim"):
        setattr(o, f, kw.pop(f, math.nan))
    o.itmax, o.history = kw.pop("itmax", 0), int(kw.pop("history", True))
    o.window, o.ldiv = kw.pop("window", 0), int(kw.pop("ldiv", False))
    o.transfer_to_lsqr = int(kw.pop("transfer_to_lsqr", False))
    itmax = o.itmax if o.itmax > 0 else m + n
    o.hist_cap = kw.pop("hist_cap", min(itmax + 2, 1 << 22))
    if kw:
        raise TypeError(f"unknown options {sorted(kw)}")
    x = np.zeros(n, dtype)
    hist = [np.zeros(o.hist_cap, dtype) for _ in range(5)]
    ptrs = (C.c_void_p * 5)(*[h.ctypes.data for h in hist])
    counts = (C.c_int * 5)()
    ewb = C.c_int()
    st = Stats()
    f = getattr(lib(), f"oracle_lslq_{suf}")
    f.argtypes = [C.c_int] * 2 + [C.c_void_p] * 12
    f(m, n, _p(rp), _p(ci), _p(va), _p(b), _p(M), _p(N), C.cast(C.byref(o), C.c_void_p), _p(x), C.cast(ptrs, C.c_void_p),
      C.cast(counts, C.c_void_p), C.cast(C.byref(ewb), C.c_void_p), C.cast(C.byref(st), C.c_void_p))
    k = [min(counts[i], o.hist_cap) for i in range(5)]
    st.nres = k[0]
    return _result(st, x, hist[0], dict(Aresiduals=hist[1][:k[1]].copy(), err_lbnds=hist[2][:k[2]].copy(),
                                        err_ubnds_lq=hist[3][:k[3]].copy(), err_ubnds_cg=hist[4][:k[4]].copy(),
                                        error_with_bnd=bool(ewb.value)))
