"""ctypes front-end of the CPU restatement of lnlq! -- TEST INFRASTRUCTURE ONLY.

Same status as oracle/oracle.py (only tests/ may import it; the product never does).  The solver lives in
krylov_oracle_lnlq.h, built into the oracle library that oracle.py builds and loads, so oracle.dot_mode (re-exported
here) switches the dot products of this solver as of every other family.  The generators of test/test_utils.jl
that the reference's test/test_lnlq.jl uses are re-exported from leastnorm_oracle.py, which restates them for CRAIG
and CRAIGMR.
Parity pinning: tests/test_oracle_lnlq.py and tests/golden/oracle_lnlq.json (frozen histories).
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import scipy.sparse as sp

from oracle.leastnorm_oracle import (over_consistent, regularization, saddle_point, small_ln, small_sp,  # noqa: F401
                                     small_sqd, sqd, square_consistent, two_preconditioners, under_consistent,
                                     zero_rhs)
from oracle.oracle import _ITER_CB, Stats, _csr, _p, _suf, _vec, dot_mode, lib  # noqa: F401


class LnlqOpts(C.Structure):
    _fields_ = [("atol", C.c_double), ("rtol", C.c_double), ("utolx", C.c_double), ("utoly", C.c_double),
                ("lambda_", C.c_double), ("sigma", C.c_double), ("itmax", C.c_int), ("history", C.c_int),
                ("ldiv", C.c_int), ("transfer_to_craig", C.c_int), ("hist_cap", C.c_int)]


def lnlq(A, b, M=None, N=None, timemax=math.inf, callback=None, dtype=np.float64, **kw):
    """lnlq! (src/lnlq.jl:168-568) -> (x, y, stats); stats also has error_bnd_x, error_bnd_y and error_with_bnd.
    M (m) / N (n): None or the diagonal of a Diagonal operator.  kwargs: lambda_, sqd, sigma, transfer_to_craig
    (default True), utolx, utoly, atol, rtol, itmax, ldiv, history.  callback(iter) -> bool."""
    suf, _ = _suf(dtype)
    A = sp.csr_matrix(A)
    m, n = A.shape
    _, rp, ci, va = _csr(A, dtype)
    _, trp, tci, tva = _csr(A.T, dtype)
    b, M, N = _vec(b, dtype), _vec(M, dtype), _vec(N, dtype)
    o = LnlqOpts()
    o.lambda_ = kw.pop("lambda_", 0.0)
    if kw.pop("sqd", False):
        if o.lambda_ != 0:
            raise ValueError("sqd cannot be set to true if λ ≠ 0 !")
        o.lambda_ = 1.0
    o.sigma = kw.pop("sigma", 0.0)
    o.atol, o.rtol = kw.pop("atol", math.nan), kw.pop("rtol", math.nan)
    o.utolx, o.utoly = kw.pop("utolx", math.nan), kw.pop("utoly", math.nan)
    o.itmax, o.history = kw.pop("itmax", 0), int(kw.pop("history", True))
    o.ldiv, o.transfer_to_craig = int(kw.pop("ldiv", False)), int(kw.pop("transfer_to_craig", True))
    itmax = o.itmax if o.itmax > 0 else m + n
    o.hist_cap = min(itmax + 3, 1 << 22)
    if kw:
        raise TypeError(f"unknown options {sorted(kw)}")
    x, y = np.zeros(n, dtype), np.zeros(m, dtype)
    res, ex, ey = (np.zeros(o.hist_cap, dtype) for _ in range(3))
    out = (C.c_int * 3)()
    st = Stats()
    cb = _ITER_CB(lambda it, _u: int(bool(callback(it)))) if callback is not None else _ITER_CB()
    f = getattr(lib(), f"oracle_lnlq_{suf}")
    f.argtypes = [C.c_int] * 2 + [C.c_void_p] * 10 + [C.c_double, _ITER_CB] + [C.c_void_p] * 8
    f(m, n, _p(rp), _p(ci), _p(va), _p(trp), _p(tci), _p(tva), _p(b), _p(M), _p(N), C.cast(C.byref(o), C.c_void_p),
      -1.0 if math.isinf(timemax) else float(timemax), cb, None, _p(x), _p(y), _p(res), _p(ex), _p(ey),
      C.cast(out, C.c_void_p), C.cast(C.byref(st), C.c_void_p))
    stats = dict(niter=st.niter, solved=bool(st.solved), inconsistent=bool(st.inconsistent), status=st.status.decode("utf-8"),
                 residuals=res[:min(st.nres, o.hist_cap)].copy(), error_bnd_x=ex[:min(out[0], o.hist_cap)].copy(),
                 error_bnd_y=ey[:min(out[1], o.hist_cap)].copy(), error_with_bnd=bool(out[2]))
    return x, y, stats
