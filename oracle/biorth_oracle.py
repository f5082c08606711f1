"""ctypes front-end of the CPU restatement of bilq! / qmr! -- TEST INFRASTRUCTURE ONLY.

Same status as oracle/oracle.py (only tests/ may import it; the product never does).  The solvers live in
krylov_oracle_biorth.h, built into the oracle library that oracle.py builds and loads.  The square problem generators of test/test_utils.jl that test/test_bilq.jl and test/test_qmr.jl use are
re-exported from oracle.py; unsymmetric_breakdown (test/test_utils.jl:196-201) is restated here.  Parity pinning:
tests/test_oracle_bilq_qmr.py and tests/golden/oracle_bilq_qmr.json (frozen histories).
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import scipy.sparse as sp

from oracle.oracle import (_ITER_CB, Stats, _csr, _opts, _p, _result, _suf, _vec, bc_breakdown, dot_mode,  # noqa: F401
                           kron_unsymmetric, lib, nonsymmetric_definite, nonsymmetric_indefinite, polar_poisson,
                           sparse_laplacian, square_preconditioned, symmetric_definite, symmetric_indefinite,
                           two_preconditioners, zero_rhs)


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
