"""ctypes front-end of the CPU restatement of cg_lanczos_shift! and cgls_lanczos_shift! -- TEST INFRASTRUCTURE ONLY.

Same status as oracle/oracle.py (only tests/ may import it; the product never does).  The solvers live in
krylov_oracle_shift.h, built with the helpers of krylov_oracle_impl.h into libkrylov_oracle_shift.so (Makefile.shift),
which has its own test knobs: `dot_mode` and `precond_block` below set them for this library.  Parity pinning:
tests/test_oracle_shift.py (the reference's assertions of test/test_cg_lanczos_shift.jl and
test/test_cgls_lanczos_shift.jl) and tests/golden/oracle_shift.json (frozen histories).
"""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess

import numpy as np
import scipy.sparse as sp

from oracle.oracle import Options, Problem, Stats, _ITER_CB, _csr, _p, _suf, _vec

_HERE = os.path.dirname(os.path.abspath(__file__))
_SOURCES = ("krylov_oracle_shift.c", "krylov_oracle_shift.h", "krylov_oracle_impl.h", "Makefile.shift")
_LIB = None


def build(force: bool = False) -> str:
    """Compile oracle/libkrylov_oracle_shift.so with Makefile.shift (when missing or older than its sources)."""
    so = os.path.join(_HERE, "libkrylov_oracle_shift.so")
    if force or not os.path.exists(so) or any(os.path.getmtime(os.path.join(_HERE, s)) > os.path.getmtime(so)
                                             for s in _SOURCES):
        subprocess.check_call(["make", "-C", _HERE, "-f", "Makefile.shift", "-s"])
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
    return _LIB


class dot_mode:
    """with dot_mode(2): ...  -- this library's dot products in the order of the device's one-CTA reduction (n <= 256);
    1 accumulates in double, 0 (default) is the sequential sum (krylov_oracle_impl.h: kdot)."""

    def __init__(self, mode):
        self.mode = int(mode)

    def __enter__(self):
        lib().oracle_set_dot_mode(self.mode)

    def __exit__(self, *a):
        lib().oracle_set_dot_mode(0)


class precond_block:
    """with precond_block(bs): ...  -- M is read as ceil(n/bs) dense bs x bs row-major diagonal blocks (block-Jacobi)."""

    def __init__(self, bs):
        self.bs = int(bs)

    def __enter__(self):
        lib().oracle_set_precond_block(self.bs)

    def __exit__(self, *a):
        lib().oracle_set_precond_block(0)


_KW = ("atol", "rtol", "itmax", "timemax", "history", "callback", "ldiv", "hist_cap")


def _solve(name, A, b, shifts, M, dtype, kw):
    if name == "cgls_lanczos_shift" and M is not None:
        raise ValueError("Preconditioner `M` is not supported.")
    unknown = sorted(set(kw) - set(_KW) - ({"check_curvature"} if name == "cg_lanczos_shift" else set()))
    if unknown:
        raise TypeError(f"unknown options {unknown}")
    suf, _ = _suf(dtype)
    A = sp.csr_matrix(A)
    m, n = A.shape
    if name == "cg_lanczos_shift" and m != n:
        raise ValueError("System must be square")
    shifts = np.ascontiguousarray(shifts, dtype=dtype)
    p = shifts.shape[0]
    P = Problem(m, n)
    _, rp, ci, va = _csr(A, dtype)
    P.rowptr, P.colind, P.val = _p(rp), _p(ci), _p(va)
    keep = [rp, ci, va]
    if name == "cgls_lanczos_shift":
        _, trp, tci, tva = _csr(A.T, dtype)
        P.trowptr, P.tcolind, P.tval = _p(trp), _p(tci), _p(tva)
        keep += [trp, tci, tva]
    bv, Mv = _vec(b, dtype), _vec(M, dtype)
    P.b, P.M = _p(bv), _p(Mv)
    o = Options()
    if kw.get("atol") is not None:
        o.atol = float(kw["atol"])
    if kw.get("rtol") is not None:
        o.rtol = float(kw["rtol"])
    o.itmax = int(kw.get("itmax", 0))
    o.history = int(bool(kw.get("history", True)))
    o.ldiv = int(bool(kw.get("ldiv", False)))
    o.check_curvature = int(bool(kw.get("check_curvature", False)))
    t = kw.get("timemax", math.inf)
    o.timemax = -1.0 if math.isinf(t) else float(t)
    f = kw.get("callback")
    o.callback = _ITER_CB() if f is None else _ITER_CB(lambda it, _u: int(bool(f(it))))
    itmax = o.itmax if o.itmax > 0 else (m + n if name == "cgls_lanczos_shift" else 2 * n)
    o.hist_cap = int(kw.get("hist_cap") or min(itmax + 2, 1 << 22))
    X = np.zeros((n, p), dtype, order="F")
    hist = np.zeros((p, o.hist_cap), dtype)
    hlen, indef = np.zeros(p, np.int32), np.zeros(p, np.int32)
    st = Stats()
    rc = getattr(lib(), f"oracle_lanczos_shift_{suf}")(
        name.encode(), C.byref(P), _p(shifts), p, C.byref(o), _p(X), _p(hist), _p(hlen), _p(indef), C.byref(st))
    if rc != 0:
        raise ValueError(st.status.decode())
    stats = dict(niter=st.niter, solved=bool(st.solved), status=st.status.decode(),
                 residuals=[hist[i, :min(int(hlen[i]), o.hist_cap)].copy() for i in range(p)],
                 indefinite=[bool(v) for v in indef], Anorm=math.nan, Acond=math.nan)
    return [X[:, i].copy() for i in range(p)], stats


def cg_lanczos_shift(A, b, shifts, M=None, dtype=np.float64, **kw):
    """cg_lanczos_shift! (src/cg_lanczos_shift.jl:110-268) -> (xs, stats): (A + σᵢ I) xᵢ = b for every σᵢ in shifts.
    M: None or the diagonal of a Diagonal preconditioner (blocks under precond_block).  kwargs: atol, rtol (default
    sqrt(eps)), itmax (0: 2n), check_curvature, ldiv, history (default True), callback(iter) -> bool, timemax."""
    return _solve("cg_lanczos_shift", A, b, shifts, M, dtype, kw)


def cgls_lanczos_shift(A, b, shifts, M=None, dtype=np.float64, **kw):
    """cgls_lanczos_shift! (src/cgls_lanczos_shift.jl:110-260) -> (xs, stats): (AᵀA + σᵢ I) xᵢ = Aᵀb, A m x n.
    kwargs as cg_lanczos_shift (itmax 0: m + n) without check_curvature; M raises as the reference does."""
    return _solve("cgls_lanczos_shift", A, b, shifts, M, dtype, kw)
