"""ctypes front-end of the CPU restatement of bilqr! / trilqr! -- TEST INFRASTRUCTURE ONLY.

Same status as oracle/oracle.py (only tests/ may import it; the product never does).  The solvers live in
krylov_oracle_adjoint.h, built with the shared BLAS-1 wrappers of krylov_oracle_impl.h by adjoint.mk into a library
that links against the shared oracle library and uses its test knobs: oracle.dot_mode (re-exported here) switches the
dot products of these solvers as of every other family.  The adjoint problem
generators of test/test_utils.jl:212-283 (and the ODE / PDE discretizations of test/get_div_grad.jl:27-138 they use)
are restated here.  Parity pinning: tests/test_oracle_adjoint.py and tests/golden/oracle_adjoint.json (frozen
histories).
"""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess

import numpy as np
import scipy.sparse as sp

from oracle import oracle as _shared
from oracle.oracle import (_ITER_CB, Stats, _csr, _opts, _p, _suf, _vec, bc_breakdown, dot_mode,  # noqa: F401
                           kron_unsymmetric)

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
_SOURCES = ("krylov_oracle_adjoint.c", "krylov_oracle_adjoint.h", "krylov_oracle_impl.h", "adjoint.mk",
            "libkrylov_oracle.so")


def build(force: bool = False) -> str:
    """Compile oracle/libkrylov_oracle_adjoint.so with adjoint.mk (when missing or older than its sources), after the
    shared oracle library it links against."""
    _shared.build()
    so = os.path.join(_HERE, "libkrylov_oracle_adjoint.so")
    srcs = [os.path.join(_HERE, f) for f in _SOURCES]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "adjoint.mk"])
    return so


def lib():
    global _LIB
    if _LIB is None:
        _shared.lib()                 # the shared library first: this one resolves the test knobs against it
        _LIB = C.CDLL(build())
    return _LIB


def _adjoint(tri, A, b, c, x0, y0, transfer, timemax, callback, dtype, kw):
    suf, _ = _suf(dtype)
    A = sp.csr_matrix(A)
    m, n = A.shape
    _, rp, ci, va = _csr(A, dtype)
    _, trp, tci, tva = _csr(A.T, dtype)
    b, c, x0, y0 = (_vec(v, dtype) for v in (b, c, x0, y0))
    if (x0 is None) != (y0 is None):
        raise ValueError("pass both x0 and y0, or neither")
    o = _opts(n, kw, 1 << 22)
    itmax = o.itmax if o.itmax > 0 else (m + n if tri else 2 * n)
    o.hist_cap = min(itmax + 2, 1 << 22)
    x, t = np.zeros(n, dtype), np.zeros(m, dtype)
    rres, sres = np.zeros(o.hist_cap, dtype), np.zeros(o.hist_cap, dtype)
    nsres, sp_, sd_ = C.c_int(0), C.c_int(0), C.c_int(0)
    st = Stats()
    cb = _ITER_CB(lambda it, _u: int(bool(callback(it)))) if callback is not None else _ITER_CB()
    f = getattr(lib(), f"oracle_adjoint_{suf}")
    f.argtypes = [C.c_int] * 3 + [C.c_void_p] * 10 + [C.c_int, C.c_double, _ITER_CB] + [C.c_void_p] * 9
    f(int(tri), m, n, _p(rp), _p(ci), _p(va), _p(trp), _p(tci), _p(tva), _p(b), _p(c), _p(x0), _p(y0), int(transfer),
      -1.0 if math.isinf(timemax) else float(timemax), cb, None, C.cast(C.byref(o), C.c_void_p), _p(x), _p(t), _p(rres),
      _p(sres), C.cast(C.byref(nsres), C.c_void_p), C.cast(C.byref(sp_), C.c_void_p), C.cast(C.byref(sd_), C.c_void_p),
      C.cast(C.byref(st), C.c_void_p))
    stats = dict(niter=st.niter, solved=bool(st.solved), solved_primal=bool(sp_.value), solved_dual=bool(sd_.value),
                 status=st.status.decode("utf-8"), residuals_primal=rres[:min(st.nres, o.hist_cap)].copy(),
                 residuals_dual=sres[:min(nsres.value, o.hist_cap)].copy())
    return x, t, stats


def bilqr(A, b, c, x0=None, y0=None, transfer_to_bicg=True, timemax=math.inf, callback=None, dtype=np.float64, **kw):
    """bilqr! (src/bilqr.jl:115-484) -> (x, y, stats).  callback(iter) -> bool stops the solve when true."""
    return _adjoint(False, A, b, c, x0, y0, transfer_to_bicg, timemax, callback, dtype, kw)


def trilqr(A, b, c, x0=None, y0=None, transfer_to_usymcg=True, timemax=math.inf, callback=None, dtype=np.float64, **kw):
    """trilqr! (src/trilqr.jl:114-461) -> (x, y, stats); A is m x n, b has m entries, c n."""
    return _adjoint(True, A, b, c, x0, y0, transfer_to_usymcg, timemax, callback, dtype, kw)


# ---- problem generators of test/test_utils.jl:212-283 (real case) -------------------------------------------------
def _tri_band(n, m):
    """[i == j ? 10 : i < j ? 1 : -1 for i=1:n, j=1:m]"""
    i, j = np.indices((n, m))
    return np.where(i == j, 10.0, np.where(i < j, 1.0, -1.0))


def underdetermined_adjoint(n=100, m=200):
    """test/test_utils.jl:212-218: A n x m (n < m), b = A [1..m], c = Aᵀ [-n..-1]."""
    A = _tri_band(n, m)
    return sp.csr_matrix(A), A @ np.arange(1.0, m + 1), A.T @ np.arange(-float(n), 0.0)


def square_adjoint(n=100):
    """test/test_utils.jl:221-226"""
    A = _tri_band(n, n)
    return sp.csr_matrix(A), A @ np.arange(1.0, n + 1), A.T @ np.arange(-float(n), 0.0)


def rectangular_adjoint(n=10, m=25):
    """test/test_utils.jl:229-234: Aᴴ, c = over_inconsistent(m, n); A = (Aᴴ)ᴴ (n x m), b = A 1."""
    At = np.ones((m, n))
    c = np.array([-1.0 if i == 1 else float(i) for i in range(1, m + 1)])
    A = At.T
    return sp.csr_matrix(A), A @ np.ones(m), c


def overdetermined_adjoint(n=200, m=100):
    """test/test_utils.jl:237-243: A n x m (n > m)."""
    A = _tri_band(n, m)
    return sp.csr_matrix(A), A @ np.arange(1.0, m + 1), A.T @ np.arange(-float(n), 0.0)


def ode(n, f, g, coefs):
    """ODE (test/get_div_grad.jl:28-63): central differences on ]0, 1[ with n interior points."""
    x1, x2, x3 = coefs
    dx = 1.0 / (n + 1)
    grid = np.array([i * dx for i in range(1, n + 1)])
    A = sp.lil_matrix((n, n))
    for i in range(n):
        if i != 0:
            A[i, i - 1] = x1 / (dx * dx) - x2 / (2 * dx)
        A[i, i] = -2 * x1 / (dx * dx) + x3
        if i != n - 1:
            A[i, i + 1] = x1 / (dx * dx) + x2 / (2 * dx)
    return sp.csr_matrix(A), f(grid), g(grid)


def pde(n, m, f, g, coefs):
    """PDE (test/get_div_grad.jl:66-138): central differences on ]0, 1[² with n x m interior points."""
    a, b_, c, d, e = coefs
    dx, dy = 1.0 / (n + 1), 1.0 / (m + 1)
    xs = [i * dx for i in range(1, n + 1)]
    ys = [j * dy for j in range(1, m + 1)]
    A = sp.lil_matrix((n * m, n * m))
    for i in range(n):
        for j in range(m):
            k = i + n * j
            A[k, k] = -2 * a / (dx * dx) - 2 * b_ / (dy * dy) + e
            if i >= 1:
                A[k, k - 1] = a / (dx * dx) - c / (2 * dx)
            if i <= n - 2:
                A[k, k + 1] = a / (dx * dx) + c / (2 * dx)
            if j >= 1:
                A[k, k - n] = b_ / (dy * dy) - d / (2 * dy)
            if j <= m - 2:
                A[k, k + n] = b_ / (dy * dy) + d / (2 * dy)
    bv = np.zeros(n * m)
    cv = np.zeros(n * m)
    for i in range(n):
        for j in range(m):
            bv[i + n * j] = f(xs[i], ys[j])
            cv[i + n * j] = g(xs[i], ys[j])
    return sp.csr_matrix(A), bv, cv


def adjoint_ode(n=50):
    """test/test_utils.jl:246-264"""
    x1 = x2 = x3 = 1.0
    f = lambda x: (-x1 * math.pi * math.pi + x3) * np.sin(math.pi * x) + (x2 * math.pi) * np.cos(math.pi * x)  # noqa: E731
    return ode(n, f, np.exp, [x1, x2, x3])


def adjoint_pde(n=50, m=50):
    """test/test_utils.jl:267-283"""
    k1, k2, k3 = 5.0, 20.0, 0.0

    def f(x, y):
        return ((-2 * k1 * math.pi * math.pi + k3) * math.sin(math.pi * x) * math.sin(math.pi * y)
                + k2 * math.pi * math.cos(math.pi * x) * math.sin(math.pi * y)
                + k2 * math.pi * math.sin(math.pi * x) * math.cos(math.pi * y))
    return pde(n, m, f, lambda x, y: math.exp(x + y), [k1, k1, k2, k2, k3])
