"""Problem generators of the CPU restatement of bilqr! / trilqr!, and its solver functions -- TEST INFRASTRUCTURE ONLY.

Same status as oracle/oracle.py (only tests/ may import it; the product never does).  The solvers live in
krylov_oracle_adjoint.h, built into the oracle library that oracle.py builds and loads, so oracle.dot_mode
(re-exported here) switches the dot products of these solvers as of every other family.  The adjoint problem
generators of test/test_utils.jl:212-283 (and the ODE / PDE discretizations of test/get_div_grad.jl:27-138 they use)
are restated here.  Parity pinning: tests/test_oracle_adjoint.py and tests/golden/oracle_adjoint.json (frozen
histories).
"""
from __future__ import annotations

import math

import numpy as np
import scipy.sparse as sp

from oracle.oracle import bc_breakdown, bilqr, dot_mode, kron_unsymmetric, lib, trilqr  # noqa: F401


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
