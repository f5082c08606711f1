"""Problem generators of the CPU restatement of lsqr! / lsmr!, and its solver functions -- TEST INFRASTRUCTURE ONLY.

Same status as oracle/oracle.py (only tests/ may import it; the product never does).  The solvers live in
krylov_oracle_lsq.h, built into the oracle library that oracle.py builds and loads.  The problem generators restate test/gen_lsq.jl and the least-squares helpers of test/test_utils.jl; the square
generators the reference's LSQR / LSMR tests also use (zero_rhs, two_preconditioners, ddx) are re-exported from
oracle.py.  Parity pinning: tests/test_oracle_lsq.py (the reference's assertions of test/test_lsqr.jl and
test/test_lsmr.jl) and tests/golden/oracle_lsq.json (frozen histories).
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

from oracle.oracle import ddx, lib, lsmr, lsqr, two_preconditioners, zero_rhs  # noqa: F401


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
