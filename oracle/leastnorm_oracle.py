"""Problem generators of the CPU restatement of craig! / craigmr!, and its solver functions -- TEST INFRASTRUCTURE ONLY.

Same status as oracle/oracle.py (only tests/ may import it; the product never does).  The solvers live in
krylov_oracle_leastnorm.h, built into the oracle library that oracle.py builds and loads, so oracle.dot_mode
(re-exported here) switches the dot products of these solvers as of every other family.  The generators of
test/test_utils.jl that the reference's test/test_craig.jl and test/test_craigmr.jl use are restated here, or
re-exported from oracle.py and lsq_oracle.py.
Parity pinning: tests/test_oracle_leastnorm.py and tests/golden/oracle_leastnorm.json (frozen histories).
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

from oracle.lsq_oracle import regularization, saddle_point, sqd  # noqa: F401
from oracle.oracle import (craig, craigmr, dot_mode, lib, square_inconsistent, two_preconditioners,  # noqa: F401
                           zero_rhs)


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
