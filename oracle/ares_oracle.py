"""Problem generators of the CPU restatement of car! / minares!, and its solver functions -- TEST INFRASTRUCTURE ONLY.

Same status as oracle/oracle.py (only tests/ may import it; the product never does).  The solvers live in
krylov_oracle_ares.h, built into the oracle library that oracle.py builds and loads.  The symmetric problem generators of test/test_utils.jl that test/test_car.jl and test/test_minares.jl use are
re-exported from oracle.py; symmetric_inconsistent (test/test_utils.jl:128-132) is restated here.  Parity pinning:
tests/test_oracle_car_minares.py and tests/golden/oracle_car_minares.json (frozen histories).
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

from oracle.oracle import (almost_singular, car, cartesian_poisson, dot_mode, get_div_grad, lib, minares,  # noqa: F401
                           singular_consistent, sparse_laplacian, square_inconsistent, square_preconditioned,
                           symmetric_definite, symmetric_indefinite, zero_rhs)


def symmetric_inconsistent():
    """test/test_utils.jl:128-132: a symmetric, singular 4 x 4 system whose b is outside the range of A."""
    A = np.array([[3.0, 2.0, -1.0, 5.0], [2.0, -2.0, 4.0, 0.0], [-1.0, 4.0, 1.0, 3.0], [5.0, 0.0, 3.0, 5.0]])
    return sp.csr_matrix(A), np.array([1.0, -8.0, 5.0, 2.0])
