"""Problem generators of the CPU restatement of bilq! / qmr!, and its solver functions -- TEST INFRASTRUCTURE ONLY.

Same status as oracle/oracle.py (only tests/ may import it; the product never does).  The solvers live in
krylov_oracle_biorth.h, built into the oracle library that oracle.py builds and loads.  The square problem generators of test/test_utils.jl that test/test_bilq.jl and test/test_qmr.jl use are
re-exported from oracle.py; unsymmetric_breakdown (test/test_utils.jl:196-201) is restated here.  Parity pinning:
tests/test_oracle_bilq_qmr.py and tests/golden/oracle_bilq_qmr.json (frozen histories).
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

from oracle.oracle import (bc_breakdown, bilq, dot_mode, kron_unsymmetric, lib, nonsymmetric_definite,  # noqa: F401
                           nonsymmetric_indefinite, polar_poisson, qmr, sparse_laplacian, square_preconditioned,
                           symmetric_definite, symmetric_indefinite, two_preconditioners, zero_rhs)


def unsymmetric_breakdown():
    """test/test_utils.jl:196-201: b and c start a Lanczos biorthogonalization that breaks down (pᴴq = 0)."""
    return sp.csr_matrix(np.array([[0.0, 1.0], [-1.0, 0.0]])), np.array([1.0, 0.0]), np.array([-1.0, 0.0])
