"""Problem generators of the CPU restatement of lnlq!, and its solver functions -- TEST INFRASTRUCTURE ONLY.

Same status as oracle/oracle.py (only tests/ may import it; the product never does).  The solver lives in
krylov_oracle_lnlq.h, built into the oracle library that oracle.py builds and loads, so oracle.dot_mode (re-exported
here) switches the dot products of this solver as of every other family.  The generators of test/test_utils.jl
that the reference's test/test_lnlq.jl uses are re-exported from leastnorm_oracle.py, which restates them for CRAIG
and CRAIGMR.
Parity pinning: tests/test_oracle_lnlq.py and tests/golden/oracle_lnlq.json (frozen histories).
"""
from __future__ import annotations

from oracle.leastnorm_oracle import (over_consistent, regularization, saddle_point, small_ln, small_sp,  # noqa: F401
                                     small_sqd, sqd, square_consistent, two_preconditioners, under_consistent,
                                     zero_rhs)
from oracle.oracle import dot_mode, lib, lnlq  # noqa: F401
