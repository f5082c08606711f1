"""Problem generators of the CPU restatement of cgne! and crmr!, and its solver functions -- TEST INFRASTRUCTURE ONLY.

Same status as oracle/oracle.py (only tests/ may import it; the product never does).  The solvers live in
krylov_oracle_cgne.h, built into the oracle library that oracle.py builds and loads, so oracle.dot_mode (re-exported
here) switches the dot products of these solvers as of every other family.  The generators of test/test_utils.jl
that the reference's test/test_cgne.jl and test/test_crmr.jl use are re-exported from leastnorm_oracle.py and
oracle.py.
Parity pinning: tests/test_oracle_cgne_crmr.py and tests/golden/oracle_cgne_crmr.json (frozen histories).
"""
from __future__ import annotations

from oracle.leastnorm_oracle import (over_consistent, over_inconsistent, small_sp, square_consistent,  # noqa: F401
                                     square_inconsistent, under_consistent, under_inconsistent, zero_rhs)
from oracle.oracle import cgne, crmr, dot_mode, lib, square_preconditioned  # noqa: F401
