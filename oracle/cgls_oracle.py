"""Problem generators of the CPU restatement of cgls! / crls! / lslq!, and its solver functions -- TEST INFRASTRUCTURE ONLY.

Same status as oracle/oracle.py (only tests/ may import it; the product never does).  The solvers live in
krylov_oracle_cgls.h and krylov_oracle_lslq.h, on the rectangular products of krylov_oracle_lsq.h, built into the
oracle library that oracle.py builds and loads.  The least-squares problem generators are re-exported from
lsq_oracle.py.  Parity pinning: tests/test_oracle_cgls.py (the reference's assertions of test/test_cgls.jl and
test/test_crls.jl) and tests/golden/oracle_cgls.json (frozen histories).
"""
from __future__ import annotations

import numpy as np  # noqa: F401

from oracle.lsq_oracle import lsq_test, lstp, regularization, saddle_point, sqd  # noqa: F401
from oracle.oracle import cgls, crls, lib, lslq, zero_rhs  # noqa: F401
