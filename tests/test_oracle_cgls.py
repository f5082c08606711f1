"""The CPU oracle's cgls / crls (oracle/krylov_oracle_cgls.h) against the reference's own known-answer tests
(test/test_cgls.jl, test/test_crls.jl, real case, same assertions and tolerance), and against the frozen histories of
tests/golden/oracle_cgls.json (tests/golden/gen_golden_cgls.py)."""
import json
import os

import numpy as np
import pytest

from parity import golden_module

HERE = os.path.dirname(os.path.abspath(__file__))
TOL = 1.0e-5                                                         # cgls_tol / crls_tol
G = golden_module("cgls")
GOLD = json.load(open(os.path.join(HERE, "golden", "oracle_cgls.json")))
SOLVERS = ["cgls", "crls"]


@pytest.fixture(scope="module")
def CO():
    """The CPU restatement of cgls! / crls! (oracle/cgls_oracle.py; test infrastructure)."""
    from oracle import cgls_oracle
    cgls_oracle.lib()
    return cgls_oracle


@pytest.mark.parametrize("solver", SOLVERS)
@pytest.mark.parametrize("npower", [1, 2, 3, 4])
def test_lstp_with_and_without_regularization(CO, solver, npower):
    b, A, *_ = CO.lsq_test(40, 40, 4, npower, 0)
    x, st = getattr(CO, solver)(A, b)
    assert np.linalg.norm(A.T @ (A @ x - b)) / np.linalg.norm(b) <= TOL and st["solved"]
    lam = 1.0e-3
    x, st = getattr(CO, solver)(A, b, lambda_=lam)
    assert np.linalg.norm(A.T @ (A @ x - b) + lam * x) / np.linalg.norm(b) <= TOL and st["solved"]


@pytest.mark.parametrize("solver", SOLVERS)
def test_preconditioner_and_trust_region(CO, solver):
    from oracle import lsq_oracle
    A, b, D = lsq_oracle.saddle_point()
    Minv = 1 / D
    x, _ = getattr(CO, solver)(A, b, M=Minv)
    resid = np.linalg.norm(A.T @ (Minv * (A @ x - b))) / np.sqrt(b @ (Minv * b))
    assert resid <= TOL
    x, st = getattr(CO, solver)(A, b, M=D, ldiv=True)                # the same M applied by division
    assert np.linalg.norm(A.T @ (Minv * (A @ x - b))) / np.sqrt(b @ (Minv * b)) <= TOL
    x, _ = getattr(CO, solver)(A, b)
    radius = 0.75 * np.linalg.norm(x)
    x, st = getattr(CO, solver)(A, b, radius=radius)
    assert st["solved"] and abs(radius - np.linalg.norm(x)) <= TOL * radius
    assert st["status"] == "on trust-region boundary"


@pytest.mark.parametrize("solver", SOLVERS)
def test_zero_rhs(CO, solver):
    A, b = CO.zero_rhs()
    x, st = getattr(CO, solver)(A, b)
    assert np.linalg.norm(x) == 0 and st["status"] == "x is a zero-residual solution" and st["niter"] == 0


@pytest.mark.parametrize("solver", SOLVERS)
def test_adjoint_residual_zero(CO, solver):
    """Aᴴb = 0 (b orthogonal to the range of A): x = 0 at iteration 0."""
    import scipy.sparse as sp
    A = sp.csr_matrix(sp.vstack([sp.identity(5), sp.csr_matrix((2, 5))]))
    b = np.zeros(7)
    b[6] = 1.0
    x, st = getattr(CO, solver)(A, b)
    assert st["niter"] == 0 and st["status"] == "solution good enough given atol and rtol" and not x.any()


def test_crls_positive_semidefinite():
    """test/test_crls.jl's semi-definite case (fixed orthogonal factors) and a forced zero-curvature exit."""
    from oracle import cgls_oracle as CO
    A, b = G.psd_problem()
    x, st = CO.crls(A, b, radius=10.0)
    assert st["solved"] and st["status"] in ("zero-curvature encountered", "on trust-region boundary")
    assert np.linalg.norm(x) <= 10.0 * (1 + 1e-12)
    b, A, *_ = CO.lsq_test(40, 40, 4, 1, 0)
    x, st = CO.crls(A, b, radius=1.0e3, atol=1.0, rtol=0.0)
    assert st["status"] == "zero-curvature encountered" and st["niter"] == 0 and np.linalg.norm(x) > 0


@pytest.mark.parametrize("solver", SOLVERS)
def test_float32_restatement(CO, solver):
    b, A, *_ = CO.lsq_test(40, 40, 4, 1, 0)
    x, st = getattr(CO, solver)(A.astype(np.float32), b.astype(np.float32), dtype=np.float32)
    assert st["solved"] and np.linalg.norm(A.T @ (A @ x.astype(np.float64) - b)) / np.linalg.norm(b) <= 1e-3


def _golden_case(key):
    solver, name = key.split("/")
    cs = G.cases()
    if name == "trust_region":
        A, b, _ = cs["trust_free"]
        return solver, A, b, dict(radius=G.trust_radius(solver))
    if name == "zero_curvature":
        A, b, _ = cs["lstp1"]
        return solver, A, b, dict(radius=1.0e3, atol=1.0, rtol=0.0)
    A, b, kw = cs[name]
    return solver, A, b, kw


@pytest.mark.parametrize("key", sorted(GOLD))
def test_oracle_matches_golden(CO, key):
    solver, A, b, kw = _golden_case(key)
    x, st = getattr(CO, solver)(A, b, **kw)
    g = GOLD[key]
    assert (st["niter"], st["status"], st["solved"], st["inconsistent"]) == (g["niter"], g["status"], g["solved"], g["inconsistent"])
    assert np.allclose(st["residuals"], g["residuals"], rtol=1e-12, atol=0)
    assert np.allclose(st["Aresiduals"], g["Aresiduals"], rtol=1e-12, atol=1e-300)
    assert np.allclose(x[:6], g["x_head"], rtol=1e-10, atol=1e-14)
