"""The CPU oracle's lsqr / lsmr (oracle/krylov_oracle_lsq.h) against the reference's own known-answer tests
(test/test_lsqr.jl, test/test_lsmr.jl, real case, same assertions and tolerance), and against the frozen histories of
tests/golden/oracle_lsq.json (tests/golden/gen_golden_lsq.py)."""
import json
import os

import numpy as np
import pytest
import scipy.sparse as sp

from parity import golden_module

HERE = os.path.dirname(os.path.abspath(__file__))
TOL = 1.0e-4                                                         # lsqr_tol / lsmr_tol
G = golden_module("lsq")
GOLD = json.load(open(os.path.join(HERE, "golden", "oracle_lsq.json")))
SOLVERS = ["lsqr", "lsmr"]


@pytest.fixture(scope="module")
def LO():
    """The CPU restatement of lsqr! / lsmr! and its problem generators (oracle/lsq_oracle.py; test infrastructure)."""
    from oracle import lsq_oracle
    lsq_oracle.lib()
    return lsq_oracle


@pytest.mark.parametrize("solver", SOLVERS)
@pytest.mark.parametrize("npower", [1, 2, 3, 4])
def test_lstp_with_and_without_regularization(LO, solver, npower):
    b, A, *_ = LO.lsq_test(40, 40, 4, npower, 0)
    x, st = getattr(LO, solver)(A, b)
    r = b - A @ x
    assert np.linalg.norm(A.T @ r) / np.linalg.norm(b) <= TOL and st["solved"]
    lam = 1.0e-3
    x, st = getattr(LO, solver)(A, b, lambda_=lam)
    r = b - A @ x
    assert np.linalg.norm(A.T @ r - lam * lam * x) / np.linalg.norm(b) <= TOL and st["solved"]


@pytest.mark.parametrize("solver", SOLVERS)
def test_trust_region(LO, solver):
    A = sp.csr_matrix(np.array([[i / j - j / i for j in range(1, 7)] for i in range(1, 11)]))
    b = A @ np.ones(6)
    x, _ = getattr(LO, solver)(A, b)
    radius = 0.75 * np.linalg.norm(x)
    x, st = getattr(LO, solver)(A, b, radius=radius)
    assert st["solved"] and abs(radius - np.linalg.norm(x)) <= TOL * radius


@pytest.mark.parametrize("solver", SOLVERS)
def test_zero_rhs(LO, solver):
    A, b = LO.zero_rhs()
    x, st = getattr(LO, solver)(A, b)
    assert np.linalg.norm(x) == 0 and st["status"] == "x is a zero-residual solution"


@pytest.mark.parametrize("solver", SOLVERS)
def test_preconditioners(LO, solver):
    A, b, M, N = LO.two_preconditioners()
    x, st = getattr(LO, solver)(A, b, M=M, N=N)
    r = b - A @ x
    assert np.sqrt(r @ (M * r)) / np.linalg.norm(b) <= TOL and st["solved"]


@pytest.mark.parametrize("solver", SOLVERS)
def test_regularization_saddle_point_sqd(LO, solver):
    A, b, lam = LO.regularization()
    x, _ = getattr(LO, solver)(A, b, lambda_=lam)
    r = b - A @ x
    assert np.linalg.norm(A.T @ r - lam ** 2 * x) / np.linalg.norm(b) <= TOL
    A, b, D = LO.saddle_point()
    x, _ = getattr(LO, solver)(A, b, M=1 / D)
    r = (b - A @ x) / D
    assert np.linalg.norm(A.T @ r) / np.linalg.norm(b) <= TOL
    A, b, M, N = LO.sqd()
    x, _ = getattr(LO, solver)(A, b, M=1 / M, N=1 / N, sqd=True)
    r = (b - A @ x) / M
    assert np.linalg.norm(A.T @ r - N * x) / np.linalg.norm(b) <= TOL
    lam = 4.0
    x, _ = getattr(LO, solver)(A, b, M=1 / M, N=1 / N, lambda_=lam)
    r = (b - A @ x) / M
    assert np.linalg.norm(A.T @ r - lam ** 2 * N * x) / np.linalg.norm(b) <= TOL
    with pytest.raises(ValueError):
        getattr(LO, solver)(A, b, sqd=True, lambda_=1.0)


@pytest.mark.parametrize("solver", SOLVERS)
def test_float32_restatement(LO, solver):
    b, A, *_ = LO.lsq_test(40, 40, 4, 1, 0)
    x, st = getattr(LO, solver)(A.astype(np.float32), b.astype(np.float32), dtype=np.float32)
    r = b - A @ x.astype(np.float64)
    assert st["solved"] and np.linalg.norm(A.T @ r) / np.linalg.norm(b) <= 1e-3


@pytest.mark.parametrize("key", sorted(GOLD))
def test_oracle_matches_golden(LO, key):
    solver, name = key.split("/")
    cs = G.cases()
    if name == "trust_region":
        A, b, _ = cs["trust_free"]
        kw = dict(radius=G.trust_radius(solver))
    else:
        A, b, kw = cs[name]
    x, st = getattr(LO, solver)(A, b, **kw)
    g = GOLD[key]
    assert (st["niter"], st["status"], st["solved"], st["inconsistent"]) == (g["niter"], g["status"], g["solved"], g["inconsistent"])
    assert np.allclose(st["residuals"], g["residuals"], rtol=1e-12, atol=0)
    assert np.allclose(st["Aresiduals"], g["Aresiduals"], rtol=1e-12, atol=1e-300)
    assert np.allclose(x[:6], g["x_head"], rtol=1e-10, atol=1e-14)


def test_generators_match_the_reference_formulas(LO):
    b, A, D, HY, HZ, Acond, rnorm = LO.lsq_test(40, 40, 4, 2, 0)
    assert A.shape == (40, 40) and np.allclose(HY @ HY, np.eye(40)) and np.allclose(HZ @ HZ, np.eye(40))
    d = np.diag(D)
    assert np.isclose(d[0], 0.01) and d[-1] == 1.0 and np.isclose(Acond, 100.0)
    x = 40 - np.arange(1, 41)
    assert np.allclose(b - A @ x, HY @ np.r_[HZ @ x / d][:40])
    A, b, lam = LO.regularization()
    assert A[1, 0] == 2 ** 2 * 1 + (-1) * 5 * 1 and lam == 4.0
