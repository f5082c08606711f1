"""The CPU oracle's lslq (oracle/krylov_oracle_lslq.h) against the reference's own known-answer tests
(test/test_lslq.jl, real case, same assertions and tolerance), and against the frozen histories of
tests/golden/oracle_lslq.json (tests/golden/gen_golden_lslq.py)."""
import importlib.util
import json
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
TOL = 1.0e-5                                                         # lslq_tol
_spec = importlib.util.spec_from_file_location("gen_golden_lslq", os.path.join(HERE, "golden", "gen_golden_lslq.py"))
G = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(G)
GOLD = json.load(open(os.path.join(HERE, "golden", "oracle_lslq.json")))


@pytest.fixture(scope="module")
def CO():
    from oracle import cgls_oracle
    cgls_oracle.lib()
    return cgls_oracle


def radau_problem(seed=0):
    """test/test_lslq.jl's smallest-singular-value case with fixed orthogonal factors: A = U [Σ; 0] Vᵀ, Σ = diag(1:4)."""
    rng = np.random.default_rng(seed)
    U, _ = np.linalg.qr(rng.random((6, 6)))
    V, _ = np.linalg.qr(rng.random((4, 4)))
    A = U @ np.vstack([np.diag([1.0, 2.0, 3.0, 4.0]), np.zeros((2, 4))]) @ V.T
    return A, np.ones(6)


@pytest.mark.parametrize("npower", [1, 2, 3, 4])
def test_lstp_with_and_without_regularization(CO, npower):
    b, A, *_ = CO.lsq_test(40, 40, 4, npower, 0)
    x, st = CO.lslq(A, b)
    assert np.linalg.norm(A.T @ (b - A @ x)) / np.linalg.norm(b) <= TOL and st["solved"]
    lam = 1.0e-3
    x, st = CO.lslq(A, b, lambda_=lam)
    assert np.linalg.norm(A.T @ (b - A @ x) - lam * lam * x) / np.linalg.norm(b) <= TOL and st["solved"]


def test_error_bounds(CO):
    b, A, *_ = CO.lsq_test(40, 40, 4, 4, 0)
    _, st = CO.lslq(A, b, sigma=1.0)
    assert st["error_with_bnd"]
    A, b = CO.zero_rhs()
    x, st = CO.lslq(A, b)
    assert np.linalg.norm(x) == 0 and st["status"] == "x is a zero-residual solution"
    import scipy.sparse as sp
    A, b = radau_problem()
    x_exact = np.linalg.lstsq(A, b, rcond=None)[0]
    for t in (False, True):
        x, st = CO.lslq(sp.csr_matrix(A), b, sigma=1.0 - 1.0e-10, transfer_to_lsqr=t)
        assert abs(st["err_ubnds_lq"][-1]) <= np.sqrt(2.2e-16) and abs(st["err_ubnds_cg"][-1]) <= np.sqrt(2.2e-16)
        assert np.linalg.norm(x - x_exact) <= np.sqrt(2.2e-16) * np.linalg.norm(x_exact)


@pytest.mark.parametrize("t", [False, True])
def test_preconditioners_regularization_sqd(CO, t):
    from oracle import lsq_oracle as L
    A, b, M, N = L.two_preconditioners()
    x, st = CO.lslq(A, b, M=M, N=N, transfer_to_lsqr=t)
    r = b - A @ x
    assert np.sqrt(r @ (M * r)) / np.linalg.norm(b) <= TOL and st["solved"]
    A, b, lam = L.regularization()
    x, _ = CO.lslq(A, b, lambda_=lam, transfer_to_lsqr=t)
    assert np.linalg.norm(A.T @ (b - A @ x) - lam ** 2 * x) / np.linalg.norm(b) <= TOL
    A, b, D = L.saddle_point()
    x, _ = CO.lslq(A, b, M=1 / D, transfer_to_lsqr=t)
    assert np.linalg.norm(A.T @ ((b - A @ x) / D)) / np.linalg.norm(b) <= TOL
    A, b, M, N = L.sqd()
    x, _ = CO.lslq(A, b, M=1 / M, N=1 / N, sqd=True, transfer_to_lsqr=t)
    assert np.linalg.norm(A.T @ ((b - A @ x) / M) - N * x) / np.linalg.norm(b) <= TOL
    x, _ = CO.lslq(A, b, M=1 / M, N=1 / N, lambda_=4.0, transfer_to_lsqr=t)
    assert np.linalg.norm(A.T @ ((b - A @ x) / M) - 16.0 * N * x) / np.linalg.norm(b) <= TOL
    with pytest.raises(ValueError):
        CO.lslq(A, b, sqd=True, lambda_=1.0)


def test_adjoint_residual_zero(CO):
    import scipy.sparse as sp
    A = sp.csr_matrix(sp.vstack([sp.identity(5), sp.csr_matrix((2, 5))]))
    b = np.zeros(7)
    b[6] = 1.0
    x, st = CO.lslq(A, b)
    assert st["niter"] == 0 and st["status"] == "x is a minimum least-squares solution" and not x.any()
    assert list(st["residuals"]) == [1.0] and list(st["Aresiduals"]) == [0.0]


@pytest.mark.parametrize("key", sorted(GOLD))
def test_oracle_matches_golden(CO, key):
    A, b, kw = G.cases()[key.split("/")[1]]
    x, st = CO.lslq(A, b, **kw)
    g = GOLD[key]
    assert (st["niter"], st["status"], st["solved"], st["inconsistent"], st["error_with_bnd"]) == \
        (g["niter"], g["status"], g["solved"], g["inconsistent"], g["error_with_bnd"])
    for k in G.KEYS:
        assert len(st[k]) == len(g[k]) and np.allclose(st[k], g[k], rtol=1e-12, atol=1e-300), k
    assert np.allclose(x[:6], g["x_head"], rtol=1e-10, atol=1e-14)
