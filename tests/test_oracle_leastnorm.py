"""The CPU oracle's craig and craigmr (oracle/krylov_oracle_leastnorm.h) against the reference's own assertions
(test/test_craig.jl, test/test_craigmr.jl, real case, same tolerance), and against the frozen histories of
tests/golden/oracle_leastnorm.json (tests/golden/gen_golden_leastnorm.py)."""
import importlib.util
import json
import os

import numpy as np
import pytest

from oracle import leastnorm_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
TOL = 1.0e-6                                                         # craig_tol / craigmr_tol
_spec = importlib.util.spec_from_file_location("gen_golden_leastnorm", os.path.join(HERE, "golden", "gen_golden_leastnorm.py"))
G = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(G)
GOLD = json.load(open(os.path.join(HERE, "golden", "oracle_leastnorm.json")))
SOLVERS = ["craig", "craigmr"]


def _min_norm(A, b, x):
    """check_min_norm.jl (λ = 0): the least-norm solution from a QR factorization of Aᵀ."""
    Q, R = np.linalg.qr(A.toarray().T)
    xmin = Q @ np.linalg.lstsq(R.T, b, rcond=None)[0]             # R' \ b: least squares when R is wide
    return x, xmin, np.linalg.norm(xmin)


@pytest.mark.parametrize("solver", SOLVERS)
@pytest.mark.parametrize("name", ["under_consistent", "square_consistent", "over_consistent"])
def test_consistent_systems(solver, name):
    A, b = getattr(O, name)()
    x, y, st = getattr(O, solver)(A, b)
    assert np.linalg.norm(x - A.T @ y) <= TOL * np.linalg.norm(x)
    assert np.linalg.norm(b - A @ x) / np.linalg.norm(b) <= TOL
    assert st["solved"]
    xI, xmin, xmin_norm = _min_norm(A, b, x)
    assert np.linalg.norm(xI - xmin) <= np.linalg.cond(A.toarray()) * TOL * xmin_norm


@pytest.mark.parametrize("name", ["under_inconsistent", "square_inconsistent", "over_inconsistent"])
def test_craig_inconsistent_systems(name):
    A, b = getattr(O, name)()
    _, _, st = O.craig(A, b)
    assert st["inconsistent"] or st["status"] == "condition number exceeds tolerance"


@pytest.mark.parametrize("name", ["under_inconsistent", "square_inconsistent", "over_inconsistent"])
def test_craigmr_inconsistent_systems(name):
    A, b = getattr(O, name)()
    x, y, st = O.craigmr(A, b, history=True)
    assert np.linalg.norm(x - A.T @ y) <= TOL * np.linalg.norm(x)
    assert st["inconsistent"]
    assert st["Aresiduals"][-1] <= TOL


@pytest.mark.parametrize("solver", SOLVERS)
def test_zero_rhs(solver):
    A, b = O.zero_rhs()
    x, y, st = getattr(O, solver)(A, b, lambda_=1.0e-3)
    assert np.linalg.norm(x) == 0 and np.linalg.norm(y) == 0
    assert st["status"] == "x is a zero-residual solution"


@pytest.mark.parametrize("solver", SOLVERS)
def test_regularization(solver):
    A, b, lam = O.regularization()
    x, y, _ = getattr(O, solver)(A, b, lambda_=lam)
    s = lam * y
    assert np.linalg.norm(b - (A @ x + lam * s)) / np.linalg.norm(b) <= TOL
    r2 = b - (A @ A.T @ y + lam ** 2 * y)
    assert np.linalg.norm(r2) / np.linalg.norm(b) <= TOL


@pytest.mark.parametrize("solver", SOLVERS)
def test_saddle_point_with_N(solver):
    A, b, D = O.saddle_point()
    x, y, _ = getattr(O, solver)(A, b, N=1.0 / D)
    assert np.linalg.norm(b - A @ x) / np.linalg.norm(b) <= TOL
    assert np.linalg.norm(b - A @ ((A.T @ y) / D)) / np.linalg.norm(b) <= TOL


@pytest.mark.parametrize("solver", SOLVERS)
def test_two_preconditioners(solver):
    A, b, Mi, Ni = O.two_preconditioners()
    x, y, _ = getattr(O, solver)(A, b, M=Mi, N=Ni, sqd=False)
    r = b - A @ x
    assert np.sqrt(r @ (Mi * r)) / np.linalg.norm(b) <= TOL
    assert np.linalg.norm(x - Ni * (A.T @ y)) <= TOL * np.linalg.norm(x)


@pytest.mark.parametrize("solver", SOLVERS)
def test_sqd_and_lambda4_with_M_N(solver):
    A, b, M, N = O.sqd()
    x, y, _ = getattr(O, solver)(A, b, M=1.0 / M, N=1.0 / N, sqd=True)
    assert np.linalg.norm(b - (A @ x + M * y)) / np.linalg.norm(b) <= TOL
    assert np.linalg.norm(b - (A @ ((A.T @ y) / N) + M * y)) / np.linalg.norm(b) <= TOL
    lam = 4.0
    x, y, _ = getattr(O, solver)(A, b, M=1.0 / M, N=1.0 / N, lambda_=lam)
    assert np.linalg.norm(b - (A @ x + lam ** 2 * M * y)) / np.linalg.norm(b) <= TOL
    assert np.linalg.norm(b - (A @ ((A.T @ y) / N) + lam ** 2 * M * y)) / np.linalg.norm(b) <= TOL


@pytest.mark.parametrize("solver", SOLVERS)
def test_small_least_norm(solver):
    A, b = O.small_ln()
    x, y, st = getattr(O, solver)(A, b)
    assert st["solved"]
    assert np.linalg.norm(b - A @ x) / np.linalg.norm(b) <= TOL
    assert np.linalg.norm(x - A.T @ y) <= TOL * np.linalg.norm(x)


def test_sqd_with_lambda_raises():
    A, b = O.small_ln()
    with pytest.raises(ValueError, match="sqd cannot be set to true if λ ≠ 0 !"):
        O.craig(A, b, sqd=True, lambda_=1.0)


def test_callback_stops_and_sees_the_iteration():
    A, b = O.over_consistent()
    seen = []
    _, _, st = O.craig(A, b, callback=lambda it: seen.append(it) or True)
    assert st["status"] == "user-requested exit" and seen == [1] and st["niter"] == 1


def test_craig_transfer_to_lsqr_moves_x_only_with_lambda():
    A, b, lam = O.regularization()
    x0, _, _ = O.craig(A, b, lambda_=lam)
    x1, _, _ = O.craig(A, b, lambda_=lam, transfer_to_lsqr=True)
    assert not np.array_equal(x0, x1)
    A, b = O.over_consistent()
    assert np.array_equal(O.craig(A, b)[0], O.craig(A, b, transfer_to_lsqr=True)[0])


@pytest.mark.parametrize("name", sorted(GOLD))
def test_oracle_reproduces_golden(name):
    solver, case = name.split("/")
    A, b, kw = G.cases()[case]
    x, y, st = G.run(solver, A, b, **kw)
    g = GOLD[name]
    assert (st["niter"], st["solved"], st["inconsistent"], st["status"]) == (g["niter"], g["solved"], g["inconsistent"],
                                                                            g["status"])
    assert [float(v) for v in st["residuals"]] == g["residuals"]
    assert [float(v) for v in st.get("Aresiduals", [])] == g["Aresiduals"]
    assert [float(v) for v in x[:6]] == g["x_head"] and [float(v) for v in y[:6]] == g["y_head"]
