"""The CPU oracle's car and minares (oracle/krylov_oracle_ares.h) against the reference's own known-answer tests
(test/test_car.jl, test/test_minares.jl, real case, same assertions and tolerance), and against the frozen histories of
tests/golden/oracle_car_minares.json (tests/golden/gen_golden_car_minares.py)."""
import json
import os

import numpy as np
import pytest

from oracle import ares_oracle as O
from parity import golden_module

HERE = os.path.dirname(os.path.abspath(__file__))
TOL = 1.0e-6                                                         # car_tol / minares_tol
G = golden_module("car_minares")
GOLD = json.load(open(os.path.join(HERE, "golden", "oracle_car_minares.json")))


@pytest.mark.parametrize("name", ["symmetric_definite", "sparse_laplacian", "cartesian_poisson"])
def test_car_known_answer_problems_are_solved(name):
    A, b, _ = G.cases()["car"][name]
    x, st = O.car(A, b)
    assert np.linalg.norm(b - A @ x) / np.linalg.norm(b) <= TOL
    assert st["solved"]


def test_car_preconditioned_and_singular_consistent():
    A, b, M = O.square_preconditioned()
    x, st = O.car(A, b, M=M)
    assert np.linalg.norm(M * (b - A @ x)) / np.linalg.norm(M * b) <= TOL and st["solved"]
    A, b = O.singular_consistent()
    x, st = O.car(A, b)
    assert np.linalg.norm(b - A @ x) / np.linalg.norm(b) <= TOL and not st["inconsistent"]


@pytest.mark.parametrize("name", ["symmetric_definite", "symmetric_indefinite", "sparse_laplacian", "almost_singular"])
def test_minares_known_answer_problems_are_solved(name):
    A, b, _ = G.cases()["minares"][name]
    x, st = O.minares(A, b)
    resid = np.linalg.norm(b - A @ x) / np.linalg.norm(b)
    assert resid <= TOL * np.linalg.norm(A.toarray(), 2) * np.linalg.norm(x)
    assert st["solved"]


@pytest.mark.parametrize("name", ["square_inconsistent", "symmetric_inconsistent"])
def test_minares_inconsistent_systems_minimize_the_a_residual(name):
    A, b, _ = G.cases()["minares"][name]
    x, st = O.minares(A, b)
    r = b - A @ x
    assert np.linalg.norm(A @ r) / np.linalg.norm(A @ b) <= TOL


def test_minares_shifted_system():
    A, b = O.symmetric_indefinite()
    x, st = O.minares(A, b, lambda_=2.0)
    resid = np.linalg.norm(b - A @ x - 2.0 * x) / np.linalg.norm(b)
    assert resid <= TOL * np.linalg.norm(A.toarray(), 2) * np.linalg.norm(x) and st["solved"]


@pytest.mark.parametrize("solver", ["car", "minares"])
def test_zero_rhs(solver):
    A, b = O.zero_rhs()
    x, st = getattr(O, solver)(A, b)
    assert np.linalg.norm(x) == 0 and st["status"] == "x is a zero-residual solution" and st["niter"] == 0


@pytest.mark.parametrize("solver", ["car", "minares"])
def test_callback_exit_itmax_and_time_limit(solver):
    A, b = O.sparse_laplacian()
    f = getattr(O, solver)
    kw = dict(atol=0.0, rtol=0.0) if solver == "car" else dict(atol=0.0, rtol=0.0, artol=0.0)
    x, st = f(A, b, callback=lambda it: it >= 4, **kw)
    assert st["status"] == "user-requested exit" and st["niter"] == 4
    x, st = f(A, b, timemax=0.0)
    assert st["status"] == "time limit exceeded" and st["niter"] == 1
    x, st = f(A, b, itmax=5)
    assert st["status"] == "maximum number of iterations exceeded" and st["niter"] == 5


@pytest.mark.parametrize("solver", ["car", "minares"])
def test_warm_start_continues_from_x0(solver):
    A, b = O.sparse_laplacian()
    x0 = np.ones(A.shape[0])
    x, st = getattr(O, solver)(A, b, x0=x0)
    assert st["solved"] and np.linalg.norm(b - A @ x) / np.linalg.norm(b - A @ x0) <= 10 * TOL


def test_minares_artol_stops_on_the_a_residual():
    A, b = O.sparse_laplacian()
    _, st = O.minares(A, b, atol=0.0, rtol=0.0, artol=1e-3)
    ar = np.asarray(st["Aresiduals"])
    assert st["solved"] and ar[-1] <= 1e-3 * ar[0] and np.all(ar[:-1] > 1e-3 * ar[0])


@pytest.mark.parametrize("key", sorted(GOLD))
def test_matches_golden_history(key):
    solver, name = key.split("/")
    A, b, kw = G.cases()[solver][name]
    x, st = getattr(O, solver)(A, b, history=True, **kw)
    g = GOLD[key]
    assert (st["niter"], st["solved"], st["status"]) == (g["niter"], g["solved"], g["status"])
    np.testing.assert_array_equal(np.asarray(st["residuals"]), np.asarray(g["residuals"]))
    np.testing.assert_array_equal(np.asarray(st["Aresiduals"]), np.asarray(g["Aresiduals"]))
    np.testing.assert_array_equal(x[:6], np.asarray(g["x_head"]))
