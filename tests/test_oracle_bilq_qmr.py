"""The CPU oracle's bilq and qmr (oracle/krylov_oracle_biorth.h) against the reference's own known-answer tests
(test/test_bilq.jl, test/test_qmr.jl, real case, same assertions and tolerance), and against the frozen histories of
tests/golden/oracle_bilq_qmr.json (tests/golden/gen_golden_bilq_qmr.py)."""
import json
import os

import numpy as np
import pytest

from oracle import biorth_oracle as O
from parity import golden_module

HERE = os.path.dirname(os.path.abspath(__file__))
TOL = 1.0e-6                                                         # bilq_tol / qmr_tol
G = golden_module("bilq_qmr")
GOLD = json.load(open(os.path.join(HERE, "golden", "oracle_bilq_qmr.json")))
SOLVERS = ("bilq", "qmr")
SOLVED = {"bilq": ("solution xᴸ good enough given atol and rtol", "solution xᶜ good enough given atol and rtol"),
          "qmr": ("solution good enough given atol and rtol",)}


@pytest.mark.parametrize("solver", SOLVERS)
@pytest.mark.parametrize("name", ["symmetric_definite", "symmetric_indefinite", "nonsymmetric_definite",
                                  "nonsymmetric_indefinite", "sparse_laplacian", "polar_poisson", "unsymmetric_breakdown"])
def test_known_answer_problems_are_solved(solver, name):
    A, b, kw = G.cases()[name]
    x, st = getattr(O, solver)(A, b, **kw)
    assert np.linalg.norm(b - A @ x) / np.linalg.norm(b) <= TOL
    assert st["solved"] and st["status"] in SOLVED[solver]


@pytest.mark.parametrize("solver", SOLVERS)
def test_preconditioned_problems_are_solved(solver):
    f = getattr(O, solver)
    A, b, M = O.square_preconditioned()
    x, st = f(A, b, M=M)
    assert np.linalg.norm(M * (b - A @ x)) / np.linalg.norm(M * b) <= TOL and st["solved"]
    x, st = f(A, b, N=M)
    assert np.linalg.norm(b - A @ x) / np.linalg.norm(b) <= TOL and st["solved"]
    A, b, M, N = O.two_preconditioners()
    x, st = f(A, b, M=M, N=N)
    assert np.linalg.norm(M * (b - A @ x)) / np.linalg.norm(M * b) <= TOL and st["solved"]


@pytest.mark.parametrize("solver", SOLVERS)
def test_exit_statuses(solver):
    f = getattr(O, solver)
    A, b = O.zero_rhs()
    x, st = f(A, b)
    assert np.linalg.norm(x) == 0 and st["status"] == "x is a zero-residual solution" and st["niter"] == 0
    A, b, c = O.bc_breakdown()
    x, st = f(A, b, c=c)
    assert st["status"] == "Breakdown bᴴc = 0" and not st["solved"] and st["niter"] == 0
    A, b = O.polar_poisson()
    x, st = f(A, b, callback=lambda it: it >= 3)
    assert st["status"] == "user-requested exit" and st["niter"] == 3
    x, st = f(A, b, timemax=0.0)
    assert st["status"] == "time limit exceeded" and st["niter"] == 1
    x, st = f(A, b, itmax=5)
    assert st["status"] == "maximum number of iterations exceeded" and st["niter"] == 5


def test_bilq_takes_the_bicg_point_when_it_converges_first():
    A, b = O.polar_poisson()
    x, st = O.bilq(A, b)
    assert st["status"] == "solution xᶜ good enough given atol and rtol"
    xl, stl = O.bilq(A, b, transfer_to_bicg=False)
    assert stl["status"] == "solution xᴸ good enough given atol and rtol" and stl["niter"] > st["niter"]
    assert np.linalg.norm(b - A @ xl) / np.linalg.norm(b) <= TOL


@pytest.mark.parametrize("solver", SOLVERS)
def test_warm_start_continues_from_x0(solver):
    A, b = O.nonsymmetric_definite()
    x0 = np.ones(A.shape[0])
    x, st = getattr(O, solver)(A, b, x0=x0)
    assert st["solved"] and np.linalg.norm(b - A @ x) / np.linalg.norm(b - A @ x0) <= TOL


@pytest.mark.parametrize("key", sorted(GOLD))
def test_matches_golden_history(key):
    solver, name = key.split("/")
    A, b, kw = G.cases()[name]
    x, st = getattr(O, solver)(A, b, history=True, **kw)
    g = GOLD[key]
    assert (st["niter"], st["solved"], st["status"]) == (g["niter"], g["solved"], g["status"])
    np.testing.assert_array_equal(np.asarray(st["residuals"]), np.asarray(g["residuals"]))
    np.testing.assert_array_equal(x[:6], np.asarray(g["x_head"]))
