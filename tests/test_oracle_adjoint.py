"""The CPU oracle's bilqr and trilqr (oracle/krylov_oracle_adjoint.h) against the reference's own known-answer tests
(test/test_bilqr.jl, test/test_trilqr.jl, real case, same assertions and tolerance), and against the frozen histories
of tests/golden/oracle_adjoint.json (tests/golden/gen_golden_adjoint.py)."""
import json
import os

import numpy as np
import pytest

from oracle import adjoint_oracle as O
from parity import golden_module

HERE = os.path.dirname(os.path.abspath(__file__))
TOL = 1.0e-6                                                         # bilqr_tol / trilqr_tol
G = golden_module("adjoint")
GOLD = json.load(open(os.path.join(HERE, "golden", "oracle_adjoint.json")))


def _resid(A, b, c, x, y):
    return np.linalg.norm(b - A @ x) / np.linalg.norm(b), np.linalg.norm(c - A.T @ y) / np.linalg.norm(c)


@pytest.mark.parametrize("name", ["square_adjoint", "adjoint_ode", "adjoint_pde"])
def test_bilqr_known_answer_problems_are_solved(name):
    A, b, c = getattr(O, name)()
    x, y, st = O.bilqr(A, b, c)
    rp, rd = _resid(A, b, c, x, y)
    assert rp <= TOL and st["solved_primal"]
    assert rd <= TOL and st["solved_dual"]


@pytest.mark.parametrize("name", ["underdetermined_adjoint", "square_adjoint", "overdetermined_adjoint", "adjoint_ode",
                                  "adjoint_pde"])
def test_trilqr_known_answer_problems_are_solved(name):
    A, b, c = getattr(O, name)()
    x, y, st = O.trilqr(A, b, c)
    rp, rd = _resid(A, b, c, x, y)
    assert rp <= TOL and st["solved_primal"]
    assert rd <= TOL and st["solved_dual"]


def test_trilqr_inconsistent_dual_is_solved_in_the_normal_equations():
    A, b, c = O.rectangular_adjoint()
    x, y, st = O.trilqr(A, b, c)
    s = c - A.T @ y
    assert np.linalg.norm(b - A @ x) / np.linalg.norm(b) <= TOL and st["solved_primal"]
    assert np.linalg.norm(A @ s) / np.linalg.norm(A @ c) <= TOL and st["solved_dual"]


def test_bc_breakdown_status():
    A, b, c = O.bc_breakdown()
    x, y, st = O.bilqr(A, b, c)
    assert st["status"] == "Breakdown bᴴc = 0" and st["niter"] == 0
    assert not st["solved_primal"] and not st["solved_dual"]


@pytest.mark.parametrize("solver", ["bilqr", "trilqr"])
def test_callback_user_requested_exit(solver):
    A, b, c = O.adjoint_pde()
    seen = []
    x, y, st = getattr(O, solver)(A, b, c, atol=0.0, rtol=0.0, callback=lambda it: (seen.append(it) or it >= 5))
    assert st["status"] == "user-requested exit" and st["niter"] == 5 and seen == [1, 2, 3, 4, 5]


@pytest.mark.parametrize("solver", ["bilqr", "trilqr"])
def test_warm_start_finishes_in_fewer_iterations(solver):
    A, b, c = O.adjoint_pde(20, 20)
    tol = dict(atol=1e-7 * min(np.linalg.norm(b), np.linalg.norm(c)), rtol=0.0)   # the same bar for both starts
    x, y, st = getattr(O, solver)(A, b, c, **tol)
    x1, y1, st1 = getattr(O, solver)(A, b, c, x0=x + 1e-6, y0=y - 1e-6, **tol)
    assert st1["solved_primal"] and st1["solved_dual"] and st1["niter"] < st["niter"]
    rp, rd = _resid(A, b, c, x1, y1)
    assert rp <= 10 * TOL and rd <= 10 * TOL


def test_split_cases_converge_one_half_first():
    for name, (want_p, want_d) in (("bilqr/primal_first", (True, False)), ("bilqr/dual_first", (False, True)),
                                   ("trilqr/primal_first", (True, False)), ("trilqr/dual_first", (False, True))):
        g = GOLD[name]
        lp, ld = len(g["residuals_primal"]), len(g["residuals_dual"])
        assert (lp < ld) == want_p and (ld < lp) == want_d, (name, lp, ld)
        assert abs(lp - ld) >= 20, (name, lp, ld)


@pytest.mark.parametrize("name", sorted(G.cases()))
def test_golden_histories_reproduce(name):
    solver, A, b, c, kw = G.cases()[name]
    x, y, st = G.run(solver, A, b, c, **kw)
    g = GOLD[name]
    assert (st["niter"], st["solved_primal"], st["solved_dual"], st["status"]) == \
        (g["niter"], g["solved_primal"], g["solved_dual"], g["status"])
    for key in ("residuals_primal", "residuals_dual"):
        assert np.array_equal(np.asarray(st[key]), np.asarray(g[key])), key
    assert np.array_equal(x[:6], np.asarray(g["x_head"])) and np.array_equal(y[:6], np.asarray(g["y_head"]))
